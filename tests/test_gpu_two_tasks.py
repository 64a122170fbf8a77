"""Two tasks calling one engine at once, bit for bit against a serial twin.

The ABI promises two concurrent callers (include/b200rwkv.h, INTEGRATION.md §2 and §4): one task makes the infer and state
calls, another makes the softmax and sampling calls, and a dropped snapshot handle calls b200rwkv_state_free on whatever
thread drops it.  Every scenario here builds two engines from the same image with the same options: `live` is driven by
threads, `twin` gets the same calls serially on the main thread.  The threads only ever overlap on disjoint slots, as the
contract allows, so every output of `live` must be the twin's bits.  Each scenario also asserts that calls really overlapped
(a sampling-group call lying entirely inside an infer-group call), so a test that passes with the two tasks serialised is
not possible.

What the engine relies on, per member that run-time calls touch (engine.cu, struct b200rwkv_engine):

Infer group -- infer / infer_ex / infer_snapshots, state_load / back / read / write / free, snapshot_back / load,
cache_stats, launch_count, bind / load / unload_adapter, update_weights, head_format, keep_hidden*, score_top, last_*;
all under `mu`:
  - `stream`, the step graphs `graphs` (captured in cudaStreamCaptureModeThreadLocal, so the sampling thread may allocate
    and free while a capture is open), `launch_total`, `last_T`, `last_sh`;
  - the step buffers (`d_meta` / `h_meta` / `meta_ev`, activations, `gemm_ws`, `d_logits`, `d_hidden`, the snapshot step
    block `snap_dev` / `snap_host` / `snap_logits`);
  - slot states `att_shift` / `ffn_shift` / `wkv_state`, the host staging row `d_api`;
  - snapshots `snaps` / `next_snap` (a cudaMalloc per snapshot, a cudaFree in state_free -- from any thread, under `mu`);
  - grown buffers `sc_dev` / `sc_host` (SCORE), `hid_all`, `d_hidden_all`, `pool_dev` / `pool_host`;
  - settings and plans: `hid_layers`, `pool_layers`, `top_n`, `qhead`, adapter places and bindings, the weights.
Sampling group -- softmax, sample_topk, sample_probs; all under `sm_mu`, on `sm_stream`:
  - `sm_in` / `sm_out` (softmax), `sp_dev` (sample_probs), `tk_dev` / pinned `tk_host` (the staging blob), all grown by
    a cudaFree followed by a cudaMalloc (Buf::grow); `tk_cand_x` / `tk_cand_id` / `tk_stats` / `tk_out_id` / `tk_out_p`.
Shared between the groups:
  - `d_keep` (one kept logits row per slot): written on `stream` by the steps of the slots they contain and by
    state_write, read on `sm_stream` by the sampler for the slots it lists.  Disjoint slots make the rows disjoint;
  - `keep_valid`, under `keep_mu`: written by infer (NONE entries, steps with rows), state_load, state_write and the decode
    routes; read by the sampler's slot check, state_read and SCORE;
  - `step_done`: recorded on `stream` after every step and by state_write; `sm_stream` waits on it before it reads kept rows;
  - immutable after creation, read without a lock: V, S, C, L, N, dev, rank, world;
  - the error text `g_err` is thread_local: each task reads its own last failure.

What each scenario catches:
  - a sampler entry that takes `mu`: sampling can no longer run inside an infer call, and the overlap assertions of
    scenarios 1-3 fail;
  - a buffer shared between the groups: the bit comparisons of scenarios 1-3 fail;
  - a capture mode that forbids other threads' allocations: scenario 2's infer call fails with ERR_CUDA, or its
    launch_count differs from the twin's;
  - a global (not thread_local) `g_err`: scenario 4 fails (and tests/test_two_tasks_cpu.py without a GPU).

A sampler prepares its arguments before a round starts and waits (at most a bounded time) for an infer call to be in flight
before it issues its calls, so the overlap does not hinge on thread scheduling.  A sampler call blocked behind the infer
call cannot finish inside it, so the overlap assertions still catch a serialising lock.

Rules: every loop is bounded, nothing retries a failed call, threads are daemons joined with a timeout, and on a timeout
the test fails with the last call each thread entered."""
import dataclasses
import hashlib
import threading
import time
import traceback

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

TIMEOUT = 300.0          # seconds for all threads of one scenario
MAX_REPEATS = 64         # identical sampler repeats per round while the round's infer call is in flight
S = 16
GROUPS = (list(range(0, 8)), list(range(8, 16)))
ROUNDS = 24


def preset(name):
    """small6 with the production vocabulary (sampler rows and kept rows of 256 KiB), small7 as it is."""
    return dataclasses.replace(synth.PRESETS["small6"], V=65536) if name == "small6" else synth.PRESETS[name]


_IMAGES = {}


def image(name, seed=0):
    key = (name, seed)
    if key not in _IMAGES:
        _IMAGES[key] = synth.make_st(preset(name) if name in ("small6", "small7") else name, seed)
    return _IMAGES[key]


# ---------------------------------------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------------------------------------
class Trace:
    """The call intervals of one run (perf_counter_ns around each call; every entry ends in a stream synchronise, so an
    interval is the call's true extent) and the progress list of its threads.  With record=False it only calls."""

    def __init__(self, record=True):
        self.record = record
        self.progress = []            # (thread name, call) in the order the calls were entered
        self.spans = {}               # group -> [(t0, t1, call)]
        self.lock = threading.Lock()
        # set while a call of the group is in flight: a sampler may wait (bounded) for one before it issues its calls
        self.busy = {"infer": threading.Event(), "capture": threading.Event()}

    def call(self, group, what, fn, *args, **kw):
        if not self.record:
            return fn(*args, **kw)
        with self.lock:
            self.progress.append((threading.current_thread().name, what))
        busy = self.busy.get(group)
        t0 = time.perf_counter_ns()
        if busy:
            busy.set()
        try:
            return fn(*args, **kw)
        finally:
            if busy:
                busy.clear()
            t1 = time.perf_counter_ns()
            with self.lock:
                self.spans.setdefault(group, []).append((t0, t1, what))

    def inside(self, inner, outer):
        """(calls of group `inner`, how many of them lie entirely inside a call of group `outer`)."""
        outs = sorted((a, b) for a, b, _ in self.spans.get(outer, []))
        ins = self.spans.get(inner, [])
        starts = np.array([a for a, _ in outs], np.int64)
        n = 0
        for a, b, _ in ins:
            # the latest call of `outer` that started at or before a: one thread makes a group's calls, so they never
            # overlap and that call is the only candidate
            k = int(np.searchsorted(starts, a, side="right")) - 1
            if k >= 0 and outs[k][1] >= b:
                n += 1
        return len(ins), n


def run_threads(trace, bodies, barriers=()):
    """Runs {name: body} on daemon threads and joins them within TIMEOUT.  A thread that raises aborts the barriers, so the
    others stop too; the first real failure is reported.  A thread still alive at the deadline fails the test with the last
    call each thread entered (the threads are daemons: they do not keep the process alive)."""
    errors = []

    def wrap(body):
        def run():
            try:
                body()
            except BaseException as ex:                      # noqa: BLE001 -- reported by the main thread
                errors.append((threading.current_thread().name, ex, traceback.format_exc()))
                for b in barriers:
                    b.abort()
        return run

    threads = [threading.Thread(target=wrap(b), name=n, daemon=True) for n, b in bodies.items()]
    for t in threads:
        t.start()
    deadline = time.monotonic() + TIMEOUT
    for t in threads:
        t.join(max(0.0, deadline - time.monotonic()))
    alive = [t.name for t in threads if t.is_alive()]
    if alive:
        last = {}
        with trace.lock:
            for name, what in trace.progress:
                last[name] = what
        pytest.fail(f"threads {alive} still running after {TIMEOUT:.0f} s; last call entered per thread: {last}")
    if errors:
        real = [e for e in errors if not isinstance(e[1], threading.BrokenBarrierError)] or errors
        name, _, tb = real[0]
        pytest.fail(f"thread {name} raised:\n{tb}")


def assert_same(live, twin, where):
    """Bit identity of two results: arrays on their uint views, tuples / lists / dicts member by member, the rest by ==."""
    if isinstance(twin, np.ndarray):
        assert isinstance(live, np.ndarray) and live.shape == twin.shape and live.dtype == twin.dtype, where
        if live.dtype.itemsize in (2, 4, 8):
            u = {2: np.uint16, 4: np.uint32, 8: np.uint64}[live.dtype.itemsize]
            bad = int(np.count_nonzero(live.view(u) != twin.view(u)))
        else:
            bad = int(np.count_nonzero(live != twin))
        assert bad == 0, f"{where}: {bad} of {twin.size} elements differ from the serial twin"
    elif isinstance(twin, (tuple, list)):
        assert isinstance(live, (tuple, list)) and len(live) == len(twin), where
        for i, (a, b) in enumerate(zip(live, twin)):
            assert_same(a, b, f"{where}[{i}]")
    elif isinstance(twin, dict):
        assert isinstance(live, dict) and live.keys() == twin.keys(), f"{where}: {sorted(live)} vs {sorted(twin)}"
        for k in twin:
            assert_same(live[k], twin[k], f"{where}[{k!r}]")
    else:
        assert live == twin, f"{where}: {live!r} vs {twin!r}"


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def code_of(fn, *args, **kw):
    """The result of fn, or ('error', code) if it raised B200Error."""
    try:
        return fn(*args, **kw)
    except capi.B200Error as ex:
        return ("error", ex.code)


def sample_requests(V, seed, slots, pen=24, bias=8, with_allow=False):
    """Penalty and bias lists (the reference's HashMaps) and an optional allow mask for `slots`, from `seed`."""
    rng = np.random.default_rng(seed)
    pens = [{int(t): float(v) for t, v in zip(rng.choice(V, pen, replace=False), rng.random(pen) * 2)} for _ in slots]
    biases = [{int(t): float(v) for t, v in zip(rng.choice(V, bias, replace=False), rng.random(bias) - 0.5)} for _ in slots]
    allow = (rng.random((len(slots), V)) > 0.1) if with_allow else None
    return pens, biases, allow


def end_state(m):
    """state_back of every slot, launch_count, and the snapshot cache's count and bytes."""
    cs = m.state.cache_stats()
    return {"states": [m.state.back(s) for s in range(m.max_batch)], "launches": m.launch_count(),
            "snapshots": cs["snapshots"], "bytes_used": cs["bytes_used"]}


# ---------------------------------------------------------------------------------------------------------------------
# scenario 1: pipelined generation, the run.rs shape
# ---------------------------------------------------------------------------------------------------------------------
class Pipeline:
    """Rounds of the run.rs shape on one engine.  In round r the infer task makes one call for group r % 2 while two sampler
    threads work on the other group's kept rows (sampler k on its half).  A slot's next token is ids[row, (r + slot) % 7]
    of its sample_topk result, so the token sequence depends on every sampling result.  Round kinds, by r % 6:
      2, 3: rich -- one prefill of 40-300 tokens (LAST), one FULL entry, one SCORE entry, score_top lists and snapshots
            (infer_snapshots);
      4, 5: slot 3 of the group feeds a prefill as a NONE chunk; the group's next round finishes it with LAST.  In the
            round between, sampling that slot answers ERR_STATE;
      else: decode, one token per slot, LAST.
    Snapshots are read back by the infer task when they are taken and freed by sampler 0 two rounds later."""

    def __init__(self, m, trace):
        self.m, self.t = m, trace
        self.V = m.info["num_vocab"]
        self.tok = {s: 1 + 37 * s for s in range(S)}
        self.rest = {}                 # slot -> tokens still to feed after a NONE chunk
        self.snaps = []                # (round taken, TensorGpu): appended by the infer task, freed by sampler 0
        self.snap_lock = threading.Lock()
        self.res = {}
        self.r = -1
        self.infer_done = threading.Event()

    def start(self):
        """Both groups get a kept row: a short prefill per slot, before any thread runs."""
        m = self.m
        for s in range(S):
            m.state.load(m.state.init(), s)
        for g in GROUPS:
            toks = [[self.tok[s], 2 * s + 3, 5 * s + 7] for s in g]
            self.res[("start", g[0])] = m.infer_raw(g, [3] * len(g), sum(toks, []), [capi.OPTION_LAST] * len(g))

    def next_round(self):
        """Between rounds (the barrier's action): the round number and each sampler's requests, made before the round
        starts so that the samplers' first calls go out while the infer call is in flight."""
        self.r += 1
        self.infer_done.clear()
        r, V = self.r, self.V
        h = GROUPS[1 - r % 2]
        self.req = []
        for k in (0, 1):
            mine = h[4 * k:4 * k + 4]
            slots = [s for s in mine if s not in self.rest]
            pens, biases, allow = sample_requests(V, 100 * r + k, slots, with_allow=(r % 3 == 0))
            sm_rows = np.random.default_rng(9000 + 10 * r + k).standard_normal((1 + (r + k) % 3, V)).astype(np.float32)
            # slots with a NONE chunk pending have no kept row
            self.req.append(([s for s in mine if s in self.rest], slots, pens, biases, allow, 16 + 8 * (r % 5), sm_rows))

    # -- the infer task --
    def infer_round(self):
        r, m, t, V = self.r, self.m, self.t, self.V
        g = GROUPS[r % 2]
        rng = np.random.default_rng(7000 + r)
        kind = r % 6
        slots, ntok, toks, opts = [], [], [], []
        for s in g:
            if s in self.rest:
                seq, opt = self.rest.pop(s), capi.OPTION_LAST
            elif kind in (2, 3) and s == g[0]:
                seq, opt = [self.tok[s]] + rng.integers(1, V, int(rng.integers(40, 300))).tolist(), capi.OPTION_LAST
            elif kind in (2, 3) and s == g[1]:
                seq, opt = [self.tok[s]] + rng.integers(1, V, 3).tolist(), capi.OPTION_FULL
            elif kind in (2, 3) and s == g[2]:
                seq, opt = [self.tok[s]] + rng.integers(1, V, 5).tolist(), capi.OPTION_SCORE
            elif kind in (4, 5) and s == g[3]:
                full = [self.tok[s]] + rng.integers(1, V, int(rng.integers(40, 200))).tolist()
                cut = int(rng.integers(8, len(full) - 1))
                seq, opt = full[:cut], capi.OPTION_NONE
                self.rest[s] = full[cut:]
            else:
                seq, opt = [self.tok[s]], capi.OPTION_LAST
            slots.append(s)
            ntok.append(len(seq))
            toks += seq
            opts.append(opt)
        if kind in (2, 3):
            at = [(0, 17), (0, ntok[0]), (1, 2), (2, ntok[2]), (4, 1)]
            t.call("infer", f"score_top r{r}", m.score_top, 8)
            rows, scores, snaps = t.call("infer", f"infer_snapshots r{r}", m.infer_snapshots, slots, ntok, toks, opts, at)
            tops = t.call("infer", f"last_score_top r{r}", m.last_score_top)
            t.call("infer", f"score_top r{r}", m.score_top, 0)
            self.res[(r, "rows")] = [x.copy() for x in rows]
            self.res[(r, "scores")] = [None if x is None else (x[0].copy(), x[1].copy()) for x in scores]
            self.res[(r, "tops")] = tops
            for j, sn in enumerate(snaps):
                self.res[(r, "snap", j)] = t.call("infer", f"snapshot_back r{r}", m.state.snapshot_back, sn, True)
                with self.snap_lock:
                    self.snaps.append((r, sn))
        else:
            rows = t.call("infer", f"infer r{r}", m.infer_raw, slots, ntok, toks, opts)
            self.res[(r, "rows")] = [x.copy() for x in rows]
        self.infer_done.set()

    # -- the sampler tasks --
    def sampler_round(self, k, repeat):
        r, m, t = self.r, self.m, self.t
        without, slots, pens, biases, allow, top_k, sm_rows = self.req[k]
        calls = [
            ("topk", lambda: t.call("sample", f"sample_topk r{r}", m.sample_topk, slots, pens, biases, allow, top_k)),
            ("probs", lambda: t.call("sample", f"sample_probs r{r}", m.sample_probs, slots, pens, biases, allow)),
            ("softmax", lambda: t.call("sample", f"softmax r{r}", m.softmax, list(sm_rows))),
        ]
        if repeat and not self.infer_done.is_set():
            t.busy["infer"].wait(0.5)
        first = {}
        for name, fn in calls:
            first[name] = fn()
            self.res[(r, k, name)] = first[name]
        for s in without:
            self.res[(r, k, "no_row", s)] = t.call("sample", f"sample_topk r{r} no row", code_of, m.sample_topk, [s], top_k=4)
        ids = first["topk"][0]
        for row, s in enumerate(slots):
            self.tok[s] = int(ids[row, (r + s) % 7])
        if k == 0:                     # TensorGpu drop: state_free from the sampling thread (an infer-group call)
            with self.snap_lock:
                old = [sn for rr, sn in self.snaps if rr <= r - 2]
                self.snaps = [x for x in self.snaps if x[0] > r - 2]
            for sn in old:
                t.call("free", f"state_free r{r}", sn.free)
        reps = 0
        while repeat and not self.infer_done.is_set() and reps < MAX_REPEATS:
            for name, fn in calls:
                assert_same(fn(), first[name], f"round {r} sampler {k} {name} repeat {reps}")
            reps += 1


def drive_pipeline(m, trace, threaded):
    p = Pipeline(m, trace)
    p.start()
    if not threaded:
        for _ in range(ROUNDS):
            p.next_round()
            p.infer_round()
            for k in (0, 1):
                p.sampler_round(k, repeat=False)
    else:
        bar = threading.Barrier(3, action=p.next_round, timeout=TIMEOUT)

        def infer_body():
            for _ in range(ROUNDS):
                bar.wait()
                p.infer_round()

        def sampler_body(k):
            def body():
                for _ in range(ROUNDS):
                    bar.wait()
                    p.sampler_round(k, repeat=True)
            return body

        run_threads(trace, {"infer": infer_body, "sampler0": sampler_body(0), "sampler1": sampler_body(1)}, [bar])
    p.res["end"] = end_state(m)
    for _, sn in p.snaps:
        sn.free()
    return p.res


@pytest.mark.parametrize("name,chunk,precision", [("small6", 32, 0), ("small6", 128, 0), ("small6", 32, 1),
                                                  ("small7", 32, 0), ("small7", 128, 0)])
def test_pipelined_generation(name, chunk, precision):
    st = image(name)
    live = runtime.Model(st, max_batch=S, token_chunk_size=chunk, precision=precision)
    twin = runtime.Model(st, max_batch=S, token_chunk_size=chunk, precision=precision)
    try:
        trace = Trace()
        got = drive_pipeline(live, trace, threaded=True)
        want = drive_pipeline(twin, Trace(record=False), threaded=False)
    finally:
        live.close()
        twin.close()
    n, inside = trace.inside("sample", "infer")
    print(f"[two-tasks] pipelined {name} V{preset(name).V} chunk{chunk} p{precision}: {n} sampler calls, {inside} inside infer")
    assert_same(got, want, "pipelined")
    # the ERR_STATE answers between a NONE chunk and its LAST: present, and the same on both engines
    no_rows = [v for key, v in want.items() if isinstance(key, tuple) and "no_row" in key]
    assert no_rows and all(v == ("error", capi.ERR_STATE) for v in no_rows)
    assert inside >= 1, "no sampling call ran inside an infer call: the two tasks were serialised"


# ---------------------------------------------------------------------------------------------------------------------
# scenario 2: first captures while the sampler grows its buffers
# ---------------------------------------------------------------------------------------------------------------------
def capture_program(m, V):
    """The infer task's calls on slots 0-15 of a fresh engine (max_batch 32, token_chunk_size 128).  Each call is one step
    whose graph key -- (token tiles, head-row tiles, snapshot-row tiles) as run_step keys its graphs -- is new, so every
    call captures a graph.  Returns [(key, name, fn(trace) -> result)]."""
    rng = np.random.default_rng(11)

    def tk(n):
        return rng.integers(1, V, n).tolist()

    def infer(slots, ntok, opts):
        toks = tk(sum(ntok))
        return lambda t: [x.copy() for x in t.call("capture", f"infer {ntok}", m.infer_raw, slots, ntok, toks, opts)]

    def score(slot, n):
        toks = tk(n)

        def run(t):
            m.score_top(8)
            try:
                _, scores = t.call("capture", f"score {n}", m.infer_ex, [slot], [n], toks, [capi.OPTION_SCORE])
                return [scores[0][0].copy(), scores[0][1].copy(), m.last_score_top()]
            finally:
                m.score_top(0)
        return run

    def hidden(slot, n, layers):
        toks = tk(n)

        def run(t):
            m.keep_hidden(layers=layers)
            try:
                rows = t.call("capture", f"hidden {n}", m.infer_raw, [slot], [n], toks, [capi.OPTION_LAST])
                return [rows[0].copy()] + [m.last_hidden(max_rows=n, layer=l) for l in layers]
            finally:
                m.keep_hidden(layers=[])
        return run

    def pooled(slots, n, layers):
        toks = tk(n * len(slots))

        def run(t):
            m.keep_hidden_pooled(layers, "mean")
            try:
                rows = t.call("capture", f"pooled {n}", m.infer_raw, slots, [n] * len(slots), toks,
                              [capi.OPTION_LAST] * len(slots))
                return [x.copy() for x in rows] + [m.last_hidden_pooled(l, max_rows=len(slots)) for l in layers]
            finally:
                m.keep_hidden_pooled([])
        return run

    def snapshots(slot, n, opt, at):
        toks = tk(n)

        def run(t):
            rows, _, snaps = t.call("capture", f"snapshots {n}x{len(at)}", m.infer_snapshots, [slot], [n], toks, [opt],
                                    [(0, p) for p in at])
            out = [x.copy() for x in rows]
            for sn in snaps:                # contents by digest: a 70-snapshot call holds 0.9 GB of records
                out.append(digest(*m.state.snapshot_back(sn, with_logits=True)))
                sn.free()
            return out
        return run

    LAST, FULL, NONE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE
    return [
        ((1, 1, None), "1 token, LAST", infer([0], [1], [LAST])),
        ((1, 0, None), "9 tokens, NONE", infer([1], [9], [NONE])),
        ((2, 2, None), "2 x 12 tokens, FULL", infer([2, 3], [12, 12], [FULL, FULL])),
        ((4, 1, None), "50 tokens, LAST", infer([4], [50], [LAST])),
        ((8, 0, None), "2 x 50 tokens, NONE", infer([5, 6], [50, 50], [NONE, NONE])),
        ((4, 4, None), "SCORE 40 tokens, top 8", score(7, 40)),
        ((2, 1, None), "20 tokens, LAST, layers 2 and 11 recorded", hidden(8, 20, [2, 11])),
        ((8, 1, None), "2 x 64 tokens, LAST, layers 5 and 23 pooled", pooled([9, 10], 64, [5, 23])),
        ((8, 8, None), "100 tokens, FULL", infer([11], [100], [FULL])),
        ((1, 1, 0), "snapshots: 10 tokens FULL, 2 snapshots with rows", snapshots(12, 10, FULL, [3, 10])),
        ((2, 0, 1), "snapshots: 20 tokens NONE, 5", snapshots(13, 20, NONE, [1, 2, 3, 4, 5])),
        ((4, 0, 2), "snapshots: 40 tokens NONE, 20", snapshots(14, 40, NONE, list(range(1, 41, 2)))),
        ((8, 0, 4), "snapshots: 70 tokens NONE, 40", snapshots(15, 70, NONE, list(range(1, 41)))),
        ((8, 0, 8), "snapshots: 128 tokens NONE, 70", snapshots(0, 128, NONE, list(range(30, 100)))),
    ]


def grow_program(m, V):
    """The sampler task's calls on slots 16-31: each grows one of its buffers with a cudaFree + cudaMalloc (the first
    sample_probs and sample_topk calls make the first blocks).  softmax with 1 .. 64 rows; sample_probs with 1, 5, 16 rows
    (past sp_dev's first 1 MiB); sample_topk with penalty and bias lists of 5, then 2 x 40000, then 16 x 20000 entries (past
    the staging blob's first 1 MiB, regrowing pinned tk_host and tk_dev).  Results are kept as digests."""
    x = np.random.default_rng(12).standard_normal((64, V)).astype(np.float32)
    slots = list(range(16, 32))

    def softmax(n):
        return lambda t: digest(*t.call("sample", f"softmax {n}", m.softmax, list(x[:n])))

    def probs(n):
        return lambda t: digest(t.call("sample", f"sample_probs {n}", m.sample_probs, slots[:n]))

    def topk(n, entries):
        pens, biases, _ = sample_requests(V, 13 + n, slots[:n], pen=entries, bias=entries)
        return lambda t: list(t.call("sample", f"sample_topk {n}x{entries}", m.sample_topk, slots[:n], pens, biases, None, 64))

    prog = [("topk 1x5", topk(1, 5)), ("probs 1", probs(1))]
    prog += [(f"softmax {n}", softmax(n)) for n in range(1, 22)]
    prog += [("topk 2x40000", topk(2, 40000)), ("probs 5", probs(5))]
    prog += [(f"softmax {n}", softmax(n)) for n in range(22, 43)]
    prog += [("topk 16x20000", topk(16, 20000)), ("probs 16", probs(16))]
    prog += [(f"softmax {n}", softmax(n)) for n in range(43, 65)]
    return prog


def capture_engine(st):
    m = runtime.Model(st, max_batch=32, token_chunk_size=128)
    V, rng = m.info["num_vocab"], np.random.default_rng(10)
    for s in range(16):
        m.state.load(m.state.init(), s)
    for s in range(16, 32):            # kept rows by copies only: snapshot_load + state_write capture no graph
        init = m.state.init()
        sn = m.state.snapshot_load(init + rng.standard_normal(init.shape).astype(np.float32) * 0.1,
                                   rng.standard_normal(V).astype(np.float32) * 3)
        m.state.write(sn, s)
        sn.free()
    return m


def test_first_captures_while_the_sampler_grows_its_buffers():
    st = synth.make_st("v6-1b6", 0)
    live, twin = capture_engine(st), capture_engine(st)
    del st
    try:
        V = live.info["num_vocab"]
        assert live.launch_count() == twin.launch_count() == 0
        cap_l, grow_l = capture_program(live, V), grow_program(live, V)
        cap_t, grow_t = capture_program(twin, V), grow_program(twin, V)
        keys = [k for k, _, _ in cap_l]
        assert len(set(keys)) == len(keys), "every infer call of this scenario must capture a new step graph"
        trace, got, want = Trace(), {}, {}
        bar = threading.Barrier(2, timeout=TIMEOUT)
        done = threading.Event()

        def infer_body():
            bar.wait()
            for _, name, fn in cap_l:
                got[name] = fn(trace)
            done.set()

        def sampler_body():
            bar.wait()
            for name, fn in grow_l:
                if not done.is_set():          # issue the call while a capturing infer call is in flight
                    trace.busy["capture"].wait(2.0)
                got[name] = fn(trace)

        run_threads(trace, {"infer": infer_body, "sampler": sampler_body}, [bar])
        serial = Trace(record=False)
        for _, name, fn in cap_t:
            want[name] = fn(serial)
        for name, fn in grow_t:
            want[name] = fn(serial)
        got["end"], want["end"] = end_state(live), end_state(twin)
    finally:
        live.close()
        twin.close()
    n, inside = trace.inside("sample", "capture")
    print(f"[two-tasks] first captures v6-1b6 V{V}: {n} growing sampler calls, {inside} inside a capturing infer call")
    assert_same(got, want, "first captures")        # launch_count included: no capture was lost or redone
    assert inside >= 1, "no growing sampler call ran inside a capturing infer call"


# ---------------------------------------------------------------------------------------------------------------------
# scenario 3: infer-group calls that rewrite engine state while sampling reads it
# ---------------------------------------------------------------------------------------------------------------------
KINDS3 = ("att.key", "att.value", "ffn.key")


def adapter_image():
    """An adapter file on the places' kinds, without the head pair make_lora_st adds (the places do not plan the head, so
    head_format stays available)."""
    w = O.parse_st(synth.make_lora_st(preset("small6"), rank=8, seed=41, targets=KINDS3))
    return synth.pack_st({k: np.ascontiguousarray(v) for k, v in w.items() if not k.startswith("head.")})


def rewrite_program(m, adapter, update):
    """The infer task's calls on group A (slots 0-7) and engine-wide ones.  Every op ends with a decode of group A (LAST,
    one token per slot), whose rows are recorded."""
    V, A = m.info["num_vocab"], GROUPS[0]
    rng = np.random.default_rng(21)
    box = {}

    def decode(t, tag):
        toks = rng.integers(1, V, len(A)).tolist()
        return [x.copy() for x in t.call("infer", f"decode {tag}", m.infer_raw, A, [1] * len(A), toks, [capi.OPTION_LAST] * len(A))]

    def read_write(t):
        box["a"] = t.call("infer", "state_read", m.state.read, 0)
        out = list(t.call("infer", "snapshot_back", m.state.snapshot_back, box["a"], True))
        t.call("infer", "state_write", m.state.write, box["a"], 1)
        return out + decode(t, "read_write")

    def loads(t):
        r2, init = np.random.default_rng(22), m.state.init()
        t.call("infer", "state_load", m.state.load, init, 2)
        box["b"] = t.call("infer", "snapshot_load", m.state.snapshot_load,
                          init + r2.standard_normal(init.shape).astype(np.float32) * 0.1, r2.standard_normal(V).astype(np.float32))
        t.call("infer", "state_write", m.state.write, box["b"], 3)
        cs = t.call("infer", "cache_stats", m.state.cache_stats)
        return [cs["snapshots"], cs["bytes_used"]] + decode(t, "loads")

    def load_bind(t):
        t.call("infer", "load_adapter", m.load_adapter, 1, adapter, 0.75)
        t.call("infer", "bind_adapter", m.bind_adapter, A[:4], [1] * 4)
        return decode(t, "bound")

    def head(kind):
        def run(t):
            t.call("infer", f"head_format {kind}", m.head_format, kind)
            return decode(t, f"head {kind}")
        return run

    def unload(t):
        t.call("infer", "bind_adapter", m.bind_adapter, A[:4], [0] * 4)
        t.call("infer", "unload_adapter", m.unload_adapter, 1)
        return decode(t, "unloaded")

    def update_weights(t):
        t.call("infer", "update_weights", m.update_weights, update)
        return decode(t, "updated")

    def frees(t):
        for k in ("a", "b"):
            t.call("infer", "state_free", box.pop(k).free)
        cs = t.call("infer", "cache_stats", m.state.cache_stats)
        return [cs["snapshots"], cs["bytes_used"]] + decode(t, "freed")

    return [("decode", lambda t: decode(t, "first")), ("state_read / state_write", read_write),
            ("state_load / snapshot_load / cache_stats", loads), ("load_adapter / bind_adapter", load_bind),
            ("head_format Int8", head("Int8")), ("head_format None", head("None")),
            ("bind 0 / unload_adapter", unload), ("update_weights", update_weights), ("state_free", frees)]


def sample_group_b(m, k):
    """Sampler k's fixed requests on its half of group B (slots 8-15), whose kept rows nothing in scenario 3 rewrites."""
    V, slots = m.info["num_vocab"], GROUPS[1][4 * k:4 * k + 4]
    pens, biases, allow = sample_requests(V, 31 + k, slots, with_allow=True)
    return [("topk", lambda t: t.call("sample", "sample_topk B", m.sample_topk, slots, pens, biases, allow, 32)),
            ("probs", lambda t: t.call("sample", "sample_probs B", m.sample_probs, slots, pens, biases, None))]


def rewrite_engine(st):
    m = runtime.Model(st, max_batch=S, token_chunk_size=32, adapter_places=2, adapter_targets=KINDS3)
    for s in range(S):
        m.state.load(m.state.init(), s)
    toks = [t for s in range(S) for t in (s + 1, 3 * s + 2, 7 * s + 5)]
    m.infer_raw(list(range(S)), [3] * S, toks, [capi.OPTION_LAST] * S, keep_on_device=True)
    return m


def test_state_rewrites_while_sampling():
    st = image("small6")
    adapter, update = adapter_image(), image("small6", 1)
    live, twin = rewrite_engine(st), rewrite_engine(st)
    try:
        ops_l, ops_t = rewrite_program(live, adapter, update), rewrite_program(twin, adapter, update)
        smp_l = [sample_group_b(live, k) for k in (0, 1)]
        smp_t = [sample_group_b(twin, k) for k in (0, 1)]
        serial = Trace(record=False)
        want_b = {(k, name): fn(serial) for k in (0, 1) for name, fn in smp_t[k]}
        want = {name: fn(serial) for name, fn in ops_t}
        for k in (0, 1):                 # group B's results did not change across all of this
            for name, fn in smp_t[k]:
                assert_same(fn(serial), want_b[(k, name)], f"twin group B {name} after the rewrites")
        want["end"] = end_state(twin)

        trace, got = Trace(), {}
        done = threading.Event()
        bar = threading.Barrier(3, action=done.clear, timeout=TIMEOUT)

        def infer_body():
            for name, fn in ops_l:
                bar.wait()
                got[name] = fn(trace)
                done.set()

        def sampler_body(k):
            def body():
                for i in range(len(ops_l)):
                    bar.wait()
                    reps = 0
                    while reps == 0 or (not done.is_set() and reps < MAX_REPEATS):
                        for name, fn in smp_l[k]:
                            assert_same(fn(trace), want_b[(k, name)], f"group B sampler {k} {name} during op {i} repeat {reps}")
                        reps += 1
            return body

        run_threads(trace, {"infer": infer_body, "sampler0": sampler_body(0), "sampler1": sampler_body(1)}, [bar])
        got["end"] = end_state(live)
    finally:
        live.close()
        twin.close()
    n, inside = trace.inside("sample", "infer")
    print(f"[two-tasks] state rewrites small6 V65536: {n} sampler calls, {inside} inside infer-group calls")
    assert_same(got, want, "state rewrites")
    assert inside >= 1, "no sampling call ran inside an infer-group call: the two tasks were serialised"


# ---------------------------------------------------------------------------------------------------------------------
# scenario 4: error text per thread
# ---------------------------------------------------------------------------------------------------------------------
def last_error():
    msg = capi.lib().b200rwkv_last_error(None)
    return msg.decode("utf-8", "replace") if msg else ""


def raw_infer(m, slots, toks):
    """b200rwkv_infer with LAST entries of one token each and rows to the host: (status, rows)."""
    V = m.info["num_vocab"]
    a = [np.asarray(x, dt) for x, dt in ((slots, np.int32), ([1] * len(slots), np.int32), (toks, np.uint32),
                                          ([capi.OPTION_LAST] * len(slots), np.int32))]
    out, rows = np.zeros((len(slots), V), np.float32), np.zeros(len(slots), np.int32)
    code = capi.lib().b200rwkv_infer(m._h, len(slots), *(capi.ptr(x) for x in a), capi.ptr(out), out.size, capi.ptr(rows))
    return code, out


def raw_topk(m, slots, top_k):
    """b200rwkv_sample_topk without adjustment lists: (status, ids, probs)."""
    a = np.asarray(slots, np.int32)
    ids, p = np.zeros((len(slots), max(top_k, 1)), np.uint32), np.zeros((len(slots), max(top_k, 1)), np.float32)
    code = capi.lib().b200rwkv_sample_topk(m._h, len(slots), capi.ptr(a), None, None, None, None, None, None, None, top_k,
                                           capi.ptr(ids), capi.ptr(p))
    return code, ids, p


def error_engine(st):
    m = runtime.Model(st, max_batch=S, token_chunk_size=32)
    for s in range(S):
        m.state.load(m.state.init(), s)
    m.infer_raw(list(range(8)), [2] * 8, [t for s in range(8) for t in (s + 1, s + 9)], [capi.OPTION_LAST] * 8,
                keep_on_device=True)
    return m                           # slots 8-15: no kept row


def test_error_text_per_thread():
    st = image("small7")
    live, twin = error_engine(st), error_engine(st)
    try:
        V = live.info["num_vocab"]
        # (sampler request, its expected status and a fragment of its message); slot 15 has no kept row
        cases = [(([15], 4), capi.ERR_STATE, "slot 15 has produced no logits row yet"),
                 (([0], 0), capi.ERR_INVALID, "top_k must be in [1, 128]")]
        bad_tok = V + 5
        trace, got = Trace(), {}
        bar = threading.Barrier(2, timeout=TIMEOUT)

        def infer_body():
            for i in range(len(cases)):
                bar.wait()                                    # the two failures start together
                got[(i, "infer fail")] = trace.call("infer", "infer bad token", raw_infer, live, [0, 1], [3, bad_tok])[0]
                bar.wait()                                    # both failed before either reads its text
                got[(i, "infer text")] = last_error()
                bar.wait()
                got[(i, "infer ok")] = trace.call("infer", "infer", raw_infer, live, [2, 3, 4, 5], [11 + i, 12, 13, 14])
                bar.wait()                                    # the other thread's successful call has returned
                got[(i, "infer text again")] = last_error()

        def sampler_body():
            for i, ((slots, top_k), _, _) in enumerate(cases):
                bar.wait()
                got[(i, "sample fail")] = trace.call("sample", "sample_topk fails", raw_topk, live, slots, top_k)[0]
                bar.wait()
                got[(i, "sample text")] = last_error()
                bar.wait()
                got[(i, "sample ok")] = trace.call("sample", "sample_topk", raw_topk, live, [6, 7], 8 + i)
                bar.wait()
                got[(i, "sample text again")] = last_error()

        run_threads(trace, {"infer": infer_body, "sampler": sampler_body}, [bar])
        for i, ((slots, top_k), code, frag) in enumerate(cases):
            where = f"case {i}"
            assert got[(i, "infer fail")] == capi.ERR_INVALID, where
            assert got[(i, "sample fail")] == code, where
            assert f"token id {bad_tok} is outside the vocabulary" in got[(i, "infer text")], (where, got[(i, "infer text")])
            assert frag in got[(i, "sample text")], (where, got[(i, "sample text")])
            assert got[(i, "infer text again")] == got[(i, "infer text")], where
            assert got[(i, "sample text again")] == got[(i, "sample text")], where
            # neither failure is fatal: the next calls give the twin's bits, and the twin fails the same way
            assert raw_infer(twin, [0, 1], [3, bad_tok])[0] == capi.ERR_INVALID
            assert raw_topk(twin, slots, top_k)[0] == code
            want_i = raw_infer(twin, [2, 3, 4, 5], [11 + i, 12, 13, 14])
            want_s = raw_topk(twin, [6, 7], 8 + i)
            assert want_i[0] == want_s[0] == capi.OK
            assert_same(got[(i, "infer ok")], want_i, f"{where} infer after the failures")
            assert_same(got[(i, "sample ok")], want_s, f"{where} sample_topk after the failures")
        assert_same(end_state(live), end_state(twin), "error text end state")
    finally:
        live.close()
        twin.close()
    print(f"[two-tasks] error text small7 V{V}: {len(cases)} overlapping failures, each thread read its own text")
