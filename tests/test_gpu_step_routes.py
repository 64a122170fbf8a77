"""The three entry points that run whole decode steps outside b200rwkv_infer, held to infer and to the oracle.

  - b200rwkv_bench_decode (the headline number, and what bench.py --dump-outputs writes) builds every step's metadata up
    front, copies it device to device between graph replays, takes its step shape from step_shape(nslot, nslot) and marks
    the kept rows on the host afterwards.  On a fresh engine whose slots were primed with a NONE prompt (as bench.py does,
    so the decode graph is first captured inside bench_decode), it must give bit for bit what a twin engine -- built from the
    same image, with the same slot history -- gives when the same tokens go through b200rwkv_infer one LAST step at a time:
    every listed slot's state, its kept row as every reader sees it (state_read + snapshot_back, sample_topk, sample_probs,
    SCORE token 0), the unlisted slots' states and rows unchanged, and `steps` times infer's launches per step.
  - At the bench shape (one layer of v6-7b / v7-2b9, V = 4096, batch 16 / 8) the bench route stays within the oracle's
    bounds of test_gpu_quant.py: kept row and state within 1e-3 relative, argmax exact, for fp16 activations, precision 1
    (the "f32" oracle), and Int8 / NF4 layers (oracle on the dequantised weights), after a 128-token NONE prompt per slot
    and warmup 3 + 5 steps.  The oracle keeps its matrices converted to f32 (Oracle.keep_all_matrices), without which the
    channel-mix matrices of this shape are converted again for every token.
  - b200rwkv_profile_step runs one step with no graph and no programmatic dependent launch (PDL): every kernel starts after
    its predecessor has finished.  It must equal a graph step, where each kernel's prologue before griddepcontrol.wait
    overlaps its predecessors, bit for bit (states of all slots and the last layer's residual rows, debug_read("hidden")).
    b200rwkv_profile_insitu(reps = r) replays a traced copy of the step graph r + 1 times and must equal r + 1 infer steps
    of the same tokens.  A mismatch means some kernel reads before its wait what a predecessor writes, or writes before its
    wait what a predecessor still reads.  Find it from the evidence of one run, by comparing the debug_read buffers of the
    two engines (x_a, xx1, r, k, v, ..., part_att, part_ffn, hidden) for a model with L = 1 and then growing L: the first
    buffer that differs names the kernel whose ordering is wrong.  Do not rerun to see whether it happens again.
  - Both profiling calls advance the listed slots' states without writing kept rows, so afterwards those slots have none
    (sample_topk / sample_probs ERR_STATE, SCORE token 0 NaN / UINT32_MAX, a state_read snapshot without a row), and every
    other slot keeps its row's bits.
  - All three refuse, before any CUDA work and with nothing changed (launch count, every slot's state): a slot out of range
    (ERR_STATE), a duplicate slot, a token id >= num_vocab, nslot 0 or above max_batch (ERR_INVALID).
  - bench.dump_outputs after bench_decode writes the twin's LAST rows and a sample of the backed states, bit for bit.

Configurations are those of test_gpu_step_program.py, plus NF4 layers and a model with two adapters bound to half the slots.
"""
import contextlib
import dataclasses
import functools
import os

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

f32 = np.float32
MAX_BATCH = 8
CHUNK = 64
QUANT_LAYERS = 2
REL_TOL = 1e-3
SLOTS = [5, 0, 3]                        # permuted, not contiguous
BOUND = ([0, 2, 4, 6], [1, 2, 1, 2])     # the adapter configuration: half the slots bound, to two adapters

# id: (preset, shape overrides, exact, quant type, adapters)
CONFIGS = {
    "tiny5": ("tiny5", {}, False, None, False),
    "tiny6": ("tiny6", {}, False, None, False),
    "tiny7": ("tiny7", {}, False, None, False),
    "small6": ("small6", {}, False, None, False),                 # front half, decay fold
    "small6-Dm16": ("small6", dict(Dm=16), False, None, False),   # no front half: LN1 + W1 + W2
    "small6-Dd192": ("small6", dict(Dd=192), False, None, False),  # decay LoRA stage 2 as its own launch
    "small6-exact": ("small6", {}, True, None, False),            # precision 1: split operands
    "small6-int8": ("small6", {}, False, "Int8", False),
    "tiny7-nf4": ("tiny7", {}, False, "NF4", False),
    "small6-adapters": ("small6", {}, False, None, True),
}


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def same_bits(a, b):
    return np.array_equal(bits(a), bits(b))


def rel_err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


@functools.lru_cache(maxsize=None)
def image(name):
    preset, over, _, _, ads = CONFIGS[name]
    shp = dataclasses.replace(synth.PRESETS[preset], **over)
    adapters = None
    if ads:
        adapters = [(synth.make_lora_st(shp, rank=8, seed=11, targets=("att.key", "att.value", "att.output", "ffn.key")), 0.1),
                    (synth.make_lora_st(shp, rank=16, seed=12, targets=("att.receptance", "att.gate", "ffn.value")), -0.15)]
    return shp, synth.make_st(shp, 0), adapters


def engine(name, **extra):
    _, _, exact, qt, ads = CONFIGS[name]
    shp, st, adapters = image(name)
    kw = dict(extra)
    if qt:
        kw.update(quant=QUANT_LAYERS, quant_type=qt)
    if ads:
        kw["adapters"] = adapters
    m = runtime.Model(st, max_batch=MAX_BATCH, token_chunk_size=CHUNK, exact=exact, **kw)
    if ads:
        m.bind_adapter(*BOUND)
    return m


@contextlib.contextmanager
def twins(name, **extra):
    """Two fresh engines from one image: the route under test runs on the first, infer on the second."""
    a = engine(name, **extra)
    try:
        b = engine(name, **extra)
        try:
            yield a, b
        finally:
            b.close()
    finally:
        a.close()


def fill_slots(engines, rng, with_rows=True):
    """Every slot gets a distinct random state and (with_rows) a random kept row, the same on every engine.  Returns
    (states, rows)."""
    m0 = engines[0]
    shape, V = m0.state.init().shape, m0.info["num_vocab"]
    states = [(0.5 * rng.standard_normal(shape)).astype(f32) for _ in range(MAX_BATCH)]
    rows = [(3.0 * rng.standard_normal(V)).astype(f32) for _ in range(MAX_BATCH)] if with_rows else None
    for m in engines:
        for s in range(MAX_BATCH):
            if not with_rows:
                m.state.load(states[s], s)
                continue
            snap = m.state.snapshot_load(states[s], rows[s])
            try:
                m.state.write(snap, s)
            finally:
                snap.free()
    return states, rows


def kept_row(m, slot):
    """The slot's kept row as bench.dump_outputs reads it: state_read + snapshot_back(with_logits); None without one."""
    snap = m.state.read(slot)
    try:
        return m.state.snapshot_back(snap, with_logits=True)[1]
    except capi.B200Error as e:
        assert e.code == capi.ERR_STATE
        return None
    finally:
        snap.free()


def bench_pair(a, b, slots, warmup, steps, rng, flush_l2=False, prime=8, count_launches=True):
    """Prime `slots` on both engines with a NONE prompt, run bench_decode on `a` and the same tokens through infer one
    LAST step at a time on `b`; check the launch count.  Returns the twin's last LAST rows, [nslot, V]."""
    n, V = len(slots), a.info["num_vocab"]
    prompt = rng.integers(0, V, size=n * prime).tolist()
    for m in (a, b):
        m.infer_raw(slots, [prime] * n, prompt, [capi.OPTION_NONE] * n)
    toks = rng.integers(0, V, size=(warmup + steps, n)).astype(np.uint32)
    _, launches = a.bench_decode(slots, toks, warmup, steps, flush_l2=flush_l2)
    per_step = set()
    for st in range(warmup + steps):
        before = b.launch_count()
        out = b.infer_raw(slots, [1] * n, toks[st].tolist(), [capi.OPTION_LAST] * n)
        per_step.add(b.launch_count() - before)
    if count_launches:
        assert len(per_step) == 1, per_step
        assert launches == steps * per_step.pop()
    return np.stack([r[0] for r in out])


def check_bench_pair(a, b, slots, states, rows, last, tag):
    """After bench_pair: states, kept rows and every reader of them, bit for bit against the twin."""
    for s in range(MAX_BATCH):
        got = a.state.back(s)
        assert same_bits(got, b.state.back(s)), (tag, "state", s)
        if s not in slots:
            assert same_bits(got, states[s]), (tag, "unlisted state", s)
        row = kept_row(a, s)
        want = last[slots.index(s)] if s in slots else rows[s]
        assert row is not None and same_bits(row, want), (tag, "kept row", s)
    every = list(range(MAX_BATCH))
    ids_a, p_a = a.sample_topk(every, top_k=32)
    ids_b, p_b = b.sample_topk(every, top_k=32)
    assert np.array_equal(ids_a, ids_b) and same_bits(p_a, p_b), tag
    assert same_bits(a.sample_probs(every), b.sample_probs(every)), tag
    tok = [int(t) for t in np.arange(MAX_BATCH) * 7 + 1]
    _, sa = a.infer_ex(every, [1] * MAX_BATCH, tok, [capi.OPTION_SCORE] * MAX_BATCH)
    _, sb = b.infer_ex(every, [1] * MAX_BATCH, tok, [capi.OPTION_SCORE] * MAX_BATCH)
    for s in every:
        assert not np.isnan(sa[s][0][0]), (tag, "SCORE token 0 found no kept row", s)
        assert same_bits(sa[s][0], sb[s][0]) and np.array_equal(sa[s][1], sb[s][1]), (tag, "SCORE token 0", s)


# ---------------------------------------------------------------------------------------------------------------------------
# A. bench_decode against infer
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CONFIGS))
def test_bench_decode_equals_infer(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    with twins(name) as (a, b):
        states, rows = fill_slots((a, b), rng)
        last = bench_pair(a, b, SLOTS, 2, 3, rng)
        check_bench_pair(a, b, SLOTS, states, rows, last, name)


# (config, slots, warmup, steps, flush_l2)
SHAPES = {
    "batch 1": ("small6", [6], 2, 3, False),
    "batch max": ("small6", [3, 7, 1, 0, 6, 2, 5, 4], 2, 3, False),
    "batch max exact": ("small6-exact", list(range(MAX_BATCH)), 1, 2, False),
    "batch max adapters": ("small6-adapters", [7, 6, 5, 4, 3, 2, 1, 0], 1, 2, False),
    "tiny7 batch 1": ("tiny7", [2], 1, 4, False),
    "tiny7 batch max": ("tiny7", list(range(MAX_BATCH))[::-1], 1, 2, False),
    "warmup 0": ("small6", SLOTS, 0, 4, False),
    "warmup 0 tiny5": ("tiny5", [1, 4], 0, 1, False),
    "flush_l2": ("small6", SLOTS, 1, 2, True),
}


@pytest.mark.parametrize("case", list(SHAPES))
def test_bench_decode_equals_infer_shapes(case):
    name, slots, warmup, steps, flush = SHAPES[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    with twins(name) as (a, b):
        states, rows = fill_slots((a, b), rng)
        last = bench_pair(a, b, slots, warmup, steps, rng, flush_l2=flush)
        check_bench_pair(a, b, slots, states, rows, last, case)


def _gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_gpu_count() < 2, reason="tensor parallelism needs two GPUs")
def test_tensor_parallel_bench_decode_equals_infer():
    """Two in-process ranks: states (merged by head in state_back) and the sampler's view of rank 0's gathered kept rows."""
    rng = np.random.default_rng(2)
    with twins("small6", devices=[0, 1]) as (a, b):
        fill_slots((a, b), rng, with_rows=False)
        bench_pair(a, b, SLOTS, 1, 3, rng, count_launches=False)
        for s in range(MAX_BATCH):
            assert same_bits(a.state.back(s), b.state.back(s)), s
        ids_a, p_a = a.sample_topk(SLOTS, top_k=32)
        ids_b, p_b = b.sample_topk(SLOTS, top_k=32)
        assert np.array_equal(ids_a, ids_b) and same_bits(p_a, p_b)


# ---------------------------------------------------------------------------------------------------------------------------
# B. the bench route against the oracle at the bench shape
# ---------------------------------------------------------------------------------------------------------------------------
PROMPT = 128
# id: (preset, batch, exact, quant type)
ORACLE_CASES = {
    "v6-7b": ("v6-7b", 16, False, None),
    "v6-7b-exact": ("v6-7b", 16, True, None),
    "v6-7b-int8": ("v6-7b", 16, False, "Int8"),
    "v6-7b-nf4": ("v6-7b", 16, False, "NF4"),
    "v7-2b9": ("v7-2b9", 8, False, None),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_bench_route_matches_the_oracle(case):
    preset, batch, exact, qt = ORACLE_CASES[case]
    shp = dataclasses.replace(synth.PRESETS[preset], L=1, V=4096)
    st = synth.make_st(shp, 0)
    w = O.parse_st(st)
    kw = {}
    if qt:
        kw = dict(quant=1, quant_type=qt)
        w = Q.quantize_model(w, 1, {"Int8": Q.QUANT_INT8, "NF4": Q.QUANT_NF4}[qt])
    orc = O.Oracle(w, "f32" if exact else "f16").keep_all_matrices()
    m = runtime.Model(st, max_batch=batch, token_chunk_size=CHUNK, exact=exact, **kw)
    try:
        rng = np.random.default_rng(9)
        slots = list(range(batch))
        for s in slots:
            m.state.load(m.state.init(), s)
        prompt = rng.integers(1, shp.V, size=(batch, PROMPT))
        m.infer_raw(slots, [PROMPT] * batch, prompt.reshape(-1).tolist(), [capi.OPTION_NONE] * batch)
        dec = rng.integers(1, shp.V, size=(3 + 5, batch)).astype(np.uint32)
        m.bench_decode(slots, dec, 3, 5)
        for s in (0, batch // 2 - 1, batch - 1):
            snap = m.state.read(s)
            try:
                state, row = m.state.snapshot_back(snap, with_logits=True)
            finally:
                snap.free()
            want, want_state = orc.run(prompt[s].tolist() + dec[:, s].tolist(), orc.state_init())
            assert rel_err(row, want[0]) <= REL_TOL, (case, s)
            assert row.argmax() == want[0].argmax(), (case, s)
            assert rel_err(state, want_state) <= REL_TOL, (case, s)
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------------------------------------
# C. the serialised step and the traced graph step against PDL graph steps
# ---------------------------------------------------------------------------------------------------------------------------
def profile_pair(a, b, slots, route, reps, rng):
    """The same preceding LAST call on both engines (debug_read's row count is the last infer step's token count), then
    the route on `a` and as many NONE steps of the same tokens on `b`."""
    n, V = len(slots), a.info["num_vocab"]
    first = rng.integers(0, V, size=n).tolist()
    for m in (a, b):
        m.infer_raw(slots, [1] * n, first, [capi.OPTION_LAST] * n)
    toks = rng.integers(0, V, size=n).astype(np.uint32)
    if route == "profile_step":
        a.profile_step(slots, toks)
        nsteps = 1
    else:
        a.profile_insitu(slots, toks, reps=reps)
        nsteps = reps + 1
    for _ in range(nsteps):
        b.infer_raw(slots, [1] * n, toks.tolist(), [capi.OPTION_NONE] * n)


ROUTES = [("profile_step", 1), ("profile_insitu", 1), ("profile_insitu", 2)]


@pytest.mark.parametrize("route,reps", ROUTES, ids=["step", "insitu-1", "insitu-2"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_profiling_steps_equal_graph_steps(name, route, reps):
    rng = np.random.default_rng([sum(map(ord, name)), reps])
    with twins(name) as (a, b):
        states, _ = fill_slots((a, b), rng, with_rows=False)
        profile_pair(a, b, SLOTS, route, reps, rng)
        n = len(SLOTS)
        assert same_bits(a.debug_read("hidden", rows=n), b.debug_read("hidden", rows=n)), (name, route, "hidden")
        for s in range(MAX_BATCH):
            got = a.state.back(s)
            assert same_bits(got, b.state.back(s)), (name, route, "state", s)
            if s not in SLOTS:
                assert same_bits(got, states[s]), (name, route, "unlisted state", s)
            else:
                assert not same_bits(got, states[s]), (name, route, "state did not advance", s)


# ---------------------------------------------------------------------------------------------------------------------------
# D. the kept row after a profiling step
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route,reps", ROUTES[:2], ids=["step", "insitu"])
@pytest.mark.parametrize("name", ["tiny6", "small6-adapters"])
def test_profiling_steps_drop_the_kept_row(name, route, reps):
    rng = np.random.default_rng(5)
    with twins(name) as (a, b):
        _, rows = fill_slots((a, b), rng)
        profile_pair(a, b, SLOTS, route, reps, rng)
        for s in range(MAX_BATCH):
            row = kept_row(a, s)
            if s not in SLOTS:
                assert row is not None and same_bits(row, rows[s]), (name, route, "unlisted row", s)
                continue
            assert row is None, (name, route, "a stale kept row", s)
            for read in (lambda: a.sample_topk([s], top_k=8), lambda: a.sample_probs([s])):
                with pytest.raises(capi.B200Error) as ei:
                    read()
                assert ei.value.code == capi.ERR_STATE, (name, route, s)
        _, sc = a.infer_ex(SLOTS, [1] * len(SLOTS), [3] * len(SLOTS), [capi.OPTION_SCORE] * len(SLOTS))
        for i, s in enumerate(SLOTS):
            assert np.isnan(sc[i][0][0]) and int(sc[i][1][0]) == 0xFFFFFFFF, (name, route, s)


# ---------------------------------------------------------------------------------------------------------------------------
# E. refusals
# ---------------------------------------------------------------------------------------------------------------------------
def _call(route, m, slots, bad_token):
    """Run `route` on `slots`; with bad_token the last token id it reads is num_vocab."""
    V = m.info["num_vocab"]
    nrows = 3 if route == "bench_decode" else 1
    toks = (np.arange(nrows * len(slots), dtype=np.uint32) % V).reshape(nrows, len(slots))
    if bad_token:
        toks[-1, -1] = V
    if route == "bench_decode":
        return m.bench_decode(slots, toks, 1, 2)
    if route == "profile_step":
        return m.profile_step(slots, toks[0])
    return m.profile_insitu(slots, toks[0], reps=1)


REFUSALS = {
    "slot -1": ([0, -1], False, capi.ERR_STATE),
    "slot S": ([1, MAX_BATCH], False, capi.ERR_STATE),
    "duplicate slot": ([2, 5, 2], False, capi.ERR_INVALID),
    "token V": ([1, 4], True, capi.ERR_INVALID),
    "nslot 0": ([], False, capi.ERR_INVALID),
    "nslot above max_batch": (list(range(MAX_BATCH)) + [0], False, capi.ERR_INVALID),
}


@pytest.fixture(scope="module")
def refusal_engine():
    m = engine("tiny6")
    yield m
    m.close()


@pytest.mark.parametrize("case", list(REFUSALS))
@pytest.mark.parametrize("route", ["bench_decode", "profile_step", "profile_insitu"])
def test_decode_routes_refuse_bad_arguments(refusal_engine, route, case):
    m = refusal_engine
    slots, bad_token, code = REFUSALS[case]
    fill_slots((m,), np.random.default_rng(6))
    before = [m.state.back(s) for s in range(MAX_BATCH)]
    launches = m.launch_count()
    with pytest.raises(capi.B200Error) as ei:
        _call(route, m, slots, bad_token)
    assert ei.value.code == code, (route, case, ei.value)
    assert m.launch_count() == launches, (route, case)
    for s in range(MAX_BATCH):
        assert same_bits(m.state.back(s), before[s]), (route, case, s)
    _call(route, m, [1, 4], False)                 # and the engine still runs the route
    assert not same_bits(m.state.back(1), before[1])


# ---------------------------------------------------------------------------------------------------------------------------
# F. bench.py --dump-outputs after the bench route
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small6", "tiny7-nf4"])
def test_dump_outputs_hold_the_infer_route(tmp_path, name):
    import bench
    rng = np.random.default_rng(8)
    slots = [4, 1, 6, 2]
    with twins(name) as (a, b):
        fill_slots((a, b), rng)
        last = bench_pair(a, b, slots, 2, 3, rng)
        bench.dump_outputs(str(tmp_path), a, slots)
        logits = np.load(os.path.join(tmp_path, "logits.npy"))
        assert logits.shape == last.shape and same_bits(logits, last)
        idx = np.load(os.path.join(tmp_path, "state_sample_index.npy")).astype(np.int64)
        sample = np.load(os.path.join(tmp_path, "state_sample.npy"))
        for i, s in enumerate(slots):
            assert same_bits(sample[i], b.state.back(s).reshape(-1)[idx]), s
        ids, probs = b.sample_topk(slots, top_k=128)
        assert np.array_equal(np.load(os.path.join(tmp_path, "topk_ids.npy")), ids.astype(np.float64))
        assert same_bits(np.load(os.path.join(tmp_path, "topk_probs.npy")), probs)
