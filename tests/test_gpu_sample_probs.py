"""The whole adjusted distribution on the GPU (b200rwkv_sample_probs, csrc/sample.cuh probs_stats_kernel / probs_write_kernel)
through the C ABI: against a float64 softmax of the oracle's adjusted row (oracle/sampling_numpy.py adjusted_logits) on the
same kept row, against b200rwkv_sample_topk and b200rwkv_softmax, over vocabulary sizes above 65536 and not a multiple of 4,
with no side effect on the kept rows, states, candidates or launch counts, deterministic per row, and in generation loops of
the reference's Mirostat, Typical and Nucleus (top_k > 128) samplers, restated below from sampler/mirostat.rs:44-90,
sampler/typical.rs:70-131 and sampler/nucleus.rs:69-123.

Error bound of one probability p = expf(x - M) * (1 / S), S = sum over segments of s_g expf(m_g - M), u = 2^-24:
  - x - M is rounded once: an absolute error <= u |x - M| in the exponent, a relative error <= u |x - M| in p;
  - expf is within 2 ulp (CUDA C Programming Guide, maximum ulp errors): 2u;
  - S: each element's term expf(x - m_g) (2u + u |x - m_g|), 8 sequential adds per thread, 5 + 3 levels of the block tree,
    one expf (2u) and one product (u) per segment rescale, at most 2 sequential adds per lane and 5 levels of the xor tree:
    a relative error below (2 + 8 + 8 + 3 + 2 + 5) u + u max |x - m_g| <= 28u + u |x_min - M|; 1 / S and the product: 2u.
So |p - p64| <= p64 (32 + 2 |x - M|) u for every element that is not -inf, where |x - M| stays below 104 for any p that is
not below the f32 subnormal range (e^-104 < 2^-149).  The tests assert |p - p64| <= 2e-6 + 2e-5 p64: 2e-5 = 335u covers
(32 + 2 * 104) u = 240u, and the absolute 2e-6 covers p64 below 2^-126 rounding to f32 subnormals or zero.
The row sum: sum_i p_i (1 + e_i) - 1 = sum_i p_i e_i, at most the largest relative error above (<< V u for V >= 509), plus
the float64 summation's own rounding; the tests assert |sum - 1| <= V 2^-24.
"""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import sampling_numpy as S

pytestmark = pytest.mark.gpu

ATOL, RTOL = 2e-6, 2e-5
f32 = np.float32


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(preset, max_batch=4, **over):
        key = (preset, max_batch, tuple(sorted(over.items())))
        if key not in cache:
            shp = synth.PRESETS[preset] if not over else dataclasses.replace(synth.PRESETS[preset], **over)
            cache[key] = runtime.Model(synth.make_st(shp, 0), max_batch=max_batch, token_chunk_size=32)
        return cache[key]

    yield get
    for m in cache.values():
        m.close()


def softmax64(adjusted: np.ndarray) -> np.ndarray:
    x = np.asarray(adjusted, np.float64)
    m = x.max()
    if not np.isfinite(m):
        return np.zeros_like(x)
    e = np.exp(x - m)
    return e / e.sum()


def fill_rows(m, slots, seed=0):
    """Fresh states, a few prompt tokens per slot, LAST rows to the host: the kept row of every slot, as host copies."""
    rng = np.random.default_rng(seed)
    V = m.info["num_vocab"]
    toks = [rng.integers(0, V, size=1 + (i % 3)).tolist() for i in range(len(slots))]
    for s in slots:
        m.state.load(m.state.init(), s)
    rows = m.infer_raw(list(slots), [len(t) for t in toks], sum(toks, []), [capi.OPTION_LAST] * len(slots))
    return [r[0].copy() for r in rows]


def mixes(rows, seed=1):
    """The adjustment mixes, per row: (penalties, allow, bias) lists over the rows."""
    rng = np.random.default_rng(seed)
    n, V = len(rows), rows[0].size
    none = ([None] * n, None, [None] * n)
    pen = [{int(t): float(v) for t, v in zip(rng.choice(V, 50, replace=False), rng.random(50) * 3)} for _ in range(n)]
    sparse = rng.random((n, V)) < 0.1
    for i in range(n):
        sparse[i, rng.integers(0, V)] = True
    # the row's best token is masked off; its neighbour is biased to the top; the masked token's own bias changes nothing
    nb_allow = np.ones((n, V), bool)
    nb_bias = []
    for i, r in enumerate(rows):
        a = int(r.argmax())
        b = a + 1 if a + 1 < V else a - 1
        nb_allow[i, a] = False
        nb_bias.append({b: float(r.max() - r[b]) + 3.0, a: 100.0})
    allb = [{**pb, **{int(t): -2.0 for t in rng.choice(V, 5, replace=False) if int(t) not in pb}} for pb in nb_bias]
    both = sparse.copy()
    for i, pb in enumerate(nb_bias):
        b, a = list(pb)
        both[i, a], both[i, b] = False, True
    return {"none": none, "penalties": (pen, None, [None] * n), "sparse mask": ([None] * n, sparse, [None] * n),
            "masked neighbour": ([None] * n, nb_allow, nb_bias), "all": (pen, both, allb)}


def adjusted(row, pen, allow, bias):
    return S.adjusted_logits(row, pen, allow, bias)


def check_row(got, row, pen, allow, bias, tag):
    adj = adjusted(row, pen, allow, bias)
    want = softmax64(adj)
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= ATOL + RTOL * want), (tag, float((err - RTOL * want).max()))
    assert np.all(got[np.isneginf(adj)] == 0), tag
    if np.isfinite(adj.max()):
        assert abs(got.astype(np.float64).sum() - 1.0) <= row.size * 2.0 ** -24, tag


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_matches_the_oracle(models, preset):
    m = models(preset)
    slots = [2, 0, 3, 1]
    rows = fill_rows(m, slots)
    for name, (pen, allow, bias) in mixes(rows).items():
        probs = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
        assert probs.shape == (4, m.info["num_vocab"]) and probs.dtype == np.float32
        for i in range(4):
            check_row(probs[i], rows[i], pen[i], None if allow is None else allow[i], bias[i], (preset, name, i))
        if name == "masked neighbour":
            for i in range(4):
                a = int(rows[i].argmax())
                assert probs[i, a] == 0 and int(probs[i].argmax()) == list(bias[i])[0]


@pytest.mark.parametrize("V", [2048, 65536])
def test_sample_topk_candidates_are_entries_of_the_row(models, V):
    m = models("tiny6", V=V)
    slots = [0, 1, 2, 3]
    rows = fill_rows(m, slots, seed=3)
    for name, (pen, allow, bias) in mixes(rows, seed=4).items():
        ids, p = m.sample_topk(slots, penalties=pen, bias=bias, allow=allow, top_k=128)
        probs = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
        for i in range(4):
            row = probs[i]
            # the same segment statistics, combine and expression: bit for bit (so also within the bound)
            assert np.array_equal(p[i], row[ids[i]]), (V, name, i)
            # the candidates are the 128 largest entries, in non-increasing order
            assert np.all(np.diff(row[ids[i]]) <= 0), (V, name, i)
            rest = np.ones(V, bool)
            rest[ids[i]] = False
            assert row[rest].max() <= row[ids[i]].min(), (V, name, i)


def test_matches_b200rwkv_softmax_on_the_host_adjusted_row(models):
    m = models("small6")
    slots = [1, 3]
    rows = fill_rows(m, slots, seed=5)
    for name, (pen, allow, bias) in mixes(rows, seed=6).items():
        probs = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
        adj = [adjusted(rows[i], pen[i], None if allow is None else allow[i], bias[i]) for i in range(2)]
        host = m.softmax(adj)
        for i in range(2):
            b = host[i].astype(np.float64)
            assert np.all(np.abs(probs[i] - b) <= ATOL + RTOL * b), (name, i)


@pytest.mark.parametrize("V", [65536, 70003, 509])
def test_vocabulary_sizes(models, V):
    """V = 65536 (32 segments), V = 70003 (35 segments: more than one per lane of the combine, and V % 4 = 3) and V = 509
    (one partial segment, V % 4 = 1).  The last token is biased to the top so the scalar tail carries the largest entry."""
    m = models("tiny6", V=V)
    slots = [0, 1, 2]
    rows = fill_rows(m, slots, seed=7)
    ms = mixes(rows, seed=8)
    ms["last token"] = ([None] * 3, None, [{V - 1: float(r.max() - r[V - 1]) + 2.0} for r in rows])
    for name, (pen, allow, bias) in ms.items():
        probs = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
        for i in range(3):
            check_row(probs[i], rows[i], pen[i], None if allow is None else allow[i], bias[i], (V, name, i))
        if name == "last token":
            assert all(int(probs[i].argmax()) == V - 1 for i in range(3))
    if V > 65536:
        with pytest.raises(capi.B200Error) as ei:
            m.sample_topk(slots, top_k=4)
        assert ei.value.code == capi.ERR_UNSUPPORTED


@pytest.mark.parametrize("V", [2048, 70003])
def test_all_tokens_masked(models, V):
    """Every token disallowed: the row is all zeros, as sample_topk's probabilities are (ids 0 .. top_k-1 there)."""
    m = models("tiny6", V=V)
    slots = [0, 2]
    fill_rows(m, slots, seed=9)
    allow = np.zeros((2, V), bool)
    bias = [{5: 10.0}, {}]
    probs = m.sample_probs(slots, bias=bias, allow=allow)
    assert not np.any(probs) and not np.any(np.isnan(probs))
    if V <= 65536:
        ids, p = m.sample_topk(slots, bias=bias, allow=allow, top_k=16)
        assert not np.any(p) and ids.tolist() == [list(range(16))] * 2


def test_no_side_effects(models):
    m = models("small6")
    slots = [0, 1, 2, 3]
    fill_rows(m, slots, seed=10)
    ms = mixes([np.zeros(m.info["num_vocab"], np.float32)] * 4, seed=11)
    pen, allow, bias = ms["all"]
    ids0, p0 = m.sample_topk(slots, penalties=pen, bias=bias, allow=allow, top_k=128)
    states0 = [m.state.back(s) for s in slots]
    snaps = [m.state.read(s) for s in slots]
    kept0 = [m.state.snapshot_back(t, with_logits=True)[1] for t in snaps]
    for t in snaps:
        t.free()
    launches0 = m.launch_count()
    for name, (pn, al, bs) in ms.items():
        m.sample_probs(slots, penalties=pn, bias=bs, allow=al)
        m.sample_probs(slots[::-1][:2])
    assert m.launch_count() == launches0
    ids1, p1 = m.sample_topk(slots, penalties=pen, bias=bias, allow=allow, top_k=128)
    assert np.array_equal(ids0, ids1) and np.array_equal(p0.view(np.uint32), p1.view(np.uint32))
    for s, want in zip(slots, states0):
        assert np.array_equal(m.state.back(s).view(np.uint32), want.view(np.uint32))
    snaps = [m.state.read(s) for s in slots]
    for t, want in zip(snaps, kept0):
        assert np.array_equal(m.state.snapshot_back(t, with_logits=True)[1].view(np.uint32), want.view(np.uint32))
        t.free()


def test_deterministic_and_independent_of_the_other_rows(models):
    m = models("tiny7", V=70003)
    slots = [0, 1, 2, 3]
    rows = fill_rows(m, slots, seed=12)
    pen, allow, bias = mixes(rows, seed=13)["all"]
    a = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
    b = m.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for order in ([3, 1, 0, 2], [2], [1, 3]):
        c = m.sample_probs([slots[i] for i in order], penalties=[pen[i] for i in order], bias=[bias[i] for i in order],
                           allow=allow[order])
        for k, i in enumerate(order):
            assert np.array_equal(c[k].view(np.uint32), a[i].view(np.uint32)), (order, i)


# ---- the reference's whole-distribution samplers, restated (f32 like the Rust code; `rand` is fastrand::f32()) ----
# Ties: the reference sorts with voracious_sort (unstable), so the order of equal keys is unspecified there; these
# restatements break ties by token id ascending, one of the reference's possible outcomes.

class MirostatSampler:
    """sampler/mirostat.rs:30-90."""

    def __init__(self, tau=3.0, rate=0.1):
        self.tau, self.rate = f32(tau), f32(rate)
        self.max_surprise = f32(self.tau * f32(2.0))
        self.penalties = {}                 # transform is a no-op

    def init(self, model_tokens):
        pass

    def sample(self, probs, rand: float) -> int:
        probs = np.asarray(probs, f32)
        order = np.lexsort((np.arange(probs.size), -probs.astype(np.float64)))          # probability descending
        x = probs[order]
        cum = np.cumsum(x, dtype=f32)                                                   # sequential f32 scan
        with np.errstate(divide="ignore"):
            surprise = -np.log2(x)
        over = np.nonzero(surprise > self.max_surprise)[0]
        k = int(over[0]) + 1 if over.size else x.size
        total = cum[k - 1]
        r = f32(f32(rand) * total)
        hit = np.nonzero(r <= cum[:k])[0]
        j = int(hit[0]) if hit.size else 0
        token, prob = int(order[j]), x[j]
        token_surprise = f32(np.log2(total) - np.log2(prob))
        self.max_surprise = f32(self.max_surprise - f32(self.rate * f32(token_surprise - self.tau)))
        self.max_surprise = min(self.max_surprise, f32(f32(4.0) * self.tau))
        return token


class TypicalSampler:
    """sampler/typical.rs:40-131."""

    def __init__(self, tau=0.5, top_k=128, temperature=1.0, presence_penalty=0.3, frequency_penalty=0.3,
                 penalty_decay=0.99654026):
        self.tau, self.top_k, self.temperature = f32(tau), int(top_k), f32(temperature)
        self.presence_penalty, self.frequency_penalty, self.penalty_decay = f32(presence_penalty), f32(frequency_penalty), f32(penalty_decay)
        self.penalties: dict[int, np.float32] = {}

    def init(self, model_tokens):
        for index, token in enumerate(reversed(list(model_tokens))):
            pen = self.penalties.pop(int(token), self.presence_penalty)
            pen = f32(pen + self.frequency_penalty * f32(np.power(self.penalty_decay, f32(index))))
            self.penalties[int(token)] = pen

    def sample(self, probs, rand: float) -> int:
        probs = np.asarray(probs, f32)
        ids = np.nonzero(probs > 0)[0]
        x = probs[ids]
        y = (-np.log(x)).astype(f32)
        entropy = np.cumsum((x * y).astype(f32), dtype=f32)[-1]                        # sequential f32 sum
        key = np.abs((y - entropy).astype(f32))
        order = np.lexsort((ids, key.astype(np.float64)))[: self.top_k]                 # |y - entropy| ascending
        kept, cum = [], f32(0.0)
        for j in order:
            if cum > self.tau:
                break
            cum = f32(cum + x[j])
            kept.append((int(ids[j]), f32(np.power(x[j], f32(1.0) / self.temperature))))
        total = f32(0.0)
        for _, v in kept:
            total = f32(total + v)
        token, cum = kept[0][0], f32(0.0)
        for i, v in kept:
            cum = f32(cum + f32(v / total))
            if f32(rand) <= cum:
                token = i
                break
        for t in self.penalties:
            self.penalties[t] = f32(self.penalties[t] * self.penalty_decay)
        self.penalties[token] = f32(self.penalties[token] + self.frequency_penalty) if token in self.penalties else self.presence_penalty
        return token


SAMPLERS = {
    "mirostat": lambda: MirostatSampler(tau=3.0, rate=0.1),
    "typical": lambda: TypicalSampler(tau=0.6, top_k=256, temperature=1.2),
    # nucleus.rs:69-123 sorts the probabilities it is given (no order_key): the same on both routes
    "nucleus500": lambda: S.NucleusSampler(top_p=0.95, top_k=500, temperature=1.1),
}


@pytest.mark.parametrize("kind", list(SAMPLERS))
def test_generation_loop_device_route_equals_host_route(models, kind):
    """24 tokens on two slots: (a) logits to the host, adjusted_logits + softmax on the host (the reference's route);
    (b) logits kept in HBM, b200rwkv_sample_probs.  The same sampler and the same uniform draws give the same tokens."""
    m = models("small6")
    draws = np.random.default_rng(14).random((24, 2))
    prompt = [[3, 4, 5], [9]]
    outs = []
    for route in ("host", "device"):
        for s in range(2):
            m.state.load(m.state.init(), s)
        smp = [SAMPLERS[kind]() for _ in range(2)]
        for s in range(2):
            smp[s].init(prompt[s])
        toks = [p[:] for p in prompt]
        feed = [p[:] for p in prompt]
        for step in range(24):
            pens = [dict(x.penalties) for x in smp]
            if route == "host":
                rows = m.infer_raw([0, 1], [len(f) for f in feed], sum(feed, []), [capi.OPTION_LAST] * 2)
                probs = [S.softmax_row(S.adjusted_logits(rows[s][0], pens[s], None, None)) for s in range(2)]
            else:
                m.infer_raw([0, 1], [len(f) for f in feed], sum(feed, []), [capi.OPTION_LAST] * 2, keep_on_device=True)
                probs = m.sample_probs([0, 1], penalties=pens)
            nxt = [smp[s].sample(probs[s], draws[step, s]) for s in range(2)]
            for s in range(2):
                toks[s].append(nxt[s])
            feed = [[t] for t in nxt]
        outs.append(toks)
    assert outs[0] == outs[1]
    assert len({t for seq in outs[0] for t in seq[3:]}) > 2          # the loop really samples, not a fixed point


def _call(m, slots, pen_off=None, out=True, nrows=None):
    """Raw b200rwkv_sample_probs with a valid output buffer unless out=False."""
    a_slot = np.asarray(slots, np.int32)
    n = len(slots) if nrows is None else nrows
    buf = np.empty((max(len(slots), 1), m.info["num_vocab"]), np.float32)
    po = None if pen_off is None else np.asarray(pen_off, np.int32)
    pt = np.arange(8, dtype=np.uint32)
    pv = np.zeros(8, np.float32)
    return capi.lib().b200rwkv_sample_probs(m._h, n, capi.ptr(a_slot), None if po is None else capi.ptr(po), capi.ptr(pt),
                                            capi.ptr(pv), None, None, None, None, capi.ptr(buf) if out else None)


def test_argument_errors(models):
    """Each refusal returns its status before any CUDA work: a valid call right after still succeeds with the same row."""
    m = models("small6", max_batch=5)                 # an engine of its own: slot 3 never produces a row
    fill_rows(m, [0, 1, 2], seed=15)
    want = m.sample_probs([0, 1])
    cases = {
        "slot without a row": (_call(m, [0, 3]), capi.ERR_STATE),
        "slot out of range": (_call(m, [0, 5]), capi.ERR_STATE),
        "negative slot": (_call(m, [-1]), capi.ERR_STATE),
        "duplicate slot": (_call(m, [1, 1]), capi.ERR_INVALID),
        "descending offsets": (_call(m, [0, 1], pen_off=[0, 2, 1]), capi.ERR_INVALID),
        "null output": (_call(m, [0], out=False), capi.ERR_INVALID),
        "nrows = 0": (_call(m, [0], nrows=0), capi.ERR_INVALID),
        "nrows > max_batch": (_call(m, [0, 1, 2, 3, 4, 0], nrows=6), capi.ERR_INVALID),
    }
    for name, (got, code) in cases.items():
        assert got == code, name
        again = m.sample_probs([0, 1])
        assert np.array_equal(again.view(np.uint32), want.view(np.uint32)), name
    assert _call(m, [2, 0], pen_off=[0, 1, 3]) == capi.OK


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
def test_tensor_parallel_engine_gives_the_same_distribution():
    """In-process tensor parallelism: rank 0 holds the gathered kept rows and runs the kernels; the distribution of each row
    (the gathered row the same infer call returned) is within the bound of the oracle, as on one GPU."""
    st = synth.make_st("small6", 0)
    multi = runtime.Model(st, max_batch=4, token_chunk_size=32, devices=[0, 1])
    try:
        slots = [0, 1]
        rows = fill_rows(multi, slots, seed=16)
        for name, (pen, allow, bias) in mixes(rows, seed=17).items():
            probs = multi.sample_probs(slots, penalties=pen, bias=bias, allow=allow)
            for i in range(2):
                check_row(probs[i], rows[i], pen[i], None if allow is None else allow[i], bias[i], ("tp", name, i))
    finally:
        multi.close()
