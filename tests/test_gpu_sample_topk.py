"""The top-k sampler (b200rwkv_sample_topk, csrc/sample.cuh topk_segment_kernel / topk_merge_kernel), the per-slot kept
logits row every sampling reader takes (keep_rows_kernel and the engine's keep_valid flags) and b200rwkv_softmax
(csrc/misc.cuh softmax_kernel), through the C ABI on rows constructed to hit the sort's edges: exact ties across and inside
segments, the best tokens all in one segment or one per segment, monotone rows, +0.0 beside -0.0, neighbours one ulp apart,
magnitudes near 1e38, -inf entries, fewer allowed tokens than top_k, and penalty / bias lists that make or break ties.  Rows
are injected as the kept row of a slot with b200rwkv_snapshot_load + b200rwkv_state_write.  NaN logits are outside this
file.

References:
  - ids: the f32 adjusted row of oracle/sampling_numpy.adjusted_logits (the f32 operations of adjust_segment, in its
    order), ordered by np.lexsort((ids, -adjusted)): logit descending, id ascending, +0.0 == -0.0.  The ids must be equal.
    Penalty and bias tokens >= num_vocab are ignored by adjust_segment, so the reference drops them.
  - sample_topk probabilities: a float64 softmax of that f32 row, within 2e-6 + 2e-5 p64 -- the bound derived in
    tests/test_gpu_sample_probs.py (|p - p64| <= p64 (32 + 2 |x - M|) u, u = 2^-24, |x - M| < 104 for any p above the f32
    subnormal range; 2e-5 = 335u covers 240u, 2e-6 covers p64 that round to subnormals).  Each probability also equals
    sample_probs's entry for the same row and lists bit for bit.
  - SCORE token 0 from the kept row: test_gpu_score.py's bound 2^-16 + 2^-22 |x_t - m|, restated in `score_bound`.
  - softmax_kernel, one CTA of 1024 threads per row: out = expf(x - m) * (1 / S), S = sum expf(x - m), m the row max (exact).
      * x - m is rounded once: relative error d u in expf's result, d = m - x;  expf within 2 ulp: 2u;
      * S: each term (2 + d_j) u; k = ceil(V / 1024) sequential adds per thread, then 5 levels of the warp xor tree and 5
        over the 32 warps' results, each level one rounding of a sum of positive terms: (k + 10) u.  A term with d_j >= 104
        underflows (e^-104 < 2^-149), and a subnormal term is off by at most 2^-148, so together they move S (>= 1) by less
        than V 2^-147; every other term has d_j < 104: S is within (k + 12 + min(max d, 104)) u + V 2^-147 relative;
      * 1 / S and the product: u each.
    So |out - p64| <= p64 (k + 16 + min(max d, 104) + d) u (1 + 1e-3) + 4 * 2^-149 (the absolute term: results in the f32
    subnormal range, whose expf and product round to 2^-149).  A -inf entry gives exactly 0; a row with one finite entry
    gives exactly 1 there.  A row of only -inf has no finite maximum (the result is NaN) and is outside the contract.

Kept-row lifecycle: after each operation every reader (sample_topk or ERR_STATE, sample_probs or ERR_STATE,
snapshot_back(state_read(slot), with_logits) or ERR_STATE, SCORE token 0 or NaN / UINT32_MAX) sees the row of the slot's
current state, and the other slots' rows keep their bits.
"""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import sampling_numpy as S

pytestmark = pytest.mark.gpu

f32 = np.float32
U = 2.0 ** -24
ATOL, RTOL = 2e-6, 2e-5
SEG = 2048                        # elements per topk_segment_kernel segment
SCORE_THREADS = 256
VOCABS = [509, 2048, 2049, 4095, 6144, 65535, 65536]
TOP_KS = [1, 2, 3, 17, 64, 127, 128]
WORST = {}


def _note(tag, ratio):
    WORST[tag] = max(WORST.get(tag, 0.0), float(ratio))


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(V, max_batch=16, chunk=32):
        key = (V, max_batch, chunk)
        if key not in cache:
            st = synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], V=V), 0)
            cache[key] = runtime.Model(st, max_batch=max_batch, token_chunk_size=chunk)
        return cache[key]

    yield get
    for m in cache.values():
        m.close()
    if WORST:
        print("\nworst error / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


# ---- references ----

def expect_ids(adj, k):
    key = -np.asarray(adj, np.float64) + 0.0                 # + 0.0: -0.0 and +0.0 are one key
    return np.lexsort((np.arange(adj.size), key))[:k]


def softmax64(adj):
    x = np.asarray(adj, np.float64)
    m = x.max()
    if not np.isfinite(m):
        return np.zeros_like(x)
    e = np.exp(x - m)
    return e / e.sum()


def check_probs(got, p64, tag):
    """sample_topk / sample_probs probabilities against the float64 softmax of the adjusted row."""
    err = np.abs(np.asarray(got, np.float64) - p64)
    lim = ATOL + RTOL * p64
    assert np.all(err <= lim), (tag, float((err - lim).max()))
    _note(tag.split(":")[0], (err / lim).max())


def score_bound(row, t):
    """test_gpu_score.py's derived bound of one score and the headline bound it stays inside."""
    V = row.size
    k = -(-V // (4 * SCORE_THREADS)) * 4 + 1
    d = abs(float(row[t]) - float(row.max()))
    derived = (4 + 6 * k + 8) * U + 3 * U * np.log(V) + 2 * U * d
    headline = 2.0 ** -16 + 2.0 ** -22 * d
    assert derived <= headline
    return headline


def log_softmax64(row):
    x = np.asarray(row, np.float64)
    m = x.max()
    return x - m - np.log(np.exp(x - m).sum())


# ---- constructed rows: (family, row, penalties, allow, bias) ----

@dataclasses.dataclass
class Case:
    family: str
    row: np.ndarray
    pen: dict | None = None
    allow: np.ndarray | None = None
    bias: dict | None = None

    def adjusted(self):
        V = self.row.size
        keep = lambda d: {t: v for t, v in (d or {}).items() if t < V}
        return S.adjusted_logits(self.row, keep(self.pen), self.allow, keep(self.bias))


def segments(V):
    return [(g * SEG, min(V, (g + 1) * SEG)) for g in range(-(-V // SEG))]


def low(rng, V, centre=-10.0):
    return (centre + rng.standard_normal(V)).astype(f32)


def cases_for(V, k, rng):
    segs = segments(V)
    out = [Case("all equal", np.full(V, 0.75, f32))]
    # a block of exact ties straddling rank k, spread over the row (and so over the segments)
    row = (-5.0 - np.abs(rng.standard_normal(V))).astype(f32)
    n_top = k // 2
    pos = rng.choice(V, n_top + (k - n_top + 2), replace=False)
    row[pos[:n_top]] = (10.0 + 10.0 * rng.random(n_top)).astype(f32)
    row[pos[n_top:]] = 1.0
    out.append(Case("ties across rank k", row))
    # the best min(128, segment length) tokens all in one segment
    picks = {"first": 0, "middle": len(segs) // 2}
    full = [g for g, (a, b) in enumerate(segs) if b - a == SEG]
    if full:
        picks["last full"] = full[-1]
    if segs[-1][1] - segs[-1][0] < SEG:
        picks["last partial"] = len(segs) - 1
    for g in sorted(set(picks.values())):
        a, b = segs[g]
        row = low(rng, V)
        n = min(128, b - a)
        row[a + rng.choice(b - a, n, replace=False)] = (5.0 + rng.standard_normal(n)).astype(f32)
        out.append(Case("best in one segment", row))
    # one winner per segment, in a random order of value
    row = low(rng, V)
    for g, (a, b) in enumerate(segs):
        row[a + int(rng.integers(0, b - a))] = f32(10.0 + 0.5 * rng.permutation(len(segs))[g])
    out.append(Case("one winner per segment", row))
    out.append(Case("descending in id", (-np.arange(V) * 1e-3).astype(f32)))
    out.append(Case("ascending in id", (np.arange(V) * 1e-3).astype(f32)))
    # +0.0 beside -0.0 at the top, both orders
    row = (-1.0 - np.abs(rng.standard_normal(V))).astype(f32)
    npair = min(k // 2 + 2, V // 4)
    for i, j in enumerate(np.sort(rng.choice(V // 2 - 1, npair, replace=False)) * 2):
        row[j], row[j + 1] = (f32(-0.0), f32(0.0)) if i % 2 == 0 else (f32(0.0), f32(-0.0))
    out.append(Case("+0.0 beside -0.0", row))
    # a chain of values one ulp apart above 1.0 and one below -3.5, scattered
    row = low(rng, V, -20.0)
    up = [f32(1.0)]
    while len(up) < k + 20:
        up.append(np.nextafter(up[-1], f32(np.inf)))
    down = [f32(-3.5)]
    while len(down) < 20:
        down.append(np.nextafter(down[-1], f32(-np.inf)))
    chain = np.array(up + down, f32)
    row[rng.choice(V, chain.size, replace=False)] = rng.permutation(chain)
    out.append(Case("1 ulp neighbours", row))
    # magnitudes near +-1e38 (|x - max| <= 2e38 stays finite in f32)
    row = rng.uniform(-1e38, 1e38, V).astype(f32)
    row[rng.choice(V, 4, replace=False)] = np.array([1e38, -1e38, 1e38, np.nextafter(f32(1e38), f32(0))], f32)
    out.append(Case("near 1e38", row))
    # -inf entries in the row itself, a whole segment of them where there are several segments
    row = (3.0 * rng.standard_normal(V)).astype(f32)
    row[rng.random(V) < 0.4] = -np.inf
    if len(segs) > 1:
        a, b = segs[len(segs) // 2]
        row[a:b] = -np.inf
    out.append(Case("-inf in the row", row, bias={int(np.flatnonzero(np.isneginf(row))[0]): 50.0}))
    # allowed-token counts around k
    for c in sorted({0, 1, max(k - 1, 0), k, k + 1}):
        allow = np.zeros(V, bool)
        allow[rng.choice(V, c, replace=False)] = True
        out.append(Case("allowed count", (3.0 * rng.standard_normal(V)).astype(f32), allow=allow))
    # lists that create exact ties: x_p - 0.5 == x_q, x_a + 0.5 == x_b
    row = (-5.0 - np.abs(rng.standard_normal(V))).astype(f32)
    pos = rng.choice(V, 24, replace=False)
    pen, bias = {}, {}
    for i in range(6):
        p, q, a, b = (int(x) for x in pos[4 * i:4 * i + 4])
        row[p], row[q] = f32(100.5 - 4 * i), f32(100.0 - 4 * i)
        row[a], row[b] = f32(97.5 - 4 * i), f32(98.0 - 4 * i)
        pen[p], bias[a] = 0.5, 0.5
    out.append(Case("lists make ties", row, pen=pen, bias=bias))
    # lists that break exact ties: groups of six equal values, the lowest id of one group pushed down one ulp, the highest
    # id of another pushed up one ulp, one of the third moved below the others
    row = (-5.0 - np.abs(rng.standard_normal(V))).astype(f32)
    pos = rng.choice(V, 18, replace=False)
    g1, g2, g3 = np.sort(pos[:6]), np.sort(pos[6:12]), np.sort(pos[12:])
    row[g1], row[g2], row[g3] = 50.0, 40.0, 30.0
    out.append(Case("lists break ties", row, pen={int(g1[0]): 2.0 ** -18, int(g3[2]): 10.0}, bias={int(g2[-1]): 2.0 ** -18}))
    # a bias on a masked token leaves it masked
    row = (3.0 * rng.standard_normal(V)).astype(f32)
    a = int(row.argmax())
    allow = np.ones(V, bool)
    allow[[a, (a + 7) % V]] = False
    out.append(Case("bias on a masked token", row, allow=allow, bias={a: 100.0, (a + 7) % V: 1e30, (a + 1) % V: 0.25}))
    # penalty / bias tokens >= num_vocab are ignored
    row = (3.0 * rng.standard_normal(V)).astype(f32)
    out.append(Case("list tokens >= V", row, pen={V: 5.0, V + 1: 1.0, 0x7FFFFFFF: 2.0, 3: 0.3},
                    bias={V + 7: 50.0, 0xFFFFFFFF: 1.0, 5: 0.2}))
    return out


def inject(m, slot, row, state=None):
    """Make `row` the kept row of `slot` (and the slot's state `state`, the initial state by default)."""
    snap = m.state.snapshot_load(m.state.init() if state is None else state, row)
    try:
        m.state.write(snap, slot)
    finally:
        snap.free()


def allow_matrix(cases):
    if all(c.allow is None for c in cases):
        return None
    return np.stack([np.ones(c.row.size, bool) if c.allow is None else c.allow for c in cases])


@pytest.mark.parametrize("top_k", TOP_KS)
@pytest.mark.parametrize("V", VOCABS)
def test_sample_topk_on_constructed_rows(models, V, top_k):
    m = models(V)
    rng = np.random.default_rng([V, top_k])
    cases = cases_for(V, top_k, rng)
    nb = -(-len(cases) // 16)
    cases = cases + cases[:16 * nb - len(cases)]                # whole batches of 16 rows
    for b in range(nb):
        batch = cases[16 * b:16 * (b + 1)]
        slot_of = rng.permutation(16)                           # case i lives in slot slot_of[i]
        for c, s in zip(batch, slot_of):
            inject(m, int(s), c.row)
        order = rng.permutation(16)                             # the call lists case order[j] at position j
        listed = [batch[i] for i in order]
        slots = [int(slot_of[i]) for i in order]
        args = dict(penalties=[c.pen for c in listed], bias=[c.bias for c in listed], allow=allow_matrix(listed))
        ids, p = m.sample_topk(slots, top_k=top_k, **args)
        probs = m.sample_probs(slots, **args)
        for j, c in enumerate(listed):
            tag = f"{c.family}:V{V}/k{top_k}/{j}"
            adj = c.adjusted()
            want = expect_ids(adj, top_k)
            assert np.array_equal(ids[j], want), (tag, ids[j][:8], want[:8])
            p64 = softmax64(adj)
            check_probs(p[j], p64[ids[j]], tag)
            check_probs(probs[j], p64, "sample_probs row:" + tag)
            assert np.array_equal(p[j].view(np.uint32), probs[j][ids[j]].view(np.uint32)), tag
            if c.family == "all equal":
                assert ids[j].tolist() == list(range(top_k)), tag
            if c.family == "allowed count":
                fin = np.isfinite(adj)
                n_fin = min(int(fin.sum()), top_k)
                assert np.all(fin[ids[j][:n_fin]]), tag
                assert ids[j][n_fin:].tolist() == np.flatnonzero(~fin)[:top_k - n_fin].tolist(), tag
                assert not np.any(p[j][n_fin:]), tag
            if c.family == "bias on a masked token":
                assert not np.any(probs[j][~c.allow]), tag
            # the same row alone gives the same bits
            one_ids, one_p = m.sample_topk([slots[j]], top_k=top_k, penalties=[c.pen], bias=[c.bias],
                                           allow=None if c.allow is None else c.allow[None])
            assert np.array_equal(one_ids[0], ids[j]), tag
            assert np.array_equal(one_p[0].view(np.uint32), p[j].view(np.uint32)), tag


# ---- b200rwkv_softmax ----

def softmax_bound(x, p64):
    """Per-element bound of softmax_kernel (module docstring) on row x; meaningful for its finite entries."""
    V = x.size
    k = -(-V // 1024)
    xd = np.asarray(x, np.float64)
    fin = np.isfinite(xd)
    d = np.where(fin, xd.max() - xd, 0.0)
    dmax = min(float(d[fin].max()), 104.0)
    rel = (k + 16 + dmax + d) * U * (1 + 1e-3) + V * 2.0 ** -147
    return p64 * rel + 4 * 2.0 ** -149


def softmax_rows(V, rng):
    neg = (3.0 * rng.standard_normal(V)).astype(f32)
    neg[rng.random(V) < 0.3] = -np.inf
    neg[int(rng.integers(0, V))] = f32(2.0)
    single = np.full(V, -np.inf, f32)
    single[int(rng.integers(0, V))] = f32(7.3)
    return {"-inf entries": neg, "one finite entry": single, "constant": np.full(V, -2.25, f32),
            "spread over 1e4": rng.uniform(-5e3, 5e3, V).astype(f32), "normal": (4.0 * rng.standard_normal(V)).astype(f32)}


@pytest.mark.parametrize("V", [509, 2049, 65536, 70003])
def test_softmax(models, V):
    m = models(V)
    rng = np.random.default_rng(V)
    fams = softmax_rows(V, rng)
    rows, names = list(fams.values()), list(fams)
    while len(rows) < 33:
        for name, r in softmax_rows(V, rng).items():
            rows.append(r)
            names.append(name)
    rows, names = rows[:33], names[:33]
    many = m.softmax(rows)
    for i, (name, x, y) in enumerate(zip(names, rows, many)):
        tag = f"softmax {name}:V{V}/{i}"
        p64 = softmax64(x)
        fin = np.isfinite(x)
        assert np.all(y[~fin] == 0), tag
        lim = softmax_bound(x, p64)[fin]
        err = np.abs(y[fin].astype(np.float64) - p64[fin])
        assert np.all(err <= lim), (tag, float((err - lim).max()))
        _note(f"softmax {name}", (err / lim).max())
        if name == "one finite entry":
            assert y[fin][0] == 1.0 and not np.any(y[~fin]), tag
    for i in range(len(fams)):                                 # one row per call: the same bits as in the 33-row call
        one = m.softmax([rows[i]])[0]
        assert np.array_equal(one.view(np.uint32), many[i].view(np.uint32)), (V, names[i])


# ---- the kept row through every reader ----

def observe(m, slot, want, tag):
    """The slot's kept row as sample_topk, sample_probs and state_read + snapshot_back see it: `want` (bits) or none."""
    if want is None:
        for read in (lambda: m.sample_topk([slot], top_k=8), lambda: m.sample_probs([slot])):
            with pytest.raises(capi.B200Error) as ei:
                read()
            assert ei.value.code == capi.ERR_STATE, tag
        snap = m.state.read(slot)
        try:
            with pytest.raises(capi.B200Error) as ei:
                m.state.snapshot_back(snap, with_logits=True)
            assert ei.value.code == capi.ERR_STATE, tag
        finally:
            snap.free()
        return
    ids, p = m.sample_topk([slot], top_k=8)
    assert np.array_equal(ids[0], expect_ids(want, 8)), tag
    probs = m.sample_probs([slot])[0]
    check_probs(probs, softmax64(want), "lifecycle:" + tag)
    assert np.array_equal(p[0].view(np.uint32), probs[ids[0]].view(np.uint32)), tag
    snap = m.state.read(slot)
    try:
        _, row = m.state.snapshot_back(snap, with_logits=True)
    finally:
        snap.free()
    assert np.array_equal(row.view(np.uint32), want.view(np.uint32)), tag


def observe_score(m, slot, want, tag, token=5):
    """SCORE token 0 on the slot (advances its state: the last reader)."""
    _, sc = m.infer_ex([slot], [1], [token], [capi.OPTION_SCORE])
    s, a = float(sc[0][0][0]), int(sc[0][1][0])
    if want is None:
        assert np.isnan(s) and a == 0xFFFFFFFF, (tag, s, a)
        return
    b = score_bound(want, token)
    err = abs(s - log_softmax64(want)[token])
    assert err <= b, (tag, err, b)
    _note("lifecycle SCORE token 0", err / b)
    assert a == int(np.argmax(want)), tag


def random_rows(V, n, rng):
    return {s: (3.0 * rng.standard_normal(V)).astype(f32) for s in range(n)}


TGT = 3


def op_state_load(m, rng, rows):
    m.state.load(m.state.init(), TGT)
    return {TGT: None}


def op_none_tokens(m, rng, rows):
    m.infer_raw([TGT], [5], rng.integers(0, m.info["num_vocab"], 5).tolist(), [capi.OPTION_NONE])
    return {TGT: None}


def op_none_beside_last(m, rng, rows):
    out = m.infer_raw([TGT, 6], [5, 3], rng.integers(0, m.info["num_vocab"], 8).tolist(), [capi.OPTION_NONE, capi.OPTION_LAST])
    return {TGT: None, 6: out[1][0].copy()}


def op_none_empty(m, rng, rows):
    m.infer_raw([TGT], [0], [], [capi.OPTION_NONE])
    return {}


def op_last_empty(m, rng, rows):
    m.infer_raw([TGT, 5], [0, 0], [], [capi.OPTION_LAST, capi.OPTION_FULL])
    return {}


def op_write_with_row(m, rng, rows):
    new = (5.0 * rng.standard_normal(m.info["num_vocab"])).astype(f32)
    inject(m, TGT, new)
    return {TGT: new}


def op_write_without_row(m, rng, rows):
    snap = m.state.snapshot_load(m.state.init())
    try:
        m.state.write(snap, TGT)
    finally:
        snap.free()
    return {TGT: None}


def op_read_after_none(m, rng, rows):
    """A snapshot taken after a NONE entry carries no row, and writes none."""
    op_none_tokens(m, rng, rows)
    snap = m.state.read(TGT)
    try:
        m.state.write(snap, 5)
    finally:
        snap.free()
    return {TGT: None, 5: None}


def op_prompt_cut_by_the_chunk(m, rng, rows):
    """Runtime.infer on a 20-token Last prompt with a chunk of 8: the first call sends NONE."""
    inp = runtime.RnnInput([runtime.RnnInputBatch([]) for _ in range(TGT)]
                           + [runtime.RnnInputBatch(rng.integers(0, m.info["num_vocab"], 20).tolist())], 8)
    rest, out = m.runtime.infer(inp)
    assert out[TGT].is_empty() and len(rest.batches[TGT].tokens) == 12
    return {TGT: None}


def op_none_then_last(m, rng, rows):
    V = m.info["num_vocab"]
    m.infer_raw([TGT], [6], rng.integers(0, V, 6).tolist(), [capi.OPTION_NONE])
    out = m.infer_raw([TGT], [4], rng.integers(0, V, 4).tolist(), [capi.OPTION_LAST])
    return {TGT: out[0][0].copy()}


OPS = {f.__name__[3:]: f for f in (op_state_load, op_none_tokens, op_none_beside_last, op_none_empty, op_last_empty,
                                   op_write_with_row, op_write_without_row, op_read_after_none, op_prompt_cut_by_the_chunk,
                                   op_none_then_last)}


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("V", [509, 2049])
def test_kept_row_follows_the_state(models, V, op):
    m = models(V, max_batch=8, chunk=8)
    rng = np.random.default_rng([V, len(op)])
    rows = random_rows(V, 8, rng)
    for s, r in rows.items():
        inject(m, s, r)
    want = {**rows, **OPS[op](m, rng, rows)}
    for s in range(8):
        observe(m, s, want[s], f"{op}:V{V}/slot{s}")
    observe_score(m, TGT, want[TGT], f"{op}:V{V}")


@pytest.mark.parametrize("option", ["LAST", "FULL", "SCORE"])
@pytest.mark.parametrize("V", [509, 2049])
def test_kept_row_after_a_call_cut_into_steps(models, V, option):
    """Two entries of 41 and 38 tokens, chunk 8: each slot's kept row is the host copy of its entry's last row, bit for bit.
    Slot 3 (odd) and slot 4 (even): at V = 509 and 2049 the kept row of slot 3 starts 12 bytes past a 16-byte boundary and
    that of slot 4 on one, and the rows of a step start anywhere, so keep_rows_kernel runs all its load / store paths."""
    m = models(V, max_batch=8, chunk=8)
    rng = np.random.default_rng([V, len(option), 7])
    rows = random_rows(V, 8, rng)
    for s, r in rows.items():
        inject(m, s, r)
    slots, ntok = [3, 4], [41, 38]
    toks = rng.integers(0, V, sum(ntok)).tolist()
    opt = {"LAST": capi.OPTION_LAST, "FULL": capi.OPTION_FULL, "SCORE": capi.OPTION_FULL}[option]
    snaps = [m.state.read(s) for s in slots]
    try:
        out = m.infer_raw(slots, ntok, toks, [opt] * 2)
        full = [r.copy() for r in out]
        want = dict(rows)
        want.update({s: full[i][-1].copy() for i, s in enumerate(slots)})
        if option == "SCORE":
            for s, t in zip(slots, snaps):
                m.state.write(t, s)
            res, sc = m.infer_ex(slots, ntok, toks, [capi.OPTION_SCORE] * 2)
            assert [r.shape[0] for r in res] == [0, 0]
            for i, s in enumerate(slots):
                mine = toks[sum(ntok[:i]):sum(ntok[:i + 1])]
                preds = [rows[s]] + list(full[i][:-1])
                for j, (row, t) in enumerate(zip(preds, mine)):
                    b = score_bound(row, t)
                    err = abs(float(sc[i][0][j]) - log_softmax64(row)[t])
                    assert err <= b and int(sc[i][1][j]) == int(np.argmax(row)), (option, V, s, j, err, b)
    finally:
        for t in snaps:
            t.free()
    for s in range(8):
        observe(m, s, want[s], f"{option} cut:V{V}/slot{s}")
    for s in slots:
        observe_score(m, s, want[s], f"{option} cut:V{V}/slot{s}")


# ---- refusal ----

def test_top_k_above_num_vocab_is_refused(models):
    """V = 100 < 128: top_k = V returns the whole row sorted; top_k > V is ERR_INVALID, before any CUDA work."""
    V = 100
    m = models(V, max_batch=2)
    m.state.load(m.state.init(), 0)
    row = m.infer_raw([0], [3], [1, 2, 3], [capi.OPTION_LAST])[0][0].copy()
    ids, p = m.sample_topk([0], top_k=V)
    assert np.array_equal(ids[0], expect_ids(row, V))
    check_probs(p[0], softmax64(row)[ids[0]], f"refusal:V{V}")
    for k in (V + 1, 128):
        with pytest.raises(capi.B200Error) as ei:
            m.sample_topk([0], top_k=k)
        assert ei.value.code == capi.ERR_INVALID, k
        again_ids, again_p = m.sample_topk([0], top_k=V)
        assert np.array_equal(again_ids, ids) and np.array_equal(again_p.view(np.uint32), p.view(np.uint32)), k
