"""Top-n log-probabilities of every scored row (b200rwkv_score_top / b200rwkv_last_score_top, csrc/sample.cuh
score_top_segment_kernel + score_top_merge_kernel).

Constructed rows are injected as the kept row of a slot (b200rwkv_snapshot_load + b200rwkv_state_write), as
test_gpu_score_rows.py does; an infer_ex call with one SCORE token per slot then lists that row's best entries.  Checks:
  - ids: exactly the non-NaN ids ordered by (logit descending, id ascending), np.lexsort((ids, -row)), then UINT32_MAX;
  - the target's entry, when listed, is bit-identical to score_out; ids[:, 0] == argmax_out when the row's maximum is finite;
  - every other logprob is within the bound below of the float64 log-softmax of the f32 row;
  - special values: a row with a NaN gives NaN logprobs with its ids still ranked; -inf entries follow the finite ones by
    ascending id; slots past the non-NaN entries and tokens with no row are UINT32_MAX / NaN.

Bound.  The logprob of entry i is (x_i - m) - logf(S~) with score_rows_kernel's m and S~, so the derivation in
test_gpu_score_rows.py applies with the target replaced by i.  Coarsened to what a row's size gives: a thread adds at most
k = 4 ceil(V / 1024) + 1 elements and its running max rises at most k times, and only terms with |d_j| <= 87 count, so
  eps = u (1 + 1e-3) (64 + 6 k + 87) + V 2^-123,  b = -log(1 - eps) + 2u (log S + e),
  |lp_i - (d_i - log S)| <= (2 + u) u |d_i| + (1 + u) b + u log S.

Through real engines (tiny5/6/7, small6, FP8 layers) the lists of a SCORE entry match the FULL rows of a twin slot fed the
same tokens in the same call; infer_snapshots leaves them unchanged; a batch-invariant engine gives the same bits under any
chunking, call cut or mix; and with the setting off an engine's outputs and launch counts equal those of one that never set
it."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
U = 2.0 ** -24
SLOTS = 16
NO_ID = 0xFFFFFFFF
VOCABS = [509, 2048, 2049, 4095, 65535, 65536]
TOP_NS = [1, 5, 20, 128]


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(V):
        if V not in cache:
            st = synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], V=V), 0)
            m = runtime.Model(st, max_batch=SLOTS, token_chunk_size=32)
            cache[V] = (m, m.state.init())
        return cache[V]

    yield get
    for m, _ in cache.values():
        m.close()


def inject(m, init, slot, row):
    snap = m.state.snapshot_load(init, row)
    try:
        m.state.write(snap, slot)
    finally:
        snap.free()


def run_rows(m, init, pairs, n, rng):
    """pairs: [(row, target)] -> [(score, argmax, ids [n], logprobs [n])], 16 per call in shuffled slots."""
    out = [None] * len(pairs)
    for b in range(0, len(pairs), SLOTS):
        batch = list(range(b, min(b + SLOTS, len(pairs))))
        slot_of = rng.permutation(SLOTS)[:len(batch)]
        for i, s in zip(batch, slot_of):
            inject(m, init, int(s), pairs[i][0])
        order = rng.permutation(len(batch))
        slots = [int(slot_of[j]) for j in order]
        toks = [int(pairs[batch[j]][1]) for j in order]
        _, sc, tops = m.infer_ex(slots, [1] * len(slots), toks, [capi.OPTION_SCORE] * len(slots), top_n=n)
        for pos, j in enumerate(order):
            out[batch[j]] = (sc[pos][0][0], int(sc[pos][1][0]), tops[pos][0][0], tops[pos][1][0])
    return out


def expect_ids(row, n):
    ok = np.flatnonzero(~np.isnan(row))
    order = ok[np.lexsort((ok, -row[ok].astype(np.float64)))]
    ids = np.full(n, NO_ID, np.uint32)
    ids[:min(n, order.size)] = order[:n]
    return ids


def check(tag, row, t, s, a, ids, lp):
    """One row's list against the reference; returns the worst error / bound over its finite entries (0 if none)."""
    n = ids.size
    want = expect_ids(row, n)
    assert np.array_equal(ids, want), (tag, ids[:8], want[:8])
    listed = ids != NO_ID
    assert np.all(np.isnan(lp[~listed])), tag
    if np.isnan(row).any():
        assert np.all(np.isnan(lp)), tag
        return 0.0
    hit = np.flatnonzero(ids == t)
    if hit.size:
        assert f32(lp[hit[0]]).view(np.uint32) == f32(s).view(np.uint32), (tag, t, lp[hit[0]], s)
    x = row.astype(np.float64)
    M = float(x.max())
    if not np.isfinite(M):                                   # only -inf: every logprob NaN, as the score
        assert np.all(np.isnan(lp)), tag
        return 0.0
    assert ids[0] == a, (tag, ids[0], a)
    V = row.size
    log_s = float(np.log(np.exp(x - M).sum()))
    k = 4 * -(-V // 1024) + 1
    eps = U * (1 + 1e-3) * (64 + 6 * k + 87) + V * 2.0 ** -123
    e = -np.log1p(-eps)
    b = e + 2 * U * (log_s + e)
    worst = 0.0
    for r in np.flatnonzero(listed):
        xi = float(row[ids[r]])
        if xi == -np.inf:
            assert lp[r] == -np.inf, (tag, r)
            continue
        d = xi - M
        bound = (2 + U) * U * abs(d) + (1 + U) * b + U * log_s
        err = abs(float(lp[r]) - (d - log_s))
        assert err <= bound, (tag, r, float(lp[r]), d - log_s, err, bound)
        worst = max(worst, err / bound)
    return worst


def base(rng, V, centre=0.0, scale=3.0):
    return (centre + scale * rng.standard_normal(V)).astype(f32)


def constructed_rows(V, n, rng):
    """[(family, row, target)]."""
    out = []
    row = base(rng, V)
    out += [("normal", row, int(np.argmax(row))), ("normal", row, int(rng.integers(0, V)))]
    # ties across rank n: n + 3 equal values straddling the cut, at ids spread over every segment
    row = base(rng, V, -10.0, 1.0)
    tie = rng.choice(V, min(V, n + 3), replace=False)
    row[tie] = f32(4.0)
    row[tie[:max(0, n - 2)]] = f32(5.0)
    out.append(("ties across rank n", row, int(tie[-1])))
    # equal maxima in different 2048-element segments, the higher id listed first in memory order of candidates
    row = base(rng, V, -10.0, 1.0)
    at = [V - 1, V // 2, 2047 if V > 2047 else V // 3, 0]
    row[at] = f32(6.0)
    out.append(("ties across segments", row, V - 1))
    # +0.0 / -0.0 and 1-ulp neighbours as the top entries
    row = (-1.0 - np.abs(rng.standard_normal(V))).astype(f32)
    zs = rng.choice(V, 6, replace=False)
    row[zs[:3]] = f32(0.0)
    row[zs[3:]] = f32(-0.0)
    one = f32(1.0)
    nb = rng.choice(np.setdiff1d(np.arange(V), zs), 3, replace=False)
    row[nb] = [np.nextafter(one, f32(0)), one, np.nextafter(one, f32(2))]
    out.append(("+-0.0 and 1-ulp neighbours", row, int(zs[4])))
    steps = np.array([np.nextafter(f32(0.75), f32(-1)), f32(0.75), np.nextafter(f32(0.75), f32(2))], f32)
    out.append(("uniform 1 ulp", steps[rng.integers(0, 3, V)], 0))
    out.append(("all equal", np.full(V, 0.75, f32), V - 1))
    # -inf entries: most of the row, so some lists reach them
    row = base(rng, V)
    row[rng.random(V) < 0.97] = -np.inf
    out.append(("-inf entries", row, int(np.flatnonzero(row == -np.inf)[0])))
    row = np.full(V, -np.inf, f32)
    row[[3, V - 2]] = f32(1.5)
    out.append(("two finite entries", row, 3))
    out.append(("all -inf", np.full(V, -np.inf, f32), 0))
    # NaN entries: ranked around, logprobs NaN
    row = base(rng, V)
    row[[0, V // 2, V - 1]] = np.nan
    out.append(("NaN entries", row, 1))
    row = np.full(V, np.nan, f32)
    row[rng.choice(V, 3, replace=False)] = [f32(2.0), -np.inf, f32(-1.0)]
    out.append(("NaN with 3 non-NaN", row, 0))
    out.append(("all NaN", np.full(V, np.nan, f32), 0))
    return out


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("n", TOP_NS)
def test_constructed_rows(models, V, n):
    m, init = models(V)
    rng = np.random.default_rng([V, n])
    rows = constructed_rows(V, n, rng)
    got = run_rows(m, init, [(r, t) for _, r, t in rows], n, rng)
    worst = 0.0
    for (family, row, t), (s, a, ids, lp) in zip(rows, got):
        worst = max(worst, check(f"{family}:V{V}:n{n}", row, t, s, a, ids, lp))
    print(f"V{V} n{n}: worst logprob error / bound {worst:.3g}")


def test_no_row_and_setting_off(models):
    """A SCORE token with no row (the slot has no kept row) lists UINT32_MAX / NaN; last_score_top after a call with the
    setting off is ERR_STATE; a small buffer is ERR_INVALID."""
    m, init = models(509)
    m.state.load(init, 0)
    _, sc, tops = m.infer_ex([0], [3], [5, 6, 7], [capi.OPTION_SCORE], top_n=5)
    ids, lp = tops[0]
    assert ids.shape == (3, 5) and np.all(ids[0] == NO_ID) and np.all(np.isnan(lp[0]))
    assert np.all(ids[1:] != NO_ID) and ids[1, 0] == sc[0][1][1]
    L = capi.lib()
    small = np.zeros(14, np.uint32)
    assert L.b200rwkv_last_score_top(m._h, capi.ptr(small), capi.ptr(small.view(np.float32)), 14) == capi.ERR_INVALID
    assert m._top_n == 0
    m.infer_ex([0], [1], [5], [capi.OPTION_SCORE])
    assert L.b200rwkv_last_score_top(m._h, None, None, 0) == capi.ERR_STATE


def test_refusals_that_need_an_engine():
    st = synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], V=65537), 0)
    m = runtime.Model(st, max_batch=2, token_chunk_size=32)
    try:
        assert capi.lib().b200rwkv_score_top(m._h, 5) == capi.ERR_UNSUPPORTED
        assert capi.lib().b200rwkv_score_top(m._h, 0) == capi.OK
        assert capi.lib().b200rwkv_score_top(m._h, 129) == capi.ERR_INVALID
    finally:
        m.close()


# ---- real engines ----

ENGINES = {
    "tiny5": ("tiny5", {}), "tiny6": ("tiny6", {}), "tiny7": ("tiny7", {}), "small6": ("small6", {}),
    "tiny6-fp8": ("tiny6", {"quant": 2, "quant_type": "FP8"}),
}


def host_lists(rows, n):
    """(ids, float64 log-softmax at those ids) of each f32 row."""
    ids = np.stack([expect_ids(r, n) for r in rows])
    x = rows.astype(np.float64)
    M = x.max(1, keepdims=True)
    ls = x - M - np.log(np.exp(x - M).sum(1, keepdims=True))
    return ids, np.take_along_axis(ls, ids.astype(np.int64), 1)


@pytest.mark.parametrize("name", list(ENGINES))
def test_engine_lists_match_full_rows_of_a_twin(name):
    """Slot 0 (SCORE) and slot 1 (FULL) start from the same state and kept row and are fed the same tokens in one call: the
    lists of slot 0 are the lexsort of slot 1's rows (the kept row for token 0), target entries equal the scores."""
    preset, kw = ENGINES[name]
    m = runtime.Model(synth.make_st(preset, 0), max_batch=4, token_chunk_size=32, **kw)
    try:
        rng = np.random.default_rng(7)
        V = m.info["num_vocab"]
        prefix = rng.integers(0, V, 5).tolist()
        toks = rng.integers(0, V, 40).tolist()
        n = 20
        for s in (0, 1):
            m.state.load(m.state.init(), s)
        kept = m.infer_raw([0, 1], [5, 5], prefix + prefix, [capi.OPTION_LAST] * 2)
        rows, sc, tops = m.infer_ex([0, 1], [40, 40], toks + toks, [capi.OPTION_SCORE, capi.OPTION_FULL], top_n=n)
        full = np.vstack([kept[1], rows[1][:-1]])
        ids, lp = tops[0]
        want_ids, want_lp = host_lists(full, n)
        assert np.array_equal(ids, want_ids), name
        assert np.all(np.abs(lp - want_lp) <= 1e-5 * (1 + np.abs(want_lp))), name
        assert np.array_equal(ids[:, 0], sc[0][1]), name
        for j, t in enumerate(toks):
            hit = np.flatnonzero(ids[j] == t)
            if hit.size:
                assert lp[j, hit[0]].view(np.uint32) == sc[0][0][j].view(np.uint32), (name, j)
    finally:
        m.close()


def test_snapshots_leave_the_lists_unchanged():
    m = runtime.Model(synth.make_st("tiny6", 0), max_batch=4, token_chunk_size=32)
    try:
        rng = np.random.default_rng(3)
        toks = rng.integers(0, 512, 30).tolist()
        m.score_top(8)
        outs = []
        for snap in (False, True):
            m.state.load(m.state.init(), 0)
            m.infer_raw([0], [2], [1, 2], [capi.OPTION_LAST])
            if snap:
                _, sc, snaps = m.infer_snapshots([0], [30], toks, [capi.OPTION_SCORE], [(0, 7), (0, 30)])
                for s in snaps:
                    s.free()
            else:
                _, sc = m.infer_ex([0], [30], toks, [capi.OPTION_SCORE])
            outs.append(m.last_score_top())
        assert np.array_equal(outs[0][0], outs[1][0])
        assert np.array_equal(outs[0][1].view(np.uint32), outs[1][1].view(np.uint32))
    finally:
        m.close()


def test_batch_invariant_lists_across_cuts_and_mixes():
    """One 100-token SCORE entry on a batch-invariant engine, whole at chunk 128, at chunk 16 beside LAST / FULL / NONE
    neighbours, and cut into three calls: bit-identical lists."""
    st = synth.make_st("tiny6", 0)
    rng = np.random.default_rng(11)
    toks = rng.integers(0, 512, 100).tolist()
    other = rng.integers(0, 512, 37).tolist()
    results = []
    for chunk, cuts, mix in ((128, [100], False), (16, [100], True), (32, [13, 50, 37], True)):
        m = runtime.Model(st, max_batch=4, token_chunk_size=chunk, batch_invariant=True)
        try:
            m.score_top(20)
            for s in range(4):
                m.state.load(m.state.init(), s)
            m.infer_raw([0], [3], [4, 5, 6], [capi.OPTION_LAST])
            ids, lps, p = [], [], 0
            for c in cuts:
                part = toks[p:p + c]
                if mix:
                    slots = [1, 0, 2, 3]
                    ntok = [len(other), c, 9, 4]
                    opts = [capi.OPTION_FULL, capi.OPTION_SCORE, capi.OPTION_NONE, capi.OPTION_LAST]
                    m.infer_ex(slots, ntok, other + part + other[:9] + other[:4], opts)
                else:
                    m.infer_ex([0], [c], part, [capi.OPTION_SCORE])
                i, l = m.last_score_top()
                ids.append(i)
                lps.append(l)
                p += c
            results.append((np.vstack(ids), np.vstack(lps)))
        finally:
            m.close()
    for ids, lp in results[1:]:
        assert np.array_equal(ids, results[0][0])
        assert np.array_equal(lp.view(np.uint32), results[0][1].view(np.uint32))


def test_setting_off_is_the_engine_that_never_set_it():
    """An engine that turned score_top on and off again: same logits rows, scores, argmax ids and launch counts as an
    engine that never set it; with the setting on the launch count is unchanged too (the top launches ride beside SCORE)."""
    st = synth.make_st("tiny6", 0)
    rng = np.random.default_rng(5)
    toks = rng.integers(0, 512, 60).tolist()
    outs = []
    for toggle in (False, True):
        m = runtime.Model(st, max_batch=4, token_chunk_size=32)
        try:
            if toggle:
                m.score_top(16)
                m.infer_ex([2], [3], [1, 2, 3], [capi.OPTION_SCORE])
                m.score_top(0)
            for s in range(3):
                m.state.load(m.state.init(), s)
            n0 = m.launch_count()
            rows, sc = m.infer_ex([0, 1, 2], [20, 20, 20], toks,
                                  [capi.OPTION_FULL, capi.OPTION_SCORE, capi.OPTION_LAST])
            outs.append((rows, sc, m.launch_count() - n0))
            assert capi.lib().b200rwkv_last_score_top(m._h, None, None, 0) == capi.ERR_STATE
        finally:
            m.close()
    (r0, s0, n0), (r1, s1, n1) = outs
    assert n0 == n1
    for a, b in zip(r0, r1):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(s0[1][0].view(np.uint32), s1[1][0].view(np.uint32)) and np.array_equal(s0[1][1], s1[1][1])
