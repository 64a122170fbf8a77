"""SCORE's row kernel (b200rwkv_infer_ex with B200RWKV_OPTION_SCORE, csrc/sample.cuh score_rows_kernel) on constructed rows
at every vocabulary size, against a float64 log-softmax of the f32 row and np.argmax (the first index of the maximum).

Rows are injected as the kept row of a slot (b200rwkv_snapshot_load + b200rwkv_state_write); an infer_ex call with one SCORE
token per slot then scores that token against the slot's row.  Sixteen slots per call, on a tiny6 model whose vocabulary is
overridden.  Every call replaces the kept rows, so they are injected again before each call.  Slot s's kept row starts 4 s V
bytes into the keep buffer: for V % 4 != 0 only the rows of slots s % 4 == 0 are 16-byte aligned, and the kernel reads the
others through its scalar loads.

Thread map: with n4 = V / 4, element i < 4 n4 goes to thread (i / 4) % 256, in increasing i; tail element 4 n4 + j goes to
thread j, last.  For each thread t of a row the test counts k_t, the elements it adds (entries above -inf), and r_t, the
times its running max rises after its first element (the first one sets s = 0 * expf(-inf) + 1 = 1 exactly).

Error bound of one score.  u = 2^-24, M the row maximum, d_j = x_j - M <= 0, S = sum_j exp(d_j) >= 1, w_j = exp(d_j) / S.
  - All partial sums are sums of positive terms, so each rounding of one multiplies each of its terms by the same (1 + e),
    and the computed S~ is sum_j exp(d_j) times the product of the factors on term j's path:
      * the exponents: d_j is the sum of the arguments of the expf calls on the path (x_j - m at its add, m - x at each later
        rise of its thread, m - M at each merge), all <= 0 and each rounded once: a factor within exp(u |d_j|);
      * its own add: expf (2 ulp <= 4u) and the add, or for a rise the exact 1 and the add: 5u;
      * each later rise of its thread: expf, the product and the add, 6u; each later plain add, u: with the own add
        4 + k_t + 5 r_t in all;
      * 10 merge levels (5 xor levels inside each warp, then 5 in warp 0 over the 8 warps' results), each an expf, a product
        and an add on the term's side: 60u.
    A term with d_j < -87 is below 2^-125, the bottom of the f32 normal range; computed, it and any subnormal it passes
    through stay below 2^-123, so such terms move S~ by less than V 2^-123 in all.  The other terms never meet a subnormal
    (their partial sums only grow).  First order, with 1 + 1e-3 for the products of (1 + e) factors (sum |e| < 1e-3):
      |S~ - S| / S <= eps = u (1 + 1e-3) sum_{d_j >= -87} w_j (64 + k_t(j) + 5 r_t(j) + |d_j|) + V 2^-123.
  - logf within 1 ulp <= 2u |log S~|:  |logf(S~) - log S| <= b = e + 2u (log S + e),  e = -log(1 - eps).
  - x_t - M rounded once (u |d_t|) and the final subtraction once (u |result|):
      |score - (d_t - log S)| <= (2 + u) u |d_t| + (1 + u) b + u log S.
This holds at every vocabulary; tests/test_gpu_score.py's headline bound 2^-16 + 2^-22 |x_t - m| covers it only for V <= 2048.
Each family prints its worst error / bound per V; a ratio above 1 fails.

Special values, as the header of b200rwkv_infer_ex states them: a -inf target scores -inf; a target so far below the maximum
that x_t - M overflows f32 scores -inf, the correctly rounded answer; a row of only -inf scores NaN with argmax 0; a NaN
anywhere in the row makes the score NaN, and the argmax is the lowest id of the largest non-NaN entry (UINT32_MAX for a row of
only NaN).
"""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
U = 2.0 ** -24
SCORE_THREADS = 256
SLOTS = 16
VOCABS = [509, 2048, 2049, 4095, 65535, 65536, 70003]
NO_ID = 0xFFFFFFFF
WORST = {}


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(V, exact=False):
        key = (V, exact)
        if key not in cache:
            st = synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], V=V), 0)
            m = runtime.Model(st, max_batch=SLOTS, token_chunk_size=32, exact=exact)
            cache[key] = (m, m.state.init())
        return cache[key]

    yield get
    for m, _ in cache.values():
        m.close()
    if WORST:
        print("\nworst score error / bound:\n  " + "\n  ".join(f"{f} V{V}: {r:.3g}" for (f, V), r in sorted(WORST.items())))


def _note(family, V, ratio):
    WORST[family, V] = max(WORST.get((family, V), 0.0), float(ratio))


# ---- reference and bound ----

def thread_sequences(x):
    """[256, L] float64: thread t's elements in the order it adds them, -inf (no operation) as padding."""
    V = x.size
    n4 = V // 4
    passes = -(-n4 // SCORE_THREADS)
    body = np.full(passes * 4 * SCORE_THREADS, -np.inf)
    body[:4 * n4] = x[:4 * n4]
    seq = body.reshape(passes, SCORE_THREADS, 4).transpose(1, 0, 2).reshape(SCORE_THREADS, 4 * passes)
    tail = np.full((SCORE_THREADS, 1), -np.inf)
    tail[:V & 3, 0] = x[4 * n4:]
    return np.hstack([seq, tail])


@dataclasses.dataclass
class RowStats:
    M: float          # row maximum
    log_s: float      # log sum exp(x - M)
    b: float          # bound on |logf(S~) - log S|


def row_stats(row):
    """The parts of the bound (module docstring) that depend on the whole row; None for a row without a finite maximum."""
    x = np.asarray(row, np.float64)
    M = float(x.max())
    if not np.isfinite(M):
        return None
    V = x.size
    log_s = float(np.log(np.exp(x - M).sum()))
    seq = thread_sequences(x)
    k = (seq > -np.inf).sum(1)
    prev = np.hstack([np.full((SCORE_THREADS, 1), -np.inf), np.maximum.accumulate(seq, axis=1)[:, :-1]])
    r = (seq > prev).sum(1) - (k > 0)
    c = 64 + k + 5 * r
    d = seq - M
    normal = d >= -87.0
    w = np.where(normal, np.exp(np.where(normal, d, 0.0)), 0.0) / np.exp(log_s)
    eps = U * (1 + 1e-3) * float((w * (c[:, None] + np.abs(np.where(normal, d, 0.0)))).sum()) + V * 2.0 ** -123
    e = -np.log1p(-eps)
    return RowStats(M, log_s, e + 2 * U * (log_s + e))


def expect_argmax(row):
    """Lowest id of the largest non-NaN entry (+0.0 == -0.0), UINT32_MAX if every entry is NaN."""
    ok = np.flatnonzero(~np.isnan(row))
    return NO_ID if ok.size == 0 else int(ok[np.argmax(row[ok])])


def check_score(tag, row, stats, t, s, a):
    """One kernel result (score s, argmax a) for target t of `row` against the reference; returns error / bound or None."""
    assert a == expect_argmax(row), (tag, t, a, expect_argmax(row))
    if np.isnan(row).any():
        assert np.isnan(s), (tag, t, s)
        return None
    if stats is None:                                    # only -inf: (-inf - -inf) - logf(0)
        assert np.isnan(s) and a == 0, (tag, t, s, a)
        return None
    with np.errstate(over="ignore"):
        dt32 = np.subtract(row[t], f32(stats.M), dtype=f32)
    if np.isneginf(dt32):                                # a -inf target, or x_t - M below -FLT_MAX
        assert s == -np.inf, (tag, t, s, float(row[t]), stats.M)
        return None
    dt = float(row[t]) - stats.M
    want = dt - stats.log_s
    bound = (2 + U) * U * abs(dt) + (1 + U) * stats.b + U * stats.log_s
    err = abs(float(s) - want)
    assert err <= bound, (tag, t, float(s), want, err, bound)
    return err / bound


# ---- driving the kernel ----

def inject(m, init, slot, row):
    snap = m.state.snapshot_load(init, row)
    try:
        m.state.write(snap, slot)
    finally:
        snap.free()


def score_pairs(m, init, pairs, rng):
    """pairs: [(row, target)] -> [(score, argmax)], 16 per call: pair i in slot slot_of[i], listed at a random position."""
    out = [None] * len(pairs)
    for b in range(0, len(pairs), SLOTS):
        batch = list(range(b, min(b + SLOTS, len(pairs))))
        slot_of = rng.permutation(SLOTS)[:len(batch)]
        for i, s in zip(batch, slot_of):
            inject(m, init, int(s), pairs[i][0])
        order = rng.permutation(len(batch))
        slots = [int(slot_of[j]) for j in order]
        toks = [int(pairs[batch[j]][1]) for j in order]
        _, sc = m.infer_ex(slots, [1] * len(slots), toks, [capi.OPTION_SCORE] * len(slots))
        for pos, j in enumerate(order):
            out[batch[j]] = (sc[pos][0][0], int(sc[pos][1][0]))
    return out


# ---- constructed rows ----

def targets(row, rng, extra=()):
    """The argmax, the minimum, id 0, the last id, a tail id (the last float4 element if V % 4 == 0), three random ids."""
    V = row.size
    n4 = V // 4
    tail = 4 * n4 + (V & 3) // 2 if V & 3 else 4 * n4 - 1
    finite = np.where(np.isnan(row), 0.0, row)
    ts = [int(np.argmax(finite)), int(np.argmin(finite)), 0, V - 1, tail] + rng.integers(0, V, 3).tolist() + list(extra)
    return list(dict.fromkeys(int(t) for t in ts))


def base(rng, V, centre=-10.0, scale=1.0):
    return (centre + scale * rng.standard_normal(V)).astype(f32)


def tie_pairs(V):
    """(family, lower id, higher id): two equal maxima straddling each boundary of the kernel's thread map."""
    n4, tail = V // 4, V & 3
    q = n4 // 2
    last_pass = 402 + 1024 * ((4 * n4 - 1 - 402) // 1024)
    pairs = [("tie inside one float4", 4 * q + 1, 4 * q + 3), ("tie inside one float4", 4 * q, 4 * q + 1),
             ("tie across adjacent threads", 148, 152), ("tie across adjacent threads", 4 * n4 - 8, 4 * n4 - 4),
             ("tie across warps", 284, 412), ("tie across warps", 124, 128),
             ("tie across passes", 402, 1426), ("tie across passes", 402, last_pass),
             ("tie across passes", 1020, 1024)]              # thread 255 of pass 0, thread 0 of pass 1
    if tail:
        pairs += [("tie float4 / tail", 4 * n4 - 1, 4 * n4), ("tie float4 / tail", 5, V - 1),
                  ("tie float4 / tail", 0, 4 * n4 + tail - 1)]
    return [(f, i, j) for f, i, j in pairs if i < j < V]


def constructed_rows(V, rng):
    """[(family, row, targets)]."""
    n4, tail = V // 4, V & 3
    out = []

    def add(family, row, extra=()):
        out.append((family, row, targets(row, rng, extra)))

    add("normal", base(rng, V, 0.0, 3.0))
    asc = np.linspace(-20.0, 8.0, V).astype(f32)
    assert np.all(np.diff(asc) > 0)
    add("ascending (every element rescales)", asc)
    add("descending", asc[::-1].copy())
    add("random order", rng.permutation(asc))
    add("uniform", np.full(V, 0.75, f32))
    add("uniform", np.full(V, -3e4, f32))
    steps = np.array([np.nextafter(f32(0.75), f32(-1)), f32(0.75), np.nextafter(f32(0.75), f32(2))], f32)
    add("uniform 1 ulp", steps[rng.integers(0, 3, V)])
    for family, i, j in tie_pairs(V):
        row = base(rng, V)
        row[[i, j]] = f32(5.0)
        assert expect_argmax(row) == i
        add(family, row, (i, j))
    for i, j in [(3, 4), (9, V - 1)]:
        for lo, hi in [(f32(-0.0), f32(0.0)), (f32(0.0), f32(-0.0))]:
            row = (-1.0 - np.abs(rng.standard_normal(V))).astype(f32)
            row[i], row[j] = lo, hi
            assert expect_argmax(row) == i
            add("tie +0.0 / -0.0", row, (i, j))
    last_g = SCORE_THREADS - 1 + SCORE_THREADS * ((n4 - SCORE_THREADS) // SCORE_THREADS)
    places = {"max at id 0": 0, "max at the last float4": 4 * n4 - 1, "max at the first of the last float4": 4 * n4 - 4,
              "max in the last thread of the last warp": 4 * last_g + 3}
    if tail:
        places["max in the tail"] = V - 1
    for family, p in places.items():
        if 0 <= p < V:
            row = base(rng, V, 0.0, 3.0)
            row[p] = row.max() + f32(2.0)
            add(family, row, (p,))
    row = base(rng, V, -5.0, 2.0)
    row[V // 3] = f32(60.0)
    add("one dominant outlier", row)
    row = base(rng, V, 0.0, 3.0)
    row[rng.random(V) < 0.4] = -np.inf
    row[[1, V - 1]] = -np.inf
    add("-inf entries", row, (1,))
    row = np.full(V, -np.inf, f32)
    row[4 * n4 - 3] = f32(7.3)
    add("one finite entry", row)
    add("only -inf", np.full(V, -np.inf, f32))
    row = rng.uniform(-1e38, 1e38, V).astype(f32)
    big = rng.choice(V, 4, replace=False)
    row[big] = np.array([1e38, -1e38, 1e38, np.nextafter(f32(1e38), f32(0))], f32)
    add("near 1e38", row, tuple(big))
    row = base(rng, V, 0.0, 1.0)
    a, b, c, e = (int(x) for x in rng.choice(V, 4, replace=False))
    row[a], row[b], row[c], row[e] = f32(3e38), f32(-3e38), f32(-1e38), f32(-3e37)
    add("x_t - m overflows", row, (b, c, e))          # 3e38 - (-3e37) = 3.3e38 stays finite
    return out


@pytest.mark.parametrize("V", VOCABS)
def test_constructed_rows(models, V):
    """Every family of `constructed_rows`, each row scored at its targets, 16 rows per call in shuffled slots."""
    m, init = models(V)
    rng = np.random.default_rng([V, 1])
    rows = constructed_rows(V, rng)
    pairs = [(row, t) for _, row, ts in rows for t in ts]
    got = score_pairs(m, init, pairs, rng)
    results = iter(got)
    for family, row, ts in rows:
        stats = row_stats(row)
        for t in ts:
            s, a = next(results)
            ratio = check_score(f"{family}:V{V}", row, stats, t, s, a)
            if ratio is not None:
                _note(family, V, ratio)
            if family == "one finite entry" and t == a:
                assert s == 0.0, (V, t, s)                   # 0 - logf(1)


@pytest.mark.parametrize("V", VOCABS)
def test_nan_reaches_the_score(models, V):
    """A NaN anywhere in the row makes the score NaN; the argmax skips it.  Rows without NaN scored in the same call keep
    their bits."""
    m, init = models(V)
    rng = np.random.default_rng([V, 2])
    nan_pairs = []
    for at in (0, V // 2, V - 1):                            # V - 1: in the tail when V % 4 != 0
        row = base(rng, V, 0.0, 3.0)
        row[at] = np.nan
        nan_pairs += [(row, t) for t in targets(row, rng)]
        nan_pairs.append((row, at))                          # the NaN is the target
    row = base(rng, V, 0.0, 3.0)
    t = int(np.argmax(row))
    row[t + 1 if t + 1 < V else t - 1] = np.nan               # beside the maximum
    nan_pairs.append((row, t))
    row = np.full(V, np.nan, f32)                            # only NaN: UINT32_MAX
    nan_pairs += [(row, 0), (row, V - 1)]
    row = np.full(V, -np.inf, f32)                           # NaN and -inf only: the argmax is the first -inf
    row[rng.random(V) < 0.5] = np.nan
    row[0] = np.nan
    nan_pairs += [(row, 0), (row, int(np.flatnonzero(~np.isnan(row))[0]))]
    clean = [(base(rng, V, 0.0, 3.0), 0), (np.linspace(-20.0, 8.0, V).astype(f32), V - 1)]
    pairs = nan_pairs[:SLOTS - 2] + clean + nan_pairs[SLOTS - 2:]        # the first call: 14 NaN rows and the clean two
    got = score_pairs(m, init, pairs, rng)
    for (r, t), (s, a) in zip(pairs, got):
        check_score(f"NaN:V{V}", r, row_stats(r), t, s, a)
    # the clean rows alone in a call: the same bits as beside the NaN rows
    alone = score_pairs(m, init, clean, rng)
    for (s0, a0), (s1, a1) in zip(alone, got[SLOTS - 2:SLOTS]):
        assert f32(s0).view(np.uint32) == f32(s1).view(np.uint32) and a0 == a1, V


@pytest.mark.parametrize("V", VOCABS)
def test_result_does_not_depend_on_slot_or_neighbours(models, V):
    """One row in all 16 slots (for V % 4 != 0, 4 read through float4 loads and 12 through scalar loads), listed in a random
    order; then in slots 0 and 1 alone among other rows, listed first and last: the same score and argmax bits everywhere."""
    m, init = models(V)
    rng = np.random.default_rng([V, 3])
    tie = base(rng, V)
    tie[[148, 152]] = f32(5.0)
    inf = base(rng, V, 0.0, 3.0)
    inf[rng.random(V) < 0.3] = -np.inf
    for name, row in [("normal", base(rng, V, 0.0, 3.0)), ("ascending", np.linspace(-20.0, 8.0, V).astype(f32)),
                      ("tie", tie), ("-inf entries", inf)]:
        t = int(rng.integers(0, V))
        for s in range(SLOTS):
            inject(m, init, s, row)
        order = rng.permutation(SLOTS).tolist()
        _, sc = m.infer_ex(order, [1] * SLOTS, [t] * SLOTS, [capi.OPTION_SCORE] * SLOTS)
        bits = {(int(f32(x[0][0]).view(np.uint32)), int(x[1][0])) for x in sc}
        assert len(bits) == 1, (name, V, bits)
        check_score(f"{name}:V{V}", row, row_stats(row), t, sc[0][0][0], int(sc[0][1][0]))
        for s in range(2, SLOTS):
            inject(m, init, s, base(rng, V, 0.0, 3.0))
        for s in (0, 1):
            inject(m, init, s, row)
        others = list(range(2, SLOTS))
        slots = [0] + others + [1]
        toks = [t] + rng.integers(0, V, len(others)).tolist() + [t]
        _, sc = m.infer_ex(slots, [1] * SLOTS, toks, [capi.OPTION_SCORE] * SLOTS)
        for j in (0, SLOTS - 1):
            assert (int(f32(sc[j][0][0]).view(np.uint32)), int(sc[j][1][0])) in bits, (name, V, j)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("V", [65536, 70003])
def test_scores_match_the_full_rows(models, V, precision):
    """20 tokens scored in one step, against the float64 log-softmax of the FULL rows of the same call.  The rows come from
    the step's logits (unaligned rows for V % 4 != 0) and, for token 0, from the kept row."""
    m, init = models(V, exact=precision == 1)
    rng = np.random.default_rng([V, precision])
    m.state.load(init, 0)
    m.infer_raw([0], [3], rng.integers(1, V, 3).tolist(), [capi.OPTION_LAST], keep_on_device=True)
    snap = m.state.read(0)
    try:
        _, kept0 = m.state.snapshot_back(snap, with_logits=True)
        toks = rng.integers(0, V, 20).tolist()
        m.state.write(snap, 0)
        full = m.infer_raw([0], [len(toks)], toks, [capi.OPTION_FULL])[0].copy()
        m.state.write(snap, 0)
        rows, sc = m.infer_ex([0], [len(toks)], toks, [capi.OPTION_SCORE])
    finally:
        snap.free()
    assert rows[0].shape[0] == 0
    for j, (row, t) in enumerate(zip([kept0] + list(full[:-1]), toks)):
        ratio = check_score(f"in-step p{precision}:V{V}/{j}", row, row_stats(row), t, sc[0][0][j], int(sc[0][1][j]))
        _note(f"in-step rows p{precision}", V, ratio)
