"""Scoring on the GPU (b200rwkv_infer_ex with B200RWKV_OPTION_SCORE, csrc/sample.cuh score_rows_kernel): per-token
log-probabilities and argmax ids of a known continuation, against a float64 log-softmax of the engine's own FULL rows, with
the state and the kept row bit-identical to FULL, through every cut and mixed batch the shim sends, and the reference's
perplexity() (run.rs:699-755) against the oracle's logits.

Error bound of one score (derived in `score_bound`): the kernel computes (x_t - m) - logf(S), S = sum expf(x - m) >= 1.
  - every term of S: expf within 2 ulp, and each online rescale of a thread's partial sum one more expf (2 ulp) and one
    product rounding; at most k rescales for the k elements a thread reads;
  - the f32 sum: k sequential adds per thread, then 5 + 3 levels of the fixed combine tree (32 lanes, 8 warps), each
    level one rounding of a sum of positive terms;
  - logf within 1 ulp of log S (<= log V), x_t - m rounded once, the final subtraction rounded once.
With u = 2^-24:  |err| <= (4 + 5k + k + 8) u + 2u log V + u (|x_t - m| + log V) + u |x_t - m|.  For the vocabularies here
(V <= 2048, k <= 8) that is below 2^-16 + 2^-22 |x_t - m|, the bound the tests assert and report ratios against.
tests/test_gpu_score_rows.py derives the bound per row from the kernel's thread map, with the rounding of every expf argument
counted as well, for every vocabulary (65536 and above included) and for rows built to hit the kernel's edges; at V <= 2048 it
stays inside this headline.
"""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SCORE_THREADS = 256
WORST = {}


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(preset, max_batch=4, chunk=32, exact=False, **over):
        key = (preset, max_batch, chunk, exact, tuple(sorted(over.items())))
        if key not in cache:
            shp = synth.PRESETS[preset] if not over else dataclasses.replace(synth.PRESETS[preset], **over)
            st = synth.make_st(shp, 0)
            cache[key] = (runtime.Model(st, max_batch=max_batch, token_chunk_size=chunk, exact=exact), st)
        return cache[key]

    yield get
    for m, _ in cache.values():
        m.close()
    if WORST:
        print("\nworst score error / (2^-16 + 2^-22 |x_t - m|): " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def log_softmax64(row):
    x = np.asarray(row, np.float64)
    m = x.max()
    return x - m - np.log(np.exp(x - m).sum())


def score_bound(row, t):
    """Derived bound (module docstring) and the headline bound 2^-16 + 2^-22 |x_t - m| it must stay inside."""
    V = row.size
    k = -(-V // (4 * SCORE_THREADS)) * 4 + 1          # elements one thread reads: float4 groups + the scalar tail
    d = abs(float(row[t]) - float(row.max()))
    derived = (4 + 6 * k + 8) * U + 3 * U * np.log(V) + 2 * U * d
    headline = 2.0 ** -16 + 2.0 ** -22 * d
    assert derived <= headline
    return headline


def check_scores(tag, scores, argmax, rows, targets):
    """scores[j] / argmax[j] against row j of `rows` and token targets[j]."""
    worst = 0.0
    for j, (s, a, row, t) in enumerate(zip(scores, argmax, rows, targets)):
        want = log_softmax64(row)[t]
        b = score_bound(row, t)
        err = abs(float(s) - want)
        assert err <= b, (tag, j, float(s), want, err, b)
        worst = max(worst, err / b)
        assert int(a) == int(np.argmax(row)), (tag, j)          # np.argmax: first (lowest) id of the maximum
    WORST[tag.split(":")[0]] = max(WORST.get(tag.split(":")[0], 0.0), worst)
    return worst


def primed_snapshot(m, slot, rng):
    """A state with a kept row: a few LAST tokens from the initial state."""
    m.state.load(m.state.init(), slot)
    m.infer_raw([slot], [3], rng.integers(1, m.info["num_vocab"], 3).tolist(), [capi.OPTION_LAST], keep_on_device=True)
    return m.state.read(slot)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_scores_match_the_full_rows(models, preset, precision):
    m, _ = models(preset, exact=precision == 1)
    rng = np.random.default_rng(3)
    snap = primed_snapshot(m, 0, rng)
    _, kept0 = m.state.snapshot_back(snap, with_logits=True)
    toks = rng.integers(0, m.info["num_vocab"], 20).tolist()
    m.state.write(snap, 0)
    full = m.infer_raw([0], [len(toks)], toks, [capi.OPTION_FULL])[0].copy()
    state_full = m.state.back(0)
    s_full = m.state.read(0)
    _, kept_full = m.state.snapshot_back(s_full, with_logits=True)
    m.state.write(snap, 0)
    rows, sc = m.infer_ex([0], [len(toks)], toks, [capi.OPTION_SCORE])
    assert rows[0].shape[0] == 0
    scores, argmax = sc[0]
    check_scores(f"{preset}/p{precision}", scores, argmax, [kept0] + list(full[:-1]), toks)
    assert np.array_equal(m.state.back(0), state_full)
    s_score = m.state.read(0)
    _, kept_score = m.state.snapshot_back(s_score, with_logits=True)
    assert np.array_equal(kept_score, kept_full) and np.array_equal(kept_full, full[-1])
    # a forced tie in the kept row: the lower id wins
    tie = kept0.copy()
    hi = float(tie.max()) + 1.0
    tie[[37, 11]] = hi
    snap_tie = m.state.snapshot_load(m.state.back(0), tie)
    m.state.write(snap_tie, 1)
    _, sc = m.infer_ex([1], [2], [37, 5], [capi.OPTION_SCORE])
    assert int(sc[0][1][0]) == 11
    check_scores(f"{preset}/p{precision}:tie", sc[0][0][:1], sc[0][1][:1], [tie], [37])
    for s in (snap, s_full, s_score, snap_tie):
        s.free()


def test_first_token_comes_from_the_kept_row(models):
    m, _ = models("tiny6")
    rng = np.random.default_rng(4)
    row = (rng.standard_normal(m.info["num_vocab"]) * 5).astype(np.float32)
    state = m.state.init()
    with_row = m.state.snapshot_load(state, row)
    m.state.write(with_row, 2)
    _, sc = m.infer_ex([2], [3], [9, 4, 1], [capi.OPTION_SCORE])
    check_scores("tiny6:first", sc[0][0][:1], sc[0][1][:1], [row], [9])
    # a slot whose state came without a row: NaN and UINT32_MAX for token 0, ordinary scores after it
    no_row = m.state.snapshot_load(state)
    m.state.write(no_row, 3)
    _, sc = m.infer_ex([3], [3], [9, 4, 1], [capi.OPTION_SCORE])
    assert np.isnan(sc[0][0][0]) and int(sc[0][1][0]) == 0xFFFFFFFF
    assert np.isfinite(sc[0][0][1:]).all()
    with_row.free(); no_row.free()


@pytest.mark.parametrize("chunk", [8, 32])
def test_cuts(models, chunk):
    """45 tokens in one call (six or two internal steps) against FULL rows of the same cut; the same continuation split over
    two calls chains through the kept row; different cuts agree within what their logits differ by."""
    m, _ = models("tiny6", chunk=chunk)
    rng = np.random.default_rng(5)
    toks = rng.integers(1, 500, 45).tolist()
    snap = primed_snapshot(m, 0, rng)
    _, kept0 = m.state.snapshot_back(snap, with_logits=True)
    m.state.write(snap, 0)
    full = m.infer_raw([0], [45], toks, [capi.OPTION_FULL])[0].copy()
    m.state.write(snap, 0)
    _, sc = m.infer_ex([0], [45], toks, [capi.OPTION_SCORE])
    one_call = sc[0][0].copy()
    check_scores(f"tiny6/chunk{chunk}", one_call, sc[0][1], [kept0] + list(full[:-1]), toks)
    # split 20 + 25: the second call's token 0 is scored from the first call's last row
    m.state.write(snap, 0)
    _, a = m.infer_ex([0], [20], toks[:20], [capi.OPTION_SCORE])
    mid = m.state.read(0)
    _, kept_mid = m.state.snapshot_back(mid, with_logits=True)
    _, b = m.infer_ex([0], [25], toks[20:], [capi.OPTION_SCORE])
    check_scores(f"tiny6/chunk{chunk}:chain", b[0][0][:1], b[0][1][:1], [kept_mid], toks[20:21])
    split = np.concatenate([a[0][0], b[0][0]])
    # the split cut's rows, to measure how far the two cuts' logits are apart
    m.state.write(snap, 0)
    rows_a = m.infer_raw([0], [20], toks[:20], [capi.OPTION_FULL])[0].copy()
    rows_b = m.infer_raw([0], [25], toks[20:], [capi.OPTION_FULL])[0].copy()
    split_rows = np.concatenate([rows_a, rows_b])
    delta = float(np.abs(split_rows - full).max())
    assert delta <= 5e-4 * float(np.abs(full).max())
    # log-softmax moves by at most 2 max|dx|; plus each side's own rounding bound
    lim = 2 * delta + 2 * max(score_bound(r, t) for r, t in zip([kept0] + list(full[:-1]), toks))
    assert float(np.abs(split - one_call).max()) <= lim
    snap.free(); mid.free()


def test_mixed_batch(models):
    """SCORE / LAST / FULL / NONE in one call with ragged counts over interleaved steps (chunk 8).  The same call with the
    SCORE entry as FULL packs the steps identically: every other entry's rows and rows_out, and all states, are
    bit-identical; the SCORE entry's scores match its FULL rows, and do not change when the other entries' tokens do."""
    m, _ = models("tiny6", chunk=8)
    rng = np.random.default_rng(6)
    counts = [13, 5, 9, 7]
    toks = [rng.integers(1, 500, n).tolist() for n in counts]
    snaps = [primed_snapshot(m, s, rng) for s in range(4)]
    _, kept0 = m.state.snapshot_back(snaps[0], with_logits=True)

    def run(options, tok_lists):
        for s in range(4):
            m.state.write(snaps[s], s)
        rows, sc = m.infer_ex([0, 1, 2, 3], counts, sum(tok_lists, []), options)
        return [r.copy() for r in rows], sc, [m.state.back(s) for s in range(4)]

    opts = [capi.OPTION_SCORE, capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE]
    rows, sc, states = run(opts, toks)
    rows_f, _, states_f = run([capi.OPTION_FULL] + opts[1:], toks)
    assert [r.shape[0] for r in rows] == [0, 1, 9, 0] and [r.shape[0] for r in rows_f] == [13, 1, 9, 0]
    assert np.array_equal(rows[1], rows_f[1]) and np.array_equal(rows[2], rows_f[2])
    for a, b in zip(states, states_f):
        assert np.array_equal(a, b)
    assert sc[1] is None and sc[2] is None and sc[3] is None
    check_scores("tiny6:mixed", sc[0][0], sc[0][1], [kept0] + list(rows_f[0][:-1]), toks[0])
    other = [toks[0]] + [rng.integers(1, 500, n).tolist() for n in counts[1:]]
    _, sc2, _ = run(opts, other)
    assert np.array_equal(sc[0][0], sc2[0][0]) and np.array_equal(sc[0][1], sc2[0][1])
    for s in snaps:
        s.free()


def perplexity_from_rows(rows, tokens, head=None):
    """run.rs:699-755 restated literally in f32 over FULL rows of the fed tokens (a 0 in front of `tokens` when head is None):
    p = exp(x)[token] / sum exp(x), ln, sum, divided by the fed length."""
    fed = list(tokens) if head is not None else [0] + list(tokens)
    p = [np.float32(head)] if head is not None else []
    for index in range(1, len(fed)):
        data = np.exp(np.asarray(rows[index - 1], np.float32))
        total = np.float32(0.0)
        for x in data:
            total = np.float32(total + x)
        p.append(np.float32(data[fed[index]] / total))
    ppl = np.float32(0.0)
    for x in p:
        ppl = np.float32(ppl + np.float32(np.log(x)))
    return float(np.float32(-ppl / np.float32(len(fed))))


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_perplexity_matches_the_oracle(models, preset):
    m, st = models(preset)
    orc = O.Oracle(O.parse_st(st), "f16")
    toks = np.random.default_rng(7).integers(1, 500, 17).tolist()
    for head in (None, 0.3):
        fed = toks if head is not None else [0] + toks
        want_rows, _ = orc.run(fed, orc.state_init(), full=True)
        want = perplexity_from_rows(want_rows, toks, head)
        m.state.load(m.state.init(), 1)
        got = m.perplexity(1, toks, head=head)
        assert abs(got - want) <= 1e-3 * abs(want), (head, got, want)


def test_odd_vocabulary_keeps_the_row(models):
    """V = 509 (V % 4 != 0): the kept row is the last FULL row, so sample_topk reads it."""
    m, _ = models("tiny6", V=509)
    m.state.load(m.state.init(), 0)
    full = m.infer_raw([0], [6], [3, 1, 4, 1, 5, 9], [capi.OPTION_FULL])[0].copy()
    ids, _ = m.sample_topk([0], top_k=4)
    want = np.lexsort((np.arange(509), -full[-1].astype(np.float64)))[:4]
    assert ids[0].tolist() == want.tolist()


def test_odd_vocabulary_scores(models):
    m, _ = models("tiny6", V=509)
    m.state.load(m.state.init(), 1)
    full = m.infer_raw([1], [6], [3, 1, 4, 1, 5, 9], [capi.OPTION_FULL])[0].copy()
    toks = [2, 508, 7]
    snap = m.state.read(1)
    full2 = m.infer_raw([1], [3], toks, [capi.OPTION_FULL])[0].copy()
    m.state.write(snap, 1)
    _, sc = m.infer_ex([1], [3], toks, [capi.OPTION_SCORE])
    check_scores("tiny6/V509", sc[0][0], sc[0][1], [full[-1], full2[0], full2[1]], toks)
    snap.free()


def test_steps_without_score_entries_launch_the_same_kernels(models):
    m, _ = models("tiny6")
    for s in range(3):
        m.state.load(m.state.init(), s)
    args = ([0, 1, 2], [1, 4, 2], [5, 6, 7, 8, 9, 10, 11], [capi.OPTION_LAST] * 3)
    m.infer_raw(*args)                                   # captures the step graph
    n0 = m.launch_count()
    m.infer_raw(*args)
    n1 = m.launch_count()
    m.infer_ex(*args)
    n2 = m.launch_count()
    assert n1 - n0 == n2 - n1 > 0


def test_tensor_parallel_refuses_score_entries():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    m = runtime.Model(synth.make_st("small5", 0), max_batch=2, token_chunk_size=16, devices=[0, 1])
    try:
        m.state.load(m.state.init(), 0)
        with pytest.raises(capi.B200Error) as ei:
            m.infer_ex([0], [2], [1, 2], [capi.OPTION_SCORE])
        assert ei.value.code == capi.ERR_UNSUPPORTED
        rows, _ = m.infer_ex([0], [2], [1, 2], [capi.OPTION_LAST])
        assert rows[0].shape[0] == 1
    finally:
        m.close()
