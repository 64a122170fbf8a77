"""Pooled hidden rows (b200rwkv_keep_hidden_pooled / b200rwkv_last_hidden_pooled): one [num_emb] row per entry of an infer
call, reduced on the device by hidden_pool_kernel from the step buffers the LN stages record the residual stream into.

The per-token recording (b200rwkv_keep_hidden_layers) is the yardstick: with both on in one call, POOL_LAST must equal the
entry's last recorded row and POOL_MEAN the float32 sum of the entry's recorded rows in token order divided once by the
count, bit for bit, however the call is cut into steps.  (The rows themselves may move in their last bits with the cut, as
the projections sum in another order; the reduction adds no dependence of its own.)  Also checked: pooling changes no other
output, costs one launch per step and no per-token copy, the refusals that need an engine, and the NumPy oracle."""
import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3                      # tests/test_gpu_hidden.py's tolerance against the oracle
RAGGED = (1, 3, 17, 130, 300)
SLOTS = [6, 0, 3, 7, 2]             # permuted and sparse in an engine of 8 slots


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(preset, max_batch=8, chunk=32, exact=False):
        key = (preset, max_batch, chunk, exact)
        if key not in cache:
            cache[key] = runtime.Model(synth.make_st(synth.PRESETS[preset], 0), max_batch=max_batch, token_chunk_size=chunk,
                                       exact=exact)
        return cache[key]

    yield get
    for m in cache.values():
        m.close()


def make_runs(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(1, 500, size=n).tolist() for n in sizes]


def run_both(m, slots, runs, layers, mode, options=None, kept=None):
    """One infer call over fresh slots with `layers` pooled and `kept` (default: the same layers) recorded per token.
    Returns ({layer: (pooled rows, counts)}, {layer: per-token rows})."""
    kept = layers if kept is None else kept
    for s in slots:
        m.state.load(m.state.init(), s)
    m.keep_hidden(layers=kept)
    m.keep_hidden_pooled(layers, mode)
    try:
        ntok = [len(r) for r in runs]
        m.infer_ex(slots, ntok, sum(runs, []), options or [capi.OPTION_NONE] * len(runs))
        pooled = {l: m.last_hidden_pooled(l) for l in layers}
        rows = {l: m.last_hidden(max_rows=max(sum(ntok), 1), layer=l) for l in kept}
        return pooled, rows
    finally:
        m.keep_hidden(layers=[])
        m.keep_hidden_pooled([])


def split_rows(rows, runs):
    out, off = [], 0
    for r in runs:
        out.append(rows[off:off + len(r)])
        off += len(r)
    return out


def mean_f32(rows):
    """The definition of POOL_MEAN: from +0.0, one float32 addition per token in token order, then one float32 division."""
    acc = np.zeros(rows.shape[1], np.float32)
    for r in rows:
        acc = np.add(acc, r, dtype=np.float32)
    return np.divide(acc, np.float32(rows.shape[0]), dtype=np.float32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check_last(pooled, rows, runs):
    got, ntok = pooled
    assert ntok.tolist() == [len(r) for r in runs]
    for i, part in enumerate(split_rows(rows, runs)):
        assert same_bits(got[i], part[-1]), i


def check_mean(pooled, rows, runs):
    got, ntok = pooled
    assert ntok.tolist() == [len(r) for r in runs]
    for i, part in enumerate(split_rows(rows, runs)):
        assert same_bits(got[i], mean_f32(part)), i
        mean64 = part.astype(np.float64).mean(axis=0)
        assert np.abs(got[i] - mean64).max() <= len(part) * 2.0 ** -23 * np.abs(part).max(), i


def three_layers(m):
    """First, middle and last layer (two layers where the model has only two), the last one first."""
    L = m.info["num_layer"]
    return sorted({0, L // 2, L - 1}, reverse=True)


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_pool_last_is_the_last_recorded_row(models, preset):
    m = models(preset)
    runs = make_runs(RAGGED, 71)
    layers = three_layers(m)
    pooled, rows = run_both(m, SLOTS, runs, layers, "last")
    for l in layers:
        assert pooled[l][0].shape == (len(runs), m.info["num_emb"])
        check_last(pooled[l], rows[l], runs)


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_pool_mean_is_the_sequential_f32_mean(models, preset):
    m = models(preset)
    runs = make_runs(RAGGED, 72)
    layers = three_layers(m)
    pooled, rows = run_both(m, SLOTS, runs, layers, "mean")
    for l in layers:
        check_mean(pooled[l], rows[l], runs)


@pytest.mark.parametrize("chunk", [16, 32, 128])
@pytest.mark.parametrize("preset", ["tiny7", "small6"])
def test_every_cut_follows_the_definition(models, preset, chunk):
    """token_chunk_size 16 / 32 / 128, each input alone in its call and sharing its steps with the others: the pooled rows
    are the definition applied to that call's rows, so no cut adds a rounding of its own; where two cuts record the same
    rows they pool the same bits."""
    m = models(preset, chunk=chunk)
    runs = make_runs((45, 1, 130, 6), 73)
    L = m.info["num_layer"]
    layers = [0, L - 1]
    for mode, check in (("last", check_last), ("mean", check_mean)):
        shared, shared_rows = run_both(m, [3, 1, 0, 2], runs, layers, mode)
        for l in layers:
            check(shared[l], shared_rows[l], runs)
        for i, r in enumerate(runs):
            alone, alone_rows = run_both(m, [i], [r], layers, mode)
            for l in layers:
                check(alone[l], alone_rows[l], [r])
                if same_bits(alone_rows[l], split_rows(shared_rows[l], runs)[i]):
                    assert same_bits(alone[l][0][0], shared[l][0][i])


def test_mixed_options_and_an_entry_without_tokens(models):
    m = models("small6")
    runs = make_runs((9, 40, 0, 5, 33), 74)
    options = [capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_LAST, capi.OPTION_NONE, capi.OPTION_SCORE]
    layers = three_layers(m)
    for mode, ref in (("last", lambda part: part[-1]), ("mean", mean_f32)):
        pooled, rows = run_both(m, SLOTS, runs, layers, mode, options)
        for l in layers:
            got, ntok = pooled[l]
            assert ntok.tolist() == [9, 40, 0, 5, 33] and got.shape[0] == 5
            for i, part in enumerate(split_rows(rows[l], runs)):
                if len(part) == 0:
                    assert same_bits(got[i], np.zeros_like(got[i]))          # +0.0 in every channel
                else:
                    assert same_bits(got[i], ref(part)), (mode, l, i)


def _outputs(m, runs, pooled_layers, mode, steps):
    """A mixed call (FULL, LAST, SCORE entries), then one decode call: logits rows, scores, kept rows (sample_topk), states,
    and the kernel launches of the two calls minus `steps` launches per pooled step."""
    n = len(runs)
    for s in range(n):
        m.state.load(m.state.init(), s)
    m.keep_hidden_pooled(pooled_layers, mode)
    try:
        before = m.launch_count()
        options = [capi.OPTION_FULL, capi.OPTION_LAST, capi.OPTION_SCORE][:n]
        rows, scores = m.infer_ex(list(range(n)), [len(r) for r in runs], sum(runs, []), options)
        last = m.infer_raw(list(range(n)), [1] * n, [5, 6, 7][:n], [capi.OPTION_LAST] * n)
        launches = m.launch_count() - before
        ids, probs = m.sample_topk(list(range(n)), top_k=16)
        states = [m.state.back(s) for s in range(n)]
    finally:
        m.keep_hidden_pooled([])
    arrays = [np.concatenate(rows), np.concatenate(last), scores[2][0], scores[2][1], ids, probs] + states
    return arrays, launches - (steps if pooled_layers else 0)


@pytest.mark.parametrize("preset,exact,chunk,sizes,steps", [("small6", False, 32, (20, 2, 8), 2), ("tiny5", False, 16, (20, 2, 8), 3),
                                                            ("tiny7", False, 32, (3, 1, 2), 2), ("tiny6", True, 32, (20, 2, 8), 3)])
def test_pooling_changes_no_other_output_and_costs_one_launch_per_step(models, preset, exact, chunk, sizes, steps):
    """Logits, scores, kept rows and states are bit-identical with pooling off, on (every layer, either mode) and off again;
    the launches differ by exactly one per step.  `steps`: the prefill's steps (30 tokens: one at chunk 32, two at 16 or
    with precision 1, which runs steps of at most 16 tokens) plus the decode step."""
    m = models(preset, chunk=chunk, exact=exact)
    runs = make_runs(sizes, 75)
    every = list(range(min(m.info["num_layer"], 8)))
    off, n_off = _outputs(m, runs, [], "last", steps)
    on_last, n_last = _outputs(m, runs, every, "last", steps)
    on_mean, n_mean = _outputs(m, runs, every[:1], "mean", steps)
    off2, n_off2 = _outputs(m, runs, [], "last", steps)
    for a, b, c, d in zip(off, on_last, on_mean, off2):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(a, c, equal_nan=True) and np.array_equal(a, d, equal_nan=True)
    assert n_off == n_last == n_mean == n_off2


def test_a_layer_only_pooling_asked_for_is_not_gathered(models):
    """keep_hidden_layers on layer 1, pooling on layers 0 and 1: both see layer 1, the per-token getter refuses layer 0."""
    m = models("small6")
    runs = make_runs((20, 5), 76)
    pooled, rows = run_both(m, [1, 0], runs, [0, 1], "last", kept=[1])
    check_last(pooled[1], rows[1], runs)
    m.keep_hidden_pooled([0], "last")
    try:
        m.infer_raw([0], [3], [1, 2, 3], [capi.OPTION_NONE])
        for layer in (0, 1):
            with pytest.raises(capi.B200Error) as ei:
                m.last_hidden(max_rows=3, layer=layer)
            assert ei.value.code == capi.ERR_STATE
        assert m.last_hidden_pooled(0)[1].tolist() == [3]
    finally:
        m.keep_hidden_pooled([])
    # and the other way round: the rows pooled from a buffer of its own equal the rows recorded per token
    alone, _ = run_both(m, [1, 0], runs, [0], "last", kept=[])
    both, rows = run_both(m, [1, 0], runs, [0], "last")
    assert same_bits(alone[0][0], both[0][0])
    check_last(alone[0], rows[0], runs)


def test_refusals_with_an_engine():
    m = runtime.Model(synth.make_st(synth.PRESETS["tiny7"], 0), max_batch=4, token_chunk_size=32)
    try:
        L, C = m.info["num_layer"], m.info["num_emb"]
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(0)                     # no infer call yet
        assert ei.value.code == capi.ERR_STATE
        m.infer_raw([0], [2], [4, 5], [capi.OPTION_NONE])
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(0)                     # a call made with pooling off
        assert ei.value.code == capi.ERR_STATE
        for bad in ([L], [0, L + 3], list(range(9)), [1, 1]):
            with pytest.raises(capi.B200Error) as ei:
                m.keep_hidden_pooled(bad)
            assert ei.value.code == capi.ERR_INVALID
        with pytest.raises(capi.B200Error) as ei:
            m.keep_hidden_pooled([0], 2)
        assert ei.value.code == capi.ERR_INVALID
        m.keep_hidden_pooled([0, L - 1], "mean")
        m.infer_raw([2, 0, 1], [2, 1, 3], [4, 5, 6, 7, 8, 9], [capi.OPTION_NONE] * 3)
        rows, ntok = m.last_hidden_pooled(0)
        assert rows.shape == (3, C) and ntok.tolist() == [2, 1, 3]
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(1)                     # a layer the call did not pool
        assert ei.value.code == capi.ERR_STATE
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(L)
        assert ei.value.code == capi.ERR_INVALID
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(0, max_rows=2)         # cap too small for three entries
        assert ei.value.code == capi.ERR_INVALID
        buf = np.empty((3, C), np.float32)              # ntok_out may be NULL
        assert capi.lib().b200rwkv_last_hidden_pooled(m._h, 0, capi.ptr(buf), buf.size, None) == 3
        assert same_bits(buf, rows)
        # off, then on again with another layer and mode, on the same engine
        m.keep_hidden_pooled([])
        assert same_bits(m.last_hidden_pooled(0)[0], rows)          # the pooled call's rows are still there
        m.infer_raw([0], [1], [4], [capi.OPTION_NONE])
        with pytest.raises(capi.B200Error) as ei:
            m.last_hidden_pooled(0)
        assert ei.value.code == capi.ERR_STATE
        m.keep_hidden_pooled([1], "last")
        m.infer_raw([3], [4], [4, 5, 6, 7], [capi.OPTION_NONE])
        assert m.last_hidden_pooled(1)[1].tolist() == [4]
        m.keep_hidden_pooled([])
    finally:
        m.close()


@pytest.mark.parametrize("exact,sizes", [(True, RAGGED), (False, (5, 1, 3, 6)), (True, (5, 1, 3, 6))])
def test_rwkv6_precision_1_and_decode_shaped_calls(models, exact, sizes):
    """Precision 1 (steps of at most 16 tokens, split operands) and a call of one decode-shaped step, where the RWKV-6 LN1
    stage runs in pre6_kernel: both modes against the recorded rows."""
    m = models("small6", exact=exact)
    runs = make_runs(sizes, 77)
    slots = SLOTS[:len(runs)]
    layers = three_layers(m)
    for mode, check in (("last", check_last), ("mean", check_mean)):
        pooled, rows = run_both(m, slots, runs, layers, mode)
        for l in layers:
            check(pooled[l], rows[l], runs)


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_pool_last_at_the_last_layer_matches_the_oracle(models, preset):
    m = models(preset)
    orc = O.Oracle(O.parse_st(synth.make_st(synth.PRESETS[preset], 0)), "f16")
    runs = make_runs((20, 1, 8), 78)
    L = m.info["num_layer"]
    got = {}
    for mode in ("last", "mean"):
        for s in range(3):
            m.state.load(m.state.init(), s)
        got[mode] = m.embed_many([2, 0, 1], runs, L - 1, mode=mode)
        assert got[mode].shape == (3, m.info["num_emb"])
    for i, r in enumerate(runs):
        want, _ = orc.hidden(r, orc.state_init())
        scale = max(np.abs(want).max(), 1e-30)
        assert np.abs(got["last"][i] - want[-1]).max() / scale <= REL_TOL, i
        assert np.abs(got["mean"][i] - want.astype(np.float64).mean(axis=0)).max() / scale <= REL_TOL, i
