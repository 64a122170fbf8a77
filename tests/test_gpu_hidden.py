"""Per-layer hidden states (b200rwkv_keep_hidden_layers / b200rwkv_last_hidden_layer): the `layer` parameter of the
embeddings route (reference docs/doc-api/openai.md:376-437).  "Layer l" is the f32 residual stream after block l, before any
LayerNorm.  The rows of layer l < L - 1 are stored by the LN1 stage of block l + 1, which runs in one of three kernels
depending on the step: pre6_kernel (RWKV-6, <= 16 tokens), ln_mix_cluster_kernel (RWKV-5 / 7, <= 16 tokens) and
ln_mix_kernel (more than 16 tokens); layer L - 1 comes from ln_out_kernel, the rows b200rwkv_last_hidden returns.

Checked here: every layer against the NumPy oracle, each of those kernels (and both ddlerp LoRA ranks of pre6_kernel),
bit-identical outputs, states and launch counts with recording on and off, ragged multi-step calls, the refusals that need
an engine, and the in-process tensor-parallel engine."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
PRE_MAX_C = 4096          # pre6.cuh: widest row of the fused RWKV-6 front half


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def oracle_layers(orc, tokens, state):
    """The oracle's token loop (Oracle._token) with the residual stream recorded after every block: ([T, L, C], state)."""
    w, info = orc.w, orc.info
    state = state.copy()
    out = []
    for tok in tokens:
        x = O.layer_norm(O._f(w["emb.weight"][int(tok)]), O._vec(w, "blocks.0.ln0.weight"), O._vec(w, "blocks.0.ln0.bias"))
        v_first, rows = None, []
        for l in range(info.num_layer):
            if info.version == 7:
                x, v_first = orc._att_v7(l, x, state[l], v_first)
                x = orc._ffn_v7(l, x, state[l])
            else:
                x = orc._att_v56(l, x, state[l])
                x = orc._ffn_v56(l, x, state[l])
            rows.append(x)
        out.append(np.stack(rows))
    return np.stack(out), state


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(preset, max_batch=4, chunk=32, exact=False, **over):
        key = (preset, max_batch, chunk, exact, tuple(sorted(over.items())))
        if key not in cache:
            shp = synth.PRESETS[preset] if not over else dataclasses.replace(synth.PRESETS[preset], **over)
            st = synth.make_st(shp, 0)
            m = runtime.Model(st, max_batch=max_batch, token_chunk_size=chunk, exact=exact)
            cache[key] = (m, O.Oracle(O.parse_st(st), "f32" if exact else "f16"))
        return cache[key]

    yield get
    for m, _ in cache.values():
        m.close()


def run_recorded(m, layers, runs, option=capi.OPTION_NONE):
    """One infer call over fresh slots 0.. with `layers` recorded; returns {layer: rows [sum(len(runs)), C]}."""
    for s in range(len(runs)):
        m.state.load(m.state.init(), s)
    m.keep_hidden(layers=layers)
    try:
        m.infer_raw(list(range(len(runs))), [len(r) for r in runs], sum(runs, []), [option] * len(runs))
        n = sum(len(r) for r in runs)
        return {l: m.last_hidden(max_rows=n, layer=l) for l in layers}
    finally:
        m.keep_hidden(layers=[])


def check_against_oracle(m, orc, runs, layers=None):
    L = m.info["num_layer"]
    layers = list(range(L)) if layers is None else layers
    got = run_recorded(m, layers, runs)
    off = 0
    for r in runs:
        want, _ = oracle_layers(orc, r, orc.state_init())
        for l in layers:
            rows = got[l][off:off + len(r)]
            assert rows.shape == (len(r), m.info["num_emb"])
            assert rel_err(rows, want[:, l]) <= REL_TOL, (l, rel_err(rows, want[:, l]))
        off += len(r)
    return got


def test_oracle_hook_matches_the_oracle():
    """oracle_layers is Oracle._token with a record per block: its last layer is Oracle.hidden, bit for bit."""
    orc = O.Oracle(O.parse_st(synth.make_st("tiny7", 0)), "f16")
    toks = [3, 70, 9, 41]
    rows, st = oracle_layers(orc, toks, orc.state_init())
    want, want_st = orc.hidden(toks, orc.state_init())
    assert np.array_equal(rows[:, -1], want) and np.array_equal(st, want_st)


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_every_layer_matches_the_oracle(models, preset, exact):
    """All layers recorded at once, a ragged decode-shaped call (9 tokens in one step) at precision 0 and 1."""
    m, orc = models(preset, exact=exact)
    rng = np.random.default_rng(61)
    runs = [rng.integers(1, 500, size=n).tolist() for n in (5, 1, 3)]
    check_against_oracle(m, orc, runs)


def test_decode_rwkv6_front_half_with_lora_rank_32(models):
    """pre6_kernel<2, ·>: RWKV-6, ddlerp LoRA rank 32, a step of <= 16 tokens."""
    m, orc = models("small6")
    info = m.info
    assert info["version"] == 6 and info["time_mix_adapter"] == 32 and info["num_emb"] % 128 == 0 and info["num_emb"] <= PRE_MAX_C
    runs = [[4, 99, 7], [12], [301, 2, 2, 60]]
    assert sum(map(len, runs)) <= 16
    check_against_oracle(m, orc, runs)


def test_decode_rwkv6_front_half_with_the_7b_lora_rank():
    """pre6_kernel<4, ·>: the ddlerp LoRA rank 64 of the 7B model, on a two-layer model of the 7B width."""
    shp = dataclasses.replace(synth.PRESETS["v6-7b"], L=2, V=2048)
    st = synth.make_st(shp, 0)
    m = runtime.Model(st, max_batch=2, token_chunk_size=32)
    try:
        info = m.info
        assert info["time_mix_adapter"] == 64 and info["num_emb"] % 128 == 0 and info["num_emb"] <= PRE_MAX_C
        orc = O.Oracle(O.parse_st(st), "f16")
        runs = [[5, 1700, 33], [808]]
        got = check_against_oracle(m, orc, runs)
        m.keep_hidden(True)
        try:
            for s in range(2):
                m.state.load(m.state.init(), s)
            m.keep_hidden(layers=[1])
            m.infer_raw([0, 1], [3, 1], sum(runs, []), [capi.OPTION_NONE] * 2)
            assert np.array_equal(m.last_hidden(max_rows=4, layer=1), m.last_hidden(max_rows=4))
            assert np.array_equal(m.last_hidden(max_rows=4, layer=1), got[1])
        finally:
            m.keep_hidden(False)
            m.keep_hidden(layers=[])
    finally:
        m.close()


@pytest.mark.parametrize("preset", ["tiny5", "tiny7"])
def test_decode_cluster_ln_kernel(models, preset):
    """ln_mix_cluster_kernel: RWKV-5 / 7 time-mix LN stage of a step of <= 16 tokens (num_emb / 32 <= 256 threads)."""
    m, orc = models(preset)
    C = m.info["num_emb"]
    assert C % 32 == 0 and C // 32 <= 256
    runs = [[8, 6, 100, 2, 9, 9], [44], [71, 13]]
    assert sum(map(len, runs)) <= 16
    check_against_oracle(m, orc, runs)


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_steps_of_more_than_16_tokens(models, preset):
    """ln_mix_kernel: one step of 29 tokens (token_chunk_size 32, precision 0)."""
    m, orc = models(preset)
    rng = np.random.default_rng(62)
    runs = [rng.integers(1, 500, size=n).tolist() for n in (20, 1, 8)]
    T = sum(map(len, runs))
    assert 16 < T <= m.token_chunk_size              # one step, too wide for the decode-shaped kernels
    check_against_oracle(m, orc, runs)


def test_last_layer_rows_equal_last_hidden(models):
    m, _ = models("small6", chunk=8)
    L = m.info["num_layer"]
    rng = np.random.default_rng(63)
    runs = [rng.integers(1, 500, size=n).tolist() for n in (13, 1, 6)]       # several steps
    for s in range(3):
        m.state.load(m.state.init(), s)
    m.keep_hidden(True)
    m.keep_hidden(layers=[L - 1, 0])
    try:
        m.infer_raw([0, 1, 2], [len(r) for r in runs], sum(runs, []), [capi.OPTION_NONE] * 3)
        assert np.array_equal(m.last_hidden(max_rows=20, layer=L - 1), m.last_hidden(max_rows=20))
    finally:
        m.keep_hidden(False)
        m.keep_hidden(layers=[])


def _outputs(m, runs, layers, decode_tokens):
    """FULL rows of one ragged call, then one decode call; the states, kept rows (sample_topk) and kernel launches."""
    n = len(runs)
    for s in range(n):
        m.state.load(m.state.init(), s)
    m.keep_hidden(layers=layers)
    try:
        before = m.launch_count()
        full = np.concatenate(m.infer_raw(list(range(n)), [len(r) for r in runs], sum(runs, []), [capi.OPTION_FULL] * n))
        last = np.concatenate(m.infer_raw(list(range(n)), [1] * n, decode_tokens, [capi.OPTION_LAST] * n))
        launches = m.launch_count() - before
        ids, probs = m.sample_topk(list(range(n)), top_k=16)
        states = [m.state.back(s) for s in range(n)]
    finally:
        m.keep_hidden(layers=[])
    return full, last, ids, probs, states, launches


@pytest.mark.parametrize("preset,exact,sizes", [("small6", False, (20, 1, 8)), ("small6", False, (3, 1, 2)),
                                               ("tiny5", False, (20, 1, 8)), ("tiny7", False, (3, 1, 2)),
                                               ("tiny6", True, (3, 1, 2)), ("tiny7", True, (7, 1, 2))])
def test_recording_changes_no_other_output(models, preset, exact, sizes):
    """Logits, states, kept rows and launch counts are bit-identical with recording on and off: the same step graphs run,
    the LN kernels only add a store."""
    m, _ = models(preset, exact=exact)
    rng = np.random.default_rng(64)
    runs = [rng.integers(1, 500, size=n).tolist() for n in sizes]
    dec = rng.integers(1, 500, size=len(sizes)).tolist()
    L = m.info["num_layer"]
    off = _outputs(m, runs, [], dec)
    on = _outputs(m, runs, list(range(L)), dec)
    off2 = _outputs(m, runs, [], dec)
    for a, b, c in zip(off[:4], on[:4], off2[:4]):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    for a, b in zip(off[4], on[4]):
        assert np.array_equal(a, b)
    assert off[5] == on[5] == off2[5]


def test_unrecorded_layers_write_nothing(models):
    """The LN1 stage of an unrecorded layer stores nothing: step buffers keep their bits while recording is off, and
    only the buffers of the recorded layers change."""
    m, _ = models("small6", max_batch=3)                # an engine of its own: no earlier test has used its step buffers
    C = m.info["num_emb"]
    step = lambda k: m.debug_read(f"hid_step{k}", rows=3).copy()
    run = lambda layers, toks: run_recorded(m, layers, [[t] for t in toks])

    got = run([1], [5, 6, 7])
    b0 = step(0)
    assert np.array_equal(b0, got[1])                   # buffer 0 holds layer 1's rows of the (only) step
    zeros = np.zeros((3, C), np.float32)
    for k in range(1, 8):
        assert np.array_equal(step(k), zeros)
    run([], [9, 10, 11])                                 # recording off: nothing is stored
    assert np.array_equal(step(0), b0)
    got = run([2, 0], [9, 10, 11])                       # buffer 0 <- layer 2, buffer 1 <- layer 0; layers 1 and 3 write nothing
    assert np.array_equal(step(0), got[2]) and np.array_equal(step(1), got[0])
    for k in range(2, 8):
        assert np.array_equal(step(k), zeros)
    run([3], [12, 13, 14])                               # the last layer comes from ln_out_kernel: no step buffer is written
    assert np.array_equal(step(0), got[2]) and np.array_equal(step(1), got[0])


def test_ragged_multi_step_calls_and_chunk_sizes(models):
    """Four entries (one of a single token) over several internal steps with three layers recorded at once: rows in entry
    order, matching the oracle; the cut into steps (token_chunk_size 32 vs 8) moves them only by summation order."""
    rng = np.random.default_rng(65)
    runs = [rng.integers(1, 500, size=n).tolist() for n in (45, 1, 20, 6)]
    layers = [2, 0, 3]
    got = {}
    for chunk in (32, 8):
        m, orc = models("small6", chunk=chunk)
        got[chunk] = check_against_oracle(m, orc, runs, layers)
        assert all(got[chunk][l].shape[0] == 72 for l in layers)
    for l in layers:
        assert rel_err(got[8][l], got[32][l]) <= 5e-4, l


def test_refusals_with_an_engine(models):
    m, _ = models("tiny7")
    L = m.info["num_layer"]
    runs = [[1, 2, 3]]
    run_recorded(m, [0, L - 1], runs)
    for bad in ([L], [0, L + 3], list(range(9))):
        with pytest.raises(capi.B200Error) as ei:
            m.keep_hidden(layers=bad)
        assert ei.value.code == capi.ERR_INVALID
    with pytest.raises(capi.B200Error) as ei:
        m.keep_hidden(layers=[1, 1])
    assert ei.value.code == capi.ERR_INVALID
    # the recorded call's rows are still there; a layer it did not record is ERR_STATE, a layer outside the model INVALID
    assert m.last_hidden(max_rows=3, layer=0).shape == (3, m.info["num_emb"])
    with pytest.raises(capi.B200Error) as ei:
        m.last_hidden(max_rows=3, layer=1)
    assert ei.value.code == capi.ERR_STATE
    with pytest.raises(capi.B200Error) as ei:
        m.last_hidden(max_rows=3, layer=L)
    assert ei.value.code == capi.ERR_INVALID
    with pytest.raises(capi.B200Error) as ei:
        m.last_hidden(max_rows=2, layer=0)              # cap too small
    assert ei.value.code == capi.ERR_INVALID
    # a call made with recording off records nothing
    m.infer_raw([0], [1], [4], [capi.OPTION_NONE])
    with pytest.raises(capi.B200Error) as ei:
        m.last_hidden(max_rows=3, layer=0)
    assert ei.value.code == capi.ERR_STATE


def test_embed_returns_the_last_token_row(models):
    m, orc = models("small6")
    toks = [17, 3, 250, 8, 64]
    want, _ = oracle_layers(orc, toks, orc.state_init())
    for layer in (0, 2):
        m.state.load(m.state.init(), 1)
        e = m.embed(1, toks, layer)
        assert e.shape == (m.info["num_emb"],)
        assert rel_err(e, want[-1, layer]) <= REL_TOL


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
def test_tensor_parallel_engine_records_the_same_rows():
    """In-process tensor parallelism: rank 0 records the (replicated) residual stream; it matches the single-GPU engine up
    to summation order."""
    world = 2
    st = synth.make_st("small6", 0)
    single = runtime.Model(st, max_batch=4, token_chunk_size=32, device=0)
    multi = runtime.Model(st, max_batch=4, token_chunk_size=32, devices=list(range(world)))
    try:
        rng = np.random.default_rng(66)
        runs = [rng.integers(1, 500, size=n).tolist() for n in (5, 1, 20)]
        a, b = run_recorded(single, [0, 1, 3], runs), run_recorded(multi, [0, 1, 3], runs)
        for l in (0, 1, 3):
            assert rel_err(b[l], a[l]) <= REL_TOL, l
    finally:
        single.close()
        multi.close()
