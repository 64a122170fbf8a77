"""GPU tests of the Int4 weight-only layers (B200RWKV_QUANT_INT4, csrc/int4gemm.cuh): the load-time quantiser against
tests/int4_oracle.py bit for bit; the projection kernel through b200rwkv_op_gemm against float64 with the bound and the
sentinel / repeat checks of tests/test_gpu_gemm.py (W^ = fma_f16(q, scale, min), the engine contract), blocks whose scale is
below 2^-10 included; and engines with Int4 layers against the forward-pass oracle on the same dequantised weights (1e-3
relative, argmax exact)."""
import dataclasses
import functools

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

import int4_oracle as I
import test_gpu_gemm as G
from test_gpu_quant import _matrix, feed, rel_err

pytestmark = pytest.mark.gpu

INT4 = capi.QUANT_INT4
REL_TOL = 1e-3


def _small_range_rows(n, k, seed):
    """Blocks whose scale is below 2^-10 (ranges ~2^-9 around +-0.5 and 0) and subnormal (ranges ~2^-20 around 0)."""
    rng = np.random.default_rng(seed)
    w = np.empty((n, k), np.float32)
    for r in range(n):
        off = (0.5, -0.5, 0.0, 0.0)[r % 4]
        amp = (2.0 ** -9, 2.0 ** -9, 2.0 ** -9, 2.0 ** -20)[r % 4]
        w[r] = off + rng.uniform(-amp, amp, k)
    return w.astype(np.float16)


def _tie_rows(k):
    """Rows whose codes sit exactly on the .5 boundaries: every block keeps min 0 and max 15 (scale 1), the rest j + 0.5."""
    rows = []
    for j in range(15):
        r = np.full(k, j + 0.5, np.float32)
        r[::128], r[1::128] = 0.0, 15.0
        rows.append(r)
    return np.array(rows, np.float16)


# ----------------------------------------------------------------------------------------------------------------------
# quantiser
# ----------------------------------------------------------------------------------------------------------------------
def _check_quantiser(w):
    codes, mn, scale = capi.op_quantize(INT4, w)
    q, m, s = I.quant_int4(w)
    assert (mn.view(np.uint16) == m.view(np.uint16)).all()
    assert (scale.view(np.uint16) == s.view(np.uint16)).all()
    bad = np.argwhere(codes != q)
    assert bad.size == 0, f"{len(bad)} codes differ, first at {tuple(bad[0])}: {codes[tuple(bad[0])]} vs {q[tuple(bad[0])]}"


@pytest.mark.parametrize("shape", [(200, 384), (128, 128), (1, 256), (130, 1024), (1, 128), (17, 1024)])
def test_quantiser_is_bit_exact_on_the_edge_rows(shape):
    """N not a multiple of 128, one row, K = 128 and 1024; _matrix holds a constant block, a zero row, a ramp and an outlier."""
    w = _matrix(max(shape[0], 16), max(shape[1], 256), 4)[:shape[0], :shape[1]].copy()
    _check_quantiser(w)


def test_quantiser_is_bit_exact_on_ties_and_small_scales():
    ties = _tie_rows(512)
    assert (I.quant_int4(ties)[0][:, 2:128] == np.arange(1, 16)[:, None]).all()
    _check_quantiser(ties)
    small = _small_range_rows(64, 1024, 3)
    s = I.quant_int4(small)[2]
    assert (s < np.float16(2.0 ** -10)).all() and (s[3::4] < np.float16(2.0 ** -14)).all() and (s > 0).all()
    _check_quantiser(small)
    # every finite f16 value, shuffled into rows (wide ranges) and sorted into rows (ranges down to the subnormal spacing)
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    h = h[np.isfinite(h)]
    _check_quantiser(np.random.default_rng(8).permutation(h).reshape(-1, 1024))
    _check_quantiser(np.sort(h.astype(np.float32)).astype(np.float16).reshape(-1, 1024))


# ----------------------------------------------------------------------------------------------------------------------
# projection kernel through b200rwkv_op_gemm
# ----------------------------------------------------------------------------------------------------------------------
_dequantised_int = G.dequantised


@functools.lru_cache(maxsize=4)
def _dequantised(N, K, seed, edge, qtype):
    if qtype == INT4:
        return I.dequant_int4(*I.quant_int4(G.weights(N, K, seed, edge)))
    return _dequantised_int(N, K, seed, edge, qtype)


@pytest.fixture(autouse=True)
def _int4_reference_weights(monkeypatch):
    """test_gpu_gemm's float64 reference multiplies with the weights of the engine contract: fma_f16(q, scale, min)."""
    monkeypatch.setattr(G, "dequantised", _dequantised)


@pytest.mark.parametrize("T,grid", [(T, 0) for T in (1, 2, 15, 16, 17, 31, 32, 33, 64, 65, 100, 128)] + [(16, 1), (17, 6), (128, 7)])
def test_token_tiles_and_partial_tiles(T, grid):
    segs = [G.seg(200, 384, bias=True, edge=True), G.seg(200, 384, capi.ACT_RELU2, capi.OUT_A16, edge=True, seed=1)]
    plan = G.run("int4", T, segs, quant=INT4, grid=grid)
    if grid == 6:                             # 6 blocks over 6 CTAs: every tile of 3 k blocks is cut
        assert plan == (6, 12, 4, 2)


@pytest.mark.parametrize("which", ["one", "blocks", "prime"])
@pytest.mark.parametrize("T", [1, 16, 32, 64, 128])
def test_forced_stream_k_grids(T, which):
    segs = [G.seg(256, 4096, bias=True), G.seg(128, 4096, capi.ACT_SIGMOID, capi.OUT_A16), G.seg(96, 384, capi.ACT_SILU, pad=0)]
    blocks = 2 * 32 + 32 + 3
    grid = {"one": 1, "blocks": blocks, "prime": 37}[which]
    plan = G.run("int4-forced", T, segs, quant=INT4, grid=grid)
    assert plan[:3] == (grid, blocks, 4)
    if which == "blocks":
        assert plan[3] == 32                  # one block per CTA: 32 partial tiles summed by the fix-up
    if which == "prime":
        assert plan[1] % plan[0] != 0 and plan[3] > 1


@pytest.mark.parametrize("act", range(capi.ACT_V7DECAY + 1))
def test_every_activation_and_output_mode(act):
    segs = [G.seg(256, 512, act, bias=True, edge=True), G.seg(320, 512, act, capi.OUT_A16, grp=64, pad=64, seed=1),
            G.seg(256, 256, act, capi.OUT_LERP_A16, seed=2)]
    G.run("int4-modes", 16, segs, quant=INT4)
    G.run("int4-modes", 40, segs, quant=INT4, grid=5)


@pytest.mark.parametrize("T", [1, 16, 128])
def test_small_scales_and_ties_through_the_kernel(T):
    """Blocks with scales below 2^-10 (normal and subnormal) and codes on the .5 boundaries, multiplied as fma_f16(q, scale,
    min): within the float64 bound 2^-14 sum_k |x_k W^_nk| of the dequantised weights."""
    K = 1024
    w = np.concatenate([_small_range_rows(113, K, 5), _tie_rows(K)])
    N = w.shape[0]
    x = np.random.default_rng(T).standard_normal((1, T, K)).astype(np.float32)
    out = np.full((1, capi.gemm_rows(T), N), np.nan, np.float32)
    capi.op_gemm(T, [dict(w=w, x=x, out=out)], quant_type=INT4)
    wd = I.dequant_int4(*I.quant_int4(w)).astype(np.float64)
    x16 = x[0].astype(np.float16).astype(np.float64)
    want = x16 @ wd.T
    bound = 2.0 ** -14 * (np.abs(x16) @ np.abs(wd).T) + 1e-30
    assert (np.abs(out[0, :T] - want) <= bound).all(), float((np.abs(out[0, :T] - want) / bound).max())


# the launches of the 7B / 3B / RWKV-7 2.9B layers whose matrices a quantised layer holds (K % 128 == 0), split-K slices included
LAUNCHES = {
    "7b-rkvg": (16, lambda: G.launch_7b_rkvg()),
    "7b-o": (16, lambda: G.launch_row_parallel(4096, 4096)),
    "7b-ffn-kr": (16, lambda: ([G.seg(14336, 4096, capi.ACT_RELU2, capi.OUT_A16), G.seg(4096, 4096, capi.ACT_SIGMOID)], 0)),
    "7b-ffn-v": (16, lambda: G.launch_row_parallel(4096, 14336)),
    "7b-ffn-v-prefill": (64, lambda: G.launch_row_parallel(4096, 14336)),
    "3b-rkvg": (1, lambda: G.launch_7b_rkvg(2560, 64)),
    "3b-ffn-v": (1, lambda: G.launch_row_parallel(2560, 8960)),
    "v7-2b9-ffn-k": (8, lambda: ([G.seg(10240, 2560, capi.ACT_RELU2, capi.OUT_A16)], 0)),
    "v7-2b9-ffn-v": (8, lambda: G.launch_row_parallel(2560, 10240)),
}


@pytest.mark.parametrize("name", list(LAUNCHES))
def test_model_layer_launches(name):
    T, make = LAUNCHES[name]
    segs, grid = make()
    G.run(name, T, segs, quant=INT4, grid=grid)


def test_forced_grid_gives_each_token_the_bits_of_a_16_token_launch():
    """The batch-invariant mode's premise for Int4 projections: at a forced grid, 128 tokens in one launch give every token
    the bits of launches of 16."""
    rng = np.random.default_rng(6)
    N, K, grid = 384, 1024, 10
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((1, 128, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    xx, sx = rng.standard_normal((1, 128, N)).astype(np.float32), rng.standard_normal((1, 128, N)).astype(np.float32)
    mu = rng.random(N).astype(np.float32)
    for act, mode in [(capi.ACT_NONE, capi.OUT_F32), (capi.ACT_TANH, capi.OUT_F32), (capi.ACT_TANH, capi.OUT_A16),
                      (capi.ACT_NONE, capi.OUT_LERP_A16)]:
        def run(T, t0):
            dt = np.float32 if mode == capi.OUT_F32 else np.uint16
            d = dict(w=w, x=x[:, t0:t0 + T], act=act, out_mode=mode, out=np.zeros((1, capi.gemm_rows(T), N), dt))
            if mode == capi.OUT_F32:
                d["bias"] = bias
            if mode == capi.OUT_LERP_A16:
                d.update(xx=xx[:, t0:t0 + T], sx=sx[:, t0:t0 + T], mu=mu)
            capi.op_gemm(T, [d], quant_type=INT4, grid=grid)
            out = d["out"][0, :T]
            return out.view(np.uint16 if out.dtype == np.uint16 else np.uint32)
        wide = run(128, 0)
        narrow = np.concatenate([run(16, t0) for t0 in range(0, 128, 16)])
        assert np.array_equal(wide, narrow), (act, mode)


# ----------------------------------------------------------------------------------------------------------------------
# engines with Int4 layers
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def int4models():
    cache = {}

    def get(preset, layers=None, max_batch=4, chunk=128):
        key = (preset, layers, max_batch, chunk)
        if key not in cache:
            st = synth.make_st(synth.PRESETS[preset], 0)
            w = O.parse_st(st)
            L = synth.PRESETS[preset].L if layers is None else layers
            m = runtime.Model(st, max_batch=max_batch, token_chunk_size=chunk, quant=L, quant_type="Int4")
            cache[key] = (m, O.Oracle(I.quantize_model(w, L, INT4), "f16"), w)
        return cache[key]

    yield get
    for m, _, _ in cache.values():
        m.close()


@pytest.mark.parametrize("preset", ["tiny6", "tiny5", "tiny7", "small6"])
def test_logits_and_states_match_the_oracle(int4models, preset):
    m, orc, w = int4models(preset)
    toks = [1, 5, 9, 33, 2, 7, 300, 41, 41, 8, 0, 17]
    m.state.load(m.state.init(), 0)
    got = np.stack([feed(m, 0, [t])[0] for t in toks])
    want, want_state = orc.run(toks, orc.state_init(), full=True)
    assert rel_err(got, want) <= REL_TOL
    assert (got.argmax(1) == want.argmax(1)).all()
    assert rel_err(m.state.back(0), want_state) <= REL_TOL
    # the format is really in effect: the f16 model answers differently
    plain, _ = O.Oracle(w, "f16").run(toks, orc.state_init(), full=True)
    assert rel_err(want, plain) > 1e-3


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_prefill_shapes(int4models, preset):
    m, orc, _ = int4models(preset)
    rng = np.random.default_rng(11)
    for n, slot in ((20, 0), (50, 1), (128, 2), (300, 3)):
        toks = rng.integers(1, 500, size=n).tolist()
        m.state.load(m.state.init(), slot)
        got = feed(m, slot, toks)
        want, want_state = orc.run(toks, orc.state_init())
        assert rel_err(got, want) <= REL_TOL, n
        assert got.argmax() == want.argmax()
        assert rel_err(m.state.back(slot), want_state) <= REL_TOL, n


def test_only_the_first_layers_are_int4(int4models):
    m, orc, _ = int4models("small6", layers=2)
    seqs = [[3, 4, 5, 6, 7], [100, 200], [9] * 17, [1]]
    for s in range(4):
        m.state.load(m.state.init(), s)
    rows = m.infer_raw([0, 1, 2, 3], [len(x) for x in seqs], [t for x in seqs for t in x], [capi.OPTION_LAST] * 4)
    for s, x in enumerate(seqs):
        want, _ = orc.run(x, orc.state_init())
        assert rel_err(rows[s][0], want[0]) <= REL_TOL
        assert rows[s][0].argmax() == want[0].argmax()


def test_7b_layer_at_batch_16():
    """One layer with the 7B dimensions: the O and channel-mix value projections run as split-K slices."""
    shp = dataclasses.replace(synth.PRESETS["v6-7b"], L=1, V=4096)
    st = synth.make_st(shp, 0)
    w = O.parse_st(st)
    orc = O.Oracle(I.quantize_model(w, 1, INT4), "f16").keep_all_matrices()
    m = runtime.Model(st, max_batch=16, token_chunk_size=64, quant=1, quant_type="Int4")
    try:
        rng = np.random.default_rng(5)
        toks = rng.integers(1, 4000, size=(16, 3))
        slots = list(range(16))
        for s in slots:
            m.state.load(m.state.init(), s)
        for j in range(3):
            rows = m.infer_raw(slots, [1] * 16, toks[:, j].tolist(), [capi.OPTION_LAST] * 16)
        for s in (0, 7, 15):
            want, want_state = orc.run(toks[s].tolist(), orc.state_init())
            assert rel_err(rows[s][0], want[0]) <= REL_TOL
            assert rows[s][0].argmax() == want[0].argmax()
            assert rel_err(m.state.back(s), want_state) <= REL_TOL
        ptoks = rng.integers(1, 4000, size=40).tolist()
        m.state.load(m.state.init(), 1)
        got = m.infer_raw([1], [40], ptoks, [capi.OPTION_LAST])[0][0]
        want, _ = orc.run(ptoks, orc.state_init())
        assert rel_err(got, want[0]) <= REL_TOL
        assert got.argmax() == want[0].argmax()
    finally:
        m.close()


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_batch_invariant_int4_engine(preset):
    """A 300-token FULL prompt (steps of 128, 128 and 44 tokens) gives the bits of the same tokens fed one per call."""
    st = synth.make_st(synth.PRESETS[preset], 0)
    m = runtime.Model(st, max_batch=4, token_chunk_size=128, quant=synth.PRESETS[preset].L, quant_type="Int4",
                      batch_invariant=True)
    try:
        for s in range(2):
            m.state.load(m.state.init(), s)
        toks = np.random.default_rng(1).integers(1, m.info["num_vocab"], size=300).tolist()
        full = m.infer_raw([0], [300], toks, [capi.OPTION_FULL])[0].copy()
        ref = np.stack([m.infer_raw([1], [1], [t], [capi.OPTION_LAST])[0][0].copy() for t in toks])
        assert np.array_equal(full.view(np.uint32), ref.view(np.uint32))
        assert np.array_equal(m.state.back(0).view(np.uint32), m.state.back(1).view(np.uint32))
    finally:
        m.close()


def test_refusals_on_the_gpu():
    st = synth.make_st(synth.PRESETS["tiny6"], 0)
    with pytest.raises(capi.B200Error) as e:
        runtime.Model(st, max_batch=2, token_chunk_size=32, quant=2, quant_type="Int4", exact=True)      # precision 1
    assert e.value.code == capi.ERR_UNSUPPORTED
    with pytest.raises(capi.B200Error) as e:
        runtime.Model(st, max_batch=2, token_chunk_size=32, quant=2, quant_type="Int4",
                      adapters=[(synth.make_lora_st("tiny6", rank=8, seed=1), 1.0)])
    assert e.value.code == capi.ERR_UNSUPPORTED
    w = np.zeros((64, 256), np.float16)
    x = np.zeros((1, 4, 256), np.float32)
    with pytest.raises(capi.B200Error) as e:
        capi.op_gemm(4, [dict(w=w, x=x, out=np.zeros((1, 32, 64), np.float32))], precision=1, quant_type=INT4)
    assert e.value.code == capi.ERR_UNSUPPORTED
    # quant = 0 is the plain f16 model
    runtime.Model(st, max_batch=2, token_chunk_size=32, quant=0, quant_type="Int4").close()
