"""CPU tests of the FP8 (E4M3) weight-only format (tests/fp8_oracle.py, B200RWKV_QUANT_FP8): the E4M3 restatement against the
format definition and against torch's float8_e4m3fn conversion, the quantiser's rounding, saturation and zero rows, which
matrices a model quantises, the bytes a pass streams, and the refusals the C entries make before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

import fp8_oracle as F


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_e4m3_table_follows_the_format_definition():
    v = F.E4M3_VALUES
    assert v[0x00] == 0 and not np.signbit(v[0x00]) and v[0x80] == 0 and np.signbit(v[0x80])
    assert v[0x01] == 2.0 ** -9 and v[0x07] == 7 * 2.0 ** -9           # subnormals: m / 8 * 2^-6
    assert v[0x08] == 2.0 ** -6 and v[0x38] == 1.0 and v[0x39] == 1.125  # bias 7
    assert v[0x7E] == 448 and v[0xFE] == -448                            # largest finite value
    assert np.isnan(v[0x7F]) and np.isnan(v[0xFF])                       # S.1111.111 is NaN, nothing else is
    assert np.isnan(v).sum() == 2 and not np.isinf(v).any()
    assert (v[0x80:] == -v[:0x80])[~np.isnan(v[:0x80])].all()
    pos = v[:0x7F]
    assert (np.diff(pos) > 0).all()                                      # codes ascend with their magnitude
    # every value is exact in f16 (the engine feeds them to the tensor cores as f16)
    fin = v[~np.isnan(v)]
    assert (fin.astype(np.float16).astype(np.float64) == fin).all()
    # an independent decoding: torch's float8_e4m3fn reinterpretation of the 256 bit patterns
    torch = pytest.importorskip("torch")
    t = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float64).numpy()
    assert ((t == v) | (np.isnan(t) & np.isnan(v))).all()
    # encoding a code's value gives the code back
    codes = np.array([c for c in range(256) if not np.isnan(v[c])], np.uint8)
    assert (F.e4m3_encode(v[codes].astype(np.float32)) == codes).all()


def test_e4m3_encode_matches_torch_on_every_finite_f16_up_to_448():
    torch = pytest.importorskip("torch")
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    h = h[np.isfinite(h) & (np.abs(h.astype(np.float32)) <= 448)]
    x = h.astype(np.float32)
    want = torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert (F.e4m3_encode(x) == want).all()
    # the f32 quotients the quantiser rounds are not f16 values: random f32 in the whole range, all exponents
    rng = np.random.default_rng(3)
    x = (rng.uniform(-1, 1, 1 << 18) * np.exp2(rng.integers(-14, 9, 1 << 18))).astype(np.float32)
    x = np.clip(x, -448, 448)
    assert (F.e4m3_encode(x) == torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy()).all()


def test_e4m3_encode_rounds_ties_to_even_and_saturates():
    v = F.E4M3_VALUES
    for c in range(0x7E):                       # the midpoint of codes c and c + 1 goes to the even one
        mid = np.float32((v[c] + v[c + 1]) / 2)
        assert float(mid) == (v[c] + v[c + 1]) / 2
        assert F.e4m3_encode(mid) == (c if c % 2 == 0 else c + 1), hex(c)
        assert F.e4m3_encode(-mid) == 0x80 | (c if c % 2 == 0 else c + 1)
        below, above = np.nextafter(mid, np.float32(0)), np.nextafter(mid, np.float32(1e9))
        assert F.e4m3_encode(below) == c and F.e4m3_encode(above) == c + 1
    big = np.array([448.0, 448.5, 464.0, 479.9, 480.0, 60000.0, 3.0e38], np.float32)
    assert (F.e4m3_encode(big) == 0x7E).all() and (F.e4m3_encode(-big) == 0xFE).all()
    assert F.e4m3_encode(np.float32(np.nan)) == 0x7F
    assert F.e4m3_encode(np.float32(2.0 ** -10)) == 0x00                # half the smallest subnormal: ties to +0
    assert F.e4m3_encode(np.float32(-2.0 ** -10)) == 0x80


def test_quant_fp8_scales_rows_of_the_whole_matrix():
    rng = np.random.default_rng(1)
    w = (rng.standard_normal((64, 512)) * 0.05).astype(np.float16)
    w[5] = 0                                    # zero row: scale 0, codes +0
    w[7, 300] = np.float16(-3.0)                # the row's absmax sits in its third k block
    w[9, :] = np.float16(1e-6)                  # a row of f16 subnormals
    q, s = F.quant_fp8(w)
    assert q.dtype == np.uint8 and s.dtype == np.float32 and q.shape == w.shape and s.shape == (64,)
    a = np.abs(w.astype(np.float32)).max(axis=1)
    assert (s == (a / np.float32(448)).astype(np.float32)).all()
    assert s[5] == 0 and (q[5] == 0).all()
    assert q[7, 300] == 0xFE and s[7] == np.float32(3.0) / np.float32(448)
    # every row with a nonzero absmax reaches +-448 at it
    rows = np.nonzero(a > 0)[0]
    assert (np.abs(F.e4m3_decode(q[rows])).max(axis=1) == 448).all()
    # the dequantised weight: s * value(q) in f32; within E4M3's half-ulp (2^-4 relative) plus the subnormal spacing
    d = F.dequant_fp8(q, s)
    assert d.dtype == np.float32
    err = np.abs(d - w.astype(np.float32))
    assert (err <= np.abs(w.astype(np.float32)) * (2.0 ** -4 + 2.0 ** -20) + s[:, None] * 2.0 ** -10).all()
    # relative RMS error of N(0, 0.05) weights sits between Int8 and NF4
    big = (np.random.default_rng(2).standard_normal((256, 4096)) * 0.05).astype(np.float16)
    ref = big.astype(np.float32)
    rms = lambda x: float(np.sqrt(((x - ref) ** 2).mean() / (ref ** 2).mean()))
    e_fp8 = rms(F.dequant_fp8(*F.quant_fp8(big)))
    e_int8 = rms(Q.dequant_int8(*Q.quant_int8(big), contract="f32"))
    e_nf4 = rms(Q.dequant_nf4(*Q.quant_nf4(big), contract="f32"))
    assert e_int8 < e_fp8 < e_nf4 and e_fp8 < 0.03


def test_quantize_model_touches_the_projection_matrices_of_the_first_layers():
    w = O.parse_st(synth.make_st("tiny6", 0))
    wq = F.quantize_model(w, 1, F.QUANT_FP8)
    changed = sorted(k for k in w if wq[k] is not w[k])
    assert changed == sorted(f"blocks.0.{m}" for m in Q.QUANT_MATRICES)
    for k in changed:
        assert wq[k].dtype == np.float32 and wq[k].shape == w[k].shape
        assert (wq[k] != w[k].astype(np.float32)).any()
    # the other formats go to oracle/quant_numpy.py unchanged
    wi = F.quantize_model(w, 1, Q.QUANT_INT8)
    assert (wi["blocks.0.att.key.weight"] == Q.quantize_model(w, 1, Q.QUANT_INT8)["blocks.0.att.key.weight"]).all()


def test_fp8_weight_bytes():
    assert F.quant_weight_bytes(4096, 4096, F.QUANT_FP8) == 4096 * 4096 + 4096 * 4
    assert F.quant_weight_bytes(4096, 14336, F.QUANT_FP8) == 4096 * 14336 + 4096 * 4
    for qt in (Q.QUANT_NONE, Q.QUANT_INT8, Q.QUANT_NF4):
        assert F.quant_weight_bytes(512, 1024, qt) == Q.quant_weight_bytes(512, 1024, qt)
    assert capi.QUANT_FP8 == F.QUANT_FP8 == 4


def test_fp8_refusals_without_a_gpu():
    """The refusals the C entries make for FP8 before their first CUDA call."""
    INV, UNS = capi.ERR_INVALID, capi.ERR_UNSUPPORTED
    N, K, T = 64, 256, 4
    w = np.zeros((N, K), np.float16)
    x = np.zeros((1, T, K), np.float32)
    out = np.zeros((1, 16, N), np.float32)

    def gemm(K_=K, T_=T, precision=0, quant=capi.QUANT_FP8):
        seg = capi.GemmSeg(N, K_, capi.ptr(w), capi.ptr(x), None, capi.ACT_NONE, capi.OUT_F32, 0, None, None, None, N, capi.ptr(out))
        return capi.lib().b200rwkv_op_gemm(0, T_, precision, quant, 0, 1, 1, (capi.GemmSeg * 1)(seg), None)

    assert gemm(precision=1) == UNS                         # precision 1 over FP8 weights
    assert gemm(K_=200) == UNS                              # K % 128
    assert gemm(quant=5) == UNS
    codes = np.zeros((N, 200), np.uint8)
    scale = np.zeros(N, np.float32)
    w200 = np.zeros((N, 200), np.float16)
    assert capi.lib().b200rwkv_op_quantize(0, capi.QUANT_FP8, N, 200, capi.ptr(w200), capi.ptr(codes), capi.ptr(scale), None) == INV
    assert capi.lib().b200rwkv_op_quantize(0, capi.QUANT_FP8, N, K, capi.ptr(w), None, capi.ptr(scale), None) == INV
    assert capi.lib().b200rwkv_op_quantize(0, 5, N, K, capi.ptr(w), capi.ptr(codes), capi.ptr(scale), None) == UNS
    # create_ex: FP8 layers are single-GPU
    st = synth.make_st("tiny6", 0)
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    opt.quant_layers, opt.quant_type = 2, capi.QUANT_FP8
    opt.num_devices = 2
    opt.devices[0], opt.devices[1] = 0, 1
    h = C.c_void_p()
    assert capi.lib().b200rwkv_create_ex(capi.ptr(st), st.size, C.byref(opt), C.byref(h)) == UNS
    assert not h and "single-GPU" in _last_error()
    # adapters: a pair on an FP8 layer is refused, as on Int8 / NF4 layers
    good = synth.make_lora_st("tiny6", rank=8, seed=1)
    opt.num_devices, opt.quant_layers = 1, 1
    ptrs, lens, alphas = (C.c_void_p * 1)(good.ctypes.data), (C.c_size_t * 1)(good.size), (C.c_float * 1)(1.0)
    rc = capi.lib().b200rwkv_create_adapters(capi.ptr(st), st.size, C.byref(opt), 1, C.cast(ptrs, C.c_void_p),
                                             C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p), C.byref(h))
    assert rc == UNS and "quantised" in _last_error()
    # adapter places: every layer FP8 leaves no f16 projection matrix of the targeted kinds
    opt.quant_layers = synth.PRESETS["tiny6"].L
    rc = capi.lib().b200rwkv_create_adapter_places(capi.ptr(st), st.size, opt, 2, capi.TARGET_ATT_K | capi.TARGET_FFN_V, C.byref(h))
    assert rc == UNS and "name no f16 projection matrix" in _last_error()
    # the Python surface spells the format "FP8"; unknown names are refused before anything is built
    with pytest.raises(capi.B200Error) as e:
        runtime.Model(st, max_batch=2, token_chunk_size=32, quant=2, quant_type="FP16")
    assert e.value.code == INV and "FP8" in str(e.value)
