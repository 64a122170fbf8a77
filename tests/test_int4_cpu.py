"""CPU tests of the Int4 weight-only format (tests/int4_oracle.py, B200RWKV_QUANT_INT4): the restatement's codes, parameters
and round-trip error, constant blocks and ties, blocks whose scale is below 2^-10, which matrices a model quantises, the bytes
a pass streams, the weight error next to the other formats, and the refusals the C entries make before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

import fp8_oracle as F
import int4_oracle as I


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def _blocks(w):
    n, k = w.shape
    return w.astype(np.float32).reshape(n, k // 128, 128)


def test_codes_and_parameters_follow_the_definition():
    rng = np.random.default_rng(1)
    w = (rng.standard_normal((48, 512)) * 0.05).astype(np.float16)
    w[2, 128:256] = np.float16(60000.0)         # one outlier block
    w[2, 130] = np.float16(-60000.0)
    q, mn, s = I.quant_int4(w)
    assert q.dtype == np.uint8 and mn.dtype == np.float16 and s.dtype == np.float16
    assert q.shape == w.shape and mn.shape == s.shape == (48, 4)
    assert q.max() <= 15
    b = _blocks(w)
    lo, hi = b.min(axis=2), b.max(axis=2)
    assert (mn.astype(np.float32) == lo).all()                                     # f16(min) is exact
    assert (s == ((hi - lo).astype(np.float32) / np.float32(15)).astype(np.float16)).all()
    # every block with a range reaches code 0 at its minimum and code 15 at its maximum
    qb = q.reshape(48, 4, 128)
    assert (qb.min(axis=2) == 0).all() and (qb.max(axis=2) == 15).all()


def test_round_trip_error_is_half_a_step_plus_roundings():
    rng = np.random.default_rng(2)
    w = (rng.standard_normal((64, 1024)) * 0.05).astype(np.float16)
    w[4, :128] = (rng.standard_normal(128) * 2.0 ** -14).astype(np.float16)    # range ~2^-12: scale below 2^-10
    w[6, 128:256] = (rng.standard_normal(128) * 2.0 ** -22).astype(np.float16)  # f16 subnormals: subnormal scale
    w[8, :] = (rng.standard_normal(1024) * 1000).astype(np.float16)
    q, mn, s = I.quant_int4(w)
    d = I.dequant_int4(q, mn, s)
    assert d.dtype == np.float16
    b = _blocks(w).astype(np.float64)
    rng_ = (b.max(axis=2) - b.min(axis=2))[..., None]
    step = rng_ / 15                                                   # the exact code spacing
    s64 = s.astype(np.float64)[..., None]
    dd = d.astype(np.float64).reshape(b.shape)
    err = np.abs(dd - b)
    # half a step, the rounding of the scale to f16 over up to 15 steps, the one f16 rounding of the weight, f32 slack
    bound = step / 2 + 15 * np.abs(s64 - step) + np.abs(dd) * 2.0 ** -11 + 2.0 ** -25 + rng_ * 2.0 ** -20
    assert (err <= bound).all()
    # the small-range blocks are really below 2^-10 and subnormal, and still resolve 16 levels
    assert s[4, 0] < np.float16(2.0 ** -10) and s[6, 1] < np.float16(2.0 ** -14) and s[6, 1] > 0
    assert len(np.unique(q[4, :128])) > 8 and len(np.unique(q[6, 128:256])) > 8


def test_constant_and_zero_blocks():
    w = np.zeros((3, 256), np.float16)
    w[0, :128] = np.float16(0.125)
    w[1, 128:] = np.float16(-3.0)
    q, mn, s = I.quant_int4(w)
    assert (q == 0).all() and (s == 0).all()
    assert (I.dequant_int4(q, mn, s) == w).all()


def test_ties_round_up():
    """mn = 0, rng = 15: w = j + 0.5 lands exactly on the tie j + 0.5 in f32, and floor(x + 0.5) takes it up (not to even)."""
    for j in range(15):
        w = np.array([[0.0, 15.0] + [j + 0.5] * 126], np.float16)
        t = np.float32(np.float32(j + 0.5) / np.float32(15))
        assert np.float32(t * np.float32(15)) == np.float32(j + 0.5)
        q, _, s = I.quant_int4(w)
        assert s[0, 0] == 1 and (q[0, 2:] == j + 1).all(), j


def test_quantize_model_touches_the_projection_matrices_of_the_first_layers():
    w = O.parse_st(synth.make_st("tiny6", 0))
    wq = I.quantize_model(w, 1, I.QUANT_INT4)
    changed = sorted(k for k in w if wq[k] is not w[k])
    assert changed == sorted(f"blocks.0.{m}" for m in Q.QUANT_MATRICES)
    for k in changed:
        assert wq[k].dtype == np.float16 and wq[k].shape == w[k].shape
        assert (wq[k] != w[k]).any()
    wi = I.quantize_model(w, 1, Q.QUANT_INT8)
    assert (wi["blocks.0.att.key.weight"] == Q.quantize_model(w, 1, Q.QUANT_INT8)["blocks.0.att.key.weight"]).all()


def test_int4_weight_bytes():
    assert I.quant_weight_bytes(4096, 4096) == 4096 * 4096 // 2 + 4096 * 32 * 4
    assert I.quant_weight_bytes(4096, 14336) == 4096 * 14336 // 2 + 4096 * 112 * 4
    # 0.531 bytes per weight, the same as NF4, half of Int8's and FP8's
    for n, k in ((4096, 4096), (14336, 4096), (2560, 8960)):
        assert I.quant_weight_bytes(n, k) == Q.quant_weight_bytes(n, k, Q.QUANT_NF4)
        assert I.quant_weight_bytes(n, k) / (n * k) == pytest.approx(0.53125)
    for qt in (Q.QUANT_NONE, Q.QUANT_INT8, Q.QUANT_NF4):
        assert I.quant_weight_bytes(512, 1024, qt) == Q.quant_weight_bytes(512, 1024, qt)
    assert capi.QUANT_INT4 == I.QUANT_INT4 == 6


def test_weight_error_next_to_the_other_formats():
    """Relative RMS error on N(0, 0.05) weights (DESIGN.md §4a): Int8 0.006 < FP8 0.027 < NF4 0.092 < Int4 0.100."""
    big = (np.random.default_rng(2).standard_normal((256, 4096)) * 0.05).astype(np.float16)
    ref = big.astype(np.float32)
    rms = lambda x: float(np.sqrt(((x.astype(np.float32) - ref) ** 2).mean() / (ref ** 2).mean()))
    e_int4 = rms(I.dequant_int4(*I.quant_int4(big)))
    e_int8 = rms(Q.dequant_int8(*Q.quant_int8(big), contract="f32"))
    e_nf4 = rms(Q.dequant_nf4(*Q.quant_nf4(big), contract="f32"))
    e_fp8 = rms(F.dequant_fp8(*F.quant_fp8(big)))
    assert e_int8 < e_fp8 < e_nf4 < e_int4 < 0.11
    assert abs(e_int4 - 0.100) < 0.002


def test_int4_refusals_without_a_gpu():
    """The refusals the C entries make for Int4 before their first CUDA call."""
    INV, UNS = capi.ERR_INVALID, capi.ERR_UNSUPPORTED
    N, K, T = 64, 256, 4
    w = np.zeros((N, K), np.float16)
    x = np.zeros((1, T, K), np.float32)
    out = np.zeros((1, 16, N), np.float32)

    def gemm(K_=K, T_=T, precision=0, quant=capi.QUANT_INT4):
        seg = capi.GemmSeg(N, K_, capi.ptr(w), capi.ptr(x), None, capi.ACT_NONE, capi.OUT_F32, 0, None, None, None, N, capi.ptr(out))
        return capi.lib().b200rwkv_op_gemm(0, T_, precision, quant, 0, 1, 1, (capi.GemmSeg * 1)(seg), None)

    assert gemm(precision=1) == UNS                         # precision 1 over Int4 weights
    assert gemm(K_=200) == UNS                              # K % 128
    assert gemm(quant=5) == UNS and gemm(quant=3) == UNS    # unassigned, SF4
    codes = np.zeros((N, K), np.uint8)
    p = np.zeros((N, K // 128), np.float16)
    w200 = np.zeros((N, 200), np.float16)
    op_q = capi.lib().b200rwkv_op_quantize
    assert op_q(0, capi.QUANT_INT4, N, 200, capi.ptr(w200), capi.ptr(codes), capi.ptr(p), capi.ptr(p)) == INV
    assert op_q(0, capi.QUANT_INT4, N, K, capi.ptr(w), None, capi.ptr(p), capi.ptr(p)) == INV
    assert op_q(0, capi.QUANT_INT4, N, K, capi.ptr(w), capi.ptr(codes), capi.ptr(p), None) == INV      # Int4 needs the scales
    assert op_q(0, 5, N, K, capi.ptr(w), capi.ptr(codes), capi.ptr(p), capi.ptr(p)) == UNS
    # create_ex: Int4 layers are single-GPU
    st = synth.make_st("tiny6", 0)
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    opt.quant_layers, opt.quant_type = 2, capi.QUANT_INT4
    opt.num_devices = 2
    opt.devices[0], opt.devices[1] = 0, 1
    h = C.c_void_p()
    assert capi.lib().b200rwkv_create_ex(capi.ptr(st), st.size, C.byref(opt), C.byref(h)) == UNS
    assert not h and "single-GPU" in _last_error()
    # adapters: a pair on an Int4 layer is refused, as on the other quantised layers
    good = synth.make_lora_st("tiny6", rank=8, seed=1)
    opt.num_devices, opt.quant_layers = 1, 1
    ptrs, lens, alphas = (C.c_void_p * 1)(good.ctypes.data), (C.c_size_t * 1)(good.size), (C.c_float * 1)(1.0)
    rc = capi.lib().b200rwkv_create_adapters(capi.ptr(st), st.size, C.byref(opt), 1, C.cast(ptrs, C.c_void_p),
                                             C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p), C.byref(h))
    assert rc == UNS and "quantised" in _last_error()
    # adapter places: every layer Int4 leaves no f16 projection matrix of the targeted kinds
    opt.quant_layers = synth.PRESETS["tiny6"].L
    rc = capi.lib().b200rwkv_create_adapter_places(capi.ptr(st), st.size, opt, 2, capi.TARGET_ATT_K | capi.TARGET_FFN_V, C.byref(h))
    assert rc == UNS and "name no f16 projection matrix" in _last_error()
    # the Python surface spells the format "Int4" (any case); unknown names are refused before anything is built
    with pytest.raises(capi.B200Error) as e:
        runtime.Model(st, max_batch=2, token_chunk_size=32, quant=2, quant_type="Int3")
    assert e.value.code == INV and "Int4" in str(e.value) and "FP8" in str(e.value)
