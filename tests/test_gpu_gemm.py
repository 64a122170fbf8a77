"""The projection GEMM kernels (csrc/gemm.cuh, csrc/qgemm.cuh) driven alone through b200rwkv_op_gemm -- the engine's own
planner and launcher over caller-supplied matrices -- against a float64 reference of the same operation.

Reference: y64 = x^ W^T + bias in float64, with x^ the f16-rounded input (precision 0) or the f32 input itself (precision 1,
hi + lo operands), W^ the f16 weight or, for Int8 / NF4 layers, the dequantised weight of oracle/quant_numpy.py's engine
contract (which tests/test_gpu_quant.py holds bit-identical to what the kernels expand); activation and ddlerp in float64.

Bound, per element, scaled by the data rather than by the largest output:  |y - y64| <= 2^-14 sum_k |x^_k W^_nk|  (the f32
accumulation of f16 products over K, stream-K partial sums included), carried through the activation over the interval it
spans, plus a few f32 ulps; f16 outputs get one f16 ulp of the reference on top.  Every case prints its worst ratio
error / bound.  Beyond the values: every cell the kernel must not write keeps its NaN sentinel bit for bit (token rows
T..rows-1, columns N..ldo-1), and each case runs its plan three times back to back on inputs A, B, A: every slice matches its
own reference and slices 0 and 2 are bit-identical (tile counters back to zero after every launch, deterministic fix-up).
"""
import functools
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi
from oracle import quant_numpy as Q

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -14
SENT32 = np.uint32(0x7FA5A5A5)      # NaN bit patterns no arithmetic produces
SENT16 = np.uint16(0x7E5A)
V7_DECAY = float(np.float32(0.606531))   # the constant of csrc/common.cuh ACT_V7DECAY
F16_MAX = 65504.0


@functools.lru_cache(maxsize=1)
def num_sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_split(K: int, tiles: int) -> int:
    """The engine's static split-K factor of a row-parallel projection (b200rwkv_engine::pick_split, one GPU)."""
    if K % 128:
        return 1
    best = 1
    for s in range(2, 9):
        if (K // 128) % s == 0 and tiles * s <= num_sms():
            best = s
    return best


@functools.lru_cache(maxsize=8)
def weights(N: int, K: int, seed: int, edge: bool = False, positive: bool = False) -> np.ndarray:
    """f16 [N, K] with unit-variance outputs for unit inputs; `edge` adds the rows that stress the quantisers (constant block,
    zero row, linear ramp, one outlier, exact NF4 levels and the midpoints between them)."""
    rng = np.random.default_rng(seed)
    if positive:
        w = rng.random((N, K), dtype=np.float32) * np.float32(2.0 / K)
    else:
        w = rng.standard_normal((N, K), dtype=np.float32) * np.float32(K ** -0.5)
    w = w.astype(np.float16)
    if edge:
        w[3, :128] = np.float16(0.125)
        w[5, :] = 0
        w[7, 128:256] = np.linspace(-1, 1, 128).astype(np.float16)
        w[9, 0] = np.float16(60000.0)
        w[11, :64] = (Q.NF4_LEVELS[:, None].repeat(4, 1).reshape(-1) * 0.5).astype(np.float16)
        w[12, :15] = ((Q.NF4_LEVELS[:-1] + Q.NF4_LEVELS[1:]) / 2).astype(np.float16)
        w[12, 15] = 1.0
    w.setflags(write=False)
    return w


@functools.lru_cache(maxsize=4)
def dequantised(N: int, K: int, seed: int, edge: bool, qtype: int) -> np.ndarray:
    w = weights(N, K, seed, edge)
    if qtype == capi.QUANT_INT8:
        return Q.dequant_int8(*Q.quant_int8(w), contract="engine")
    return Q.dequant_nf4(*Q.quant_nf4(w), contract="engine")


def act64(z, act):
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    with np.errstate(over="ignore"):
        if act == capi.ACT_TANH:
            return np.tanh(z)
        if act == capi.ACT_SIGMOID:
            return sig(z)
        if act == capi.ACT_SILU:
            return z * sig(z)
        if act == capi.ACT_RELU2:
            return np.maximum(z, 0.0) ** 2
        if act == capi.ACT_EXPNEGEXP:
            return np.exp(-np.exp(z))
        if act == capi.ACT_V7DECAY:
            return np.exp(-V7_DECAY * sig(z))
    return z


def seg(N, K, act=capi.ACT_NONE, mode=capi.OUT_F32, bias=False, grp=0, pad=5, seed=0, **kw):
    return dict(N=N, K=K, act=act, out_mode=mode, has_bias=bias, grp=grp, pad=pad, seed=seed, **kw)


def run(name, T, segs, precision=0, quant=capi.QUANT_NONE, grid=0, launches=3, eps=EPS, x_fill=None):
    """Build inputs for every segment, run the plan through b200rwkv_op_gemm, check every slice of every segment against the
    float64 reference and the sentinels.  Returns the plan (grid, blocks, tiles, most contributors of one tile)."""
    rows = capi.gemm_rows(T, precision)
    rng = np.random.default_rng(zlib.crc32(repr((name, T, grid, precision, quant)).encode()))
    args = []
    for i, s in enumerate(segs):
        N, K = s["N"], s["K"]
        w = weights(N, K, 1000 + s["seed"] * 17 + i, s.get("edge", False), s.get("positive", False))
        if x_fill is not None:
            a = np.full((T, K), x_fill, np.float32)
        elif s.get("positive"):
            a = rng.random((T, K), dtype=np.float32)
        else:
            a = rng.standard_normal((T, K), dtype=np.float32)
        b = rng.standard_normal((T, K), dtype=np.float32) if x_fill is None else a * np.float32(0.5)
        x = np.stack([a, b, a][:launches]) if launches == 3 else np.stack([a] * launches)
        ldo = N + s["pad"]
        a16 = s["out_mode"] != capi.OUT_F32
        out = np.empty((launches, rows, ldo), np.uint16 if a16 else np.float32)
        out.view(np.uint16 if a16 else np.uint32)[...] = SENT16 if a16 else SENT32
        d = dict(w=w, x=x, act=s["act"], out_mode=s["out_mode"], grp=s["grp"], out=out)
        if s["has_bias"]:
            d["bias"] = rng.standard_normal(N, dtype=np.float32) * np.float32(0.5)
        if s["out_mode"] == capi.OUT_LERP_A16:
            xx = rng.standard_normal((T, N), dtype=np.float32)
            sx = rng.standard_normal((T, N), dtype=np.float32)
            d["xx"], d["sx"] = np.stack([xx, sx * 2, xx][:launches]), np.stack([sx, xx, sx][:launches])
            d["mu"] = rng.standard_normal(N, dtype=np.float32) * np.float32(0.5)
        args.append(d)
    plan = capi.op_gemm(T, args, precision=precision, quant_type=quant, grid=grid, launches=launches)
    worst = 0.0
    for i, (s, d) in enumerate(zip(segs, args)):
        worst = max(worst, check(s, d, T, precision, quant, eps, 1000 + s["seed"] * 17 + i))
    print(f"\n[gemm] {name} T={T} p{precision} q{quant} grid={grid}: plan {plan}, worst |err|/bound = {worst:.4f}")
    return plan


def project64(xf, w, bias, act, eps=EPS, dz=0.0):
    """float64 act(xf W^T + bias) of operand rows xf [M, K] (the values the kernel multiplies) and its per-element bound
    before any f16 hand-off: eps sum_k |x_k W_nk| + dz (an error the caller knows its operand carries, already multiplied
    through |W|) and the bias add, carried through the activation over the interval it spans, plus a few f32 ulps."""
    N = w.shape[0]
    xa = np.abs(xf)
    z = np.empty((xf.shape[0], N))
    S = np.empty_like(z)
    for n0 in range(0, N, 8192):                               # the 65536-row head in chunks
        wc = w[n0:n0 + 8192].astype(np.float64)
        z[:, n0:n0 + 8192] = xf @ wc.T
        S[:, n0:n0 + 8192] = xa @ np.abs(wc).T
    if bias is not None:
        z += np.asarray(bias, np.float64)
    e = eps * S + dz + 2.0 ** -22 * np.abs(z)                  # error of the pre-activation value (accumulation, bias add)
    y = act64(z, act)
    dev = np.maximum(np.abs(act64(z - e, act) - y), np.abs(act64(z + e, act) - y))
    return y, dev + 8 * 2.0 ** -24 * np.abs(y) + 1e-30


def check(s, d, T, precision, quant, eps, wseed):
    N, K = s["N"], s["K"]
    out, launches = d["out"], d["x"].shape[0]
    split = precision == 1
    a16 = s["out_mode"] != capi.OUT_F32
    w = dequantised(N, K, wseed, s.get("edge", False), quant) if quant else d["w"]
    x = d["x"].astype(np.float64) if split else d["x"].astype(np.float16).astype(np.float64)
    y, bound = project64(x.reshape(-1, K), w, d.get("bias"), s["act"], eps)
    y, bound = y.reshape(launches, T, N), bound.reshape(launches, T, N)
    if s["out_mode"] == capi.OUT_LERP_A16:
        xx, sx, mu = (d[k].astype(np.float64) for k in ("xx", "sx", "mu"))
        lerp = xx + sx * (mu + y)
        bound = np.abs(sx) * bound + 2.0 ** -22 * (np.abs(xx) + np.abs(sx) * (np.abs(mu) + np.abs(y))) + 1e-30
        y = lerp
    written = np.zeros(out.shape[1:], bool)
    if a16:
        f = lambda r: out[:, r, :N].view(np.float16).astype(np.float64)
        if split:                                              # hi + lo halves of the same 16 tokens
            got = f(slice(0, T)) + f(slice(16, 16 + T))
            bound = bound + 2.0 ** -21 * np.abs(y) + 2.0 ** -24
            written[16:16 + T, :N] = True
        else:
            got = f(slice(0, T))
            y = np.clip(y, -F16_MAX, F16_MAX)                  # f16 outputs saturate
            with np.errstate(over="ignore"):                   # the spacing above 65504 is inf: one ulp there is 32
                ulp = np.minimum(np.spacing(np.abs(y).astype(np.float16)).astype(np.float64), 32.0)
            bound = bound + ulp
    else:
        got = out[:, :T, :N].astype(np.float64)
    written[:T, :N] = True
    ratio = np.abs(got - y) / bound
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    worst = float(ratio.max())
    bad = np.argwhere(ratio > 1.0)
    assert worst <= 1.0, (f"{len(bad)} cells over the bound, first (launch, token, column) {tuple(bad[0])}: "
                          f"got {got[tuple(bad[0])]!r}, want {y[tuple(bad[0])]!r}, bound {bound[tuple(bad[0])]!r}")
    bits = out.view(np.uint16 if a16 else np.uint32)
    assert (bits[:, ~written] == (SENT16 if a16 else SENT32)).all(), "a cell outside [T, N] was written"
    if launches == 3:
        assert np.array_equal(bits[0], bits[2]), "the same input gave different bits in launch 0 and launch 2"
    return worst


# ----------------------------------------------------------------------------------------------------------------------
# token counts: every token-tile bucket, partial last tiles, the production plan and a forced prime grid
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", [0, 7])
@pytest.mark.parametrize("T", [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128])
def test_token_counts(T, grid):
    segs = [seg(320, 320, bias=True, pad=3), seg(136, 320, capi.ACT_TANH, capi.OUT_A16, pad=8)]
    plan = run("tokens", T, segs, grid=grid)
    if grid == 0:
        assert plan == (5, 15, 5, 1)          # 5 tiles of 3 k blocks each: whole tiles per CTA, no fix-up
    else:
        assert plan[:3] == (7, 15, 5) and plan[3] == 2 and plan[1] % plan[0] != 0


# ----------------------------------------------------------------------------------------------------------------------
# N (row masking, tile counts) and K (padding, k-block counts)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K,T", [
    (8, 64, 1), (96, 96, 2), (120, 128, 17), (128, 320, 33), (136, 2560, 16), (320, 4096, 65), (2560, 14336, 1),
    (4096, 2560, 128), (14336, 4096, 16), (4096, 4096, 64), (8, 14336, 100), (14336, 64, 31)])
def test_shapes(N, K, T):
    run("shape", T, [seg(N, K, bias=True)])


@pytest.mark.parametrize("T", [1, 16])
def test_vocabulary_head(T):
    plan = run("head", T, [seg(65536, 4096, pad=0)], launches=1)
    assert plan[1:3] == (16384, 512)


def test_positive_operands_at_k_14336():
    """No cancellation: sum |x W| = y, so the bound is as tight as it gets, along the longest K of the models."""
    segs = [seg(256, 14336, positive=True)]
    run("positive", 16, segs)
    plan = run("positive", 16, segs, grid=2 * 112)         # one block per CTA: 112 partial tiles summed by the fix-up
    assert plan == (224, 224, 2, 112)


# ----------------------------------------------------------------------------------------------------------------------
# the launches of the real models
# ----------------------------------------------------------------------------------------------------------------------
def launch_7b_rkvg(C=4096, Dd=128):
    return [seg(C, C), seg(C, C), seg(C, C), seg(C, C, capi.ACT_SILU), seg(Dd, C, capi.ACT_TANH, capi.OUT_A16)], 0


def launch_row_parallel(N, K):
    """O / channel-mix value: K cut into static slices, one partial output each, grid = tiles x slices (whole tiles)."""
    tiles = -(-N // 128)
    S = pick_split(K, tiles)
    return [seg(N, K // S, seed=sp) for sp in range(S)], (tiles * S if S > 1 else 0)


LAUNCHES = {
    "7b-rkvg-wd1": (16, lambda: launch_7b_rkvg()),
    "7b-wd2": (16, lambda: ([seg(4096, 128, capi.ACT_EXPNEGEXP, bias=True)], 0)),
    "7b-o": (16, lambda: launch_row_parallel(4096, 4096)),
    "7b-ffn-kr": (16, lambda: ([seg(14336, 4096, capi.ACT_RELU2, capi.OUT_A16), seg(4096, 4096, capi.ACT_SIGMOID)], 0)),
    "7b-ffn-v": (16, lambda: launch_row_parallel(4096, 14336)),
    "3b-rkvg-wd1": (1, lambda: launch_7b_rkvg(2560, 64)),
    "v7-lora1": (8, lambda: ([seg(96, 2560, capi.ACT_TANH, capi.OUT_A16), seg(96, 2560, mode=capi.OUT_A16),
                             seg(64, 2560, mode=capi.OUT_A16), seg(320, 2560, capi.ACT_SIGMOID, capi.OUT_A16)], 0)),
    "v7-lora2": (8, lambda: ([seg(2560, 96, capi.ACT_V7DECAY, bias=True), seg(2560, 96, capi.ACT_SIGMOID, bias=True),
                             seg(2560, 64, capi.ACT_SIGMOID, bias=True), seg(2560, 320)], 0)),
    "v7-ffn-k": (8, lambda: ([seg(10240, 2560, capi.ACT_RELU2, capi.OUT_A16)], 0)),
    "v6-ddlerp-w1": (16, lambda: ([seg(5 * 64, 4096, capi.ACT_TANH, capi.OUT_A16, grp=64, pad=64)], 0)),
    "v6-ddlerp-w2": (16, lambda: ([seg(4096, 64, mode=capi.OUT_LERP_A16, seed=i) for i in range(5)], 0)),
}


@pytest.mark.parametrize("name", list(LAUNCHES))
def test_model_launches(name):
    T, make = LAUNCHES[name]
    segs, grid = make()
    plan = run(name, T, segs, grid=grid)
    if name == "3b-rkvg-wd1":
        # 81 tiles of 20 blocks: the production grid cuts them unevenly, several CTAs per tile
        assert plan[1] % plan[0] != 0 and plan[3] > 1


# ----------------------------------------------------------------------------------------------------------------------
# forced grids: one CTA for everything, one block per CTA (32 contributors to a K = 4096 tile), a prime in between
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["one", "blocks", "prime"])
@pytest.mark.parametrize("T", [16, 32, 64, 128])
def test_forced_grids(T, which):
    segs = [seg(256, 4096, bias=True), seg(128, 4096, capi.ACT_SIGMOID, capi.OUT_A16), seg(96, 320, capi.ACT_SILU, pad=0)]
    blocks = 2 * 32 + 32 + 3
    grid = {"one": 1, "blocks": blocks, "prime": 37}[which]
    plan = run("forced", T, segs, grid=grid)
    assert plan[:3] == (grid, blocks, 4)
    if which == "blocks":
        assert plan[3] == 32                  # > 4 contributors at one token tile, > 2 at two: several rounds of the fix-up
    if which == "prime":
        assert plan[1] % plan[0] != 0 and plan[3] > 1


# ----------------------------------------------------------------------------------------------------------------------
# precision 1: f32 inputs as f16 hi + lo operand pairs
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 5, 16])
@pytest.mark.parametrize("name", ["3b-rkvg-wd1", "v7-lora1", "v6-ddlerp-w2"])
def test_precision1_launches(name, T):
    segs, grid = LAUNCHES[name][1]()
    run(name, T, segs, precision=1, grid=grid)


def test_precision1_lo_half_counts():
    """x = 1 + 2^-12 rounds to 1 in f16: only the lo operand carries the 2^-12, and the bound is four times tighter than the
    error a plain f16 operand would make."""
    segs = [seg(128, 512, positive=True), seg(128, 512, mode=capi.OUT_A16, positive=True, seed=1)]
    x = 1.0 + 2.0 ** -12
    assert np.float16(x) == 1.0
    run("lo-half", 4, segs, precision=1, x_fill=x, eps=2.0 ** -16)
    run("lo-half", 4, segs, precision=1, x_fill=x, eps=2.0 ** -16, grid=8)


# ----------------------------------------------------------------------------------------------------------------------
# Int8 / NF4 weights, expanded in shared memory in front of the MMAs
# ----------------------------------------------------------------------------------------------------------------------
QCASES = [((200, 384), T, 0) for T in (1, 16, 17, 64, 128)] + [((200, 384), 16, 1), ((200, 384), 17, 6)] + [
    ((4096, 4096), 1, 0), ((4096, 4096), 64, 0), ((4096, 4096), 16, 29), ((14336, 4096), 16, 0), ((14336, 4096), 128, 0),
    ((4096, 14336), 1, 0), ((4096, 14336), 17, 0)]


@pytest.mark.parametrize("qtype", [capi.QUANT_INT8, capi.QUANT_NF4])
@pytest.mark.parametrize("shape,T,grid", QCASES)
def test_quantised(qtype, shape, T, grid):
    N, K = shape
    segs = [seg(N, K, edge=True)]
    if N == 200:
        segs.append(seg(N, K, capi.ACT_RELU2, capi.OUT_A16, edge=True, seed=1))
    plan = run("quant", T, segs, quant=qtype, grid=grid)
    if grid == 6:                             # 6 blocks over 6 CTAs: every tile of 3 k blocks is cut
        assert plan == (6, 12, 4, 2)


# ----------------------------------------------------------------------------------------------------------------------
# f16 outputs saturate
# ----------------------------------------------------------------------------------------------------------------------
def test_f16_output_saturates():
    w = np.asarray(weights(16, 128, 7)).copy()
    w[0], w[1] = np.float16(1024), np.float16(-1024)
    x = np.full((1, 3, 128), 64.0, np.float32)              # row 0: 64 * 1024 * 128 = 8.4e6
    out = np.empty((1, 16, 16), np.uint16)
    out[...] = SENT16
    capi.op_gemm(3, [dict(w=w, x=x, out_mode=capi.OUT_A16, out=out)])
    assert (out[0, :3, 0] == 0x7BFF).all() and (out[0, :3, 1] == 0xFBFF).all()     # +-65504, not inf
    assert np.isfinite(out[0, :3].view(np.float16)).all() and (out[0, 3:] == SENT16).all()
