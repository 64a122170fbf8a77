"""The kernels that prepare weights at load (csrc/misc.cuh lora_blend_kernel, f16_to_f32_kernel, decay_table_kernel and
csrc/gemm.cuh repack_weight_kernel), each alone through b200rwkv_op_weight with the launch shape the model build gives it,
against an exact reference.  Whole-model logits see these kernels only through a 1e-3 tolerance; here every output is
compared bit for bit, except the decay table, whose bound is derived below.

Arithmetic the references model:
  - nvcc contracts `a * b + c` in these kernels to one FFMA (the default --fmad=true; `cuobjdump -sass` of the sm_90a library shows
    `FFMA acc, alpha, w` feeding F2FP.F16.F32 in lora_blend_kernel, one FFMA in f16_to_f32_kernel, and no FMUL / FADD in
    either).  fma_f32 below rounds a * b + c
    once, exactly: a * b of two f32 values is exact in float64 (24 + 24 significant bits), and TwoSum gives the exact
    float64 sum s plus its error e, so s + e is the exact result.  Rounding s to f32 is one correct rounding of s + e except
    when s is exactly halfway between two f32 neighbours and e != 0, where the sign of e picks the side.
    test_fma_f32_is_one_rounding checks this against fractions.Fraction.
  - lora_blend_kernel: acc = fmaf(b[k], a[k], acc) for k = 0 .. r-1 from +0.0.  b[k] * a[k] of two f16 values has at most
    22 significant bits and lies in [2^-48, 2^32]: it is exact in f32, so each fmaf is one round-to-nearest f32 addition and
    the chain equals an ordered f32 add chain.  Then w' = f16_rn(fma_f32(alpha, acc, f32(w))).  Two LoRAs blend one after
    the other, each rounding to f16.
  - f16_to_f32_kernel: dst = fma_f32(f32(src), scale, bias).
  - repack_weight_kernel: written from the layout in gemm.cuh's comment, block(tile, kb) = [k8 chunk 16][row group 16][row 8]
    [8 halves], zero padded, not from the kernel's index arithmetic.
"""
from fractions import Fraction

import numpy as np
import pytest

from ai00_server_b200 import capi

gpu = pytest.mark.gpu
f16, f32, f64 = np.float16, np.float32, np.float64


# ---- references ----

def fma_f32(a, b, c):
    """a * b + c for f32 arrays, rounded once to f32 (nearest, ties to even): what one FFMA computes."""
    a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
    p = a.astype(f64) * b.astype(f64)                       # exact
    c64 = c.astype(f64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                         # TwoSum: s + e == p + c exactly
    r = s.astype(f32)
    r64 = r.astype(f64)
    other = np.nextafter(r, np.where(s > r64, f32(np.inf), f32(-np.inf)).astype(f32))    # the f32 neighbour on s's side
    o64 = other.astype(f64)
    tie = (r64 != s) & ((r64 + o64) / 2 == s) & (e != 0)
    return np.where(tie & (np.sign(e) == np.sign(o64 - r64)), other, r)


def round_f32_exact(x: Fraction) -> np.float32:
    """The f32 nearest to the rational x, ties to even (finite, nonzero results only)."""
    f = f32(float(x))
    cands = [np.nextafter(f, f32(-np.inf)), f, np.nextafter(f, f32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c, f32).view(np.uint32)) & 1))


def lora_ref(w16, b16, a16, alpha):
    """f16(f32(w) + alpha * acc) with acc the ordered f32 sum of the exact products b[o][j] a[i][j]."""
    bf, af = b16.astype(f32), a16.astype(f32)
    acc = np.zeros((bf.shape[0], af.shape[0]), f32)
    for j in range(bf.shape[1]):
        p = np.outer(bf[:, j], af[:, j])                   # f32
        assert np.array_equal(p.astype(f64), np.outer(bf[:, j].astype(f64), af[:, j].astype(f64)))    # exact in f32
        acc = acc + p
    return fma_f32(f32(alpha), acc, w16.astype(f32)).astype(f16)


def repack_ref(src, n0, k0, N, K):
    """Rows [n0, n0 + N), columns [k0, k0 + K) of src as blocks [tiles][KB][k8 16][row group 16][row 8][8 halves], zero padded:
    element (tile, kb, k8, g, row, e) is sub[tile * 128 + 8 g + row][kb * 128 + 8 k8 + e]."""
    tiles, KB = -(-N // 128), -(-K // 128)
    sub = np.zeros((tiles * 128, KB * 128), np.uint16)
    sub[:N, :K] = src.view(np.uint16)[n0:n0 + N, k0:k0 + K]
    return sub.reshape(tiles, 16, 8, KB, 16, 8).transpose(0, 3, 4, 1, 2, 5)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint16 if a.dtype == f16 else np.uint32)


def finite_f16():
    """Every finite f16 value, +-0 and the subnormals included (63488 values)."""
    x = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(f16)
    return x[np.isfinite(x)]


def random_f16(rng, shape, scale=1.0):
    return (rng.uniform(-scale, scale, shape)).astype(f16)


# ---- the reference itself ----

def test_fma_f32_is_one_rounding():
    """fma_f32 equals the exactly rounded a * b + c on random operands, on operands whose sum is exact, and on constructed
    ties: c an f32 halfway point minus / plus a tiny product, where rounding the float64 sum would pick the wrong side."""
    rng = np.random.default_rng(7)
    a = rng.standard_normal(3000).astype(f32) * f32(2) ** rng.integers(-30, 30, 3000).astype(f32)
    b = rng.standard_normal(3000).astype(f32)
    c = rng.standard_normal(3000).astype(f32) * f32(2) ** rng.integers(-30, 30, 3000).astype(f32)
    # ties: c = 1 + 2^-23 (odd), a * b = +-(1 + 2^-23)(1 - 2^-23) 2^-24 = +-(2^-24 - 2^-70).  The float64 sum loses the 2^-70
    # and lands on the halfway point 1 + 3 * 2^-24 (resp. 1 + 2^-24), where ties-to-even picks the side away from the exact sum
    a_t = np.array([1.0 + 2.0 ** -23, -(1.0 + 2.0 ** -23)], f64) * 2.0 ** -24
    b_t = np.full(2, 1.0 - 2.0 ** -23)
    c_t = np.full(2, 1.0 + 2.0 ** -23)
    a, b, c = (np.concatenate([x, y.astype(f32)]) for x, y in ((a, a_t), (b, b_t), (c, c_t)))
    got = fma_f32(a, b, c)
    for i in range(a.size):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        want = round_f32_exact(exact) if exact != 0 else f32(0)
        assert np.array(got[i], f32).view(np.uint32) == np.array(want, f32).view(np.uint32) or (exact == 0 and got[i] == 0), i
    assert np.array_equal(got[-2:], np.full(2, 1.0 + 2.0 ** -23, f32))
    # the constructed cases really are float64 double-rounding traps
    s64 = a_t * b_t + c_t
    assert np.all(s64.astype(f32) != got[-2:])


def test_repack_reference_reads_the_documented_layout():
    """repack_ref's block order, spelled out element by element for one small sub-matrix."""
    src = np.arange(300 * 140, dtype=np.uint32).astype(np.uint16).view(f16).reshape(300, 140)
    n0, k0, N, K = 3, 5, 130, 131
    blk = repack_ref(src, n0, k0, N, K)
    assert blk.shape == (2, 2, 16, 16, 8, 8)
    s16 = src.view(np.uint16)
    rng = np.random.default_rng(0)
    for tile, kb, k8, g, row, e in zip(*(rng.integers(0, m, 500) for m in (2, 2, 16, 16, 8, 8))):
        n, k = tile * 128 + 8 * g + row, kb * 128 + 8 * k8 + e
        want = s16[n0 + n, k0 + k] if n < N and k < K else 0
        assert blk[tile, kb, k8, g, row, e] == want


# ---- LoRA blend ----

LORA_CASES = [  # (out, in, r)
    (96, 136, 1), (136, 96, 7), (257, 40, 8), (40, 257, 64), (72, 200, 320), (640, 520, 8),
]


@gpu
@pytest.mark.parametrize("alpha", [0.75, -1.5, 0.0])
@pytest.mark.parametrize("out,inp,r", LORA_CASES)
def test_lora_blend_is_bit_exact(out, inp, r, alpha):
    """One LoRA pair: w' = f16(fma(alpha, acc, w)), acc the ordered f32 chain.  The matrix carries +-0, f16 subnormals and
    values near the f16 maximum, so rounding, signed zeros and overflow to inf are all exercised.  640 x 520 has more elements
    than the launch has threads (num_sms * 8 CTAs of 256): the grid-stride loop runs twice."""
    rng = np.random.default_rng(out * 1000 + inp + r)
    w = random_f16(rng, (out, inp))
    w.reshape(-1)[:6] = np.array([0.0, -0.0, 6e-8, -6e-8, 65504.0, -65000.0], f16)
    b = random_f16(rng, (out, r), np.sqrt(3.0 / r))
    a = random_f16(rng, (inp, r), np.sqrt(3.0 / r))
    got = capi.op_lora_blend(w, b, a, alpha)
    want = lora_ref(w, b, a, alpha)
    assert np.array_equal(bits(got), bits(want)), int((bits(got) != bits(want)).sum())
    if alpha != 0.0:
        assert not np.array_equal(got, w)


@gpu
def test_two_loras_round_to_f16_one_after_the_other():
    """Two LoRA pairs on one matrix, as b200rwkv_create_ex applies two LoRA files: each blend rounds to f16 before the next,
    which differs from blending the sum of the two updates once."""
    rng = np.random.default_rng(11)
    out, inp = 200, 136
    w = random_f16(rng, (out, inp))
    b1, a1 = random_f16(rng, (out, 7), 0.6), random_f16(rng, (inp, 7), 0.6)
    b2, a2 = random_f16(rng, (out, 64), 0.2), random_f16(rng, (inp, 64), 0.2)
    got = capi.op_lora_blend(capi.op_lora_blend(w, b1, a1, 0.75), b2, a2, -1.5)
    want = lora_ref(lora_ref(w, b1, a1, 0.75), b2, a2, -1.5)
    assert np.array_equal(bits(got), bits(want))
    acc1 = sum(np.outer(b1[:, j].astype(f64), a1[:, j].astype(f64)) for j in range(7))
    acc2 = sum(np.outer(b2[:, j].astype(f64), a2[:, j].astype(f64)) for j in range(64))
    once = (w.astype(f64) + 0.75 * acc1 - 1.5 * acc2).astype(f16)
    assert not np.array_equal(bits(got), bits(once))


# ---- f16 -> f32 vectors ----

@gpu
@pytest.mark.parametrize("scale,bias", [(1.0, 0.0), (-1.0, 1.0), (0.7, -0.3), (3.0e-5, 1.0e4)])
def test_f16_to_f32_is_one_fma(scale, bias):
    """dst = fma_f32(f32(src), scale, bias) over every finite f16 (the engine's vectors use (1, 0) and, for the RWKV-5 mixes,
    (-1, 1)), and over 1001 values, a count that is not a multiple of the 256-thread CTA."""
    x = finite_f16()
    for src in (x, np.random.default_rng(3).permutation(x)[:1001]):
        got = capi.op_vector(capi.WEIGHT_F32, src, scale, bias)
        want = fma_f32(src.astype(f32), f32(scale), f32(bias))
        assert np.array_equal(bits(got), bits(want)), int((bits(got) != bits(want)).sum())


# ---- RWKV-5 decay table ----

@gpu
def test_decay_table_within_the_derived_bound():
    """w = expf(-expf(x)) for every finite f16 x, against float64 exp(-exp(x)) = z.

    Bound, from CUDA's documented maximum error of expf, 2 ulp over its whole range (CUDA C Programming Guide, Mathematical
    Functions, single precision), u = 2^-24, ulp(v) <= 2u |v| for a normal v and 2^-149 below:
      - inner: y = expf(x) = e^x + d1 with |d1| <= D = 2^-22 e^x + 2^-148 (x = f32(f16) is exact, so is the negation);
      - outer: e^-y = z e^(-d1), so |e^-y - z| <= z (e^D - 1); expf(-y) = e^-y + d2 with |d2| <= 2^-22 e^-y + 2^-148
        <= 2^-22 z e^D + 2^-148;
      - together |w - z| <= z ((1 + 2^-22) e^D - 1) + 2^-148, plus the float64 reference's own error, under 2^-50 (1 + e^x) z.
    For x > 88.72 expf(x) is inf and w must be 0 (z is 0 in float64 too); for x below about -17, e^x < 2^-24 and w rounds
    to 1 within the bound.  The test also checks that these regions are reached: results of exactly 0 and exactly 1."""
    x = finite_f16()
    w = capi.op_vector(capi.WEIGHT_DECAY, x)
    x64 = x.astype(f64)
    with np.errstate(over="ignore", invalid="ignore"):
        ex = np.exp(x64)
        z = np.exp(-ex)
        D = 2.0 ** -22 * ex + 2.0 ** -148
        # z ((1 + 2^-22) e^D - 1) written as (1 + 2^-22) (e^(D - e^x) - z) + 2^-22 z, finite where e^D alone is not
        bound = (1 + 2.0 ** -22) * (np.exp(D - ex) - z) + 2.0 ** -22 * z + 2.0 ** -148 + 2.0 ** -50 * (1 + ex) * z
    bound = np.where(np.isfinite(ex), bound, 2.0 ** -148)
    err = np.abs(w.astype(f64) - z)
    assert np.all(np.isfinite(w)) and np.all(w >= 0) and np.all(w <= 1)
    assert np.all(err <= bound), float(np.max(err / bound))
    assert np.all(w[x64 > 88.8] == 0) and np.any(w == 0) and np.any(w == 1) and np.any((w > 0) & (w < 2.0 ** -126))
    print(f"\ndecay table: worst error / bound {float(np.max(err / bound)):.3g}")


# ---- repack ----

def rand_bits16(rng, shape):
    """Random f16 bit patterns without NaN / inf, so that a misplaced element almost never matches by accident."""
    b = rng.integers(0, 1 << 16, shape, dtype=np.uint32).astype(np.uint16)
    b[(b & 0x7C00) == 0x7C00] ^= 0x4000
    return b.view(f16)


REPACK_CASES = [  # (rows, ld, n0, k0, N, K)
    (256, 256, 0, 0, 256, 256),            # whole tiles, every chunk on the aligned path
    (256, 256, 128, 128, 128, 128),        # one aligned tile inside a larger matrix
    (300, 203, 5, 3, 290, 197),            # odd k0 and odd ld: every chunk on the scalar path; N % 128, K % 8 != 0
    (130, 1000, 1, 7, 129, 993),           # a tile of one row, a k block of 97 columns
    (40, 77, 2, 4, 37, 70),                # even k0, odd ld: rows alternate between aligned and unaligned starts
    (64, 264, 0, 8, 64, 250),              # aligned rows, a last chunk of 2 columns (scalar tail)
    (9, 16, 8, 0, 1, 1),                   # one element
]


@gpu
@pytest.mark.parametrize("rows,ld,n0,k0,N,K", REPACK_CASES)
def test_repack_is_bit_exact(rows, ld, n0, k0, N, K):
    src = rand_bits16(np.random.default_rng(rows * ld + n0 + k0), (rows, ld))
    got = capi.op_repack(src, n0, k0, N, K)
    assert np.array_equal(bits(got), repack_ref(src, n0, k0, N, K))


def pick_split(K, tiles, world, num_sms=132):
    """engine.cu pick_split: static K slices of a row-parallel projection (H100: 132 SMs)."""
    if K % 128:
        return 1
    best = 1
    for S in range(2, 8 // world + 1):
        if (K // 128) % S == 0 and tiles * S <= num_sms:
            best = S
    return best


@gpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_repack_small6_tensor_parallel_cuts(world):
    """Every sub-matrix a rank of small6 (C 512, F 1792, V 2048) repacks at this world size: column-parallel cuts (rows
    [r Cl, ...) of the C x C projections, [r Fl, ...) of ffn.key, [r Vl, ...) of the head) and row-parallel cuts (columns
    [r Cl + s Cl / S_att, ...) of att.output and [r Fl + s Fl / S_ffn, ...) of ffn.value, S the static K split).  At W = 8 a
    row-parallel att.output slice is 64 columns and an ffn slice 224: K blocks that are not whole."""
    C, F, V = 512, 1792, 2048
    Cl, Fl, Vl = C // world, F // world, V // world
    rng = np.random.default_rng(world)
    mats = {"CxC": rand_bits16(rng, (C, C)), "FxC": rand_bits16(rng, (F, C)), "CxF": rand_bits16(rng, (C, F)),
            "VxC": rand_bits16(rng, (V, C))}
    s_att, s_ffn = pick_split(Cl, C // 128, world), pick_split(Fl, C // 128, world)
    cuts = []
    for r in range(world):
        cuts += [("CxC", r * Cl, 0, Cl, C), ("FxC", r * Fl, 0, Fl, C), ("VxC", r * Vl, 0, Vl, C)]
        cuts += [("CxC", 0, r * Cl + s * (Cl // s_att), C, Cl // s_att) for s in range(s_att)]
        cuts += [("CxF", 0, r * Fl + s * (Fl // s_ffn), C, Fl // s_ffn) for s in range(s_ffn)]
    for name, n0, k0, N, K in cuts:
        got = capi.op_repack(mats[name], n0, k0, N, K)
        assert np.array_equal(bits(got), repack_ref(mats[name], n0, k0, N, K)), (name, n0, k0, N, K)
