"""NumPy restatement of the FP8 (E4M3) weight-only format (B200RWKV_QUANT_FP8, ai00_server_b200/csrc/fp8gemm.cuh), shared by
tests/test_fp8_cpu.py, tests/test_gpu_fp8.py and scripts/gpu_fp8.py.  The format goes beyond the reference's `Quant` enum, so
there is no reference arithmetic to pin; what is restated is the format's definition and the engine contract:

* E4M3 (the OCP 8-bit floating point "E4M3" / torch.float8_e4m3fn): sign, 4 exponent bits with bias 7, 3 mantissa bits;
  exponent 0 is subnormal (m / 8 * 2^-6), S.1111.111 is NaN, there are no infinities and the largest finite value is 448.
* Scale: for output row n of the whole [N, K] f16 matrix, a = max_k |w_nk| and s_n = a / 448, in f32 (round to nearest).
* Codes: q_nk = e4m3(w_nk / s_n), the f32 quotient rounded to nearest even and saturated to +-448.  A zero row keeps s_n = 0
  and +0 codes.
* Engine contract: the tensor cores multiply each code's exact value with the f16 operand and accumulate in f32; each output
  is multiplied by s_n in f32.  The forward-pass oracle therefore multiplies with f32(s_n * value(q)).
"""
from __future__ import annotations

import numpy as np

from oracle import quant_numpy as Q

QUANT_FP8 = 4
E4M3_MAX = 448.0


def e4m3_value(code: int) -> float:
    """The value of one E4M3 code, from the format definition."""
    sign = -1.0 if code & 0x80 else 1.0
    e, m = (code >> 3) & 15, code & 7
    if e == 15 and m == 7:
        return float("nan")
    if e == 0:
        return sign * (m / 8.0) * 2.0 ** -6
    return sign * (1.0 + m / 8.0) * 2.0 ** (e - 7)


E4M3_VALUES = np.array([e4m3_value(c) for c in range(256)], np.float64)    # exact in f16, f32 and f64
_POS = E4M3_VALUES[:127]                                                     # codes 0x00 .. 0x7E: +0 .. 448, ascending
_MID = (_POS[:-1] + _POS[1:]) / 2                                            # exact in f64


def e4m3_decode(q) -> np.ndarray:
    return E4M3_VALUES[np.asarray(q, np.uint8)]


def e4m3_encode(x) -> np.ndarray:
    """f32 -> E4M3 codes: round to nearest, ties to the even code (= even mantissa), magnitudes above 448 saturate to 448,
    NaN -> 0x7F; the sign bit is kept (-0 -> 0x80)."""
    x = np.asarray(x, np.float32)
    a = np.abs(x).astype(np.float64)
    i = np.searchsorted(_MID, a, side="left")              # _MID[i - 1] < a <= _MID[i]: nearest code i, or a tie with i + 1
    tie = (i < len(_MID)) & (a == _MID[np.minimum(i, len(_MID) - 1)])
    i = np.where(tie & (i % 2 == 1), i + 1, i)
    q = i.astype(np.uint8) | (np.signbit(x).astype(np.uint8) << 7)
    return np.where(np.isnan(x), np.uint8(0x7F), q).astype(np.uint8)


def quant_fp8(w16: np.ndarray):
    """[N, K] f16 -> (codes u8 [N, K], scale f32 [N])."""
    w = np.asarray(w16, np.float16).astype(np.float32)
    a = np.abs(w).max(axis=1)
    s = (a / np.float32(E4M3_MAX)).astype(np.float32)
    safe = np.where(a > 0, s, np.float32(1))
    q = e4m3_encode((w / safe[:, None]).astype(np.float32))
    q[a <= 0] = 0
    return q, s


def dequant_fp8(q: np.ndarray, s: np.ndarray) -> np.ndarray:
    """f32(s_n * value(q_nk)): the weights the engine contract multiplies with."""
    return (np.asarray(s, np.float32)[:, None] * e4m3_decode(q).astype(np.float32)).astype(np.float32)


def quantize_model(weights: dict[str, np.ndarray], layers: int, qtype: int, contract: str = "engine") -> dict[str, np.ndarray]:
    """oracle/quant_numpy.py's quantize_model, with FP8 added: the eight projection matrices of the first `layers` layers."""
    if qtype != QUANT_FP8:
        return Q.quantize_model(weights, layers, qtype, contract)
    out = dict(weights)
    for l in range(layers):
        for m in Q.QUANT_MATRICES:
            name = f"blocks.{l}.{m}"
            if name in weights:
                out[name] = dequant_fp8(*quant_fp8(weights[name]))
    return out


def quant_weight_bytes(n: int, k: int, qtype: int) -> int:
    """Bytes one pass over an [n, k] matrix streams: FP8 = one byte per code + one f32 scale per row."""
    if qtype == QUANT_FP8:
        return n * k + n * 4
    return Q.quant_weight_bytes(n, k, qtype)
