"""NumPy restatement of the Int4 weight-only format (B200RWKV_QUANT_INT4, ai00_server_b200/csrc/int4gemm.cuh), shared by
tests/test_int4_cpu.py and tests/test_gpu_int4.py.  The format goes beyond the reference's `Quant` enum, so there is no
reference arithmetic to pin; what is restated is the format's definition and the engine contract.  It is oracle/quant_numpy.py's
Int8 at 4 bits:

* Blocks: runs of 128 consecutive inputs of one output row of the [N, K] f16 matrix.
* Parameters, in f32: mn = min, mx = max, rng = mx - mn; the block keeps scale = f16(rng / 15) and min = f16(mn) (exact).
* Codes: q = floor(15 clamp((w - mn) / rng, 0, 1) + 0.5), 0..15, every step an f32 operation rounded to nearest; a block with
  rng == 0 keeps q = 0.
* Engine contract: the weight is fma_f16(q, scale, min) -- the exact product plus min, rounded once to f16 -- which the tensor
  cores multiply with the f16 operand, accumulating in f32.
"""
from __future__ import annotations

import numpy as np

from oracle import quant_numpy as Q

QUANT_INT4 = 6
BLOCK = 128


def quant_int4(w16: np.ndarray):
    """[N, K] f16 -> (codes u8 0..15 [N, K], min f16 [N, K/128], scale f16 [N, K/128])."""
    w16 = np.asarray(w16, np.float16)
    n, k = w16.shape
    assert k % BLOCK == 0, "Int4 blocks are 128 consecutive input elements"
    b = w16.astype(np.float32).reshape(n, k // BLOCK, BLOCK)
    mn, mx = b.min(axis=2), b.max(axis=2)
    rng = (mx - mn).astype(np.float32)
    safe = np.where(rng > 0, rng, np.float32(1))
    x = ((b - mn[..., None]).astype(np.float32) / safe[..., None]).astype(np.float32)
    x = np.clip(x, np.float32(0), np.float32(1))
    q = np.floor((x * np.float32(15)).astype(np.float32) + np.float32(0.5)).astype(np.uint8)
    q[rng <= 0] = 0
    scale = (rng / np.float32(15)).astype(np.float32).astype(np.float16)
    return q.reshape(n, k), mn.astype(np.float16), scale


def dequant_int4(q: np.ndarray, mn16: np.ndarray, scale16: np.ndarray) -> np.ndarray:
    """fma_f16(q, scale, min): float64 product and sum (both exact), one rounding to f16."""
    n, k = q.shape
    qb = q.reshape(n, k // BLOCK, BLOCK).astype(np.float64)
    w = qb * scale16.astype(np.float64)[..., None] + mn16.astype(np.float64)[..., None]
    return w.astype(np.float16).reshape(n, k)


def quantize_model(weights: dict[str, np.ndarray], layers: int, qtype: int = QUANT_INT4,
                   contract: str = "engine") -> dict[str, np.ndarray]:
    """oracle/quant_numpy.py's quantize_model, with Int4 added: the eight projection matrices of the first `layers` layers."""
    if qtype != QUANT_INT4:
        return Q.quantize_model(weights, layers, qtype, contract)
    out = dict(weights)
    for l in range(layers):
        for m in Q.QUANT_MATRICES:
            name = f"blocks.{l}.{m}"
            if name in weights:
                out[name] = dequant_int4(*quant_int4(weights[name]))
    return out


def quant_weight_bytes(n: int, k: int, qtype: int = QUANT_INT4) -> int:
    """Bytes one pass over an [n, k] matrix streams: Int4 = half a byte per code + f16 (scale, min) per 128 inputs."""
    if qtype == QUANT_INT4:
        return n * k // 2 + (n * k // BLOCK) * 4
    return Q.quant_weight_bytes(n, k, qtype)
