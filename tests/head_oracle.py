"""The quantised vocabulary head (b200rwkv_head_format) on top of the NumPy oracles, shared by tests/test_quant_head_cpu.py and
tests/test_gpu_quant_head.py: head.weight through the quantiser of a quantised layer's matrices, in each of the four formats
(oracle/quant_numpy.py for Int8 and NF4, tests/fp8_oracle.py for FP8, tests/int4_oracle.py for Int4)."""
from __future__ import annotations

import numpy as np

from oracle import quant_numpy as Q

import fp8_oracle as F8
import int4_oracle as I4

QUANT_INT8, QUANT_NF4, QUANT_FP8, QUANT_INT4 = Q.QUANT_INT8, Q.QUANT_NF4, F8.QUANT_FP8, I4.QUANT_INT4

# each format's quantize_model: the layers' arithmetic, which the engine applies to head.weight too
QUANTIZE = {QUANT_INT8: Q.quantize_model, QUANT_NF4: Q.quantize_model, QUANT_FP8: F8.quantize_model, QUANT_INT4: I4.quantize_model}


def quantize_head(weights: dict[str, np.ndarray], qtype: int, contract: str = "engine") -> dict[str, np.ndarray]:
    """The weights the forward pass multiplies with after `b200rwkv_head_format(qtype)`: head.weight as a quantised layer
    matrix of that format, everything else as given (so it composes with a quantize_model of the layers)."""
    out = dict(weights)
    if qtype == Q.QUANT_NONE:
        return out
    probe = "blocks.0.att.key.weight"          # any name quantize_model quantises in layer 0
    out["head.weight"] = QUANTIZE[qtype]({probe: weights["head.weight"]}, 1, qtype, contract)[probe]
    return out


def head_bytes(V: int, C: int, qtype: int) -> int:
    """Bytes one pass over the quantised head streams (codes + block parameters)."""
    return (F8 if qtype == QUANT_FP8 else I4).quant_weight_bytes(V, C, qtype)
