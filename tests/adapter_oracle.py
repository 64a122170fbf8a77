"""The unblended adapter path on top of the NumPy oracle, shared by the adapter tests (tests/test_adapters_cpu.py,
tests/test_gpu_adapters.py): what an engine from b200rwkv_create_adapters computes for a slot bound to one adapter."""
import numpy as np

from oracle import rwkv_numpy as O


class AdapterOracle(O.Oracle):
    """The oracle with one adapter applied unblended, as an engine from b200rwkv_create_adapters runs a bound slot: every
    projection W with a pair computes W q(x) + f16(alpha lora.1) r(lora.0^T q(x)), r rounding u like an operand (f16 in the
    "f16" contract; the hi + lo pair of precision 1 is f32 to ~2^-22, so none in "f32")."""

    def __init__(self, weights, act="f16", adapter=None):
        super().__init__(weights, act)
        self.adapter = adapter          # (lora dict, alpha) or None

    def _mv(self, name, x):
        y = super()._mv(name, x)
        if self.adapter is not None and name.endswith(".weight"):
            lora, alpha = self.adapter
            base = name[:-7]
            if base + ".lora.0" in lora:
                u = self._q(O._f(lora[base + ".lora.0"]).T @ self._q(x))
                bb = (np.float32(alpha) * O._f(lora[base + ".lora.1"])).astype(np.float16).astype(np.float32)
                y = y + bb @ u
        return y
