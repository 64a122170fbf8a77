"""How far apart can two correct implementations of the same contract be at full depth?

TEST INFRASTRUCTURE (CPU only).  On a synthetic model of the given preset this compares, token by token,
  (a) the C/OpenMP oracle under the f16-operand contract vs the same code under the pure-f32 contract, and
  (b) the C oracle vs the NumPy oracle, both under the f16-operand contract (they differ only in f32 summation order).
(b) is the noise floor of ANY parity check at that depth: a rounding flip of one f16 operand is 1e-3 of that element and
32 layers of LayerNorm + projections amplify it.

    python -m oracle.noise_floor v6-3b [steps]
"""
import sys
import time

import numpy as np

from ai00_server_b200 import synth
from oracle import ref_c
from oracle import rwkv_numpy as O


def main():
    preset = sys.argv[1] if len(sys.argv) > 1 else "v6-3b"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    w = O.parse_st(synth.make_st(preset, 0))
    rng = np.random.default_rng(0)
    c16, c32, n16 = ref_c.RefC(w, "f16"), ref_c.RefC(w, "f32"), O.Oracle(w, "f16")
    s16, s32, sn = c16.state_init(1), c32.state_init(1), n16.state_init()
    for step in range(steps):
        tok = int(rng.integers(1, min(60000, c16.info.num_vocab)))
        t0 = time.time()
        a = c16.decode_step([tok], s16)[0]
        b = c32.decode_step([tok], s32)[0]
        want, sn = n16.run([tok], sn)
        n = want[0]
        rel = lambda x, y: float(np.abs(x - y).max() / np.abs(y).max())
        print(f"{preset} step {step}: C f16-contract vs C f32-contract {rel(a, b):.2e} | C f16 vs NumPy f16 {rel(a, n):.2e} | "
              f"argmax equal {a.argmax() == b.argmax() == n.argmax()} | {time.time() - t0:.1f} s", flush=True)


if __name__ == "__main__":
    main()
