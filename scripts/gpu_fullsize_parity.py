"""Engine vs the C/OpenMP oracle at a BASELINE shape (default v6-3b, B=2; use v6-7b on a machine with >= 64 host cores):
relative logits error against BOTH oracle contracts, argmax agreement, and the oracle-vs-oracle noise floor beside it
(see DESIGN.md §2, oracle/noise_floor.py).

    python scripts/gpu_fullsize_parity.py v6-3b 2 4
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth          # noqa: E402
from oracle import ref_c                                   # noqa: E402
from oracle import rwkv_numpy as O                         # noqa: E402

preset = sys.argv[1] if len(sys.argv) > 1 else "v6-3b"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 2
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 4
st = synth.make_st(preset, 0)
w = O.parse_st(st)
m = runtime.Model(st, max_batch=B, token_chunk_size=32)
c16, c32 = ref_c.RefC(w, "f16"), ref_c.RefC(w, "f32")
s16, s32 = c16.state_init(B), c32.state_init(B)
for s in range(B):
    m.state.load(m.state.init(), s)
rng = np.random.default_rng(3)
rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
for i in range(steps):
    toks = rng.integers(1, min(60000, c16.info.num_vocab), B)
    rows = np.concatenate(m.infer_raw(list(range(B)), [1] * B, toks.tolist(), [capi.OPTION_LAST] * B))
    a, b = c16.decode_step(toks, s16), c32.decode_step(toks, s32)
    print(f"{preset} step {i}: engine vs C f16-contract {rel(rows, a):.2e} | engine vs C f32-contract {rel(rows, b):.2e} | "
          f"C f16 vs C f32 {rel(a, b):.2e} | argmax engine==f16 {(rows.argmax(1) == a.argmax(1)).all()} engine==f32 "
          f"{(rows.argmax(1) == b.argmax(1)).all()}", flush=True)
m.close()
