"""Cost of snapshots inside an infer call (b200rwkv_infer_snapshots), on one GPU.

  verify:  7B shape, one SCORE entry of 4 tokens per slot, ms per call with no snapshots, with 4 new snapshots per slot
           (allocated and freed every call) and with 4 reused ones, at batch 16 and 1.
  prefix:  16 slots x 512 tokens of NONE entries, one snapshot per entry at token 256, against the same prefill without
           snapshots and against the cut route (infer 256, state_read, infer 256).

Prints one JSON line with the card's name and power limit.  python scripts/gpu_snapshots.py [--preset v6-7b]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) * 1e3 / reps      # every call ends in a device synchronise


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    st = synth.make_st(a.preset, 0)
    m = runtime.Model(st, max_batch=16, token_chunk_size=128)
    V = m.info["num_vocab"]
    rng = np.random.default_rng(0)
    out = {"card": card(), "preset": a.preset}
    for B in (16, 1):
        slots = list(range(B))
        toks = [int(x) for x in rng.integers(0, V, 4 * B)]
        at = [(e, p) for e in range(B) for p in range(1, 5)]
        args = (slots, [4] * B, toks, [capi.OPTION_SCORE] * B)

        def fresh():
            for s in m.infer_snapshots(*args, at)[2]:
                s.free()

        reuse = m.infer_snapshots(*args, at)[2]
        out[f"verify_b{B}_ms"] = {
            "none": timed(lambda: m.infer_ex(*args), a.reps),
            "new": timed(fresh, a.reps),
            "reused": timed(lambda: m.infer_snapshots(*args, at, reuse=reuse), a.reps),
        }
        for s in reuse:
            s.free()
    slots = list(range(16))
    toks = [int(x) for x in rng.integers(0, V, 512 * 16)]
    opt = [capi.OPTION_NONE] * 16
    half = [t for s in slots for t in toks[s * 512:s * 512 + 256]], [t for s in slots for t in toks[s * 512 + 256:(s + 1) * 512]]

    def cut():
        m.infer_ex(slots, [256] * 16, half[0], opt)
        snaps = [m.state.read(s) for s in slots]
        m.infer_ex(slots, [256] * 16, half[1], opt)
        return snaps

    reuse = m.infer_snapshots(slots, [512] * 16, toks, opt, [(s, 256) for s in slots])[2]
    reps = max(3, a.reps // 4)

    def cut_free():
        for s in cut():
            s.free()

    out["prefix_16x512_ms"] = {
        "none": timed(lambda: m.infer_ex(slots, [512] * 16, toks, opt), reps),
        "snap_reused": timed(lambda: m.infer_snapshots(slots, [512] * 16, toks, opt, [(s, 256) for s in slots], reuse=reuse), reps),
        "cut_state_read": timed(cut_free, reps),
    }
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
