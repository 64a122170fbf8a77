"""What a quantised vocabulary head (b200rwkv_head_format) buys on the GPU, with f16 layers and with Int4 layers.

    python scripts/gpu_quant_head.py [--runs 3] [--json out.json]

Shapes: RWKV-6 7B at batch 16, RWKV-6 3B at batch 1, RWKV-7 2.9B at batch 8 (synthetic weights).  For each shape two engines,
f16 layers and Int4 layers (every layer), and on each the five head formats, switched on the same engine between arms:
  decode      bench_decode, 128 timed steps after 8 (CUDA events over graph replays); the arms rotate run by run and the
              median and range of the runs are reported
  head alone  debug_gemm_time(which = 30): the head launch over 16 rows, timed over repeated launches; its weight bytes and
              bytes / time
  logits      max |logit - f16 head| and top-1 agreement with the f16 head, same engine and layers, over a seeded decode
              stream of 32 steps (synthetic weights: this says nothing about trained checkpoints)
The card name, power limit and max SM clock are read by the same process."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402

HEADS = ["None", "Int8", "NF4", "FP8", "Int4"]
SHAPES = [("v6-7b", 16), ("v6-3b", 1), ("v7-2b9", 8)]


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "runs": len(xs)}


def decode(m, B, runs, rng):
    V = m.info["num_vocab"]
    toks = rng.integers(1, V, size=(8 + 128) * B).astype(np.uint32)
    res = {h: [] for h in HEADS}
    for r in range(runs):
        for h in HEADS[r % len(HEADS):] + HEADS[:r % len(HEADS)]:
            m.head_format(h)
            t, _ = m.bench_decode(list(range(B)), toks, 8, 128)
            res[h].append(t / 128)
    return {h: stats(v) for h, v in res.items()}


def head_alone(m):
    out = {}
    for h in HEADS:
        m.head_format(h)
        ms, nb = C.c_float(0), C.c_int64(0)
        capi.check(capi.lib().b200rwkv_debug_gemm_time(m._h, 30, 4, C.byref(ms), C.byref(nb), None), m._h)
        out[h] = {"us": ms.value * 1e3, "weight_bytes": nb.value, "GB_per_s": nb.value / (ms.value * 1e-3) / 1e9}
    return out


def logits(m, B, rng):
    V = m.info["num_vocab"]
    toks = rng.integers(1, V, size=(32, B)).tolist()
    rows = {}
    for h in HEADS:
        m.head_format(h)
        for s in range(B):
            m.state.load(m.state.init(), s)
        rows[h] = np.stack([np.stack([r[0] for r in m.infer_raw(list(range(B)), [1] * B, t, [capi.OPTION_LAST] * B)])
                            for t in toks])
    ref = rows["None"]
    return {h: {"max_abs_dlogit": float(np.abs(v - ref).max()), "max_abs_logit": float(np.abs(ref).max()),
                "top1_agreement": float((v.argmax(-1) == ref.argmax(-1)).mean())}
            for h, v in rows.items() if h != "None"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    out = {"card": card}
    rng = np.random.default_rng(0)
    for preset, B in SHAPES:
        st = synth.make_st(preset, 0)
        L = synth.PRESETS[preset].L
        for layers in ("f16", "Int4"):
            kw = dict(quant=L, quant_type="Int4") if layers == "Int4" else {}
            m = runtime.Model(st, max_batch=B, token_chunk_size=64, **kw)
            try:
                for s in range(B):
                    m.state.load(m.state.init(), s)
                key = f"{preset}_b{B}_{layers}_layers"
                res = {"decode_ms_per_step": decode(m, B, args.runs, rng), "head_alone": head_alone(m),
                       "logits_vs_f16_head": logits(m, B, rng)}
                out[key] = res
                print(key, json.dumps(res), flush=True)
            finally:
                m.close()
        del st
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
