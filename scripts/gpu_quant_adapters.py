"""Adapters on quantised layers (b200rwkv_options.quant_adapters): the decode step of Int4 and FP8 adapter-places engines,
unbound and with every slot bound, against the f16 places engine bound, and each engine's resident device memory.

    python scripts/gpu_quant_adapters.py [--preset v6-7b] [--batch 16] [--rank 64] [--runs 3] [--steps 128] [--json out.json]

Every engine has 1 place targeting all eight projection kinds and the head, loaded with one file of rank `rank`; the quantised
engines quantise every layer.  Arms (`b200rwkv_bench_decode`: CUDA events around `steps` graph replays after `warmup`),
alternated in an order that rotates from run to run:
  int4_unbound, int4_bound, fp8_unbound, fp8_bound, f16_bound
Resident memory is the drop in free device memory across each engine's creation.  The card name and power limit are read by
the same process."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402

TARGETS = ("att.receptance", "att.key", "att.value", "att.gate", "att.output", "ffn.key", "ffn.value", "ffn.receptance")


def stats(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1], "all": v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rank", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    shp = synth.PRESETS[args.preset]
    B = args.batch
    slots = list(range(B))
    st = synth.make_st(shp, 0)
    f = synth.make_lora_st(shp, rank=args.rank, seed=31, targets=TARGETS)
    every = TARGETS + ("head",)
    out = {"card": card, "preset": args.preset, "batch": B, "rank": args.rank, "resident_gb": {}}
    torch.cuda.init()
    engines = {}
    for name, q in (("int4", "Int4"), ("fp8", "FP8"), ("f16", None)):
        free0 = torch.cuda.mem_get_info()[0]
        kw = dict(quant=shp.L, quant_type=q, quant_adapters=True) if q else {}
        m = runtime.Model(st, max_batch=B, token_chunk_size=128, adapter_places=1, adapter_targets=every, **kw)
        m.load_adapter(1, f, 0.1)
        out["resident_gb"][name] = (free0 - torch.cuda.mem_get_info()[0]) / 1e9
        print(f"{name}: resident {out['resident_gb'][name]:.2f} GB", flush=True)
        engines[name] = m
    V = engines["f16"].info["num_vocab"]
    tokens = np.random.default_rng(0).integers(1, V, size=(args.warmup + args.steps) * B).astype(np.uint32)
    arms = {"int4_unbound": ("int4", 0), "int4_bound": ("int4", 1), "fp8_unbound": ("fp8", 0), "fp8_bound": ("fp8", 1),
            "f16_bound": ("f16", 1)}
    names = list(arms)
    res, launches = {}, {}
    for run in range(args.runs):
        for name in names[run % len(names):] + names[:run % len(names)]:
            eng, bound = arms[name]
            m = engines[eng]
            m.bind_adapter(slots, [bound] * B)
            ms, n = m.bench_decode(slots, tokens, args.warmup, args.steps)
            res.setdefault(name, []).append(ms / args.steps)
            launches[name] = n // args.steps
            print(f"run {run} {name}: {ms / args.steps:.4f} ms/step, {n // args.steps} launches/step", flush=True)
    for m in engines.values():
        m.close()
    out["step_ms"] = {k: stats(v) | {"launches": launches[k]} for k, v in res.items()}
    for k, v in out["step_ms"].items():
        print(f"{k:13s} {v['median']:.4f} ms/step ({v['min']:.4f}-{v['max']:.4f}), {v['launches']} launches", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
