"""What FP8 (E4M3) and Int4 weight-only layers buy on the GPU, against f16, Int8 and NF4 layers (every layer quantised).

    python scripts/gpu_fp8.py [--runs 3] [--json out.json]

Arms, alternated in a rotating order run by run (median and range of the runs):
  7B decode at batch 16   bench_decode, 128 timed steps after 8 (CUDA events over graph replays)
  7B in-situ windows      profile_insitu of one decode step at batch 16: the projection launches' windows, their algorithmic
                          weight bytes (codes + scales as streamed) and bytes / window
  3B decode at batch 1    bench_decode, 128 timed steps after 8
Also the largest relative logits distance of each arm to the f16 engine over the same decode calls (synthetic weights: this
says nothing about the quality of trained checkpoints).  The card name, power limit and max SM clock are read by the same
process."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402

ARMS = {"fp16": None, "int8": "Int8", "nf4": "NF4", "fp8": "FP8", "int4": "Int4"}


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "runs": len(xs)}


def build(preset, B):
    st = synth.make_st(preset, 0)
    L = synth.PRESETS[preset].L
    ms = {}
    for k, qt in ARMS.items():
        kw = dict(quant=L, quant_type=qt) if qt else {}
        m = runtime.Model(st, max_batch=B, token_chunk_size=64, **kw)
        for s in range(B):
            m.state.load(m.state.init(), s)
        ms[k] = m
    return ms


def decode_arms(ms, B, runs, rng, label):
    V = ms["fp16"].info["num_vocab"]
    toks = rng.integers(1, V, size=(8 + 128) * B).astype(np.uint32)
    res = {k: [] for k in ms}
    order = list(ms)
    for r in range(runs):
        for k in order[r % len(order):] + order[:r % len(order)]:
            t, _ = ms[k].bench_decode(list(range(B)), toks, 8, 128)
            res[k].append(t / 128)
    out = {k: stats(v) for k, v in res.items()}
    print(f"{label} ms/step:", json.dumps(out), flush=True)
    return out


def logits_distance(ms, B, rng):
    """Every arm from the zero state over the same 8 decode calls; max |logits - fp16| / max |fp16| per arm."""
    V = ms["fp16"].info["num_vocab"]
    toks = rng.integers(1, V, size=(8, B)).tolist()
    rows = {}
    for k, m in ms.items():
        for s in range(B):
            m.state.load(m.state.init(), s)
        rows[k] = np.stack([np.stack([r[0] for r in m.infer_raw(list(range(B)), [1] * B, t, [capi.OPTION_LAST] * B)])
                            for t in toks])
    ref = rows["fp16"]
    return {k: float(np.abs(v - ref).max() / np.abs(ref).max()) for k, v in rows.items() if k != "fp16"}


def insitu(ms, B, rng):
    V = ms["fp16"].info["num_vocab"]
    toks = rng.integers(1, V, size=B).astype(np.uint32)
    out = {}
    for k, m in ms.items():
        wins, step_us = m.profile_insitu(list(range(B)), toks, reps=5)
        g = [w for w in wins if w["type"] >= 1000000]
        us = sum(w["end_us"] - w["start_us"] for w in g)
        by = sum(w["bytes"] for w in g)
        out[k] = {"step_us": step_us, "projection_us": us, "weight_bytes": by, "GB_per_s": by / us / 1e3, "launches": len(g)}
    print("7B in-situ projection windows:", json.dumps(out), flush=True)
    return out


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

    ms = build("v6-7b", 16)
    out["7b_b16"] = decode_arms(ms, 16, args.runs, rng, "7B decode batch 16")
    out["7b_insitu"] = insitu(ms, 16, rng)
    out["7b_logits_distance"] = logits_distance(ms, 16, rng)
    print("7B max relative logits distance to fp16:", json.dumps(out["7b_logits_distance"]), flush=True)
    for m in ms.values():
        m.close()
    del ms

    ms = build("v6-3b", 1)
    out["3b_b1"] = decode_arms(ms, 1, args.runs, rng, "3B decode batch 1")
    out["3b_logits_distance"] = logits_distance(ms, 1, rng)
    print("3B max relative logits distance to fp16:", json.dumps(out["3b_logits_distance"]), flush=True)
    for m in ms.values():
        m.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
