"""What the batch-invariant mode (b200rwkv_options.batch_invariant) costs, against a default engine and against a default
engine at token_chunk_size 16 (the other way to keep every step decode-shaped).

    python scripts/gpu_invariant.py [--runs 3] [--json out.json]

Arms, alternated run by run (median and range of the runs):
  7B decode at batch 16   bench_decode, 128 timed steps after 8: default against mode (same launches and bits expected)
  7B decode at 32 / 64    one LAST token per slot per infer call (logits stay on the device), 32 calls per run: default,
                          mode, default at chunk 16
  3B prefill 16 x 512     one NONE infer call of 16 entries of 512 tokens: default at chunk 128, mode at chunk 128, default
                          at chunk 16
Wall times end in the engine's stream synchronise (infer is host-synchronous).  The card name and power limit are read by the
same process."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "runs": len(xs)}


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

    # ---- 7B decode ----
    st = synth.make_st("v6-7b", 0)
    arms = {"default": dict(), "mode": dict(batch_invariant=True), "chunk16": dict(token_chunk_size=16)}
    ms = {k: runtime.Model(st, max_batch=64, **{"token_chunk_size": 128, **kw}) for k, kw in arms.items()}
    V = ms["default"].info["num_vocab"]
    for m in ms.values():
        for s in range(64):
            m.state.load(m.state.init(), s)
    toks = rng.integers(1, V, size=(8 + 128) * 16).astype(np.uint32)
    res = {k: [] for k in ("default", "mode")}
    launches, rows = {}, {}
    for r in range(args.runs):
        for k in (("default", "mode") if r % 2 == 0 else ("mode", "default")):
            t, n = ms[k].bench_decode(list(range(16)), toks, 8, 128)
            res[k].append(t / 128)
            launches[k] = n
            rows[k] = ms[k].infer_raw(list(range(16)), [1] * 16, toks[:16].tolist(), [capi.OPTION_LAST] * 16)
    same = all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(rows["default"], rows["mode"]))
    out["decode16"] = {k: stats(v) for k, v in res.items()}
    out["decode16"].update(launches=launches, rows_identical=bool(same))
    print("7B decode batch 16 ms/step:", json.dumps(out["decode16"]), flush=True)
    for B in (32, 64):
        res = {k: [] for k in arms}
        calls = 32
        tk = rng.integers(1, V, size=(calls, B)).tolist()
        for m in ms.values():                    # warm up: capture every step shape the timed calls use
            for j in range(2):
                m.infer_raw(list(range(B)), [1] * B, tk[j], [capi.OPTION_LAST] * B, keep_on_device=True)
        order = list(arms)
        for r in range(args.runs):
            for k in order[r % 3:] + order[:r % 3]:
                m = ms[k]
                t0 = time.perf_counter()
                for j in range(calls):
                    m.infer_raw(list(range(B)), [1] * B, tk[j], [capi.OPTION_LAST] * B, keep_on_device=True)
                res[k].append((time.perf_counter() - t0) * 1e3 / calls)
        out[f"decode{B}"] = {k: stats(v) for k, v in res.items()}
        print(f"7B decode batch {B} ms/call:", json.dumps(out[f"decode{B}"]), flush=True)
    for m in ms.values():
        m.close()
    del ms, st

    # ---- 3B prefill ----
    st = synth.make_st("v6-3b", 0)
    arms = {"default": dict(), "mode": dict(batch_invariant=True), "chunk16": dict(token_chunk_size=16)}
    ms = {k: runtime.Model(st, max_batch=16, **{"token_chunk_size": 128, **kw}) for k, kw in arms.items()}
    V = ms["default"].info["num_vocab"]
    tk = rng.integers(1, V, size=16 * 512).tolist()
    res = {k: [] for k in arms}
    for m in ms.values():
        for s in range(16):
            m.state.load(m.state.init(), s)
        m.infer_raw(list(range(16)), [512] * 16, tk, [capi.OPTION_NONE] * 16)       # warm-up: every step shape
    order = list(arms)
    for r in range(args.runs):
        for k in order[r % 3:] + order[:r % 3]:
            m = ms[k]
            for s in range(16):
                m.state.load(m.state.init(), s)
            t0 = time.perf_counter()
            m.infer_raw(list(range(16)), [512] * 16, tk, [capi.OPTION_NONE] * 16)
            res[k].append((time.perf_counter() - t0) * 1e3)
    out["prefill3b"] = {k: stats(v) for k, v in res.items()}
    print("3B prefill 16 x 512 ms/call:", json.dumps(out["prefill3b"]), flush=True)
    for m in ms.values():
        m.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
