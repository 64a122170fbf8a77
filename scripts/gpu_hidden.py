"""Cost of recording per-layer hidden states (b200rwkv_keep_hidden_layers) against the same call with recording off.

    python scripts/gpu_hidden.py [--preset v6-3b] [--slots 16] [--tokens 512] [--runs 5] [--json out.json]

Arms, alternated run by run, each one infer call of `slots` x `tokens` tokens (LAST rows, token_chunk_size 128, so
128-token prefill steps through ln_mix_kernel) from the same snapshot in every slot:
  off       no layer recorded
  1 layer   the middle layer
  3 layers  first, middle and last layer (the last one comes from ln_out_kernel: only its gather copies are extra)
Then the same three arms for decode-shaped calls (one token per slot, pre6_kernel), `--decode-calls` calls per timing.
Wall time of the engine call (it ends in a stream synchronise), medians and ranges.  The last logits rows of every arm must
be bit-identical.  The card name and power limit are read by the same process."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-3b")
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=512)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--decode-calls", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    B, T = args.slots, args.tokens
    m = runtime.Model(synth.make_st(args.preset, 0), max_batch=B, token_chunk_size=128)
    L, C, V = m.info["num_layer"], m.info["num_emb"], m.info["num_vocab"]
    arms = {"off": [], "1 layer": [L // 2], "3 layers": [0, L // 2, L - 1]}
    rng = np.random.default_rng(0)
    m.state.load(m.state.init(), 0)
    m.infer_raw([0], [4], [11, 12, 13, 14], [capi.OPTION_LAST])
    snap = m.state.read(0)
    slots = list(range(B))
    toks = rng.integers(1, V, (B, T)).astype(np.uint32).reshape(-1).tolist()
    dec = rng.integers(1, V, (args.decode_calls, B)).astype(np.uint32)

    def reset():
        for s in slots:
            m.state.write(snap, s)

    def prefill(layers):
        reset()
        m.keep_hidden(layers=layers)
        t0 = time.perf_counter()
        rows = m.infer_raw(slots, [T] * B, toks, [capi.OPTION_LAST] * B)
        t1 = time.perf_counter()
        m.keep_hidden(layers=[])
        return (t1 - t0) * 1e3, np.concatenate(rows)

    def decode(layers):
        reset()
        m.keep_hidden(layers=layers)
        out = []
        t0 = time.perf_counter()
        for i in range(args.decode_calls):
            out.append(m.infer_raw(slots, [1] * B, dec[i].tolist(), [capi.OPTION_LAST] * B))
        t1 = time.perf_counter()
        m.keep_hidden(layers=[])
        return (t1 - t0) * 1e3 / args.decode_calls, np.concatenate([np.concatenate(r) for r in out])

    for a in arms.values():             # warm-up: graphs, call buffers
        prefill(a); decode(a)
    res = {"prefill": {k: [] for k in arms}, "decode": {k: [] for k in arms}}
    same = True
    for _ in range(args.runs):
        for kind, fn in (("prefill", prefill), ("decode", decode)):
            ref = None
            for name, layers in arms.items():
                ms, rows = fn(layers)
                res[kind][name].append(ms)
                ref = rows if ref is None else ref
                same = same and np.array_equal(rows, ref)
    summ = {kind: {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
                   for k, v in r.items()} for kind, r in res.items()}
    out = {
        "card": card, "preset": args.preset, "slots": B, "tokens_per_slot": T, "runs": args.runs,
        "layers": {k: v for k, v in arms.items()},
        "prefill_call": summ["prefill"], "decode_call": summ["decode"],
        "recorded_bytes_per_layer_per_call": {"prefill": B * T * C * 4, "decode": B * C * 4},
        "outputs_bit_identical": bool(same),
        "all_runs_ms": res,
    }
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    snap.free()
    m.close()
    if not same:
        sys.exit("logits rows differ between arms")


if __name__ == "__main__":
    main()
