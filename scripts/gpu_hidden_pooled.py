"""Cost of one embedding row per input: pooled hidden rows (b200rwkv_keep_hidden_pooled) against per-token recording
(b200rwkv_keep_hidden_layers) with the row picked on the host, and against the same call with neither.

    python scripts/gpu_hidden_pooled.py [--preset v6-3b] [--slots 16] [--tokens 512] [--runs 5] [--json out.json]

Arms, alternated within every run in an order that rotates from run to run, each one infer call of `slots` x `tokens` tokens (NONE entries as the embeddings route runs
them, token_chunk_size 128) from the same snapshot in every slot, timed up to the rows being in host memory:
  off            nothing recorded, nothing fetched
  kept 1         keep_hidden_layers on the middle layer, all rows fetched, row sum(ntok[0..=i]) - 1 of every entry picked
  pooled last    keep_hidden_pooled on the middle layer, POOL_LAST, [slots][num_emb] fetched
  pooled mean    the same with POOL_MEAN
  pooled 3       POOL_LAST on first, middle and last layer, three fetches
Then the same arms for decode-shaped calls (one token per slot), `--decode-calls` calls per timing.  Wall time of the engine
calls (each ends in a stream synchronise), medians and ranges, and the bytes each arm moves to the host.  `pooled last` must
equal the picked rows of `kept 1` bit for bit.  hidden_pool_kernel's own time comes from torch.profiler (CUDA activities)
around one more call per pooled arm, in a run of its own.  The card name and power limit are read by the same process."""
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
    mid = L // 2
    # name -> (kept layers, pooled layers, mode)
    arms = {"off": ([], [], "last"), "kept 1": ([mid], [], "last"), "pooled last": ([], [mid], "last"),
            "pooled mean": ([], [mid], "mean"), "pooled 3": ([], [0, mid, L - 1], "last")}
    rng = np.random.default_rng(0)
    m.state.load(m.state.init(), 0)
    m.infer_raw([0], [4], [11, 12, 13, 14], [capi.OPTION_LAST])
    snap = m.state.read(0)
    slots = list(range(B))
    toks = rng.integers(1, V, (B, T)).astype(np.uint32).reshape(-1).tolist()
    dec = rng.integers(1, V, (args.decode_calls, B)).astype(np.uint32)
    none = [capi.OPTION_NONE] * B

    def reset():
        for s in slots:
            m.state.write(snap, s)

    def call(arm, ntok, tokens):
        """One infer call and the fetch of its embedding rows: ([B][C] rows of the middle layer or None, bytes to the host)."""
        kept, pooled, _ = arms[arm]
        m.infer_raw(slots, [ntok] * B, tokens, none)
        if kept:
            rows = m.last_hidden(max_rows=B * ntok, layer=mid)
            return rows[np.arange(1, B + 1) * ntok - 1].copy(), rows.nbytes
        got = [m.last_hidden_pooled(l, max_rows=B)[0] for l in pooled]
        return (got[pooled.index(mid)].copy() if pooled else None), sum(g.nbytes for g in got)

    def timed(arm, fn):
        kept, pooled, mode = arms[arm]
        reset()
        m.keep_hidden(layers=kept)
        m.keep_hidden_pooled(pooled, mode)
        t0 = time.perf_counter()
        out = fn(arm)
        t1 = time.perf_counter()
        m.keep_hidden(layers=[])
        m.keep_hidden_pooled([])
        return (t1 - t0) * 1e3, out

    def prefill(arm):
        return call(arm, T, toks)

    def decode(arm):
        out = [call(arm, 1, dec[i].tolist()) for i in range(args.decode_calls)]
        return out[-1][0], out[-1][1]

    for a in arms:                      # warm-up: graphs, call buffers
        timed(a, prefill); timed(a, decode)
    res = {"prefill": {k: [] for k in arms}, "decode": {k: [] for k in arms}}
    moved = {"prefill": {}, "decode": {}}
    same = True
    names = list(arms)
    for run in range(args.runs):
        order = names[run % len(names):] + names[:run % len(names)]      # every arm takes every place in the sequence
        for kind, fn in (("prefill", prefill), ("decode", decode)):
            got = {}
            for name in order:
                ms, (rows, nbytes) = timed(name, fn)
                res[kind][name].append(ms / (args.decode_calls if kind == "decode" else 1))
                moved[kind][name] = int(nbytes)
                got[name] = rows
            same = same and np.array_equal(got["kept 1"].view(np.uint32), got["pooled last"].view(np.uint32))
            same = same and np.array_equal(got["pooled 3"].view(np.uint32), got["pooled last"].view(np.uint32))

    # kernel time, profiler on, separate run
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    kernel = {}
    for name in ("pooled last", "pooled mean", "pooled 3"):
        for kind, fn in (("prefill", prefill), ("decode", lambda arm: call(arm, 1, dec[0].tolist()))):
            reset()
            m.keep_hidden_pooled(arms[name][1], arms[name][2])
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn(name)
                torch.cuda.synchronize()
            m.keep_hidden_pooled([])
            kern = [e for e in prof.key_averages() if "hidden_pool_kernel" in e.key]
            t_attr = "device_time_total" if kern and hasattr(kern[0], "device_time_total") else "cuda_time_total"
            kernel.setdefault(kind, {})[name] = {"launches": int(sum(e.count for e in kern)),
                                                 "total_us": float(sum(getattr(e, t_attr) for e in kern))}

    summ = {kind: {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
                   for k, v in r.items()} for kind, r in res.items()}
    out = {
        "card": card, "preset": args.preset, "slots": B, "tokens_per_slot": T, "runs": args.runs,
        "arms": {k: {"kept": v[0], "pooled": v[1], "mode": v[2]} for k, v in arms.items()},
        "prefill_call": summ["prefill"], "decode_call": summ["decode"],
        "bytes_to_host_per_call": moved,
        "hidden_pool_kernel_per_call": kernel,
        "pooled_last_equals_picked_rows": bool(same),
        "all_runs_ms": res,
    }
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    snap.free()
    m.close()
    if not same:
        sys.exit("pooled rows differ from the picked per-token rows")


if __name__ == "__main__":
    main()
