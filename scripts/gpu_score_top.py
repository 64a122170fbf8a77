"""Top-n log-probabilities of every scored token: SCORE alone against SCORE plus b200rwkv_score_top(5 / 20 / 128), and the
FULL + host sort route they replace.

    python scripts/gpu_score_top.py [--preset v6-7b] [--slots 16] [--tokens 256] [--runs 5] [--json out.json]

Every slot starts from the same snapshot before each call, so all arms score the same tokens on the same states.  Arms,
alternated run by run (wall time of the engine call, which ends in a stream synchronise):
  score          infer_ex with SCORE entries
  top5 / top20 / top128   the same call with score_top(n) on, plus last_score_top
  full_sort      b200rwkv_infer with FULL into pinned host memory, then the n = 20 best entries of every row on the host
                 (np.argpartition + a lexsort of the survivors) and an f32 log-softmax at them; host time reported apart
Median and range over the runs.  Kernel times of score_rows_kernel and the two score_top kernels come from torch.profiler
(CUDA activities) around one top-20 call, in a run of its own.  The card name and power limit are read by the same process."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402


def host_top(rows: np.ndarray, n: int):
    """(ids, f32 log-probabilities) of the n best entries of each row, logit descending then id ascending."""
    ids = np.empty((rows.shape[0], n), np.int64)
    lp = np.empty((rows.shape[0], n), np.float32)
    for b in range(0, rows.shape[0], 256):
        x = rows[b:b + 256]
        part = np.argpartition(-x, n, axis=1)[:, :n + 1]
        # ties at the cut: widen to every entry equal to the n-th best before ordering
        for r in range(x.shape[0]):
            cand = part[r]
            kth = np.sort(x[r, cand])[::-1][n - 1]
            cand = np.union1d(cand, np.flatnonzero(x[r] == kth))
            order = cand[np.lexsort((cand, -x[r, cand]))][:n]
            ids[b + r] = order
        m = x.max(1, keepdims=True)
        lse = np.log(np.exp(x - m).sum(1, dtype=np.float32))
        lp[b:b + 256] = (np.take_along_axis(x, ids[b:b + 256], 1) - m) - lse[:, None]
    return ids, lp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    B, T = args.slots, args.tokens
    m = runtime.Model(synth.make_st(args.preset, 0), max_batch=B, token_chunk_size=128)
    V = m.info["num_vocab"]
    rng = np.random.default_rng(0)
    m.state.load(m.state.init(), 0)
    m.infer_raw([0], [4], [11, 12, 13, 14], [capi.OPTION_LAST], keep_on_device=True)
    snap = m.state.read(0)
    toks = rng.integers(1, V, (B, T)).astype(np.uint32)
    slots, ntok, flat = list(range(B)), [T] * B, toks.reshape(-1).tolist()
    n_tok = B * T
    pinned = C.c_void_p()
    capi.check(capi.lib().b200rwkv_host_alloc(n_tok * V * 4, C.byref(pinned)))
    pin = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (n_tok, V))

    def reset():
        for s in slots:
            m.state.write(snap, s)

    def score(n):
        reset()
        m.score_top(n)
        t0 = time.perf_counter()
        _, sc = m.infer_ex(slots, ntok, flat, [capi.OPTION_SCORE] * B)
        lists = m.last_score_top() if n else None
        t1 = time.perf_counter()
        return (t1 - t0) * 1e3, sc, lists

    def full_sort():
        reset()
        a = [np.asarray(x, t) for x, t in ((slots, np.int32), (ntok, np.int32), (flat, np.uint32))]
        a_opt = np.full(B, capi.OPTION_FULL, np.int32)
        rows = np.zeros(B, np.int32)
        t0 = time.perf_counter()
        capi.check(capi.lib().b200rwkv_infer(m._h, B, capi.ptr(a[0]), capi.ptr(a[1]), capi.ptr(a[2]), capi.ptr(a_opt),
                                             pin.ctypes.data_as(C.c_void_p), pin.size, capi.ptr(rows)), m._h)
        t1 = time.perf_counter()
        ids, _ = host_top(pin, 20)
        t2 = time.perf_counter()
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3, ids

    arms = {"score": 0, "top5": 5, "top20": 20, "top128": 128}
    for n in arms.values():
        score(n)                              # warm-up: graphs, allocations
    full_sort()
    res = {k: [] for k in list(arms) + ["full_sort_engine", "full_sort_host"]}
    same_ids = True
    for _ in range(args.runs):
        for k, n in arms.items():
            ms, _, lists = score(n)
            res[k].append(ms)
            if n == 20:
                dev_ids = lists[0]
        e_ms, h_ms, ids = full_sort()
        res["full_sort_engine"].append(e_ms)
        res["full_sort_host"].append(h_ms)
        # FULL row j of a slot is the row SCORE token j + 1 was scored from
        dev = dev_ids.reshape(B, T, 20)[:, 1:].reshape(-1, 20)
        host = ids.reshape(B, T, 20)[:, :-1].reshape(-1, 20)
        same_ids &= bool(np.array_equal(dev, host))
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    reset()
    m.score_top(20)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.infer_ex(slots, ntok, flat, [capi.OPTION_SCORE] * B)
        torch.cuda.synchronize()
    m.score_top(0)
    kernels = {}
    for e in prof.key_averages():
        for name in ("score_rows_kernel", "score_top_segment_kernel", "score_top_merge_kernel"):
            if name in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                kernels[name] = {"launches": int(e.count), "us_total": float(t)}
    stat = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in res.items()}
    out = {
        "card": card, "preset": args.preset, "slots": B, "tokens_per_slot": T, "runs": args.runs,
        "call_ms": stat,
        "d2h_bytes_per_call": {"score": n_tok * 8, **{k: n_tok * (8 + 8 * n) for k, n in arms.items() if n},
                               "full": n_tok * V * 4},
        "kernels_top20_call": kernels,
        "top20_ids_equal_full_sort": same_ids,
        "all_runs_ms": res,
    }
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    snap.free()
    capi.lib().b200rwkv_host_free(pinned)
    m.close()


if __name__ == "__main__":
    main()
