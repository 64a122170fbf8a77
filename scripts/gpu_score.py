"""Scoring continuations: FULL rows to the host + NumPy log-softmax against OPTION_SCORE on the device (b200rwkv_infer_ex).

    python scripts/gpu_score.py [--preset v6-7b] [--slots 16] [--tokens 256] [--runs 5] [--json out.json]

Every slot starts from the same snapshot (a state with a kept row) before each call, so all arms score the same tokens on the
same states.  Arms, alternated run by run:
  full_pinned    b200rwkv_infer with FULL into pinned host memory (b200rwkv_host_alloc), then a NumPy f32 log-softmax
  full_pageable  the same into ordinary (pageable) NumPy memory
  score          b200rwkv_infer_ex with SCORE: 8 bytes per token come back
Wall time of the engine call (it ends in a stream synchronise) and of the NumPy pass are reported separately, as medians.
The score_rows_kernel time comes from torch.profiler (CUDA activities) around one more SCORE call, in a run of its own.
The card name and power limit are read by the same process."""
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


def log_softmax_at(rows: np.ndarray, targets: np.ndarray) -> np.ndarray:
    """f32 log softmax(rows)[targets], row by row in blocks (what a host caller of FULL does with the rows)."""
    out = np.empty(rows.shape[0], np.float32)
    for b in range(0, rows.shape[0], 256):
        x = rows[b:b + 256]
        m = x.max(1, keepdims=True)
        lse = np.log(np.exp(x - m).sum(1, dtype=np.float32))
        out[b:b + 256] = (x[np.arange(x.shape[0]), targets[b:b + 256]] - m[:, 0]) - lse
    return out


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
    _, kept = m.state.snapshot_back(snap, with_logits=True)
    toks = rng.integers(1, V, (B, T)).astype(np.uint32)
    slots, ntok, flat = list(range(B)), [T] * B, toks.reshape(-1).tolist()
    n = B * T
    pinned = C.c_void_p()
    capi.check(capi.lib().b200rwkv_host_alloc(n * V * 4, C.byref(pinned)))
    pin = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (n, V))
    pageable = np.empty((n, V), np.float32)
    # targets of the FULL rows: row j of a slot predicts token j + 1; token 0 is scored from the kept row
    tgt = toks[:, 1:].reshape(-1)
    keep_rows = np.concatenate([np.arange(s * T, s * T + T - 1) for s in range(B)])

    def reset():
        for s in slots:
            m.state.write(snap, s)

    def full(buf):
        reset()
        a = [np.asarray(x, t) for x, t in ((slots, np.int32), (ntok, np.int32), (flat, np.uint32))]
        a_opt = np.full(B, capi.OPTION_FULL, np.int32)
        rows = np.zeros(B, np.int32)
        t0 = time.perf_counter()
        capi.check(capi.lib().b200rwkv_infer(m._h, B, capi.ptr(a[0]), capi.ptr(a[1]), capi.ptr(a[2]), capi.ptr(a_opt),
                                             buf.ctypes.data_as(C.c_void_p), buf.size, capi.ptr(rows)), m._h)
        t1 = time.perf_counter()
        sc = np.empty((B, T), np.float32)
        sc[:, 1:] = log_softmax_at(buf[keep_rows], tgt).reshape(B, T - 1)
        sc[:, 0] = log_softmax_at(np.repeat(kept[None], B, 0), toks[:, 0])
        t2 = time.perf_counter()
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3, sc

    def score():
        reset()
        t0 = time.perf_counter()
        _, sc = m.infer_ex(slots, ntok, flat, [capi.OPTION_SCORE] * B)
        t1 = time.perf_counter()
        return (t1 - t0) * 1e3, np.stack([s for s, _ in sc])

    full(pin); full(pageable); score()          # warm-up: graphs, allocations, page faults of the pageable buffer
    res = {"full_pinned": [], "full_pageable": [], "score": [], "numpy_ms": []}
    worst = 0.0
    for _ in range(args.runs):
        a_ms, np_ms, a_sc = full(pin)
        p_ms, _, _ = full(pageable)
        b_ms, b_sc = score()
        res["full_pinned"].append(a_ms); res["full_pageable"].append(p_ms); res["score"].append(b_ms); res["numpy_ms"].append(np_ms)
        worst = max(worst, float(np.abs(a_sc - b_sc).max()))
    # kernel time, profiler on, separate run
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.infer_ex(slots, ntok, flat, [capi.OPTION_SCORE] * B)
        torch.cuda.synchronize()
    kern = [e for e in prof.key_averages() if "score_rows_kernel" in e.key]
    t_attr = "device_time_total" if kern and hasattr(kern[0], "device_time_total") else "cuda_time_total"
    kernel_us = float(sum(getattr(e, t_attr) for e in kern))
    n_launch = int(sum(e.count for e in kern))
    med = {k: float(np.median(v)) for k, v in res.items()}
    out = {
        "card": card, "preset": args.preset, "slots": B, "tokens_per_slot": T, "runs": args.runs,
        "engine_call_ms_median": {k: med[k] for k in ("full_pinned", "full_pageable", "score")},
        "numpy_log_softmax_ms_median": med["numpy_ms"],
        "full_pinned_total_ms": med["full_pinned"] + med["numpy_ms"],
        "full_pageable_total_ms": med["full_pageable"] + med["numpy_ms"],
        "d2h_bytes_per_call": {"full": n * V * 4, "score": n * 8},
        "score_rows_kernel_launches": n_launch, "score_rows_kernel_us_total": kernel_us,
        "max_abs_diff_full_vs_score": worst,
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
