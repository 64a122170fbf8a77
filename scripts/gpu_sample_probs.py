"""Whole-distribution sampling per generated token: the reference's host route against b200rwkv_sample_probs.

    python scripts/gpu_sample_probs.py [--preset v6-7b] [--slots 16] [--tokens 32] [--runs 5] [--json out.json]

Every run decodes `tokens` steps of one token per slot from the same snapshot, with fixed token ids, and produces for every
slot and step the vector run.rs:673-691 hands to Sampler::sample: softmax(logits - penalties, + bias).  Each slot carries 64
penalties and 4 bias entries (a Typical / Nucleus penalty map and a request bias; no grammar mask).  Routes, alternated run by
run:
  host           the reference's: b200rwkv_infer into a host logits buffer, NumPy f32 adjustment of each row
                 (oracle/sampling_numpy.py adjusted_logits, as Sampler::transform and the bias add do), b200rwkv_softmax on the
                 adjusted rows (one upload, one copy back)
  device         b200rwkv_infer(logits_out = NULL), then b200rwkv_sample_probs into ordinary (pageable) NumPy memory
  device_pinned  the same into pinned memory from b200rwkv_host_alloc
Wall times of the calls (each ends in a stream synchronise) are reported per step, as medians and ranges over the runs, with
the split between infer, the host pass and the sampling call.  The kernel time of probs_stats_kernel + probs_write_kernel
comes from torch.profiler (CUDA activities) around `tokens` more sample_probs calls, in a pass of its own.  The card's name and
power limit are read by the same process."""
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
from oracle import sampling_numpy as S  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=32)
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
    slots = list(range(B))
    toks = rng.integers(1, V, (T, B)).astype(np.uint32)
    pens = [{int(t): float(v) for t, v in zip(rng.choice(V, 64, replace=False), rng.random(64))} for _ in slots]
    bias = [{int(t): float(v) for t, v in zip(rng.choice(V, 4, replace=False), rng.standard_normal(4))} for _ in slots]
    logits = np.empty((B, V), np.float32)
    pinned = C.c_void_p()
    capi.check(capi.lib().b200rwkv_host_alloc(B * V * 4, C.byref(pinned)))
    pin = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (B, V))
    args_c = m._sample_args(slots, pens, bias, None)

    def reset():
        for s in slots:
            m.state.write(snap, s)

    def infer(step, out):
        a_slot, a_ntok, a_opt = np.asarray(slots, np.int32), np.ones(B, np.int32), np.full(B, capi.OPTION_LAST, np.int32)
        rows = np.zeros(B, np.int32)
        tok = np.ascontiguousarray(toks[step])
        capi.check(capi.lib().b200rwkv_infer(m._h, B, capi.ptr(a_slot), capi.ptr(a_ntok), capi.ptr(tok), capi.ptr(a_opt),
                                             None if out is None else capi.ptr(out), 0 if out is None else out.size,
                                             capi.ptr(rows)), m._h)

    def sample_probs(out):
        a_slot, po, pt, pv, _, bo, bt, bv = args_c
        capi.check(capi.lib().b200rwkv_sample_probs(m._h, B, capi.ptr(a_slot), capi.ptr(po), capi.ptr(pt), capi.ptr(pv), None,
                                                    capi.ptr(bo), capi.ptr(bt), capi.ptr(bv), capi.ptr(out)), m._h)

    def host_route():
        reset()
        t = np.zeros(3)
        last = None
        for step in range(T):
            t0 = time.perf_counter()
            infer(step, logits)
            t1 = time.perf_counter()
            adj = np.stack([S.adjusted_logits(logits[i], pens[i], None, bias[i]) for i in range(B)])
            t2 = time.perf_counter()
            probs = m.softmax(list(adj))
            t3 = time.perf_counter()
            t += (t1 - t0, t2 - t1, t3 - t2)
            last = np.stack(probs)
        return t * 1e3 / T, last

    def device_route(out):
        reset()
        t = np.zeros(2)
        for step in range(T):
            t0 = time.perf_counter()
            infer(step, None)
            t1 = time.perf_counter()
            sample_probs(out)
            t2 = time.perf_counter()
            t += (t1 - t0, t2 - t1)
        return t * 1e3 / T, out.copy()

    pageable = np.empty((B, V), np.float32)
    host_route(); device_route(pageable); device_route(pin)          # warm-up: graphs, allocations, page faults
    res = {"host": [], "device": [], "device_pinned": []}
    worst = 0.0
    for _ in range(args.runs):
        th, ph = host_route()
        td, pd = device_route(pageable)
        tp, pp = device_route(pin)
        res["host"].append(th.tolist()); res["device"].append(td.tolist()); res["device_pinned"].append(tp.tolist())
        worst = max(worst, float(np.abs(ph - pd).max()), float(np.abs(ph - pp).max()))
    # kernel time, profiler on, separate pass
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    reset()
    infer(0, None)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(T):
            sample_probs(pageable)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for name in ("probs_stats_kernel", "probs_write_kernel"):
            if name in e.key:
                t_attr = "device_time_total" if hasattr(e, "device_time_total") else "cuda_time_total"
                kern[name] = (float(getattr(e, t_attr)) / max(e.count, 1), int(e.count))

    def summary(k, parts):
        per = np.asarray(res[k])
        tot = per.sum(1)
        return {"per_step_ms_median": float(np.median(tot)), "per_step_ms_range": [float(tot.min()), float(tot.max())],
                "split_ms_median": {p: float(np.median(per[:, j])) for j, p in enumerate(parts)}}

    out = {
        "card": card, "preset": args.preset, "slots": B, "num_vocab": V, "tokens_per_run": T, "runs": args.runs,
        "host": summary("host", ["infer_to_host", "numpy_adjust", "softmax_round_trip"]),
        "device": summary("device", ["infer_no_logits", "sample_probs"]),
        "device_pinned": summary("device_pinned", ["infer_no_logits", "sample_probs"]),
        "pcie_bytes_per_step": {"host": 3 * B * V * 4, "device": B * V * 4},
        "kernel_us_per_call": {k: v[0] for k, v in kern.items()},
        "kernel_launches": {k: v[1] for k, v in kern.items()},
        "max_abs_diff_host_vs_device": worst,
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
