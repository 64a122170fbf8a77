"""Cost of unblended LoRA adapters (b200rwkv_create_adapters) on the decode step.

    python scripts/gpu_adapters.py [--preset v6-7b] [--batch 16] [--rank 64] [--runs 3] [--steps 128] [--json out.json]

Arms, each `b200rwkv_bench_decode` (CUDA events around `steps` graph replays after `warmup`), alternated within every run in
an order that rotates from run to run:
  (a) base      an engine from b200rwkv_create_ex, created first
  (a') base2    a second create_ex engine, created after the adapter engine (the same launches, weights elsewhere in HBM)
  (b) unbound   an engine from b200rwkv_create_adapters with 4 adapters of rank `rank` on all eight projection kinds and the
                head, no slot bound
  (c) one       the same engine, adapter 1 bound to every slot
  (d) four      the same engine, adapters 1..4 bound to `batch / 4` slots each
Also printed: the algorithmic weight bytes of each arm's step, the outputs of (a) and (b) on the same decode calls (logits and
states, which must be byte-identical), and, from torch.profiler (CUDA activities) around one more bench call of (c) and (d)
in a run of its own, the shrink kernels' own time per step.  The card name and power limit are read by the same process."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth  # noqa: E402

TARGETS = ("att.receptance", "att.key", "att.value", "att.gate", "att.output", "ffn.key", "ffn.value", "ffn.receptance")


def step_bytes(shp, rank, n_registered, bound):
    """Algorithmic weight bytes of one decode step: the base step's f16 weights, + the alpha B tail blocks (N x 128 per
    adapted projection and registered adapter) when a slot is bound, + every bound adapter's A ([r][K] per projection)."""
    C, F, V, L = shp.C, shp.F, shp.V, shp.L
    base = synth.algorithmic_bytes_per_step(shp, 0)
    proj = [(C, C)] * 5 + [(F, C), (C, F), (C, C)]          # (N, K) of r, k, v, g, o, ffn key, ffn value, ffn receptance
    if shp.version == 7:
        proj = [(C, C)] * 4 + [(F, C), (C, F)]
    proj = proj * L + [(V, C)]
    if not bound:
        return base
    tails = sum(n * 128 * 2 for n, _ in proj) * n_registered
    a_read = sum(rank * k * 2 for _, k in proj) * bound
    return base + tails + a_read


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
    st = synth.make_st(shp, 0)
    ads = [(synth.make_lora_st(shp, rank=args.rank, seed=31 + i, targets=TARGETS), 0.1) for i in range(4)]
    base = runtime.Model(st, max_batch=B, token_chunk_size=128, devices=[0])
    ad = runtime.Model(st, max_batch=B, token_chunk_size=128, adapters=ads)
    base2 = runtime.Model(st, max_batch=B, token_chunk_size=128, devices=[0])
    slots = list(range(B))
    rng = np.random.default_rng(0)
    V = base.info["num_vocab"]

    # (a) and (b) on the same decode calls
    outs = []
    for m in (base, ad):
        for s in slots:
            m.state.load(m.state.init(), s)
        r = np.random.default_rng(1)
        rows = [m.infer_raw(slots, [1] * B, r.integers(1, V, size=B).tolist(), [capi.OPTION_LAST] * B) for _ in range(4)]
        outs.append(np.concatenate([np.concatenate(x, 0).ravel() for x in rows] + [m.state.back(s).ravel() for s in slots]))
    identical = bool(np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)))
    print("outputs of (a) and (b) byte-identical:", identical, flush=True)

    binds = {"base": None, "base2": None, "unbound": [0] * B, "one": [1] * B, "four": [1 + (s * 4) // B for s in slots]}
    nbound = {"base": 0, "base2": 0, "unbound": 0, "one": 1, "four": 4}
    engines = {"base": base, "base2": base2}
    tokens = rng.integers(1, V, size=(args.warmup + args.steps) * B).astype(np.uint32)
    res = {k: [] for k in binds}
    launches = {}
    names = list(binds)
    for run in range(args.runs):
        order = names[run % len(names):] + names[:run % len(names)]
        for name in order:
            m = engines.get(name, ad)
            if binds[name] is not None:
                m.bind_adapter(slots, binds[name])
            ms, n = m.bench_decode(slots, tokens, args.warmup, args.steps)
            res[name].append(ms / args.steps)
            launches[name] = n // args.steps
            print(f"run {run} {name}: {ms / args.steps:.4f} ms/step, {n // args.steps} launches/step", flush=True)
    summary = {}
    for name in names:
        v = sorted(res[name])
        gb = step_bytes(shp, args.rank, 4, nbound[name]) / 1e9
        summary[name] = {"ms_median": v[len(v) // 2], "ms_min": v[0], "ms_max": v[-1], "launches": launches[name], "weight_GB": gb}
        print(f"{name:8s} {v[len(v) // 2]:.4f} ms/step ({v[0]:.4f}-{v[-1]:.4f}), {launches[name]} launches, "
              f"{gb:.3f} GB algorithmic weight bytes", flush=True)

    # shrink kernels' own time, a run of its own
    import torch
    from torch.profiler import ProfilerActivity, profile
    shrink = {}
    prof_steps = 16
    tok2 = tokens[:(2 + prof_steps) * B]
    for name in ("one", "four"):
        ad.bind_adapter(slots, binds[name])
        ad.bench_decode(slots, tok2, 2, prof_steps)
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            ad.bench_decode(slots, tok2, 2, prof_steps)
            torch.cuda.synchronize()
        tot = n = 0
        for e in p.events():
            if "adapter_shrink" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                tot += e.device_time
                n += 1
        steps = 2 + prof_steps
        shrink[name] = {"us_per_step": tot / steps, "launches_per_step": n / steps}
        print(f"shrink kernels ({name}): {tot / steps:.1f} us per step in {n / steps:.0f} launches", flush=True)
    out = {"card": card, "preset": args.preset, "batch": B, "rank": args.rank, "identical_a_b": identical,
           "arms": summary, "runs": res, "shrink": shrink}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for m in (base, base2, ad):
        m.close()


if __name__ == "__main__":
    main()
