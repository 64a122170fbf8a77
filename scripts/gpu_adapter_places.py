"""Cost of adapter places (b200rwkv_create_adapter_places): loading and unloading an adapter against rebuilding the engine,
and the bound decode step of a places engine against an engine created with the same number of files.

    python scripts/gpu_adapter_places.py [--preset v6-7b] [--batch 16] [--rank 64] [--runs 3] [--steps 128] [--json out.json]

Every place and file pairs all eight projection kinds and the head at rank `rank`.  Two phases, so that at most two engines of
the 7B shape are resident at once:
  1. P8, a places engine with 8 places (all kinds and the head targeted), and C8, an engine from b200rwkv_create_adapters with
     the 8 files.  First the outputs of P8 (all 8 places loaded) and C8 on the same decode calls, which must be
     byte-identical.  Then the host wall time of unload_adapter and load_adapter on P8 (each call ends in a stream
     synchronise; 5 of each), and the decode step (`b200rwkv_bench_decode`: CUDA events around `steps` graph replays), every
     slot bound, alternated in an order that rotates from run to run:
       p8_full8  P8 with all 8 places loaded, slot s bound to place 1 + s % 8
       c8        C8, the same binding
       p8_full1  P8 with only place 1 loaded, every slot bound to it
       p8_full8_one, c8_one  all 8 loaded, every slot bound to id 1: against p8_full1, what loaded places cost by themselves
     Last, the host wall time of destroying C8 and creating it again with the same files (`--rebuilds` times).
  2. P1 (1 place, loaded) and C1 (1 file), every slot bound to id 1, alternated the same way.
The card name and power limit are read by the same process."""
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

TARGETS = ("att.receptance", "att.key", "att.value", "att.gate", "att.output", "ffn.key", "ffn.value", "ffn.receptance")


def stats(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1], "all": v}


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def alternate(arms, slots, tokens, args, res, launches):
    """arms: name -> (model, set-up callable run before each measurement); fills res[name] with ms per step"""
    names = list(arms)
    for run in range(args.runs):
        for name in names[run % len(names):] + names[:run % len(names)]:
            m, setup = arms[name]
            setup()
            ms, n = m.bench_decode(slots, tokens, args.warmup, args.steps)
            res.setdefault(name, []).append(ms / args.steps)
            launches[name] = n // args.steps
            print(f"run {run} {name}: {ms / args.steps:.4f} ms/step, {n // args.steps} launches/step", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rank", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rebuilds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    shp = synth.PRESETS[args.preset]
    B = args.batch
    slots = list(range(B))
    st = synth.make_st(shp, 0)
    files = [(synth.make_lora_st(shp, rank=args.rank, seed=31 + i, targets=TARGETS), 0.1) for i in range(8)]
    every = TARGETS + ("head",)
    kw = dict(max_batch=B, token_chunk_size=128)
    out = {"card": card, "preset": args.preset, "batch": B, "rank": args.rank}

    # ---- phase 1: 8 places against 8 files ----
    p8 = runtime.Model(st, adapter_places=8, adapter_targets=every, **kw)
    for i, (img, a) in enumerate(files):
        p8.load_adapter(i + 1, img, a)
    c8 = runtime.Model(st, adapters=files, **kw)
    V = p8.info["num_vocab"]
    spread = [1 + s % 8 for s in slots]
    outs = []
    for m in (p8, c8):
        m.bind_adapter(slots, spread)
        for s in slots:
            m.state.load(m.state.init(), s)
        r = np.random.default_rng(1)
        rows = [m.infer_raw(slots, [1] * B, r.integers(1, V, size=B).tolist(), [capi.OPTION_LAST] * B) for _ in range(4)]
        outs.append(np.concatenate([np.concatenate(x, 0).ravel() for x in rows] + [m.state.back(s).ravel() for s in slots]))
    out["identical_p8_c8"] = bool(np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)))
    print("outputs of P8 and C8 byte-identical:", out["identical_p8_c8"], flush=True)

    p8.bind_adapter(slots, [1] * B)
    load_ms, unload_ms = [], []
    for _ in range(args.reps):
        unload_ms.append(timed(lambda: p8.unload_adapter(8)))
        load_ms.append(timed(lambda: p8.load_adapter(8, *files[7])))
    out["load_ms"], out["unload_ms"] = stats(load_ms), stats(unload_ms)
    print(f"load_adapter   {out['load_ms']['median']:.1f} ms ({out['load_ms']['min']:.1f}-{out['load_ms']['max']:.1f})", flush=True)
    print(f"unload_adapter {out['unload_ms']['median']:.1f} ms ({out['unload_ms']['min']:.1f}-{out['unload_ms']['max']:.1f})",
          flush=True)

    full = {"n": 8}

    def p8_with(k, bind):
        def setup():
            p8.bind_adapter(slots, [1] * B)          # no slot on a place about to be emptied, none on an empty one
            while full["n"] > k:
                p8.unload_adapter(full["n"])
                full["n"] -= 1
            while full["n"] < k:
                full["n"] += 1
                p8.load_adapter(full["n"], *files[full["n"] - 1])
            p8.bind_adapter(slots, bind)
        return setup

    tokens = np.random.default_rng(0).integers(1, V, size=(args.warmup + args.steps) * B).astype(np.uint32)
    res, launches = {}, {}
    alternate({"p8_full8": (p8, p8_with(8, spread)), "c8": (c8, lambda: c8.bind_adapter(slots, spread)),
               "p8_full1": (p8, p8_with(1, [1] * B)), "p8_full8_one": (p8, p8_with(8, [1] * B)),
               "c8_one": (c8, lambda: c8.bind_adapter(slots, [1] * B))}, slots, tokens, args, res, launches)
    p8.close()
    rebuild, holder = [], [c8]

    def rebuild_c8():
        holder.pop().close()
        holder.append(runtime.Model(st, adapters=files, **kw))

    for _ in range(args.rebuilds):
        rebuild.append(timed(rebuild_c8))
    holder[0].close()
    out["rebuild_c8_ms"] = stats(rebuild)
    print(f"destroy + create_adapters (8 files): {out['rebuild_c8_ms']['median']:.0f} ms "
          f"({out['rebuild_c8_ms']['min']:.0f}-{out['rebuild_c8_ms']['max']:.0f})", flush=True)

    # ---- phase 2: 1 place against 1 file ----
    p1 = runtime.Model(st, adapter_places=1, adapter_targets=every, **kw)
    p1.load_adapter(1, *files[0])
    c1 = runtime.Model(st, adapters=files[:1], **kw)
    for m in (p1, c1):
        m.bind_adapter(slots, [1] * B)
    alternate({"p1": (p1, lambda: None), "c1": (c1, lambda: None)}, slots, tokens, args, res, launches)
    p1.close()
    c1.close()

    out["step_ms"] = {k: stats(v) | {"launches": launches[k]} for k, v in res.items()}
    for k, v in out["step_ms"].items():
        print(f"{k:9s} {v['median']:.4f} ms/step ({v['min']:.4f}-{v['max']:.4f}), {v['launches']} launches", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
