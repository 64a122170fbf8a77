"""New weights for a live engine: in-place updates against destroying the engine and creating it again.

    python scripts/gpu_update_weights.py [--preset v6-7b] [--quant none,fp8,int4] [--runs 3] [--json out.json]

For each weight format (f16; FP8 or Int4 on every layer) one engine of the preset's shape is created from a synthetic image,
then four arms run alternated, in an order that rotates from run to run, each timed by the host clock around the call (every
call returns after its writes are complete):
  recreate     b200rwkv_destroy + b200rwkv_create_ex from the same image (pageable)
  upd_pageable b200rwkv_update_weights with the whole image in pageable memory
  upd_pinned   b200rwkv_update_weights with the image copied once into b200rwkv_host_alloc (pinned) memory
  upd_device   b200rwkv_update_weights_device from BF16 torch tensors of every model tensor on the engine's device
The image is the same in every arm, so after each host-side arm the engine's decode logits must equal the first engine's
bit for bit; after every upd_device they must equal those of the first upd_device (the BF16 tensors round the image's F16
values), and differ from the image's (checked).  Reported: median, min and max of each arm, the image's bytes and the rate
they imply, and the card name, power limit and max SM clock, read by the same process."""
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
from oracle import rwkv_numpy as O  # noqa: E402

QUANTS = {"none": (0, capi.QUANT_NONE), "fp8": (None, capi.QUANT_FP8), "int4": (None, capi.QUANT_INT4)}


def stats(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1], "all": v}


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="v6-7b")
    ap.add_argument("--quant", default="none,fp8,int4")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("gpu_update_weights.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    shp = synth.PRESETS[args.preset]
    st = synth.make_st(shp, 0)
    nbytes = int(st.size)
    pinned_p = C.c_void_p()
    capi.check(capi.lib().b200rwkv_host_alloc(nbytes, C.byref(pinned_p)))
    pinned = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(pinned_p.value))
    pinned[:] = st
    dev = {n: torch.from_numpy(np.array(v)).to("cuda").to(torch.bfloat16) for n, v in O.parse_st(st).items()}
    torch.cuda.synchronize()
    B = args.batch
    slots = list(range(B))
    toks = [1 + 17 * s for s in range(B)]
    want_dev = {}
    out = {"card": card, "preset": args.preset, "image_bytes": nbytes, "runs": args.runs, "arms": {}}

    def logits(m):
        for s in slots:
            m.state.load(m.state.init(), s)
        return m.infer_raw(slots, [1] * B, toks, [capi.OPTION_LAST] * B)

    try:
        for q in args.quant.split(","):
            layers, qt = QUANTS[q]
            kw = dict(quant=shp.L if layers is None else 0, quant_type=qt) if qt != capi.QUANT_NONE else dict(devices=[0])
            box = {"m": runtime.Model(st, max_batch=B, token_chunk_size=128, **kw)}
            want = logits(box["m"])

            def recreate():
                box["m"].close()
                box["m"] = runtime.Model(st, max_batch=B, token_chunk_size=128, **kw)

            arms = {"recreate": recreate,
                    "upd_pageable": lambda: box["m"].update_weights(st),
                    "upd_pinned": lambda: box["m"].update_weights(pinned),
                    "upd_device": lambda: box["m"].update_weights_from_tensors(dev)}
            res = {}
            names = list(arms)
            for run in range(args.runs):
                for name in names[run % len(names):] + names[:run % len(names)]:
                    ms = timed(arms[name])
                    got = logits(box["m"])
                    ref = want
                    if name == "upd_device":
                        ref = want_dev.setdefault(q, got)
                        if all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, want)):
                            raise SystemExit(f"{q} {name}: the BF16 weights gave the F16 image's logits")
                    if not all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, ref)):
                        raise SystemExit(f"{q} {name}: the logits changed")
                    res.setdefault(name, []).append(ms)
                    print(f"{q} run {run} {name}: {ms:.1f} ms", flush=True)
            box["m"].close()
            out["arms"][q] = {n: dict(stats(v), image_gb_per_s=nbytes / (stats(v)["median"] * 1e-3) / 1e9) for n, v in res.items()}
            for n, v in out["arms"][q].items():
                print(f"{q} {n}: median {v['median']:.1f} ms (min {v['min']:.1f}, max {v['max']:.1f}), "
                      f"{v['image_gb_per_s']:.1f} GB/s of image", flush=True)
    finally:
        del pinned
        capi.lib().b200rwkv_host_free(pinned_p)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
