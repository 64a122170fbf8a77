"""One engine object over N GPUs of the machine (b200rwkv_create_ex, worker thread per rank): decode throughput of the bench
workload and the in-situ windows of rank 0's step.  usage: gpu_inproc_tp.py N [preset] [batch]"""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth

N = int(sys.argv[1]) if len(sys.argv) > 1 else 2
preset = sys.argv[2] if len(sys.argv) > 2 else "v6-7b"
B = int(sys.argv[3]) if len(sys.argv) > 3 else 16
st = synth.make_st(preset, 0)
t0 = time.time()
m = runtime.Model(st, max_batch=B, token_chunk_size=64, devices=list(range(N)))
print(f"build {time.time() - t0:.1f} s over {N} GPUs")
slots = list(range(B))
rng = np.random.default_rng(1234)
for s in slots:
    m.state.load(m.state.init(), s)
m.infer_raw(slots, [16] * B, rng.integers(1, 60000, 16 * B).tolist(), [capi.OPTION_NONE] * B)
steps, warm = 64, 4
toks = rng.integers(1, 60000, size=(steps + warm, B)).astype(np.uint32)
ms, launches = m.bench_decode(slots, toks, warm, steps)
print(f"in-process TP{N}: {ms / steps:.4f} ms/step  {B * steps / (ms * 1e-3):.1f} tokens/s  launches/step {launches // steps}")
wins, step_us = m.profile_insitu(slots, toks[0], reps=5)
cls = {}
for w in wins:
    ty = w["type"]
    name = f"gemm_{ty - 1000000}MiB" if ty >= 1000000 else {0: "ln_mix", 2: "wkv", 6: "front_half"}.get(ty, str(ty))
    a = cls.setdefault(name, [0.0, 0])
    a[0] += w["end_us"] - w["start_us"]; a[1] += 1
tot = sum(v[0] for v in cls.values())
print(f"rank 0 in-situ step {step_us:.1f} us, windows {tot:.1f} us, between windows {step_us - tot:.1f} us")
for k, v in sorted(cls.items()):
    print(f"  {k:14s} n={v[1]:3d} avg {v[0] / v[1]:7.2f} us  sum {v[0]:8.1f}")
# e2e through the one-object API
out = np.empty((B, m.info["num_vocab"]), np.float32)
t0 = time.perf_counter()
for i in range(32):
    m.infer_raw(slots, [1] * B, toks[i % toks.shape[0]].tolist(), [0] * B, out=out)
dt = time.perf_counter() - t0
print(f"e2e infer (host logits): {dt / 32 * 1e3:.4f} ms/step  {B * 32 / dt:.1f} tokens/s")
m.close()
