"""Per-CTA skew of the projection launches of one graph-replayed decode step.

    python scripts/gpu_cta_skew.py [--json out.json]

Prints the decode step time (bench_decode, CUDA events over graph replays), then per projection launch class (label = weight
MiB), over every layer of one traced replay: the window [griddepcontrol.wait released, last CTA exit], and the median / p90 /
last CTA "MMAs done" stamp relative to the release; `trail` is (last - median) / window, the share of the window the slowest
CTA adds.  The stamps are the per-CTA {SM id, MMAs done, exit} that gemm_kernel writes when its trace pointer is set.  Last,
the big launches' MMA-done lateness (stamp - launch median, in % of the window) averaged per SM id."""
import ctypes as C, json, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth

args = sys.argv[1:]
out_json = args[args.index("--json") + 1] if "--json" in args else None
preset = os.environ.get("B200RWKV_BENCH_PRESET", "v6-7b")
B = int(os.environ.get("B200RWKV_BENCH_BATCH", "16"))
BIG_MIB = 100                   # launches of at least this many weight MiB get the per-SM table

st = synth.make_st(preset, 0)
rng = np.random.default_rng(0)
ROW = 512
m = runtime.Model(st, max_batch=B, token_chunk_size=64)
slots = list(range(B))
V = m.info["num_vocab"]
for _ in range(4):
    m.infer_raw(slots, [1] * B, rng.integers(1, V, B).tolist(), [0] * B)
steps, warm = 64, 8
ms, _ = m.bench_decode(slots, rng.integers(1, V, (warm + steps, B)).astype(np.uint32), warm, steps)
windows, step_us = m.profile_insitu(slots, rng.integers(1, V, B).astype(np.uint32), reps=3)
gemm_us = sum(w["end_us"] - w["start_us"] for w in windows if w["type"] >= 1000000)
buf = np.zeros(1024 * ROW, np.uint64); types = np.zeros(1024, np.int32); n = C.c_int32(0)
capi.check(capi.lib().b200rwkv_debug_trace(m._h, capi.ptr(buf), buf.size, capi.ptr(types), C.byref(n)), m._h)
n = n.value
full = buf[:n * ROW].reshape(n, ROW).astype(np.int64)
m.close()
print(f"{ms / steps:.4f} ms/step (bench_decode), traced step {step_us:.1f} us, projection windows {gemm_us:.1f} us", flush=True)
cls = {}
per_sm = {}
for i in range(n):
    if types[i] < 1000000: continue
    rel = full[i, 2]                                     # CTA 0's producer released by griddepcontrol.wait
    c = full[i, 8:ROW - (ROW - 8) % 3].reshape(-1, 3)
    ok = c[:, 2] > 0
    if not ok.any() or rel == 0: continue
    mma = (c[ok, 1] - rel) / 1e3
    win = (c[ok, 2].max() - rel) / 1e3
    med = float(np.median(mma))
    a = cls.setdefault(int(types[i]) - 1000000, {"n": 0, "ctas": int(ok.sum()), "win": [], "med": [], "p90": [], "last": []})
    a["n"] += 1; a["win"].append(win); a["med"].append(med)
    a["p90"].append(float(np.percentile(mma, 90))); a["last"].append(float(mma.max()))
    if types[i] - 1000000 >= BIG_MIB:
        for smid, t in zip(c[ok, 0], mma):
            per_sm.setdefault(int(smid), []).append(100.0 * (t - med) / win)
print(f"  {'MiB':>5s} {'n':>3s} {'ctas':>4s} {'window us':>9s} {'median':>7s} {'p90':>7s} {'last':>7s} {'trail %':>7s}")
rows = []
for mib in sorted(cls):
    a = cls[mib]
    win, med, p90, last = (float(np.mean(a[k])) for k in ("win", "med", "p90", "last"))
    trail = float(np.mean([(l - md) / w for l, md, w in zip(a["last"], a["med"], a["win"])])) * 100
    print(f"  {mib:5d} {a['n']:3d} {a['ctas']:4d} {win:9.2f} {med:7.2f} {p90:7.2f} {last:7.2f} {trail:7.2f}")
    rows.append({"mib": mib, "launches": a["n"], "ctas": a["ctas"], "window_us": win, "median_us": med, "p90_us": p90,
                 "last_us": last, "trail_pct": trail})
sm = sorted((s, float(np.mean(v))) for s, v in per_sm.items())
if sm:
    print(f"  launches >= {BIG_MIB} MiB, mean MMA-done lateness per SM id (% of window, vs the launch median):")
    for k in range(0, len(sm), 12):
        print("   " + " ".join(f"{s:3d}:{v:+5.1f}" for s, v in sm[k:k + 12]))
if out_json:
    with open(out_json, "w") as f:
        json.dump({"ms_per_step": ms / steps, "traced_step_us": step_us, "gemm_us": gemm_us, "classes": rows,
                   "lateness_per_sm_pct": sm}, f, indent=1)
