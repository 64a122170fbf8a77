"""Timeline of one graph-replayed decode step (b200rwkv_profile_insitu + b200rwkv_debug_trace): globaltimer stamps of CTA 0 of every launch.
Rows: label, entry, past griddepcontrol.wait, ..., exit -- all in us relative to the first launch of the printed layer."""
import ctypes as C, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth

preset = os.environ.get("B200RWKV_BENCH_PRESET", "v6-7b")
B = int(os.environ.get("B200RWKV_BENCH_BATCH", "16"))
st = synth.make_st(preset, 0)
m = runtime.Model(st, max_batch=B, token_chunk_size=128)
slots = list(range(B))
rng = np.random.default_rng(0)
for i in range(8):
    m.infer_raw(slots, [1] * B, rng.integers(1, 60000, B).tolist(), [0] * B)
m.profile_insitu(slots, rng.integers(1, 60000, B).astype(np.uint32), reps=2)      # traced replays leave their stamp rows behind
ROW = 512
buf = np.zeros(1024 * ROW, np.uint64); types = np.zeros(1024, np.int32); n = C.c_int32(0)
capi.check(capi.lib().b200rwkv_debug_trace(m._h, capi.ptr(buf), buf.size, capi.ptr(types), C.byref(n)), m._h)
n = n.value
full = buf[:n * ROW].reshape(n, ROW).astype(np.int64)
tr = full[:, :8]
def name(ty):
    if ty >= 1000000: return f"gemm{ty - 1000000}MB"
    return {0: "ln", 2: "wkv", 6: "pre6"}.get(ty, str(ty))
# find launches of layer 8 (skip warm layers): per layer launches = (n - 3) / L
L = m.info["num_layer"]
per = (n - 3) // L
print(f"{n} launches, {per} per layer; step total {(tr[:, [0, 7]].max() - tr[0, 0]) / 1e3:.1f} us")
for layer in (8, 9):
    i0 = 1 + layer * per
    base = tr[i0, 0]
    for i in range(i0, i0 + per):
        row = " ".join(f"{(x - base) / 1e3:7.2f}" if x > 0 else "      -" for x in tr[i])
        print(f"  L{layer} {name(types[i]):10s} {row}")
# aggregate: per label, mean (exit - previous exit) = marginal time on the critical path
prev_exit = np.concatenate([[tr[0, 0]], tr[:-1, 7]])
for ty in sorted(set(types[:n].tolist())):
    sel = np.where(types[:n] == ty)[0]
    sel = sel[sel > 0]
    marg = (tr[sel, 7] - np.maximum.accumulate(tr[:, 7])[sel - 1]) / 1e3
    inside = (tr[sel, 7] - tr[sel, 1]) / 1e3
    print(f"{name(ty):10s} n={len(sel):3d} marginal (exit - prev exit) avg {marg.mean():6.2f} us sum {marg.sum():8.1f} | wait->exit avg {inside.mean():6.2f}")
# skew across the grid of the projection launches of layers 8..11: per CTA {SM id, last MMA issued, exit}
G = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
for layer in (8, 9, 10, 11):
    i0 = 1 + layer * per
    for i in range(i0, i0 + per):
        if types[i] == 6:
            c = full[i, 8:8 + 3 * 128].reshape(128, 3)
            base = c[:, 1].min()
            ent = (c[:, 0] - base) / 1e3; rel = (c[:, 1] - base) / 1e3; p1 = (c[:, 2] - base) / 1e3
            print(f"  L{layer} pre6 per-CTA (us from first release): entry min/med/max {ent.min():6.2f} {np.median(ent):6.2f} {ent.max():6.2f} | released {rel.min():5.2f} {np.median(rel):5.2f} {rel.max():5.2f} | phase1 done {p1.min():5.2f} {np.median(p1):5.2f} {p1.max():5.2f} | slowest clusters {sorted(set((np.argsort(p1)[-8:] // 8).tolist()))}")
            continue
        if types[i] < 1000000: continue
        c = full[i, 8:8 + 3 * G].reshape(G, 3)
        ok = c[:, 2] > 0
        if ok.sum() == 0: continue
        base = tr[i, 2]                      # producer of CTA 0 released by griddepcontrol.wait
        mma = (c[ok, 1] - base) / 1e3; ex = (c[ok, 2] - base) / 1e3
        order = np.argsort(ex)
        slow = np.where(ok)[0][order[-6:]]
        print(f"  L{layer} {name(types[i]):10s} ctas {ok.sum():3d} lastMMA min/med/max {mma.min():6.2f} {np.median(mma):6.2f} {mma.max():6.2f} | exit min/med/max {ex.min():6.2f} {np.median(ex):6.2f} {ex.max():6.2f} | slowest ctas {slow.tolist()} on SMs {c[slow, 0].tolist()}")
if len(sys.argv) > 1:                    # optional: save the raw stamps to this .npy path
    np.save(sys.argv[1], full[:, :8 + 3 * G])
m.close()
