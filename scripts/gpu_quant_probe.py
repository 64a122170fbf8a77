"""Where a quantised projection launch spends its time (debug build): per-role cycle accounts of CTA 0 (qgemm.cuh) and the launch
windows, for the hand-off variants / diagnostic switches of B200RWKV_QVAR: bit 0: one arrive per expansion warp instead of one
per thread (production); bit 1: skip the expansion; bit 2: skip the MMAs; bit 3: skip the proxy fence (bits 1-3 give wrong
results: timing only)."""
import ctypes as C, dataclasses, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi, runtime, synth

capi._lib = capi.debug_lib()
B = 16
shape = dataclasses.replace(synth.PRESETS["v6-7b"], L=6, V=8192)
st = synth.make_st(shape, 0)
rng = np.random.default_rng(0)
ROW, QTR = 512, 460
for qt in ("int8", "nf4"):
    for qv in (1, 0, 3, 5, 9, 7):
        os.environ["B200RWKV_QVAR"] = str(qv)
        m = runtime.Model(st, max_batch=B, token_chunk_size=64, quant=shape.L, quant_type=qt)
        slots = list(range(B))
        for i in range(4):
            m.infer_raw(slots, [1] * B, rng.integers(1, 8000, B).tolist(), [0] * B)
        win, step_us = m.profile_insitu(slots, rng.integers(1, 8000, B).astype(np.uint32), reps=3)
        buf = np.zeros(1024 * ROW, np.uint64); types = np.zeros(1024, np.int32); n = C.c_int32(0)
        capi.check(capi.lib().b200rwkv_debug_trace(m._h, capi.ptr(buf), buf.size, capi.ptr(types), C.byref(n)), m._h)
        n = n.value
        full = buf[:n * ROW].reshape(n, ROW).astype(np.int64)
        agg = {}
        for i in range(n):
            if types[i] < 1000000 or full[i, QTR + 4] == 0:
                continue
            a = agg.setdefault(int(types[i]) - 1000000, [])
            q = full[i, QTR:QTR + 12]
            a.append([(full[i, 7] - full[i, 2]) / 1e3] + q.tolist())
        print(f"{qt} qvar={qv} step {step_us:.1f} us")
        for mb, rows in sorted(agg.items()):
            r = np.asarray(rows, np.float64).mean(0)
            nb = r[5]
            print(f"  gemm {mb:4d} MiB x{len(rows)}: window {r[0]:6.2f} us, {nb:.0f} blocks/CTA = {r[0] / nb:5.3f} us/block | expand warps (cycles/block): "
                  f"wait full {r[1]/nb:6.0f} wait dfree {r[2]/nb:6.0f} expand {r[3]/nb:6.0f} fence+arrive {r[4]/nb:6.0f} | consumer: wait full {r[6]/nb:6.0f} "
                  f"wait dfull {r[7]/nb:6.0f} total {r[9]/nb:6.0f} | producer: wait empty {r[11]/nb:6.0f} total {r[12]/nb:6.0f}")
        m.close()
