import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from ai00_server_b200 import capi, runtime, synth
st = synth.make_st("v6-7b", 0)
m = runtime.Model(st, max_batch=16, token_chunk_size=64)
for which, name in [(0, "W1"), (1, "W2"), (2, "RKVG+d1"), (10, "O"), (20, "ffnKR"), (21, "ffnV"), (30, "head")]:
    ms = C.c_float(0); nb = C.c_int64(0)
    tr = np.zeros((32, 16), np.uint64)
    capi.check(capi.lib().b200rwkv_debug_gemm_time(m._h, which, 3, C.byref(ms), C.byref(nb), capi.ptr(tr)), m._h)
    t = tr.astype(np.int64)
    rel = (t - t[:, :1]) / 1e3
    gap = (t[1:, 0] - t[:-1, 7]) / 1e3            # next launch entry - this launch exit (cta 0)
    names = ["entry", "setup", "pdlwait(prod)", "1st full", "mma done", "pdlwait(epi)", "epi done", "exit", "tfull(last seg)", "tmem read", "fixup done"]
    print(f"{name:8s} {ms.value*1e3:8.2f} us/launch  {nb.value/1e6:8.2f} MB  {nb.value/(ms.value*1e-3)/1e12:6.2f} TB/s | cta0 stamps(us): " +
          " ".join(f"{n}={np.median(rel[4:, i]):.1f}" for i, n in enumerate(names)) + f" | entry->next entry {np.median(t[5:,0]-t[4:-1,0])/1e3:.1f} gap(exit->next entry) {np.median(gap[4:]):.1f}")
m.close()
