import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ai00_server_b200 import capi
L = capi.debug_lib()        # python -m ai00_server_b200.build --debug
def run(kind, gb=4.0, stage=16384, nstage=12, hint=1, split=1, producers=1, reps=5):
    ms = C.c_float(0)
    capi.check(L.b200rwkv_debug_stream(0, kind, gb, stage, nstage, hint, split, producers, reps, C.byref(ms)))
    return gb / (ms.value * 1e-3) / 1e3
print("ldg.128 streaming            %.2f TB/s" % run(0))
for (stage, ns) in [(16384, 12), (8192, 24), (4096, 48), (2048, 96), (32768, 6), (65536, 3)]:
    print("ring stage=%6d nstage=%2d trivial consumer 1 producer  %.2f TB/s" % (stage, ns, run(1, stage=stage, nstage=ns)))
for (stage, ns) in [(8192, 24), (4096, 48), (2048, 96)]:
    print("ring stage=%6d nstage=%2d trivial consumer 2 producers %.2f TB/s   3 producers %.2f TB/s" % (stage, ns, run(1, stage=stage, nstage=ns, producers=2), run(1, stage=stage, nstage=ns, producers=3)))
print("ring 16K split=2 (2 copies/stage)  %.2f TB/s" % run(1, split=2))
print("ring 16K split=4                   %.2f TB/s" % run(1, split=4))
print("ring 18K = 16K + 2K extra copy x11 %.2f TB/s" % run(1, stage=18432, nstage=11))
print("ring 18K = 16K + 2K, 2 producers   %.2f TB/s" % run(1, stage=18432, nstage=11, producers=2))
print("ring 36K = 32K + 4K extra copy x6  %.2f TB/s" % run(1, stage=36864, nstage=6))
for gb in (0.135,):
    print("ring 16K x12 trivial, %.3f GB per launch (ramp/tail)   %.2f TB/s" % (gb, run(1, gb=gb, reps=20)))
