"""Diagnostic: per-step device time of the resident configs[1] tick over a long run (clock ramp check).
usage: python profiles/ab_build.py [path/to/libevgsched.so] [iterations]"""
import sys, os, time, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from evergreen_b200 import _lib as L
path = sys.argv[1] if len(sys.argv) > 1 else L.LIB_PATH
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3000
lib = C.CDLL(path)
for name, (res, args) in list(L.SYMBOLS.items()):
    if hasattr(lib, name):
        fn = getattr(lib, name); fn.restype = res; fn.argtypes = args
L._lib = lib
from evergreen_b200 import scheduler, synth
eng = scheduler.Engine(0)
w = synth.config(2)
eng.upload(w.tasks, w.distros, w.hosts)
ms, wall = [], []
t0 = time.perf_counter()
for i in range(iters):
    eng.run(w.now); ms.append(eng.last_timing_ms()[0]); wall.append(time.perf_counter() - t0)
ms = np.array(ms); wall = np.array(wall)
print(os.path.basename(path), "first10 %s" % np.round(ms[:10], 3).tolist())
for a in range(0, iters, max(iters // 10, 1)):
    b = min(a + max(iters // 10, 1), iters)
    print("  steps %5d-%5d  wall %.2fs  median %.4f ms  min %.4f" % (a, b, wall[b - 1], float(np.median(ms[a:b])), float(ms[a:b].min())))
