"""General-path shapes for ncu: `python profiles/prof_general.py c3|1m|plain [ticks]`
c3: 48 distros x 100k tasks in configs[2]'s mix (Zipf, dependencies, task groups); 1m: 8 x 1M tasks; plain: no multi-member units."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np
from evergreen_b200 import _lib as L
if len(sys.argv) > 3:  # another build of the library, e.g. another commit's, to compare the two
    lib = C.CDLL(sys.argv[3])
    for name, (res, args) in L.SYMBOLS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name); fn.restype = res; fn.argtypes = args
    L._lib = lib
from evergreen_b200 import scheduler, synth
which = sys.argv[1] if len(sys.argv) > 1 else "c3"
eng = scheduler.Engine(0)
if which == "c3":
    w = synth.config(3, 0.0048, each=True)
elif which == "1m":
    w = synth.config(4, 0.0008, each=True)
elif which == "c5":  # BASELINE configs[4]: 100k power-law distros, every route in one tick
    w = synth.config(5)
elif which == "c2":
    w = synth.config(2)
elif which == "c4":  # BASELINE configs[3], total reading: 10k distros, 1M tasks, 50k hosts
    w = synth.config(4)
elif which == "c3t":  # BASELINE configs[2], total reading: 10k distros, 100k tasks
    w = synth.config(3)
else:
    w = synth.make(np.full(48, 100000), synth.SEED_BASE + 3, tg_frac=0.0, zipf_priority=True, n_hosts=96)
eng.upload(w.tasks, w.distros, w.hosts)
ms = []
for _ in range(int(sys.argv[2]) if len(sys.argv) > 2 else 3):
    eng.run(w.now)
    ms.append(eng.last_timing_ms()[0])
po, ao = eng.download()
try:
    gt = eng.general_timing_ms()
except Exception:  # noqa: BLE001  (a tick without general-path distros)
    gt = None
print("ok", which, os.path.basename(sys.argv[3]) if len(sys.argv) > 3 else "in-tree", w.n_tasks, "tick median %.4f ms min %.4f" % (float(np.median(ms)), float(min(ms))),
      "tasks/s %.3e" % (w.n_tasks / (float(np.median(ms)) * 1e-3)), gt, eng.last_launch_count(),
      "checksum", int(ao.result["new_hosts"].sum()) + int(po.order[::997].sum()))
