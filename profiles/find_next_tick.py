#!/usr/bin/env python3
"""FindNextTask for every distro of a resident tick: evg_find_next_tasks on the dispatchers evg_rebuild_dispatchers left
on the device, on the shapes profiles/dispatch_tick.py uses (configs[4]: 100 000 ragged distros; a block of --distros
queues of --tasks tasks with persisted heads of 10 000), with one request per distro and with --many per distro.
Every call ends in a stream synchronise, so the host clock around it spans its copies and kernels; torch.profiler gives
the k_next_* kernel times of one call.  Each timed call follows a rebuild (not timed), so every repetition serves the same
requests against the same state.  The snapshot has a document for every item and nothing started, so each request walks
to the first item it can hand out.  What the host route would copy back instead (sorted, unit_items, unit_off per distro)
is reported in bytes; its walk is not timed here.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import scheduler, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--distros", type=int, default=200)
ap.add_argument("--tasks", type=int, default=20_000)
ap.add_argument("--many", type=int, default=16)
ap.add_argument("--c5-scale", type=float, default=1.0)
args = ap.parse_args()


def kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "k_next_" in e.name:
            name = e.name[e.name.index("k_next_"):].split("(")[0]
            out[name] = out.get(name, 0.0) + (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
    return out


def measure(name, w):
    eng = scheduler.Engine(0)
    eng.upload(w.tasks, w.distros)
    eng.run(w.now)
    r = eng.rebuild_dispatchers(0)
    D, (N, G) = w.distros.n_distros, eng._n_disp
    db = {"flags": np.full(N, L.EVG_ND_FOUND | L.EVG_ND_DEPS_MET_NOW, np.uint8), "est_generated": np.zeros(N, np.int32),
          "ingest_ns": np.zeros(N, np.int64), "running_hosts": np.zeros(G, np.int32), "generate_limit": 0, "pending_generate": 0,
          "max_large_parser": 0, "num_large_parser": 0}
    res = {"shape": name, "distros": D, "items": N, "groups": G, "reps": args.reps,
           "copy_back_bytes": 4 * (2 * N + G + 2 * D), "runs": {}}
    for per in (1, args.many):
        n_req = np.where(np.diff(r["item_off"]) > 0, per, 0)
        req_off = np.concatenate([[0], np.cumsum(n_req)]).astype(np.int64)
        R = int(req_off[-1])
        req = (req_off, np.full(R, -1, np.int32), np.zeros(R, np.int64))
        eng.find_next_tasks(db, req)  # warm-up: first allocations
        ms = []
        for _ in range(args.reps):
            eng.rebuild_dispatchers(0)
            t0 = time.perf_counter()
            item, outcome = eng.find_next_tasks(db, req)
            ms.append((time.perf_counter() - t0) * 1e3)
        eng.rebuild_dispatchers(0)
        res["runs"][str(per)] = {"requests": R, "found": int((item >= 0).sum()), "ms": [round(x, 3) for x in ms],
                                 "median_ms": float(np.median(ms)), "launches": int(eng.last_launch_count()),
                                 "h2d_bytes": 13 * N + 4 * G + 8 * (D + 1) + 12 * R, "d2h_bytes": 8 * R,
                                 "kernel_ms": kernels(lambda: eng.find_next_tasks(db, req))}
    eng.close()
    return res


try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown"
runs = [measure("configs[4]", synth.config(5, args.c5_scale)),
        measure("long queues", synth.make(np.full(args.distros, args.tasks, dtype=np.int64), synth.SEED_BASE + 3, zipf_priority=True,
                                          unmet_dep_frac=0.05, met_dep_frac=0.02, includes_dependencies=True, tg_frac=0.1))]
print(json.dumps({"card": card, "runs": runs}))
