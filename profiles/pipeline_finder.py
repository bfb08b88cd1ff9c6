#!/usr/bin/env python3
"""The pipeline task finder against the legacy finder at the f.1 size (3000 distros, ~8.12e6 candidates), through the
public API: evg_find_runnable_ex vs evg_find_runnable_batch, and evg_plan_from_finder_ex vs evg_plan_from_finder.  Each
call ends in a stream synchronise, so the host clock around it spans H2D, the kernels and D2H.  The four calls are
alternated over `--reps` rounds after one warm-up each; medians and minima in ms.  Prints one JSON line with the card's
name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import model as M  # noqa: E402
from evergreen_b200 import scheduler, soa, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--distros", type=int, default=3000)
ap.add_argument("--mean", type=int, default=2707, help="mean candidates per distro (2707 x 3000 = 8.12e6)")
args = ap.parse_args()

NOW = synth.NOW_NS
rnd = np.random.default_rng(17)
D, P, X, NS = args.distros, 64, 4000, 8
sizes = rnd.integers(0, 2 * args.mean, D)
off = np.zeros(D + 1, np.int64); np.cumsum(sizes, out=off[1:])
T = int(off[-1])
sched = (rnd.integers(0, 256, T) | 0x0F * (rnd.random(T) < 0.85)).astype(np.uint8)
project = rnd.integers(-1, P, T).astype(np.int32)
pflags = (rnd.integers(0, 16, P) | 1).astype(np.uint8)
praw = (rnd.integers(0, 8, P) | 1).astype(np.uint8)
nvalid = np.where(rnd.random(D) < 0.3, rnd.integers(1, 6, D), 0)
voff = np.zeros(D + 1, np.int64); np.cumsum(nvalid, out=voff[1:])
vidx = rnd.integers(-1, P, int(voff[-1])).astype(np.int32)
n_dep = rnd.integers(0, 3, T)
doff = np.zeros(T + 1, np.int64); np.cumsum(n_dep, out=doff[1:])
E = int(doff[-1])
distro_of = np.repeat(np.arange(D), sizes)
owner = np.repeat(np.arange(T), n_dep)
ref = (off[distro_of][owner] + rnd.integers(0, 1 << 30, E) % np.maximum(sizes[distro_of][owner], 1)).astype(np.int32)
kind = rnd.integers(0, 3, E).astype(np.uint8)
ref[kind == 1] %= X
deps = soa.DepsTable(doff, kind, ref, rnd.integers(0, 4, E).astype(np.uint8), rnd.integers(0, 3, T).astype(np.uint8),
                     (rnd.random(T) < 0.1).astype(np.uint8), rnd.integers(0, 3, X).astype(np.uint8))
pipe = soa.PipelineTable(NS, rnd.integers(0, NS, E).astype(np.int32), rnd.integers(0, NS, T).astype(np.int32),
                         rnd.integers(0, NS, X).astype(np.int32), (rnd.random(T) < 0.05).astype(np.uint8),
                         (rnd.random(X) < 0.1).astype(np.uint8), praw)
legacy = soa.RunnableTable(off, sched, project, pflags, voff, vidx, np.full(D, L.EVG_FINDER_LEGACY, np.uint8), deps)
pipeline = soa.RunnableTable(off, sched, project, pflags, voff, vidx, np.full(D, L.EVG_FINDER_PIPELINE, np.uint8), deps, pipe)
wc = synth.make(sizes, 91, zipf_priority=True, tg_frac=0.1, met_dep_frac=0.03, includes_dependencies=True)
wc.tasks.flags &= ~np.uint32(L.EVG_TF_DEPS_MET)
fin = np.where(rnd.random(E) < 0.5, NOW - rnd.integers(0, 10 ** 12, E), M.ZERO_TIME).astype(np.int64)

eng = scheduler.Engine(0)
calls = {
    "find_legacy": lambda: eng.find_runnable_batch(legacy),
    "find_pipeline": lambda: eng.find_runnable_batch(pipeline),
    "plan_legacy": lambda: eng.plan_from_finder(legacy, wc.tasks, wc.distros, None, fin, NOW),
    "plan_pipeline": lambda: eng.plan_from_finder(pipeline, wc.tasks, wc.distros, None, fin, NOW),
}
kept = {}
for name, fn in calls.items():  # warm-up: module load, first allocations
    _, count = fn()
    kept[name] = int(count.sum())
ms = {name: [] for name in calls}
for _ in range(args.reps):
    for name, fn in calls.items():
        t0 = time.perf_counter()
        fn()
        ms[name].append((time.perf_counter() - t0) * 1e3)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown"
out = {"card": card, "candidates": T, "distros": D, "in_queue_edges": int(wc.tasks.n_edges), "dependency_entries": E,
       "reps": args.reps, "kept": kept,
       "median_ms": {k: float(np.median(v)) for k, v in ms.items()}, "min_ms": {k: float(np.min(v)) for k, v in ms.items()}}
print(json.dumps(out))
