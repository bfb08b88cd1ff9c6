#!/usr/bin/env python3
"""evg_resolve_durations at the flagship size: 200 distros x 100 000 tasks (2e7 task rows) plus hosts, 1e7 history rows
over 1e5 Zipf-skewed keys (synth.make_duration_cache).  The call ends in a stream synchronise, so the host clock
around it spans H2D, the kernels and the error-word read-back.  Two row lists: every task and host row, and a 5 %
sample (what a shim sends after checking freshness on the host).  torch.profiler gives the k_dur_* share of one
all-rows call.  The Python host route (marshal_tasks resolving FetchExpectedDuration per Task object) is timed at a
smaller size and labelled as such: the aggregate through scheduler.get_expected_durations_for_window, then
marshal_tasks with and without model.fetch_expected_duration per task.  Prints one JSON line with the card's name and power limit."""
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
ap.add_argument("--distros", type=int, default=200)
ap.add_argument("--tasks", type=int, default=100_000, help="tasks per distro")
ap.add_argument("--hosts", type=int, default=20_000)
ap.add_argument("--history", type=int, default=10_000_000)
ap.add_argument("--keys", type=int, default=100_000)
ap.add_argument("--host-route-tasks", type=int, default=20_000)
args = ap.parse_args()

w = synth.make(np.full(args.distros, args.tasks), 5, n_hosts=args.hosts)
dw = synth.make_duration_cache(w, 5, n_rows=args.history, n_keys=args.keys)
eng = scheduler.Engine(0)
eng.upload(w.tasks, w.distros, w.hosts)
rng = np.random.default_rng(5)


def sample(c: soa.DurationCache, frac: float) -> soa.DurationCache:
    r = np.sort(rng.choice(c.n_rows, int(c.n_rows * frac), replace=False)).astype(np.int64)
    return soa.DurationCache(*[getattr(c, f)[r] for f in L.DURATION_CACHE_COLUMNS], c.key[r], r)


lists = {"all_rows": (dw.tasks, dw.hosts), "stale_5pct": (sample(dw.tasks, 0.05), sample(dw.hosts, 0.05))}
hist_bytes = dw.history.rows.n_rows * (4 + 3 * 8 + 1) + dw.history.pair_key_off.nbytes
h2d = {k: hist_bytes + sum(c.nbytes() for c in v) for k, v in lists.items()}
for t, h in lists.values():  # warm-up: first allocations
    eng.resolve_durations(dw.history, w.now, t, h)
ms = {k: [] for k in lists}
for _ in range(args.reps):
    for k, (t, h) in lists.items():
        t0 = time.perf_counter()
        eng.resolve_durations(dw.history, w.now, t, h)
        ms[k].append((time.perf_counter() - t0) * 1e3)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    eng.resolve_durations(dw.history, w.now, *lists["all_rows"])
    torch.cuda.synchronize()
kern, copies = {}, 0.0
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if e.name.startswith("_Z") or e.name.startswith("k_") or "k_dur" in e.name:
            name = next((n for n in ("k_dur_sum", "k_dur_dev", "k_dur_final", "k_dur_pair", "k_dur_resolve", "k_dur_commit") if n in e.name), e.name)
            kern[name] = kern.get(name, 0.0) + us / 1e3
        elif "Memcpy" in e.name or "Memset" in e.name:
            copies += us / 1e3
kern_total = sum(kern.values())

# the Python host route, smaller: marshal_tasks resolving FetchExpectedDuration per Task
n = args.host_route_tasks
finished = [M.Task(id=f"f{i}", project="p", build_variant=f"bv{i % 50}", display_name=f"n{i % 997}", status="success",
                   time_taken=(1 + i % 60) * M.MINUTE, start_time=w.now - 2 * M.HOUR, finish_time=w.now - M.HOUR)
            for i in range(10 * n)]
# the host route's aggregate is the product's scheduler.get_expected_durations_for_window: soa.marshal_durations on the
# host, then the one-shot evg_expected_durations_batch (its own context); timed separately from the marshalling
scheduler.get_expected_durations_for_window(finished[:10], w.now - 7 * 24 * M.HOUR, w.now)  # warm-up: its context
t0 = time.perf_counter()
hist = scheduler.get_expected_durations_for_window(finished, w.now - 7 * 24 * M.HOUR, w.now)
agg_ms = (time.perf_counter() - t0) * 1e3
tasks = [M.Task(id=f"t{i}", project="p", build_variant=f"bv{i % 50}", display_name=f"n{i % 1200}",
                duration_prediction=M.CachedDurationValue(0, 0, 0, M.ZERO_TIME)) for i in range(n)]
t0 = time.perf_counter()
soa.marshal_tasks([(M.Distro(id="d"), tasks)], w.now, duration_history=hist)
marshal_ms = (time.perf_counter() - t0) * 1e3
t0 = time.perf_counter()
soa.marshal_tasks([(M.Distro(id="d"), tasks)], w.now, resolve_durations=False)
marshal_plain_ms = (time.perf_counter() - t0) * 1e3

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown"
out = {"card": card, "task_rows": w.n_tasks, "host_rows": w.hosts.n_hosts, "history_rows": dw.history.rows.n_rows,
       "keys": dw.history.rows.n_keys, "pairs": dw.history.n_pairs, "reps": args.reps,
       "listed_rows": {k: int(t.n_rows + h.n_rows) for k, (t, h) in lists.items()},
       "median_ms": {k: float(np.median(v)) for k, v in ms.items()}, "min_ms": {k: float(np.min(v)) for k, v in ms.items()},
       "h2d_bytes": h2d, "kernel_ms_all_rows": kern, "k_dur_ms_all_rows": kern_total, "copy_ms_all_rows": copies,
       "host_route": {"tasks": n, "history_rows": len(finished), "aggregate_ms": agg_ms,
                      "marshal_with_fetch_ms": marshal_ms, "marshal_without_fetch_ms": marshal_plain_ms,
                      "fetch_us_per_task": (marshal_ms - marshal_plain_ms) * 1e3 / n}}
print(json.dumps(out))
