#!/usr/bin/env python3
"""What the full SortingValueBreakdown of the persisted queues costs on a resident tick.  Per shape, with the tick's
inputs resident (evg_upload once):
  run ms    evg_run_resident with no option, with EVG_OPT_QUEUE_BREAKDOWN and with EVG_OPT_BREAKDOWN ("does not fit"
            when its T x 104 B buffer cannot be allocated), device time of the whole tick (evg_last_timing_ms), medians of
            --reps alternating rounds after a warm-up round; the kernel launches of each;
  download  evg_download_queue (40 B per persisted rank) and evg_download_queue_breakdown (104 B per persisted rank) after
            an EVG_OPT_QUEUE_BREAKDOWN run, host clock around each call (both end in a stream synchronise), medians.
Shapes: configs[1] (1 000 distros x 10 000 tasks, task groups only: every distro narrow), a block of configs[2]'s
headline mix (--block distros x 100 000 tasks, 5 % unmet in-queue dependencies: every distro complex), configs[4]
(100 000 power-law distros, GroupVersions on a fifth, dependencies) and a GroupVersions / dependency-heavy shape (500
distros x 5 000 tasks, all GroupVersions).  Every rank's TotalValue of the breakdown rows is checked against the items'.
Prints one JSON line with the card's name and power limit."""
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
ap.add_argument("--block", type=int, default=300, help="distros of 100 000 tasks in the configs[2] shape")
args = ap.parse_args()


def gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def shapes():
    yield "configs[1]: 1000 distros x 10k tasks (narrow)", lambda: synth.config(2)
    yield (f"configs[2] block: {args.block} distros x 100k tasks, 5% unmet deps (complex)",
           lambda: synth.make(np.full(args.block, 100_000), synth.SEED_BASE + 3, zipf_priority=True, unmet_dep_frac=0.05,
                              met_dep_frac=0.02, includes_dependencies=True))
    yield "configs[4]: 100k power-law distros", lambda: synth.config(5)
    yield ("GroupVersions + dependencies: 500 distros x 5k tasks",
           lambda: synth.make(np.full(500, 5000), 7100, zipf_priority=True, tg_frac=0.2, group_versions_frac=1.0,
                              unmet_dep_frac=0.05, met_dep_frac=0.05, includes_dependencies=True))


def timed_run(eng, now, opts):
    eng.run(now, opts)
    total, _ = eng.last_timing_ms()
    return total, eng.last_launch_count()


def main():
    eng = scheduler.Engine(0)
    out = {"gpu": gpu(), "reps": args.reps, "shapes": []}
    for name, make in shapes():
        w = make()
        eng.upload(w.tasks, w.distros)
        task_off = w.distros.task_off
        narrow = sum(1 for d in range(w.distros.n_distros) if not int(w.distros.cfg["group_versions"][d]) and
                     (w.tasks.n_edges == 0 or w.tasks.dep_off[task_off[d + 1]] == w.tasks.dep_off[task_off[d]]))
        opts = {"none": 0, "queue_breakdown": L.EVG_OPT_QUEUE_BREAKDOWN, "breakdown": L.EVG_OPT_BREAKDOWN}
        ms = {k: [] for k in opts}
        launches = {}
        fits = True
        for rep in range(args.reps + 1):  # round 0 warms every option up
            for k, o in opts.items():
                if k == "breakdown" and not fits:
                    continue
                try:
                    t, n = timed_run(eng, w.now, o)
                except L.EvgError as e:
                    if e.code != L.EVG_ERR_NOMEM:
                        raise
                    fits = False
                    continue
                launches[k] = n
                if rep:
                    ms[k].append(t)
        eng.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
        dq, dqb = [], []
        for rep in range(args.reps + 1):
            t0 = time.perf_counter()
            item_off, items = eng.download_queue(0, task_off)
            t1 = time.perf_counter()
            bd_off, bd = eng.download_queue_breakdown(0, task_off)
            t2 = time.perf_counter()
            if rep:
                dq.append((t1 - t0) * 1e3)
                dqb.append((t2 - t1) * 1e3)
        assert np.array_equal(item_off, bd_off) and np.array_equal(items["total_value"], bd[:, L.EVG_BD_TOTAL_VALUE])
        rows = int(item_off[-1])
        med = lambda v: round(float(np.median(v)), 3) if v else None  # noqa: E731
        out["shapes"].append({
            "shape": name, "tasks": int(w.n_tasks), "distros": int(w.distros.n_distros), "narrow_distros": narrow,
            "run_ms": {k: (med(v) if (k != "breakdown" or fits) else "does not fit") for k, v in ms.items()},
            "launches": launches,
            "persisted_rows": rows,
            "download_queue": {"ms": med(dq), "bytes": rows * L.QUEUE_ITEM_DTYPE.itemsize},
            "download_queue_breakdown": {"ms": med(dqb), "bytes": rows * 8 * L.EVG_BD_N},
            "breakdown_buffer_bytes": int(w.n_tasks) * 8 * L.EVG_BD_N,
        })
        del w
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
