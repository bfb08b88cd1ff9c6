#!/usr/bin/env python3
"""The legacy prioritiser with EVG_LEGACY_MODE_GO_STABLE (the device replay of Go's sort.Stable) next to the key sort,
on two shapes:
  1 000 distros x 10 000 tasks   (about half commit builds, half patch tasks, a few high-priority patch tasks)
  4 distros x 1 000 000 tasks
Each shape runs twice: "exact" with the commit builds spread over three projects, so the repotracker list is one on
which the chain is not a strict weak order and goes GO_STABLE (as soa.marshal_legacy(exact=True) marks it), and
"key" with every commit build in one project, so that list is REVISION and is key-sorted.  The patch and high-priority
lists are INGEST in both.  Per run: the call's wall time (a host clock around evg_prioritize_legacy_batch, which
uploads the columns and ends in a stream synchronise; median of --reps after a warm-up), the kernels' device time
summed from torch.profiler in a call of its own, the launch count, and a spot-check of --check
distros of the first shape against oracle/oracle_legacy.py.  Prints one JSON line with the card's name and power
limit."""
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
from evergreen_b200 import scheduler  # noqa: E402
from evergreen_b200 import soa as S  # noqa: E402
from oracle import oracle_legacy as OL  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--check", type=int, default=3, help="distros of the first shape compared with the oracle")
args = ap.parse_args()
NOW = 1_700_000_000 * M.SECOND


def make_table(D, n, projects, seed):
    rng = np.random.default_rng(seed)
    T = D * n
    system = rng.random(T) < 0.5
    prio = np.where(~system & (rng.random(T) < 0.02), 150, rng.choice(np.array([0, 0, 1, 5]), T)).astype(np.int64)
    flags = (np.where(system, L.EVG_LF_REQ_SYSTEM, L.EVG_LF_REQ_PATCH) | np.where(rng.random(T) < 0.05, L.EVG_LF_GENERATE, 0)).astype(np.uint32)
    presort = np.concatenate([rng.permutation(n) for _ in range(D)]).astype(np.int32)
    repo = L.EVG_LEGACY_MODE_GO_STABLE if projects > 1 else L.EVG_LEGACY_MODE_REVISION
    return S.LegacyTable(
        priority=prio, ingest_ns=(NOW - rng.integers(0, 48, T) * M.HOUR).astype(np.int64),
        expected_ns=(rng.integers(1, 60, T) * M.MINUTE).astype(np.int64), num_dependents=rng.choice(np.array([0, 0, 0, 1, 3], np.int32), T),
        revision_order=rng.integers(0, 200, T).astype(np.int32), project_id=rng.integers(0, projects, T).astype(np.int32),
        tg_rank=np.full(T, -1, np.int32), tg_pair_id=np.full(T, -1, np.int32), task_group_order=np.zeros(T, np.int32),
        presort_rank=presort, flags=flags, task_off=(np.arange(D + 1, dtype=np.int64) * n),
        list_mode=np.tile(np.array([L.EVG_LEGACY_MODE_INGEST, L.EVG_LEGACY_MODE_INGEST, repo], np.uint8), D))


def tasks_of(tb, d):
    """Distro d of the table as model tasks: ids whose descending order is the presort, no task groups."""
    a, b = int(tb.task_off[d]), int(tb.task_off[d + 1])
    n = b - a
    return [M.Task(id=f"{n - 1 - int(tb.presort_rank[i]):08d}", priority=int(tb.priority[i]), ingest_time=int(tb.ingest_ns[i]),
                   expected_duration=int(tb.expected_ns[i]), num_dependents=int(tb.num_dependents[i]),
                   revision_order_number=int(tb.revision_order[i]), project=f"p{int(tb.project_id[i])}",
                   generate_task=bool(tb.flags[i] & L.EVG_LF_GENERATE),
                   requester=M.REPOTRACKER_VERSION_REQUESTER if (tb.flags[i] & 3) == L.EVG_LF_REQ_SYSTEM else M.PATCH_VERSION_REQUESTER)
            for i in range(a, b)]


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1000.0


def measure(eng, name, tb, check):
    call = lambda: eng.prioritize_legacy_batch(tb)  # noqa: E731
    order, count, status = (x.copy() for x in call())
    launches = eng.last_launch_count()
    res = {"shape": name, "distros": tb.n_distros, "tasks": tb.n_tasks, "launches": launches,
           "go_stable_lists": int((tb.list_mode == L.EVG_LEGACY_MODE_GO_STABLE).sum()), "all_ok": bool((status == L.EVG_LEGACY_OK).all())}
    if check:
        same = []
        for d in np.linspace(0, tb.n_distros - 1, check).astype(int).tolist():
            tasks = tasks_of(tb, d)
            a = int(tb.task_off[d])
            got = [tasks[int(i)].id for i in order[a:a + int(count[d])]]
            same.append(got == [t.id for t in OL.prioritize_tasks(tasks, {}, None)])
        res["oracle_checked"], res["oracle_equal"] = len(same), all(same)
    for _ in range(2):
        call()
    t = []
    for _ in range(args.reps):
        t0 = time.perf_counter(); call(); t.append(time.perf_counter() - t0)
    res["call_ms"] = round(1e3 * float(np.median(t)), 2)
    res["kernel_ms"] = round(kernel_ms(call), 3)
    return res


eng = scheduler.Engine(0)
out = {"results": []}
for name, D, n in (("1000 x 10k", 1000, 10_000), ("4 x 1M", 4, 1_000_000)):
    for label, projects in (("exact", 3), ("key", 1)):
        tb = make_table(D, n, projects, seed=D)
        out["results"].append(measure(eng, f"{name} {label}", tb, args.check if D > 4 else 0))
        del tb
eng.close()
try:
    out["gpu"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]).decode().strip()
except Exception as e:  # noqa: BLE001
    out["gpu"] = f"unknown ({e})"
print(json.dumps(out))
