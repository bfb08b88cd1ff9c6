#!/usr/bin/env python3
"""The DAG dispatcher of every persisted queue of a resident tick, two routes, alternated in one process:
  host:   evg_download_queue (40 B per persisted item to the host) -> the persisted queue's dependency CSR and dense group
          ids in numpy (soa.persisted_dag_input, from the shim's own columns) -> evg_dag_rebuild_batch on a second
          context (it ends the tick of the context it runs on);
  device: evg_rebuild_dispatchers on the tick itself.
Shapes: the flagship (--distros distros x --tasks tasks in configs[2]'s mix, a generated block of --block distros tiled
as bench.py tiles it; persisted heads of 10 000 items) and configs[4] (100 000 ragged distros).  Both calls end in a
stream synchronise, so the host clock around each spans its copies and kernels.  Per shape: warm-up, --reps alternating
pairs, the launch count, the bytes each route moves over PCIe (computed from the shapes), torch.profiler's k_dag_*,
k_seg_merge_pass and k_dp_* kernel times of one device call, and an equality check of every output array.  Prints one
JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import scheduler, soa, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--distros", type=int, default=2000)
ap.add_argument("--tasks", type=int, default=100_000, help="tasks per distro of the flagship shape")
ap.add_argument("--block", type=int, default=10, help="distros generated, then tiled")
ap.add_argument("--c5-scale", type=float, default=1.0)
args = ap.parse_args()


def tiled(n_distros: int, per: int, block: int) -> synth.Workload:
    """configs[2]'s mix (synth.config(3, each=True)'s arguments) on a block of distros, tiled to n_distros: task groups,
    versions and edges are distro-local, so the tiles are valid queues of their own."""
    b = synth.make(np.full(block, per, dtype=np.int64), synth.SEED_BASE + 3, zipf_priority=True, unmet_dep_frac=0.05,
                   met_dep_frac=0.02, includes_dependencies=True, tg_frac=0.1)
    reps = n_distros // block
    t, dt = b.tasks, b.distros
    cols = {name: np.tile(getattr(t, name), reps) for name, _ in soa.TaskSoA.COLUMNS}
    E = t.n_edges
    dep_off = np.concatenate([[0], (t.dep_off[1:][None, :] + E * np.arange(reps)[:, None]).ravel()]).astype(np.int64)
    tasks = soa.TaskSoA(**cols, dep_off=dep_off, dep_idx=np.tile(t.dep_idx, reps)).normalize()
    T, G = b.n_tasks, dt.n_groups
    task_off = np.concatenate([[0], (dt.task_off[1:][None, :] + T * np.arange(reps)[:, None]).ravel()]).astype(np.int64)
    group_off = np.concatenate([[0], (dt.group_off[1:][None, :] + G * np.arange(reps)[:, None]).ravel()]).astype(np.int64)
    distros = soa.DistroTable(task_off, group_off, np.tile(dt.cfg, reps), np.tile(dt.group_max_hosts, reps)).normalize()
    return synth.Workload(f"{reps * block} distros x {per} tasks", b.now, tasks, distros, None)


def host_route(eng, other, w):
    item_off, items = eng.download_queue(0, w.distros.task_off)
    D = w.distros.n_distros
    lens = np.diff(item_off)
    d_of = np.repeat(np.arange(D), lens)
    order = np.zeros(max(w.n_tasks, 1), dtype=np.int32)
    order[w.distros.task_off[d_of] + np.arange(int(item_off[-1])) - item_off[d_of]] = items["task"]
    io, go, dep_off, dep_item, gid, gidx, gslot = soa.persisted_dag_input(w.tasks, w.distros, order, 0)
    srt, ns, nc, ui, uo = other.dag_rebuild_batch(io, go, dep_off, dep_item, gid, gidx)
    return {"item_off": io, "sorted": srt, "n_sorted": ns, "n_cycles": nc, "group_off": go, "group_slot": gslot,
            "unit_items": ui, "unit_off": uo}, int(dep_item.shape[0])


def profile_device(eng):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        eng.rebuild_dispatchers(0)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = next((n for n in ("k_dag_topo", "k_dag_group_init", "k_seg_merge_pass", "k_dag_units", "k_dp_gather",
                                     "k_dp_edges", "k_dp_groups", "k_scan_") if n in e.name), None)
            if name:
                us = e.device_time if hasattr(e, "device_time") else e.cuda_time
                kern[name] = kern.get(name, 0.0) + us / 1e3
    return kern


def measure(name, w):
    eng, other = scheduler.Engine(0), scheduler.Engine(0)
    eng.upload(w.tasks, w.distros)
    eng.run(w.now)
    eng.rebuild_dispatchers(0)  # warm-up: first allocations on both contexts
    host_route(eng, other, w)
    ms = {"host": [], "device": []}
    for _ in range(args.reps):
        n0 = eng.last_launch_count()
        t0 = time.perf_counter()
        h, E_items = host_route(eng, other, w)
        ms["host"].append((time.perf_counter() - t0) * 1e3)
        host_launches = eng.last_launch_count() - n0 + other.last_launch_count()  # k_project_queue, then the DAG kernels
        t0 = time.perf_counter()
        d = eng.rebuild_dispatchers(0)
        ms["device"].append((time.perf_counter() - t0) * 1e3)
        dev_launches = eng.last_launch_count()
    same = all(np.array_equal(d[f], h[f]) for f in L.DISPATCH_OUT_FIELDS)
    D, N, G2 = w.distros.n_distros, int(d["item_off"][-1]), int(d["group_off"][-1])
    out_bytes = 4 * (2 * N + 2 * D + G2 + G2 + D)  # sorted, unit_items, n_sorted, n_cycles, unit_off, (group_slot: device only)
    pcie = {"host": {"d2h": 40 * N + 8 * (D + 1) + out_bytes - 4 * G2,
                     "h2d": 8 * 2 * (D + 1) + 8 * (N + 1) + 4 * E_items + 8 * N + 4 * D},
            "device": {"d2h": 8 * (D + 1) + out_bytes, "h2d": 8 * (D + 1)}}
    res = {"shape": name, "distros": D, "tasks": w.n_tasks, "items": N, "item_edges": E_items, "groups": G2,
           "cycles": int(d["n_cycles"].sum()), "identical": bool(same), "reps": args.reps,
           "ms": {k: [round(x, 3) for x in v] for k, v in ms.items()},
           "median_ms": {k: float(np.median(v)) for k, v in ms.items()}, "launches": {"host": host_launches, "device": dev_launches},
           "pcie_bytes": pcie, "device_kernel_ms": profile_device(eng)}
    eng.close()
    other.close()
    return res


try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "unknown"
runs = [measure("flagship", tiled(args.distros, args.tasks, args.block))]
runs.append(measure("configs[4]", synth.config(5, args.c5_scale)))
print(json.dumps({"card": card, "runs": runs}))
