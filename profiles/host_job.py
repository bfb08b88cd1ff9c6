#!/usr/bin/env python3
"""hostAllocatorJob.Run past the allocator for every distro of a resident tick, two routes, alternated in one process:
  host:   evg_download of the queue infos, group infos and allocator results (152 + 72 per group slot + 20 B per
          distro to the host), then the job in numpy, vectorised over distros;
  device: evg_host_job on the tick (24 B per distro in, 116 B per distro out).
Shapes: configs[4] (100 000 ragged distros, synth.config(5)) and configs[3] total (10 000 distros x 100 tasks,
synth.config(4)).  Both routes end in a stream synchronise, so the host clock around each spans its copies and kernels.
Per shape: warm-up, --reps alternating pairs (median reported), k_host_job's time from torch.profiler in a run of its
own, and an equality check of the two routes (floats as bits).  Prints one JSON line with the card's name and power
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
from evergreen_b200 import scheduler, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--scale", type=float, default=1.0)
args = ap.parse_args()
MAXT = np.int64(2532000 * 3600 * 10 ** 9)


def host_job(po, ao, group_off, host_off, acfg, cfg):
    """The job (units/host_allocator.go:180-337, 394-425) in numpy over all distros; spawned = max(n_hosts, 0)."""
    q, g = po.info, po.group_info
    single = cfg["single_task_distro"] != 0
    n_slots = np.diff(group_off)
    has = n_slots > 0
    starts = np.minimum(group_off[:-1], max(g.shape[0] - 1, 0))

    def gsum(f, zero_single=False):
        s = np.add.reduceat(g[f], starts) if g.shape[0] else np.zeros_like(n_slots)
        s = np.where(has, s, 0)
        return np.where(single, 0, s) if zero_single else s
    with np.errstate(over="ignore"):
        n_hosts = np.where(single, q["length_with_dependencies_met"] - cfg["n_provisioning"], ao.result["new_hosts"].astype(np.int64))
        n_free = np.where(single, 0, ao.result["free_hosts"].astype(np.int64))
        status = np.where(single, 0, ao.status)
        spawned = np.maximum(n_hosts, 0)
        free, required = gsum("count_free", True), gsum("count_required", True)
        sched = (q["expected_duration"] - gsum("expected_duration")) - (q["duration_over_threshold"] - gsum("duration_over_threshold"))
        over = q["count_duration_over_threshold"] - gsum("count_duration_over_threshold")
        corr = spawned - required
        avail = (n_free - free) + corr - over
        avail_ns = avail - corr
        pos = sched > 0
        tte = np.where(pos, np.where(avail <= 0, MAXT, sched // np.where(avail > 0, avail, 1)), 0)
        tte_ns = np.where(pos, np.where((avail <= 0) | (avail_ns <= 0), MAXT, sched // np.where(avail_ns > 0, avail_ns, 1)), 0)
    thr = q["max_duration_threshold"].astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = tte.astype(np.float32) / thr
        ratio_ns = tte_ns.astype(np.float32) / thr
    n_up = np.diff(host_off)
    cond = (cfg["terminate_when_overallocated"] != 0) & (acfg["provider"] != L.EVG_PROVIDER_STATIC) & (ratio < np.float32(0.25)) \
        & (n_up > 0) & (cfg["hourly_billing"] == 0) & (status == 0)
    with np.errstate(over="ignore", invalid="ignore"):
        prod = n_up.astype(np.float32) * (np.float32(1) - ratio)
        kill = np.where(ratio == 0, n_up, np.where(prod >= np.float32(2.0 ** 63), np.iinfo(np.int64).max,
                                                    np.trunc(np.where(cond, prod, 0)).astype(np.int64)))
    cap = np.maximum(np.where(ratio == 0, 0, n_up - kill), acfg["minimum_hosts"])
    ok = status == 0
    rep = np.zeros(n_up.shape[0], L.HOST_REPORT_DTYPE)
    for f, v in (("time_to_empty_ns", tte), ("time_to_empty_no_spawns_ns", tte_ns), ("scheduled_duration_ns", sched),
                 ("hosts_avail", avail), ("hosts_spawned", spawned), ("overdue_in_groups", gsum("count_wait_over_threshold")),
                 ("free_in_groups", free), ("required_in_groups", required), ("host_queue_ratio", ratio),
                 ("no_spawns_ratio", ratio_ns)):
        rep[f] = np.where(ok, v, 0)
    rep["killable_hosts"] = np.where(cond, kill, 0)
    rep["new_cap_target"] = np.where(cond, cap, 0)
    rep["drawdown"] = cond & (kill > 0)
    return {"n_hosts": n_hosts, "n_hosts_free": n_free, "status": status, "report": rep}


def measure(name, w):
    eng = scheduler.Engine(0)
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    D = w.distros.n_distros
    rng = np.random.default_rng(7)
    cfg = np.zeros(D, L.HOST_JOB_CFG_DTYPE)
    cfg["n_provisioning"] = rng.integers(0, 3, D)
    cfg["single_task_distro"] = rng.random(D) < 0.1
    cfg["terminate_when_overallocated"] = rng.random(D) < 0.7
    cfg["hourly_billing"] = rng.random(D) < 0.3

    def host():
        po, ao = eng.download(want_alloc=True)
        return host_job(po, ao, w.distros.group_off, w.hosts.host_off, w.hosts.cfg, cfg)

    def device():
        return eng.host_job(cfg)
    a, b = device(), host()
    same = all(np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).astype(a[k].dtype).view(np.uint8))
               for k in ("n_hosts", "n_hosts_free", "status")) and \
        all(np.array_equal(a["report"][f].view(np.uint32 if a["report"][f].dtype == np.float32 else a["report"][f].dtype),
                           b["report"][f].astype(a["report"][f].dtype).view(np.uint32 if a["report"][f].dtype == np.float32
                                                                            else a["report"][f].dtype))
            for f in L.HOST_REPORT_FIELDS)
    t_dev, t_host = [], []
    for _ in range(3):
        device(), host()
    for _ in range(args.reps):
        t0 = time.perf_counter(); device(); t_dev.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); host(); t_host.append(time.perf_counter() - t0)
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device()
        torch.cuda.synchronize()
    k_ms = sum(e.device_time_total for e in prof.key_averages() if "k_host_job" in e.key) / 1000.0
    G = int(w.distros.group_off[-1])
    eng.close()
    return {"shape": name, "distros": D, "group_slots": G, "tasks": int(w.n_tasks), "same": bool(same),
            "device_ms": round(1e3 * float(np.median(t_dev)), 3), "host_ms": round(1e3 * float(np.median(t_host)), 3),
            "k_host_job_ms": round(k_ms, 4), "bytes_to_host_device": D * 116, "bytes_to_host_host": D * (152 + 20) + G * 72}


out = {"results": [measure("configs[4]", synth.config(5, args.scale)), measure("configs[3]", synth.config(4, args.scale))]}
try:
    out["gpu"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().strip()
except Exception as e:  # noqa: BLE001
    out["gpu"] = f"unknown ({e})"
print(json.dumps(out))
