#!/usr/bin/env python3
"""GetEstimatedStartTime for every persisted queue position of a resident tick, two routes, alternated in one process:
  host:   evg_download_queue (40 B per persisted item to the host), then the simulation on the CPU, one distro per task
          of a thread pool as wide as the machine (Python and numpy: what the mirror has, not a tuned C++ build);
  device: evg_estimate_start_times on the tick (17 B per host in, 8 B per persisted item and 4 B per distro out).
Shapes: configs[4] (100 000 ragged distros, synth.config(5), its own host counts) and the headline block (40 distros x
100 000 tasks: 40 persisted queues of 10 000 items, 1 000 hosts each).  Both routes end in a stream synchronise, so the
host clock around each spans its copies and kernels.  Per shape: warm-up, --reps alternating pairs of the device call and
the host route's download (medians), the CPU simulation timed once on its own (it does not touch the device), k_es_sim's
time from torch.profiler in a run of its own -- for the whole tick and for the distro with the most items x hosts alone,
the critical path -- and an equality check of the two routes.  Prints one JSON line with the card's name and power
limit."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import scheduler, synth  # noqa: E402
from evergreen_b200 import soa as S  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--scale", type=float, default=1.0)
args = ap.parse_args()
MINUTE = 60 * 10 ** 9
FIXED = np.array([4 * MINUTE, 3 * MINUTE, MINUTE, 0, 0, 0], np.int64)


def simulate(dur, pool):
    """One fresh run (model/task_start_estimation.go:53-96) over a sorted pool: the estimate of every position."""
    if pool.shape[0] == 0 or dur.shape[0] == 0:
        return np.full(dur.shape[0], -1, np.int64)
    out = np.empty(dur.shape[0], np.int64)
    if pool.shape[0] <= 24:  # a short pool: Python lists beat numpy's per-call cost
        p, e = pool.tolist(), 0
        for j, d in enumerate(dur.tolist()):
            ff = p[0]
            e += ff
            p = [v - ff for v in p[1:]]
            k = len(p)
            for i in range(len(p) - 1):
                if p[i] <= d <= p[i + 1]:
                    k = i
                    break
            p.insert(k, d)
            out[j] = e
        return out
    p, e = pool.copy(), np.zeros(1, np.int64)
    for j, d in enumerate(dur):
        ff = p[0]
        e += ff
        p = p[1:] - ff
        hit = (p[:-1] <= d) & (p[1:] >= d)
        p = np.insert(p, int(np.argmax(hit)) if hit.any() else p.shape[0], d)
        out[j] = e[0]
    return out


def random_hosts(rng, counts, now):
    H = int(np.sum(counts))
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return S.EstHostTable(rng.integers(0, 5, H).astype(np.uint8), rng.integers(MINUTE, 120 * MINUTE, H),
                          now - rng.integers(0, 60 * MINUTE, H), off)  # no overflow: the host route uses plain int64


def k_sim_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "k_es_sim" in e.key) / 1000.0


def measure(name, w, counts):
    eng = scheduler.Engine(0)
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    D = w.distros.n_distros
    hosts = random_hosts(np.random.default_rng(11), counts, w.now)
    ttc = np.where(hosts.kind == L.EVG_EH_RUNNING, hosts.expected_ns - (w.now - hosts.dispatch_ns), FIXED[hosts.kind])
    ho = hosts.est_host_off
    pools = [np.sort(ttc[ho[d]:ho[d + 1]]) for d in range(D)]

    def device():
        return eng.estimate_start_times(hosts, w.now, 0, w.distros.task_off)

    def download():
        return eng.download_queue(0, w.distros.task_off)

    def cpu(io, dur):
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            parts = list(ex.map(lambda d: simulate(dur[io[d]:io[d + 1]], pools[d]), range(D)))
        return np.concatenate(parts) if parts else np.zeros(0, np.int64)

    io, start, used = [x.copy() for x in device()]
    _, items = download()
    dur = items["expected_ns"].copy()
    t0 = time.perf_counter()
    want = cpu(io, dur)
    cpu_s = time.perf_counter() - t0
    same = bool(np.array_equal(start, want) and np.array_equal(used, np.diff(ho)))
    t_dev, t_dl = [], []
    for _ in range(3):
        device(), download()
    for _ in range(args.reps):
        t0 = time.perf_counter(); device(); t_dev.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); download(); t_dl.append(time.perf_counter() - t0)
    all_ms = k_sim_ms(device)
    work = np.diff(io) * np.diff(ho)
    top = int(np.argmax(work))
    alone = S.EstHostTable(hosts.kind[ho[top]:ho[top + 1]].copy(), hosts.expected_ns[ho[top]:ho[top + 1]].copy(),
                           hosts.dispatch_ns[ho[top]:ho[top + 1]].copy(), np.where(np.arange(D + 1) > top, ho[top + 1] - ho[top], 0).astype(np.int64))
    eng.estimate_start_times(alone, w.now, 0, w.distros.task_off)
    top_ms = k_sim_ms(lambda: eng.estimate_start_times(alone, w.now, 0, w.distros.task_off))
    N, H = int(io[-1]), hosts.n_hosts
    eng.close()
    return {"shape": name, "distros": D, "items": N, "hosts": H, "same": same, "threads": os.cpu_count(),
            "device_ms": round(1e3 * float(np.median(t_dev)), 3), "host_download_ms": round(1e3 * float(np.median(t_dl)), 3),
            "host_cpu_simulation_ms": round(1e3 * cpu_s, 1), "k_es_sim_ms": round(all_ms, 4),
            "largest_distro": {"items": int(np.diff(io)[top]), "hosts": int(np.diff(ho)[top]), "k_es_sim_ms": round(top_ms, 4)},
            "bytes_device_route": {"to_device": 17 * H + 8 * (D + 1), "to_host": 8 * N + 4 * D},
            "bytes_host_route": {"to_device": 8 * (D + 1), "to_host": 40 * N}}


c5 = synth.config(5, args.scale)
block = synth.make(np.full(40, 100_000, dtype=np.int64), synth.SEED_BASE + 3, zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02,
                   includes_dependencies=True, n_hosts=80)
out = {"results": [measure("configs[4]", c5, np.diff(c5.hosts.host_off)),
                   measure("headline block: 40 distros x 100k tasks", block, np.full(40, 1000))]}
try:
    out["gpu"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]).decode().strip()
except Exception as e:  # noqa: BLE001
    out["gpu"] = f"unknown ({e})"
print(json.dumps(out))
