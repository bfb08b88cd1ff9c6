#!/usr/bin/env python3
"""The drawdown job and the idle-host job for every distro, device against the Python restatement:
  device: evg_host_drawdown (standalone) and evg_idle_hosts on the idle-host table, host clock around each call (each
          ends in a stream synchronise, so the time spans the table's upload, the kernels and the copies back);
  python: tests/oracle_host_termination.py over the same Host objects (one pass; it is seconds, not milliseconds).
Shapes: C4 (50 000 idle hosts over 10 000 distros) and 1e6 idle hosts over 100 000 distros, from synth.make_idle_hosts.
Per shape: warm-up, --reps calls of each (median reported), the kernels' times from torch.profiler in a run of their
own, and an equality check of device and restatement.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import oracle_host_termination as OT  # noqa: E402
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import model as M  # noqa: E402
from evergreen_b200 import scheduler, synth  # noqa: E402
from evergreen_b200 import soa as S  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=None, help="also write the JSON line to OUT/host_termination.json")
args = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.name.startswith("k_"):
            out[e.name] = out.get(e.name, 0.0) + e.device_time_total / 1000.0
    return out


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def shape(eng, name, sizes, seed):
    w = synth.make_idle_hosts(sizes, seed)
    cap = np.array([L.EVG_NO_DRAWDOWN if x is None else x.new_cap_target for x in w.drawdown], np.int64)
    ex, qlen = np.asarray(w.existing, np.int64), np.asarray(w.queue_lengths, np.int64)
    t_dd = S.marshal_idle_hosts(w.groups)
    t_id = S.marshal_idle_hosts(w.groups, [(d or M.Distro()).default_ami for d in w.distros])
    cfg = np.zeros(len(w.distros), L.IDLE_CFG_DTYPE)
    for i, d in enumerate(w.distros):
        d = d or M.Distro()
        cfg[i] = (d.host_allocator_settings.minimum_hosts, int(w.running_counts[i]),
                  d.host_allocator_settings.acceptable_host_idle_time or w.sched_idle_seconds * M.SECOND)
    dd = lambda: eng.host_drawdown(t_dd, ex, w.now, cap, qlen)  # noqa: E731
    ih = lambda: eng.idle_hosts(t_id, cfg, w.now)  # noqa: E731
    for _ in range(3):
        dd(), ih()
    dev_dd, dev_ih = median_ms(dd, args.reps), median_ms(ih, args.reps)
    t = time.perf_counter()
    want_dd = []
    for d, g in enumerate(w.groups):
        want_dd += ([OT.NOT_CHECKED] * len(g) if w.drawdown[d] is None else
                    OT.drawdown_job(f"d{d}", g, int(ex[d]), int(cap[d]), int(qlen[d]), w.now)[1])
    py_dd = (time.perf_counter() - t) * 1e3
    t = time.perf_counter()
    want_ih = []
    for d, g in enumerate(w.groups):
        want_ih += OT.idle_job(w.distros[d], g, int(w.running_counts[d]), w.now, w.sched_idle_seconds)[1]
    py_ih = (time.perf_counter() - t) * 1e3
    fields = ("decision", "idle_ns", "communication_ns", "threshold_ns", "since_teardown_ns")
    same = all([tuple(int(v[f]) for f in fields) for v in res["hosts"]] == want
               for res, want in ((dd(), want_dd), (ih(), want_ih)))
    return {"shape": name, "hosts": t_dd.n_hosts, "distros": t_dd.n_distros, "same_as_restatement": same,
            "drawdown_ms": round(dev_dd, 3), "idle_ms": round(dev_ih, 3), "python_drawdown_ms": round(py_dd, 1),
            "python_idle_ms": round(py_ih, 1), "drawdown_kernels_ms": kernel_ms(dd), "idle_kernels_ms": kernel_ms(ih),
            "table_bytes": int(t_dd.n_hosts * (8 * 8 + 4))}


def main():
    eng = scheduler.Engine(0)
    try:
        rows = [shape(eng, "C4", np.full(10_000, 5, np.int64), 2602),
                shape(eng, "1e6", np.full(100_000, 10, np.int64), 2603)]
    finally:
        eng.close()
    line = json.dumps({"card": card(), "reps": args.reps, "rows": rows})
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "host_termination.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
