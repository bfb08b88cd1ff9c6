#!/usr/bin/env python3
"""Device interning against host interning at the intern_bench shape:
`python profiles/intern_device.py [steps] [out.json]`.

For D x 10 000 tasks (D = 200, 2 000), per step and in alternating order:
  host     evg_intern_columns on every host core;
  device   evg_intern_batch end to end (strings H2D, kernels, outputs D2H);
  upload   evg_intern_columns + evg_upload + evg_run_resident, against
  strings  evg_upload_strings + evg_run_resident (each until the device is idle).
Outputs are compared at every step.  A separate torch.profiler pass over one evg_intern_batch gives its kernel and copy
time.  Prints one JSON line (and writes it to out.json when given) with the card's name and power limit, read in the
same process."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from evergreen_b200 import _lib as L  # noqa: E402
from evergreen_b200 import scheduler  # noqa: E402
from evergreen_b200 import soa as S  # noqa: E402
from evergreen_b200 import synth  # noqa: E402
import intern_bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def numeric_tasks(T, seed):
    rng = np.random.default_rng(seed)
    cols = {"priority": rng.integers(0, 100, T), "expected_ns": rng.integers(1, 3_600_000_000_000, T),
            "queue_basis_ns": synth.NOW_NS - rng.integers(0, 86_400_000_000_000, T),
            "wait_basis_ns": synth.NOW_NS - rng.integers(0, 86_400_000_000_000, T), "num_dependents": rng.integers(0, 5, T),
            "task_group_order": rng.integers(0, 25, T), "group_id": np.zeros(T), "version_id": np.zeros(T),
            "flags": rng.integers(0, 2, T) | L.EVG_TF_DEPS_MET}
    return S.TaskSoA(**{name: np.ascontiguousarray(cols[name], dt) for name, dt in S.TaskSoA.COLUMNS})


def kernel_ms(eng, sc):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.intern_batch(sc)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    k = sum(e.device_time for e in ev if e.name.startswith("k_") or e.name.startswith("void k_")) / 1e3
    copy = sum(e.device_time for e in ev if "Memcpy" in e.name) / 1e3
    return k, copy


def shape(D, per, steps):
    import torch
    T, ids, vers, gk, dep_off, tgt = intern_bench.make(D, per)
    sc = S.StringCols.pack(np.arange(D + 1, dtype=np.int64) * per, ids, vers, gk, np.ones(T, np.int32), dep_off, tgt)
    del ids, vers, gk, tgt
    nbytes = sum(c[0].nbytes for c in (sc.id, sc.version, sc.group_key, sc.dep_id))
    tasks = numeric_tasks(T, D)
    cfg = np.zeros(D, L.DISTRO_CFG_DTYPE)
    lib = L.load()
    eng = scheduler.Engine(0)
    times = {k: [] for k in ("host", "device", "upload", "strings")}

    def host():
        out, outs = sc.intern_out()
        L.check(lib.evg_intern_columns(C.byref(sc.struct()), C.byref(outs), 0))
        return sc.trim(out)

    def timed(key, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        times[key].append(time.perf_counter() - t0)
        return r

    def upload_arm():
        h = host()
        t = S.TaskSoA(**{name: getattr(tasks, name) for name, _ in S.TaskSoA.COLUMNS}, dep_off=h["dep_off"], dep_idx=h["dep_idx"])
        t.group_id, t.version_id = h["group_id"], h["version_id"]
        c = cfg.copy()
        c["n_versions"] = h["n_versions"]
        eng.upload(t.normalize(), S.DistroTable(sc.task_off, h["group_off"], c, h["group_max_hosts"]).normalize())
        eng.run(synth.NOW_NS)
        return h

    def strings_arm():
        h = eng.upload_strings(tasks, sc, cfg)
        eng.run(synth.NOW_NS)
        return h

    def ranks():
        po, _ = eng.download()
        return po.order.copy(), po.total_value.copy()

    for step in range(steps + 1):  # step 0 warms every arm up and is not kept
        arms = [("host", host), ("device", lambda: eng.intern_batch(sc))]
        for key, fn in (arms if step % 2 == 0 else arms[::-1]):
            got = timed(key, fn)
            if key == "host":
                want = got
            else:
                dev = got
        for k in S.INTERN_OUT_FIELDS:
            assert np.array_equal(want[k], dev[k]), k
        res = {}
        for key, fn in ([("upload", upload_arm), ("strings", strings_arm)] if step % 2 == 0 else [("strings", strings_arm), ("upload", upload_arm)]):
            timed(key, fn)
            res[key] = ranks()
        for a, b in zip(res["upload"], res["strings"]):
            assert np.array_equal(a, b)
        if step == 0:
            for v in times.values():
                v.clear()
    k_ms, copy_ms = kernel_ms(eng, sc)
    eng.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {"distros": D, "tasks": T, "string_bytes": int(nbytes), "edges": int(sc.dep_off[-1]), "steps": steps,
            "median_s": med, "tasks_per_s": {k: T / v for k, v in med.items()},
            "intern_batch_kernel_ms": k_ms, "intern_batch_copy_ms": copy_ms,
            "intern_batch_kernel_GB_per_s": nbytes / (k_ms / 1e3) / 1e9,
            "intern_batch_end_to_end_GB_per_s": nbytes / med["device"] / 1e9}


if __name__ == "__main__":
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 4
    res = {"card": card(), "host_cores": os.cpu_count(), "shapes": [shape(D, 10_000, steps) for D in (200, 2000)]}
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            f.write(line + "\n")
