"""Tick-to-tick cost of a shim's tick loop with the strings interned on the host vs kept on the device.  Three arms on
the same Go-level batches, alternating their order per step in one process:
  (a) ResidentTick().plan -- marshal_tasks interns every string of the batch on the host, diff() rebuilds the remaps
      and gained edges, evg_edit_tasks + evg_update_tasks send the edit;
  (b) evg_upload_strings of the whole composed batch (numeric columns marshalled on the host, every string shipped);
  (c) ResidentTick(device_strings=True).plan -- the numeric columns only on the host, evg_edit_strings ships the
      departures' rows and the arrivals' columns and strings, evg_update_tasks the changed scalars.
Workload: tests/edit_strings_scripts.Script -- task groups and versions that appear and vanish, DependsOn lists with
forward references, departed targets, other distros' and external ids -- with `--frac` of each queue leaving and
arriving per step.  After each step every arm's download_queue rows must be equal.  Per arm: the median and range per
step of the wall time, of the time inside the engine's calls (host clock around synchronised calls: upload / edit /
update / run / download), and of the rest (host marshalling); the H2D bytes per step; the device memory the arm's
context holds after its first tick (cudaMemGetInfo deltas); and the card's name and power limit.

    python profiles/edit_strings_tick.py --distros 200 --tasks-per-distro 2000 --steps 6 --warmup 1
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ENGINE_CALLS = ("upload", "upload_strings", "edit_tasks", "edit_strings", "update_tasks", "run", "download")


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def timed_engine(eng, acc, torch):
    """Wrap the engine's tick calls: each is synchronised and its wall time added to acc[0]."""
    for name in ENGINE_CALLS:
        f = getattr(eng, name)

        def wrapped(*a, _f=f, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = _f(*a, **kw)
            torch.cuda.synchronize()
            acc[0] += time.perf_counter() - t0
            return r
        setattr(eng, name, wrapped)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--distros", type=int, default=200)
    ap.add_argument("--tasks-per-distro", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frac", type=float, default=0.05)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from evergreen_b200 import scheduler, soa as S
    import edit_strings_scripts as X

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures on the GPU only")
    script = X.Script(2024, sizes=(args.tasks_per_distro,) * args.distros)
    keys = ("a_host_interning", "b_upload_strings", "c_device_strings")
    engines, acc, mem = {}, {}, {}
    for a in keys:
        engines[a] = scheduler.Engine(0)
        acc[a] = [0.0]
        mem[a] = 0
        timed_engine(engines[a], acc[a], torch)
    rts = {"a_host_interning": scheduler.ResidentTick(engines["a_host_interning"]),
           "c_device_strings": scheduler.ResidentTick(engines["c_device_strings"], device_strings=True)}
    wall, call, h2d = ({a: [] for a in keys} for _ in range(3))
    batch = script.batch
    for k in range(1 + args.warmup + args.steps):
        if k > 0:
            batch = script.next_batch(leave=args.frac, arrive=args.frac)
        copies = {a: copy.deepcopy(batch) for a in keys}  # each arm stamps its own Task objects
        res = {}

        def arm_rt(a):
            def run():
                acc[a][0] = 0.0
                t0 = time.perf_counter()
                rts[a].plan(copies[a], X.NOW)
                t1 = time.perf_counter()
                last = rts[a].last
                if last is None:
                    n = rts[a].soa.nbytes() + sum(len(t.id) + len(t.version) for _, ts in batch for t in ts)
                else:
                    n = last[0].nbytes() + 48 * int(last[1].shape[0])
                res[a] = ((t1 - t0) * 1e3, acc[a][0] * 1e3, n)
            return run

        def arm_b():
            a = "b_upload_strings"
            eng = engines[a]
            acc[a][0] = 0.0
            t0 = time.perf_counter()
            canon = rts["c_device_strings"].canonical(copies[a]) if k > 0 else copies[a]
            soa, table, _ = S.marshal_tasks(canon, X.NOW, resolve_deps=True, intern=False)
            sc = S.string_cols(canon)
            eng.upload_strings(soa, sc, table.cfg)
            eng.run(X.NOW, 0)
            eng.download(want_alloc=False)
            t1 = time.perf_counter()
            n = soa.nbytes() - soa.group_id.nbytes - soa.version_id.nbytes + sc.group_max_hosts.nbytes + sc.dep_off.nbytes
            n += sum(c[0].nbytes + c[1].nbytes for c in (sc.id, sc.version, sc.group_key, sc.dep_id))
            res[a] = ((t1 - t0) * 1e3, acc[a][0] * 1e3, n)

        # arm (b) takes the canonical order arm (c) will plan, so it runs before (c) has remembered this step
        arms = {"a_host_interning": arm_rt("a_host_interning"), "b_upload_strings": arm_b, "c_device_strings": arm_rt("c_device_strings")}
        for a in (keys if k % 2 == 0 else ("b_upload_strings", "c_device_strings", "a_host_interning")):
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            arms[a]()
            mem[a] += free0 - torch.cuda.mem_get_info()[0]  # what the arm's context added (its buffers only grow)
        q = []
        for a in keys:
            eng = engines[a]
            eng.run(X.NOW, 0)
            task_off = rts["c_device_strings"].table.task_off
            off, items = eng.download_queue(0, task_off)
            q.append((off.copy(), items.copy()))
        for j in (1, 2):
            assert np.array_equal(q[0][0], q[j][0]) and np.array_equal(q[0][1], q[j][1]), f"step {k}: download_queue of {keys[j]}"
        print(json.dumps({"step": k, "wall_ms": {a: round(res[a][0], 1) for a in keys}}), flush=True)
        if k > args.warmup:
            for a in keys:
                wall[a].append(res[a][0])
                call[a].append(res[a][1])
                h2d[a].append(res[a][2])
    free_end = torch.cuda.mem_get_info()[0]
    rng_of = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}  # noqa: E731
    out = {"gpu": gpu_info(), "distros": args.distros, "tasks": int(rts["c_device_strings"].table.task_off[-1]),
           "steps": args.steps, "frac": args.frac,
           "wall_ms_per_step": {a: rng_of(v) for a, v in wall.items()},
           "engine_call_ms_per_step": {a: rng_of(v) for a, v in call.items()},
           "host_ms_per_step": {a: rng_of(np.array(wall[a]) - np.array(call[a])) for a in keys},
           "h2d_bytes_per_step": {a: int(np.mean(v)) for a, v in h2d.items()},
           "device_bytes_per_context": {a: int(v) for a, v in mem.items()},
           "device_free_bytes_end": int(free_end),
           "outputs_equal_every_step": True}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
