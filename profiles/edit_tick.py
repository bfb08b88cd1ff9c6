"""Tick-to-tick cost of a changing queue: (a) evg_upload of the composed table vs (b) evg_edit_tasks + evg_update_tasks,
each followed by evg_run_resident and evg_download_queue, alternating per step on the bench's headline mix (configs[2]
per-distro: Zipf priorities, 5 % unmet + 2 % met in-queue dependencies, 10 % of tasks in task groups).  Every step
dispatches 5 % of the rows (biased to the heads of the last ranked queues), inserts 5 % and changes 5 %.  Reports ms per
step (host clock around synchronised work), H2D bytes per step and device memory in use, and asserts that both arms'
download_queue rows are equal at every step.

    python profiles/edit_tick.py --distros 2000 --tasks-per-distro 100000 --steps 10 --warmup 2
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--distros", type=int, default=2000)
    ap.add_argument("--tasks-per-distro", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frac", type=float, default=0.05)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from evergreen_b200 import scheduler, synth

    w = synth.make(np.full(args.distros, args.tasks_per_distro, dtype=np.int64), synth.SEED_BASE + 3, zipf_priority=True,
                   unmet_dep_frac=0.05, met_dep_frac=0.02, includes_dependencies=True, n_hosts=2 * args.distros)
    eng_a, eng_b = scheduler.Engine(0), scheduler.Engine(0)
    eng_a.upload(w.tasks, w.distros, w.hosts)
    eng_b.upload(w.tasks, w.distros, w.hosts)
    eng_a.run(w.now)
    po, _ = eng_a.download(want_alloc=False)
    order = po.order.copy()
    free, total = torch.cuda.mem_get_info()
    mem_before = total - free
    mem_after_first_edit = None
    ms = {"a_upload": [], "b_edit": []}
    h2d = {"a_upload": [], "b_edit": []}
    for k in range(args.warmup + args.steps):
        e = synth.next_tick(w, 1000 + k, dispatch=args.frac, arrive=args.frac, change=args.frac, order=order)
        nw = e.workload
        res = {}

        def arm_a():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng_a.upload(nw.tasks, nw.distros, nw.hosts)
            eng_a.run(nw.now)
            off, items = eng_a.download_queue(0, nw.distros.task_off)
            res["a_upload"] = (time.perf_counter() - t0, off.copy(), items.copy())

        def arm_b():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng_b.edit_tasks(e.edit, nw.distros, nw.hosts)
            if e.rows.shape[0]:
                eng_b.update_tasks(e.rows, e.values)
            eng_b.run(nw.now)
            off, items = eng_b.download_queue(0, nw.distros.task_off)
            res["b_edit"] = (time.perf_counter() - t0, off.copy(), items.copy())

        for f in ((arm_a, arm_b) if k % 2 == 0 else (arm_b, arm_a)):
            f()
        if mem_after_first_edit is None:
            free, total = torch.cuda.mem_get_info()
            mem_after_first_edit = total - free
        assert np.array_equal(res["a_upload"][1], res["b_edit"][1]) and np.array_equal(res["a_upload"][2], res["b_edit"][2]), f"step {k}"
        if k >= args.warmup:
            for arm in ms:
                ms[arm].append(res[arm][0] * 1e3)
            h2d["a_upload"].append(nw.tasks.nbytes() + nw.distros.nbytes() + nw.hosts.nbytes())
            h2d["b_edit"].append(e.edit.nbytes() + nw.distros.nbytes() + nw.hosts.nbytes() + 48 * int(e.rows.shape[0]))
        eng_b.run(nw.now)
        po, _ = eng_b.download(want_alloc=False)
        order = po.order.copy()
        w = nw
    out ={"gpu": gpu_info(), "distros": args.distros, "tasks": w.n_tasks, "steps": args.steps, "frac": args.frac,
           "ms_per_step": {a: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for a, v in ms.items()},
           "h2d_bytes_per_step": {a: int(np.mean(v)) for a, v in h2d.items()},
           "device_mem_in_use_bytes": {"two contexts after upload": int(mem_before), "after the first edit (shadow set allocated)": int(mem_after_first_edit)},
           "download_queue_equal_every_step": True}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    eng_a.close()
    eng_b.close()


if __name__ == "__main__":
    main()
