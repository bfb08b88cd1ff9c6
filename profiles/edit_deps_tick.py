"""Tick-to-tick cost of keeping DependenciesMet right on an edited tick: (a) the host evaluates the composed dependency
table (soa.apply_deps_edit + soa.deps_verdicts, a vectorised restatement of Task.DependenciesMet) and sends the changed
bits and stamped wait bases with evg_edit_tasks + evg_update_tasks -- what ResidentTick does today -- vs (b) one
evg_edit_tasks_with_deps, which composes and evaluates the table on the device.  DESIGN.md §8.6's workload: synth.next_tick
on 200 distros x 100 000 tasks (configs[2] mix: Zipf priorities, 5 % unmet + 2 % met in-queue dependencies), 5 % of the
rows dispatched / inserted / changed per step, plus one external dependency per 20 tasks.  The arms alternate per
step in one process; after each step both run, and their download_queue rows must be equal.  Reports per-step median
and range of the device-side call time (host clock around synchronised calls) and of the host time spent on verdicts,
the H2D bytes per step, and the card's name and power limit.

    python profiles/edit_deps_tick.py --distros 200 --tasks-per-distro 100000 --steps 10 --warmup 2
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


def initial_deps(w, rng, n_ext):
    """The workload's in-queue edges as EVG_DEP_IN_QUEUE entries (global rows), one external entry per 20 tasks."""
    from evergreen_b200 import _lib as L, soa as S
    t, toff = w.tasks, w.distros.task_off
    T = t.n_tasks
    distro_of = np.repeat(np.arange(w.distros.n_distros), np.diff(toff))
    own = np.repeat(np.arange(T), np.diff(t.dep_off))
    ext = np.nonzero(rng.random(T) < 0.05)[0]
    owner = np.concatenate([own, ext])
    kind = np.concatenate([np.zeros(own.shape[0], np.uint8), np.ones(ext.shape[0], np.uint8)])
    ref = np.concatenate([toff[distro_of[own]] + t.dep_idx, rng.integers(0, n_ext, ext.shape[0])]).astype(np.int32)
    o = np.argsort(owner, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=T))]).astype(np.int64)
    E = owner.shape[0]
    return S.DepsTable(off, kind[o], ref[o], rng.integers(0, 3, E).astype(np.uint8), np.full(T, 2, np.uint8),
                       np.zeros(T, np.uint8), rng.integers(0, 3, n_ext).astype(np.uint8)), np.full(E, L.EVG_TIME_ZERO, np.int64)


def deps_edit(e, w, n_ext, rng, now):
    """The DepsEdit of step e: every departure becomes a new external id (finished now), the arrivals' in-queue edges
    and the survivors' added edges are entries, 1 % of the external ids change state."""
    from evergreen_b200 import soa as S
    toff_new = e.workload.distros.task_off
    R = e.edit.remove_rows.shape[0]
    ext_state = rng.integers(0, 3, n_ext + R).astype(np.uint8)
    ins, io = e.edit.insert, e.edit.insert_off
    ins_d = np.repeat(np.arange(io.shape[0] - 1), np.diff(io))
    own = np.repeat(np.arange(ins.n_tasks), np.diff(ins.dep_off))
    insert = S.DepsTable(ins.dep_off.copy(), np.zeros(own.shape[0], np.uint8), (toff_new[ins_d[own]] + ins.dep_idx).astype(np.int32),
                         np.zeros(own.shape[0], np.uint8), np.full(ins.n_tasks, 2, np.uint8), np.zeros(ins.n_tasks, np.uint8),
                         np.zeros(0, np.uint8))
    at = e.edit.add_edge_task
    add_d = np.searchsorted(toff_new, at, side="right") - 1
    z = np.zeros(at.shape[0], np.uint8)
    return S.DepsEdit(np.arange(n_ext, n_ext + R, dtype=np.int32), ext_state, insert, at.copy(), z,
                      (toff_new[add_d] + e.edit.add_edge_dep).astype(np.int32), z, np.zeros(0, np.int64), np.zeros(0, np.uint8),
                      np.zeros(0, np.uint8), depart_finished=np.full(R, now, np.int64)).normalize(), n_ext + R


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--distros", type=int, default=200)
    ap.add_argument("--tasks-per-distro", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frac", type=float, default=0.05)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from evergreen_b200 import _lib as L, scheduler, soa as S, synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures on the GPU only")
    rng = np.random.default_rng(11)
    w = synth.make(np.full(args.distros, args.tasks_per_distro, dtype=np.int64), synth.SEED_BASE + 3, zipf_priority=True,
                   unmet_dep_frac=0.05, met_dep_frac=0.02, includes_dependencies=True)
    n_ext = 1000
    deps, fin = initial_deps(w, rng, n_ext)
    eng_a, eng_b = scheduler.Engine(0), scheduler.Engine(0)
    now = int(w.now)
    for eng in (eng_a, eng_b):
        eng.upload_with_deps(w.tasks, w.distros, None, deps, fin, now)
    _, stamp = eng_b.download_deps()
    stamp = stamp.copy()
    # the host mirror of arm (a)'s resident columns (the device's verdict bit and stamped wait basis applied)
    met0, _ = S.deps_verdicts(deps, fin, now)
    mirror = w.tasks
    mirror.flags = (mirror.flags & ~np.uint32(L.EVG_TF_DEPS_MET)) | np.where(met0 == 1, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
    mirror.wait_basis_ns = np.where((stamp != L.EVG_TIME_ZERO) & (stamp > mirror.wait_basis_ns), stamp, mirror.wait_basis_ns)
    eng_b.run(now)
    po, _ = eng_b.download(want_alloc=False)
    order = po.order.copy()
    keys = ("a_host_verdicts", "b_device_deps")
    call_ms, verdict_ms, h2d = {k: [] for k in keys}, {k: [] for k in keys}, {k: [] for k in keys}
    for k in range(args.warmup + args.steps):
        now += 60 * 10 ** 9
        e = synth.next_tick(w, 1000 + k, dispatch=args.frac, arrive=args.frac, change=args.frac, order=order)
        nw = e.workload
        dx, n_ext2 = deps_edit(e, w, n_ext, rng, now)
        res = {}

        def arm_a():
            t0 = time.perf_counter()
            new_deps, new_fin = S.apply_deps_edit(deps, w.distros.task_off, e.edit, dx, fin, stamp)
            met, st = S.deps_verdicts(new_deps, new_fin, now)
            t1 = time.perf_counter()
            composed, _ = S.apply_edit(mirror, w.distros, e.edit)
            for name, _ in S.TaskSoA.COLUMNS:
                getattr(composed, name)[e.rows] = getattr(e.values, name)
            want_flags = (composed.flags & ~np.uint32(L.EVG_TF_DEPS_MET)) | np.where(met == 1, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
            want_wb = np.where((st != L.EVG_TIME_ZERO) & (st > composed.wait_basis_ns), st, composed.wait_basis_ns)
            before, _ = S.apply_edit(mirror, w.distros, e.edit)
            changed = np.zeros(composed.n_tasks, bool)
            changed[e.rows] = True
            changed |= (want_flags != before.flags) | (want_wb != before.wait_basis_ns)
            composed.flags, composed.wait_basis_ns = want_flags, want_wb
            rows = np.nonzero(changed)[0].astype(np.int64)
            values = S.TaskSoA(**{name: getattr(composed, name)[rows] for name, _ in S.TaskSoA.COLUMNS}).normalize()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            eng_a.edit_tasks(e.edit, nw.distros)
            if rows.shape[0]:
                eng_a.update_tasks(rows, values)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            res["a_host_verdicts"] = ((t3 - t2) * 1e3, (t1 - t0) * 1e3, e.edit.nbytes() + nw.distros.nbytes() + 48 * int(rows.shape[0]),
                                      (new_deps, new_fin, st, composed))

        def arm_b():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng_b.edit_tasks_with_deps(e.edit, nw.distros, e.rows, e.values, dx, now)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            res["b_device_deps"] = ((t1 - t0) * 1e3, 0.0, e.edit.nbytes() + nw.distros.nbytes() + 48 * int(e.rows.shape[0]) + dx.nbytes(), None)

        for f in ((arm_a, arm_b) if k % 2 == 0 else (arm_b, arm_a)):
            f()
        _, st_b = eng_b.download_deps()
        new_deps, new_fin, st_a, composed = res["a_host_verdicts"][3]
        assert np.array_equal(st_a, st_b), f"step {k}: stamps"
        q = []
        for eng in (eng_a, eng_b):
            eng.run(now)
            off, items = eng.download_queue(0, nw.distros.task_off)
            q.append((off.copy(), items.copy()))
        assert np.array_equal(q[0][0], q[1][0]) and np.array_equal(q[0][1], q[1][1]), f"step {k}: download_queue"
        if k >= args.warmup:
            for a in keys:
                call_ms[a].append(res[a][0])
                verdict_ms[a].append(res[a][1])
                h2d[a].append(res[a][2])
        po, _ = eng_b.download(want_alloc=False)
        order = po.order.copy()
        deps, fin, stamp, mirror, n_ext, w = new_deps, new_fin, st_b.copy(), composed, n_ext2, nw
    rng_of = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}  # noqa: E731
    out = {"gpu": gpu_info(), "distros": args.distros, "tasks": w.n_tasks, "steps": args.steps, "frac": args.frac,
           "device_call_ms_per_step": {a: rng_of(v) for a, v in call_ms.items()},
           "host_verdict_ms_per_step": {a: rng_of(v) for a, v in verdict_ms.items()},
           "h2d_bytes_per_step": {a: int(np.mean(v)) for a, v in h2d.items()},
           "outputs_equal_every_step": True}
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
