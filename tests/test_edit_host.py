"""evg_edit_tasks without a GPU: the composed table soa.apply_edit defines, ResidentTick's diff of two Go-level batches,
and the evg_task_edit layout the ctypes mirror assumes."""
import copy
import ctypes
import os
import random
import subprocess

import numpy as np

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth

NOW = synth.NOW_NS
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cols(**kw):
    n = len(next(iter(kw.values())))
    base = {name: np.zeros(n, dtype=dt) for name, dt in S.TaskSoA.COLUMNS}
    base.update({k: np.array(v) for k, v in kw.items() if k not in ("dep_off", "dep_idx")})
    arr = lambda k: None if k not in kw else np.array(kw[k])  # noqa: E731
    return S.TaskSoA(**base, dep_off=arr("dep_off"), dep_idx=arr("dep_idx")).normalize()


def edges(t):
    return [t.dep_idx[t.dep_off[i]:t.dep_off[i + 1]].tolist() if t.n_edges else [] for i in range(t.n_tasks)]


def test_apply_edit_by_hand():
    # distro 0: rows 0..3, groups g0 (row 0) and g1 (row 2), versions 0/1; distro 1: rows 4..6, no groups
    tasks = cols(priority=[10, 11, 12, 13, 20, 21, 22], group_id=[0, -1, 1, -1, -1, -1, -1], version_id=[0, 1, 1, 0, 0, 0, 0],
                 dep_off=[0, 0, 2, 2, 3, 3, 4, 4], dep_idx=[0, 2, 1, 0])
    cfg = np.zeros(2, dtype=L.DISTRO_CFG_DTYPE)
    cfg["n_versions"] = [2, 1]
    distros = S.DistroTable(np.array([0, 4, 7]), np.array([0, 2, 2]), cfg, np.array([1, 2], dtype=np.int32)).normalize()
    ins = cols(priority=[30, 40], group_id=[1, -1], version_id=[2, 0], dep_off=[0, 1, 1], dep_idx=[0])
    new_cfg = cfg.copy()
    new_cfg["n_versions"] = [3, 1]
    edit = S.TaskEdit(remove_rows=[2, 4], insert=ins, insert_off=[0, 1, 2], add_edge_task=[2, 2], add_edge_dep=[3, 0],
                      group_remap=[0, -1], version_remap=[1, 0, 0], group_off=np.array([0, 2, 2]),
                      group_max_hosts=np.array([1, 3], dtype=np.int32), cfg=new_cfg)
    t, d = S.apply_edit(tasks, distros, edit)
    assert d.task_off.tolist() == [0, 4, 7] and d.group_off.tolist() == [0, 2, 2]
    assert d.cfg["n_versions"].tolist() == [3, 1] and d.group_max_hosts.tolist() == [1, 3]
    assert t.priority.tolist() == [10, 11, 13, 30, 21, 22, 40]  # survivors in order, then the inserted row
    assert t.group_id.tolist() == [0, -1, -1, 1, -1, -1, -1]
    assert t.version_id.tolist() == [1, 0, 1, 2, 0, 0, 0]      # survivors' versions remapped, inserted rows' kept
    # row 1 lost its edge to the removed row 2; row 3 (now 2) keeps its edge to row 1, then gains two;
    # row 5 (now 4) depended on the removed row 4; the inserted row of distro 0 brings its own edge
    assert edges(t) == [[], [0], [1, 3, 0], [0], [], [], []]


def test_apply_edit_rejects_a_survivor_in_a_dropped_group():
    tasks = cols(priority=[1, 2], group_id=[0, 0])
    cfg = np.zeros(1, dtype=L.DISTRO_CFG_DTYPE)
    cfg["n_versions"] = 1
    distros = S.DistroTable(np.array([0, 2]), np.array([0, 1]), cfg, np.array([1], dtype=np.int32)).normalize()
    edit = S.TaskEdit([0], None, [0, 0], [], [], group_remap=[-1])
    try:
        S.apply_edit(tasks, distros, edit)
    except ValueError:
        return
    raise AssertionError("a survivor in a group mapped to -1 must be rejected")


def go_batch(rng, n_distros=3, n_tasks=40, prefix="t"):
    batch = []
    for k in range(n_distros):
        d = M.Distro(id=f"d{k}", dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
        d.planner_settings.group_versions = k == 2
        tasks = [go_task(rng, f"{prefix}{k}-{i}", d.id) for i in range(n_tasks)]
        link(rng, tasks)
        batch.append((d, tasks))
    return batch


def go_task(rng, tid, distro_id):
    t = M.Task(id=tid, version=f"v{rng.randrange(4)}", project="p", build_variant="bv", distro_id=distro_id,
               priority=rng.choice([0, 0, 5, 50]), requester=rng.choice(["gitter_request", "patch_request"]),
               num_dependents=rng.randrange(3), activated_time=NOW - rng.randrange(10 ** 13),
               scheduled_time=NOW - rng.randrange(10 ** 12), expected_duration=rng.randrange(1, 3600) * 10 ** 9)
    if rng.random() < 0.3:
        t.task_group, t.task_group_order, t.task_group_max_hosts = f"tg{rng.randrange(3)}", rng.randrange(1, 5), 2
    return t


def link(rng, tasks):
    for t in tasks:
        if rng.random() < 0.2:
            dep = rng.choice(tasks)
            if dep is not t:
                t.depends_on.append(M.Dependency(dep.id, status="success"))


def evolve(rng, batch, tick):
    """Next Go-level batch: dispatch, arrivals (a new task group among them), a dependency finishing, priority changes."""
    out = []
    for d, tasks in batch:
        # dispatched tasks leave; a task others depend on leaving is a dependency finishing
        kept = [copy.copy(t) for t in tasks if rng.random() >= 0.15]
        for t in kept:
            t.depends_on = list(t.depends_on)
            if rng.random() < 0.1:
                t.priority += 7
        arrivals = [go_task(rng, f"n{tick}-{d.id}-{i}", d.id) for i in range(6)]
        for i, t in enumerate(arrivals[:3]):
            t.task_group, t.task_group_order, t.task_group_max_hosts = f"new{tick}", i + 1, 1
        pool = kept + arrivals
        for t in arrivals:
            if rng.random() < 0.5:
                t.depends_on.append(M.Dependency(rng.choice(pool).id, status="success"))
            t.depends_on = [dep for dep in t.depends_on if dep.task_id != t.id]
        if kept and rng.random() < 0.7:
            kept[0].depends_on.append(M.Dependency(arrivals[-1].id, status="success"))
        rng.shuffle(kept)
        out.append((d, kept + arrivals))
    return out


def test_resident_tick_diff_composes_the_marshalled_batch():
    rng = random.Random(7)
    batch = go_batch(rng)
    rt = scheduler.ResidentTick()
    canon = rt.canonical(batch)
    soa, table, keys = S.marshal_tasks(canon, NOW, resolve_deps=True)
    rt.remember(canon, soa, table, keys)
    n_edits = 0
    for tick in range(4):
        batch = evolve(rng, batch, tick)
        canon = rt.canonical(batch)
        prev_ids = {i for ids in rt.ids for i in ids}
        # canonical order: survivors in their previous order, then arrivals in batch order
        for (d, ts), prev in zip(canon, rt.ids):
            surv = [t.id for t in ts if t.id in prev_ids]
            assert surv == [i for i in prev if i in set(surv)]
            assert all(t.id in prev_ids for t in ts[:len(surv)])
        new, new_table, new_keys = S.marshal_tasks(canon, NOW, resolve_deps=True)
        change = rt.diff(canon, new, new_table, new_keys)
        if change is not None:
            n_edits += 1
            edit, rows, values = change
            got, got_table = S.apply_edit(rt.soa, rt.table, edit)
            for name, _ in S.TaskSoA.COLUMNS:
                getattr(got, name)[rows] = getattr(values, name)
            for name, _ in S.TaskSoA.COLUMNS:
                assert np.array_equal(getattr(got, name), getattr(new, name)), name
            for f in ("task_off", "group_off", "group_max_hosts"):
                assert np.array_equal(getattr(got_table, f), getattr(new_table, f)), f
            assert np.array_equal(got_table.cfg, new_table.cfg)
            # the same edges per task; their order inside a task may differ (the GPU test shows it is not observable)
            assert [sorted(e) for e in edges(got)] == [sorted(e) for e in edges(new)]
        rt.remember(canon, new, new_table, new_keys)
    assert n_edits >= 1


def test_resident_tick_uploads_when_a_survivor_loses_a_queued_dependency():
    rng = random.Random(3)
    d = M.Distro(id="d")
    a, b = go_task(rng, "a", "d"), go_task(rng, "b", "d")
    for t in (a, b):
        t.task_group = ""
    b.depends_on = [M.Dependency("a")]
    rt = scheduler.ResidentTick()
    canon = rt.canonical([(d, [a, b])])
    rt.remember(canon, *S.marshal_tasks(canon, NOW, resolve_deps=True))
    b2 = copy.copy(b)
    b2.depends_on = []
    canon = rt.canonical([(d, [a, b2])])
    assert rt.diff(canon, *S.marshal_tasks(canon, NOW, resolve_deps=True)) is None


def test_next_tick_composes_a_valid_tick():
    w = synth.make(np.array([1, 40, 700, 0, 3000]), 11, zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02,
                   group_versions_frac=0.3, n_hosts=30)
    for remap in (True, False):
        x = w
        for k in range(3):
            e = synth.next_tick(x, k, remap=remap)
            t, d = e.workload.tasks, e.workload.distros
            dof = np.repeat(np.arange(d.n_distros), np.diff(d.task_off))
            assert np.all((t.group_id >= -1) & (t.group_id < np.diff(d.group_off)[dof]))
            assert np.all((t.version_id >= 0) & (t.version_id < d.cfg["n_versions"][dof]))
            own = np.repeat(np.arange(t.n_tasks), np.diff(t.dep_off))
            assert np.all(t.dep_idx < np.diff(d.task_off)[dof[own]]) and np.all(t.dep_idx != own - d.task_off[dof[own]])
            if remap:  # dense ids: every group slot has a member
                assert np.unique(d.group_off[dof[t.group_id >= 0]] + t.group_id[t.group_id >= 0]).shape[0] == d.n_groups
            assert e.edit.remove_rows.shape[0] > 0 and e.edit.insert.n_tasks > 0 and e.rows.shape[0] > 0
            x = e.workload


def test_task_edit_struct_layout(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(evg_task_edit), offsetof(evg_task_edit, n_remove),
         offsetof(evg_task_edit, remove_rows), offsetof(evg_task_edit, insert), offsetof(evg_task_edit, insert_off),
         offsetof(evg_task_edit, n_add_edges), offsetof(evg_task_edit, add_edge_task), offsetof(evg_task_edit, add_edge_dep),
         offsetof(evg_task_edit, group_remap), offsetof(evg_task_edit, version_remap));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    E = L.TaskEditStruct
    assert got == [ctypes.sizeof(E), E.n_remove.offset, E.remove_rows.offset, E.insert.offset, E.insert_off.offset,
                   E.n_add_edges.offset, E.add_edge_task.offset, E.add_edge_dep.offset, E.group_remap.offset,
                   E.version_remap.offset]
