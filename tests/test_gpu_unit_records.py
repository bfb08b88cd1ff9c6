"""The general path's unit records: k_galloc numbers every multi-member unit of the tick, k_gfill hands the number to its
memberships, and every later kernel finds the unit by that number.  Ticks that put the hand-off at its edges, against
the oracle: units of 2, 8 / 9 (the one-thread ranking limit), 64 / 65 (the emitted-rank mask and the counting fallback)
and several hundred members, duplicate edges into one unit, GroupVersions tasks that are both an own-key and a version
member, a unit count exactly at the record capacity the host reserves, the pipelined one-shot call with several chunks
and a resident tick after evg_edit_tasks."""
import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import synth

pytestmark = pytest.mark.gpu

RANK_ONE = 8  # units up to this many members are ranked by the thread that folds them


def set_edges(w, lists):
    """Dependency edges from {global task: [distro-local targets]}; every other task has none."""
    T = w.n_tasks
    n = np.zeros(T, dtype=np.int64)
    for t, ds in lists.items():
        n[t] = len(ds)
    off = np.zeros(T + 1, dtype=np.int64)
    np.cumsum(n, out=off[1:])
    idx = np.zeros(int(off[-1]), dtype=np.int32)
    for t, ds in lists.items():
        idx[off[t]:off[t + 1]] = ds
    w.tasks.dep_off, w.tasks.dep_idx = off, idx


def resize_group(t, a, b, g, size, pool):
    """Task group g of the distro [a, b) gets exactly `size` members: extra members leave it, tasks from `pool`
    (ungrouped, distro-local) join it in its first member's version."""
    gid = t.group_id[a:b]
    m = np.nonzero(gid == g)[0]
    if m.shape[0] > size:
        gid[m[size:]] = -1
    else:
        add = [pool.pop() for _ in range(size - m.shape[0])]
        gid[add] = g
        t.version_id[a:b][add] = t.version_id[a + m[0]]
    assert int((gid == g).sum()) == size


def finish(w):
    w.tasks.normalize()
    w.distros.normalize()
    return w


def check(engine, w, breakdown=True):
    po, ao = engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now, breakdown=breakdown)
    ref = parity.check_against_oracle(w, po, ao)
    if breakdown:
        assert np.array_equal(po.breakdown, ref["breakdown"])
    parity.check_properties(w, po, ao)
    return po, ao


def unit_sizes_tick():
    """Distro 0 (general path): task groups and dependency fan-ins of 2, 8, 9, 64, 65 and 300 / 401 members, and
    duplicate edges into one unit.  Distro 1: GroupVersions, grouped tasks with a version membership too."""
    sizes = np.array([20000, 14000])
    w = synth.make(sizes, 91, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    t, dt = w.tasks, w.distros
    a0, b0, b1 = (int(x) for x in dt.task_off)
    assert int(dt.group_off[1] - dt.group_off[0]) >= 6
    pool = list(np.nonzero(t.group_id[a0:b0] < 0)[0][::-1])
    for g, s in enumerate((2, RANK_ONE, RANK_ONE + 1, 64, 65, 300)):
        resize_group(t, a0, b0, g, s, pool)
    lists = {}
    free = [x for x in pool if t.group_id[a0 + x] < 0]
    # fan-ins: a target and its distinct dependents form a unit of 1 + dependents members
    for members in (2, RANK_ONE, RANK_ONE + 1, 64, 65, 401):
        target = free.pop()
        for _ in range(members - 1):
            lists[a0 + free.pop()] = [target]
    # duplicate edges: the same target twice, two members of one task group, and a member of a task group into its own
    target = free.pop()
    lists[a0 + free.pop()] = [target, target]
    g3 = np.nonzero(t.group_id[a0:b0] == 3)[0]
    lists[a0 + free.pop()] = [int(g3[0]), int(g3[1]), target]
    lists[a0 + int(g3[2])] = [int(g3[4])]
    # distro 1: GroupVersions, 20 versions of 700 tasks (a task group stays in its first member's version), a few edges
    dt.cfg["group_versions"][1] = 1
    dt.cfg["n_versions"][1] = 20
    ver = (np.arange(b1 - b0) // 700).astype(np.int32)
    gid = t.group_id[b0:b1]
    for g in np.unique(gid[gid >= 0]):
        m = np.nonzero(gid == g)[0]
        ver[m] = ver[m[0]]
    t.version_id[b0:b1] = ver
    for k in range(50):
        lists[b0 + 7 * k + 3] = [7 * k + 1, 7 * k + 2]
    set_edges(w, dict(sorted(lists.items())))
    return finish(w)


def test_unit_sizes_around_the_rank_and_mask_limits_with_breakdown(engine):
    w = unit_sizes_tick()
    gid = w.tasks.group_id[:20000]
    assert sorted(np.bincount(gid[gid >= 0])[:6].tolist()) == [2, 8, 9, 64, 65, 300]
    check(engine, w)


def test_unit_sizes_on_the_resident_tick(engine):
    w = unit_sizes_tick()
    engine.upload(w.tasks, w.distros, w.hosts)
    for opts in (L.EVG_OPT_BREAKDOWN, 0, L.EVG_OPT_BREAKDOWN):  # records rebuilt tick after tick, with and without breakdown
        engine.run(w.now, opts)
        po, ao = engine.download(want_breakdown=bool(opts))
        ref = parity.check_against_oracle(w, po, ao)
        if opts:
            assert np.array_equal(po.breakdown, ref["breakdown"])


def units_at_capacity_tick():
    """Every unit the record capacity allows: distro 0 is a dependency ring (every task is a target, so every task's
    own-key unit has two members); distro 1 is GroupVersions with one task group per task and two tasks per version
    (a unit per group and per version)."""
    n0, n1 = 13000, 14000
    w = synth.make(np.array([n0, n1]), 92, zipf_priority=True, tg_frac=0.0, n_hosts=10)
    t, dt = w.tasks, w.distros
    t.group_id[:] = -1
    t.group_id[n0:] = np.arange(n1, dtype=np.int32)
    t.version_id[:n0] = 0
    t.version_id[n0:] = (np.arange(n1) // 2).astype(np.int32)
    dt.group_off = np.array([0, 0, n1], dtype=np.int64)
    dt.group_max_hosts = np.full(n1, 3, dtype=np.int32)
    dt.cfg["group_versions"][:] = [0, 1]
    dt.cfg["n_versions"][:] = [1, n1 // 2]
    set_edges(w, {k: [(k + 1) % n0] for k in range(n0)})
    return finish(w), n0 + n1 + n1 // 2


def test_unit_count_at_the_record_capacity(engine):
    w, bound = units_at_capacity_tick()
    # distinct units: the ring's n0 own-key units, n1 group units and n1 / 2 version units
    assert bound == 13000 + 14000 + 7000
    check(engine, w)


def test_pipelined_call_with_several_chunks(engine):
    """The one-shot call cuts a tick of 2^21 tasks or more into chunks of whole distros and numbers each chunk's units
    afresh; the later chunks' general-path tiles start past tile 0."""
    sizes = np.array([360_000] * 6)
    w = synth.make(sizes, 93, zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02, tg_frac=0.1,
                   group_versions_frac=0.5, includes_dependencies=True, n_hosts=60)
    assert w.n_tasks >= 2 * (1 << 20)
    check(engine, finish(w), breakdown=False)


def test_resident_tick_after_an_edit(engine):
    w = unit_sizes_tick()
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now, 0)
    po, _ = engine.download()
    e = synth.next_tick(w, 94, order=po.order, dep_frac=0.2, add_edge_frac=0.02)
    w2 = e.workload
    engine.edit_tasks(e.edit, w2.distros, w2.hosts)
    if e.rows.shape[0]:
        engine.update_tasks(e.rows, e.values)
    engine.run(w2.now, L.EVG_OPT_BREAKDOWN)
    po, ao = engine.download(want_breakdown=True)
    ref = parity.check_against_oracle(w2, po, ao)
    assert np.array_equal(po.breakdown, ref["breakdown"])
