"""General-path distros whose multi-member units are large, against the oracle with the breakdown on: a fan-in of
10 000 dependents on one task, GroupVersions version units of 1300 members and a task group past 64 members.  These
cross the unit table's one-thread ranking limit, the 64-rank emitted-rank masks and the counting fallback of the
displaced-task placement, which the smaller general-path ticks never reach."""
import numpy as np
import pytest

import parity
from evergreen_b200 import synth

pytestmark = pytest.mark.gpu


def big_units_tick(fan_in=True, big_group=True):
    sizes = np.array([30000, 13000])
    w = synth.make(sizes, 77, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    t, dt = w.tasks, w.distros
    a0, b0, b1 = (int(x) for x in dt.task_off)
    # distro 0: a third of the queue depends on its task 5
    fan = np.arange(1, sizes[0], 3) if fan_in else np.zeros(0, dtype=np.int64)
    dep_off = np.zeros(w.n_tasks + 1, dtype=np.int64)
    n_dep = np.zeros(w.n_tasks, dtype=np.int64)
    n_dep[a0 + fan] = 1
    np.cumsum(n_dep, out=dep_off[1:])
    t.dep_off, t.dep_idx = dep_off, np.full(fan.shape[0], 5, dtype=np.int32)
    if big_group:
        # distro 0: 100 ungrouped tasks join its task group 0 (every other group keeps its members), with repeated
        # TaskGroupOrders so that the in-unit order needs the later keys and the input index
        rng = np.random.default_rng(5)
        grp = a0 + 200 + np.nonzero(t.group_id[a0 + 200:b0] < 0)[0][:100]
        first = a0 + int(np.nonzero(t.group_id[a0:b0] == 0)[0][0])
        t.group_id[grp] = 0
        t.version_id[grp] = t.version_id[first]  # a task group lives in one version (the oracle keys it by version too)
        t.task_group_order[grp] = rng.integers(1, 30, grp.shape[0]).astype(np.int32)
        t.num_dependents[grp] = rng.integers(0, 3, grp.shape[0]).astype(np.int32)
    # distro 1: GroupVersions with ten versions of 1300 tasks; a task group stays inside its first member's version
    cfg = dt.cfg
    cfg["group_versions"][1] = 1
    cfg["n_versions"][1] = 10
    loc = np.arange(b1 - b0)
    ver = (loc // 1300).astype(np.int32)
    gid = t.group_id[b0:b1]
    for g in np.unique(gid[gid >= 0]):
        m = np.nonzero(gid == g)[0]
        ver[m] = ver[m[0]]
    t.version_id[b0:b1] = ver
    assert np.bincount(ver).min() > 1000
    return finish(w)


def finish(w):
    w.tasks.normalize()
    w.distros.normalize()
    return w


def check(engine, w):
    po, ao = engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now, breakdown=True)
    ref = parity.check_against_oracle(w, po, ao)
    assert np.array_equal(po.breakdown, ref["breakdown"])
    parity.check_properties(w, po, ao)


def test_general_path_fan_in_and_version_units(engine):
    check(engine, big_units_tick(big_group=False))


def test_general_path_big_task_group_fan_in_and_version_units(engine):
    w = big_units_tick()
    g0 = np.nonzero(w.tasks.group_id[:30000] == 0)[0]
    assert g0.shape[0] > 64 and np.unique(w.tasks.version_id[g0]).shape[0] == 1
    check(engine, w)
