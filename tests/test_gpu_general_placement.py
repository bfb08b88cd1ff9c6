"""The general path's placement writes every slot of a distro's pre-arrangement exactly once, and nothing else: a tile
writes the slots of the tasks emitted from their own single-task unit, a multi-member unit the run of its anchor, and no
writer fills the other's slots with a placeholder.  A slot nobody writes keeps what an earlier tick left in the buffer,
so two different general-path ticks run back to back on one resident context, and each is checked against the oracle.
The second tick holds:
  * a distro whose first tile's stretch exceeds the 3072 slots k_gplace stages in shared memory (written from registers);
  * a unit above kRankOne (8) members anchored in a distro's first tile, and one anchored in its last tile (a warp per
    unit).
A third tick puts a distro's last task at both edges of the tile's anchor test (the slots past the distro read as 0):
  * the last task, alone in its distro's last tile, anchors a small unit;
  * the last task is emitted from a small unit it does not anchor, in a last tile whose stretch exceeds the stage, with
    a general-path distro after it.
Every case is asserted on the oracle's queue."""
import numpy as np
import pytest

import parity
from evergreen_b200 import synth
from test_gpu_unit_emit import emitted_value, set_edges

pytestmark = pytest.mark.gpu

SIZES = np.array([30000, 20000])
K_STAGE, K_RANK_ONE, TILE = 3072, 8, 2048


def ungrouped(w, d):
    a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
    return np.nonzero(w.tasks.group_id[a:b] < 0)[0]


def last_tile_start(w, d):
    """Distro-local index of the first task of d's last tile (tiles start at (base & ~3) + k * 2048)."""
    a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
    a0 = a & ~3
    return a0 + (b - 1 - a0) // TILE * TILE - a


def placement_tick():
    """Returns the tick and its fan-ins: (distro, target, dependents), distro-local."""
    w = synth.make(SIZES, 131, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    free0, free1 = ungrouped(w, 0), ungrouped(w, 1)
    n1 = int(SIZES[1])
    # distro 0: every fifth ungrouped task from index 100 on depends on the first ungrouped task
    t0 = int(free0[0])
    fan0 = free0[free0 >= 100][::5]
    # distro 1: 20 dependents on an ungrouped task of its first tile, 40 on one of its last tile
    t1 = int(free1[1])
    t2 = int(free1[free1 >= last_tile_start(w, 1)][-1])
    mid = free1[(free1 > 4000) & (free1 < n1 - 4000)]
    fan1, fan2 = mid[:20], mid[20:60]
    a1 = int(w.distros.task_off[1])
    lists = {int(x): [t0] for x in fan0}
    lists.update({a1 + int(x): [t1] for x in fan1})
    lists.update({a1 + int(x): [t2] for x in fan2})
    set_edges(w, dict(sorted(lists.items())))
    w.tasks.normalize()
    w.distros.normalize()
    return w, [(0, t0, fan0), (1, t1, fan1), (1, t2, fan2)]


def run(engine, w):
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now, 0)
    po, ao = engine.download()
    ref = parity.check_against_oracle(w, po, ao)
    parity.check_properties(w, po, ao)
    return ref


def test_second_tick_writes_every_slot(engine):
    other = synth.make(SIZES, 37, zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02, tg_frac=0.2, n_hosts=20)
    w, fans = placement_tick()
    run(engine, other)
    ref = run(engine, w)
    run(engine, other)  # and back: the crafted tick's runs are stale under this one
    assert last_tile_start(w, 1) <= fans[2][1] and fans[1][1] < TILE
    for d, target, deps in fans:
        val, _ = emitted_value(ref, d)
        emitted = int(np.count_nonzero(val == val[target]))  # the unit's tasks share its TotalValue
        assert emitted > K_RANK_ONE, (d, target, emitted)
        assert np.all(val[deps] == val[target]), (d, target)
    # the target's unit alone fills more than the stage of distro 0's first tile
    assert np.count_nonzero(emitted_value(ref, 0)[0] == emitted_value(ref, 0)[0][fans[0][1]]) > K_STAGE


END_SIZES = np.array([14337, 30000, 20000])  # the first distro's last tile holds one task; all three are general-path


def distro_end_tick():
    """The distro's last task at both edges of the anchor test.  Distro 0: its last task, alone in its last tile, anchors
    a unit of 5 members.  Distro 1: its last task is a dependent emitted from a 5-member unit anchored in the last tile
    (it anchors nothing), whose stretch a dependency target of 3500 dependents pushes past the stage; distro 2 follows
    it on the general path.  Returns the tick and the cases: (distro, target, dependents), distro-local."""
    w = synth.make(END_SIZES, 1, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    t = w.tasks
    cases, lists = [], {}
    for d, (n_small, n_big) in enumerate(((4, 0), (4, 3500))):
        a, n = int(w.distros.task_off[d]), int(END_SIZES[d])
        last = n - 1
        assert t.group_id[a + last] < 0
        free = ungrouped(w, d)
        mid = free[(free > 100) & (free < last_tile_start(w, d) - 100)]
        if d == 0:
            target, deps = last, mid[:n_small]
        else:
            tail = free[(free >= last_tile_start(w, d)) & (free < last)]
            target, big = int(tail[0]), int(tail[1])
            deps = np.append(mid[:n_small - 1], last)
            cases.append((d, big, mid[n_small:n_small + n_big]))
            lists.update({a + int(x): [big] for x in mid[n_small:n_small + n_big]})
        cases.append((d, int(target), deps))
        lists.update({a + int(x): [int(target)] for x in deps})
    set_edges(w, dict(sorted(lists.items())))
    w.tasks.normalize()
    w.distros.normalize()
    return w, cases


def test_distro_last_task_at_the_anchor_test(engine):
    other = synth.make(END_SIZES, 41, zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02, tg_frac=0.2, n_hosts=20)
    w, cases = distro_end_tick()
    assert last_tile_start(w, 0) == END_SIZES[0] - 1
    run(engine, other)
    ref = run(engine, w)
    run(engine, other)
    for d, target, deps in cases:
        val, _ = emitted_value(ref, d)
        emitted = int(np.count_nonzero(val == val[target]))
        assert np.all(val[deps] == val[target]), (d, target)
        assert emitted == deps.shape[0] + 1 and (emitted <= K_RANK_ONE) == (deps.shape[0] < K_RANK_ONE), (d, target, emitted)
    # distro 1's last tile: its own tasks and the 3501 of the big unit exceed the stage
    assert END_SIZES[1] - last_tile_start(w, 1) + cases[1][2].shape[0] + 1 > K_STAGE
