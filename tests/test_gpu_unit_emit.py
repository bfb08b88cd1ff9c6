"""The general path writes the tasks a multi-member unit emits from the unit itself: at its anchor's run start, in
rank order, skipping the members another unit emits first.  Ticks that put that walk at its edges, bit for bit against
the oracle (order, TotalValue, breakdown):
  * a unit whose anchor is not its rank-0 member (a task group whose smallest index has the largest TaskGroupOrder, a
    dependency target that ranks behind its dependents);
  * units that emit only some of their members, because the others go to a higher-valued unit they also belong to:
    dependency units over a task group, both ways round (the task group wins the shared members, or the dependency
    unit does);
  * such a partial emission in units of 6 (one thread per unit), 40, 100 (past 64) and 3000 members (a warp per unit);
  * a resident tick re-run after evg_update_tasks moves the shared members from one unit to the other and back.
Every tick asserts on the oracle's queue that the case it is named for happens."""
import numpy as np
import pytest

import parity
from evergreen_b200 import soa as S
from evergreen_b200 import synth

pytestmark = pytest.mark.gpu

HIGH = 5000  # a priority far above synth's: the unit holding such a task outranks every unit without one
SIZES = np.array([24000, 20000])  # both general-path distros; the second starts past slot 0
# (dependency-unit members, of which also in the task group): partial emissions at every placement path's size
FAN_INS = ((6, 2), (40, 5), (100, 10), (3000, 20))


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


def take_group(t, a, g, size, pool):
    """Task group g of the distro starting at a gets exactly `size` members: extra members leave it, ungrouped tasks
    from `pool` join it in its first member's version.  Returns the members (distro-local, ascending)."""
    gid = t.group_id[a:a + pool.limit]  # a view
    m = np.nonzero(gid == g)[0]
    if m.shape[0] > size:
        gid[m[size:]] = -1
        pool.give(m[size:])
    else:
        add = pool.take(size - m.shape[0])
        gid[add] = g
        t.version_id[a + add] = t.version_id[a + m[0]]
    return np.nonzero(gid == g)[0]


class Pool:
    """Ungrouped tasks of one distro that no case has used yet (distro-local indices)."""

    def __init__(self, t, a, b):
        self.limit = b - a
        self.free = list(np.nonzero(t.group_id[a:b] < 0)[0][::-1])

    def take(self, n):
        out = [int(self.free.pop()) for _ in range(n)]
        return np.array(out, dtype=np.int64)

    def give(self, xs):
        self.free.extend(int(x) for x in xs)


def build_cases(w, d, first_group):
    """Writes the cases into distro d and returns what the checks need: per case, the members of the two units and
    which one is meant to win the shared members."""
    t = w.tasks
    a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
    pool = Pool(t, a, b)
    cases, lists = [], {}
    g = first_group
    ng = int(w.distros.group_off[d + 1] - w.distros.group_off[d])
    # (a) a task group of 12 whose smallest index has the largest TaskGroupOrder: its anchor is not its rank-0 member
    grp = take_group(t, a, g, 12, pool)
    t.task_group_order[a + grp] = np.arange(12, 0, -1, dtype=np.int32)
    cases.append(dict(kind="anchor", group=grp))
    g += 1
    # (b), (c) a dependency target X, its dependents, and a task group whose members are some of the dependents
    for k, (members, shared) in enumerate(FAN_INS):
        for group_wins in (True, False):
            assert g < ng
            grp = take_group(t, a, g, shared + 6, pool)
            g += 1
            x = int(pool.take(1)[0])
            deps = np.concatenate([grp[:shared], pool.take(members - 1 - shared)])
            for q in deps:
                lists[a + int(q)] = [x]
            fan = np.concatenate([[x], deps])
            t.priority[a + fan] = 1
            t.priority[a + grp] = 1
            # TaskList.Less puts more dependents first: the target ranks behind every dependent
            t.num_dependents[a + fan] = 1
            t.num_dependents[a + x] = 0
            t.task_group_order[a + grp] = np.arange(1, grp.shape[0] + 1, dtype=np.int32)
            boost = grp[-1] if group_wins else deps[-1]  # never a shared member: each unit keeps a task of its own
            t.priority[a + boost] = HIGH
            cases.append(dict(kind="partial", group=grp, fan=fan, target=x, shared=grp[:shared], group_wins=group_wins,
                              boost=boost))
    return lists, cases


def emit_tick():
    w = synth.make(SIZES, 95, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    lists, cases = {}, []
    for d in range(SIZES.shape[0]):
        ld, cd = build_cases(w, d, 0)
        lists.update(ld)
        cases.append(cd)
    set_edges(w, dict(sorted(lists.items())))
    w.tasks.normalize()
    w.distros.normalize()
    return w, cases


def emitted_value(ref, j):
    """TotalValue each task of the j-th distro was emitted with (by distro-local index), and its rank."""
    ra, rb = int(ref["task_off"][j]), int(ref["task_off"][j + 1])
    order = np.asarray(ref["order"][ra:rb])
    val = np.empty(rb - ra, dtype=np.int64)
    val[order] = np.asarray(ref["total_value"][ra:rb])
    rank = np.empty(rb - ra, dtype=np.int64)
    rank[order] = np.arange(rb - ra)
    return val, rank


def assert_cases(ref, cases):
    """The oracle's queue shows every case: the anchor behind another member, and partial emissions."""
    for j, cd in enumerate(cases):
        val, rank = emitted_value(ref, j)
        for c in cd:
            if c["kind"] == "anchor":
                grp = c["group"]
                assert np.unique(val[grp]).shape[0] == 1
                assert rank[grp[0]] == rank[grp].max()  # the anchor (smallest index) is emitted last of the unit
                continue
            grp, fan, shared = c["group"], c["fan"], c["shared"]
            v_grp, v_fan = val[grp[-1]], val[c["target"]]
            assert v_grp != v_fan
            winner = v_grp if c["group_wins"] else v_fan
            assert np.all(val[shared] == winner)
            loser_members = fan if c["group_wins"] else grp
            loser = v_fan if c["group_wins"] else v_grp
            kept = loser_members[val[loser_members] == loser]
            # the losing unit emits some of its members, not all
            assert 2 <= kept.shape[0] < loser_members.shape[0]
            if c["group_wins"]:
                # its anchor (the target) ranks behind the dependents it still emits
                assert rank[c["target"]] == rank[kept].max()


def check(engine, w, cases, po, ao):
    ref = parity.check_against_oracle(w, po, ao)
    assert_cases(ref, cases)
    return ref


def test_partial_emission_and_anchor_behind_rank_zero(engine):
    w, cases = emit_tick()
    po, ao = engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now, breakdown=True)
    ref = check(engine, w, cases, po, ao)
    assert np.array_equal(po.breakdown, ref["breakdown"])
    parity.check_properties(w, po, ao)


def flip(w, cases):
    """Moves every case's boost from one unit to the other: the shared members change the unit that emits them.
    Returns the task slots whose priority changed."""
    rows = []
    for j, cd in enumerate(cases):
        a = int(w.distros.task_off[j])
        for c in cd:
            if c["kind"] != "partial":
                continue
            old = c["boost"]
            new = c["fan"][-1] if c["group_wins"] else c["group"][-1]
            w.tasks.priority[a + old] = 1
            w.tasks.priority[a + new] = HIGH
            c["boost"], c["group_wins"] = new, not c["group_wins"]
            rows += [a + int(old), a + int(new)]
    return np.array(sorted(rows), dtype=np.int64)


def test_resident_tick_after_update_moves_shared_members(engine):
    w, cases = emit_tick()
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now, 0)
    po, ao = engine.download()
    check(engine, w, cases, po, ao)
    for _ in range(2):  # there and back: every unit's emitted-by-rank slots of the previous run are stale
        rows = flip(w, cases)
        engine.update_tasks(rows, S.TaskSoA(**{name: getattr(w.tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
        engine.run(w.now, 0)
        po, ao = engine.download()
        check(engine, w, cases, po, ao)
