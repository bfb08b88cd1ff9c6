"""evg_plan_aliases on the device: the alias queues it builds from the tick's schedulable tasks (each given once) plan
exactly like a fresh evg_upload_with_deps of the same queues built on the host (soa.compose_aliases) -- order,
TotalValue, queue and group info, breakdown, the persisted queue -- on every route, with the oracle; each rule of
FindHostSchedulableForAlias on its own; the calls that follow; the error contract; and plan_alias_queues against
find_host_schedulable_for_alias + plan_distros(secondary=True)."""
import copy
import ctypes as C

import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_edit import SIZES, check_equal, edit

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fresh():
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def host_route(fresh, at, cfg, now):
    """The alias queues built on the host and uploaded with evg_upload_with_deps; the device's dependency verdicts and
    stamps are folded into the columns, so the returned workload re-uploads (and feeds the oracle) as it stands."""
    soa, table, deps, fin, src, gsrc = S.compose_aliases(at, cfg)
    fresh.upload_with_deps(soa, table, None, deps, fin, now)
    met, stamp = (x.copy() for x in fresh.download_deps())
    soa.flags = np.where(met & 1, soa.flags | L.EVG_TF_DEPS_MET, soa.flags & ~np.uint32(L.EVG_TF_DEPS_MET)).astype(np.uint32)
    soa.wait_basis_ns = np.where((stamp != M.ZERO_TIME) & (stamp > soa.wait_basis_ns), stamp, soa.wait_basis_ns).astype(np.int64)
    return synth.Workload("alias", now, soa, table, None), src, gsrc


def plan_and_check(engine, fresh, at, cfg, now, breakdown=False, oracle=False):
    task_off, group_off, n_versions = engine.plan_aliases(at, cfg, now)
    w, src, gsrc = host_route(fresh, at, cfg, now)
    assert np.array_equal(task_off, w.distros.task_off) and np.array_equal(group_off, w.distros.group_off)
    assert np.array_equal(n_versions, w.distros.cfg["n_versions"])
    got_src, got_gsrc = engine.download_alias_map()
    assert np.array_equal(got_src, src) and np.array_equal(got_gsrc, gsrc)
    po, _, _, _ = check_equal(engine, fresh, w, breakdown)
    if oracle:
        parity.check_against_oracle(w, po, None)
    return w


def test_every_size_class_equals_the_host_route(engine, fresh):
    w0 = synth.make(np.array(SIZES), 801, zipf_priority=True, unmet_dep_frac=0.03, met_dep_frac=0.03, tg_frac=0.15,
                    group_versions_frac=0.3, includes_dependencies=True)
    # one alias queue above 12 288 tasks (the general path) and on-chip queues from the names; then tiny queues
    sizes = []
    for k, (name_frac, big) in enumerate(((0.05, 14000), (0.001, 0))):
        at, cfg = synth.make_aliases(w0, 802 + k, name_frac=name_frac, big=big)
        w = plan_and_check(engine, fresh, at, cfg, w0.now, breakdown=k == 0, oracle=True)
        assert k > 0 or (w.tasks.n_edges > 0 and w.distros.n_groups > 0 and (w.distros.cfg["group_versions"] != 0).any())
        sizes.extend(np.diff(w.distros.task_off).tolist())
    sizes = np.array(sizes)
    assert (sizes > 12288).any() and ((sizes > 1280) & (sizes <= 12288)).any() and ((sizes > 32) & (sizes <= 384)).any()
    assert (sizes <= 32).any(), sizes


def test_follow_up_calls_equal_a_fresh_upload(engine, fresh):
    w0 = synth.make(np.array([40, 900, 6000, 300]), 803, tg_frac=0.1, met_dep_frac=0.05, group_versions_frac=0.5)
    at, cfg = synth.make_aliases(w0, 804, name_frac=0.7)
    w = plan_and_check(engine, fresh, at, cfg, w0.now)
    rows = np.array([0, w.n_tasks // 2, w.n_tasks - 1], dtype=np.int64)
    w.tasks.priority[rows] = 77
    engine.update_tasks(rows, S.TaskSoA(**{name: getattr(w.tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
    check_equal(engine, fresh, w, breakdown=True)
    for k in range(2):
        e = synth.next_tick(w, 805 + k)
        edit(engine, e)
        w = e.workload
        check_equal(engine, fresh, w, breakdown=True)
    # the rows are no longer the alias queues' rows
    assert engine.lib.evg_download_alias_map(engine.ctx, None, None) == L.EVG_ERR_STATE


def raw_plan(eng, at, cfg):
    st, keep = at.struct()
    D = int(cfg.shape[0])
    cfg = np.ascontiguousarray(cfg, dtype=L.DISTRO_CFG_DTYPE)
    bufs = [np.zeros(D + 1, np.int64), np.zeros(D + 1, np.int64), np.zeros(D + 1, np.int32)]
    out = L.AliasOutStruct(*[L.ptr(b) for b in bufs])
    rc = eng.lib.evg_plan_aliases(eng.ctx, C.byref(st), L.ptr(cfg) if D else None, D, synth.NOW_NS, C.byref(out))
    del keep
    return rc


def test_errors(engine, fresh):
    w0 = synth.make(np.array([60, 500, 3000]), 806, tg_frac=0.1, met_dep_frac=0.05)
    at, cfg = synth.make_aliases(w0, 807, name_frac=0.8)
    w = plan_and_check(engine, fresh, at, cfg, w0.now)

    def variant(**kw):
        v = copy.copy(at)
        for k, x in kw.items():
            setattr(v, k, x)
        return v
    so, do = at.secondary_off, at.dest_off
    bad_so = so.copy()
    bad_so[3], bad_so[4] = bad_so[4] + 1, bad_so[3]             # decreases
    bad_do = do.copy()
    bad_do[1] = bad_do[2] + 1                                   # decreases
    deps_short = copy.copy(at.deps)
    deps_short.task_state, deps_short.task_pre = at.deps.task_state[:-1], at.deps.task_pre[:-1]
    deps_short.dep_off = at.deps.dep_off[:-1]
    t_off = copy.copy(at.tasks)
    t_off.dep_off = at.tasks.dep_off.copy()
    t_off.dep_off[-1] += 1
    host_cases = [
        variant(secondary_off=bad_so),
        variant(dest_off=bad_do),
        variant(dest_idx=np.where(np.arange(at.dest_idx.shape[0]) == 0, cfg.shape[0], at.dest_idx).astype(np.int32)),
        variant(dest_idx=np.where(np.arange(at.dest_idx.shape[0]) == 0, -1, at.dest_idx).astype(np.int32)),
        variant(deps=deps_short),                                # sizes disagree
        variant(tasks=t_off),                                    # dep_off does not span n_edges
    ]
    for v in host_cases:
        assert raw_plan(engine, v, cfg) == L.EVG_ERR_INVALID, L.last_error()
        check_equal(engine, fresh, w)  # the previous tick, still resident and runnable
    st, keep = at.struct()
    st.n_groups = -1
    bufs = [np.zeros(8, np.int64) for _ in range(3)]
    out = L.AliasOutStruct(*[L.ptr(b) for b in bufs])
    assert engine.lib.evg_plan_aliases(engine.ctx, C.byref(st), L.ptr(cfg), int(cfg.shape[0]), 0, C.byref(out)) == L.EVG_ERR_INVALID
    check_equal(engine, fresh, w)
    # ids found out of range on the device: no resident tick
    named = int(np.nonzero(at.secondary_idx >= 0)[0][0])
    gt = copy.copy(at.tasks)
    gt.group_id = at.tasks.group_id.copy()
    gt.group_id[0] = at.group_max_hosts.shape[0]
    for v in (variant(secondary_idx=np.where(np.arange(at.secondary_idx.shape[0]) == named, -2, at.secondary_idx).astype(np.int32)),
              variant(primary=np.full(at.n_tasks, cfg.shape[0], np.int32)), variant(tasks=gt)):
        engine.plan_aliases(at, cfg, w0.now)
        assert raw_plan(engine, v, cfg) == L.EVG_ERR_INVALID, L.last_error()
        assert engine.lib.evg_run_resident(engine.ctx, 0, 0) == L.EVG_ERR_STATE
    # empty inputs are valid: no rows (every queue empty), no distros (no queue)
    empty = synth.make_aliases(synth.make(np.array([0, 0]), 808), 809)[0]
    task_off, group_off, _ = engine.plan_aliases(empty, cfg, w0.now)
    assert task_off.tolist() == [0, 0, 0, 0] and group_off.tolist() == [0, 0, 0, 0]
    engine.run(w0.now)
    po, _ = engine.download()
    assert po.info["length"].tolist() == [0, 0, 0]
    none = variant(secondary_idx=np.full(at.secondary_idx.shape[0], -1, np.int32), dest_off=np.zeros(1, np.int64),
                   dest_idx=np.zeros(0, np.int32), primary=np.full(at.n_tasks, -1, np.int32))
    task_off, _, _ = engine.plan_aliases(none, cfg[:0], w0.now)
    assert task_off.tolist() == [0]
    engine.run(w0.now)


# ---- the rules of FindHostSchedulableForAlias, one task each, through the Task-level API
NOW = synth.NOW_NS


def task(i, distro, secondary, **kw):
    base = dict(id=f"t{i}", project="p", version=f"v{i % 3}", build_variant="bv", distro_id=distro, secondary_distros=secondary,
                requester=M.REPOTRACKER_VERSION_REQUESTER, priority=i % 5, expected_duration=(1 + i % 7) * M.MINUTE,
                activated_time=NOW - (1 + i) * M.MINUTE, scheduled_time=NOW - M.HOUR)
    base.update(kw)
    return M.Task(**base)


def rule_tick():
    distros = [M.Distro(id="d0", aliases=["a1"]), M.Distro(id="d1", aliases=["a1", "a2"]), M.Distro(id="d2"),
               M.Distro(id="d3", aliases=["nobody-uses-this"])]
    done = M.Task(id="done", status=M.TASK_SUCCEEDED, distro_id="d2")
    tasks = [
        task(0, "d0", ["d1", "a1"]),                                   # reaches d1 twice: once there; d0 through a1
        task(1, "d0", ["d0"]),                                         # its own distro: OTHER_DISTRO clear
        task(2, "d0", ["a2"], task_group="g1", task_group_max_hosts=1),  # single-host task group: out
        task(3, "d0", ["a2"], task_group_max_hosts=1),                 # TaskGroupMaxHosts == 1 without a group: out
        task(4, "d0", ["a2"], activated=False),                        # each base-query bit
        task(5, "d0", ["a2"], status="started"),
        task(6, "d0", ["a2"], priority=-1),
        task(7, "d0", ["a2"], execution_platform="container"),
        task(8, "d0", ["a2"], unattainable_dependency=True),           # unattainable: out
        task(9, "d0", ["a2"], unattainable_dependency=True, override_dependencies=True,
             depends_on=[M.Dependency("done")]),                       # ... unless overridden
        task(10, "d0", ["zzz"]),                                       # a name no distro has
        task(11, "d0", ["a2"], task_group="tg", task_group_max_hosts=3, version="vx", task_group_order=1),
        task(12, "d2", ["a2"], task_group="tg", task_group_max_hosts=3, version="vx", task_group_order=2),  # one group in d1
        task(13, "d0", ["a2"], depends_on=[M.Dependency("t14"), M.Dependency("t9")]),  # t14 is not in d1's queue
        task(14, "d0", []),
        task(15, "d0", ["a2"], depends_on=[M.Dependency("t9"), M.Dependency("t9")]),   # duplicate DependsOn entries
        task(16, "elsewhere", ["a2", "d1"], num_dependents=3),   # two names, one queue
    ]
    return distros, tasks, {t.id: t for t in tasks + [done]}


def compare_plans(got, want):
    for (gr, gi), (wr, wi) in zip(got, want):
        assert [t.id for t in gr] == [t.id for t in wr]
        assert [t.sorting_value_breakdown.total_value for t in gr] == [t.sorting_value_breakdown.total_value for t in wr]
        for f in parity.INFO_FIELDS:
            assert getattr(gi, f) == getattr(wi, f), f
        key = lambda infos: sorted((g.name,) + tuple(getattr(g, f) for f in L.GROUP_INFO_FIELDS) for g in infos)  # noqa: E731
        assert key(gi.task_group_infos) == key(wi.task_group_infos)


def test_each_rule_and_the_mirror(engine, fresh):
    distros, tasks, db = rule_tick()
    want_ids = {"d0": ["t0", "t1"], "d1": ["t0", "t9", "t11", "t12", "t13", "t15", "t16"], "d2": [], "d3": []}
    for d in distros:
        assert [t.id for t in scheduler.find_host_schedulable_for_alias(d.id, tasks, distros)] == want_ids[d.id]
    got = scheduler.plan_alias_queues(distros, copy.deepcopy(tasks), NOW, engine=engine, dependency_db=copy.deepcopy(db),
                                      breakdown=True, started_at=NOW - 5)
    # the raw queue info (before the scheduler.go:44 overwrite): d0's alias queue holds only tasks of d0, so no task
    # has OTHER_DISTRO there; d1's holds tasks of other distros
    po, _ = engine.download()
    assert po.info["secondary_queue"].tolist() == [0, 1, 0, 0]
    tasks2, db2 = copy.deepcopy(tasks), copy.deepcopy(db)
    batch = [(d, scheduler.find_host_schedulable_for_alias(d.id, tasks2, distros)) for d in distros]
    want = scheduler.plan_distros(batch, NOW, engine=fresh, dependency_db=db2, secondary=True)
    compare_plans(got, want)
    assert all(i.secondary_queue and i.plan_created_at == NOW - 5 for _, i in got)
    assert sorted(t.id for t in got[1][0]).count("t0") == 1 and got[2][0] == [] and got[3][0] == []
    tg = [g for g in got[1][1].task_group_infos if g.name.startswith("tg")]
    assert len(tg) == 1 and tg[0].count == 2 and tg[0].max_hosts == 3
    # in d1's queue t13 keeps its edge to t9 only, t15 both of its duplicate edges (in-queue dependencies join units)
    soa, table, _ = S.marshal_tasks([batch[1]], NOW, db2)
    assert soa.dep_idx.tolist() == [1, 1, 1]
    # the persisted alias queues: one document per distro, routed to the alias queues' collection
    qs = scheduler.persist_alias_task_queues(distros, copy.deepcopy(tasks), NOW, engine=engine, dependency_db=copy.deepcopy(db))
    assert [[it.id for it in q.queue] for q in qs] == [[t.id for t in r] for r, _ in got]
    assert all(q.collection() == M.TASK_SECONDARY_QUEUES_COLLECTION for q in qs)
    assert [[it.sorting_value_breakdown.total_value for it in q.queue] for q in qs] == \
        [[t.sorting_value_breakdown.total_value for t in r] for r, _ in got]
