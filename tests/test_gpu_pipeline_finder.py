"""The pipeline task finder on the device (evg_find_runnable_ex, evg_plan_from_finder_ex): the golden cases and random
batches of all five finder codes against the stage-by-stage oracle, a 2e6-candidate run against a numpy restatement,
the planned tick against the host route (oracle finder -> the tasks as returned -> plan), resident edits after a
pipeline tick, and the error contract."""
import copy
import ctypes
import random

import numpy as np
import pytest

import golden_loader as G
import oracle_pipeline as OP
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from oracle import oracle as O
from test_gpu_edit import BOUNDS, size_class
from test_pipeline_finder_host import PIPELINE, check_case, pipeline_case

pytestmark = pytest.mark.gpu

NOW = 1_700_000_000 * 10 ** 9
CODES = {L.EVG_FINDER_NO_DEPS: ("legacy", "revised-with-dependencies"), L.EVG_FINDER_LEGACY: ("legacy", ""),
         L.EVG_FINDER_ALTERNATE: ("alternate", ""), L.EVG_FINDER_PIPELINE: ("pipeline", ""),
         L.EVG_FINDER_PIPELINE_NO_DEPS: ("pipeline", "revised-with-dependencies")}


def without(db, tasks):
    """The collection as seen from one distro: its own candidates are not external documents."""
    own = {t.id for t in tasks}
    return {k: v for k, v in db.items() if k not in own}


def expected(code, d, tasks, refs, db):
    kind, version = CODES[code]
    d = copy.copy(d)
    d.dispatcher_settings = M.DispatcherSettings(version=version)
    if kind == "pipeline":
        return [t.id for t in OP.find_runnable(d, tasks, refs, db)]
    return [t.id for t in O.find_runnable(d, tasks, refs, db, kind)]


@pytest.mark.parametrize("case", PIPELINE["cases"], ids=lambda c: c["name"])
def test_pipeline_golden_on_device(engine, case):
    d, tasks, refs = pipeline_case(case)
    got = scheduler.find_runnable_tasks([(d, tasks)], refs, finder="pipeline", engine=engine)[0]
    assert [t.id for t in got] == [t.id for t in OP.find_runnable(d, tasks, refs)]
    check_case(case, scheduler.pipeline_returned_tasks(d, got))
    assert [t.id for t in scheduler.RunnableTasksPipeline(d, tasks, refs, engine=engine)] == [t.id for t in got]


STATUSES = ["undispatched", "success", "failed", "", "started", "inactive"]
WANTS = ["success", "failed", "*", "", "started"]
REQUESTERS = ["gitter_request", "patch_request", "github_pull_request", "github_merge_request", "ad_hoc", "trigger_request"]


def gate_all(refs):
    """Every raw project_ref lets every task through (for the planner tests)."""
    for r in refs:
        r.enabled, r.dispatching_disabled, r.patching_disabled = True, None, False
    return refs


def random_refs(rng):
    out = []
    for i in range(8):
        out.append(M.ProjectRef(id=f"p{i}", enabled=rng.random() < 0.8, hidden=rng.choice([None, True, False]),
                                dispatching_disabled=rng.choice([None, None, True, False]),
                                patching_disabled=rng.choice([None, True, False])))
    return out


def random_batch(rng, sizes, *, planner=False, version=""):
    """Candidates of every distro with dependencies inside the distro, on other distros' tasks and on finished tasks of
    the collection (dependency_db), on missing ids; "" and odd statuses; unattainable entries; raw project flags."""
    refs = random_refs(rng)
    db = {f"x{i}": M.Task(id=f"x{i}", status=rng.choice(STATUSES), override_dependencies=rng.random() < 0.2,
                          depends_on=[M.Dependency("gone", "*", unattainable=rng.random() < 0.3)] if rng.random() < 0.5 else [])
          for i in range(40)}
    batch = []
    for d, n in enumerate(sizes):
        tasks = []
        for i in range(n):
            t = M.Task(id=f"d{d}-t{i}", project=rng.choice([f"p{rng.randrange(8)}"] * 9 + ["nowhere"]),
                       requester=rng.choice(REQUESTERS), activated=rng.random() < 0.95,
                       status=rng.choice(["undispatched"] * 12 + STATUSES[1:]), priority=rng.choice([0, 0, 0, 5, 50, -1]),
                       distro_id=f"d{d}", override_dependencies=rng.random() < 0.03,
                       dependencies_met_time=NOW - 10 ** 9 if rng.random() < 0.03 else M.ZERO_TIME)
            if planner:  # nearly every candidate passes the base query and the gating: the kept sizes stay near n
                t.project, t.activated, t.status = f"p{rng.randrange(8)}", True, "undispatched"
                t.priority = rng.choice([0, 0, 5, 50])
                t.version = f"v{rng.randrange(6)}"
                t.build_variant = f"bv{rng.randrange(3)}"
                if rng.random() < 0.15:
                    t.task_group = f"g{rng.randrange(4)}"
                    t.task_group_max_hosts = 1 + (int(t.task_group[1:]) + int(t.version[1:])) % 3
                    t.task_group_order = rng.randrange(5)
                t.expected_duration = rng.randrange(1, 4 * 3600) * 10 ** 9
                t.activated_time = NOW - rng.randrange(1, 10 ** 5) * 10 ** 9
                t.scheduled_time = NOW - rng.randrange(1, 10 ** 5) * 10 ** 9
                t.num_dependents = rng.randrange(4)
                t.generate_task = rng.random() < 0.05
            k = rng.choice([0] * 16 + [1, 2]) if planner else rng.choice([0, 0, 0, 1, 1, 2, 3])
            seen = set()
            for _ in range(k):
                u = rng.random()
                if u < 0.5 and i > 0:
                    target = f"d{d}-t{rng.randrange(i)}"
                elif u < 0.8:
                    target = f"x{rng.randrange(40)}"
                elif u < 0.9:
                    target = f"d{rng.randrange(len(sizes))}-t0"
                else:
                    target = f"missing{rng.randrange(5)}"
                if target in seen:  # one entry per dependency: SatisfiesDependency reads the first match only
                    continue
                seen.add(target)
                t.depends_on.append(M.Dependency(target, rng.choice(WANTS + ["*"] * 2), unattainable=rng.random() < 0.2,
                                                 finished_at=rng.choice([M.ZERO_TIME, 0, NOW - 5 * 10 ** 9])))
            tasks.append(t)
        batch.append((M.Distro(id=f"d{d}", dispatcher_settings=M.DispatcherSettings(version=version)), tasks))
    # a task of another distro is a document of the collection too
    for _, tasks in batch:
        for t in tasks:
            db.setdefault(t.id, t)
    return batch, refs, db


@pytest.mark.parametrize("seed", range(3))
def test_random_batches_mix_all_five_codes(engine, seed):
    rng = random.Random(900 + seed)
    batch, refs, db = random_batch(rng, [rng.randrange(0, 60) for _ in range(15)] + [700])
    table = S.marshal_runnable(batch, refs, "pipeline", db)
    codes = np.array([rng.randrange(5) for _ in batch], np.uint8)
    table.finder = codes
    runnable, count = engine.find_runnable_batch(table)
    for i, (d, tasks) in enumerate(batch):
        a = int(table.task_off[i])
        got = [tasks[int(j)].id for j in runnable[a:a + int(count[i])]]
        # the other distros' candidates are documents of the collection, not of this distro's candidates
        others = without(db, tasks)
        assert got == expected(int(codes[i]), d, tasks, refs, others), (i, int(codes[i]))


def test_pipeline_at_scale(engine):
    """2e6 candidates over 3000 distros, every code: device result vs a numpy restatement of the same tables."""
    rng = np.random.default_rng(11)
    D, P, X, NS = 3000, 64, 4000, 6
    sizes = rng.integers(0, 1300, D)
    sizes[5] = 40_000
    off = np.zeros(D + 1, np.int64); np.cumsum(sizes, out=off[1:])
    T = int(off[-1])
    sched = (rng.integers(0, 256, T) | 0x0F * (rng.random(T) < 0.85)).astype(np.uint8)
    project = rng.integers(-1, P, T).astype(np.int32)
    pflags = rng.integers(0, 16, P).astype(np.uint8)
    praw = rng.integers(0, 8, P).astype(np.uint8) | (rng.random(P) < 0.7).astype(np.uint8)
    nvalid = np.where(rng.random(D) < 0.3, rng.integers(1, 6, D), 0)
    voff = np.zeros(D + 1, np.int64); np.cumsum(nvalid, out=voff[1:])
    vidx = rng.integers(-1, P, int(voff[-1])).astype(np.int32)
    finder = rng.integers(0, 5, D).astype(np.uint8)
    n_dep = rng.choice([0, 0, 1, 2, 3], T)
    doff = np.zeros(T + 1, np.int64); np.cumsum(n_dep, out=doff[1:])
    E = int(doff[-1])
    kind = rng.choice([0, 1, 2], E, p=[0.5, 0.4, 0.1]).astype(np.uint8)
    ref = np.where(kind == 0, rng.integers(0, T, E), rng.integers(0, X, E)).astype(np.int32)
    want = rng.integers(0, 4, E).astype(np.uint8)
    tstate = (rng.integers(0, 3, T) | 4 * (rng.random(T) < 0.2)).astype(np.uint8)
    tpre = ((rng.random(T) < 0.1) | ((rng.random(T) < 0.1) << 1)).astype(np.uint8)
    xstate = (rng.integers(0, 3, X) | 4 * (rng.random(X) < 0.2)).astype(np.uint8)
    deps = S.DepsTable(doff, kind, ref, want, tstate, tpre, xstate)
    pipe = S.PipelineTable(NS, rng.integers(0, NS, E).astype(np.int32), rng.integers(0, NS, T).astype(np.int32),
                           rng.integers(0, NS, X).astype(np.int32), (rng.random(T) < 0.1).astype(np.uint8),
                           (rng.random(X) < 0.2).astype(np.uint8), praw)
    table = S.RunnableTable(off, sched, project, pflags, voff, vidx, finder, deps, pipe)
    runnable, count = engine.find_runnable_batch(table)

    # ---- numpy restatement
    owner = np.repeat(np.arange(T), n_dep)
    st = np.where(kind == 0, tstate[np.minimum(ref, T - 1)], xstate[np.minimum(ref, X - 1)])
    status = st & 3
    ok_e = np.select([want == 0, want == 1, want == 2], [status == 0, status == 1, (status < 2) | ((st & 4) != 0)], False)
    ok_e &= kind != 2
    bad = np.bincount(owner, weights=~ok_e, minlength=T) > 0
    short = (tpre & 3) != 0
    met_legacy = ~bad | short
    met_alt = ~bad
    pst = np.where(kind == 0, pipe.task_status[np.minimum(ref, T - 1)], pipe.ext_status[np.minimum(ref, X - 1)])
    pun = np.where(kind == 0, pipe.task_unattainable[np.minimum(ref, T - 1)], pipe.ext_unattainable[np.minimum(ref, X - 1)]) != 0
    sat = (pipe.dep_status == pst) | ((pipe.dep_status == 2) & ((pst == 0) | (pst == 1) | pun))
    exists = kind != 2
    unsat = np.bincount(owner, weights=exists & ~sat, minlength=T) > 0
    paired = np.bincount(owner, weights=exists, minlength=T) > 0
    met_pipe = ~unsat & (paired | (n_dep == 0))
    distro_of = np.repeat(np.arange(D), sizes)
    f = finder[distro_of]
    base = ((sched & 0x0F) == 0x0F) & (((sched & 0x10) == 0) | ((sched & 0x20) != 0))
    pj = np.maximum(project, 0)
    has_p = project >= 0
    pf, pr = pflags[pj], praw[pj]
    legacy_gate = (((pf & 1) != 0) | (((sched & 0x40) != 0) & ((pf & 2) != 0))) & ((pf & 4) == 0) & \
        ~(((sched & 0x80) != 0) & ((pf & 8) != 0))
    pipe_gate = ((pr & 1) != 0) & ((pr & 2) == 0) & (((sched & 0x80) == 0) | ((pr & 4) != 0))
    valid = np.ones(T, bool)
    for d in np.nonzero(nvalid)[0]:
        a, b = off[d], off[d + 1]
        valid[a:b] = np.isin(project[a:b], vidx[voff[d]:voff[d + 1]])
    gate = np.where(f >= 3, pipe_gate, legacy_gate)
    dep_ok = np.select([f == 1, f == 2, f == 3], [met_legacy, met_alt, met_pipe], True)
    keep = base & has_p & gate & valid & dep_ok
    for d in range(D):
        a, b = int(off[d]), int(off[d + 1])
        want_idx = np.nonzero(keep[a:b])[0]
        assert int(count[d]) == want_idx.size, d
        assert np.array_equal(runnable[a:a + want_idx.size], want_idx), d
        assert (runnable[a + want_idx.size:b] == -1).all()


# ---------------------------------------------------------------- the planned tick against the host route

def device_route(eng, batch, refs, db):
    """plan_candidates' calls: the candidates through evg_plan_from_finder_ex, then run + download."""
    table = S.marshal_runnable(batch, refs, "pipeline", db)
    if table.deps is None:
        table.deps = S.marshal_deps(batch, db)
    soa, dtable, keys = S.marshal_tasks(batch, NOW, db)
    runnable, count = eng.plan_from_finder(table, soa, dtable, None, S.marshal_dep_finished(batch), NOW)
    return collect(eng, np.concatenate([[0], np.cumsum(count)]).astype(np.int64), dtable, keys), count.copy()


def returned_view(batch, refs, db):
    """Per distro, the oracle finder's tasks as the aggregation decodes them."""
    return [(d, scheduler.pipeline_returned_tasks(d, OP.find_runnable(d, tasks, refs, without(db, tasks)))) for d, tasks in batch]


def host_route(eng, batch, refs, db):
    """The oracle finder, the returned tasks as decoded, marshalled and planned like plan_distros does."""
    view = returned_view(batch, refs, db)
    # what the depCache misses is fetched whole from the collection: every candidate of every distro is in it
    soa, dtable, keys = S.marshal_tasks(view, NOW, db)
    scheduler._upload_with_device_deps(eng, view, soa, dtable, None, NOW, db)
    return collect(eng, dtable.task_off.copy(), dtable, keys), np.diff(dtable.task_off)


def collect(eng, task_off, dtable, keys):
    """The tick's outputs; task groups by name, the live ones only (the finder's tick keeps the candidates' group
    slots, empty ones included)."""
    eng.run(NOW, L.EVG_OPT_BREAKDOWN)
    po, _ = eng.download(want_breakdown=True, want_alloc=False)
    item_off, items = eng.download_queue(0, task_off)
    groups = []
    for d in range(dtable.n_distros):
        ga, gb = int(dtable.group_off[d]), int(dtable.group_off[d + 1])
        groups.append(sorted((name, tuple(int(g[f]) for f in L.GROUP_INFO_FIELDS))
                             for name, g in zip(keys[d].group_names, po.group_info[ga:gb]) if int(g["count"])))
    return (po.order.copy(), po.total_value.copy(), po.info.copy(), groups, po.breakdown.copy(), item_off.copy(), items.copy())


@pytest.fixture(scope="module")
def other():
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


@pytest.mark.parametrize("version", ["", "revised-with-dependencies"])
def test_planned_tick_equals_the_host_route(engine, other, version):
    """EVG_FINDER_PIPELINE ("") and EVG_FINDER_PIPELINE_NO_DEPS distros, every route."""
    rng = random.Random(77 + len(version))
    sizes = [20, 300, 1000, 4000, 9000, 11500, 14000]
    batch, refs, db = random_batch(rng, sizes, planner=True, version=version)
    gate_all(refs)  # keep most candidates so that every size class is planned
    a, count = device_route(engine, batch, refs, db)
    b, count_b = host_route(other, batch, refs, db)
    assert np.array_equal(count, count_b)
    assert {size_class(int(n)) for n in count} == set(range(len(BOUNDS) + 1))  # every route, one distro above 12288
    for name, x, y in zip(("order", "total_value", "info", "groups", "breakdown", "item_off", "items"), a, b):
        assert (x == y) if name == "groups" else np.array_equal(x, y), name
    if version == "":
        assert int(a[2]["length_with_dependencies_met"].sum()) == int(count.sum())  # nothing waits on a dependency


def test_plan_candidates_pipeline(engine):
    rng = random.Random(5)
    batch, refs, db = random_batch(rng, [30, 400], planner=True)
    gate_all(refs)
    ranked = scheduler.plan_candidates(batch, refs, NOW, finder="pipeline", dependency_db=db, engine=engine)
    host = scheduler.plan_distros(returned_view(batch, refs, db), NOW, engine=engine, dependency_db=db, breakdown=False)
    live = lambda infos: sorted((g.name, g.count, g.expected_duration, g.count_duration_over_threshold,  # noqa: E731
                                 g.count_wait_over_threshold) for g in infos if g.count or g.name == "")
    for (ra, qa), (rb, qb) in zip(ranked, host):
        assert [(t.id, t.sorting_value_breakdown.total_value) for t in ra] == \
            [(t.id, t.sorting_value_breakdown.total_value) for t in rb]
        assert live(qa.task_group_infos) == live(qb.task_group_infos)
        qa.task_group_infos, qb.task_group_infos = [], []
        assert qa == qb


def test_update_and_edit_after_a_pipeline_tick(engine, other):
    from test_gpu_edit import check_equal
    from test_gpu_finder_compaction import drop, kept_mask
    from evergreen_b200 import synth
    rng = random.Random(31)
    batch, refs, db = random_batch(rng, [50, 700, 2000], planner=True)
    gate_all(refs)
    table = S.marshal_runnable(batch, refs, "pipeline", db)
    soa, dtable, _ = S.marshal_tasks(batch, NOW, db)
    runnable, count = engine.plan_from_finder(table, soa, dtable, None, S.marshal_dep_finished(batch), NOW)
    runnable, count = runnable.copy(), count.copy()
    # the same tick built on the host: the candidates' columns without the dropped rows and, the DependsOn of the
    # returned tasks being empty, without edges; the verdicts of the returned tasks (met, nothing stamped)
    view = [(d, scheduler.pipeline_returned_tasks(d, [tasks[int(j)] for j in runnable[int(table.task_off[i]):
                                                                                    int(table.task_off[i]) + int(count[i])]]))
            for i, (d, tasks) in enumerate(batch)]
    vsoa, vtable, _ = S.marshal_tasks(view, NOW, db)
    other.upload_with_deps(vsoa, vtable, None, S.marshal_deps(view, db), S.marshal_dep_finished(view), NOW)
    met, stamp = (x.copy() for x in other.download_deps())
    assert (met & 1).all() and (stamp == L.EVG_TIME_ZERO).all()
    _, tasks, distros = drop(soa, dtable, kept_mask(table, runnable, count))
    tasks.dep_off = np.zeros_like(tasks.dep_off)
    tasks.dep_idx = np.zeros(0, np.int32)
    tasks.flags = tasks.flags | np.uint32(L.EVG_TF_DEPS_MET)
    engine.run(NOW)
    check_equal(engine, other, synth.Workload("pipeline", NOW, tasks, distros, None), breakdown=True)
    # an update of a tenth of the rows
    nr = np.random.default_rng(3)
    rows = np.sort(nr.choice(tasks.n_tasks, size=tasks.n_tasks // 10, replace=False)).astype(np.int64)
    tasks.priority[rows] = nr.integers(0, 101, rows.size)
    tasks.flags[rows] ^= np.uint32(L.EVG_TF_DEPS_MET)
    engine.update_tasks(rows, S.TaskSoA(**{name: getattr(tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
    check_equal(engine, other, synth.Workload("pipeline", NOW, tasks, distros, None), breakdown=True)
    # then an edit that removes every fifth row
    keep = np.ones(tasks.n_tasks, bool)
    keep[::5] = False
    ed, tasks2, distros2 = drop(tasks, distros, keep)
    engine.edit_tasks(ed, distros2)
    check_equal(engine, other, synth.Workload("pipeline", NOW, tasks2, distros2, None), breakdown=True)


def test_invalid_pipeline_input(engine):
    """Inputs the host can reject leave the previous tick resident and runnable; a status id out of range is found on
    the device and leaves no tick, as for the other ids the device checks."""
    rng = random.Random(41)
    batch, refs, db = random_batch(rng, [40, 600], planner=True)
    table = S.marshal_runnable(batch, refs, "pipeline", db)
    soa, dtable, _ = S.marshal_tasks(batch, NOW, db)
    fin = S.marshal_dep_finished(batch)
    engine.plan_from_finder(table, soa, dtable, None, fin, NOW)
    engine.run(NOW)
    before = engine.download(want_alloc=False)[0].order.copy()

    def rejected(t):
        for call in (lambda: engine.plan_from_finder(t, soa, dtable, None, fin, NOW), lambda: engine.find_runnable_batch(t)):
            with pytest.raises(L.EvgError) as e:
                call()
            assert e.value.code == L.EVG_ERR_INVALID, str(e.value)

    no_pipe = copy.copy(table)
    no_pipe.pipe = None  # a pipeline code without an evg_pipeline_in
    rejected(no_pipe)
    unknown = copy.copy(table)
    unknown.finder = np.full_like(table.finder, 5)
    rejected(unknown)
    small = copy.deepcopy(table)
    small.pipe.n_status = 2
    rejected(small)
    # the old entry points refuse the pipeline codes whatever the caller passes
    st, keep = table.struct()
    with pytest.raises(L.EvgError) as e:
        L.check(engine.lib.evg_find_runnable_batch(engine.ctx, ctypes.byref(st), L.ptr(np.zeros(table.n_tasks, np.int32)),
                                                   L.ptr(np.zeros(table.n_distros, np.int64))))
    assert e.value.code == L.EVG_ERR_INVALID
    engine.run(NOW)
    assert np.array_equal(engine.download(want_alloc=False)[0].order, before)
    for field in ("dep_status", "task_status"):
        bad = copy.deepcopy(table)
        col = getattr(bad.pipe, field)
        col[len(col) // 2] = bad.pipe.n_status
        rejected(bad)
    with pytest.raises(L.EvgError):
        engine.run(NOW)
    engine.plan_from_finder(table, soa, dtable, None, fin, NOW)
    engine.run(NOW)
    assert np.array_equal(engine.download(want_alloc=False)[0].order, before)
