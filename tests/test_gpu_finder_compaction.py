"""evg_plan_from_finder builds its tick with evg_edit_tasks' compaction: the finder's tick equals an upload of every
candidate (evg_upload_with_deps) edited down to the kept ones, it may be updated like any resident tick, and malformed
candidate edges are rejected before they index anything.  Also: evg_download_deps after evg_deps_met_batch."""
import copy

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_edit import SIZES, check_equal, outputs, size_class

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def other():
    """A second context: the upload-and-edit route, or a fresh upload."""
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


FINDERS = {"no_deps": L.EVG_FINDER_NO_DEPS, "legacy": L.EVG_FINDER_LEGACY, "alternate": L.EVG_FINDER_ALTERNATE}


def candidates(sizes, seed, finder):
    """A candidate tick: the planner columns (task groups, GroupVersions, in-queue edges; no EVG_TF_DEPS_MET), the finder
    table over it (`finder`: one kind for every distro, or "mixed"), a dependency table holding every in-queue edge plus
    some external and missing dependencies, and dep_finished_ns with real, zero and unset times."""
    w = synth.make(np.array(sizes), seed, zipf_priority=True, unmet_dep_frac=0.03, met_dep_frac=0.05, tg_frac=0.1,
                   group_versions_frac=0.3, includes_dependencies=True, n_hosts=200)
    t, dt = w.tasks, w.distros
    t.flags &= ~np.uint32(L.EVG_TF_DEPS_MET)
    rng = np.random.default_rng(seed)
    T, D, X = t.n_tasks, dt.n_distros, 50
    distro_of = np.repeat(np.arange(D), np.diff(dt.task_off))
    owner_q = np.repeat(np.arange(T), np.diff(t.dep_off))
    extra = np.nonzero(rng.random(T) < 0.05)[0]
    kind_x = np.where(rng.random(extra.size) < 0.8, L.EVG_DEP_EXTERNAL, L.EVG_DEP_MISSING)
    owner = np.concatenate([owner_q, extra])
    kind = np.concatenate([np.full(owner_q.size, L.EVG_DEP_IN_QUEUE), kind_x])
    ref = np.concatenate([dt.task_off[distro_of[owner_q]] + t.dep_idx, np.where(kind_x == L.EVG_DEP_EXTERNAL, rng.integers(0, X, extra.size), 0)])
    o = np.argsort(owner, kind="stable")
    E = owner.size
    blocked = lambda n: np.where(rng.random(n) < 0.05, L.EVG_TS_BLOCKED, 0)  # noqa: E731
    deps = S.DepsTable(np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=T))]).astype(np.int64),
                       kind[o].astype(np.uint8), ref[o].astype(np.int32),
                       rng.choice([L.EVG_WANT_SUCCESS, L.EVG_WANT_FAILED, L.EVG_WANT_ANY, L.EVG_WANT_OTHER], size=E,
                                  p=[0.7, 0.1, 0.15, 0.05]).astype(np.uint8),
                       (rng.choice([0, 1, 2], size=T, p=[0.8, 0.1, 0.1]) | blocked(T)).astype(np.uint8),
                       (np.where(rng.random(T) < 0.05, L.EVG_TP_OVERRIDE, 0) | np.where(rng.random(T) < 0.05, L.EVG_TP_MET_TIME, 0)).astype(np.uint8),
                       (rng.integers(0, 3, X) | blocked(X)).astype(np.uint8))
    u = rng.random(E)
    fin = np.where(u < 0.5, w.now - rng.integers(0, 10 ** 12, E), np.where(u < 0.8, L.EVG_TIME_ZERO, 0)).astype(np.int64)
    sched = np.full(T, L.EVG_SQ_ACTIVATED | L.EVG_SQ_UNDISPATCHED | L.EVG_SQ_PRIORITY_OK | L.EVG_SQ_HOST_PLATFORM, np.uint8)
    sched[rng.random(T) < 0.02] &= ~np.uint8(L.EVG_SQ_ACTIVATED)
    sched |= np.where(rng.random(T) < 0.02, L.EVG_SQ_UNATTAINABLE, 0).astype(np.uint8)
    sched |= np.where(rng.random(T) < 0.3, L.EVG_SQ_PATCH_REQUEST, 0).astype(np.uint8)
    pflags = np.array([L.EVG_PF_ENABLED, L.EVG_PF_ENABLED, L.EVG_PF_ENABLED | L.EVG_PF_PATCHING_DISABLED, 0], np.uint8)
    project = rng.choice([0, 1, 2, 3, -1], size=T, p=[0.6, 0.35, 0.03, 0.01, 0.01]).astype(np.int32)
    nvalid = np.where(rng.random(D) < 0.3, 3, 0)
    voff = np.concatenate([[0], np.cumsum(nvalid)]).astype(np.int64)
    vidx = np.tile(np.array([0, 1, 2], np.int32), int(voff[-1]) // 3)
    kinds = rng.integers(0, 3, D) if finder == "mixed" else np.full(D, FINDERS[finder])
    table = S.RunnableTable(dt.task_off.copy(), sched, project, pflags, voff, vidx, kinds.astype(np.uint8), deps)
    return w, table, fin


def kept_mask(table, runnable, count):
    off = table.task_off
    distro_of = np.repeat(np.arange(table.n_distros), np.diff(off))
    slot = np.arange(table.n_tasks) - off[distro_of]
    used = slot < count[distro_of]
    keep = np.zeros(table.n_tasks, dtype=bool)
    keep[off[distro_of[used]] + runnable[used]] = True
    return keep


def drop(tasks, distros, keep):
    """The edit that removes every candidate the finder dropped, and the kept table it composes."""
    ed = S.TaskEdit(np.nonzero(~keep)[0], None, np.zeros(distros.n_distros + 1, np.int64), np.zeros(0, np.int64),
                    np.zeros(0, np.int32)).normalize()
    return (ed,) + S.apply_edit(tasks, distros, ed)


@pytest.mark.parametrize("finder", ["no_deps", "legacy", "alternate", "mixed"])
def test_finders_tick_is_an_edit(engine, other, finder):
    w, table, fin = candidates(SIZES + [300], 601, finder)  # 300: a kept queue in (32, 384] whatever the finder drops
    runnable, count = engine.plan_from_finder(table, w.tasks, w.distros, w.hosts, fin, w.now)
    keep = kept_mask(table, runnable.copy(), count.copy())
    other.upload_with_deps(w.tasks, w.distros, w.hosts, table.deps, fin, w.now)
    ed, tasks, distros = drop(w.tasks, w.distros, keep)
    other.edit_tasks(ed, distros, w.hosts)
    kw = synth.Workload(w.name, w.now, tasks, distros, w.hosts)
    assert {size_class(int(n)) for n in np.diff(distros.task_off)} == set(range(7))  # every route
    assert 0 < tasks.n_edges < w.tasks.n_edges and 0 < keep.sum() < keep.size
    a, b = outputs(engine, kw, True), outputs(other, kw, True)
    for f in ("order", "total_value", "info", "group_info", "breakdown"):
        assert np.array_equal(getattr(a[0], f), getattr(b[0], f)), f
    assert np.array_equal(a[1].result, b[1].result) and np.array_equal(a[1].status, b[1].status)
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])


def test_update_tasks_after_plan_from_finder(engine, other):
    w, table, fin = candidates([40, 900, 6000, 13000], 602, "mixed")
    runnable, count = engine.plan_from_finder(table, w.tasks, w.distros, w.hosts, fin, w.now)
    keep = kept_mask(table, runnable.copy(), count.copy())
    # the candidates with the device's verdict applied, as the finder's tick holds them
    other.upload_with_deps(w.tasks, w.distros, None, table.deps, fin, w.now)
    met, stamp = (x.copy() for x in other.download_deps())
    t = copy.deepcopy(w.tasks)
    t.flags = (t.flags & ~np.uint32(L.EVG_TF_DEPS_MET)) | np.where(met & 1, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
    t.wait_basis_ns = np.where((stamp != L.EVG_TIME_ZERO) & (stamp > t.wait_basis_ns), stamp, t.wait_basis_ns)
    _, tasks, distros = drop(t, w.distros, keep)
    kw = synth.Workload(w.name, w.now, tasks, distros, w.hosts)
    rng = np.random.default_rng(7)
    rows = np.sort(rng.choice(tasks.n_tasks, size=tasks.n_tasks // 10, replace=False)).astype(np.int64)
    tasks.priority[rows] = rng.integers(0, 101, rows.size)
    tasks.expected_ns[rows] += rng.integers(0, 10 ** 10, rows.size)
    tasks.flags[rows] ^= np.uint32(L.EVG_TF_DEPS_MET)
    engine.update_tasks(rows, S.TaskSoA(**{name: getattr(tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
    check_equal(engine, other, kw, breakdown=True)


def test_download_deps_after_deps_met_batch_is_a_state_error(engine):
    w, table, fin = candidates([300, 2000], 603, "legacy")
    engine.upload_with_deps(w.tasks, w.distros, None, table.deps, fin, w.now)
    engine.download_deps()
    d = table.deps
    n = int(d.dep_off[10])
    batch = S.DepsTable(d.dep_off[:11].copy(), d.dep_kind[:n], np.where(d.dep_kind[:n] == L.EVG_DEP_IN_QUEUE, 0, d.dep_ref[:n]).astype(np.int32),
                        d.dep_want[:n], d.task_state[:10], d.task_pre[:10], d.ext_state)
    engine.deps_met_batch(batch)
    with pytest.raises(L.EvgError) as e:
        engine.download_deps()
    assert e.value.code == L.EVG_ERR_STATE
    engine.run(w.now)  # the tick itself stays resident
    engine.download()


def test_plan_from_finder_rejects_malformed_candidate_edges(engine):
    w, table, fin = candidates([300, 2000, 40], 604, "legacy")
    t = w.tasks
    runnable, count = engine.plan_from_finder(table, t, w.distros, None, fin, w.now)
    runnable, count = runnable.copy(), count.copy()
    keep = kept_mask(table, runnable, count)

    def rejected(**cols):
        bad = copy.copy(t)
        for k, v in cols.items():
            setattr(bad, k, v)
        with pytest.raises(L.EvgError) as e:
            engine.plan_from_finder(table, bad, w.distros, None, fin, w.now)
        assert e.value.code == L.EVG_ERR_INVALID, str(e.value)

    off = t.dep_off
    start = off.copy(); start[0] = 1
    end = off.copy(); end[-1] -= 1
    j = int(np.nonzero((off[2:-1] > off[1:-2]))[0][0]) + 1
    down = off.copy(); down[j], down[j + 1] = off[j + 1], off[j]
    for o in (start, end, down):
        rejected(dep_off=o)
    # a dependency one past the end of its distro, on a kept candidate
    distro_of = np.repeat(np.arange(w.distros.n_distros), np.diff(w.distros.task_off))
    row = int(np.nonzero(keep & (np.diff(off) > 0))[0][0])
    idx = t.dep_idx.copy()
    idx[off[row]] = w.distros.task_off[distro_of[row] + 1] - w.distros.task_off[distro_of[row]]
    rejected(dep_idx=idx)
    with pytest.raises(L.EvgError):
        engine.run(w.now)  # a table rejected on the device leaves no resident tick
    r2, c2 = engine.plan_from_finder(table, t, w.distros, None, fin, w.now)
    assert np.array_equal(c2, count) and np.array_equal(r2, runnable)
