"""evg_edit_tasks_with_deps on the device: over seeded multi-tick scripts the edited context holds, tick after tick,
what evg_upload_with_deps of the composed tick (soa.apply_deps_edit's table) holds in a second context -- verdicts and
stamps, the planner's outputs (which read the resident flags and wait basis), the persisted queue and its breakdown --
at small sizes and on the general path; ResidentTick(device_deps=True) returns what the host-evaluated ResidentTick
returns and leaves the same stamps on the Task objects; and the call's state and validation rules."""
import copy
import ctypes as C

import numpy as np
import pytest

import edit_deps_scripts as X
from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pair():
    a, b = scheduler.Engine(0), scheduler.Engine(0)
    yield a, b
    a.close()
    b.close()


def outputs(eng, table, now):
    met, stamp = eng.download_deps()
    met, stamp = met.copy(), stamp.copy()
    eng.run(now, L.EVG_OPT_BREAKDOWN)
    po, _ = eng.download(want_breakdown=True, want_alloc=False)
    po = [po.order.copy(), po.total_value.copy(), po.info.copy(), po.group_info.copy(), po.breakdown.copy()]
    off, items = eng.download_queue(0, table.task_off)
    boff, bd = eng.download_queue_breakdown(0, table.task_off)
    return [met, stamp] + po + [off.copy(), items.copy(), boff.copy(), bd.copy()]


def assert_same(a, b, table, now, where):
    for k, (x, y) in enumerate(zip(outputs(a, table, now), outputs(b, table, now))):
        assert np.array_equal(x, y), (where, k)


def drive(pair, seed, sizes, ticks):
    a, b = pair
    sc = X.Script(seed, sizes)
    rt = scheduler.ResidentTick()  # its canonical order, diff and memory only; the engines are driven here
    shim = S.DepsShim(sc.db)
    canon = rt.canonical(sc.batch)
    now = X.NOW
    soa, table, keys = S.marshal_tasks(canon, now, sc.db)
    deps, fin = shim.upload(canon)
    a.upload_with_deps(soa, table, None, deps, fin, now)
    b.upload_with_deps(soa, table, None, deps, fin, now)
    n_edit = 0
    for tick in range(ticks + 1):
        assert_same(a, b, table, now, (seed, tick))
        _, stamp = b.download_deps()
        stamp = stamp.copy()
        X.write_back(canon, stamp)
        shim.remember(canon)
        rt.remember(canon, soa, table, keys)
        if tick == ticks:
            break
        now = X.NOW + (tick + 1) * 10 ** 11
        canon = rt.canonical(sc.step(tick))
        soa, table, keys = S.marshal_tasks(canon, now, sc.db)
        change = rt.diff(canon, soa, table, keys)
        dx = None if change is None else shim.edit(rt.ids, canon, change[0].remove_rows)
        if dx is None:
            deps, fin = shim.upload(canon)
            a.upload_with_deps(soa, table, None, deps, fin, now)
        else:
            n_edit += 1
            edit, rows, values = change
            a.edit_tasks_with_deps(edit, table, rows, values, dx, now)
            deps, fin = S.apply_deps_edit(deps, rt.table.task_off, edit, dx, fin, stamp)
        b.upload_with_deps(soa, table, None, deps, fin, now)
    return n_edit


@pytest.mark.parametrize("seed", range(4))
def test_scripts_equal_a_fresh_upload_with_deps(pair, seed):
    assert drive(pair, seed, [1, 7, 33, 90, 700], ticks=6) >= 3


def test_general_path_script(pair):
    assert drive(pair, 77, [13000, 40], ticks=3) >= 2


def test_resident_tick_device_deps_equals_host_deps(pair):
    a, b = pair
    sc = X.Script(5, [3, 30, 200])
    host = scheduler.ResidentTick(engine=a, dependency_db=sc.db)
    dev = scheduler.ResidentTick(engine=b, dependency_db=sc.db, device_deps=True)
    batch = sc.batch
    for tick in range(6):
        now = X.NOW + tick * 10 ** 11
        mine = copy.deepcopy(batch)
        ra = host.plan(batch, now)
        rb = dev.plan(mine, now)
        for (ta, ia), (tb, ib) in zip(ra, rb):
            assert [t.id for t in ta] == [t.id for t in tb], tick
            assert [t.sorting_value_breakdown for t in ta] == [t.sorting_value_breakdown for t in tb], tick
            assert ia == ib, tick
        assert [t.dependencies_met_time for _, ts in batch for t in ts] == [t.dependencies_met_time for _, ts in mine for t in ts]
        assert (dev.last is not None) == (host.last is not None)
        batch = sc.step(tick)
    assert host.last is not None


def first_two_ticks():
    """A script's first tick (soa, table, deps, FinishedAt) and the edit to its second, (change, table, DepsEdit): the
    first seed whose step is an edit with updated rows and a departure some survivor depends on (the -1 probe needs one)."""
    for seed in range(11, 40):
        sc = X.Script(seed, [5, 60])
        rt = scheduler.ResidentTick()
        shim = S.DepsShim(sc.db)
        canon = rt.canonical(sc.batch)
        soa, table, keys = S.marshal_tasks(canon, X.NOW, sc.db)
        deps, fin = shim.upload(canon)
        shim.remember(canon)
        rt.remember(canon, soa, table, keys)
        canon2 = rt.canonical(sc.step(0))
        soa2, table2, keys2 = S.marshal_tasks(canon2, X.NOW, sc.db)
        change = rt.diff(canon2, soa2, table2, keys2)
        dx = None if change is None else shim.edit(rt.ids, canon2, change[0].remove_rows)
        if dx is not None and np.any(dx.depart_ext >= 0) and change[1].shape[0] and dx.insert.n_tasks:
            return (soa, table, deps, fin), (change, table2, dx)
    raise AssertionError("no script step fits")


def raw(eng, change, table, dx, now=X.NOW):
    edit, rows, values = change
    es, keep = edit.normalize().struct()
    xs, xkeep = dx.struct()
    ds, vs = table.struct(), values.normalize().struct()
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    rc = eng.lib.evg_edit_tasks_with_deps(eng.ctx, C.byref(es), C.byref(ds), None, None, None, int(rows.shape[0]),
                                          L.ptr(rows) if rows.shape[0] else None, C.byref(vs), C.byref(xs), int(now))
    del keep, xkeep
    return rc


def runnable(eng, table):
    eng.run(X.NOW)
    po, _ = eng.download(want_alloc=False)
    return po.order.copy(), po.total_value.copy()


def test_needs_the_dependency_table(engine):
    (soa, table, deps, fin), (change, table2, dx) = first_two_ticks()
    # plain upload: no table
    engine.upload(soa, table)
    assert raw(engine, change, table2, dx) == L.EVG_ERR_STATE
    assert "dependency table" in L.last_error()
    runnable(engine, table)
    # evg_deps_met_batch after evg_upload_with_deps replaces the staged table
    engine.upload_with_deps(soa, table, None, deps, fin, X.NOW)
    engine.deps_met_batch(deps)
    assert raw(engine, change, table2, dx) == L.EVG_ERR_STATE
    runnable(engine, table)
    # plain evg_edit_tasks drops it
    engine.upload_with_deps(soa, table, None, deps, fin, X.NOW)
    engine.edit_tasks(change[0], table2)
    before = runnable(engine, table2)
    assert raw(engine, change, table2, dx) == L.EVG_ERR_STATE
    after = runnable(engine, table2)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    # evg_update_tasks keeps it (and drops only the verdicts)
    engine.upload_with_deps(soa, table, None, deps, fin, X.NOW)
    engine.update_tasks(np.array([0]), S.TaskSoA(**{n: getattr(soa, n)[:1] for n, _ in S.TaskSoA.COLUMNS}))
    with pytest.raises(L.EvgError):
        engine.download_deps()
    assert raw(engine, change, table2, dx) == L.EVG_OK, L.last_error()
    engine.download_deps()
    runnable(engine, table2)


def test_rejected_inputs(engine):
    (soa, table, deps, fin), (change, table2, dx) = first_two_ticks()
    engine.upload_with_deps(soa, table, None, deps, fin, X.NOW)
    before = runnable(engine, table)
    n_ext = dx.ext_state.shape[0]
    bad_ext = copy.copy(dx)
    bad_ext.depart_ext = np.full_like(dx.depart_ext, n_ext)
    bad_set = copy.copy(dx)
    bad_set.set_row, bad_set.set_state, bad_set.set_pre = np.array([table2.task_off[-1]]), np.zeros(1, np.uint8), np.zeros(1, np.uint8)
    bad_ins = copy.copy(dx)
    bad_ins.insert = S.DepsTable(dx.insert.dep_off[:-1].copy(), dx.insert.dep_kind, dx.insert.dep_ref, dx.insert.dep_want,
                                 dx.insert.task_state[:-1].copy(), dx.insert.task_pre[:-1].copy(), dx.insert.ext_state)
    rows_out = (change[0], np.array([table2.task_off[-1]]), S.TaskSoA(**{n: getattr(change[2], n)[:1] for n, _ in S.TaskSoA.COLUMNS}))
    for ch, x in ((change, bad_ext), (change, bad_set), (change, bad_ins), (rows_out, dx)):
        assert raw(engine, ch, table2, x) == L.EVG_ERR_INVALID, L.last_error()
        after = runnable(engine, table)  # the previous tick, resident and runnable
        assert all(np.array_equal(p, q) for p, q in zip(before, after))
    # a departure marked -1 that a survivor still depends on is found on the device: no tick afterwards
    gone = copy.copy(dx)
    gone.depart_ext = np.full_like(dx.depart_ext, -1)
    assert raw(engine, change, table2, gone) == L.EVG_ERR_INVALID
    assert "depart_ext is -1" in L.last_error()
    assert engine.lib.evg_run_resident(engine.ctx, X.NOW, 0) == L.EVG_ERR_STATE
