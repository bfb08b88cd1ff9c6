"""Every CSR offset table the C boundary takes is checked before anything indexes with it: a table that does not start
at 0, decreases somewhere or misses its end is EVG_ERR_INVALID, and evg_last_error names the entry point and the table.
The row-sized evg_deps_in.dep_off is checked by the first kernel that reads it, every other table on the host."""
import copy
import ctypes as C
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_edit import check_equal, edit, raw_edit
from test_gpu_finder_compaction import candidates
from test_gpu_pipeline_finder import NOW, random_batch

pytestmark = pytest.mark.gpu


def first(off):
    o = off.copy()
    o[0] = 1
    return o


def middle(off):
    o = off.copy()
    k = len(o) // 2
    o[k] = o[k - 1] - 1
    return o


def last(off):
    o = off.copy()
    o[-1] += 1
    return o


ENDED = (first, middle, last)  # a table whose end is a given count
COUNTED = (first, middle)      # a table whose last entry is the count: it has no end to miss


def variant(obj, **kw):
    v = copy.copy(obj)
    for k, x in kw.items():
        setattr(v, k, x)
    return v


def expect_rejected(call, who, name):
    with pytest.raises(L.EvgError) as e:
        call()
    assert e.value.code == L.EVG_ERR_INVALID, str(e.value)
    msg = L.last_error()
    assert who in msg and name in msg, msg


def dag_call(eng, item_off, group_off, dep_off, dep_item, gid, gidx, N, E, G):
    """evg_dag_rebuild_batch with the sizes given apart from the offsets (Engine.dag_rebuild_batch reads them off the ends)."""
    D = int(item_off.shape[0]) - 1
    st = L.DagInStruct(N, E, L.ptr(dep_off), L.ptr(dep_item), L.ptr(gid), L.ptr(gidx))
    outs = [np.zeros(max(n, 1), np.int32) for n in (N, D, D, N, G + D)]
    L.check(eng.lib.evg_dag_rebuild_batch(eng.ctx, C.byref(st), L.ptr(item_off), L.ptr(group_off), D, *[L.ptr(o) for o in outs]))


# ---- per entry point: the call on unmodified input, and (table, its offsets, corruptions, call with other offsets) ----
def upload_cases(eng):
    w = synth.make(np.array([60, 500, 3000]), 901, tg_frac=0.1, n_hosts=20)
    up = lambda t=w.tasks, d=w.distros, h=w.hosts: eng.upload(t, d, h)  # noqa: E731
    return lambda: up(), [
        ("task_off", w.distros.task_off, ENDED, lambda o: up(d=variant(w.distros, task_off=o))),
        ("group_off", w.distros.group_off, COUNTED, lambda o: up(d=variant(w.distros, group_off=o))),
        ("host_off", w.hosts.host_off, ENDED, lambda o: up(h=variant(w.hosts, host_off=o))),
    ]


def alloc_cases(eng):
    w = synth.make(np.array([60, 500, 3000]), 902, tg_frac=0.1, n_hosts=20)
    po = eng.plan_batch(w.tasks, w.distros, w.now)
    info, ginfo = po.info.copy(), po.group_info.copy()
    alloc = lambda h=w.hosts, g=w.distros.group_off: eng.alloc_batch(h, info, ginfo.copy(), g, w.now)  # noqa: E731
    return lambda: alloc(), [
        ("group_off", w.distros.group_off, COUNTED, lambda o: alloc(g=o)),
        ("host_off", w.hosts.host_off, ENDED, lambda o: alloc(h=variant(w.hosts, host_off=o))),
    ]


def deps_met_cases(eng):
    _, table, _ = candidates([300, 2000, 40], 903, "legacy")
    return lambda: eng.deps_met_batch(table.deps), [
        ("deps->dep_off", table.deps.dep_off, ENDED, lambda o: eng.deps_met_batch(variant(table.deps, dep_off=o))),
    ]


def upload_with_deps_cases(eng):
    w, table, fin = candidates([300, 2000, 40], 904, "legacy")
    up = lambda d=table.deps: eng.upload_with_deps(w.tasks, w.distros, w.hosts, d, fin, w.now)  # noqa: E731
    return lambda: up(), [("deps->dep_off", table.deps.dep_off, ENDED, lambda o: up(variant(table.deps, dep_off=o)))]


def finder_cases(table, call):
    return [
        ("task_off", table.task_off, ENDED, lambda o: call(variant(table, task_off=o))),
        ("valid_off", table.valid_off, COUNTED, lambda o: call(variant(table, valid_off=o))),
        ("deps->dep_off", table.deps.dep_off, ENDED, lambda o: call(variant(table, deps=variant(table.deps, dep_off=o)))),
    ]


def find_runnable_batch_cases(eng):
    _, table, _ = candidates([300, 2000, 40], 905, "mixed")
    return lambda: eng.find_runnable_batch(table), finder_cases(table, eng.find_runnable_batch)


def pipeline_tick(seed):
    batch, refs, db = random_batch(random.Random(seed), [40, 600, 90], planner=True)
    table = S.marshal_runnable(batch, refs, "pipeline", db)
    soa, dtable, _ = S.marshal_tasks(batch, NOW, db)
    return table, soa, dtable, S.marshal_dep_finished(batch)


def find_runnable_ex_cases(eng):
    table, _, _, _ = pipeline_tick(906)
    return lambda: eng.find_runnable_batch(table), finder_cases(table, eng.find_runnable_batch)


def plan_from_finder_cases(eng):
    w, table, fin = candidates([300, 2000, 40], 907, "mixed")
    plan = lambda tb=table, t=w.tasks, d=w.distros, h=w.hosts: eng.plan_from_finder(tb, t, d, h, fin, w.now)  # noqa: E731
    return lambda: plan(), finder_cases(table, lambda tb: plan(tb=tb)) + [
        ("candidates->dep_off", w.tasks.dep_off, ENDED, lambda o: plan(t=variant(w.tasks, dep_off=o))),
        ("group_off", w.distros.group_off, COUNTED, lambda o: plan(d=variant(w.distros, group_off=o))),
        ("host_off", w.hosts.host_off, ENDED, lambda o: plan(h=variant(w.hosts, host_off=o))),
    ]


def plan_from_finder_ex_cases(eng):
    table, soa, dtable, fin = pipeline_tick(908)
    plan = lambda tb=table, t=soa: eng.plan_from_finder(tb, t, dtable, None, fin, NOW)  # noqa: E731
    return lambda: plan(), finder_cases(table, lambda tb: plan(tb=tb)) + [
        ("candidates->dep_off", soa.dep_off, ENDED, lambda o: plan(t=variant(soa, dep_off=o))),
    ]


def alias_cases(eng):
    w = synth.make(np.array([60, 500, 3000]), 909, tg_frac=0.1, met_dep_frac=0.05, unmet_dep_frac=0.03, includes_dependencies=True)
    at, cfg = synth.make_aliases(w, 909, name_frac=0.7)
    plan = lambda a=at: eng.plan_aliases(a, cfg, w.now)  # noqa: E731
    return lambda: plan(), [
        ("secondary_off", at.secondary_off, COUNTED, lambda o: plan(variant(at, secondary_off=o))),
        ("dest_off", at.dest_off, COUNTED, lambda o: plan(variant(at, dest_off=o))),
        ("tasks.dep_off", at.tasks.dep_off, ENDED, lambda o: plan(variant(at, tasks=variant(at.tasks, dep_off=o)))),
        ("deps->dep_off", at.deps.dep_off, ENDED, lambda o: plan(variant(at, deps=variant(at.deps, dep_off=o)))),
    ]


def durations_cases(eng):
    w = synth.make(np.array([40, 700, 3000]), 910, tg_frac=0.1, n_hosts=50)
    dw = synth.make_duration_cache(w, 910, n_rows=20_000, n_keys=300)
    eng.upload(w.tasks, w.distros, w.hosts)
    resolve = lambda h=dw.history: eng.resolve_durations(h, w.now, dw.tasks)  # noqa: E731
    return lambda: resolve(), [
        ("pair_key_off", dw.history.pair_key_off, ENDED, lambda o: resolve(variant(dw.history, pair_key_off=o))),
    ]


def legacy_cases(eng):
    off = np.array([0, 7, 30, 31], np.int64)
    T, D = int(off[-1]), len(off) - 1
    cols = {name: np.zeros(T, dt) for name, dt in S.LegacyTable.COLUMNS}
    cols["tg_rank"][:], cols["tg_pair_id"][:] = -1, -1  # no task groups
    table = S.LegacyTable(**cols, task_off=off, list_mode=np.zeros(3 * D, np.uint8))
    return lambda: eng.prioritize_legacy_batch(table), [
        ("task_off", off, ENDED, lambda o: eng.prioritize_legacy_batch(variant(table, task_off=o))),
    ]


def dag_cases(eng):
    rng = np.random.default_rng(911)
    lens, groups = np.array([5, 8, 7]), np.array([2, 0, 3])
    item_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    group_off = np.concatenate([[0], np.cumsum(groups)]).astype(np.int64)
    d_of = np.repeat(np.arange(3), lens)
    N, G = int(item_off[-1]), int(group_off[-1])
    dep_off = np.concatenate([[0], np.cumsum(rng.integers(0, 3, N))]).astype(np.int64)
    E = int(dep_off[-1])
    owner = np.repeat(np.arange(N), np.diff(dep_off))
    dep_item = (rng.random(E) * lens[d_of[owner]]).astype(np.int32)
    gid = np.where(rng.random(N) < 0.6, (rng.random(N) * groups[d_of]).astype(np.int32), -1)
    gid = np.where(groups[d_of] > 0, gid, -1).astype(np.int32)
    gidx = rng.integers(0, 4, N).astype(np.int32)
    dag = lambda io=item_off, go=group_off, do=dep_off: dag_call(eng, io, go, do, dep_item, gid, gidx, N, E, G)  # noqa: E731
    return lambda: dag(), [
        ("item_off", item_off, ENDED, lambda o: dag(io=o)),
        ("group_off", group_off, COUNTED, lambda o: dag(go=o)),
        ("dep_off", dep_off, ENDED, lambda o: dag(do=o)),
    ]


ENTRIES = {
    "evg_upload": upload_cases,
    "evg_alloc_batch": alloc_cases,
    "evg_deps_met_batch": deps_met_cases,
    "evg_upload_with_deps": upload_with_deps_cases,
    "evg_find_runnable_batch": find_runnable_batch_cases,
    "evg_find_runnable_ex": find_runnable_ex_cases,
    "evg_plan_from_finder": plan_from_finder_cases,
    "evg_plan_from_finder_ex": plan_from_finder_ex_cases,
    "evg_plan_aliases": alias_cases,
    "evg_resolve_durations": durations_cases,
    "evg_prioritize_legacy_batch": legacy_cases,
    "evg_dag_rebuild_batch": dag_cases,
}


@pytest.mark.parametrize("who", sorted(ENTRIES))
def test_malformed_offsets_are_rejected(engine, who):
    good, cases = ENTRIES[who](engine)
    good()  # the unmodified input is accepted
    for name, off, corruptions, call in cases:
        for corrupt in corruptions:
            expect_rejected(lambda: call(corrupt(off)), who, name)
    good()  # and still is after the rejections


@pytest.fixture(scope="module")
def fresh():
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def test_malformed_edit_offsets_leave_the_tick_intact(engine, fresh):
    w = synth.make(np.array([60, 500, 3000]), 912, tg_frac=0.1, unmet_dep_frac=0.03, met_dep_frac=0.02, includes_dependencies=True,
                   n_hosts=20)
    engine.upload(w.tasks, w.distros, w.hosts)
    e = synth.next_tick(w, 5)
    good, nd = e.edit.normalize(), e.workload.distros
    assert good.insert.n_edges > 0
    cases = [
        ("insert_off", good.insert_off, ENDED, lambda o: (variant(good, insert_off=o), nd)),
        ("insert->dep_off", good.insert.dep_off, ENDED, lambda o: (variant(good, insert=variant(good.insert, dep_off=o)), nd)),
        ("task_off", nd.task_off, ENDED, lambda o: (good, variant(nd, task_off=o))),
        ("group_off", nd.group_off, COUNTED, lambda o: (good, variant(nd, group_off=o))),
    ]
    for name, off, corruptions, args in cases:
        for corrupt in corruptions:
            assert raw_edit(engine, *args(corrupt(off))) == L.EVG_ERR_INVALID
            msg = L.last_error()
            assert "evg_edit_tasks" in msg and name in msg, msg
            check_equal(engine, fresh, w)  # the previous tick, still resident and runnable
    edit(engine, e)
    check_equal(engine, fresh, e.workload)
