"""evg_download_queue_breakdown and EVG_OPT_QUEUE_BREAKDOWN: the persisted rows carry the full SortingValueBreakdown.
Every row equals the EVG_OPT_BREAKDOWN row at the same rank (and the oracle's, where the parity tests compare one) on
every planner route, at every cap; a run with the option plans exactly what a run without it plans; the rows go through
more than one staging chunk; the state rules; and the Python mirror."""
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
from test_gpu_alias import NOW as ALIAS_NOW, rule_tick
from test_gpu_find_next import one_request
from test_gpu_host_job import job_cfg
from test_gpu_start_estimate import random_table
from test_gpu_intern import pack, random_batch
import test_gpu_tick_state as TS

pytestmark = pytest.mark.gpu

CAPS = (0, 1, 7, 10_000, 1 << 22)  # 0 = the reference's 10 000; the last is above every queue


def snap(engine, w):
    """Every plan output of the last run, copied: order, TotalValue, queue and group infos, the allocator's rows, the
    persisted items."""
    po, ao = engine.download(want_alloc=w.hosts is not None)
    out = [po.order.copy(), po.total_value.copy(), po.info.copy(), po.group_info.copy()]
    if ao is not None:
        out += [ao.result.copy(), ao.status.copy()]
    out += [x.copy() for x in engine.download_queue(0, w.distros.task_off)]
    return out


def same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))


def persisted_ranks(task_off, cap):
    cap = cap or L.EVG_PERSISTED_QUEUE_CAP
    return np.concatenate([np.arange(a, a + min(b - a, cap)) for a, b in zip(task_off[:-1], task_off[1:])] + [np.zeros(0, np.int64)])


def queue_rows(engine, task_off, cap):
    off, bd = engine.download_queue_breakdown(cap, task_off)
    return off.copy(), bd.copy()


def check_tick(engine, w, upload=None, oracle=False, narrow_only=False):
    """Run the resident tick three ways (plain, EVG_OPT_QUEUE_BREAKDOWN, EVG_OPT_BREAKDOWN): the first two plan the same
    bytes (and, on a tick of narrow distros only, launch the same kernels); the queue rows at every cap are the
    EVG_OPT_BREAKDOWN rows at those ranks."""
    (upload or (lambda: engine.upload(w.tasks, w.distros, w.hosts)))()
    task_off = np.asarray(w.distros.task_off, np.int64)
    engine.run(w.now, L.EVG_OPT_BREAKDOWN)
    full, _ = engine.download(want_breakdown=True, want_alloc=False)
    full_bd = full.breakdown.copy()
    if oracle:
        ref = parity.check_against_oracle(w, full, None)
        assert np.array_equal(full_bd, ref["breakdown"])
    engine.run(w.now, 0)
    n_plain = engine.last_launch_count()
    plain = snap(engine, w)
    engine.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
    n_qbd = engine.last_launch_count()
    same(snap(engine, w), plain)
    if narrow_only:
        assert n_qbd == n_plain
    for cap in CAPS:
        off, rows = queue_rows(engine, task_off, cap)
        assert np.array_equal(off, engine.download_queue(cap, task_off)[0])
        r = persisted_ranks(task_off, cap)
        assert np.array_equal(rows, full_bd[r]), cap
        assert np.array_equal(rows[:, L.EVG_BD_TOTAL_VALUE], plain[1][r])
    return full_bd


def narrow(w):
    return all(not int(w.distros.cfg["group_versions"][d]) and
               (w.tasks.n_edges == 0 or w.tasks.dep_off[w.distros.task_off[d + 1]] == w.tasks.dep_off[w.distros.task_off[d]])
               for d in range(w.distros.n_distros))


# ---------------------------------------------------------------------------------------------- every planner route
ROUTES = {
    # k_plan_warp: tiny distros, narrow and complex
    "warp": dict(sizes=lambda rng: rng.integers(400, 0, 32), tg_frac=0.3, group_versions_frac=0.4, unmet_dep_frac=0.08,
                 met_dep_frac=0.05),
    # the three k_plan_cta classes (and the 64-thread instance): task groups only
    "cta": dict(sizes=lambda rng: np.array([300, 1200, 4000, 9000, 200, 5000, 10_000]), tg_frac=0.2),
    # the same with values beyond 32 bits: k_plan_cta hands the distros back to k_plan_smem
    "cta_punted": dict(sizes=lambda rng: np.array([900, 4500, 9500]), tg_frac=0.2, wide=True),
    # the three k_plan_smem classes (GroupVersions / edges), and GroupVersions above kBigUnitTasks in the smallest one
    "smem": dict(sizes=lambda rng: np.array([500, 1000, 3000, 4000, 9000, 12_000, 700, 200]), tg_frac=0.15,
                 group_versions_frac=0.5, unmet_dep_frac=0.04, met_dep_frac=0.03),
    # narrow distros whose tasks are nearly all in task groups
    "smem_many_groups": dict(sizes=lambda rng: np.array([1000, 4000, 11_000]), tg_frac=0.9),
    # the general path: narrow and complex distros
    "general": dict(sizes=lambda rng: np.array([20_000, 13_000, 30_000, 15_000]), tg_frac=0.1, group_versions_frac=0.5,
                    unmet_dep_frac=0.02, met_dep_frac=0.02),
    # every kind mixed, with includes_dependencies
    "mixed": dict(sizes=lambda rng: np.concatenate([[0, 1, 2, 0, 3], rng.integers(60, 1, 3000), [13_000, 0]]), tg_frac=0.2,
                  group_versions_frac=0.3, unmet_dep_frac=0.05, met_dep_frac=0.04, custom_factor_frac=0.5,
                  includes_dependencies=True),
}


def route_tick(name, seed):
    p = dict(ROUTES[name])
    sizes = p.pop("sizes")(synth.Rng(seed))
    wide = p.pop("wide", False)
    w = synth.make(np.asarray(sizes), seed, zipf_priority=True, n_hosts=50, **p)
    if wide:
        for f in ("patch_time_in_queue_factor", "generate_task_factor", "expected_runtime_factor"):
            w.distros.cfg[f] = 100
        w.tasks.priority[::7] = 1000
    return w


@pytest.mark.parametrize("sparse", [None, "0"])
@pytest.mark.parametrize("name", list(ROUTES))
def test_rows_equal_the_breakdown_run_on_every_route(engine, monkeypatch, name, sparse):
    if sparse is not None:
        monkeypatch.setenv("EVG_SPARSE_CLASS", sparse)
    w = route_tick(name, 4100 + list(ROUTES).index(name))
    check_tick(engine, w, oracle=name in ("warp", "mixed", "cta_punted"), narrow_only=narrow(w))


def test_narrow_only_tick_launches_the_same_kernels(engine):
    w = route_tick("cta", 4200)
    assert narrow(w)
    check_tick(engine, w, narrow_only=True)


def test_route_boundaries_against_the_oracle(engine):
    sizes = np.array([32, 33, 1023, 1024, 1025, 4095, 4096, 4097, 12287, 12288, 12289, 1, 0])
    w = synth.make(sizes, 21, zipf_priority=True, tg_frac=0.15, unmet_dep_frac=0.03, met_dep_frac=0.02,
                   custom_factor_frac=0.5, includes_dependencies=True, n_hosts=120, providers=(0.7, 0.2, 0.1))
    check_tick(engine, w, oracle=True)


def test_alias_tick(engine):
    w, _, _ = TS.candidates([300, 2000, 40, 5], 4300, "mixed")
    at, cfg = synth.make_aliases(w, 4301, name_frac=0.7)
    task_off, _, _ = engine.plan_aliases(at, cfg, w.now)
    task_off = np.asarray(task_off, np.int64).copy()
    soa, atab, _, _, _, _ = S.compose_aliases(at, cfg)
    aw = synth.Workload("alias", w.now, soa, atab, None)
    assert np.array_equal(atab.task_off, task_off)
    check_tick(engine, aw, upload=lambda: engine.plan_aliases(at, cfg, w.now))


# ---------------------------------------------------------------------------------------------- chunking
def test_rows_beyond_one_staging_chunk(engine):
    """300 distros of 10 000 tasks: 3 * 10^6 persisted rows, above the 2.58 * 10^6 rows of one 256 MB chunk."""
    w = synth.make(np.full(300, 10_000), 4400, zipf_priority=True, tg_frac=0.1, group_versions_frac=0.1, unmet_dep_frac=0.01)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now, L.EVG_OPT_BREAKDOWN)
    full = engine.download(want_breakdown=True, want_alloc=False)[0].breakdown.copy()
    engine.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
    off, rows = queue_rows(engine, w.distros.task_off, 0)
    assert rows.shape[0] == 3_000_000 > (256 << 20) // (8 * L.EVG_BD_N)
    assert np.array_equal(rows, full)


# ---------------------------------------------------------------------------------------------- state and errors
def raw(engine, cap=0, capacity=1 << 16, D=8):
    off, bd = np.full(D + 1, -7, np.int64), np.full((capacity, L.EVG_BD_N), -7, np.int64)
    rc = engine.lib.evg_download_queue_breakdown(engine.ctx, cap, L.ptr(off), L.ptr(bd), capacity)
    return rc, off, bd


def test_state_errors(engine):
    W = {"w": TS.candidates([300, 2000, 40], 4500, "mixed")[0]}
    W["dw"] = synth.make_duration_cache(W["w"], 4501, n_rows=2000, n_keys=50)
    w = W["w"]
    fresh = scheduler.Engine(0)
    try:
        assert raw(fresh)[0] == L.EVG_ERR_STATE and "no resident tick" in L.last_error()
        fresh.upload(w.tasks, w.distros, w.hosts)
        assert raw(fresh)[0] == L.EVG_ERR_STATE and "evg_download_queue_breakdown" in L.last_error()
    finally:
        fresh.close()
    for then in (lambda: engine.run(w.now, 0),
                 lambda: TS.update(engine, W),
                 lambda: TS.resolve(engine, W),
                 lambda: (lambda e: engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts))(synth.next_tick(w, 4502)),
                 lambda: engine.upload(w.tasks, w.distros, w.hosts),
                 lambda: engine.plan_batch(w.tasks, w.distros, w.now, breakdown=True)):
        engine.upload(w.tasks, w.distros, w.hosts)
        engine.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
        assert raw(engine)[0] == L.EVG_OK
        then()
        assert raw(engine)[0] == L.EVG_ERR_STATE
    # the one-shot calls ignore the bit
    ts, ds = w.tasks.struct(), w.distros.struct()
    ps = L.PlanOutStruct()
    order = np.zeros(w.n_tasks, np.int32)
    ps.order = L.ptr(order)
    assert engine.lib.evg_plan_batch(engine.ctx, C.byref(ts), C.byref(ds), w.now, L.EVG_OPT_QUEUE_BREAKDOWN, C.byref(ps)) == L.EVG_OK
    assert raw(engine)[0] == L.EVG_ERR_STATE


def test_short_capacity_writes_nothing(engine):
    w = synth.make(np.array([30, 500, 20_000]), 4600, tg_frac=0.2, group_versions_frac=0.5)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
    need = 30 + 500 + 10_000
    rc, off, bd = raw(engine, 0, need - 1, D=3)
    assert rc == L.EVG_ERR_INVALID and f"{need} rows needed" in L.last_error()
    assert np.all(off == -7) and np.all(bd == -7)
    rc, off, bd = raw(engine, 0, need, D=3)
    assert rc == L.EVG_OK and off[-1] == need
    assert engine.lib.evg_download_queue_breakdown(engine.ctx, -1, L.ptr(off), L.ptr(bd), need) == L.EVG_ERR_INVALID


def test_rows_survive_the_calls_that_only_read_the_tick(engine):
    D = 3
    w = synth.make(np.array([40, 700, 15_000]), 4700, tg_frac=0.2, group_versions_frac=0.5, met_dep_frac=0.05, n_hosts=60)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now, L.EVG_OPT_QUEUE_BREAKDOWN)
    first = queue_rows(engine, w.distros.task_off, 0)
    rng = np.random.default_rng(4701)

    def dispatch():
        engine.rebuild_dispatchers(0)
        N, G = engine._n_disp
        engine.find_next_tasks(*one_request(engine, N, G, D))

    def host_job():
        engine.host_job(job_cfg(D, 4702, single=0.0, terminate=1.0, hourly=0.0))
        iw = synth.make_idle_hosts(np.array([5, 10, 3]), 4703)
        engine.host_drawdown(S.marshal_idle_hosts(iw.groups), np.asarray(iw.existing, np.int64), iw.now)

    for call in (lambda: engine.download_queue(0, w.distros.task_off),
                 dispatch,
                 host_job,
                 lambda: engine.estimate_start_times(random_table(rng, np.array([2, 5, 33])), w.now, 0, w.distros.task_off),
                 lambda: engine.intern_batch(pack([[("a", "v", "g", 2, []), ("b", "v", "", 0, ["a"])]]))):
        call()
        again = queue_rows(engine, w.distros.task_off, 0)
        for x, y in zip(first, again):
            assert np.array_equal(x, y)


# ---------------------------------------------------------------------------------------------- the Python mirror
def test_persisted_items_carry_the_planned_breakdowns(engine):
    batch = random_batch(4800)
    now = synth.NOW_NS
    got = scheduler.persist_task_queues(copy.deepcopy(batch), now, engine=engine, breakdown=True, cap=300)
    planned = scheduler.plan_distros(copy.deepcopy(batch), now, engine=engine, breakdown=True)
    assert sum(len(q.queue) for q in got) > 600
    for q, (ranked, _) in zip(got, planned):
        assert [it.id for it in q.queue] == [t.id for t in ranked[:300]]
        assert [it.sorting_value_breakdown for it in q.queue] == [t.sorting_value_breakdown for t in ranked[:300]]
    one = scheduler.PersistTaskQueue(*copy.deepcopy(batch[3]), now=now, engine=engine, breakdown=True)
    assert [it.sorting_value_breakdown for it in one.queue] == [t.sorting_value_breakdown for t in planned[3][0]]


def test_persisted_alias_items_carry_the_planned_breakdowns(engine):
    distros, tasks, db = rule_tick()
    now = ALIAS_NOW
    got = scheduler.persist_alias_task_queues(distros, copy.deepcopy(tasks), now, engine=engine, dependency_db=copy.deepcopy(db),
                                              breakdown=True)
    planned = scheduler.plan_alias_queues(distros, copy.deepcopy(tasks), now, engine=engine, dependency_db=copy.deepcopy(db),
                                          breakdown=True)
    default = scheduler.persist_alias_task_queues(distros, copy.deepcopy(tasks), now, engine=engine, dependency_db=copy.deepcopy(db))
    assert [[it.sorting_value_breakdown.row() for it in q.queue] for q in default] == \
        [[[0, t.sorting_value_breakdown.total_value] + [0] * 11 for t in r] for r, _ in planned]
    assert sum(len(q.queue) for q in got) > 0
    for q, (ranked, _) in zip(got, planned):
        assert [it.id for it in q.queue] == [t.id for t in ranked]
        assert [it.sorting_value_breakdown for it in q.queue] == [t.sorting_value_breakdown for t in ranked]
