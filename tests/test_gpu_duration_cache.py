"""evg_resolve_durations on the device: FetchExpectedDuration for a resident tick's tasks and running hosts against the
weekly aggregate -- every golden case, the reference's cases that carry a DurationPrediction, the chain into the
planner and allocator bit for bit on every route, sparse row lists, every entry point a tick can come from, the error
contract, and a scale run against the numpy restatement."""
import copy
import ctypes as C
import random

import numpy as np
import pytest

import golden_loader as G
import oracle_durations as OD
import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle as O

pytestmark = pytest.mark.gpu

GOLD = G.load("duration_cache.json")
FIELDS = ("avg_ns", "std_ns", "value_ns", "pred_std_ns", "collected_ns", "source")
EXPECT = dict(avg_ns="avg", std_ns="std", value_ns="value", pred_std_ns="pred_std", collected_ns="collected", source="source")
SIZES = [1, 20, 32, 33, 700, 1280, 3000, 5120, 9000, 10240, 12288, 14000, 40000]


@pytest.fixture(scope="module")
def fresh():
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def outputs(eng, now, task_off, breakdown=True, alloc=None):
    eng.run(now, L.EVG_OPT_BREAKDOWN if breakdown else 0)
    po, ao = eng.download(want_breakdown=breakdown, want_alloc=alloc)
    po = S.PlanOutput(po.order.copy(), po.total_value.copy(), po.info.copy(), po.group_info.copy(),
                      None if po.breakdown is None else po.breakdown.copy())
    ao = None if ao is None else S.AllocOutput(ao.result.copy(), ao.status.copy())
    item_off, items = eng.download_queue(0, task_off)
    return po, ao, item_off.copy(), items.copy()


def assert_same(a, b):
    for f in ("order", "total_value", "info", "group_info", "breakdown"):
        x, y = getattr(a[0], f), getattr(b[0], f)
        assert (x is None and y is None) or np.array_equal(x, y), f
    if a[1] is not None or b[1] is not None:
        assert np.array_equal(a[1].result, b[1].result) and np.array_equal(a[1].status, b[1].status)
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])


def copy_out(d):
    return {f: np.array(d[f]) for f in FIELDS}


def with_columns(w, texp, hexp=None, hstd=None):
    """w with the planner's expected_ns (and the hosts' expected / std) replaced."""
    t = copy.copy(w.tasks)
    t.expected_ns = np.ascontiguousarray(texp, np.int64)
    h = w.hosts
    if h is not None and hexp is not None:
        h = copy.copy(h)
        h.expected_ns, h.std_ns = np.ascontiguousarray(hexp, np.int64), np.ascontiguousarray(hstd, np.int64)
    return synth.Workload(w.name, w.now, t, w.distros, h)


def garbage(w, seed):
    rng = np.random.default_rng(seed)
    H = w.hosts.n_hosts if w.hosts is not None else 0
    return with_columns(w, rng.integers(-2 ** 62, 2 ** 62, w.n_tasks), rng.integers(-2 ** 40, 2 ** 40, H),
                        rng.integers(-2 ** 40, 2 ** 40, H))


# ---- golden cases -------------------------------------------------------------------------------------------------
def golden_tick():
    """Every golden case as one task of one distro; each case's history under its own project."""
    now = GOLD["now"]
    tasks, finished = [], []
    for i, c in enumerate(GOLD["cases"]):
        t = OD.golden_task(c["task"], f"t{i}")
        t.project = f"case{i}"
        t.activated_time = now - M.HOUR
        tasks.append(t)
        for f in OD.golden_finished(c["finished"], f"c{i}-"):
            f.project = f"case{i}"
            finished.append(f)
    return now, tasks, finished


def test_golden_cases(engine):
    now, tasks, finished = golden_tick()
    soa, table, _ = S.marshal_tasks([(M.Distro(id="d"), tasks)], now, resolve_durations=False)
    soa.expected_ns[:] = -12345
    engine.upload(soa, table)
    hist, codes = S.marshal_duration_history(finished, tasks, now)
    assert (codes <= -2).sum() == 2  # the two empty-name cases go through the pair rule
    engine.resolve_durations(hist, now, S.marshal_duration_cache(tasks, hist))
    got, _ = engine.download_durations()
    for i, c in enumerate(GOLD["cases"]):
        assert {f: int(got[f][i]) for f in FIELDS} == {f: c["expect"][EXPECT[f]] for f in FIELDS}, c["name"]
    # the resolved durations are what the planner reads: the persisted queue carries them
    engine.run(now)
    item_off, items = engine.download_queue(0)
    want = {i: c["expect"]["avg"] for i, c in enumerate(GOLD["cases"])}
    assert {int(it["task"]): int(it["expected_ns"]) for it in items} == want


def test_reference_planner_cases_with_a_prediction(engine, fresh):
    """planner_test.go:466-480 and task_queue_persister_test.go:33-122,203-204 through the device route."""
    kats = G.load("planner_kats.json")
    now, el = kats["now"], kats["elapsed_ns"]
    cases = [c for c in kats["task_lists"] if c["name"] == "TaskList/ExpectedDuration"] + \
        [c for c in kats["queue_infos"] if c["name"].startswith("persister/")]
    assert len(cases) == 3
    for c in cases:
        tasks = [G.make_task(t, now, el) for t in c["tasks"]]
        want = [O.fetch_expected_duration(copy.deepcopy(t), now)[0] for t in tasks]
        if "expected_durations" in c:
            assert want == c["expected_durations"], c["ref"]
        d = M.Distro(id=c.get("distro_id", ""))
        host = scheduler.plan_distros([(d, copy.deepcopy(tasks))], now, engine=fresh)
        dev_tasks = copy.deepcopy(tasks)
        dev = scheduler.plan_distros([(d, dev_tasks)], now, engine=engine, finished_tasks=[])
        assert [t.expected_duration for t in dev_tasks] == want, c["ref"]
        assert [t.id for t in dev[0][0]] == [t.id for t in host[0][0]]
        assert dev[0][1].expected_duration == host[0][1].expected_duration == sum(want)
        if "order" in c:
            assert sorted(dev_tasks, key=lambda t: t.expected_duration, reverse=True)[0].id == c["order"][0]


def test_reference_running_task_scenario(engine, fresh):
    """utilization_based_host_allocator_test.go:1702-1801: the running tasks' cached predictions resolved on the device
    give the allocator the reference's answer."""
    alloc = G.load("allocator_scenarios.json")
    s = next(x for x in alloc["scenarios"] if x["ref"].endswith("1702-1801"))
    now = s["now"]
    data = G.go_allocator_data(s, lambda t, n: (0, 0))
    docs = {}
    for rt in s["running_tasks"]:
        t = M.Task(id=rt["Id"], project=rt.get("Project", ""), build_variant=rt.get("BuildVariant", ""),
                   expected_duration=rt.get("ExpectedDuration", 0), start_time=rt.get("StartTime", M.ZERO_TIME))
        p = rt.get("DurationPrediction", {})
        t.duration_prediction = M.CachedDurationValue(p.get("Value", 0), p.get("StdDev", 0), p.get("TTL", 0),
                                                      p.get("CollectedAt", M.ZERO_TIME))
        docs[t.id] = t
    want = {k: O.fetch_expected_duration(copy.deepcopy(t), now) for k, t in docs.items()}
    # a one-task tick carries the scenario's hosts; only their durations are read back
    hosts = S.marshal_hosts([data], [[]], docs)
    soa, table, _ = S.marshal_tasks([(data.distro, [M.Task(id="q", distro_id=data.distro.id)])], now)
    engine.upload(soa, table, hosts)
    hist, _ = S.marshal_duration_history([], [], now)
    cache, listed = S.marshal_running_cache([data], docs, hist)
    assert cache.rows.tolist() == [0, 1, 2, 3]
    engine.resolve_durations(hist, now, None, cache)
    _, got = engine.download_durations()
    assert [(int(a), int(b)) for a, b in zip(got["avg_ns"], got["std_ns"])] == [want[t.id] for t in listed]
    data.running_tasks = {t.id: M.RunningTaskStats(True, int(got["avg_ns"][i]), int(got["std_ns"][i]), t.start_time)
                          for i, t in enumerate(listed)}
    (n, f, st), = scheduler.allocate_distros([data], now, engine=fresh)
    assert (n, f, st) == (s["expect_new_hosts"], s["expect_free_hosts"], 0), s["ref"]


# ---- the chain, bit for bit -----------------------------------------------------------------------------------------
def chain_workload(seed, **kw):
    w = synth.make(np.array(SIZES), seed, zipf_priority=True, unmet_dep_frac=0.03, met_dep_frac=0.02, tg_frac=0.1,
                   group_versions_frac=0.3, includes_dependencies=True, n_hosts=300, **kw)
    dw = synth.make_duration_cache(w, seed, n_rows=200_000, n_keys=2000)
    return w, dw


def host_route(w, dw):
    t = OD.resolve_np(dw.history.rows, dw.history.pair_key_off, dw.tasks, w.now)
    h = OD.resolve_np(dw.history.rows, dw.history.pair_key_off, dw.hosts, w.now)
    return t, h, with_columns(w, t["avg_ns"], h["avg_ns"], h["std_ns"])


@pytest.mark.parametrize("seed", [901, 902])
def test_chain_every_route_equals_the_host_route(engine, fresh, seed):
    w, dw = chain_workload(seed)
    want_t, want_h, wr = host_route(w, dw)
    assert set(np.unique(want_t["source"]).tolist()) == {0, 1, 2, 3, 4}
    g = garbage(w, seed)
    engine.upload(g.tasks, g.distros, g.hosts)
    engine.resolve_durations(dw.history, w.now, dw.tasks, dw.hosts)
    got_t, got_h = (copy_out(x) for x in engine.download_durations())
    for f in FIELDS:
        assert np.array_equal(got_t[f], want_t[f]), f
        assert np.array_equal(got_h[f], want_h[f]), f
    a = outputs(engine, w.now, w.distros.task_off)
    fresh.upload(wr.tasks, wr.distros, wr.hosts)
    b = outputs(fresh, w.now, w.distros.task_off)
    assert_same(a, b)
    parity.check_against_oracle(wr, a[0], a[1])


def test_sparse_rows(engine, fresh):
    w, dw = chain_workload(903)
    want_t, want_h, wr = host_route(w, dw)
    g = garbage(w, 903)
    # unlisted rows keep their uploaded values
    rows = np.arange(0, w.n_tasks, 3, dtype=np.int64)
    hrows = np.arange(1, w.hosts.n_hosts, 2, dtype=np.int64)
    sub = lambda c, r: S.DurationCache(*[getattr(c, f)[r] for f in L.DURATION_CACHE_COLUMNS], c.key[r], r)  # noqa: E731
    engine.upload(g.tasks, g.distros, g.hosts)
    engine.resolve_durations(dw.history, w.now, sub(dw.tasks, rows), sub(dw.hosts, hrows))
    got_t, got_h = (copy_out(x) for x in engine.download_durations())
    for f in FIELDS:
        assert np.array_equal(got_t[f], want_t[f][rows]) and np.array_equal(got_h[f], want_h[f][hrows]), f
    texp = g.tasks.expected_ns.copy(); texp[rows] = want_t["avg_ns"][rows]
    hexp, hstd = g.hosts.expected_ns.copy(), g.hosts.std_ns.copy()
    hexp[hrows], hstd[hrows] = want_h["avg_ns"][hrows], want_h["std_ns"][hrows]
    ws = with_columns(w, texp, hexp, hstd)
    fresh.upload(ws.tasks, ws.distros, ws.hosts)
    assert_same(outputs(engine, w.now, w.distros.task_off), outputs(fresh, w.now, w.distros.task_off))
    # listing only the stale / backfill rows after the fresh ones were uploaded as cached equals resolving all rows
    fr = want_t["source"] == OD.FRESH
    start = g.tasks.expected_ns.copy(); start[fr] = dw.tasks.value_ns[fr]
    hfr = want_h["source"] == OD.FRESH
    hs0, hd0 = g.hosts.expected_ns.copy(), g.hosts.std_ns.copy()
    hs0[hfr], hd0[hfr] = dw.hosts.value_ns[hfr], dw.hosts.std_ns[hfr]
    w0 = with_columns(w, start, hs0, hd0)
    engine.upload(w0.tasks, w0.distros, w0.hosts)
    st, hst = np.nonzero(~fr)[0].astype(np.int64), np.nonzero(~hfr)[0].astype(np.int64)
    engine.resolve_durations(dw.history, w.now, sub(dw.tasks, st), sub(dw.hosts, hst))
    fresh.upload(wr.tasks, wr.distros, wr.hosts)
    assert_same(outputs(engine, w.now, w.distros.task_off), outputs(fresh, w.now, w.distros.task_off))


# ---- where the tick comes from ---------------------------------------------------------------------------------------
def small_world(seed, n=(40, 700, 13000)):
    w = synth.make(np.array(n), seed, tg_frac=0.1, unmet_dep_frac=0.03, n_hosts=50)
    return w, synth.make_duration_cache(w, seed, n_rows=50_000, n_keys=500)


def test_after_upload_with_deps_and_update_tasks(engine, fresh):
    rng = random.Random(41)
    import test_edit_host as H
    batch = H.go_batch(rng, n_distros=3, n_tasks=200)
    now = synth.NOW_NS
    pairs = [(d, ts) for d, ts in batch]
    soa, table, _ = S.marshal_tasks(pairs, now, resolve_durations=False)
    deps, fin = S.marshal_deps(pairs), S.marshal_dep_finished(pairs)
    engine.upload_with_deps(soa, table, None, deps, fin, now)
    met0, stamp0 = (x.copy() for x in engine.download_deps())
    tasks = [t for _, ts in pairs for t in ts]
    for i, t in enumerate(tasks):
        t.display_name = f"n{i % 7}"
        t.duration_prediction = M.CachedDurationValue(0 if i % 3 else 5 * M.MINUTE, 0, 0, M.ZERO_TIME)
    finished = [M.Task(id=f"f{i}", project="p", build_variant="bv", display_name=f"n{i % 5}", status="success",
                       time_taken=(i + 1) * M.MINUTE, start_time=now - M.HOUR, finish_time=now - M.HOUR + (i + 1) * M.MINUTE)
                for i in range(20)]
    hist, _ = S.marshal_duration_history(finished, tasks, now)
    engine.resolve_durations(hist, now, S.marshal_duration_cache(tasks, hist))
    got, _ = engine.download_durations()
    want = [OD.fetch_expected_duration(t, now, finished)["avg"] for t in tasks]
    assert got["avg_ns"].tolist() == want
    met1, stamp1 = engine.download_deps()
    assert np.array_equal(met0, met1) and np.array_equal(stamp0, stamp1)
    a = outputs(engine, now, table.task_off, alloc=False)
    soa2 = copy.copy(soa); soa2.expected_ns = np.array(want, np.int64)
    fresh.upload_with_deps(soa2, table, None, deps, fin, now)
    assert_same(a, outputs(fresh, now, table.task_off, alloc=False))
    # evg_update_tasks afterwards sets expected_ns of its rows as given
    rows = np.array([0, 5, 17], np.int64)
    vals = S.TaskSoA(**{n: getattr(soa2, n)[rows].copy() for n, _ in S.TaskSoA.COLUMNS})
    vals.expected_ns[:] = [M.HOUR, 2, 3 * M.HOUR]
    engine.update_tasks(rows, vals)
    fresh.update_tasks(rows, vals)
    assert_same(outputs(engine, now, table.task_off, alloc=False), outputs(fresh, now, table.task_off, alloc=False))
    engine.download_durations()  # the rows are the same rows: still available


def test_after_edit_tasks(engine, fresh):
    w, _ = small_world(44)
    engine.upload(w.tasks, w.distros, w.hosts)
    order = outputs(engine, w.now, w.distros.task_off)[0].order
    e = synth.next_tick(w, 45, order=order)
    engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
    if e.rows.shape[0]:
        engine.update_tasks(e.rows, e.values)
    with pytest.raises(L.EvgError) as ex:
        engine.download_durations()
    assert ex.value.code == L.EVG_ERR_STATE
    w2 = e.workload
    dw = synth.make_duration_cache(w2, 46, n_rows=50_000, n_keys=500)
    want_t, want_h, wr = host_route(w2, dw)
    engine.resolve_durations(dw.history, w2.now, dw.tasks, dw.hosts)
    fresh.upload(wr.tasks, wr.distros, wr.hosts)
    assert_same(outputs(engine, w2.now, w2.distros.task_off), outputs(fresh, w2.now, w2.distros.task_off))


def test_after_plan_from_finder_ex_and_plan_aliases(engine, fresh):
    now = synth.NOW_NS
    refs = [M.ProjectRef(id="p", enabled=True)]
    batch = []
    for k, n in enumerate((50, 900, 14000)):
        d = M.Distro(id=f"d{k}", dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
        batch.append((d, [M.Task(id=f"d{k}-{i}", project="p", version=f"v{i % 5}", build_variant="bv", distro_id=d.id,
                                 display_name=f"n{i % 11}", status="undispatched", requester=M.REPOTRACKER_VERSION_REQUESTER,
                                 priority=i % 4, activated_time=now - (1 + i) * M.MINUTE, scheduled_time=now - M.HOUR,
                                 duration_prediction=M.CachedDurationValue(0, 0, 0, M.ZERO_TIME))
                          for i in range(n)]))
    finished = [M.Task(id=f"f{i}", project="p", build_variant="bv", display_name=f"n{i % 9}", status="success",
                       time_taken=(i % 13 + 1) * M.MINUTE, start_time=now - 2 * M.HOUR, finish_time=now - M.HOUR)
                for i in range(60)]
    table = S.marshal_runnable(batch, refs, "pipeline")
    if table.deps is None:
        table.deps = S.marshal_deps(batch)
    cand, dtab, _ = S.marshal_tasks(batch, now, resolve_durations=False)
    runnable, count = engine.plan_from_finder(table, cand, dtab, None, S.marshal_dep_finished(batch), now)
    assert table.pipe is not None  # evg_plan_from_finder_ex
    kept = [[ts[int(j)] for j in runnable[int(table.task_off[d]):int(table.task_off[d]) + int(count[d])]]
            for d, (_, ts) in enumerate(batch)]
    tasks = [t for ks in kept for t in ks]
    assert len(tasks) == engine._n_tasks > 0
    hist, _ = S.marshal_duration_history(finished, tasks, now)
    engine.resolve_durations(hist, now, S.marshal_duration_cache(tasks, hist))
    got, _ = engine.download_durations()
    assert got["avg_ns"].tolist() == [OD.fetch_expected_duration(t, now, finished)["avg"] for t in tasks]
    # alias queues: the rows are the alias rows
    w, _ = small_world(47, n=(30, 600, 2000))
    at, cfg = synth.make_aliases(w, 47)
    task_off, _, _ = engine.plan_aliases(at, cfg, w.now)
    src, _ = engine.download_alias_map()
    src = src.copy()
    n = int(task_off[-1])
    dw = synth.make_duration_cache(w, 48, n_rows=20_000, n_keys=300)
    cache = S.DurationCache(*[getattr(dw.tasks, f)[src] for f in L.DURATION_CACHE_COLUMNS], dw.tasks.key[src])
    engine.resolve_durations(dw.history, w.now, cache)
    with pytest.raises(L.EvgError) as ex:
        engine.resolve_durations(dw.history, w.now, None, dw.hosts)
    assert ex.value.code == L.EVG_ERR_STATE  # an alias tick has no hosts
    got, _ = engine.download_durations()
    want = OD.resolve_np(dw.history.rows, dw.history.pair_key_off, cache, w.now)
    assert np.array_equal(got["avg_ns"][:n], want["avg_ns"])
    assert np.array_equal(engine.download_alias_map()[0], src)
    engine.run(w.now)
    _, items = engine.download_queue(0, task_off)
    base = np.repeat(task_off[:-1], np.minimum(np.diff(task_off), L.EVG_PERSISTED_QUEUE_CAP))
    assert np.array_equal(items["expected_ns"], want["avg_ns"][base + items["task"]])


# ---- errors -------------------------------------------------------------------------------------------------------
def expect_error(code, fn):
    with pytest.raises(L.EvgError) as ex:
        fn()
    assert ex.value.code == code, str(ex.value)


def test_state_errors(engine):
    w, dw = small_world(50)
    eng = scheduler.Engine(0)
    try:
        expect_error(L.EVG_ERR_STATE, lambda: eng.resolve_durations(dw.history, w.now, dw.tasks))
        eng.upload(w.tasks, w.distros)
        expect_error(L.EVG_ERR_STATE, lambda: eng.resolve_durations(dw.history, w.now, dw.tasks, dw.hosts))
        eng.resolve_durations(dw.history, w.now, dw.tasks)
        eng.plan_batch(w.tasks, w.distros, w.now)
        expect_error(L.EVG_ERR_STATE, lambda: eng.resolve_durations(dw.history, w.now, dw.tasks))
        expect_error(L.EVG_ERR_STATE, eng.download_durations)
        import torch
        cols = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dt)])).cuda()
                for name, dt in S.TaskSoA.COLUMNS}
        eng.upload_device({k: v.data_ptr() for k, v in cols.items()}, w.n_tasks, w.distros)
        expect_error(L.EVG_ERR_STATE, lambda: eng.resolve_durations(dw.history, w.now, dw.tasks))
        del cols
    finally:
        eng.close()


def test_invalid_calls_leave_the_tick_intact(engine):
    w, dw = small_world(51)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.resolve_durations(dw.history, w.now, dw.tasks, dw.hosts)
    before = outputs(engine, w.now, w.distros.task_off)
    T = w.n_tasks
    sub = lambda c, r: S.DurationCache(*[getattr(c, f)[np.clip(r, 0, c.n_rows - 1)] for f in L.DURATION_CACHE_COLUMNS],  # noqa: E731
                                       c.key[np.clip(r, 0, c.n_rows - 1)], np.asarray(r, np.int64))
    bad_rows = [np.array([3, 2]), np.array([1, 1]), np.array([-1, 4]), np.array([0, T])]
    for r in bad_rows:
        expect_error(L.EVG_ERR_INVALID, lambda: engine.resolve_durations(dw.history, w.now, sub(dw.tasks, r)))
    short = S.DurationCache(*[getattr(dw.tasks, f)[:-1] for f in L.DURATION_CACHE_COLUMNS], dw.tasks.key[:-1])
    expect_error(L.EVG_ERR_INVALID, lambda: engine.resolve_durations(dw.history, w.now, short))
    for off in ([1] + dw.history.pair_key_off[1:].tolist(), dw.history.pair_key_off[:-1].tolist() + [dw.history.rows.n_keys + 1],
                [0, 5, 3] + dw.history.pair_key_off[3:].tolist()):
        h = copy.copy(dw.history)
        h.pair_key_off = np.array(off, np.int64)
        expect_error(L.EVG_ERR_INVALID, lambda: engine.resolve_durations(h, w.now, dw.tasks))
    # a null column
    din = L.DurationInStruct()
    cs = dw.tasks.struct()
    cs.ttl_ns = None
    din.tasks = C.pointer(cs)
    assert engine.lib.evg_resolve_durations(engine.ctx, C.byref(din), int(w.now)) == L.EVG_ERR_INVALID
    # keys out of range, found on the device: the staged rows are dropped, the tick is untouched.  The rejected calls
    # carry other inputs (a day later, other cached values) so that a commit that ran would change the plan.
    later = w.now + 24 * M.HOUR

    def other(c):
        c = copy.copy(c)
        c.value_ns, c.std_ns, c.key = c.value_ns + 3 * M.MINUTE, c.std_ns + M.MINUTE, c.key.copy()
        return c
    tasks2, hosts2 = other(dw.tasks), other(dw.hosts)
    for k in (dw.history.rows.n_keys, L.EVG_DK_PAIR(dw.history.n_pairs)):
        c = copy.copy(tasks2)
        c.key = tasks2.key.copy()
        c.key[T // 2] = k
        expect_error(L.EVG_ERR_INVALID, lambda: engine.resolve_durations(dw.history, later, c, hosts2))
        expect_error(L.EVG_ERR_STATE, engine.download_durations)
    h = copy.copy(dw.history)
    h.rows = copy.copy(dw.history.rows)
    h.rows.key = dw.history.rows.key.copy()
    h.rows.key[7] = h.rows.n_keys
    expect_error(L.EVG_ERR_INVALID, lambda: engine.resolve_durations(h, later, tasks2, hosts2))
    assert_same(outputs(engine, w.now, w.distros.task_off), before)
    # the same inputs with valid keys do change the plan: the comparison above could have failed
    engine.resolve_durations(dw.history, later, tasks2, hosts2)
    after = outputs(engine, w.now, w.distros.task_off)
    assert not np.array_equal(after[0].info, before[0].info)
    assert not np.array_equal(after[3], before[3])


def test_empty_row_lists(engine, fresh):
    """An explicit row list that lists nothing resolves nothing (a NULL list would mean every row)."""
    w, dw = small_world(52)
    engine.upload(w.tasks, w.distros, w.hosts)
    empty = lambda c: S.DurationCache(*[getattr(c, f)[:0] for f in L.DURATION_CACHE_COLUMNS], c.key[:0],  # noqa: E731
                                      np.zeros(0, np.int64))
    engine.resolve_durations(dw.history, w.now, empty(dw.tasks), empty(dw.hosts))
    t, h = engine.download_durations()
    assert all(t[f].shape[0] == 0 and h[f].shape[0] == 0 for f in FIELDS)
    fresh.upload(w.tasks, w.distros, w.hosts)
    assert_same(outputs(engine, w.now, w.distros.task_off), outputs(fresh, w.now, w.distros.task_off))


# ---- scale --------------------------------------------------------------------------------------------------------
def test_scale_twenty_million_rows(engine):
    sizes = np.full(200, 100_000)
    w = synth.make(sizes, 77, n_hosts=2000)
    assert w.n_tasks == 2 * 10 ** 7
    dw = synth.make_duration_cache(w, 77, n_rows=10 ** 7, n_keys=10 ** 5)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.resolve_durations(dw.history, w.now, dw.tasks, dw.hosts)
    got_t, got_h = engine.download_durations()
    want_t = OD.resolve_np(dw.history.rows, dw.history.pair_key_off, dw.tasks, w.now)
    want_h = OD.resolve_np(dw.history.rows, dw.history.pair_key_off, dw.hosts, w.now)
    for f in FIELDS:
        assert np.array_equal(got_t[f], want_t[f]), f
        assert np.array_equal(got_h[f], want_h[f]), f
    assert set(np.unique(want_t["source"]).tolist()) == {0, 1, 2, 3, 4}


# ---- the reference-shaped API -----------------------------------------------------------------------------------------
def go_world(seed):
    import test_edit_host as H
    rng = random.Random(seed)
    now = synth.NOW_NS
    batch = H.go_batch(rng, n_distros=3, n_tasks=150)
    for _, ts in batch:
        for t in ts:
            t.display_name = f"n{rng.randrange(6)}"
            t.expected_duration = rng.choice([0, 0, t.expected_duration])
            t.expected_duration_std_dev = rng.choice([0, M.MINUTE])
            t.duration_prediction = M.CachedDurationValue(
                rng.choice([0, 7 * M.MINUTE]), rng.choice([0, M.MINUTE]), rng.choice([0, M.HOUR]),
                rng.choice([M.ZERO_TIME, now - M.MINUTE, now - 9 * M.HOUR, now + M.MINUTE]))
    finished = [M.Task(id=f"f{i}", project="p", build_variant="bv", display_name=f"n{rng.randrange(5)}",
                       status=rng.choice(["success", "failed"]), time_taken=rng.randrange(1, 3600) * 10 ** 9 + rng.randrange(999),
                       start_time=now - 2 * M.HOUR, finish_time=now - M.HOUR) for i in range(80)]
    return now, batch, finished


def fields(t):
    p = t.duration_prediction
    return (t.expected_duration, t.expected_duration_std_dev, p.value, p.std_dev, p.ttl, p.collected_at)


def test_plan_distros_with_finished_tasks_equals_the_host_route(engine, fresh):
    now, batch, finished = go_world(61)
    dev_batch, host_batch = copy.deepcopy(batch), copy.deepcopy(batch)
    got = scheduler.plan_distros(dev_batch, now, engine=engine, finished_tasks=finished)
    stats = O.expected_durations_for_window(finished, now - OD.WINDOW, now)
    hist = {k: (v[1], v[2]) for k, v in stats.items()}
    soa, table, keys = S.marshal_tasks(host_batch, now, None, duration_history=hist)
    scheduler._upload_with_device_deps(fresh, host_batch, soa, table, None, now, None)
    want = scheduler._ranked_results(fresh, host_batch, table, keys, now, True, False)
    for (gr, gi), (wr, wi) in zip(got, want):
        assert [t.id for t in gr] == [t.id for t in wr]
        assert [t.sorting_value_breakdown for t in gr] == [t.sorting_value_breakdown for t in wr]
        assert gi == wi
    for (_, gts), (_, wts) in zip(dev_batch, host_batch):
        assert [fields(t) for t in gts] == [fields(t) for t in wts]
    # without finished_tasks nothing changes
    a, b = copy.deepcopy(batch), copy.deepcopy(batch)
    x = scheduler.plan_distros(a, now, engine=engine)
    y = scheduler.plan_distros(b, now, engine=fresh)
    assert [[t.id for t in r] for r, _ in x] == [[t.id for t in r] for r, _ in y]
    assert [fields(t) for _, ts in a for t in ts] == [fields(t) for _, ts in b for t in ts]


def test_plan_and_allocate_with_running_tasks_equals_the_host_route(engine, fresh):
    now, batch, finished = go_world(62)
    rng = random.Random(62)
    docs, full = {}, []
    for k, (d, ts) in enumerate(batch):
        hosts = []
        for j in range(12):
            h = M.Host(id=f"h{k}-{j}")
            if j % 3:
                tid = f"run{k}-{j}"
                h.running_task = tid
                docs[tid] = M.Task(id=tid, project="p", build_variant="bv", display_name=f"n{rng.randrange(6)}",
                                   start_time=now - rng.randrange(1, 90) * M.MINUTE,
                                   expected_duration=rng.choice([0, 20 * M.MINUTE]),
                                   duration_prediction=M.CachedDurationValue(rng.choice([0, 9 * M.MINUTE]), 0, 0,
                                                                             rng.choice([M.ZERO_TIME, now - M.MINUTE])))
            hosts.append(h)
        d.host_allocator_settings.maximum_hosts = 100
        d.provider = M.PROVIDER_EC2_FLEET
        full.append((d, ts, M.HostAllocatorData(distro=d, existing_hosts=hosts, distro_queue_info=M.DistroQueueInfo())))
    dev = copy.deepcopy(full)
    dev_docs = {}
    for _, _, data in dev:
        for h in data.existing_hosts:
            if h.running_task:
                dev_docs[h.running_task] = copy.deepcopy(docs[h.running_task])
    got = scheduler.plan_and_allocate(dev, now, engine=engine, finished_tasks=finished, running_tasks=dev_docs)
    host = copy.deepcopy(full)
    stats = O.expected_durations_for_window(finished, now - OD.WINDOW, now)
    hist = {k: (v[1], v[2]) for k, v in stats.items()}
    host_docs = copy.deepcopy(docs)
    for _, _, data in host:
        for h in data.existing_hosts:
            if h.running_task:
                t = host_docs[h.running_task]
                avg, std = M.fetch_expected_duration(t, now, hist.get((t.project, t.build_variant, t.display_name)))
                data.running_tasks[t.id] = M.RunningTaskStats(True, avg, std, t.start_time)
    soa, table, keys = S.marshal_tasks([(d, t) for d, t, _ in host], now, None, duration_history=hist)
    hs = S.marshal_hosts([h for _, _, h in host], [k.group_names for k in keys])
    scheduler._upload_with_device_deps(fresh, host, soa, table, hs, now, None)
    fresh.run(now)
    po, ao = fresh.download()
    for i, (r, info, n, f, st) in enumerate(got):
        a, b = int(table.task_off[i]), int(table.task_off[i + 1])
        assert [t.id for t in r] == [host[i][1][int(po.order[k])].id for k in range(a, b)]
        assert (n, f, st) == (int(ao.result[i]["new_hosts"]), int(ao.result[i]["free_hosts"]), int(ao.status[i]))
    assert [fields(t) for _, ts, _ in dev for t in ts] == [fields(t) for _, ts, _ in host for t in ts]
    assert {k: fields(t) for k, t in dev_docs.items()} == {k: fields(t) for k, t in host_docs.items()}


def test_plan_and_allocate_when_no_host_runs_a_listed_task(engine, fresh):
    """running_tasks may hold documents no host of the batch runs (hosts elsewhere, or every host idle by now)."""
    now, batch, finished = go_world(63)
    full = []
    for k, (d, ts) in enumerate(batch):
        hosts = [M.Host(id=f"h{k}-{j}") for j in range(4)] + [M.Host(id=f"h{k}-busy", running_task="not-listed")]
        d.host_allocator_settings.maximum_hosts = 100
        d.provider = M.PROVIDER_EC2_FLEET
        full.append((d, ts, M.HostAllocatorData(distro=d, existing_hosts=hosts, distro_queue_info=M.DistroQueueInfo())))
    running = {"elsewhere": M.Task(id="elsewhere", project="p", build_variant="bv", display_name="n1",
                                   duration_prediction=M.CachedDurationValue(0, 0, 0, M.ZERO_TIME))}
    before = fields(running["elsewhere"])
    got = scheduler.plan_and_allocate(copy.deepcopy(full), now, engine=engine, finished_tasks=finished, running_tasks=running)
    want = scheduler.plan_and_allocate(copy.deepcopy(full), now, engine=fresh, finished_tasks=finished)
    for (gr, gi, gn, gf, gs), (wr, wi, wn, wf, ws) in zip(got, want):
        assert [t.id for t in gr] == [t.id for t in wr] and gi == wi and (gn, gf, gs) == (wn, wf, ws)
    assert fields(running["elsewhere"]) == before


def route_world(seed):
    """Task objects on every planner route (warp, CTA, smem, general; task groups, dependency edges, GroupVersions),
    non-empty display names, hosts with running tasks, and a finished-task history."""
    import test_edit_host as H
    rng = random.Random(seed)
    now = synth.NOW_NS
    full, docs = [], {}
    for k, n in enumerate([1, 20, 33, 700, 3000, 9000, 2000, 14000, 40000]):
        d = M.Distro(id=f"r{k}", provider=M.PROVIDER_EC2_FLEET,
                     dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
        d.planner_settings.group_versions = k == 6
        d.host_allocator_settings.maximum_hosts = 1000
        tasks = [H.go_task(rng, f"r{k}-{i}", d.id) for i in range(n)]
        if k % 2 or k == 6:
            H.link(rng, tasks)
        for t in tasks:
            t.display_name = f"n{rng.randrange(40)}"
            t.expected_duration = rng.choice([0, 0, t.expected_duration])
            t.expected_duration_std_dev = rng.choice([0, M.MINUTE])
            t.duration_prediction = M.CachedDurationValue(
                rng.choice([0, 7 * M.MINUTE]), rng.choice([0, M.MINUTE]), rng.choice([0, M.HOUR]),
                rng.choice([M.ZERO_TIME, now - M.MINUTE, now - 9 * M.HOUR, now + M.MINUTE]))
        hosts = []
        for j in range(30):
            h = M.Host(id=f"h{k}-{j}")
            if j % 3:
                h.running_task = f"run{k}-{j}"
                docs[h.running_task] = M.Task(
                    id=h.running_task, project="p", build_variant="bv", display_name=f"n{rng.randrange(45)}",
                    start_time=now - rng.randrange(1, 90) * M.MINUTE, expected_duration=rng.choice([0, 20 * M.MINUTE]),
                    duration_prediction=M.CachedDurationValue(rng.choice([0, 9 * M.MINUTE]), 0, 0,
                                                              rng.choice([M.ZERO_TIME, now - M.MINUTE])))
            hosts.append(h)
        full.append((d, tasks, M.HostAllocatorData(distro=d, existing_hosts=hosts, distro_queue_info=M.DistroQueueInfo())))
    finished = [M.Task(id=f"f{i}", project="p", build_variant="bv", display_name=f"n{rng.randrange(42)}",
                       status=rng.choice(["success", "failed", "started"]), timed_out=rng.random() < 0.05,
                       time_taken=rng.randrange(1, 3600) * 10 ** 9 + rng.randrange(999),
                       start_time=now - rng.choice([2 * M.HOUR, 8 * 24 * M.HOUR]), finish_time=now - M.HOUR)
                for i in range(3000)]
    return now, full, docs, finished


def test_chain_every_route_equals_the_model_host_route(engine, fresh):
    """The chain on Task objects: garbage durations uploaded, resolved on the device and run, against the host route of
    marshal_tasks(duration_history=...) plus model.fetch_expected_duration for the running tasks."""
    now, full, docs, finished = route_world(71)
    rng = np.random.default_rng(71)
    dev = copy.deepcopy(full)
    pairs, datas = [(d, ts) for d, ts, _ in dev], [h for _, _, h in dev]
    dev_docs = copy.deepcopy(docs)
    soa, table, keys = S.marshal_tasks(pairs, now, resolve_durations=False)
    soa.expected_ns[:] = rng.integers(-2 ** 62, 2 ** 62, soa.n_tasks)
    hosts = S.marshal_hosts(datas, [k.group_names for k in keys], dev_docs)
    hosts.expected_ns[:] = rng.integers(-2 ** 40, 2 ** 40, hosts.n_hosts)
    hosts.std_ns[:] = rng.integers(-2 ** 40, 2 ** 40, hosts.n_hosts)
    scheduler._upload_with_device_deps(engine, pairs, soa, table, hosts, now, None)
    hist, _ = S.marshal_duration_history(finished, (), now)
    tasks = [t for _, ts in pairs for t in ts]
    hcache, listed = S.marshal_running_cache(datas, dev_docs, hist)
    assert hcache.n_rows == 2 * len(full) * 10
    engine.resolve_durations(hist, now, S.marshal_duration_cache(tasks, hist), hcache)
    a = outputs(engine, now, table.task_off)

    host = copy.deepcopy(full)
    stats = O.expected_durations_for_window(finished, now - OD.WINDOW, now)
    hd = {k: (v[1], v[2]) for k, v in stats.items()}
    for _, _, data in host:
        for h in data.existing_hosts:
            if h.running_task:
                t = copy.deepcopy(docs[h.running_task])
                avg, std = M.fetch_expected_duration(t, now, hd.get((t.project, t.build_variant, t.display_name)))
                data.running_tasks[t.id] = M.RunningTaskStats(True, avg, std, t.start_time)
    hpairs = [(d, ts) for d, ts, _ in host]
    hsoa, htable, hkeys = S.marshal_tasks(hpairs, now, None, duration_history=hd)
    hhosts = S.marshal_hosts([h for _, _, h in host], [k.group_names for k in hkeys])
    scheduler._upload_with_device_deps(fresh, hpairs, hsoa, htable, hhosts, now, None)
    b = outputs(fresh, now, htable.task_off)
    assert_same(a, b)
    # the oracle reads the columns as the device left them: the deps-met bit and the stamped wait basis applied
    met, stamp = fresh.download_deps()
    osoa = copy.copy(hsoa)
    osoa.flags = np.where(met & 1, hsoa.flags | L.EVG_TF_DEPS_MET, hsoa.flags & ~np.uint32(L.EVG_TF_DEPS_MET)).astype(np.uint32)
    osoa.wait_basis_ns = np.where((stamp != M.ZERO_TIME) & (stamp > hsoa.wait_basis_ns), stamp, hsoa.wait_basis_ns).astype(np.int64)
    parity.check_against_oracle(synth.Workload("model route", now, osoa, htable, hhosts), b[0], b[1])
