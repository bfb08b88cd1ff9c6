"""FindNextTask on the device.  Every golden sequence through evg_find_next_batch (one request per call, the state after
each sequence equal to the golden's); random dispatchers, snapshots and requests against oracle_dispatch, several calls
in a row with 1 .. many requests per distro; evg_find_next_tasks on resident ticks against the host route
(evg_download_queue -> host-built dispatchers -> evg_find_next_batch on a second context) array for array, the tick left
as it was; the state rules and the error contract."""
import copy
import ctypes as C
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle_dispatch as OX
from test_find_next_oracle import CASES, replay

pytestmark = pytest.mark.gpu
Z = M.ZERO_TIME


@pytest.fixture(scope="module")
def other():
    """A second context for the host route: evg_find_next_batch ends the tick of the context it runs on."""
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def queue_of(items):
    return M.TaskQueue(queue=[M.TaskQueueItem(id=it["id"], group=it.get("group", ""), build_variant=it.get("build_variant", ""),
                                              project=it.get("project", ""), version=it.get("version", ""),
                                              group_index=it.get("group_index", 0), group_max_hosts=it.get("group_max_hosts", 0),
                                              dependencies=list(it.get("dependencies", [])), dependencies_met=it.get("dependencies_met", False),
                                              is_dispatched=it.get("is_dispatched", False)) for it in items])


def spec_of(s):
    return None if s is None else M.TaskSpec(s.get("group", ""), s.get("build_variant", ""), s.get("project", ""), s.get("version", ""))


def as_oracle_state(state, names, a=0, g0=0, n=None):
    """A device state slice in oracle_dispatch.Dispatcher.state()'s form."""
    bits = state["item_bits"][a:a + n] if n is not None else state["item_bits"]
    return ([int(b & L.EVG_NS_NODE) for b in bits], [int(bool(b & L.EVG_NS_UNIT)) for b in bits],
            {name: (bool(state["group_deleted"][g0 + g]), int(state["group_running"][g0 + g])) for g, name in enumerate(names)})


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_one_request_per_call(engine, case):
    """The golden's ids and outcomes; and after every request the whole downloaded state equal to the oracle's."""
    svc = scheduler.DAGDispatchService(queue_of(case["items"]), engine)
    o = OX.Dispatcher(copy.deepcopy(case["items"]))

    def state():
        return as_oracle_state(svc.built[2], svc.built[1][0])

    def serve(spec, ami, db):
        it = svc.FindNextTask(spec_of(spec), ami, db)
        got = (None if it is None else it.id, svc.last_outcome)
        assert got == (o.find_next_task(spec, ami, db), o.last_outcome) and state() == o.state()
        return got

    def rebuild(items):
        svc.rebuild(queue_of(items))
        o.rebuild(copy.deepcopy(items))
    replay(case, serve, state, rebuild)


# ---------------------------------------------------------------- random dispatchers against the oracle
def random_items(rng, n, n_groups):
    items = []
    for k in range(n):
        g = rng.randrange(n_groups) if n_groups and rng.random() < 0.6 else -1
        deps = [str(rng.randrange(n)) for _ in range(rng.choice([0, 0, 0, 1, 2]))]
        if deps and rng.random() < 0.2:
            deps.append(deps[0])          # a parallel line
        if rng.random() < 0.05:
            deps.append("absent")
        gmh = rng.choice([0, 1, 1, 2, 3]) if g >= 0 or rng.random() < 0.1 else 0
        items.append({"id": str(k), "group": f"G{g}" if g >= 0 else "", "group_index": rng.randrange(4), "group_max_hosts": gmh,
                      "dependencies": deps, "dependencies_met": rng.random() < 0.8, "is_dispatched": rng.random() < 0.05})
    return items


def random_db(rng, queues, names):
    db = {"versions": {"v0": "s3", "v1": "db"}, "generate_limit": rng.choice([0, -3, 5, 50]), "pending_generate": rng.choice([-1, 0, 3, 40]),
          "max_large_parser": rng.choice([0, -1, 2, 9]), "num_large_parser": rng.choice([-1, 0, 2, 5])}
    return db  # the per-call scalars; tasks and running_hosts are drawn per queue (ids repeat across queues)


def random_doc(rng):
    if rng.random() < 0.04:
        return None
    fin = rng.choice([0, 0, Z, 9])
    return {"start": rng.choice([0, 0, 0, 0, Z, 5]), "finish": fin, "status": rng.choice(["success", "failed", ""]),
            "version": rng.choice(["v0", "v1", "v1", "gone"]), "est_generated": rng.choice([None, 0, 1, 3, 60]),
            "ingest": rng.randrange(100), "deps_met": rng.choice([True, True, True, True, False, None])}


def test_random_dispatchers_against_the_oracle(engine):
    rng = random.Random(2401)
    for trial in range(6):
        sizes = [rng.choice([0, 1, 2, 5, 33, 64, 65, 200, 700]) for _ in range(rng.randrange(1, 9))]
        all_items = [random_items(rng, n, rng.choice([0, 1, 3, 12])) for n in sizes]
        queues = [queue_of(items) for items in all_items]
        oracles = [OX.Dispatcher(copy.deepcopy(items)) for items in all_items]
        built = scheduler.next_dispatchers(queues, engine=engine)
        names = built[1]
        io, go = built[0]["item_off"], built[0]["group_off"]
        handed = 0
        for call in range(4):
            base = random_db(rng, queues, names)
            dbs = []  # one dict per queue (ids repeat across queues); the columns are concatenated per queue
            cols = None
            for d, items in enumerate(all_items):
                db = dict(base, tasks={it["id"]: doc for it in items for doc in [random_doc(rng)] if doc is not None},
                          running_hosts={nm: rng.choice([-1, 0, 0, 1, 2, 5]) for nm in names[d]})
                dbs.append(db)
                c = S.marshal_next_db([[it["id"] for it in items]], [names[d]], db)
                cols = c if cols is None else {k: (np.concatenate([cols[k], c[k]]) if isinstance(c[k], np.ndarray) else c[k]) for k in c}
            requests = []
            for d, items in enumerate(all_items):
                reqs = []
                for _ in range(rng.choice([0, 1, 1, 2, 7, 40]) if call else 1):
                    nm = rng.choice(names[d]) if names[d] and rng.random() < 0.4 else rng.choice(["", "nope___"])
                    spec = M.TaskSpec(nm[:-3]) if nm else None
                    reqs.append((spec, rng.choice([0, Z, 50])))
                requests.append(reqs)
            ids = [[it["id"] for it in items] for items in all_items]
            item, outcome, state = engine.find_next_batch(built[0], cols, S.marshal_next_requests(names, requests), built[2])
            got = scheduler._next_results(ids, requests, item, outcome)
            built = (built[0], names, state)
            for d, reqs in enumerate(requests):
                want = []
                for spec, ami in reqs:
                    o = oracles[d]
                    r = o.find_next_task(None if spec is None else {"group": spec.group}, ami, dbs[d])
                    want.append((r, o.last_outcome))
                assert got[d] == want, (trial, call, d)
                handed += sum(1 for r, _ in want if r is not None)
                assert as_oracle_state(state, names[d], int(io[d]), int(go[d]), int(io[d + 1] - io[d])) == oracles[d].state(), (trial, call, d)
        assert handed > 0


# ---------------------------------------------------------------- chained == host route
def raw_snapshot(rng, N, G):
    """Random evg_next_db columns (any bit pattern the shim could send) and scalars."""
    return {"flags": (rng.integers(0, 256, N).astype(np.uint8) | np.where(rng.random(N) < 0.95, L.EVG_ND_FOUND, 0).astype(np.uint8)),
            "est_generated": rng.choice(np.array([0, 0, 1, 5, 70], np.int32), N), "ingest_ns": rng.integers(0, 100, N).astype(np.int64),
            "running_hosts": rng.choice(np.array([-1, 0, 0, 0, 1, 3], np.int32), G), "generate_limit": int(rng.choice([0, 60])),
            "pending_generate": int(rng.choice([-1, 0, 20])), "max_large_parser": int(rng.choice([0, 3])),
            "num_large_parser": int(rng.choice([-1, 1, 3]))}


def raw_requests(rng, group_off, per_distro):
    D = group_off.shape[0] - 1
    ng = np.diff(group_off)
    counts = np.array([per_distro(d) for d in range(D)], dtype=np.int64)
    req_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    d_of = np.repeat(np.arange(D), counts)
    group = np.where((rng.random(d_of.shape[0]) < 0.4) & (ng[d_of] > 0), (rng.random(d_of.shape[0]) * ng[d_of]).astype(np.int64), -1)
    return req_off, group.astype(np.int32), rng.choice(np.array([0, 0, 50], np.int64), d_of.shape[0])


def host_dispatchers(eng, other, soa, table, cap):
    item_off, items = eng.download_queue(cap, table.task_off)
    item_off, items = item_off.copy(), items.copy()
    D = table.n_distros
    d_of = np.repeat(np.arange(D), np.diff(item_off))
    order = np.zeros(max(soa.n_tasks, 1), dtype=np.int32)
    order[table.task_off[d_of] + np.arange(int(item_off[-1])) - item_off[d_of]] = items["task"]
    io, go, dep_off, dep_item, gid, gidx, _ = S.persisted_dag_input(soa, table, order, cap)
    srt, ns, _, ui, uo = other.dag_rebuild_batch(io, go, dep_off, dep_item, gid, gidx)
    disp = {"item_off": io, "group_off": go, "sorted": srt.copy(), "n_sorted": ns.copy(), "unit_items": ui.copy(), "unit_off": uo.copy(),
            "group_id": gid, "group_max_hosts": items["group_max_hosts"].astype(np.int32),
            "dependencies_met": (items["flags"] & L.EVG_QI_DEPS_MET).astype(np.uint8)}
    return disp, (dep_off, dep_item, gid, gidx)


def tick_snapshot(eng, w):
    po, _ = eng.download(want_alloc=False)
    item_off, items = eng.download_queue(0, w.distros.task_off)
    return [x.copy() for x in (po.order, po.total_value, po.info, po.group_info, item_off, items)]


def serve_both(engine, other, disp, state, db, req):
    a_item, a_out = engine.find_next_tasks(db, req)
    b_item, b_out, state = other.find_next_batch(disp, db, req, state)
    assert np.array_equal(a_item, b_item) and np.array_equal(a_out, b_out)
    got = engine.download_dispatch_state()
    for k in state:
        assert np.array_equal(got[k], state[k]), k
    return a_item, a_out, state


def check_properties(disp, item, outcome, req_off):
    """Size-independent: outcome codes agree with item, items lie in their distro, a handed-out standalone item has
    DependenciesMet."""
    assert np.array_equal(item >= 0, outcome == L.EVG_NEXT_FOUND) and set(np.unique(outcome)) <= {0, 1, 2}
    d_of = np.repeat(np.arange(req_off.shape[0] - 1), np.diff(req_off))
    io = disp["item_off"]
    f = item >= 0
    assert np.all(item[f] < (io[d_of + 1] - io[d_of])[f])
    j = io[d_of[f]] + item[f]
    assert np.all(disp["dependencies_met"][j][disp["group_max_hosts"][j] == 0] == 1)


@pytest.mark.parametrize("cap", [0, 7, 300])
def test_chained_equals_host_route(engine, other, cap):
    rng = np.random.default_rng(2410 + cap)
    w = synth.make(np.array([0, 1, 40, 700, 3000, 12000]), 2411, zipf_priority=True, unmet_dep_frac=0.2, met_dep_frac=0.4, tg_frac=0.3,
                   group_versions_frac=0.3, includes_dependencies=True)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    before = tick_snapshot(engine, w)
    r = engine.rebuild_dispatchers(cap)
    disp, _ = host_dispatchers(engine, other, w.tasks, w.distros, cap)
    assert np.array_equal(r["sorted"], disp["sorted"]) and np.array_equal(r["unit_off"], disp["unit_off"])
    N, G = int(disp["item_off"][-1]), int(disp["group_off"][-1])
    state, found = None, 0
    for call, per in enumerate([lambda d: 1, lambda d: int(rng.integers(0, 4)), lambda d: 150 if d == 5 else 2]):
        db = raw_snapshot(rng, N, G)
        req = raw_requests(rng, disp["group_off"], per)
        item, outcome, state = serve_both(engine, other, disp, state, db, req)
        check_properties(disp, item, outcome, req[0])
        found += int((item >= 0).sum())
        if call == 0:  # between two serves: the dispatchers hold the items as persisted
            rows = np.arange(0, w.n_tasks, 3, dtype=np.int64)
            vals = S.TaskSoA(**{name: getattr(w.tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS})
            vals.flags = vals.flags ^ L.EVG_TF_DEPS_MET
            engine.update_tasks(rows, vals)
            engine.update_tasks(rows, S.TaskSoA(**{name: getattr(w.tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
    assert found > 0
    for x, y in zip(before, tick_snapshot(engine, w)):
        assert np.array_equal(x, y)
    e = synth.next_tick(w, 2412)
    engine.edit_tasks(e.edit, e.workload.distros)  # still allowed


@pytest.mark.parametrize("entry", ["edit_tasks", "plan_aliases"])
def test_chained_equals_host_route_on_other_ticks(engine, other, entry):
    rng = np.random.default_rng(2415)
    w = synth.make(np.array([40, 900, 6000, 300]), 2416, tg_frac=0.2, met_dep_frac=0.2, group_versions_frac=0.5)
    if entry == "edit_tasks":
        engine.upload(w.tasks, w.distros)
        engine.run(w.now)
        e = synth.next_tick(w, 2417, order=engine.download(want_alloc=False)[0].order.copy())
        engine.edit_tasks(e.edit, e.workload.distros)
        if e.rows.shape[0]:
            engine.update_tasks(e.rows, e.values)
        soa, table = e.workload.tasks, e.workload.distros
    else:
        at, cfg = synth.make_aliases(w, 2418, name_frac=0.7)
        engine.plan_aliases(at, cfg, w.now)
        soa, table = S.compose_aliases(at, cfg)[:2]
    engine.run(w.now)
    for cap in (0, 13):
        engine.rebuild_dispatchers(cap)
        disp, _ = host_dispatchers(engine, other, soa, table, cap)
        N, G = int(disp["item_off"][-1]), int(disp["group_off"][-1])
        state = None
        for per in (lambda d: 1, lambda d: int(rng.integers(0, 9))):
            req = raw_requests(rng, disp["group_off"], per)
            item, outcome, state = serve_both(engine, other, disp, state, raw_snapshot(rng, N, G), req)
            check_properties(disp, item, outcome, req[0])


def test_every_queue_empty(engine):
    """A quiet tick: every persisted queue is empty and agents still poll.  Every request ends its walk at once."""
    w = synth.make(np.array([0, 0, 0]), 2419)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    r = engine.rebuild_dispatchers(0)
    assert int(r["item_off"][-1]) == 0 and engine._n_disp == (0, 0)
    db, req = one_request(engine, 0, 0, 3)
    for _ in range(2):
        item, outcome = engine.find_next_tasks(db, req)
        assert item.tolist() == [-1, -1, -1] and outcome.tolist() == [L.EVG_NEXT_NONE] * 3
    st = engine.download_dispatch_state()
    assert st["item_bits"].shape[0] == 0 and st["group_deleted"].shape[0] == 0
    many = (np.array([0, 2, 2, 5], np.int64), np.full(5, -1, np.int32), np.array([0, 50, 0, 0, 50], np.int64))
    item, outcome = engine.find_next_tasks(db, many)
    assert item.tolist() == [-1] * 5 and outcome.tolist() == [L.EVG_NEXT_NONE] * 5
    bad = (many[0], np.array([-1, 0, -1, -1, -1], np.int32), many[2])  # no distro has a group
    assert code(lambda: engine.find_next_tasks(db, bad)) == L.EVG_ERR_INVALID


def oracle_items(disp, arrays, d):
    dep_off, dep_item, gid, gidx = arrays
    lo, hi = int(disp["item_off"][d]), int(disp["item_off"][d + 1])
    return [{"id": str(j - lo), "group": f"G{int(gid[j])}" if gid[j] >= 0 else "", "group_index": int(gidx[j]),
             "group_max_hosts": int(disp["group_max_hosts"][j]), "dependencies_met": bool(disp["dependencies_met"][j]),
             "dependencies": [str(int(x)) if x >= 0 else "absent" for x in dep_item[dep_off[j]:dep_off[j + 1]]]} for j in range(lo, hi)]


def test_many_distros_and_one_long_queue(engine, other):
    """Ragged small distros with one request each and one 10 000-item queue with a few hundred: chained == host route,
    the properties everywhere, the oracle on a sample of distros (clean documents, so every item is reachable)."""
    rng = np.random.default_rng(2420)
    sizes = np.concatenate([[12000, 700], rng.integers(0, 13, 100000)])
    w = synth.make(sizes, 2421, met_dep_frac=0.3, tg_frac=0.3, includes_dependencies=True)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    engine.rebuild_dispatchers(0)
    disp, arrays = host_dispatchers(engine, other, w.tasks, w.distros, 0)
    N, G = int(disp["item_off"][-1]), int(disp["group_off"][-1])
    db = {"flags": np.full(N, L.EVG_ND_FOUND | L.EVG_ND_DEPS_MET_NOW, np.uint8), "est_generated": np.zeros(N, np.int32),
          "ingest_ns": np.zeros(N, np.int64), "running_hosts": np.zeros(G, np.int32), "generate_limit": 0, "pending_generate": 0,
          "max_large_parser": 0, "num_large_parser": 0}
    req = raw_requests(rng, disp["group_off"], lambda d: 300 if d == 0 else 40 if d == 1 else 1)
    item, outcome, state = serve_both(engine, other, disp, None, db, req)
    check_properties(disp, item, outcome, req[0])
    # nothing is handed out twice, outside distros that hold an item with a group and GroupMaxHosts 0 (two copies of IsDispatched)
    d_of = np.repeat(np.arange(sizes.shape[0]), np.diff(req[0]))
    twice = (disp["group_id"] >= 0) & (disp["group_max_hosts"] == 0)
    clean = ~np.isin(d_of, np.unique(np.repeat(np.arange(sizes.shape[0]), np.diff(disp["item_off"]))[twice]))
    pairs = np.stack([d_of[(item >= 0) & clean], item[(item >= 0) & clean]], axis=1)
    assert np.unique(pairs, axis=0).shape[0] == pairs.shape[0] and pairs.shape[0] > 300
    doc = {"start": 0, "finish": 0, "status": "", "version": "", "est_generated": None, "ingest": 0, "deps_met": True}
    for d in [1] + [int(x) for x in rng.integers(2, sizes.shape[0], 60)]:
        items = oracle_items(disp, arrays, d)
        o = OX.Dispatcher(items)
        odb = {"tasks": {it["id"]: doc for it in items}}
        for r in range(int(req[0][d]), int(req[0][d + 1])):
            g = int(req[1][r])
            want = o.find_next_task({"group": f"G{g}"} if g >= 0 else None, int(req[2][r]), odb)
            assert (int(item[r]), int(outcome[r])) == (-1 if want is None else int(want), o.last_outcome), (d, r)


def test_resident_tick_objects(engine):
    tasks = [M.Task(id=f"t{k}", version=f"v{k % 2}", project="p", build_variant="bv", distro_id="d", priority=k % 9,
                    task_group=f"g{k % 3}" if k % 2 == 0 else "", task_group_max_hosts=1 + k % 2, task_group_order=k % 4,
                    status=M.TASK_UNDISPATCHED) for k in range(120)]
    tick = scheduler.ResidentTick(engine)
    (ranked, _), = tick.plan([(M.Distro(id="d"), tasks)], synth.NOW_NS)
    items = [{"id": t.id, "group": t.task_group, "build_variant": t.build_variant, "project": t.project, "version": t.version,
              "group_index": t.task_group_order, "group_max_hosts": t.task_group_max_hosts if t.task_group else 0,
              "dependencies_met": True, "dependencies": []} for t in ranked]
    o = OX.Dispatcher(items)
    doc = {"start": 0, "finish": 0, "status": "", "version": "", "est_generated": None, "ingest": 10, "deps_met": True}
    db = {"tasks": {t.id: doc for t in tasks}}
    spec = M.TaskSpec("g0", "bv", "p", "v0")
    for reqs in ([(None, 0)], [(spec, 0), (None, 5), (spec, Z)], [(None, 0)] * 130):
        (got,), want = tick.find_next_tasks([reqs], db), []
        for s, ami in reqs:
            r = o.find_next_task(None if s is None else {"group": s.group, "build_variant": "bv", "project": "p", "version": s.version}, ami, db)
            want.append((r, o.last_outcome))
        assert got == want
    assert got[-1] == (None, L.EVG_NEXT_NONE)
    (got,), o2 = tick.find_next_tasks([[(None, 0)]], db, rebuild=True), OX.Dispatcher(items)  # a rebuild resets the state
    assert got == [(o2.find_next_task(None, 0, db), L.EVG_NEXT_FOUND)]


# ---------------------------------------------------------------- state rules and errors
def one_request(eng, N, G, D, **over):
    db = dict({"flags": np.full(N, L.EVG_ND_FOUND | L.EVG_ND_DEPS_MET_NOW, np.uint8), "est_generated": np.zeros(N, np.int32),
               "ingest_ns": np.zeros(N, np.int64), "running_hosts": np.zeros(G, np.int32), "generate_limit": 0, "pending_generate": 0,
               "max_large_parser": 0, "num_large_parser": 0}, **{k: v for k, v in over.items() if k not in ("req",)})
    req = over.get("req") or (np.concatenate([[0], np.ones(D, np.int64)]).cumsum().astype(np.int64), np.full(D, -1, np.int32), np.zeros(D, np.int64))
    return db, req


def code(fn):
    try:
        fn()
    except L.EvgError as e:
        return e.code
    return L.EVG_OK


def test_state_rules(engine):
    w = synth.make(np.array([30, 500]), 2430, tg_frac=0.3, met_dep_frac=0.2)
    D = 2
    fresh = scheduler.Engine(0)
    try:
        fresh._n_disp = (0, 0)
        db, req = one_request(fresh, 0, 0, 0)
        assert code(lambda: fresh.find_next_tasks(db, req)) == L.EVG_ERR_STATE and "no resident tick" in L.last_error()
    finally:
        fresh.close()
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    engine._n_disp = (530, 0)
    db, req = one_request(engine, 530, 0, D)
    assert code(lambda: engine.find_next_tasks(db, req)) == L.EVG_ERR_STATE  # before a rebuild
    assert "evg_find_next_tasks: no evg_rebuild_dispatchers" in L.last_error()
    assert code(engine.download_dispatch_state) == L.EVG_ERR_STATE
    r = engine.rebuild_dispatchers(0)
    N, G = engine._n_disp
    db, req = one_request(engine, N, G, D)
    first = [x.copy() for x in engine.find_next_tasks(db, req)]
    second = [x.copy() for x in engine.find_next_tasks(db, req)]  # twice in a row: the state moved on
    assert np.all(first[0] >= 0) and not np.array_equal(first[0], second[0])
    engine.update_tasks(np.zeros(1, np.int64), S.TaskSoA(**{name: getattr(w.tasks, name)[:1] for name, _ in S.TaskSoA.COLUMNS}))
    engine.find_next_tasks(db, req)  # still allowed after evg_update_tasks
    engine.rebuild_dispatchers(0)    # a second rebuild starts from IsDispatched == false
    assert np.array_equal(engine.find_next_tasks(db, req)[0], first[0])
    assert not engine.download_dispatch_state()["item_bits"].sum() == 0
    engine.run(w.now)
    assert code(lambda: engine.find_next_tasks(db, req)) == L.EVG_ERR_STATE  # the run ended the dispatchers
    engine.rebuild_dispatchers(0)
    engine.find_next_tasks(db, req)
    engine.dag_rebuild_batch(np.array([0, 1], np.int64), np.array([0, 0], np.int64), np.array([0, 0], np.int64), np.zeros(0, np.int32),
                             np.array([-1], np.int32), np.array([0], np.int32))  # a one-shot call drops the tick
    assert code(lambda: engine.find_next_tasks(db, req)) == L.EVG_ERR_STATE and "no resident tick" in L.last_error()
    engine.upload(w.tasks, w.distros)  # a new tick has no dispatchers until a run and a rebuild
    assert code(lambda: engine.find_next_tasks(db, req)) == L.EVG_ERR_STATE and "no evg_rebuild_dispatchers" in L.last_error()
    engine.run(w.now)
    engine.rebuild_dispatchers(0)
    other_ctx = scheduler.Engine(0)
    try:  # the stateless call ends the tick of the context it runs on, and only that one
        q = queue_of([{"id": "a", "dependencies_met": True}])
        scheduler.find_next_tasks([q], [[(None, 0)]], {"tasks": {}}, engine=other_ctx)
        engine.find_next_tasks(db, req)
        scheduler.find_next_tasks([q], [[(None, 0)]], {"tasks": {}}, engine=engine)
        assert code(lambda: engine.find_next_tasks(db, req)) == L.EVG_ERR_STATE
    finally:
        other_ctx.close()
    del r


def test_error_contract(engine):
    w = synth.make(np.array([30, 500]), 2431, tg_frac=0.3)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    engine.rebuild_dispatchers(0)
    N, G = engine._n_disp
    D = 2
    go = engine.rebuild_dispatchers(0)["group_off"].copy()
    db, req = one_request(engine, N, G, D)
    engine.find_next_tasks(db, req)
    state = {k: v.copy() for k, v in engine.download_dispatch_state().items()}
    bad_est = db["est_generated"].copy(); bad_est[3] = -1
    bad_hosts = db["running_hosts"].copy(); bad_hosts[0] = -2
    ng0 = int(go[1] - go[0])
    rejected = [dict(est_generated=bad_est), dict(running_hosts=bad_hosts), dict(pending_generate=-2), dict(num_large_parser=-2),
                dict(flags=db["flags"][:-1]), dict(running_hosts=db["running_hosts"][:-1]),
                dict(req=(req[0], np.array([ng0, -1], np.int32), req[2])), dict(req=(req[0], np.array([-2, -1], np.int32), req[2])),
                dict(req=(np.array([0, 2, 1], np.int64), req[1], req[2])), dict(req=(np.array([1, 1, 2], np.int64), req[1], req[2]))]
    for over in rejected:
        db2, req2 = one_request(engine, N, G, D, **over)
        n_items = db2["flags"].shape[0]
        engine._n_disp = (n_items, db2["running_hosts"].shape[0])
        assert code(lambda: engine.find_next_tasks(db2, req2)) == L.EVG_ERR_INVALID, over.keys()
        assert L.last_error().startswith("evg_find_next_tasks: ")
        engine._n_disp = (N, G)
    # null pointers
    dbs, rs, os_, *_keep = engine._next_args(db, req, N, G)
    assert G > 0
    for st, f in ((dbs, "flags"), (dbs, "est_generated"), (dbs, "ingest_ns"), (dbs, "running_hosts"), (rs, "req_off"), (rs, "group"),
                  (rs, "ami_updated_ns"), (os_, "item"), (os_, "outcome")):
        keep = getattr(st, f)
        setattr(st, f, None)
        assert engine.lib.evg_find_next_tasks(engine.ctx, C.byref(dbs), C.byref(rs), C.byref(os_)) == L.EVG_ERR_INVALID, f
        setattr(st, f, keep)
    for args in ((None, C.byref(rs), C.byref(os_)), (C.byref(dbs), None, C.byref(os_)), (C.byref(dbs), C.byref(rs), None)):
        assert engine.lib.evg_find_next_tasks(engine.ctx, *args) == L.EVG_ERR_INVALID
    assert engine.lib.evg_download_dispatch_state(engine.ctx, None) == L.EVG_ERR_INVALID
    after = engine.download_dispatch_state()  # every rejected call left the state as it was
    for k in state:
        assert np.array_equal(after[k], state[k]), k
    # the stateless call: dispatcher tables that point outside their distro, sizes that disagree
    q = queue_of([{"id": "a", "dependencies_met": True}, {"id": "b", "group": "g", "group_max_hosts": 1, "dependencies_met": True}])
    disp, names, st0 = scheduler.next_dispatchers([q], engine=engine)
    cols = S.marshal_next_db([["a", "b"]], names, {"tasks": {}})
    reqs = S.marshal_next_requests(names, [[(None, 0)]])
    for f, v in (("sorted", 2), ("unit_items", -1), ("group_id", 1), ("n_sorted", 3), ("unit_off", 5)):
        bad = {k: a.copy() for k, a in disp.items()}
        bad[f][-1 if f != "unit_items" else 0] = v
        assert code(lambda: engine.find_next_batch(bad, cols, reqs, st0)) == L.EVG_ERR_INVALID, f
    item, outcome, _ = engine.find_next_batch(disp, cols, reqs, st0)
    assert (int(item[0]), int(outcome[0])) == (-1, L.EVG_NEXT_GAVE_UP)  # no document for "a"
