"""evg_rebuild_dispatchers on the device: the DAG dispatcher of every persisted queue of the resident tick equals the host
route (evg_download_queue -> the persisted queue's dependency CSR and group ids built on the host -> evg_dag_rebuild_batch)
array for array and, at the id level, rebuild_dag_dispatchers over the persisted documents and oracle_dag -- on ticks
from every entry point, at several caps; the tick survives the call; the error contract."""
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
from oracle import oracle_dag as OD

pytestmark = pytest.mark.gpu
FIELDS = L.DISPATCH_OUT_FIELDS


@pytest.fixture(scope="module")
def other():
    """A second context for the host route: evg_dag_rebuild_batch ends the tick of the context it runs on."""
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def device(eng, cap):
    return {k: v.copy() for k, v in eng.rebuild_dispatchers(cap).items()}


def host_route(eng, other, soa, table, cap):
    """evg_download_queue, the persisted queue's CSR and dense group ids in numpy, evg_dag_rebuild_batch."""
    item_off, items = eng.download_queue(cap, table.task_off)
    item_off = item_off.copy()
    D = table.n_distros
    lens = np.diff(item_off)
    d_of = np.repeat(np.arange(D), lens)
    order = np.zeros(max(soa.n_tasks, 1), dtype=np.int32)
    order[table.task_off[d_of] + np.arange(int(item_off[-1])) - item_off[d_of]] = items["task"]
    io, go, dep_off, dep_item, gid, gidx, gslot = S.persisted_dag_input(soa, table, order, cap)
    assert np.array_equal(io, item_off)
    srt, ns, nc, ui, uo = other.dag_rebuild_batch(io, go, dep_off, dep_item, gid, gidx)
    res = {"item_off": io, "sorted": srt.copy(), "n_sorted": ns.copy(), "n_cycles": nc.copy(), "group_off": go,
           "group_slot": gslot, "unit_items": ui.copy(), "unit_off": uo.copy()}
    return res, (dep_off, dep_item, gid, gidx)


def check(eng, other, soa, table, cap, oracle_max=0):
    """Device == host route on every array; distros of at most oracle_max items also against oracle_dag."""
    a = device(eng, cap)
    b, (dep_off, dep_item, gid, gidx) = host_route(eng, other, soa, table, cap)
    for f in FIELDS:
        assert np.array_equal(a[f], b[f]), f
    io, go = a["item_off"], a["group_off"]
    for d in range(table.n_distros):
        lo, hi = int(io[d]), int(io[d + 1])
        if hi - lo > oracle_max:
            continue
        ids = [str(k) for k in range(hi - lo)]
        items = [{"id": ids[j - lo], "group": f"G{int(gid[j])}" if gid[j] >= 0 else "", "group_index": int(gidx[j]),
                  "dependencies": [ids[int(x)] if x >= 0 else "absent" for x in dep_item[dep_off[j]:dep_off[j + 1]]]}
                 for j in range(lo, hi)]
        order, cycles, units = OD.rebuild(items)
        got = [None if x < 0 else ids[int(x)] for x in a["sorted"][lo:lo + int(a["n_sorted"][d])]]
        assert got == order and int(a["n_cycles"][d]) == len(cycles)
        u = int(go[d]) + d
        got_units = {f"G{g}___": [ids[int(x)] for x in a["unit_items"][lo + int(a["unit_off"][u + g]):lo + int(a["unit_off"][u + g + 1])]]
                     for g in range(int(go[d + 1] - go[d]))}
        assert got_units == units
    return a


def with_duplicates(w, seed):
    """w with the first dependency of about one row in eight repeated: parallel lines in the DAG."""
    t = w.tasks
    if not t.n_edges:
        return w
    rng = np.random.default_rng(seed)
    deg = np.diff(t.dep_off)
    dup = (deg > 0) & (rng.random(t.n_tasks) < 0.125)
    lists = [t.dep_idx[t.dep_off[r]:t.dep_off[r + 1]].tolist() for r in range(t.n_tasks)]
    for r in np.nonzero(dup)[0]:
        lists[r].append(lists[r][0])
    t.dep_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    t.dep_idx = np.array([x for lst in lists for x in lst], dtype=np.int32)
    return w


def snapshot(eng, w):
    po, _ = eng.download(want_alloc=False)
    item_off, items = eng.download_queue(0, w.distros.task_off)
    return [x.copy() for x in (po.order, po.total_value, po.info, po.group_info, item_off, items)]


SIZES = [0, 1, 2, 50, 700, 3000, 15000]


def test_random_batches_at_every_cap(engine, other):
    w = with_duplicates(synth.make(np.array(SIZES), 901, zipf_priority=True, unmet_dep_frac=0.3, met_dep_frac=0.6, tg_frac=0.3,
                                   group_versions_frac=0.3, includes_dependencies=True), 902)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    before = snapshot(engine, w)
    caps = [0, 1, 7, 100, 10000, max(SIZES) + 1]
    cycles = truncated_groups = 0
    for cap in caps:
        a = check(engine, other, w.tasks, w.distros, cap, oracle_max=3000 if cap in (0, 100) else 0)
        cycles += int(a["n_cycles"].sum())
        truncated_groups += int(a["group_off"][-1]) < sum(min(int(np.diff(w.distros.group_off)[d]), int(np.diff(a["item_off"])[d]))
                                                          for d in range(w.distros.n_distros))
    assert cycles > 0 and truncated_groups > 0
    for x, y in zip(before, snapshot(engine, w)):
        assert np.array_equal(x, y)


def test_edit_sequence(engine, other):
    w = synth.make(np.array([40, 900, 6000, 13000]), 903, tg_frac=0.15, met_dep_frac=0.2, group_versions_frac=0.3)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    order = engine.download(want_alloc=False)[0].order.copy()
    for k in range(3):
        e = synth.next_tick(w, 904 + k, order=order)
        engine.edit_tasks(e.edit, e.workload.distros)
        if e.rows.shape[0]:
            engine.update_tasks(e.rows, e.values)
        w = e.workload
        engine.run(w.now)
        check(engine, other, w.tasks, w.distros, [0, 7, 500][k])
        order = engine.download(want_alloc=False)[0].order.copy()


def documents(ranked, cap, decode=None):
    """The persisted TaskQueueItems' dispatcher fields of the ranked tasks, as persist_task_queues writes them."""
    head = ranked[:cap or L.EVG_PERSISTED_QUEUE_CAP]
    if decode is not None:
        head = decode(head)
    return M.TaskQueue(queue=[M.TaskQueueItem(id=t.id, group=t.task_group, build_variant=t.build_variant, project=t.project,
                                              version=t.version, group_index=t.task_group_order,
                                              dependencies=[x.task_id for x in t.depends_on]) for t in head])


def same_dispatchers(got, want):
    assert len(got) == len(want)
    for (go, gc, gu), (wo, wc, wu) in zip(got, want):
        assert go == wo and gc == wc and gu == wu


def test_resident_tick_objects(engine, other):
    rnd = random.Random(905)
    tasks = [M.Task(id=f"t{k}", version=f"v{k % 3}", project="p", build_variant="bv", distro_id="d", priority=rnd.randrange(50),
                    task_group=f"g{k % 4}" if k % 3 == 0 else "", task_group_max_hosts=2, task_group_order=k % 5,
                    status=M.TASK_UNDISPATCHED) for k in range(400)]
    for k, t in enumerate(tasks):
        for _ in range(rnd.choice([0, 0, 1, 2])):
            t.depends_on.append(M.Dependency(f"t{rnd.randrange(400)}", M.TASK_SUCCEEDED))
        if k % 11 == 0:
            t.depends_on.append(M.Dependency("gone"))
    distro = M.Distro(id="d")
    tick = scheduler.ResidentTick(engine)
    for step, cap in enumerate((0, 60)):
        batch = [(distro, tasks[step * 40:])]
        res = tick.plan(batch, synth.NOW_NS + step)
        got = tick.dispatchers(cap)
        want = scheduler.rebuild_dag_dispatchers([documents(r, cap) for r, _ in res], engine=other)
        same_dispatchers(got, want)


@pytest.mark.parametrize("finder,version", [("legacy", ""), ("legacy", "revised-with-dependencies"), ("alternate", ""),
                                            ("parallel", ""), ("pipeline", ""), ("pipeline", "revised-with-dependencies")])
def test_plan_candidates_every_finder(engine, other, finder, version):
    import test_gpu_pipeline_finder as PF
    rng = random.Random(906 + len(finder) + len(version))
    batch, refs, db = PF.random_batch(rng, [20, 300, 4000], planner=True, version=version)
    PF.gate_all(refs)
    _, _, keys = S.marshal_tasks(copy.deepcopy(batch), PF.NOW, copy.deepcopy(db))
    ranked = scheduler.plan_candidates(batch, refs, PF.NOW, finder=finder, dependency_db=db, engine=engine)
    for cap in (0, 7):
        got = scheduler.dispatchers_from_tick([[t.id for t in r] for r, _ in ranked], [k.group_names for k in keys], cap=cap,
                                              engine=engine)
        decode = (lambda d: (lambda ts: scheduler.pipeline_returned_tasks(d, ts))) if finder == "pipeline" else (lambda d: None)
        docs = [documents(r, cap, decode(d)) for (d, _), (r, _) in zip(batch, ranked)]
        same_dispatchers(got, scheduler.rebuild_dag_dispatchers(docs, engine=other))
        for q, (order, n_cycles, units) in zip(docs, got):
            if len(q.queue) <= 3000:
                want = OD.rebuild([{"id": it.id, "group": it.group, "build_variant": it.build_variant, "project": it.project,
                                    "version": it.version, "group_index": it.group_index, "dependencies": it.dependencies}
                                   for it in q.queue])
                assert (order, n_cycles, units) == (want[0], len(want[1]), want[2])


def test_alias_queues(engine, other):
    w0 = synth.make(np.array([40, 900, 6000, 300]), 907, tg_frac=0.2, met_dep_frac=0.2, group_versions_frac=0.5)
    at, cfg = synth.make_aliases(w0, 908, name_frac=0.7)
    engine.plan_aliases(at, cfg, w0.now)
    engine.run(w0.now)
    soa, table = S.compose_aliases(at, cfg)[:2]
    for cap in (0, 13):
        check(engine, other, soa, table, cap, oracle_max=3000)
    # Task objects: alias_dispatchers against the documents persist_alias_task_queues saves
    import test_gpu_alias as GA
    distros, tasks, db = GA.rule_tick()
    got = scheduler.alias_dispatchers(distros, copy.deepcopy(tasks), GA.NOW, engine=engine, dependency_db=copy.deepcopy(db))
    docs = scheduler.persist_alias_task_queues(distros, copy.deepcopy(tasks), GA.NOW, engine=other, dependency_db=copy.deepcopy(db))
    same_dispatchers(got, scheduler.rebuild_dag_dispatchers(docs, engine=other))
    assert any(units for _, _, units in got)


def test_upload_device(engine, other):
    import torch
    w = with_duplicates(synth.make(np.array([3, 700, 5000]), 909, tg_frac=0.2, met_dep_frac=0.3), 910)
    dev = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dtype=dt)])).cuda()
           for name, dt in S.TaskSoA.COLUMNS}
    dev["dep_off"] = torch.from_numpy(np.concatenate([w.tasks.dep_off, np.zeros(8, np.int64)])).cuda()
    dev["dep_idx"] = torch.from_numpy(np.concatenate([w.tasks.dep_idx, np.zeros(8, np.int32)])).cuda()
    torch.cuda.synchronize()
    engine.upload_device({k: v.data_ptr() for k, v in dev.items()}, w.n_tasks, w.distros, n_edges=w.tasks.n_edges)
    engine.run(w.now)
    before = {k: v.cpu().numpy().copy() for k, v in dev.items()}
    check(engine, other, w.tasks, w.distros, 0, oracle_max=1000)
    for k, v in dev.items():
        assert np.array_equal(v.cpu().numpy(), before[k]), k  # the adopted columns are only read
    del dev


def test_tick_survives(engine, other):
    w = synth.make(np.array([30, 800, 4000]), 911, tg_frac=0.2, met_dep_frac=0.1, unmet_dep_frac=0.05, n_hosts=30)
    batch = [(M.Distro(id=f"d{d}"), [M.Task(id=f"d{d}-{i}", version="v", priority=i % 7, distro_id=f"d{d}",
                                            task_group="g" if i % 5 == 0 else "", task_group_max_hosts=1,
                                            depends_on=[M.Dependency(f"d{d}-{(i * 7) % n}")] if i % 4 == 0 else [])
                                     for i in range(n)]) for d, n in enumerate((50, 600))]
    soa, table, _ = S.marshal_tasks(batch, w.now)
    deps = S.marshal_deps(batch)
    engine.upload_with_deps(soa, table, None, deps, S.marshal_dep_finished(batch), w.now)
    engine.run(w.now)
    met0 = [x.copy() for x in engine.download_deps()]
    snap0 = snapshot(engine, synth.Workload("deps", w.now, soa, table, None))
    engine.rebuild_dispatchers(0)
    engine.rebuild_dispatchers(3)
    assert all(np.array_equal(x, y) for x, y in zip(met0, engine.download_deps()))
    assert all(np.array_equal(x, y) for x, y in zip(snap0, snapshot(engine, synth.Workload("deps", w.now, soa, table, None))))
    # with hosts: then an edit, a run and a download equal a fresh upload of the composed table
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    engine.rebuild_dispatchers(0)
    e = synth.next_tick(w, 912)
    engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
    if e.rows.shape[0]:
        engine.update_tasks(e.rows, e.values)
    engine.run(w.now)
    a = engine.download()
    a = [a[0].order.copy(), a[0].total_value.copy(), a[0].info.copy(), a[1].result.copy(), a[1].status.copy()]
    other.upload(e.workload.tasks, e.workload.distros, e.workload.hosts)
    other.run(w.now)
    b = other.download()
    for x, y in zip(a, [b[0].order, b[0].total_value, b[0].info, b[1].result, b[1].status]):
        assert np.array_equal(x, y)
    check(engine, other, e.workload.tasks, e.workload.distros, 0)


def raw(eng, cap, items_capacity, groups_capacity, drop=None):
    D = eng._n_distros
    bufs = {"item_off": np.zeros(D + 1, np.int64), "group_off": np.zeros(D + 1, np.int64)}
    for f, n in (("sorted", max(items_capacity, 1)), ("unit_items", max(items_capacity, 1)), ("group_slot", max(groups_capacity, 1)),
                 ("unit_off", groups_capacity + D + 1), ("n_sorted", D + 1), ("n_cycles", D + 1)):
        bufs[f] = np.zeros(n, np.int32)
    st = L.DispatchOutStruct(*[None if f == drop else L.ptr(bufs[f]) for f in FIELDS])
    return eng.lib.evg_rebuild_dispatchers(eng.ctx, int(cap), int(items_capacity), int(groups_capacity), C.byref(st)), bufs


def test_errors(engine, other):
    fresh = scheduler.Engine(0)
    try:
        assert raw(fresh, 0, 10, 10)[0] == L.EVG_ERR_STATE  # no resident tick
    finally:
        fresh.close()
    w = synth.make(np.array([60, 500, 3000]), 913, tg_frac=0.2, met_dep_frac=0.1)
    engine.upload(w.tasks, w.distros)
    engine.run(w.now)
    before = snapshot(engine, w)
    N = int(np.minimum(np.diff(w.distros.task_off), 100).sum())
    g_need = int(np.minimum(np.diff(w.distros.group_off), np.minimum(np.diff(w.distros.task_off), 100)).sum())
    assert raw(engine, -1, N, g_need)[0] == L.EVG_ERR_INVALID
    assert raw(engine, 100, N - 1, g_need)[0] == L.EVG_ERR_INVALID
    assert f"{N} items and {g_need} groups needed" in L.last_error()
    assert raw(engine, 100, N, g_need - 1)[0] == L.EVG_ERR_INVALID
    for f in FIELDS:
        assert raw(engine, 100, N, g_need, drop=f)[0] == L.EVG_ERR_INVALID, f
    rc, bufs = raw(engine, 100, N, g_need)  # the needed sizes suffice
    assert rc == L.EVG_OK
    for x, y in zip(before, snapshot(engine, w)):
        assert np.array_equal(x, y)
    check(engine, other, w.tasks, w.distros, 100)
    assert np.array_equal(bufs["sorted"][:N], engine.rebuild_dispatchers(100)["sorted"])
