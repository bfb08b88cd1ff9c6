"""evg_edit_tasks on the device: after every edit the context holds the tick a fresh upload of the composed table
(soa.apply_edit) holds -- order, TotalValue, queue and group info, allocator results, the persisted queue and the
breakdown all equal -- across every route, route changes in both directions, the general path's big units, and the
state and validation rules of the entry point."""
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

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fresh():
    """A second context: uploads the composed table from scratch."""
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


def outputs(eng, w, breakdown):
    eng.run(w.now, L.EVG_OPT_BREAKDOWN if breakdown else 0)
    po, ao = eng.download(want_breakdown=breakdown)
    po = S.PlanOutput(po.order.copy(), po.total_value.copy(), po.info.copy(), po.group_info.copy(),
                      None if po.breakdown is None else po.breakdown.copy())
    ao = None if ao is None else S.AllocOutput(ao.result.copy(), ao.status.copy())
    item_off, items = eng.download_queue(0, w.distros.task_off)
    return po, ao, item_off.copy(), items.copy()


def check_equal(edited, fresh, w, breakdown=False):
    """`edited` holds the edited tick; `fresh` uploads w from scratch; every output must match bit for bit."""
    fresh.upload(w.tasks, w.distros, w.hosts)
    a, b = outputs(edited, w, breakdown), outputs(fresh, w, breakdown)
    for f in ("order", "total_value", "info", "group_info") + (("breakdown",) if breakdown else ()):
        assert np.array_equal(getattr(a[0], f), getattr(b[0], f)), f
    if w.hosts is not None:
        assert np.array_equal(a[1].result, b[1].result) and np.array_equal(a[1].status, b[1].status)
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
    return a


def edit(eng, e):
    w = e.workload
    eng.edit_tasks(e.edit, w.distros, w.hosts)
    if e.rows.shape[0]:
        eng.update_tasks(e.rows, e.values)


SIZES = [1, 20, 32, 33, 700, 1280, 3000, 5120, 9000, 10240, 12288, 14000, 40000]


def test_every_route_six_consecutive_edits(engine, fresh):
    w = synth.make(np.array(SIZES), 501, zipf_priority=True, unmet_dep_frac=0.03, met_dep_frac=0.02, tg_frac=0.1,
                   group_versions_frac=0.3, includes_dependencies=True, n_hosts=200)
    engine.upload(w.tasks, w.distros, w.hosts)
    order = outputs(engine, w, False)[0].order
    for k in range(6):
        e = synth.next_tick(w, 600 + k, order=order)
        assert e.edit.add_edge_task.shape[0] > 0 and e.edit.insert.n_edges > 0
        edit(engine, e)
        w = e.workload
        po, ao, _, _ = check_equal(engine, fresh, w)
        parity.check_against_oracle(w, po, ao)
        order = po.order


def test_edits_without_remaps_keep_dead_slots(engine, fresh):
    w = synth.make(np.array([40, 900, 6000, 13000]), 502, tg_frac=0.15, met_dep_frac=0.05, group_versions_frac=0.5, n_hosts=50)
    engine.upload(w.tasks, w.distros, w.hosts)
    for k in range(3):
        e = synth.next_tick(w, 700 + k, remap=False)
        assert e.edit.group_remap is None and e.edit.version_remap is None
        edit(engine, e)
        w = e.workload
        check_equal(engine, fresh, w, breakdown=True)


def resize(w, delta, seed=0):
    """An edit that removes the last -delta[d] rows of distro d or appends delta[d] lone rows (no group, version 0, no
    edges; copies of the scalars of the distro's first row or of row 0)."""
    t, dt = w.tasks, w.distros
    D = dt.n_distros
    rm, ins_rows, ins_d = [], [], []
    for d in range(D):
        a, b = int(dt.task_off[d]), int(dt.task_off[d + 1])
        if delta[d] < 0:
            rm.extend(range(b + delta[d], b))
        else:
            ins_rows.extend([a if b > a else 0] * delta[d])
            ins_d.extend([d] * delta[d])
    ins_rows = np.array(ins_rows, dtype=np.int64)
    cols = {name: getattr(t, name)[ins_rows].copy() for name, _ in S.TaskSoA.COLUMNS}
    cols["group_id"][:] = -1
    cols["version_id"][:] = 0
    cols["priority"] = (np.arange(ins_rows.shape[0]) * 7 + seed) % 50
    cfg = dt.cfg.copy()
    cfg["n_versions"] = np.maximum(cfg["n_versions"], 1)
    ed = S.TaskEdit(np.array(rm, dtype=np.int64), S.TaskSoA(**cols),
                    np.concatenate([[0], np.cumsum(np.bincount(np.array(ins_d, dtype=np.int64), minlength=D))]).astype(np.int64),
                    np.zeros(0, np.int64), np.zeros(0, np.int32), cfg=cfg).normalize()
    tasks, distros = S.apply_edit(t, dt, ed)
    return ed, synth.Workload(w.name, w.now, tasks, distros, w.hosts)


# k_plan_warp <= 32 < k_plan_cta <64,384> <= 384 < <128,1280> <= 1280 < <256,5120> <= 5120 < <512,10240> <= 10240
# < k_plan_smem<1024,12> <= 12288 < the general path (DESIGN.md §4); narrow distros (no edges, not GroupVersions)
BOUNDS = (32, 384, 1280, 5120, 10240, 12288)


def size_class(n):
    return sum(n > b for b in BOUNDS)


def test_route_crossings_both_directions(engine, fresh):
    low = list(BOUNDS)
    sizes = low + [b + 1 for b in BOUNDS] + [5, 0, 1000]
    w = synth.make(np.array(sizes), 503, zipf_priority=True, tg_frac=0.1, n_hosts=60)
    engine.upload(w.tasks, w.distros, w.hosts)
    check_equal(engine, fresh, w)
    n = len(BOUNDS)
    # up: the lower side gains a row, the upper side loses one; distro of 5 emptied, the empty one filled
    delta = [1] * n + [-1] * n + [-5, 40, 0]
    for step in range(2):
        before = np.diff(w.distros.task_off)
        ed, w = resize(w, delta, step)
        after = np.diff(w.distros.task_off)
        engine.edit_tasks(ed, w.distros, w.hosts)
        check_equal(engine, fresh, w)
        crossed = [size_class(int(x)) != size_class(int(y)) for x, y in zip(before[:2 * n], after[:2 * n])]
        assert all(crossed), (before, after)
        assert (after[2 * n], after[2 * n + 1]) == ((0, 40) if step == 0 else (5, 0))
        delta = [-x for x in delta]
    # the first and the last in-queue edge of the 1000-task distro move it off k_plan_cta and back
    d = 2 * n + 2
    a = int(w.distros.task_off[d])
    row = a + 10
    ed = S.TaskEdit(np.zeros(0, np.int64), None, np.zeros(w.distros.n_distros + 1, np.int64),
                    np.array([row], dtype=np.int64), np.array([3], dtype=np.int32)).normalize()
    tasks, distros = S.apply_edit(w.tasks, w.distros, ed)
    w = synth.Workload(w.name, w.now, tasks, distros, w.hosts)
    engine.edit_tasks(ed, w.distros, w.hosts)
    check_equal(engine, fresh, w)
    ed, w = resize(w, [0] * d + [-990] + [0] * (w.distros.n_distros - d - 1))  # row 10 goes: the last edge with it
    assert w.tasks.n_edges == 0
    engine.edit_tasks(ed, w.distros, w.hosts)
    check_equal(engine, fresh, w)


def test_sparse_class_reroutes_other_distros(engine, fresh, monkeypatch):
    # 64 dependency distros of 1100 tasks: k_plan_smem<256,16>'s class is full; one shrinking below 1025 leaves 63, and the
    # whole class moves to the general path (and back when it grows again)
    monkeypatch.delenv("EVG_SPARSE_CLASS", raising=False)
    w = synth.make(np.full(64, 1100), 504, met_dep_frac=0.05, tg_frac=0.1, n_hosts=64)
    engine.upload(w.tasks, w.distros, w.hosts)
    check_equal(engine, fresh, w)
    for delta in (-100, 100):
        ed, w = resize(w, [delta] + [0] * 63)
        engine.edit_tasks(ed, w.distros, w.hosts)
        check_equal(engine, fresh, w)


def test_general_path_big_units_with_breakdown(engine, fresh):
    sizes = np.array([100000, 13000, 300])
    w = synth.make(sizes, 505, zipf_priority=True, tg_frac=0.1, n_hosts=30)
    t, dt = w.tasks, w.distros
    # distro 0: 10 000 tasks depend on its task 5
    fan = np.arange(6, 100000, 10)[:10000]
    n_dep = np.zeros(t.n_tasks, dtype=np.int64)
    n_dep[fan] = 1
    t.dep_off = np.concatenate([[0], np.cumsum(n_dep)]).astype(np.int64)
    t.dep_idx = np.full(fan.shape[0], 5, dtype=np.int32)
    # distro 1: GroupVersions, ten versions of 1300 tasks (a task group stays in its first member's version)
    b0, b1 = int(dt.task_off[1]), int(dt.task_off[2])
    dt.cfg["group_versions"][1] = 1
    dt.cfg["n_versions"][1] = 10
    ver = (np.arange(b1 - b0) // 1300).astype(np.int32)
    gid = t.group_id[b0:b1]
    for g in np.unique(gid[gid >= 0]):
        m = np.nonzero(gid == g)[0]
        ver[m] = ver[m[0]]
    t.version_id[b0:b1] = ver
    w.tasks.normalize()
    w.distros.normalize()
    engine.upload(w.tasks, w.distros, w.hosts)
    check_equal(engine, fresh, w, breakdown=True)
    # task 5 is dispatched (its unit dissolves, 10 000 edges drop); 200 arrivals join distro 0's task group 0, in its version
    first = int(np.nonzero(t.group_id[:100000] == 0)[0][0])
    I = 200
    ins = S.TaskSoA(**{name: np.repeat(getattr(t, name)[first:first + 1], I) for name, _ in S.TaskSoA.COLUMNS})
    ins.task_group_order = (np.arange(I) % 30 + 1).astype(np.int32)
    ins.priority = (np.arange(I) % 7).astype(np.int32)
    # distro 1: versions 0 and 1 merge (version_remap), the arrivals of distro 2 are lone rows
    nv = dt.cfg["n_versions"].astype(np.int64)
    vremap = np.concatenate([np.arange(nv[0]), [0, 0] + list(range(1, 9)), np.arange(nv[2])]).astype(np.int32)
    cfg = dt.cfg.copy()
    cfg["n_versions"][1] = 9
    ed = S.TaskEdit(np.array([5], dtype=np.int64), ins, np.array([0, I, I, I]), np.zeros(0, np.int64), np.zeros(0, np.int32),
                    version_remap=vremap, cfg=cfg).normalize()
    tasks, distros = S.apply_edit(t, dt, ed)
    w = synth.Workload(w.name, w.now, tasks, distros, w.hosts)
    assert w.tasks.n_edges == 0 and int((tasks.group_id[:100199] == 0).sum()) > 200
    engine.edit_tasks(ed, w.distros, w.hosts)
    po, ao, _, _ = check_equal(engine, fresh, w, breakdown=True)
    ref = parity.check_against_oracle(w, po, ao)
    assert np.array_equal(po.breakdown, ref["breakdown"])


def test_update_tasks_after_an_edit_addresses_the_new_rows(engine, fresh):
    w = synth.make(np.array([300, 2000, 15000]), 506, zipf_priority=True, met_dep_frac=0.05, n_hosts=20)
    engine.upload(w.tasks, w.distros, w.hosts)
    e = synth.next_tick(w, 1, change=0.0)
    engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
    w = e.workload
    rows = np.array([0, 299, w.n_tasks - 1, int(w.distros.task_off[2])], dtype=np.int64)
    for r in rows:
        w.tasks.priority[r] = 99
        w.tasks.expected_ns[r] = 7 * M.HOUR
    engine.update_tasks(rows, S.TaskSoA(**{name: getattr(w.tasks, name)[rows] for name, _ in S.TaskSoA.COLUMNS}))
    check_equal(engine, fresh, w)


def test_edit_after_plan_from_finder_equals_a_fresh_upload(engine, fresh):
    NOWT = synth.NOW_NS
    refs = [M.ProjectRef(id="p", enabled=True)]
    batch = []
    for k, n in enumerate((50, 900, 14000)):
        d = M.Distro(id=f"d{k}")
        batch.append((d, [M.Task(id=f"d{k}-{i}", project="p", version=f"v{i % 5}", build_variant="bv", distro_id=d.id,
                                 status="undispatched", requester=M.REPOTRACKER_VERSION_REQUESTER, priority=i % 4,
                                 expected_duration=(1 + i % 9) * M.MINUTE, activated_time=NOWT - (1 + i) * M.MINUTE,
                                 scheduled_time=NOWT - M.HOUR, task_group="g" if i % 10 == 0 else "", task_group_max_hosts=1,
                                 task_group_order=i % 3) for i in range(n)]))
    # no dependencies: every candidate is kept and its deps-met bit is set without a DependenciesMetTime stamp
    got = scheduler.plan_candidates(copy.deepcopy(batch), refs, NOWT, engine=engine)
    assert [len(r) for r, _ in got] == [len(ts) for _, ts in batch]
    soa, table, _ = S.marshal_tasks(batch, NOWT, resolve_deps=True)
    w = synth.Workload("finder", NOWT, soa, table, None)
    e = synth.next_tick(w, 9)
    edit(engine, e)
    check_equal(engine, fresh, e.workload)


def raw_edit(eng, ed, distros):
    es, keep = ed.normalize().struct()
    ds = distros.struct()
    rc = eng.lib.evg_edit_tasks(eng.ctx, C.byref(es), C.byref(ds), None, None, None)
    del keep
    return rc


def test_state_errors(engine):
    w = synth.make(np.array([100, 40]), 507, n_hosts=4)
    e = synth.next_tick(w, 3)
    # no table
    eng = scheduler.Engine(0)
    try:
        assert raw_edit(eng, e.edit, e.workload.distros) == L.EVG_ERR_STATE
    finally:
        eng.close()
    # after a one-shot call
    engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now)
    assert raw_edit(engine, e.edit, e.workload.distros) == L.EVG_ERR_STATE
    engine.plan_batch(w.tasks, w.distros, w.now)
    assert raw_edit(engine, e.edit, e.workload.distros) == L.EVG_ERR_STATE
    # after evg_upload_device (borrowed columns)
    import torch
    dev = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dtype=dt)])).cuda()
           for name, dt in S.TaskSoA.COLUMNS}
    engine.upload_device({k: v.data_ptr() for k, v in dev.items()}, w.n_tasks, w.distros)
    torch.cuda.synchronize()
    assert raw_edit(engine, e.edit, e.workload.distros) == L.EVG_ERR_STATE
    assert "borrowed" in L.last_error()
    del dev


def test_invalid_edits_leave_the_tick_intact(engine, fresh):
    w = synth.make(np.array([60, 500, 3000]), 508, tg_frac=0.1, met_dep_frac=0.05, n_hosts=20)
    engine.upload(w.tasks, w.distros, w.hosts)
    e = synth.next_tick(w, 4)
    good, nd = e.edit, e.workload.distros

    def variant(**kw):
        v = copy.copy(good)
        for k, x in kw.items():
            setattr(v, k, x)
        return v
    rm = good.remove_rows
    wrong_off = nd.task_off.copy()
    wrong_off[1:] += 1
    other = S.DistroTable(wrong_off, nd.group_off, nd.cfg, nd.group_max_hosts).normalize()
    fewer = S.DistroTable(nd.task_off[:-1], nd.group_off[:-1], nd.cfg[:-1], nd.group_max_hosts).normalize()
    first_insert = int(nd.task_off[1]) - (int(good.insert_off[1]) - int(good.insert_off[0]))  # distro 0's first inserted row
    cases = [
        (variant(remove_rows=rm[::-1].copy()), nd),                                   # descending
        (variant(remove_rows=np.concatenate([rm[:1], rm])), nd),                      # duplicate
        (variant(remove_rows=np.concatenate([rm, [w.n_tasks]])), nd),                 # out of range
        (good, other),                                                                # counts disagree with task_off
        (good, fewer),                                                                # another n_distros
        (variant(add_edge_task=np.array([first_insert]), add_edge_dep=np.array([0], dtype=np.int32)), nd),  # not a survivor
        (variant(add_edge_task=np.array([5, 2]), add_edge_dep=np.array([0, 0], dtype=np.int32)), nd),      # not ascending
    ]
    for ed, dtab in cases:
        assert raw_edit(engine, ed, dtab) == L.EVG_ERR_INVALID, L.last_error()
        check_equal(engine, fresh, w)  # the previous tick, still resident and runnable
    edit(engine, e)
    check_equal(engine, fresh, e.workload)


def go_batches(rng, n_ticks):
    import test_edit_host as H
    batch = H.go_batch(rng, n_distros=3, n_tasks=60)
    out = [batch]
    for k in range(n_ticks - 1):
        batch = H.evolve(rng, batch, k)
        out.append(batch)
    return out


def test_resident_tick_over_five_go_ticks_equals_plan_distros(engine, fresh):
    import random
    NOWT = synth.NOW_NS
    rt = scheduler.ResidentTick(engine)
    n_edits = 0
    for k, batch in enumerate(go_batches(random.Random(31), 5)):
        now = NOWT + k * 15 * M.SECOND
        got = rt.plan(copy.deepcopy(batch), now)
        n_edits += rt.last is not None
        order = {t.id: i for _, ts in rt.canonical(batch) for i, t in enumerate(ts)}  # the canonical order it planned
        want_batch = [(d, sorted(copy.deepcopy(ts), key=lambda t: order[t.id])) for d, ts in batch]
        want = scheduler.plan_distros(want_batch, now, engine=fresh)
        for (gr, gi), (wr, wi) in zip(got, want):
            assert [t.id for t in gr] == [t.id for t in wr]
            assert [t.sorting_value_breakdown.total_value for t in gr] == [t.sorting_value_breakdown.total_value for t in wr]
            for f in ("length", "length_with_dependencies_met", "count_dep_filled_merge_queue_tasks", "expected_duration",
                      "max_duration_threshold", "count_duration_over_threshold", "duration_over_threshold",
                      "count_wait_over_threshold", "secondary_queue"):
                assert getattr(gi, f) == getattr(wi, f), f
            key = lambda infos: sorted((g.name, g.count, g.max_hosts, g.expected_duration, g.count_duration_over_threshold,  # noqa: E731
                                        g.count_wait_over_threshold, g.count_dep_filled_merge_queue_tasks,
                                        g.duration_over_threshold) for g in infos)
            assert key(gi.task_group_infos) == key(wi.task_group_infos)
    assert n_edits >= 3
