"""Task start-time estimates on the device: evg_estimate_start_batch equals the CPU restatement's fresh run bit for bit on
every golden case and on random batches (every pool size around the warp width and the shared-memory limit, every host
kind, wrapping values); evg_estimate_start_times, chained on ticks from every entry point at several caps, equals
evg_download_queue + evg_estimate_start_batch array for array and leaves the tick as it found it; both at size; the
error contract."""
import copy
import ctypes as C
import json
import os

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle_estimate as OE
from test_gpu_find_next import raw_requests, raw_snapshot
from test_gpu_finder_compaction import candidates

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "task_start_estimation.json")))
NOW = synth.NOW_NS
MAX, MIN = 2 ** 63 - 1, -(2 ** 63)
LIMIT = L.EVG_EST_ONCHIP_HOSTS
FIXED = {L.EVG_EH_UNINITIALIZED: 4 * OE.MINUTE, L.EVG_EH_STARTING: 3 * OE.MINUTE, L.EVG_EH_PROVISIONING: OE.MINUTE, L.EVG_EH_FREE: 0}


@pytest.fixture(scope="module")
def eng():
    e = scheduler.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def other():
    e = scheduler.Engine(0)
    yield e
    e.close()


def table_of(pools):
    """A host table whose rows have exactly these timeToCompletion values: running hosts dispatched at NOW."""
    flat = [v for p in pools for v in p]
    off = np.concatenate([[0], np.cumsum([len(p) for p in pools])]).astype(np.int64)
    return S.EstHostTable(np.full(len(flat), L.EVG_EH_RUNNING, np.uint8), np.array(flat, dtype=np.int64), np.full(len(flat), NOW, np.int64), off)


def random_table(rng, counts, span=3600 * 10 ** 9):
    """Every kind; a running task's elapsed time reaches twice its expected duration, so about half of them overrun."""
    H = int(np.sum(counts))
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return S.EstHostTable(rng.integers(0, 6, H).astype(np.uint8), rng.integers(0, span, H), NOW - rng.integers(0, 2 * span, H), off)


def pools_of(table, now):
    """createSimulatorModel's pool of every distro, from the table's rows."""
    out = []
    for d in range(table.n_distros):
        p = []
        for i in range(int(table.est_host_off[d]), int(table.est_host_off[d + 1])):
            k = int(table.kind[i])
            if k == L.EVG_EH_RUNNING:
                p.append(OE.wrap(int(table.expected_ns[i]) - OE.since(now, int(table.dispatch_ns[i]))))
            elif k != L.EVG_EH_IGNORED:
                p.append(FIXED[k])
        out.append(p)
    return out


def fresh(durations, pool):
    """oracle_estimate.fresh_estimates; above 64 hosts the same statements on a numpy pool (checked against it below)."""
    if len(pool) <= 64 or len(durations) == 0:
        return OE.fresh_estimates(durations, pool)
    p = np.sort(np.array(pool, dtype=np.int64))
    elapsed, out = 0, []
    for d in durations:
        ff = p[0]
        elapsed = OE.wrap(elapsed + int(ff))
        p = p[1:] - ff  # array arithmetic wraps
        hit = (p[:-1] <= d) & (p[1:] >= d)  # the pairs i < count - 2 are all the adjacent pairs of the hosts left
        k = int(np.argmax(hit)) if hit.any() else len(p)
        p = np.insert(p, k, d)
        out.append(elapsed)
    return out


def expect(durations, item_off, pools):
    out = []
    for d, p in enumerate(pools):
        out.extend(fresh([int(x) for x in durations[int(item_off[d]):int(item_off[d + 1])]], p))
    return np.array(out, dtype=np.int64), np.array([len(p) for p in pools], dtype=np.int32)


def batch(eng, queues, table, now=NOW):
    off = np.concatenate([[0], np.cumsum([len(q) for q in queues])]).astype(np.int64)
    dur = np.array([v for q in queues for v in q], dtype=np.int64)
    start, used = eng.estimate_start_batch(dur, off, table, now)
    return dur, off, start.copy(), used.copy()


def test_numpy_restatement_equals_the_oracle():
    rng = np.random.default_rng(7200)
    for m in (65, 70, 200):
        for span in (100, 2 ** 62):
            pool, dur = rng.integers(-span, span, m).tolist(), rng.integers(-span, span, 300).tolist()
            assert fresh(dur, pool) == OE.fresh_estimates(dur, pool)


def test_every_golden_case_in_one_batch(eng):
    cases = GOLDEN["cases"]
    dur, off, start, used = batch(eng, [c["tasks"] for c in cases], table_of([c["hosts"] for c in cases]))
    for d, c in enumerate(cases):
        want = OE.fresh_estimates(c["tasks"], c["hosts"])
        assert start[int(off[d]):int(off[d + 1])].tolist() == want, c["name"]
        assert c.get("fresh", want) == want and int(used[d]) == len(c["hosts"]), c["name"]


def test_golden_models_through_the_marshaller(eng):
    for m in GOLDEN["models"]:
        hosts = [M.Host(status=h["status"], running_task=h["running_task"]) for h in m["hosts"]]
        running = {k: S.TASK_LOOKUP_ERROR if v == "error" else None if v is None else M.Task(id=k, **v) for k, v in m["running"].items()}
        queue = M.TaskQueue(distro="d", queue=[M.TaskQueueItem(id=str(i), expected_duration=v) for i, v in enumerate(m["queue"])])
        got = scheduler.estimated_start_times([queue, None], [hosts, hosts], running, m["now"], engine=eng)
        assert got == [OE.fresh_estimates(m["queue"], m["expect"]), []], m["name"]
        last = scheduler.get_estimated_start_time(M.Task(id=str(len(m["queue"]) - 1)), queue, hosts, running, m["now"], engine=eng)
        assert last == got[0][-1]


POOLS = [0, 1, 2, 3, 31, 32, 33, 34, 64, 65, LIMIT - 1, LIMIT, LIMIT + 1, LIMIT + 2, 2500]


def durations_of(rng, mode, n):
    if mode == "equal":
        return [int(rng.integers(0, 10 ** 12))] * n
    if mode == "zero":
        return [0] * n
    if mode == "negative":
        return rng.integers(-10 ** 12, 10 ** 9, n).tolist()
    if mode == "huge":
        return rng.choice(np.array([MAX, MAX - 7, MIN, MIN + 3, 2 ** 62, -(2 ** 62), 0, 5], dtype=np.int64), n).tolist()
    return rng.integers(0, 7200 * 10 ** 9, n).tolist()


@pytest.mark.parametrize("mode", ["random", "equal", "zero", "negative", "huge"])
def test_random_batches_against_the_oracle(eng, mode):
    rng = np.random.default_rng(7300 + len(mode))
    counts, queues = [], []
    for m in POOLS:
        for n in (0, 1, 2, 40, 333):
            counts.append(m)
            queues.append(durations_of(rng, mode, n))
    table = random_table(rng, counts)
    if mode == "huge":  # timeToCompletion near both ends of int64: the elapsed time and the stored offsets wrap
        table.expected_ns = rng.choice(np.array([MAX, MAX - 1, MIN, MIN + 1, 2 ** 62, 1], dtype=np.int64), table.n_hosts)
        table.dispatch_ns = np.where(rng.random(table.n_hosts) < 0.1, M.ZERO_TIME, NOW - rng.integers(-5, 5, table.n_hosts))
    assert set(table.kind.tolist()) == set(range(6))
    pools = pools_of(table, NOW)
    assert any(v < 0 for p in pools for v in p)
    dur, off, start, used = batch(eng, queues, table)
    want, want_used = expect(dur, off, pools)
    assert np.array_equal(used, want_used)
    bad = np.nonzero(start != want)[0]
    assert bad.size == 0, (mode, int(bad[0]), int(np.searchsorted(off, bad[0], "right") - 1))


def test_one_long_queue_per_side_of_the_limit(eng):
    rng = np.random.default_rng(7400)
    counts = [3, 33, LIMIT, LIMIT + 1, 0]
    queues = [rng.integers(0, 3600 * 10 ** 9, 10_000).tolist() for _ in counts]
    table = random_table(rng, counts)
    table.kind[table.kind == L.EVG_EH_IGNORED] = L.EVG_EH_RUNNING  # both sides of the limit stay on their side
    dur, off, start, used = batch(eng, queues, table)
    want, want_used = expect(dur, off, pools_of(table, NOW))
    assert used.tolist() == counts and np.array_equal(used, want_used) and np.array_equal(start, want)


def test_hosts_without_items_and_items_without_hosts(eng):
    table = table_of([[5, 1], [], [], [7]])
    _, _, start, used = batch(eng, [[], [3, 3], [], [2]], table)
    assert start.tolist() == [-1, -1, 7] and used.tolist() == [2, 0, 0, 1]
    none = S.EstHostTable(np.zeros(0, np.uint8), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(3, np.int64))
    _, _, start, used = batch(eng, [[1, 2], [3]], none)
    assert start.tolist() == [-1, -1, -1] and used.tolist() == [0, 0] and eng.last_launch_count() == 0
    ignored = S.EstHostTable(np.full(2, L.EVG_EH_IGNORED, np.uint8), np.zeros(2, np.int64), np.zeros(2, np.int64), np.array([0, 2], np.int64))
    _, _, start, used = batch(eng, [[1, 2]], ignored)
    assert start.tolist() == [-1, -1] and used.tolist() == [0]


# ---------------------------------------------------------------- the chain
def snapshot(eng, table):
    po, _ = eng.download(want_alloc=False)
    item_off, items = eng.download_queue(0, table.task_off)
    return [x.copy() for x in (po.order, po.total_value, po.info, po.group_info, item_off, items)]


def check_chain(eng, other, table, cap, rng, now=NOW, big_pool=0):
    """evg_estimate_start_times == evg_download_queue + evg_estimate_start_batch (on a context of its own) == the oracle."""
    D = table.n_distros
    counts = rng.choice(np.array([0, 1, 2, 5, 33, 70]), D)
    if big_pool:
        counts[int(np.argmax(np.diff(table.task_off)))] = big_pool
    hosts = random_table(rng, counts)
    io, start, used = [x.copy() for x in eng.estimate_start_times(hosts, now, cap, table.task_off)]
    item_off, items = eng.download_queue(cap, table.task_off)
    assert np.array_equal(io, item_off)
    dur = items["expected_ns"].copy()
    b_start, b_used = other.estimate_start_batch(dur, io, hosts, now)
    assert np.array_equal(start, b_start) and np.array_equal(used, b_used)
    want, want_used = expect(dur, io, pools_of(hosts, now))
    assert np.array_equal(start, want) and np.array_equal(used, want_used)
    return hosts, start


SIZES = [0, 1, 2, 50, 700, 3000, 6000, 15000]  # every planner route; the last one is a general-path distro above the cap


def test_chain_on_every_route_at_every_cap(eng, other):
    rng = np.random.default_rng(7500)
    w = synth.make(np.array(SIZES), 7501, zipf_priority=True, unmet_dep_frac=0.2, met_dep_frac=0.3, tg_frac=0.3, group_versions_frac=0.3,
                   includes_dependencies=True, n_hosts=30)
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    before = snapshot(eng, w.distros)
    _, ao = eng.download()
    alloc_before = ao.result.copy()
    for cap in (0, 1, 7, 100, 16000):
        check_chain(eng, other, w.distros, cap, rng, big_pool=LIMIT + 300 if cap == 0 else 0)
    for x, y in zip(before, snapshot(eng, w.distros)):
        assert np.array_equal(x, y)
    assert np.array_equal(alloc_before, eng.download()[1].result)
    eng.host_job(np.zeros(w.distros.n_distros, L.HOST_JOB_CFG_DTYPE))  # the allocator's run state survived
    eng.run(w.now)  # and the tick still runs
    for x, y in zip(before, snapshot(eng, w.distros)):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("entry", ["edit_tasks", "plan_aliases", "plan_from_finder"])
def test_chain_on_other_ticks(eng, other, entry):
    rng = np.random.default_rng(7510)
    w = synth.make(np.array([40, 900, 6000, 300]), 7511, tg_frac=0.2, met_dep_frac=0.2, group_versions_frac=0.5)
    if entry == "edit_tasks":
        eng.upload(w.tasks, w.distros)
        eng.run(w.now)
        e = synth.next_tick(w, 7512, order=eng.download(want_alloc=False)[0].order.copy())
        eng.edit_tasks(e.edit, e.workload.distros)
        if e.rows.shape[0]:
            eng.update_tasks(e.rows, e.values)
        table = e.workload.distros
    elif entry == "plan_aliases":
        at, cfg = synth.make_aliases(w, 7513, name_frac=0.7)
        eng.plan_aliases(at, cfg, w.now)
        table = S.compose_aliases(at, cfg)[1]
    else:
        w, rt, fin = candidates([300, 2000, 40], 7514, "mixed")
        _, count = eng.plan_from_finder(rt, w.tasks, w.distros, w.hosts, fin, w.now)
        off = np.concatenate([[0], np.cumsum(count.copy())]).astype(np.int64)
        table = S.DistroTable(off, w.distros.group_off, w.distros.cfg, w.distros.group_max_hosts)
    eng.run(w.now)
    for cap in (0, 13):
        check_chain(eng, other, table, cap, rng)


def test_dispatchers_survive_and_a_later_now_moves_only_the_hosts(eng, other):
    rng = np.random.default_rng(7520)
    w = synth.make(np.array([0, 1, 40, 700, 3000]), 7521, zipf_priority=True, unmet_dep_frac=0.2, met_dep_frac=0.4, tg_frac=0.3,
                   includes_dependencies=True)
    results = []
    for e, estimate in ((eng, True), (other, False)):
        e.upload(w.tasks, w.distros)
        e.run(w.now)
        r = e.rebuild_dispatchers(0)
        N, G, go = int(r["item_off"][-1]), int(r["group_off"][-1]), r["group_off"].copy()
        srng = np.random.default_rng(7522)
        first = [x.copy() for x in e.find_next_tasks(raw_snapshot(srng, N, G), raw_requests(srng, go, lambda d: 2))]
        if estimate:
            hosts = random_table(rng, [3, 4, 0, 40, 70])
            a = e.estimate_start_times(hosts, NOW, 0, w.distros.task_off)[1].copy()
            later = NOW + 90 * 10 ** 9
            b = e.estimate_start_times(hosts, later, 0, w.distros.task_off)[1].copy()
            io, items = e.download_queue(0, w.distros.task_off)
            want_a, _ = expect(items["expected_ns"], io, pools_of(hosts, NOW))
            want_b, _ = expect(items["expected_ns"], io, pools_of(hosts, later))
            assert np.array_equal(a, want_a) and np.array_equal(b, want_b) and not np.array_equal(a, b)
        state = {k: v.copy() for k, v in e.download_dispatch_state().items()}
        second = [x.copy() for x in e.find_next_tasks(raw_snapshot(srng, N, G), raw_requests(srng, go, lambda d: 3))]
        results.append((first, state, second))
    (f0, s0, n0), (f1, s1, n1) = results
    assert all(np.array_equal(x, y) for x, y in zip(f0 + n0, f1 + n1)) and all(np.array_equal(s0[k], s1[k]) for k in s0)


def test_resident_tick_object(eng):
    now = NOW
    distro = M.Distro(id="d0")
    tasks = [M.Task(id=f"t{i}", distro_id="d0", version="v", project="p", expected_duration=(i % 7 + 1) * OE.MINUTE, priority=i % 5,
                    activated_time=now - i * OE.MINUTE, ingest_time=now - i * OE.MINUTE) for i in range(60)]
    rt = scheduler.ResidentTick(eng)
    (ranked, _), = rt.plan([(distro, tasks)], now, breakdown=False)
    hosts = [M.Host(status=M.HOST_RUNNING), M.Host(status=M.HOST_STARTING), M.Host(status=M.HOST_RUNNING, running_task="r"),
             M.Host(status=M.HOST_RUNNING, running_task="gone")]
    running = {"r": M.Task(id="r", expected_duration=9 * OE.MINUTE, dispatch_time=now - 2 * OE.MINUTE)}
    got = rt.estimated_start_times([hosts], running, now)[0]
    want = OE.fresh_estimates([t.expected_duration for t in ranked], [0, 3 * OE.MINUTE, 7 * OE.MINUTE])
    assert [got[t.id] for t in ranked] == want and len(got) == 60


# ---------------------------------------------------------------- at size
def test_at_size(eng, other):
    rng = np.random.default_rng(7600)
    w = synth.config(5)
    D = w.distros.n_distros
    assert D == 100_000
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    hosts = random_table(rng, np.diff(w.hosts.host_off))  # the tick's own host counts, with the estimator's columns
    io, start, used = [x.copy() for x in eng.estimate_start_times(hosts, w.now, 0, w.distros.task_off)]
    item_off, items = eng.download_queue(0, w.distros.task_off)
    assert np.array_equal(io, item_off)
    dur = items["expected_ns"].copy()
    b_start, b_used = other.estimate_start_batch(dur, io, hosts, w.now)
    assert np.array_equal(start, b_start) and np.array_equal(used, b_used)
    work = np.diff(io) * np.diff(hosts.est_host_off)
    sample = np.union1d(np.argsort(work)[-40:], rng.choice(D, 2000, replace=False))
    pools = pools_of(hosts, w.now)
    assert np.array_equal(used, np.array([len(p) for p in pools], dtype=np.int32))
    for d in sample.tolist():
        a, b = int(io[d]), int(io[d + 1])
        assert start[a:b].tolist() == fresh(dur[a:b].tolist(), pools[d]), d
    nohost = np.repeat(used == 0, np.diff(io))
    assert np.all(start[nohost] == -1)
    # one full persisted queue against a pool of a few thousand hosts
    big = random_table(rng, [3000])
    q = rng.integers(10 ** 9, 7200 * 10 ** 9, 10_000).tolist()
    dq, off, s, u = batch(other, [q], big)
    want, want_used = expect(dq, off, pools_of(big, NOW))
    assert np.array_equal(s, want) and np.array_equal(u, want_used) and int(u[0]) > 2000


# ---------------------------------------------------------------- the error contract
def raw_times(eng, table, cap=0, capacity=1 << 20, item_off=True, start=True, used=True, off=None, D=3):
    bufs = (np.zeros(D + 1, np.int64), np.zeros(max(capacity, 1), np.int64), np.zeros(max(D, 1), np.int32))
    st = table.struct() if table is not None else None
    rc = eng.lib.evg_estimate_start_times(eng.ctx, cap, C.byref(st) if st is not None else None,
                                          L.ptr(table.est_host_off if off is None else off) if table is not None else None, NOW,
                                          L.ptr(bufs[0]) if item_off else None, L.ptr(bufs[1]) if start else None, capacity,
                                          L.ptr(bufs[2]) if used else None)
    return rc, L.last_error()


def raw_batch(eng, dur, item_off, table, D=None, off=None, start=True, used=True):
    n = 0 if dur is None else dur.shape[0]
    bufs = (np.zeros(max(n, 1), np.int64), np.zeros(max(item_off.shape[0], 1), np.int32))
    st = table.struct() if table is not None else None
    rc = eng.lib.evg_estimate_start_batch(eng.ctx, L.ptr(dur) if dur is not None else None, L.ptr(item_off),
                                          item_off.shape[0] - 1 if D is None else D, C.byref(st) if st is not None else None,
                                          L.ptr(table.est_host_off if off is None else off) if table is not None else None, NOW,
                                          L.ptr(bufs[0]) if start else None, L.ptr(bufs[1]) if used else None)
    return rc, L.last_error()


def test_error_contract_of_the_batch(eng):
    w = synth.make(np.array([30, 5]), 7700, n_hosts=4)
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    before = snapshot(eng, w.distros)
    dur, off, table = np.arange(5, dtype=np.int64), np.array([0, 2, 5], np.int64), table_of([[1, 2], [3]])
    assert raw_batch(eng, dur, off, table)[0] == L.EVG_OK
    bad_kind = copy.copy(table)
    bad_kind.kind = np.array([4, 6, 4], np.uint8)
    cases = {
        "null hosts": raw_batch(eng, dur, off, None),
        "null durations": raw_batch(eng, None, off, table),
        "null start": raw_batch(eng, dur, off, table, start=False),
        "null hosts_used": raw_batch(eng, dur, off, table, used=False),
        "negative n_distros": raw_batch(eng, dur, off, table, D=-1),
        "item_off": raw_batch(eng, dur, np.array([0, 3, 2], np.int64), table),
        "est_host_off": raw_batch(eng, dur, off, table, off=np.array([0, 2, 4], np.int64)),
        "kind": raw_batch(eng, dur, off, bad_kind),
    }
    for name, (rc, msg) in cases.items():
        assert rc == L.EVG_ERR_INVALID and msg.startswith("evg_estimate_start_batch: "), (name, rc, msg)
    assert "item_off[2]" in cases["item_off"][1] and "est_host_off[2]" in cases["est_host_off"][1]
    assert "host row 1 has kind 6" in cases["kind"][1]
    st = table.struct()
    st.n_hosts = -1
    assert eng.lib.evg_estimate_start_batch(eng.ctx, L.ptr(dur), L.ptr(off), 2, C.byref(st), L.ptr(table.est_host_off), NOW, L.ptr(dur.copy()),
                                            L.ptr(np.zeros(2, np.int32))) == L.EVG_ERR_INVALID
    for x, y in zip(before, snapshot(eng, w.distros)):  # the standalone call and its rejections leave the tick alone
        assert np.array_equal(x, y)


def test_error_contract_and_tick_state_of_the_chain(eng):
    fresh_eng = scheduler.Engine(0)
    try:
        rc, msg = raw_times(fresh_eng, table_of([[1], [2]]), D=2)
        assert rc == L.EVG_ERR_STATE and msg == "evg_estimate_start_times: no resident tick"
    finally:
        fresh_eng.close()
    w = synth.make(np.array([30, 5, 0]), 7710, n_hosts=6)
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    before = snapshot(eng, w.distros)
    table = table_of([[1, 2], [3], []])
    assert raw_times(eng, table)[0] == L.EVG_OK
    bad_kind = copy.copy(table)
    bad_kind.kind = np.array([4, 4, 9], np.uint8)
    cases = {
        "null hosts": raw_times(eng, None),
        "null item_off": raw_times(eng, table, item_off=False),
        "null start": raw_times(eng, table, start=False),
        "null hosts_used": raw_times(eng, table, used=False),
        "negative cap": raw_times(eng, table, cap=-1),
        "capacity": raw_times(eng, table, capacity=34),
        "est_host_off": raw_times(eng, table, off=np.array([0, 2, 1, 3], np.int64)),
        "kind": raw_times(eng, bad_kind),
    }
    for name, (rc, msg) in cases.items():
        assert rc == L.EVG_ERR_INVALID and msg.startswith("evg_estimate_start_times: "), (name, rc, msg)
    assert "35 rows needed, 34 available" in cases["capacity"][1] and "host row 2 has kind 9" in cases["kind"][1]
    assert raw_times(eng, table, cap=3, capacity=6)[0] == L.EVG_OK  # 3 + 3 + 0 rows
    for x, y in zip(before, snapshot(eng, w.distros)):
        assert np.array_equal(x, y)
    eng.run(w.now)  # a rejected call leaves the tick runnable
    # a tick nobody ran yet has no ranks worth reading but is a tick: the call is allowed wherever evg_download_queue is;
    # a one-shot call's tick and borrowed columns serve it too
    eng.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now)
    assert raw_times(eng, table)[0] == L.EVG_OK
    eng.dag_rebuild_batch(np.array([0, 1], np.int64), np.array([0, 0], np.int64), np.array([0, 0], np.int64), np.zeros(0, np.int32),
                          np.array([-1], np.int32), np.array([0], np.int32))  # ends the tick
    assert raw_times(eng, table)[0] == L.EVG_ERR_STATE
