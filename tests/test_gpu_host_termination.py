"""evg_host_drawdown and evg_idle_hosts on the device: standalone on every golden case, bit for bit against the
restatement oracle_host_termination on synthetic tables of at least 50 000 hosts, chained drawdown against standalone
fed the downloaded evg_host_job report after every tick kind that leaves one, the tick only read, launch counts, and
the error contract."""
import ctypes as C

import numpy as np
import pytest

import host_termination_cases as HT
import oracle_host_termination as OT
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_entry_guard import launched_kernels
from test_gpu_finder_compaction import candidates
from test_gpu_host_job import job_cfg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = scheduler.Engine(0)
    yield e
    e.close()


def rows(verdicts):
    return [tuple(int(v[f]) for f in ("decision", "idle_ns", "communication_ns", "threshold_ns", "since_teardown_ns")) for v in verdicts]


def drawdown_inputs(w):
    cap = np.array([L.EVG_NO_DRAWDOWN if x is None else x.new_cap_target for x in w.drawdown], np.int64)
    return np.asarray(w.existing, np.int64), cap, np.asarray(w.queue_lengths, np.int64)


def idle_cfg(distros, running, sched_idle_seconds):
    cfg = np.zeros(len(distros), L.IDLE_CFG_DTYPE)
    for i, d in enumerate(distros):
        d = d or M.Distro()
        idle = d.host_allocator_settings.acceptable_host_idle_time
        cfg[i] = (d.host_allocator_settings.minimum_hosts, int(running[i]), idle or sched_idle_seconds * M.SECOND)
    return cfg


# ---------------------------------------------------------------------------------------------------- golden cases
@pytest.mark.parametrize("name", sorted(HT.CASES))
def test_golden(eng, name):
    c = HT.CASES[name]
    jobs, want = HT.run_oracle(c)
    groups = [HT.hosts_of(d) for d in c["distros"]]
    ds = c["distros"]
    if c["job"] == "drawdown":
        jobs_dev = scheduler.host_drawdown_jobs(
            [d["id"] for d in ds], groups, [d["existing_hosts"] for d in ds], HT.NOW,
            drawdown=[None if d["new_cap_target"] is None else M.DrawdownInfo(d["id"], d["new_cap_target"]) for d in ds],
            queue_lengths=[d["queue_length_dm"] for d in ds], engine=eng)
        t = S.marshal_idle_hosts(groups)
        ex = np.array([d["existing_hosts"] for d in ds], np.int64)
        cap = np.array([L.EVG_NO_DRAWDOWN if d["new_cap_target"] is None else d["new_cap_target"] for d in ds], np.int64)
        res = eng.host_drawdown(t, ex, HT.NOW, cap, np.array([d["queue_length_dm"] for d in ds], np.int64))
    else:
        distros = [HT.distro_of(d) for d in ds]
        jobs_dev = scheduler.idle_host_jobs(distros, groups, [d["running_hosts_count"] for d in ds], HT.NOW,
                                            acceptable_host_idle_time_seconds=c["sched_idle_seconds"], engine=eng)
        t = S.marshal_idle_hosts(groups, [(d or M.Distro()).default_ami for d in distros])
        res = eng.idle_hosts(t, idle_cfg(distros, [d["running_hosts_count"] for d in ds], c["sched_idle_seconds"]), HT.NOW)
    assert rows(res["hosts"]) == want
    for j, jd in zip(jobs, jobs_dev):
        if j is None:
            assert jd is None
            continue
        assert HT.picked(jd) == HT.picked(j) and jd.errors == j.errors
        if c["job"] == "drawdown":
            assert (jd.drawdown_target, jd.new_cap_target, jd.num_idle_hosts) == (j.drawdown_target, j.new_cap_target, j.num_idle_hosts)
        else:
            assert (jd.min_hosts_to_evaluate, jd.reasons, jd.num_idle_hosts) == (j.min_hosts_to_evaluate, j.reasons, j.num_idle_hosts)
    e = c["expect"]
    if "hosts" in e:
        assert sorted(h for j in jobs_dev if j is not None for h in HT.picked(j)) == sorted(e["hosts"])


# ---------------------------------------------------------------------------------------------------- at scale
SHAPES = {
    "edges": np.array([0, 1, 31, 32, 33, 1025, 3000, 0, 2, 64] * 4 + [1] * 30000, np.int64),
    "c4": None,  # 10 000 distros, power-law sizes, about 50 000 hosts
}


@pytest.fixture(scope="module", params=sorted(SHAPES))
def big(request):
    sizes = SHAPES[request.param]
    if sizes is None:
        sizes = synth.power_law_sizes(synth.Rng(1501), 10_000, hi=2_000)
    w = synth.make_idle_hosts(sizes, 1502)
    assert sum(len(g) for g in w.groups) >= 45_000
    return w


def test_at_scale_bit_for_bit(eng, big):
    w = big
    ex, cap, qlen = drawdown_inputs(w)
    t_dd = S.marshal_idle_hosts(w.groups)
    res = eng.host_drawdown(t_dd, ex, w.now, cap, qlen)
    want, dist = [], []
    for d, g in enumerate(w.groups):
        if w.drawdown[d] is None:
            want += [OT.NOT_CHECKED] * len(g)
            dist.append((0, 0, 0))
            continue
        job, v = OT.drawdown_job(f"d{d}", g, int(ex[d]), int(cap[d]), int(qlen[d]), w.now)
        want += v
        dist.append((job.drawdown_target, job.decommissioned, 1))
    assert rows(res["hosts"]) == want
    assert [(int(r["target"]), int(r["decommissioned"]), int(r["ran"])) for r in res["distros"]] == dist
    targets = [t for t, _, ran in dist if ran]
    assert min(targets) <= 0 and any(n < t for t, n, ran in dist if ran) and any(0 < t == n for t, n, ran in dist if ran)

    t_idle = S.marshal_idle_hosts(w.groups, [(d or M.Distro()).default_ami for d in w.distros])
    res = eng.idle_hosts(t_idle, idle_cfg(w.distros, w.running_counts, w.sched_idle_seconds), w.now)
    want, dist = [], []
    for d, g in enumerate(w.groups):
        job, v = OT.idle_job(w.distros[d], g, int(w.running_counts[d]), w.now, w.sched_idle_seconds)
        want += v
        dist.append((job.min_hosts_to_evaluate, job.terminated))
    assert rows(res["hosts"]) == want
    assert [(int(r["min_evaluate"]), int(r["terminated"])) for r in res["distros"]] == dist
    assert {r[0] for r in want} == set(range(L.EVG_HT_TERM_TEARDOWN + 1)) - {L.EVG_HT_DECOMMISSION}


# ---------------------------------------------------------------------------------------------------- chained drawdown
@pytest.fixture(scope="module")
def world():
    w, table, fin = candidates([300, 2000, 40, 5], 1510, "mixed")
    return dict(w=w, table=table, fin=fin, plain=synth.make(np.array([100, 40, 700]), 1511, tg_frac=0.1, n_hosts=10),
                big=synth.make(np.full(8, 280_000), 1512, tg_frac=0.1, n_hosts=100))


def idle_for(D, seed):
    return synth.make_idle_hosts(np.random.default_rng(seed).integers(0, 40, D), seed)


def check_chained(eng, D, seed, po=None):
    """evg_host_job with drawdown-prone settings, then chained drawdown == standalone fed its downloaded report."""
    cfg = job_cfg(D, seed, single=0.0, terminate=1.0, hourly=0.0)
    rep = eng.host_job(cfg)["report"].copy()
    if po is None:
        po, _ = eng.download()
    iw = idle_for(D, seed)
    t = S.marshal_idle_hosts(iw.groups)
    ex = np.asarray(iw.existing, np.int64)
    chained = {k: v.copy() for k, v in eng.host_drawdown(t, ex, iw.now).items()}
    cap = np.where(rep["drawdown"] != 0, rep["new_cap_target"], L.EVG_NO_DRAWDOWN).astype(np.int64)
    qlen = po.info["length_with_dependencies_met"].astype(np.int64)
    alone = eng.host_drawdown(t, ex, iw.now, cap, qlen)
    for k in chained:
        assert np.array_equal(chained[k].view(np.uint8), alone[k].view(np.uint8)), k
    RAN.append(int(chained["distros"]["ran"].sum()))


RAN = []  # distros each chained check drew down


def test_chained_after_upload(eng, world):
    w = world["w"]
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    check_chained(eng, w.distros.n_distros, 1520)


def test_chained_after_upload_with_deps(eng, world):
    w = world["w"]
    eng.upload_with_deps(w.tasks, w.distros, w.hosts, world["table"].deps, world["fin"], w.now)
    eng.run(w.now)
    check_chained(eng, w.distros.n_distros, 1521)


def test_chained_after_edit(eng, world):
    w = world["w"]
    eng.upload(w.tasks, w.distros, w.hosts)
    e = synth.next_tick(w, 1522)
    eng.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
    eng.run(w.now)
    check_chained(eng, e.workload.distros.n_distros, 1523)


def test_chained_after_plan_from_finder(eng, world):
    w = world["w"]
    eng.plan_from_finder(world["table"], w.tasks, w.distros, w.hosts, world["fin"], w.now)
    eng.run(w.now)
    check_chained(eng, w.distros.n_distros, 1524)


@pytest.mark.parametrize("which", ["plain", "big"])
def test_chained_after_plan_and_alloc_batch(eng, world, which):
    w = world[which]
    po, _ = eng.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now)
    check_chained(eng, w.distros.n_distros, 1525, po)


def test_chained_after_upload_device(eng, world):
    import torch
    w = world["plain"]
    cols = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dt)])).cuda() for name, dt in S.TaskSoA.COLUMNS}
    eng.upload_device({k: v.data_ptr() for k, v in cols.items()}, w.n_tasks, w.distros, w.hosts)
    eng.run(w.now)
    check_chained(eng, w.distros.n_distros, 1526)
    torch.cuda.synchronize()
    del cols


def test_chained_with_bound_result_buffer(eng, world):
    import torch
    w = world["plain"]
    D = w.distros.n_distros
    buf = torch.zeros(D * L.ALLOC_RESULT_DTYPE.itemsize + 64, dtype=torch.uint8, device="cuda")
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.bind_result_buffer(buf.data_ptr(), D)
    try:
        eng.run(w.now)
        check_chained(eng, D, 1527)
    finally:
        eng.bind_result_buffer(0, 0)


def test_chained_checks_drew_down_somewhere():
    assert len(RAN) == 8 and sum(RAN) > 0, RAN


def test_tick_is_only_read(eng, world):
    w = world["w"]
    D = w.distros.n_distros
    eng.upload(w.tasks, w.distros, w.hosts)
    eng.run(w.now)
    eng.host_job(job_cfg(D, 1530, single=0.0, terminate=1.0, hourly=0.0))
    po, ao = eng.download(want_alloc=True)
    before = [a.copy() for a in (po.order, po.total_value, po.info, po.group_info, ao.result, ao.status)]
    iw = idle_for(D, 1531)
    t = S.marshal_idle_hosts(iw.groups)
    first = {k: v.copy() for k, v in eng.host_drawdown(t, iw.existing, iw.now).items()}
    eng.idle_hosts(S.marshal_idle_hosts(iw.groups, [""] * D), idle_cfg(iw.distros, iw.running_counts, 60), iw.now)
    second = eng.host_drawdown(t, iw.existing, iw.now)
    for k in first:
        assert np.array_equal(first[k].view(np.uint8), second[k].view(np.uint8)), k
    po, ao = eng.download(want_alloc=True)
    for a, b in zip(before, (po.order, po.total_value, po.info, po.group_info, ao.result, ao.status)):
        assert np.array_equal(a, b)
    e = synth.next_tick(w, 1532)
    eng.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)  # still the editable tick it was


def test_launch_counts(eng):
    """torch.profiler can miss the first kernels of a window that opens straight onto them (as in
    test_gpu_onchip_sort.profiled): a torch kernel opens each window, and a list that differs from the context's count
    is taken again, a few times.  The calls are pure, so every try launches the same kernels."""
    import torch
    iw = idle_for(50, 1540)
    t = S.marshal_idle_hosts(iw.groups)
    ex, cap, qlen = drawdown_inputs(iw)
    for fn in (lambda: eng.host_drawdown(t, ex, iw.now, cap, qlen),
               lambda: eng.idle_hosts(S.marshal_idle_hosts(iw.groups, [""] * 50), idle_cfg(iw.distros, iw.running_counts, 60), iw.now)):
        def call():
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
            fn()
        for _ in range(6):
            names = launched_kernels(call)
            if eng.last_launch_count() == len(names):
                break
        assert eng.last_launch_count() == len(names) and names, names


# ---------------------------------------------------------------------------------------------------- errors
def test_error_contract(world):
    p = world["plain"]
    eng = scheduler.Engine(0)
    try:
        D = p.distros.n_distros
        iw = idle_for(D, 1550)
        t = S.marshal_idle_hosts(iw.groups)
        ex, cap, qlen = drawdown_inputs(iw)
        vout = np.zeros(max(t.n_hosts, 1), L.HOST_VERDICT_DTYPE)
        dout = np.zeros(D, L.DRAWDOWN_DISTRO_DTYPE)
        iout = np.zeros(D, L.IDLE_DISTRO_DTYPE)
        cfg = idle_cfg(iw.distros, iw.running_counts, 60)

        def dd(table=None, off=None, e=ex, c=cap, q=qlen, out=True):
            table = table or t.struct()
            ins = L.DrawdownInStruct(L.ptr(e), L.ptr(c), L.ptr(q))
            o = L.HostTermOutStruct(L.ptr(vout), L.ptr(dout))
            return eng.lib.evg_host_drawdown(eng.ctx, C.byref(table), L.ptr(t.idle_off if off is None else off), C.byref(ins), iw.now,
                                             C.byref(o) if out else None)

        def idle(table=None, off=None, c=cfg):
            o = L.HostTermOutStruct(L.ptr(vout), L.ptr(iout))
            return eng.lib.evg_idle_hosts(eng.ctx, C.byref(table or t.struct()), L.ptr(t.idle_off if off is None else off),
                                          L.ptr(c), iw.now, C.byref(o))

        assert dd() == L.EVG_OK and idle() == L.EVG_OK  # standalone: no tick needed
        assert dd(c=None, q=None) == L.EVG_ERR_STATE and "no resident tick" in L.last_error()
        eng.upload(p.tasks, p.distros, p.hosts)
        eng.run(p.now)
        assert dd(c=None, q=None) == L.EVG_ERR_STATE and "evg_host_job" in L.last_error()
        eng.host_job(job_cfg(D, 1551))
        assert dd(c=None, q=None) == L.EVG_OK
        eng.run(p.now)
        assert dd(c=None, q=None) == L.EVG_ERR_STATE  # a new run: the report is not its
        eng.host_job(job_cfg(D, 1551))
        eng.bind_result_buffer(0, 0)
        assert dd(c=None, q=None) == L.EVG_ERR_STATE
        eng.run(p.now)
        eng.host_job(job_cfg(D, 1551))
        assert dd(c=None, q=None) == L.EVG_OK
        # rejected with nothing launched
        assert dd(c=None) == L.EVG_ERR_INVALID and dd(q=None) == L.EVG_ERR_INVALID
        assert dd(e=None) == L.EVG_ERR_INVALID and dd(out=False) == L.EVG_ERR_INVALID
        neg = ex.copy()
        neg[1] = -1
        assert dd(e=neg) == L.EVG_ERR_INVALID
        negq = qlen.copy()
        negq[0] = -1
        assert dd(q=negq) == L.EVG_ERR_INVALID
        bad = t.idle_off.copy()
        bad[1], bad[2] = bad[2] + 1, bad[1]
        assert dd(off=bad) == L.EVG_ERR_INVALID and "idle_off" in L.last_error()
        assert idle(off=bad) == L.EVG_ERR_INVALID and "idle_off" in L.last_error()
        s = t.struct()
        s.n_hosts = -1
        assert dd(table=s) == L.EVG_ERR_INVALID and idle(table=s) == L.EVG_ERR_INVALID
        s = t.struct()
        s.flags = None
        assert dd(table=s) == L.EVG_ERR_INVALID and idle(table=s) == L.EVG_ERR_INVALID
        other = S.marshal_idle_hosts(iw.groups + [[]])
        s = other.struct()
        assert eng.lib.evg_host_drawdown(eng.ctx, C.byref(s), L.ptr(other.idle_off),
                                         C.byref(L.DrawdownInStruct(L.ptr(np.zeros(D + 1, np.int64)), None, None)), iw.now,
                                         C.byref(L.HostTermOutStruct(L.ptr(vout), L.ptr(np.zeros(D + 1, L.DRAWDOWN_DISTRO_DTYPE))))
                                         ) == L.EVG_ERR_INVALID  # chained on a tick of another distro count
        for f in ("minimum_hosts", "running_hosts_count"):
            c2 = cfg.copy()
            c2[f][0] = -1
            assert idle(c=c2) == L.EVG_ERR_INVALID and f in L.last_error()
        assert idle(c=None) == L.EVG_ERR_INVALID
        assert dd(c=None, q=None) == L.EVG_OK  # the rejections left the tick and the report as they were
    finally:
        eng.close()
