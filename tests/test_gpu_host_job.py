"""evg_host_job on the device: bit-exact against the restatement oracle_host_job (floats compared as bits) on every golden
case, on the ticks of the allocator scenarios and on synthetic ticks under every job setting, after every entry point
that leaves a tick with hosts, with spawned NULL and given and with a bound result buffer; the tick is only read; the
error contract."""
import ctypes as C

import numpy as np
import pytest

import golden_loader as G
import host_job_cases as HC
import oracle_host_job as OJ
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_finder_compaction import candidates
from test_host_job_host import assert_job

pytestmark = pytest.mark.gpu
PROVIDERS = {L.EVG_PROVIDER_STATIC: M.PROVIDER_STATIC, L.EVG_PROVIDER_EPHEMERAL: M.PROVIDER_EC2_FLEET,
             L.EVG_PROVIDER_DOCKER: M.PROVIDER_DOCKER}


def job_cfg(D, seed, single=0.2, terminate=0.7, hourly=0.3):
    rng = np.random.default_rng(seed)
    cfg = np.zeros(D, L.HOST_JOB_CFG_DTYPE)
    cfg["n_provisioning"] = rng.integers(0, 4, D)
    cfg["single_task_distro"] = rng.random(D) < single
    cfg["terminate_when_overallocated"] = rng.random(D) < terminate
    cfg["hourly_billing"] = rng.random(D) < hourly
    return cfg


def restate(po, ao, group_off, hosts, cfg, spawned):
    """oracle_host_job on what evg_download returns: the distro as the job settings and allocator config describe it."""
    out = []
    for d in range(cfg.shape[0]):
        a, c = hosts.cfg[d], cfg[d]
        distro = M.Distro(id=f"d{d}", provider=PROVIDERS[int(a["provider"])], arch="osx" if c["hourly_billing"] else "linux",
                          single_task_distro=bool(c["single_task_distro"]),
                          host_allocator_settings=M.HostAllocatorSettings(
                              minimum_hosts=int(a["minimum_hosts"]),
                              hosts_overallocated_rule=M.HOSTS_OVERALLOCATED_TERMINATE if c["terminate_when_overallocated"] else ""))
        q = po.info[d]
        groups = [M.TaskGroupInfo(name=f"g{k}", **{f: int(g[f]) for f in L.GROUP_INFO_FIELDS})
                  for k, g in enumerate(po.group_info[int(group_off[d]):int(group_off[d + 1])])]
        info = M.DistroQueueInfo(length_with_dependencies_met=int(q["length_with_dependencies_met"]),
                                 expected_duration=int(q["expected_duration"]), max_duration_threshold=int(q["max_duration_threshold"]),
                                 count_duration_over_threshold=int(q["count_duration_over_threshold"]),
                                 duration_over_threshold=int(q["duration_over_threshold"]), task_group_infos=groups)
        alloc = (int(ao.result[d]["new_hosts"]), int(ao.result[d]["free_hosts"]), int(ao.status[d]))
        n_up = int(hosts.host_off[d + 1] - hosts.host_off[d])
        out.append(OJ.host_allocator_job(distro, info, n_up, int(c["n_provisioning"]), alloc,
                                         None if spawned is None else int(spawned[d])))
    return out


def as_expect(r):
    return {"n_hosts": r["n_hosts"], "n_hosts_free": r["n_hosts_free"], "status": r["status"], "report": r["report"]}


def check(eng, group_off, hosts, seed, po=None, ao=None):
    """The device job against the restatement on the resident tick, spawned NULL and given; returns the NULL result."""
    if po is None:
        po, ao = eng.download(want_alloc=True)
    D = group_off.shape[0] - 1
    cfg = job_cfg(D, seed)
    first = None
    for spawned in (None, np.random.default_rng(seed).integers(0, 6, D).astype(np.int32)):
        want = restate(po, ao, group_off, hosts, cfg, spawned)
        res = {k: v.copy() for k, v in eng.host_job(cfg, spawned).items()}
        for d in range(D):
            got = {"n_hosts": int(res["n_hosts"][d]), "n_hosts_free": int(res["n_hosts_free"][d]), "status": int(res["status"][d]),
                   "report": {f: res["report"][d][f] for f in L.HOST_REPORT_FIELDS}}
            assert_job(got, as_expect(want[d]), f"distro {d}")
        if first is None:
            first = res
    return first


# ---------------------------------------------------------------------------------------------------- golden cases
@pytest.mark.parametrize("c", HC.CASES["cases"], ids=lambda c: c["name"])
def test_golden(engine, c):
    distro, tasks, data = HC.batch_entry(c)
    spawned = None if c["spawned"] is None else [c["spawned"]]
    if "raw_threshold" not in c:
        (n, f, rep, dd), = scheduler.host_allocator_jobs([(distro, tasks, data)], HC.NOW, n_provisioning=[c["n_provisioning"]],
                                                         spawned=spawned, engine=engine)
        e = c["expect"]
        assert (n, f) == (e["n_hosts"], e["n_hosts_free"])
        assert (rep is None) == (e["status"] != 0)
        if rep is not None:
            assert rep.drawdown == bool(e["report"]["drawdown"]) and (dd is not None) == rep.drawdown
            assert dd is None or (dd.distro_id, dd.new_cap_target) == (distro.id, e["report"]["new_cap_target"])
    # the raw call, also with a MaxDurationThreshold no Distro.GetTargetTime gives
    distro, tasks, data = HC.batch_entry(c)
    soa, table, keys = S.marshal_tasks([(distro, tasks)], HC.NOW)
    table.cfg["target_time_ns"] = HC.threshold(c)
    hosts = S.marshal_hosts([data], [k.group_names for k in keys])
    engine.upload_with_deps(soa, table, hosts, S.marshal_deps([(distro, tasks)]), S.marshal_dep_finished([(distro, tasks)]), HC.NOW)
    engine.run(HC.NOW)
    res = engine.host_job(S.marshal_host_job([data], [c["n_provisioning"]]), None if spawned is None else np.array(spawned))
    got = {"n_hosts": int(res["n_hosts"][0]), "n_hosts_free": int(res["n_hosts_free"][0]), "status": int(res["status"][0]),
           "report": {f: res["report"][0][f] for f in L.HOST_REPORT_FIELDS}}
    assert_job(got, c["expect"], c["name"])


# ------------------------------------------------------------------------------------- allocator scenarios' ticks
ALLOC = G.load("allocator_scenarios.json")


def scenario_tick(s):
    """A tick with the scenario's distro, hosts and running tasks, and a queue shaped like its DistroQueueInfo: per
    TaskGroupInfo, Count tasks of ExpectedDuration / Count each in that group."""
    data = G.go_allocator_data(s, M.fetch_expected_duration)
    q = s["queue_info"]
    data.distro.planner_settings.target_time = q.get("MaxDurationThreshold", 0)
    tasks = []
    for g in q.get("TaskGroupInfos", []) or [{"Name": "", "Count": q.get("LengthWithDependenciesMet", 0),
                                             "ExpectedDuration": q.get("ExpectedDuration", 0)}]:
        parts = (g.get("Name", "").split("_") + ["", "", "", ""])[:4]
        n = g.get("Count", 0)
        for i in range(n):
            t = M.Task(id=f"{g.get('Name', '')}-{i}", expected_duration=g.get("ExpectedDuration", 0) // max(n, 1),
                       scheduled_time=s["now"] - M.MINUTE)
            if parts[0]:
                t.task_group, t.build_variant, t.project, t.version = parts
                t.task_group_max_hosts = g.get("MaxHosts", 0)
            tasks.append(t)
    return data.distro, tasks, data


@pytest.mark.parametrize("setting", ["plain", "single", "terminate", "terminate_hourly"])
def test_allocator_scenarios(engine, setting):
    batch = [scenario_tick(s) for s in ALLOC["scenarios"]]
    assert len(batch) == 23
    for d, _, data in batch:
        d.single_task_distro = setting == "single"
        d.host_allocator_settings.hosts_overallocated_rule = M.HOSTS_OVERALLOCATED_TERMINATE if "terminate" in setting else ""
        d.arch = "osx" if setting == "terminate_hourly" else "linux"
    datas = [h for _, _, h in batch]
    soa, table, keys = S.marshal_tasks([(d, t) for d, t, _ in batch], ALLOC["now"])
    hosts = S.marshal_hosts(datas, [k.group_names for k in keys])
    engine.upload(soa, table, hosts)
    engine.run(ALLOC["now"])
    po, ao = engine.download(want_alloc=True)
    cfg = S.marshal_host_job(datas, [i % 3 for i in range(len(datas))])
    for spawned in (None, np.arange(len(datas), dtype=np.int32) % 4):
        res = engine.host_job(cfg, spawned)
        for i, (d, _, data) in enumerate(batch):
            ga, gb = int(table.group_off[i]), int(table.group_off[i + 1])
            info = scheduler._queue_info_from_rows(po.info[i], po.group_info[ga:gb], keys[i].group_names)
            alloc = (int(ao.result[i]["new_hosts"]), int(ao.result[i]["free_hosts"]), int(ao.status[i]))
            want = OJ.host_allocator_job(d, info, len(data.existing_hosts), i % 3, alloc, None if spawned is None else int(spawned[i]))
            got = {"n_hosts": int(res["n_hosts"][i]), "n_hosts_free": int(res["n_hosts_free"][i]), "status": int(res["status"][i]),
                   "report": {f: res["report"][i][f] for f in L.HOST_REPORT_FIELDS}}
            assert_job(got, want, ALLOC["scenarios"][i]["test"])


# ------------------------------------------------------------------------------------------------ synthetic ticks
@pytest.mark.parametrize("k,scale", [(4, 0.2), (5, 0.1)])
def test_synthetic_configs(engine, k, scale):
    w = synth.config(k, scale)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    check(engine, w.distros.group_off, w.hosts, 1400 + k)


def test_warp_and_thread_distros(engine):
    """Distros with many task-group slots (summed by their warp) beside ones with few (one thread each)."""
    w = synth.make(np.array([6000, 40, 3000, 9, 700, 13000, 1]), 1410, tg_frac=0.6, n_hosts=60)
    slots = np.diff(w.distros.group_off)
    assert (slots > 16).any() and (slots <= 16).any()
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    check(engine, w.distros.group_off, w.hosts, 1411)


@pytest.fixture(scope="module")
def world():
    w, table, fin = candidates([300, 2000, 40, 5], 1420, "mixed")
    return dict(w=w, table=table, fin=fin, plain=synth.make(np.array([100, 40, 700]), 1421, tg_frac=0.1, n_hosts=10),
                big=synth.make(np.full(8, 280_000), 1422, tg_frac=0.1, n_hosts=100))


def test_after_upload_with_deps(engine, world):
    w = world["w"]
    engine.upload_with_deps(w.tasks, w.distros, w.hosts, world["table"].deps, world["fin"], w.now)
    engine.run(w.now)
    check(engine, w.distros.group_off, w.hosts, 1430)


def test_after_edit(engine, world):
    w = world["w"]
    engine.upload(w.tasks, w.distros, w.hosts)
    e = synth.next_tick(w, 1431)
    engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
    engine.run(w.now)
    check(engine, e.workload.distros.group_off, e.workload.hosts, 1432)


def test_after_plan_from_finder(engine, world):
    w = world["w"]
    engine.plan_from_finder(world["table"], w.tasks, w.distros, w.hosts, world["fin"], w.now)
    engine.run(w.now)
    check(engine, w.distros.group_off, w.hosts, 1433)


@pytest.mark.parametrize("which", ["plain", "big"])
def test_after_plan_and_alloc_batch(engine, world, which):
    """The one-shot call, and its pipelined path (at least 2^21 tasks)."""
    w = world[which]
    po, ao = engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now)
    assert which == "plain" or w.n_tasks >= 1 << 21
    check(engine, w.distros.group_off, w.hosts, 1434, po, ao)


def test_after_upload_device(engine, world):
    import torch
    w = world["plain"]
    cols = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dt)])).cuda() for name, dt in S.TaskSoA.COLUMNS}
    engine.upload_device({k: v.data_ptr() for k, v in cols.items()}, w.n_tasks, w.distros, w.hosts)
    engine.run(w.now)
    check(engine, w.distros.group_off, w.hosts, 1435)
    torch.cuda.synchronize()
    del cols


def test_bound_result_buffer(engine, world):
    import torch
    w = world["plain"]
    D = w.distros.n_distros
    buf = torch.zeros(D * L.ALLOC_RESULT_DTYPE.itemsize + 64, dtype=torch.uint8, device="cuda")
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.bind_result_buffer(buf.data_ptr(), D)
    try:
        engine.run(w.now)
        check(engine, w.distros.group_off, w.hosts, 1436)
        rows = buf[:D * 16].cpu().numpy().view(L.ALLOC_RESULT_DTYPE)
        po, ao = engine.download(want_alloc=True)
        assert np.array_equal(rows, ao.result)
    finally:
        engine.bind_result_buffer(0, 0)


def test_tick_is_only_read(engine, world):
    w = world["w"]
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    po, ao = engine.download(want_alloc=True)
    before = [a.copy() for a in (po.order, po.total_value, po.info, po.group_info, ao.result, ao.status)]
    cfg = job_cfg(w.distros.n_distros, 1440)
    first = {k: v.copy() for k, v in engine.host_job(cfg).items()}
    second = engine.host_job(cfg)
    for k in first:
        assert np.array_equal(first[k].view(np.uint8), second[k].view(np.uint8)), k
    po, ao = engine.download(want_alloc=True)
    after = (po.order, po.total_value, po.info, po.group_info, ao.result, ao.status)
    for a, b in zip(before, after):
        assert np.array_equal(a, b)
    e = synth.next_tick(w, 1441)
    engine.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)  # still the editable tick it was


def test_error_contract(world):
    p = world["plain"]
    eng = scheduler.Engine(0)
    try:
        D = p.distros.n_distros
        cfg = job_cfg(D, 1450)
        out = {k: np.zeros(D, dt) for k, dt in (("n_hosts", np.int64), ("n_hosts_free", np.int64), ("status", np.int32),
                                                ("report", L.HOST_REPORT_DTYPE))}
        st = L.HostJobOutStruct(*[L.ptr(out[f]) for f in ("n_hosts", "n_hosts_free", "status", "report")])
        call = lambda c=cfg, o=st, sp=None: eng.lib.evg_host_job(eng.ctx, L.ptr(c) if c is not None else None,  # noqa: E731
                                                                   L.ptr(sp) if sp is not None else None,
                                                                   C.byref(o) if o is not None else None)
        assert call() == L.EVG_ERR_STATE  # no tick
        eng.upload(p.tasks, p.distros)
        eng.run(p.now)
        assert call() == L.EVG_ERR_STATE  # no hosts
        eng.upload(p.tasks, p.distros, p.hosts)
        assert call() == L.EVG_ERR_STATE  # no run since the tick was set
        assert "since it was set" in L.last_error()
        eng.run(p.now)
        assert call(c=None) == L.EVG_ERR_INVALID and call(o=None) == L.EVG_ERR_INVALID
        assert call(o=L.HostJobOutStruct()) == L.EVG_ERR_INVALID
        neg = cfg.copy()
        neg["n_provisioning"][1] = -1
        assert call(c=neg) == L.EVG_ERR_INVALID and "n_provisioning" in L.last_error()
        assert call() == L.EVG_OK
        sp = np.full(D, 2, np.int32)
        sp[D - 1] = -1  # len(hostsSpawned) is never negative
        assert call(sp=sp) == L.EVG_ERR_INVALID and f"spawned[{D - 1}]" in L.last_error()
        iw = synth.make_idle_hosts(np.full(D, 3), 1451)  # the rejected call left the last reports for a chained drawdown
        eng.host_drawdown(S.marshal_idle_hosts(iw.groups), np.asarray(iw.existing, np.int64), iw.now)
        assert call(sp=sp + 1) == L.EVG_OK
        eng.bind_result_buffer(0, 0)
        assert call() == L.EVG_ERR_STATE  # the run's rows are not in the buffer bound now
        eng.run(p.now)
        assert call() == L.EVG_OK
        po, _ = eng.download()
        eng.alloc_batch(p.hosts, po.info.copy(), po.group_info.copy(), p.distros.group_off, p.now)
        assert call() == L.EVG_ERR_STATE  # evg_alloc_batch ended the tick
        eng.plan_and_alloc_batch(p.tasks, p.distros, p.hosts, p.now)
        assert call() == L.EVG_OK
        eng.plan_batch(p.tasks, p.distros, p.now)
        assert call() == L.EVG_ERR_STATE  # planner only
    finally:
        eng.close()
