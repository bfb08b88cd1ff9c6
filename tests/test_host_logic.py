"""Host-side logic of the shim mirror (no GPU): marshalling, dependency and
duration restatements against the oracle, sharding, the synthetic generator."""
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import dist as edist
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle as O

NOW = synth.NOW_NS


def random_tasks(rng, n, n_ext=5):
    tasks = []
    for i in range(n):
        t = M.Task(id=f"t{i}", version=f"v{rng.randrange(3)}", project="p", build_variant=f"bv{rng.randrange(2)}",
                   priority=rng.choice([0, 0, 1, 50, -1]), requester=rng.choice(["gitter_request", "patch_request",
                   "github_pull_request", "github_merge_request", "ad_hoc", "trigger_request"]),
                   activated_by=rng.choice(["", "stepback", "user"]), generate_task=rng.random() < 0.1,
                   num_dependents=rng.randrange(4), distro_id=rng.choice(["d", "d", "other"]),
                   activated_time=rng.choice([M.ZERO_TIME, 0, NOW - rng.randrange(10 ** 13)]),
                   ingest_time=rng.choice([M.ZERO_TIME, NOW - rng.randrange(10 ** 13)]),
                   scheduled_time=rng.choice([M.ZERO_TIME, NOW - rng.randrange(10 ** 12)]),
                   dependencies_met_time=rng.choice([M.ZERO_TIME, M.ZERO_TIME, 0, NOW - rng.randrange(10 ** 12)]),
                   override_dependencies=rng.random() < 0.1)
        if rng.random() < 0.3:
            g = rng.randrange(2)
            # TaskGroupMaxHosts is a property of the group (per build variant / version): uniform inside one TaskGroupString
            t.task_group, t.task_group_order = f"tg{g}", rng.randrange(5)
            t.task_group_max_hosts = 1 + (g + int(t.version[1:]) + int(t.build_variant[2:])) % 3
        for _ in range(rng.choice([0, 0, 1, 2])):
            target = rng.choice([f"t{rng.randrange(n)}", f"ext{rng.randrange(n_ext)}", "missing"])
            t.depends_on.append(M.Dependency(target, status=rng.choice(["", "success", "failed", "*"]),
                                             unattainable=rng.random() < 0.1))
        tasks.append(t)
    db = {f"ext{k}": M.Task(id=f"ext{k}", status=rng.choice(["success", "failed", "undispatched", "started"]),
                            depends_on=[M.Dependency("x", unattainable=rng.random() < 0.5)]) for k in range(n_ext)}
    return tasks, db


@pytest.mark.parametrize("seed", range(5))
def test_dependencies_met_restatement_matches_oracle(seed):
    rng = random.Random(seed)
    tasks, db = random_tasks(rng, 60)
    by_id = {t.id: t for t in tasks}
    mine = [S.dependencies_met(t, by_id, db) for t in tasks]
    assert mine == O.deps_met(tasks, NOW, db).tolist()


@pytest.mark.parametrize("seed", range(3))
def test_marshal_tasks_columns(seed):
    rng = random.Random(100 + seed)
    tasks, db = random_tasks(rng, 50)
    d = M.Distro(id="d", dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
    soa, table, keys = S.marshal_tasks([(d, tasks)], NOW, db)
    assert soa.n_tasks == 50 and table.n_distros == 1 and int(table.cfg[0]["includes_dependencies"]) == 1
    names = keys[0].group_names
    for i, t in enumerate(tasks):
        g = int(soa.group_id[i])
        assert (g == -1) == (t.task_group == "")
        if g >= 0:
            assert names[g] == t.get_task_group_string()
            assert int(table.group_max_hosts[g]) == tasks[[x.get_task_group_string() if x.task_group else None for x in tasks].index(names[g])].task_group_max_hosts
        assert keys[0].versions[int(soa.version_id[i])] == t.version
        qb = t.activated_time if t.activated_time != M.ZERO_TIME else t.ingest_time
        assert int(soa.queue_basis_ns[i]) == qb
        assert int(soa.wait_basis_ns[i]) == max(t.scheduled_time, t.dependencies_met_time)
        fl = int(soa.flags[i])
        assert (fl & 3) == (2 if t.requester == "github_merge_request" else 1 if t.requester in ("patch_request", "github_pull_request") else 0)
        assert bool(fl & L.EVG_TF_GENERATE) == t.generate_task
        assert bool(fl & L.EVG_TF_STEPBACK) == (t.activated_by == "stepback")
        assert bool(fl & L.EVG_TF_OTHER_DISTRO) == (t.distro_id != "d")
        assert int(soa.expected_ns[i]) == M.DEFAULT_TASK_DURATION
    # in-queue edges only, in DependsOn order
    if soa.dep_idx is not None:
        for i, t in enumerate(tasks):
            want = [int(x.task_id[1:]) for x in t.depends_on if x.task_id.startswith("t")]
            assert soa.dep_idx[int(soa.dep_off[i]):int(soa.dep_off[i + 1])].tolist() == want


def test_fetch_expected_duration_restatement_matches_oracle():
    rng = random.Random(3)
    for _ in range(300):
        t = M.Task(id="x", expected_duration=rng.choice([0, 0, 5 * M.MINUTE]), expected_duration_std_dev=rng.choice([0, M.MINUTE]),
                   duration_prediction=M.CachedDurationValue(value=rng.choice([0, 7 * M.MINUTE]), std_dev=rng.choice([0, M.SECOND]),
                                                             ttl=rng.choice([0, M.HOUR, 24 * M.HOUR]),
                                                             collected_at=rng.choice([M.ZERO_TIME, NOW, NOW - 2 * M.HOUR, NOW - 9 * M.HOUR])))
        hist = rng.choice([None, (0, 0), (13 * M.MINUTE, 2 * M.MINUTE)])
        import copy
        want = O.fetch_expected_duration(copy.deepcopy(t), NOW, hist)
        assert M.fetch_expected_duration(t, NOW, hist) == want


def test_marshal_hosts_buckets_like_group_by_task_group():
    infos = [M.TaskGroupInfo("g1_bv_p_v", count=2), M.TaskGroupInfo("", count=1), M.TaskGroupInfo("g2_bv_p_v", count=1)]
    hosts = [M.Host("h0"), M.Host("h1", running_task="a", running_task_group="g1", running_task_build_variant="bv",
                                  running_task_project="p", running_task_version="v"),
             M.Host("h2", running_task="b"), M.Host("h3", running_task_group="g1"),
             M.Host("h4", running_task="c", running_task_group="gone"),
             M.Host("h5", task_group_teardown_start_time=5)]
    qi = M.DistroQueueInfo(task_group_infos=infos)
    data = M.HostAllocatorData(M.Distro(id="d", provider="ec2-fleet"), hosts, qi,
                               running_tasks={"a": M.RunningTaskStats(True, 10, 1, NOW - 5), "b": M.RunningTaskStats(False)})
    q, g, goff, names = S.queue_info_rows([qi])
    assert names == [["g1_bv_p_v", "g2_bv_p_v"]] and int(q[0]["has_ungrouped"]) == 1 and goff.tolist() == [0, 2]
    h = S.marshal_hosts([data], names)
    assert h.group_id.tolist() == [-1, 0, -1, -1, -2, -1]
    assert h.flags.tolist() == [0, L.EVG_HF_RUNNING | L.EVG_HF_RT_FOUND, L.EVG_HF_RUNNING, 0, L.EVG_HF_RUNNING, L.EVG_HF_TEARDOWN]
    buckets = O.group_by_task_group(hosts, infos)
    assert sorted(buckets) == ["", "g1_bv_p_v", "g2_bv_p_v", "gone___"]
    assert buckets["g1_bv_p_v"][0] == [1] and buckets[""][0] == [0, 2, 3, 5]


def test_lpt_partition():
    rng = synth.Rng(5)
    sizes = synth.power_law_sizes(rng, 3000)
    for world in (1, 2, 4, 8):
        sh = edist.lpt_partition(sizes, world)
        assert sorted(np.concatenate(sh.members).tolist()) == list(range(3000))
        assert np.array_equal(sh.load, [int(sizes[m].sum()) for m in sh.members])
        for r, m in enumerate(sh.members):
            assert np.all(sh.owner[m] == r) and np.array_equal(sh.slot[m], np.arange(len(m)))
        assert sh.load.max() <= max(sizes.max(), int(np.ceil(sizes.sum() / world)) + sizes.max())
    sh = edist.lpt_partition(np.full(16, 10), 8)
    assert sh.load.tolist() == [20] * 8
    sh = edist.lpt_partition([100, 1, 1, 1], 2)
    assert sorted(sh.load.tolist()) == [3, 100]


def test_synth_is_deterministic_and_well_formed():
    a, b = synth.config(5, 0.01), synth.config(5, 0.01)
    for name, _ in a.tasks.COLUMNS:
        assert np.array_equal(getattr(a.tasks, name), getattr(b.tasks, name))
    t, d = a.tasks, a.distros
    sizes = np.diff(d.task_off)
    distro_of = np.repeat(np.arange(d.n_distros), sizes)
    assert np.all(t.group_id < (d.group_off[1:] - d.group_off[:-1])[distro_of])
    assert np.all(t.version_id < d.cfg["n_versions"][distro_of])
    assert np.all(t.dep_idx < sizes[distro_of][np.repeat(np.arange(t.n_tasks), np.diff(t.dep_off))])
    # a task group lives in one version
    key = distro_of[t.group_id >= 0].astype(np.int64) * (1 << 32) + t.group_id[t.group_id >= 0]
    ver = t.version_id[t.group_id >= 0]
    order = np.argsort(key, kind="stable")
    same = key[order][1:] == key[order][:-1]
    assert np.all(ver[order][1:][same] == ver[order][:-1][same])
    assert a.algorithmic_bytes() == 60 * t.n_tasks + 4 * t.n_edges + 28 * a.hosts.n_hosts + 96 * d.n_groups + 16 * d.n_distros


def test_intern_columns_equals_the_python_marshaller():
    """evg_intern_columns (host C++ behind the ABI): group ids, version ids, group offsets, per-group MaxHosts, version
    counts and the in-queue dependency CSR equal what soa.marshal_tasks builds with Python dicts -- for 1 and 5 threads,
    with empty distros, repeated versions, dependencies outside the queue; mismatching TaskGroupMaxHosts is an error."""
    rng = random.Random(11)
    batch = []
    for d, n in enumerate([0, 1, 40, 700, 0, 2500, 13]):
        tasks, _ = random_tasks(rng, n)
        for t in tasks:
            t.id = f"d{d}-{t.id}"
            for dep in t.depends_on:
                if dep.task_id.startswith("t"):
                    dep.task_id = f"d{d}-{dep.task_id}"
        batch.append((M.Distro(id=f"d{d}"), tasks))
    soa, table, keys = S.marshal_tasks(batch, 10 ** 18)
    for threads in (1, 5):
        got = S.intern_columns(batch, threads)
        assert np.array_equal(got["group_id"], soa.group_id) and np.array_equal(got["version_id"], soa.version_id)
        assert np.array_equal(got["group_off"], table.group_off) and np.array_equal(got["group_max_hosts"], table.group_max_hosts)
        assert got["n_versions"].tolist() == [len(k.versions) for k in keys]
        want_off = soa.dep_off if soa.dep_off is not None else np.zeros(soa.n_tasks + 1, np.int64)
        assert np.array_equal(got["dep_off"], want_off)
        if soa.dep_idx is not None:
            assert np.array_equal(got["dep_idx"], soa.dep_idx)
        flat = [t for _, ts in batch for t in ts]
        assert [flat[int(r)].get_task_group_string() for r in got["group_first"]] == [n for k in keys for n in k.group_names]
    assert int(got["dep_off"][-1]) > 50 and int(got["group_off"][-1]) > 20
    grouped = [t for t in batch[5][1] if t.task_group != ""]
    twin = [t for t in grouped if t.get_task_group_string() == grouped[0].get_task_group_string()]
    assert len(twin) > 1
    twin[-1].task_group_max_hosts += 1
    with pytest.raises(L.EvgError):
        S.intern_columns(batch, 3)
    assert S.intern_columns([], 1)["group_off"].tolist() == [0]
    # a dep_off that decreases is refused before any row is read (its rows would outrun the caller's dep_idx)
    assert intern_raw(np.array([0, 2, 4]), np.array([0, 2, 2, 3, 3])) == L.EVG_OK
    assert intern_raw(np.array([0, 2, 4]), np.array([0, 2, 1, 2, 3])) == L.EVG_ERR_INVALID
    assert "evg_intern_columns" in L.last_error() and "dep_off" in L.last_error()


def intern_raw(task_off, dep_off):
    """evg_intern_columns over tasks t0, t1, ... cut by `task_off`, every dependency on t0, with `dep_off` as given."""
    task_off, dep_off = task_off.astype(np.int64), dep_off.astype(np.int64)
    T, D, E = len(dep_off) - 1, len(task_off) - 1, int(dep_off.max())
    ids, blank, dep = S.pack_strings([f"t{i}" for i in range(T)]), S.pack_strings([""] * T), S.pack_strings(["t0"] * E)
    col = lambda s: L.StrColStruct(L.ptr(s[0]) if s[0].shape[0] else None, L.ptr(s[1]))  # noqa: E731
    gmax = np.zeros(T, np.int32)
    ins = L.StringColsStruct(T, D, L.ptr(task_off), col(ids), col(ids), col(blank), L.ptr(gmax), L.ptr(dep_off), col(dep))
    out = [np.zeros(n, dt) for n, dt in ((T, np.int32), (T, np.int32), (D + 1, np.int64), (D, np.int32), (T, np.int32),
                                         (T, np.int64), (T + 1, np.int64), (E, np.int32))]
    import ctypes as C
    return L.load().evg_intern_columns(C.byref(ins), C.byref(L.InternOutStruct(*[L.ptr(o) for o in out])), 1)


def test_take_distros_is_the_same_tick_per_distro():
    """synth.take_distros (what a rank of the sharded bench uploads): the oracle plans a distro of the sub-tick exactly as it
    plans it inside the whole tick -- order, TotalValue, allocator decision."""
    w = synth.make(np.array([50, 0, 300, 7, 1200, 90]), 5, zipf_priority=True, tg_frac=0.2, met_dep_frac=0.05, unmet_dep_frac=0.05,
                   group_versions_frac=0.3, includes_dependencies=True, n_hosts=30)
    ids = np.array([4, 0, 2, 5, 1])
    s = synth.take_distros(w, ids)
    ref = O.SoAJob(w.tasks, w.distros, w.hosts, None).run(w.now, 4)
    sub = O.SoAJob(s.tasks, s.distros, s.hosts, None).run(s.now, 4)
    for j, d in enumerate(ids):
        a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
        a2, b2 = int(s.distros.task_off[j]), int(s.distros.task_off[j + 1])
        assert np.array_equal(ref["order"][a:b], sub["order"][a2:b2]) and np.array_equal(ref["total_value"][a:b], sub["total_value"][a2:b2])
        assert (int(ref["new_hosts"][d]), int(ref["free_hosts"][d])) == (int(sub["new_hosts"][j]), int(sub["free_hosts"][j]))


def test_score_fast_paths_equal_the_fp64_formulas(tmp_path):
    """evg_score.cuh replaces Duration.Minutes()/Hours() FP64 arithmetic by integer quotients on a proven
    range; brute-force the equivalence on the host (same header the kernels compile)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "check"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", root, "-o", str(exe),
                           os.path.join(root, "tests", "native", "score_fastpath_check.cpp")])
    out = subprocess.check_output([str(exe)]).decode()
    assert "mismatches 0" in out, out


# ---------------------------------------------------------------- the scorer's warp votes, restated
FAST_LIMIT = np.uint64((1 << 15) * M.MINUTE)


def scorer_domains(w):
    """numpy restatement of the kernels' per-task domain tests (evg_score.cuh): `bad32` is score32_bad != 0 with the
    NumDependents term resolved as k_gtask / k_plan_cta do (the per-distro table int64(factor * n) for n < 64, capped
    at 2^29; factor * n with an integral factor below 2^14 for 64 <= n < 2^15; else not representable); `fast` is
    score_fast_domain.  Also per distro: Factors32::ok_base (the 32-bit vote can pass) and the 64-bit fast form's
    preconditions."""
    t, dt, now = w.tasks, w.distros, int(w.now)
    cfg, D = dt.cfg, dt.n_distros
    sizes = np.diff(dt.task_off)
    distro_of = np.repeat(np.arange(D), sizes)
    ints = np.stack([np.where(cfg[f] > 0, cfg[f], 1) for f in synth._INT_FACTORS])
    ok_base = (now >= 0) & np.all(ints < 2 ** 14, axis=0)
    ndf = np.where(cfg["num_dependents_factor"] > 0, cfg["num_dependents_factor"], 1.0)
    nd_int = np.where((ndf < 2.0 ** 20) & (ndf == np.trunc(ndf)), np.trunc(ndf), 0).astype(np.int64)
    ok = ok_base & (nd_int != 0) & (nd_int < 2 ** 14)
    entry = np.trunc(ndf[:, None] * np.arange(64, dtype=np.float64)[None, :])
    table = np.where((entry >= 0) & (entry < 2 ** 29), entry, 0xFFFFFFFF).astype(np.int64)
    ndc = np.maximum(t.num_dependents, 0).astype(np.int64)
    mul = np.where(ok[distro_of] & (ndc < 2 ** 15), nd_int[distro_of] * ndc, 0xFFFFFFFF)
    nd_term = np.where(ndc < 64, table[distro_of, np.minimum(ndc, 63)], mul)
    qb = t.queue_basis_ns
    with np.errstate(over="ignore"):
        tiq = np.where(qb == M.ZERO_TIME, np.uint64(0), np.uint64(now % 2 ** 64) - qb.view(np.uint64))
    ex = t.expected_ns.view(np.uint64)
    bad32 = (((tiq | ex) >> np.uint64(50)) != 0) | ((np.maximum(t.priority, 0) >> 15) != 0) | ((nd_term >> 29) != 0)
    fast = ((qb == M.ZERO_TIME) | ((qb >= 0) & (tiq < FAST_LIMIT))) & (ex < FAST_LIMIT)
    fast_clock = np.full(D, now >= 0) & (nd_int != 0)
    return distro_of, bad32, fast, ok_base, fast_clock


def scoring_tasks(w, route):
    """Tasks that vote: those whose own unit is {the task} (the rest are scored as units)."""
    t, dt = w.tasks, w.distros
    D = dt.n_distros
    sizes = np.diff(dt.task_off)
    distro_of = np.repeat(np.arange(D), sizes)
    has_dependents = np.zeros(t.n_tasks, dtype=bool)
    edges = np.zeros(D, dtype=bool)
    if t.n_edges:
        owner = np.repeat(np.arange(t.n_tasks), np.diff(t.dep_off))
        has_dependents[dt.task_off[distro_of[owner]] + t.dep_idx] = True
        edges = np.bincount(distro_of[owner], minlength=D) > 0
    gv = dt.cfg["group_versions"] != 0
    complex_distro = (np.diff(dt.group_off) > 0) | gv | edges
    if route == "warp":  # k_plan_warp votes only in distros without multi-member units
        return ~complex_distro[distro_of]
    return ~(complex_distro[distro_of] & ((t.group_id >= 0) | gv[distro_of] | has_dependents))


def vote_groups(w, route):
    """Per task: the (distro, warp vote) it takes part in, as one integer, for each kernel's lane layout.
      k_plan_warp  one warp per distro
      k_plan_smem  task i of a distro is lane i % 32 of a warp covering tasks 32*(i // 32) ..
      k_plan_cta   tile k holds slots a0 + k*2*THREADS .., a0 = the distro's first task rounded down to a multiple of 4;
                   slot j of a tile is lane j % 32 of warp (j % THREADS) // 32, whose vote spans both THREADS halves
      k_gtask      2048-slot tiles from a0; thread q of half u owns slots 4*(u*256 + q) .. +3: a warp votes on 128
                   consecutive slots"""
    import test_gpu_score_edges as E
    dt = w.distros
    sizes = np.diff(dt.task_off)
    distro_of = np.repeat(np.arange(dt.n_distros), sizes)
    s = np.arange(w.n_tasks, dtype=np.int64)
    a = dt.task_off[distro_of]
    rel = s - (a & ~3)
    if route == "warp":
        g = np.zeros_like(s)
    elif route == "smem":
        g = (s - a) // 32
    elif route == "cta":
        th = np.array([E.cta_threads(int(n)) for n in sizes], dtype=np.int64)[distro_of]
        g = (rel // (2 * th)) * 64 + (rel % th) // 32
    else:
        g = rel // E.GTASK_WARP
    return distro_of * (1 << 24) + g


def mixed_votes(w, route):
    """Number of warp votes on `route` where some voting tasks are inside the scorer's domain and some are not --
    the votes that send in-domain tasks down a fallback."""
    distro_of, bad32, fast, ok_base, fast_clock = scorer_domains(w)
    if route in ("cta", "general"):
        out, live = bad32, ok_base[distro_of]
    else:
        out, live = ~fast, fast_clock[distro_of]
    sel = scoring_tasks(w, route) & live
    g = vote_groups(w, route)[sel]
    o = out[sel]
    if g.size == 0:
        return 0
    ids, inv = np.unique(g, return_inverse=True)
    n_out = np.bincount(inv, weights=o.astype(np.float64))
    n_all = np.bincount(inv)
    return int(((n_out > 0) & (n_out < n_all)).sum())


@pytest.mark.parametrize("route", ["warp", "cta", "smem", "general"])
def test_score_edge_ticks_hold_mixed_warps(route):
    """Every edge tick of test_gpu_score_edges.py (except the `thresh` kind, whose values are inside the domain by
    design) holds mixed warp votes on its route, and its edges reach task-group members (and GroupVersions members
    where the route has such distros); the undisturbed ticks hold none -- so the GPU tests cannot drift back into the
    32-bit scorer's domain unnoticed."""
    import test_gpu_score_edges as E
    assert mixed_votes(E._route_tick(route, 500), route) == 0
    # the 64-bit fast form of k_plan_warp / k_plan_smem takes any priority and NumDependents: only times leave its domain
    leaves = ("tiq", "basis", "exp", "wrap") if route in ("warp", "smem") else tuple(k for k in E.KINDS if k != "thresh")
    for density in E.DENSITIES:
        for kind in E.KINDS:
            w = E.edge_tick(route, kind, density)
            if kind in leaves:
                assert mixed_votes(w, route) > 0, (route, kind, density)
            seed = 500 + 17 * E.ROUTES.index(route) + E.KINDS.index(kind)
            base = E._route_tick(route, seed)
            changed = np.zeros(w.n_tasks, dtype=bool)
            for name, _ in w.tasks.COLUMNS:
                changed |= getattr(w.tasks, name) != getattr(base.tasks, name)
            assert changed.any(), (route, kind, density)
            if kind == "u32":  # lone tasks only: the value of a unit would add its other members' terms
                continue
            assert (changed & (w.tasks.group_id >= 0)).any(), (route, kind, density)
            gv = (w.distros.cfg["group_versions"] != 0)[np.repeat(np.arange(w.distros.n_distros), np.diff(w.distros.task_off))]
            if route != "cta":  # k_plan_cta plans no GroupVersions distro
                assert (changed & gv).any(), (route, kind, density)


def test_scorer_domain_restatement_sees_each_limit():
    """The restatement flags exactly the values past each limit of score32_bad."""
    w = synth.make(np.array([40]), 3, tg_frac=0.0)
    t, now = w.tasks, w.now
    t.num_dependents[:] = 1
    t.priority[:] = 0
    t.expected_ns[:] = M.MINUTE
    t.queue_basis_ns[:] = now
    t.queue_basis_ns[1], t.queue_basis_ns[2] = now - (2 ** 50 - 1), now - 2 ** 50
    t.expected_ns[3], t.expected_ns[4], t.expected_ns[5] = 2 ** 50 - 1, 2 ** 50, -1
    t.priority[6], t.priority[7], t.priority[8] = 2 ** 15 - 1, 2 ** 15, -2 ** 31
    t.num_dependents[9], t.num_dependents[10] = 2 ** 15 - 1, 2 ** 15
    t.queue_basis_ns[11], t.queue_basis_ns[12] = now + 1, M.ZERO_TIME
    w.distros.cfg["num_dependents_factor"] = 7.0
    w.distros.cfg["patch_factor"] = 0
    _, bad, fast, ok_base, _ = scorer_domains(w)
    assert bool(ok_base[0])
    assert np.nonzero(bad[:13])[0].tolist() == [2, 4, 5, 7, 10, 11]  # 7 * (2^15 - 1) < 2^29; 7 * 2^15 needs n < 2^15
    w.distros.cfg["num_dependents_factor"] = 2.5  # fractional: only the table (n < 64) keeps the 32-bit form
    _, bad, _, _, _ = scorer_domains(w)
    assert np.nonzero(bad[:13])[0].tolist() == [2, 4, 5, 7, 9, 10, 11]
    w.distros.cfg["num_dependents_factor"] = 2.0 ** 27 + 0.5  # table entries reach 2^29 at n = 4
    t.num_dependents[13:16] = [3, 4, 32]
    _, bad, _, _, _ = scorer_domains(w)
    assert bad[14] and bad[15] and not bad[13]


def test_sprinkle_edges_keeps_make_and_the_tick_valid():
    """The injector draws from a stream of its own (make() is unchanged for every seed), writes every value of every
    kind, and leaves group ids, versions and TaskGroupMaxHosts alone."""
    a = synth.make(np.array([300, 2000, 40]), 12, tg_frac=0.2, zipf_priority=True)
    b = synth.make(np.array([300, 2000, 40]), 12, tg_frac=0.2, zipf_priority=True)
    written = synth.sprinkle_edges(b, 12, kinds=synth.ROW_KINDS + synth.DISTRO_KINDS, frac=0.5)
    c = synth.make(np.array([300, 2000, 40]), 12, tg_frac=0.2, zipf_priority=True)
    for name, _ in a.tasks.COLUMNS:
        assert np.array_equal(getattr(a.tasks, name), getattr(c.tasks, name))
    for name in ("group_id", "version_id", "task_group_order"):
        assert np.array_equal(getattr(a.tasks, name), getattr(b.tasks, name))
    assert np.array_equal(a.distros.group_max_hosts, b.distros.group_max_hosts)
    t = b.tasks
    assert set(synth.EDGE_VALUES["nd"]) <= set(t.num_dependents[written["nd"]].tolist())
    assert set(synth.EDGE_VALUES["prio"]) <= set(t.priority[written["prio"]].tolist())
    assert set(synth.EDGE_VALUES["exp"]) <= set(t.expected_ns[written["exp"]].tolist())
    assert {b.now - v for v in synth.EDGE_VALUES["tiq"]} <= set(t.queue_basis_ns[written["tiq"]].tolist())
    assert {b.now + 1, 0, -2 ** 63 + 1, M.ZERO_TIME} <= set(t.queue_basis_ns[written["basis"]].tolist())
    assert int(b.distros.cfg["target_time_ns"][2]) > b.now
    # marshal_tasks takes the int32 edges and refuses what does not fit
    d = M.Distro(id="d")
    soa, _, _ = S.marshal_tasks([(d, [M.Task(id="t", num_dependents=2 ** 31 - 1, priority=-2 ** 31)])], NOW)
    assert soa.num_dependents.tolist() == [2 ** 31 - 1]
    with pytest.raises(ValueError):
        S.marshal_tasks([(d, [M.Task(id="t", num_dependents=2 ** 31)])], NOW)


def test_marshal_runnable_bits():
    """soa.marshal_runnable: the byte columns of evg_runnable_in against the reference's field semantics."""
    from evergreen_b200 import _lib as L
    from evergreen_b200 import soa
    refs = [M.ProjectRef(id="a", enabled=True), M.ProjectRef(id="b", hidden=True, patching_disabled=True)]
    tasks = [M.Task(id="x", project="a", requester="github_pull_request", priority=-1, execution_platform="container"),
             M.Task(id="y", project="zzz", activated=False, status="started", unattainable_dependency=True,
                    override_dependencies=True, requester="gitter_request",
                    depends_on=[M.Dependency("x", status="*")])]
    d = M.Distro(id="d", valid_projects=["b", "ghost"])
    t = soa.marshal_runnable([(d, tasks)], refs, "alternate")
    assert t.sched.tolist() == [L.EVG_SQ_ACTIVATED | L.EVG_SQ_UNDISPATCHED | L.EVG_SQ_GITHUB_PR | L.EVG_SQ_PATCH_REQUEST,
                                L.EVG_SQ_PRIORITY_OK | L.EVG_SQ_HOST_PLATFORM | L.EVG_SQ_UNATTAINABLE | L.EVG_SQ_OVERRIDE_DEPS]
    assert t.project.tolist() == [0, -1] and t.project_flags.tolist() == [L.EVG_PF_ENABLED, L.EVG_PF_HIDDEN | L.EVG_PF_PATCHING_DISABLED]
    assert t.valid_off.tolist() == [0, 2] and t.valid_idx.tolist() == [1, -1]
    assert t.finder.tolist() == [L.EVG_FINDER_ALTERNATE] and t.deps is not None and t.deps.dep_kind.tolist() == [L.EVG_DEP_IN_QUEUE]
    d2 = M.Distro(id="e", dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
    t2 = soa.marshal_runnable([(d2, tasks)], refs, "legacy")
    assert t2.finder.tolist() == [L.EVG_FINDER_NO_DEPS] and t2.deps is None


def test_lpt_partition_properties():
    """Whole distros, every distro exactly once, deterministic, and never worse than the classic LPT bound
    (max load <= mean load + heaviest distro)."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=150, deadline=None)
    @given(st.lists(st.integers(0, 2_000_000), min_size=0, max_size=300), st.integers(1, 8))
    def prop(weights, world):
        sh = edist.lpt_partition(weights, world)
        w = np.asarray(weights, dtype=np.int64)
        assert len(sh.members) == world
        seen = np.concatenate(sh.members) if len(weights) else np.zeros(0, dtype=np.int64)
        assert sorted(seen.tolist()) == list(range(len(weights)))
        for r, m in enumerate(sh.members):
            assert (sh.owner[m] == r).all() and (sh.slot[m] == np.arange(len(m))).all()
            assert int(w[m].sum()) == int(sh.load[r])
        if len(weights):
            assert int(sh.load.max()) <= int(np.ceil(w.sum() / world)) + int(w.max())
        again = edist.lpt_partition(weights, world)
        assert np.array_equal(again.owner, sh.owner) and np.array_equal(again.slot, sh.slot)

    prop()


def test_queue_info_rows_round_trip():
    """soa.queue_info_rows (DistroQueueInfo -> the 152 B / 72 B rows of the ABI) keeps every scalar and the slot
    order of the named task groups; the "" group becomes the embedded `ungrouped` row."""
    rng = random.Random(5)
    infos = []
    for d in range(6):
        groups = [M.TaskGroupInfo(name=n, count=rng.randrange(50), max_hosts=rng.randrange(4), expected_duration=rng.randrange(10 ** 12),
                                  count_duration_over_threshold=rng.randrange(5), count_wait_over_threshold=rng.randrange(5),
                                  count_dep_filled_merge_queue_tasks=rng.randrange(3), duration_over_threshold=rng.randrange(10 ** 11))
                  for n in rng.sample(["", "tg_a", "tg_b", "tg_c", "tg_d"], rng.randrange(0, 5))]
        infos.append(M.DistroQueueInfo(length=rng.randrange(1000), length_with_dependencies_met=rng.randrange(900),
                                       expected_duration=rng.randrange(10 ** 13), max_duration_threshold=30 * 60 * 10 ** 9,
                                       count_duration_over_threshold=rng.randrange(9), duration_over_threshold=rng.randrange(10 ** 12),
                                       count_wait_over_threshold=rng.randrange(9), count_dep_filled_merge_queue_tasks=rng.randrange(4),
                                       task_group_infos=groups))
    qrows, grows, goff, names = S.queue_info_rows(infos)
    assert qrows.shape[0] == 6 and goff.tolist()[0] == 0 and int(goff[-1]) == grows.shape[0]
    for d, qi in enumerate(infos):
        named = [g for g in qi.task_group_infos if g.name != ""]
        assert names[d] == [g.name for g in named]
        assert int(qrows[d]["length"]) == qi.length and int(qrows[d]["expected_duration"]) == qi.expected_duration
        assert int(qrows[d]["length_with_dependencies_met"]) == qi.length_with_dependencies_met
        unnamed = [g for g in qi.task_group_infos if g.name == ""]
        assert int(qrows[d]["has_ungrouped"]) == len(unnamed)
        if unnamed:
            assert int(qrows[d]["ungrouped"]["count"]) == unnamed[0].count
            assert int(qrows[d]["ungrouped"]["expected_duration"]) == unnamed[0].expected_duration
        for k, g in enumerate(named):
            row = grows[int(goff[d]) + k]
            for f in ("count", "max_hosts", "expected_duration", "count_duration_over_threshold", "count_wait_over_threshold",
                      "count_dep_filled_merge_queue_tasks", "duration_over_threshold"):
                assert int(row[f]) == getattr(g, f), (d, k, f)


def test_fresh_dependency_evaluation_stamps_the_met_time():
    """GetDistroQueueInfo measures the wait AFTER checkDependenciesMet ran on the task (scheduler.go:82-123), and a fresh
    evaluation that comes out met stamps DependenciesMetTime = latest non-zero dependency FinishedAt, else now
    (Task.DependenciesMet -> setDependenciesMetTime, model/task/task.go:653,673-684).  So a task seen for the first
    time with its dependencies met has waited since they finished -- not since it was scheduled."""
    sched = NOW - 3 * M.HOUR
    ext = {"e1": M.Task(id="e1", status=M.TASK_SUCCEEDED), "e2": M.Task(id="e2", status=M.TASK_SUCCEEDED)}

    def mk():
        return [
            M.Task(id="a", distro_id="d", scheduled_time=sched),                                    # no dependencies: HasDependenciesMet short-circuit
            M.Task(id="b", distro_id="d", scheduled_time=sched,
                   depends_on=[M.Dependency("e1", finished_at=NOW - 50 * M.MINUTE), M.Dependency("e2", finished_at=NOW - 20 * M.MINUTE)]),
            M.Task(id="c", distro_id="d", scheduled_time=sched, dependencies_met_time=NOW - 2 * M.HOUR),  # stamped on an earlier tick
            M.Task(id="d", distro_id="d", scheduled_time=sched, depends_on=[M.Dependency("missing")]),     # unmet
            M.Task(id="e", distro_id="d", scheduled_time=sched, depends_on=[M.Dependency("e1")]),           # met, FinishedAt unknown: now
            M.Task(id="f", distro_id="d", scheduled_time=sched, override_dependencies=True,
                   depends_on=[M.Dependency("missing", finished_at=NOW - M.MINUTE)]),                       # short-circuit: nothing stamped
        ]
    tasks = mk()
    d = M.Distro(id="d")
    soa, table, _ = S.marshal_tasks([(d, tasks)], NOW, ext, resolve_deps=True)
    assert soa.wait_basis_ns.tolist() == [sched, NOW - 20 * M.MINUTE, NOW - 2 * M.HOUR, sched, NOW, sched]
    assert [bool(f & L.EVG_TF_DEPS_MET) for f in soa.flags.tolist()] == [True, True, True, False, True, True]
    # the marshaller wrote the stamp back on the task, like tasks[i] = task (scheduler.go:137) / the UpdateOne of task.go:659
    assert [t.dependencies_met_time for t in tasks] == [M.ZERO_TIME, NOW - 20 * M.MINUTE, NOW - 2 * M.HOUR, M.ZERO_TIME, NOW, M.ZERO_TIME]
    qi = O.queue_info("d", mk(), 30 * M.MINUTE, False, NOW, ext)
    assert qi.count_wait_over_threshold == 3 and qi.length_with_dependencies_met == 5  # a and f (3 h since scheduled), c (2 h)
    # the same queue through the SoA-level oracle job the GPU parity tests use
    job = O.SoAJob(soa, table, None, None)
    ref = job.run(NOW, 1)
    assert int(ref["info"][0]["count_wait_over_threshold"]) == 3


def test_out_of_range_priority_is_an_error_not_a_clamp():
    d = M.Distro(id="d")
    for bad in (2 ** 31, -2 ** 31 - 1, 2 ** 40):
        with pytest.raises(ValueError):
            S.marshal_tasks([(d, [M.Task(id="t", priority=bad)])], NOW)
    soa, _, _ = S.marshal_tasks([(d, [M.Task(id="t", priority=2 ** 31 - 1), M.Task(id="u", priority=-2 ** 31)])], NOW)
    assert soa.priority.tolist() == [2 ** 31 - 1, -2 ** 31]


def test_task_group_max_hosts_must_agree_inside_a_group():
    d = M.Distro(id="d")
    a = M.Task(id="a", task_group="g", task_group_max_hosts=2, version="v", build_variant="bv", project="p")
    b = M.Task(id="b", task_group="g", task_group_max_hosts=3, version="v", build_variant="bv", project="p")
    with pytest.raises(ValueError):
        S.marshal_tasks([(d, [a, b])], NOW)
    b.task_group_max_hosts = 2
    _, table, _ = S.marshal_tasks([(d, [a, b])], NOW)
    assert table.group_max_hosts.tolist() == [2]
