"""Every reader of a resident tick at its edges: evg_host_job (and the chained evg_host_drawdown) and the persisted-queue
breakdown (evg_download_queue_breakdown), against the oracle and the restatements oracle_host_job and
oracle_host_termination.

A. The score-edge ticks of test_gpu_score_edges (every route, every row kind) with one narrow distro of task groups
   appended: the queue-breakdown rows against the oracle's breakdown, and evg_host_job under four job settings, with
   spawned NULL and given, against the restatement fed the device's plan rows and the oracle's.
B. k_host_job at its own edges, on crafted ticks whose landings test_tick_report_edges_host.py asserts on the CPU:
   thresholds of 0, -1, 1 and INT64_MAX and negative ones that saturate the killable count, ratios at and just below
   0.25f, killable products one float32 ulp from an integer, the MinimumHosts clamp, every branch of the time-to-empty
   calculation, single-task distros, spawned INT32_MAX, and the warp-sum layout (wide distros on every lane kind).
C. After every evg_host_job here, the chained evg_host_drawdown against oracle_host_termination fed the restatement's
   report, with drawdown targets <= 0, equal to the idle-host count and above it."""
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Callable, Optional, Sequence

import numpy as np
import pytest

import oracle_host_job as OJ
import oracle_host_termination as OT
import parity
import test_gpu_score_edges as SE
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_host_job import as_expect, job_cfg, restate
from test_gpu_host_termination import rows as verdict_rows
from test_gpu_queue_breakdown import check_tick
from test_host_job_host import assert_job

pytestmark = pytest.mark.gpu

I64_MAX, I32_MAX = 2 ** 63 - 1, 2 ** 31 - 1
BIG = 2 ** 62 + 1  # synth.EDGE_VALUES["exp"]: two of them wrap an int64 sum


# ------------------------------------------------------------------------------------------------ tick helpers
def concat(a: synth.Workload, b: synth.Workload) -> synth.Workload:
    """The distros of `a` followed by those of `b` (same clock, both with hosts): group ids, dependency indices and host
    group ids are distro-local, so only the offsets move."""
    ta, tb = a.tasks, b.tasks
    cols = {name: np.concatenate([getattr(ta, name), getattr(tb, name)]) for name, _ in S.TaskSoA.COLUMNS}
    dep_off = dep_idx = None
    if ta.n_edges or tb.n_edges:
        oa = ta.dep_off if ta.n_edges else np.zeros(ta.n_tasks + 1, np.int64)
        ob = tb.dep_off if tb.n_edges else np.zeros(tb.n_tasks + 1, np.int64)
        dep_off = np.concatenate([oa, ob[1:] + oa[-1]])
        dep_idx = np.concatenate([x.dep_idx for x in (ta, tb) if x.n_edges])
    tasks = S.TaskSoA(**cols, dep_off=dep_off, dep_idx=dep_idx).normalize()
    da, db = a.distros, b.distros
    distros = S.DistroTable(np.concatenate([da.task_off, db.task_off[1:] + da.task_off[-1]]),
                            np.concatenate([da.group_off, db.group_off[1:] + da.group_off[-1]]),
                            np.concatenate([da.cfg, db.cfg]), np.concatenate([da.group_max_hosts, db.group_max_hosts])).normalize()
    ha, hb = a.hosts, b.hosts
    hosts = S.HostSoA(*[np.concatenate([getattr(ha, n), getattr(hb, n)]) for n, _ in S.HostSoA.COLUMNS],
                      np.concatenate([ha.host_off, hb.host_off[1:] + ha.host_off[-1]]), np.concatenate([ha.cfg, hb.cfg])).normalize()
    return synth.Workload(f"{a.name} + {b.name}", a.now, tasks, distros, hosts)


def narrow_distros(w) -> list:
    t, dt = w.tasks, w.distros
    return [d for d in range(dt.n_distros) if not int(dt.cfg["group_versions"][d]) and
            (t.n_edges == 0 or t.dep_off[dt.task_off[d + 1]] == t.dep_off[dt.task_off[d]])]


def group_members(w, d) -> list:
    """Rows of each task-group slot of distro d."""
    a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
    gid = w.tasks.group_id[a:b]
    return [a + np.nonzero(gid == g)[0] for g in range(int(w.distros.group_off[d + 1] - w.distros.group_off[d]))]


# ------------------------------------------------------------------------------------------- A. score-edge ticks
DENSE_KINDS = ("exp", "wrap", "prio", "tiq", "thresh")
EDGE_TICKS = [(r, k, "sparse") for r in SE.ROUTES for k in SE.KINDS] + [(r, k, "dense") for r in SE.ROUTES for k in DENSE_KINDS]


def report_edge_tick(route, kind, density):
    """test_gpu_score_edges.edge_tick with a narrow distro of task groups appended before the edges are sprinkled (the
    smem and general ticks have none of their own), and the rows each kind exists for pinned in it:
      exp:  two members of its first group of several at 2^62 + 1 (the group's ExpectedRuntime sum wraps), and one
            member of further groups at 2^62 + 1 until the job's sum over the distro's groups wraps;
      prio: every member of that group at a negative priority (MaxPriority stays 0).
    -> (tick, {kind: rows sprinkle_edges wrote} with the pinned rows added)."""
    seed = 500 + 17 * SE.ROUTES.index(route) + SE.KINDS.index(kind)
    w = SE._route_tick(route, seed)
    probe = synth.make(np.array([300]), seed + 1, zipf_priority=True, tg_frac=0.6, n_hosts=6)
    probe.tasks.flags |= np.uint32(L.EVG_TF_DEPS_MET)
    w = concat(w, probe)
    kw = dict(positions=SE.sparse_rows(w, route)) if density == "sparse" else dict(frac=0.3)
    rows = synth.sprinkle_edges(w, seed, kinds=(kind,) + synth.DISTRO_KINDS, **kw)
    d = w.distros.n_distros - 1
    groups = group_members(w, d)
    multi = next(i for i, g in enumerate(groups) if len(g) >= 2)
    pinned = []
    if kind == "exp":
        pinned = list(groups[multi][:2])
        w.tasks.expected_ns[pinned] = BIG
        for i, g in enumerate(groups):
            if wrapped_group_sums(w, d)[1] > I64_MAX:
                break
            if i != multi and sum(int(x) for x in w.tasks.expected_ns[g]) < 2 ** 61:
                w.tasks.expected_ns[g[0]] = BIG
                pinned.append(g[0])
    elif kind == "prio":
        pinned = list(groups[multi])
        w.tasks.priority[pinned] = [(-1, -2 ** 31)[i % 2] for i in range(len(pinned))]
    if pinned:
        rows[kind] = np.union1d(rows[kind], np.asarray(pinned, np.int64))
    return w, rows


def oracle_plan(w, ref):
    """The oracle's plan rows and allocator results shaped like Engine.download's (group rows in slot order)."""
    t, dt = w.tasks, w.distros
    gi = np.zeros(dt.n_groups, L.GROUP_INFO_DTYPE)
    for d in range(dt.n_distros):
        a = int(dt.task_off[d])
        for g in range(int(ref["info"][d]["n_groups"])):
            row = ref["groups"][a + d + g]
            nt = int(row["name_task"])
            k = -1 if nt < 0 else int(t.group_id[a + nt])
            if k >= 0:
                gi[int(dt.group_off[d]) + k] = tuple(int(row[f]) for f in L.GROUP_INFO_FIELDS)
    res = np.zeros(dt.n_distros, L.ALLOC_RESULT_DTYPE)
    res["new_hosts"], res["free_hosts"] = ref["new_hosts"], ref["free_hosts"]
    return SimpleNamespace(info=ref["info"], group_info=gi), SimpleNamespace(result=res, status=ref["status"])


SETTINGS = {"plain": dict(single=0.0, terminate=0.0, hourly=0.0), "single": dict(single=1.0, terminate=0.0, hourly=0.0),
            "terminate": dict(single=0.0, terminate=1.0, hourly=0.0),
            "terminate_hourly": dict(single=0.0, terminate=1.0, hourly=1.0)}


def wrapped_group_sums(w, d):
    """Per task-group slot of distro d (includes_dependencies off: every member counts): the exact sum of its members'
    expected durations, and the job's exact sum over the slots of each slot's int64 (wrapped) sum."""
    exact = [sum(int(x) for x in w.tasks.expected_ns[g]) for g in group_members(w, d)]
    return exact, sum(OJ.w64(x) for x in exact)


def reaches(w, kind, rows):
    """What each edge tick exists for: a narrow distro's task group holds an edge row; for exp a narrow group's
    expected-duration sum wraps and so does the job's sum over a narrow distro's groups; for prio a narrow group holds
    negative priorities only."""
    narrow = [d for d in narrow_distros(w) if not int(w.distros.cfg["includes_dependencies"][d])]
    toff = w.distros.task_off
    held = [r for r in rows[kind] if w.tasks.group_id[r] >= 0 and int(np.searchsorted(toff, r, side="right") - 1) in narrow]
    assert held or kind == "u32", "no edge row in a narrow distro's task group"  # u32 rows are lone tasks by design
    if kind == "exp":
        sums = [wrapped_group_sums(w, d) for d in narrow]
        assert any(not -2 ** 63 <= x <= I64_MAX for exact, _ in sums for x in exact)
        assert any(not -2 ** 63 <= job <= I64_MAX for _, job in sums)
    if kind == "prio":
        assert any(len(g) and (w.tasks.priority[g] < 0).all() for d in narrow for g in group_members(w, d))


# ------------------------------------------------------------------------------- the job and the chained drawdown
TARGET_MODES = ("at_most_zero", "equal", "above")


def check_chained_drawdown(engine, want, qlen, seed):
    """evg_host_drawdown chained on the last evg_host_job against oracle_host_termination fed the restatement's report
    (`want`), once per target mode: existing host counts that put every drawdown distro's target (existing -
    new_cap_target) at or below 0, at its idle-host count and above it.  -> number of drawdown distros."""
    D = len(want)
    iw = synth.make_idle_hosts(np.random.default_rng(seed).integers(1, 7, D), seed)
    table = S.marshal_idle_hosts(iw.groups)
    caps = [int(r["report"]["new_cap_target"]) if r["report"]["drawdown"] else None for r in want]
    for mode in TARGET_MODES:
        ex = np.zeros(D, np.int64)
        for d, cap in enumerate(caps):
            n = len(iw.groups[d])
            ex[d] = n if cap is None else cap + {"at_most_zero": -min(cap, 1), "equal": n, "above": n + 2}[mode]
        res = engine.host_drawdown(table, ex, iw.now)
        hosts, dist = [], []
        for d, g in enumerate(iw.groups):
            if caps[d] is None:
                hosts += [OT.NOT_CHECKED] * len(g)
                dist.append((0, 0, 0))
                continue
            job, v = OT.drawdown_job(f"d{d}", g, int(ex[d]), caps[d], int(qlen[d]), iw.now)
            hosts += v
            dist.append((job.drawdown_target, job.decommissioned, 1))
            n = len(g)
            assert {"at_most_zero": job.drawdown_target <= 0, "equal": job.drawdown_target == n,
                    "above": job.drawdown_target > n}[mode]
        assert verdict_rows(res["hosts"]) == hosts, mode
        assert [(int(r["target"]), int(r["decommissioned"]), int(r["ran"])) for r in res["distros"]] == dist, mode
    return sum(c is not None for c in caps)


def check_jobs(engine, w, cfg, spawned, sources, ref, seed, where=""):
    """evg_host_job on the resident tick against the restatement fed each (plan rows, allocator rows) source, then the
    chained drawdown.  -> (restatement on the last source, drawdown distros)."""
    res = {k: v.copy() for k, v in engine.host_job(cfg, spawned).items()}
    wants = [restate(po, ao, w.distros.group_off, w.hosts, cfg, spawned) for po, ao in sources]
    for d in range(w.distros.n_distros):
        got = {"n_hosts": int(res["n_hosts"][d]), "n_hosts_free": int(res["n_hosts_free"][d]), "status": int(res["status"][d]),
               "report": {f: res["report"][d][f] for f in L.HOST_REPORT_FIELDS}}
        for k, want in enumerate(wants):
            assert_job(got, as_expect(want[d]), f"{where} distro {d} source {k} spawned {spawned is not None}")
    n = check_chained_drawdown(engine, wants[-1], ref["info"]["length_with_dependencies_met"], seed)
    return wants[-1], n


@pytest.mark.parametrize("route,kind,density", EDGE_TICKS)
def test_edge_tick_readers(engine, monkeypatch, route, kind, density):
    if route == "smem":
        monkeypatch.setenv("EVG_SPARSE_CLASS", "0")  # keep the 4097+ task classes on k_plan_smem
    w, rows = report_edge_tick(route, kind, density)
    reaches(w, kind, rows)
    check_tick(engine, w, oracle=True)  # plan unchanged by the option, breakdown rows == oracle, queue rows at every cap
    po, ao = engine.download(want_alloc=True)
    ref = parity.check_against_oracle(w, po, ao)
    sources = [(po, ao), oracle_plan(w, ref)]
    D = w.distros.n_distros
    seed = 7000 + 100 * SE.ROUTES.index(route) + 2 * SE.KINDS.index(kind) + (density == "dense")
    drew = 0
    for name, kw in SETTINGS.items():
        cfg = job_cfg(D, seed, **kw)
        for spawned in (None, np.random.default_rng(seed).integers(0, 6, D).astype(np.int32)):
            _, n = check_jobs(engine, w, cfg, spawned, sources, ref, seed, f"{route}/{kind}/{density}/{name}")
            drew += n
    DREW.append(drew)


DREW = []  # drawdown distros each edge tick's jobs reported


def test_edge_ticks_drew_down():
    """The chained drawdowns above ran on drawdown reports (the far thresholds of the "clock" distros) for most ticks."""
    assert len(DREW) == len(EDGE_TICKS) and sum(d > 0 for d in DREW) > len(DREW) // 2, DREW


# ---------------------------------------------------------------------------------------- B. k_host_job's own edges
H, MIN = M.HOUR, M.MINUTE


@dataclass
class Case:
    """One distro of a crafted tick.  Its tasks: `ungrouped` (expected durations of the lone tasks) and `groups` (of
    each task group's members), every one with dependencies met; `n_up` idle hosts, so the allocator's free_hosts is
    n_up.  A lone task longer than `thr` counts in the distro's DurationOverThreshold, which takes one host from
    hosts_avail.  The given spawned count is `spawned`, else the one at which hosts_avail is `avail`, else 0; `lands`
    holds on the restatement's result with that count (with NULL when `null`)."""
    name: str
    thr: int
    ungrouped: Sequence[int] = ()
    groups: Sequence[Sequence[int]] = ()
    n_up: int = 3
    min_hosts: int = 0
    single: bool = False
    terminate: bool = True
    n_prov: int = 0
    avail: Optional[int] = None
    spawned: Optional[int] = None
    null: bool = False
    lands: Optional[Callable] = None


def bits(x) -> int:
    return OJ.float_bits(x)


def killable_product(r, n_up):
    """float32(n_up) * (1 - ratio), the product setTargetAndTerminate truncates."""
    with np.errstate(over="ignore"):
        return np.float32(n_up) * (np.float32(1) - np.float32(r["report"]["host_queue_ratio"]))


def below(k):
    return np.nextafter(np.float32(k), np.float32(0))


def above(k):
    return np.nextafter(np.float32(k), np.float32(np.inf))


NEG = -BIG  # two of them sum to 2^63 - 2 after the wrap: a positive scheduled duration under a threshold <= 0
# Ratios q * 2^-24 come out exact: threshold 2^30, every lone task q * 2^6 ns, as many of them as hosts_avail
EDGE_CASES = [
    # threshold 0: 0 / 0 is NaN, x / 0 is +Inf; neither is < 0.25
    Case("thr0_nan", 0, [5], lands=lambda r: np.isnan(r["report"]["host_queue_ratio"]) and not r["report"]["drawdown"]),
    Case("thr0_inf", 0, [NEG, NEG], lands=lambda r: r["report"]["scheduled_duration_ns"] == 2 ** 63 - 2 and
         np.isposinf(r["report"]["host_queue_ratio"]) and not r["report"]["drawdown"]),
    # threshold -1: 0 / -1 is -0.0, which takes the ratio == 0 branch (killable = n_up)
    Case("thr-1_negzero", -1, [5], lands=lambda r: bits(r["report"]["host_queue_ratio"]) == 0x80000000 and
         r["report"]["killable_hosts"] == 3 and r["report"]["new_cap_target"] == 0),
    # negative thresholds and a large time to empty: float32(3) * (1 - ratio) is past 2^63 and saturates
    Case("thr-1_saturates", -1, [NEG, NEG, 5, 5], lands=lambda r: r["report"]["hosts_avail"] == 1 and
         killable_product(r, 3) >= 2.0 ** 63 and r["report"]["killable_hosts"] == I64_MAX and r["report"]["drawdown"]),
    Case("thr-2_saturates", -2, [NEG, NEG, 5, 5], lands=lambda r: killable_product(r, 3) >= 2.0 ** 63 and
         r["report"]["killable_hosts"] == I64_MAX),
    Case("avail0_max_time_saturates", -1, [NEG, NEG, 5, 5, 5], lands=lambda r: r["report"]["hosts_avail"] == 0 and
         r["report"]["time_to_empty_ns"] == OJ.MAX_POSSIBLE_TIME and r["report"]["killable_hosts"] == I64_MAX),
    # threshold 1: 7 ns on 3 hosts
    Case("thr1", 1, [1] * 7, lands=lambda r: r["report"]["time_to_empty_ns"] == 2 and r["report"]["host_queue_ratio"] == 2),
    # threshold INT64_MAX rounds to 2^63 in float32: (2^61 - 1) / (2^63 - 1) < 1/4 exactly, but the ratio is 0.25f
    Case("thr_max", I64_MAX, [2 ** 61 - 1] * 3, lands=lambda r: r["report"]["time_to_empty_ns"] == 2 ** 61 - 1 and
         bits(r["report"]["host_queue_ratio"]) == 0x3E800000 and not r["report"]["drawdown"]),
    # ratio exactly 0.25f (no drawdown) and the float just below it (drawdown)
    Case("ratio_quarter", 2 ** 26, [2 ** 24] * 3, lands=lambda r: bits(r["report"]["host_queue_ratio"]) == 0x3E800000 and
         not r["report"]["drawdown"]),
    Case("ratio_below_quarter", 2 ** 26, [2 ** 24 - 1] * 4, n_up=4, lands=lambda r: bits(r["report"]["host_queue_ratio"]) ==
         0x3E7FFFFF and r["report"]["drawdown"] and r["report"]["killable_hosts"] == 3),
    # the killable product one ulp below 4 (truncated: 3) and one ulp above 3
    Case("killable_below_int", 2 ** 30, [64] * 4, n_up=4, lands=lambda r: killable_product(r, 4) == below(4) and
         r["report"]["killable_hosts"] == 3 and r["report"]["new_cap_target"] == 1),
    Case("killable_above_int", 2 ** 30, [(2 ** 22 - 1) * 64] * 4, n_up=4, lands=lambda r: killable_product(r, 4) == above(3) and
         r["report"]["killable_hosts"] == 3),
    # MinimumHosts above n_up: the cap is the minimum and the drawdown still happens
    Case("clamp_min", 2 ** 26, [2 ** 22] * 3, min_hosts=5, lands=lambda r: r["report"]["killable_hosts"] == 2 and
         r["report"]["new_cap_target"] == 5 and r["report"]["drawdown"]),
    # the time-to-empty branches
    Case("sched0", H, [2 * H], lands=lambda r: r["report"]["scheduled_duration_ns"] == 0 and r["report"]["time_to_empty_ns"] == 0 and
         r["report"]["killable_hosts"] == 3),
    Case("sched1_avail1", H, [1, 2 * H, 2 * H], lands=lambda r: r["report"]["scheduled_duration_ns"] == 1 and
         r["report"]["hosts_avail"] == 1 and r["report"]["time_to_empty_ns"] == 1 and r["report"]["time_to_empty_no_spawns_ns"] == 1),
    Case("avail_negative", H, [MIN, MIN] + [2 * H] * 6, lands=lambda r: r["report"]["hosts_avail"] == -3 and
         r["report"]["time_to_empty_ns"] == r["report"]["time_to_empty_no_spawns_ns"] == OJ.MAX_POSSIBLE_TIME),
    Case("avail_ns_zero", H, [10 * MIN, 10 * MIN] + [2 * H] * 3, avail=4, lands=lambda r: r["report"]["hosts_avail"] == 4 and
         r["report"]["hosts_spawned"] == 4 and r["report"]["time_to_empty_ns"] == 5 * MIN and
         r["report"]["time_to_empty_no_spawns_ns"] == OJ.MAX_POSSIBLE_TIME),
    Case("avail_ns_negative", H, [7 * MIN] + [2 * H] * 5, avail=1, lands=lambda r: r["report"]["hosts_avail"] == 1 and
         r["report"]["hosts_spawned"] == 3 and r["report"]["time_to_empty_ns"] == 7 * MIN and
         r["report"]["time_to_empty_no_spawns_ns"] == OJ.MAX_POSSIBLE_TIME),
    # truncated quotient: 7 / 2 (both are positive in this branch, so a quotient below zero cannot occur)
    Case("inexact_quotient", H, [7, 2 * H], avail=2, lands=lambda r: r["report"]["scheduled_duration_ns"] == 7 and
         r["report"]["hosts_avail"] == 2 and r["report"]["time_to_empty_ns"] == 3),
    Case("spawned_int32_max", H, [40 * MIN] * 3, spawned=I32_MAX, lands=lambda r: r["report"]["hosts_spawned"] == I32_MAX and
         r["report"]["hosts_avail"] == 3 + I32_MAX and r["report"]["time_to_empty_ns"] == 120 * MIN // (3 + I32_MAX)),
    # single-task distros, spawned NULL: n_hosts = LengthWithDependenciesMet - n_provisioning; the groups' CountFree /
    # CountRequired stay out of the sums
    Case("single_nprov0", H, [MIN] * 4, [[MIN, MIN], [MIN]], single=True, null=True,
         lands=lambda r: r["n_hosts"] == 7 and r["report"]["hosts_spawned"] == 7 and r["report"]["required_in_groups"] == 0),
    Case("single_nprov_max", H, [MIN] * 4, [[MIN, MIN], [MIN]], single=True, n_prov=I64_MAX, null=True,
         lands=lambda r: r["n_hosts"] == 7 - I64_MAX and r["report"]["hosts_spawned"] == 0 and r["report"]["hosts_avail"] == 0),
]


def crafted_tick(cases: Sequence[Case], now: int = synth.NOW_NS):
    """-> (tick with hosts, HOST_JOB_CFG rows) for `cases`, one distro each, static-free, by-the-second billing."""
    exp, gid, tgo, sizes, ngroups = [], [], [], [], []
    for c in cases:
        exp += list(c.ungrouped)
        gid += [-1] * len(c.ungrouped)
        tgo += [0] * len(c.ungrouped)
        for g, members in enumerate(c.groups):
            exp += list(members)
            gid += [g] * len(members)
            tgo += list(range(1, len(members) + 1))
        sizes.append(len(c.ungrouped) + sum(len(m) for m in c.groups))
        ngroups.append(len(c.groups))
    T, D = len(exp), len(cases)
    tasks = S.TaskSoA(np.zeros(T), np.array(exp, dtype=np.int64), np.full(T, now - MIN), np.full(T, now - MIN), np.zeros(T),
                      np.array(tgo), np.array(gid), np.zeros(T), np.full(T, L.EVG_TF_REQ_OTHER | L.EVG_TF_DEPS_MET)).normalize()
    cfg = np.zeros(D, L.DISTRO_CFG_DTYPE)
    cfg["target_time_ns"] = [c.thr for c in cases]
    cfg["n_versions"] = 1
    distros = S.DistroTable(np.concatenate([[0], np.cumsum(sizes)]), np.concatenate([[0], np.cumsum(ngroups)]), cfg,
                            np.ones(sum(ngroups))).normalize()
    n_up = np.array([c.n_up for c in cases], np.int64)
    Hn = int(n_up.sum())
    acfg = np.zeros(D, L.ALLOC_CFG_DTYPE)
    acfg["future_host_fraction"] = 0.4
    acfg["provider"] = L.EVG_PROVIDER_EPHEMERAL
    acfg["minimum_hosts"] = [c.min_hosts for c in cases]
    acfg["maximum_hosts"] = 100_000
    hosts = S.HostSoA(np.zeros(Hn), np.full(Hn, L.EVG_HG_NONE), np.zeros(Hn), np.zeros(Hn), np.full(Hn, M.ZERO_TIME),
                      np.concatenate([[0], np.cumsum(n_up)]), acfg).normalize()
    job = np.zeros(D, L.HOST_JOB_CFG_DTYPE)
    job["n_provisioning"] = [c.n_prov for c in cases]
    job["single_task_distro"] = [c.single for c in cases]
    job["terminate_when_overallocated"] = [c.terminate for c in cases]
    return synth.Workload("crafted", now, tasks, distros, hosts), job


def given_spawned(w, cases, job, plan):
    """The given spawned counts: hosts_avail moves one for one with spawned, so the count that puts it at `avail` is
    avail minus hosts_avail at 0 spawned."""
    at0 = restate(*plan, w.distros.group_off, w.hosts, job, np.zeros(len(cases), np.int32))
    out = [c.spawned if c.spawned is not None else (c.avail - a["report"]["hosts_avail"] if c.avail is not None else 0)
           for c, a in zip(cases, at0)]
    assert all(0 <= x <= I32_MAX for x in out)
    return np.array(out, np.int32)


# Warp-sum layout: k_host_job sums a distro of more than kHostJobWarpGroups = 16 group slots with its whole warp (32
# consecutive distros), one wide distro at a time, each lane striding 32 slots; the others sum their own slots.
# name -> (distros, {distro: slots}, single-task distros, distros with one member of each of their first four slots
# at 2^62 + 1: both the group and the over-threshold sums wrap).  Every other distro has d % 5 slots.
LAYOUTS = {
    "n1": (1, {0: 17}, (), (0,)),
    "n31": (31, {0: 17, 15: 16, 16: 17, 30: 40}, (16,), (15, 30)),
    "n33": (33, {0: 17, 16: 16, 31: 17, 32: 17}, (), (16, 31)),
    # warp 0 all wide (two above 32 slots); warp 1 mixed, with single-task distros (two of them wide) between
    # ordinary ones; warp 2 partial, wide at its first and last lane
    "n95": (95, {**{d: 17 for d in range(32)}, 5: 40, 31: 70, 32: 16, 33: 17, 40: 20, 41: 40, 49: 33, 64: 17, 80: 16, 94: 17},
            (40, 41) + tuple(d for d in range(32, 64) if d % 4 == 2), (0, 31, 33, 49, 80, 94)),
}


def layout_cases(name):
    n, wide, singles, big = LAYOUTS[name]
    cases = []
    for d in range(n):
        slots = wide.get(d, d % 5)
        groups = [[MIN * (1 + (7 * d + 3 * k + i) % 50) for i in range(1 + (d + k) % 3)] for k in range(slots)]
        if d in big:
            for g in groups[:4]:
                g[0] = BIG
        cases.append(Case(f"{name}/d{d}", H, [MIN * (5 + d % 40)] * (2 + d % 3), groups, single=d in singles,
                          spawned=d % 5))
    return cases


def run_crafted(engine, cases, seed):
    """The crafted tick on the device against the oracle, then evg_host_job with spawned NULL and given, and the chained
    drawdowns."""
    w, job = crafted_tick(cases)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    po, ao = engine.download(want_alloc=True)
    ref = parity.check_against_oracle(w, po, ao)
    plan = oracle_plan(w, ref)
    drew = 0
    for spawned in (None, given_spawned(w, cases, job, plan)):
        drew += check_jobs(engine, w, job, spawned, [(po, ao), plan], ref, seed, cases[0].name)[1]
    assert drew > 0


def test_host_job_edges(engine):
    run_crafted(engine, EDGE_CASES, 7500)


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_warp_sum_layout(engine, name):
    run_crafted(engine, layout_cases(name), 7600 + list(LAYOUTS).index(name))
