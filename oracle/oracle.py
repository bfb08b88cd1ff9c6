"""ctypes wrapper of the CPU ORACLE (oracle/evg_oracle.cpp) -- TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module.  It converts reference-shaped
inputs (evergreen_b200.model dataclasses, or the synthetic SoA tables turned
back into strings) into the oracle's columnar-string structs.

The task-finder restatement (find_runnable, SURVEY.md §8f.1) is plain Python over the same dataclasses -- the
finders are a per-task predicate, small enough for a loop; pinned by tests/golden/task_finder.json (the
assertions of scheduler/task_finder_test.go).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Dict, List, Optional, Sequence

import numpy as np

from evergreen_b200 import model as M

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libevgoracle.so")
ZERO = M.ZERO_TIME
BD_N = 13


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "evg_oracle.cpp")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < max(
            os.path.getmtime(src), os.path.getmtime(os.path.join(_HERE, "evg_oracle.h"))):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libevgoracle.so"], stdout=subprocess.DEVNULL)
    return LIB_PATH


class StrCol(C.Structure):
    _fields_ = [("buf", C.c_char_p), ("off", C.c_void_p)]


class Tasks(C.Structure):
    _fields_ = [("n", C.c_int64)] + [(f, StrCol) for f in (
        "id", "version", "project", "build_variant", "task_group", "requester", "activated_by", "distro_id", "status")] + [
        (f, C.c_void_p) for f in ("priority", "task_group_order", "task_group_max_hosts", "num_dependents",
                                  "generate_task", "override_dependencies", "blocked", "activated_time", "ingest_time",
                                  "scheduled_time", "dependencies_met_time", "expected_ns", "dep_off")] + [
        ("dep_task_id", StrCol), ("dep_status", StrCol), ("dep_found", C.c_void_p), ("dep_task_status", StrCol),
        ("dep_task_blocked", C.c_void_p), ("dep_finished_at", C.c_void_p)]


class PlannerSettings(C.Structure):
    _fields_ = [(f, C.c_int64) for f in (
        "patch_factor", "patch_time_in_queue_factor", "commit_queue_factor", "mainline_time_in_queue_factor",
        "expected_runtime_factor", "generate_task_factor", "stepback_task_factor")] + [
        ("num_dependents_factor", C.c_double), ("target_time_ns", C.c_int64), ("group_versions", C.c_int32),
        ("has_container_pool", C.c_int32), ("includes_dependencies", C.c_int32), ("_pad", C.c_int32)]


GROUP_FIELDS = ("name_task", "count", "count_free", "count_required", "max_hosts", "expected_duration",
                "count_duration_over_threshold", "count_wait_over_threshold", "count_dep_filled_merge_queue_tasks",
                "duration_over_threshold")
GROUP_DTYPE = np.dtype([(f, "<i8") for f in GROUP_FIELDS])
QINFO_FIELDS = ("length", "length_with_dependencies_met", "count_dep_filled_merge_queue_tasks", "expected_duration",
                "max_duration_threshold", "count_duration_over_threshold", "duration_over_threshold",
                "count_wait_over_threshold", "secondary_queue", "n_groups")
QINFO_DTYPE = np.dtype([(f, "<i8") for f in QINFO_FIELDS])


class Hosts(C.Structure):
    _fields_ = [("n", C.c_int64)] + [(f, StrCol) for f in (
        "running_task", "running_task_group", "running_task_bv", "running_task_project", "running_task_version")] + [
        (f, C.c_void_p) for f in ("teardown_start_time", "rt_found", "rt_expected_ns", "rt_std_ns", "rt_start_time")]


class AllocSettings(C.Structure):
    _fields_ = [("provider", C.c_char_p), ("rounding_rule", C.c_char_p), ("feedback_rule", C.c_char_p),
                ("disabled", C.c_int32), ("minimum_hosts", C.c_int32), ("maximum_hosts", C.c_int32),
                ("has_pool", C.c_int32), ("pool_max_containers", C.c_int32), ("parent_found", C.c_int32),
                ("parent_maximum_hosts", C.c_int32), ("_pad", C.c_int32), ("future_host_fraction", C.c_double)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        l = C.CDLL(LIB_PATH)
        l.evo_unit_value.restype = None
        l.evo_plan.restype = C.c_int64
        l.evo_get_distro_queue_info.restype = C.c_int64
        l.evo_target_time.restype = C.c_int64
        l.evo_calc_new_hosts_needed.restype = C.c_int64
        l.evo_calc_new_hosts_needed.argtypes = [C.c_int64] * 6 + [C.c_int32]
        l.evo_calc_existing_free_hosts.restype = C.c_int32
        l.evo_calc_existing_free_hosts.argtypes = [C.c_void_p, C.c_double, C.c_int64, C.c_int64, C.c_void_p]
        l.evo_allocate.restype = C.c_int32
        l.evo_group_by_task_group.restype = C.c_int64
        l.evo_fetch_expected_duration.restype = None
        l.evo_fetch_expected_duration.argtypes = [C.c_int64] * 7 + [C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        l.evo_job_batch.restype = None
        _lib = l
    return _lib


class _Keep:
    """Holds the numpy/bytes objects a ctypes struct points into."""

    def __init__(self):
        self.refs = []

    def strcol(self, strings: Sequence[str]) -> StrCol:
        enc = [s.encode("utf-8") for s in strings]
        off = np.zeros(len(enc) + 1, dtype=np.int64)
        if enc:
            np.cumsum([len(b) for b in enc], out=off[1:])
        buf = b"".join(enc) + b"\0"
        self.refs += [buf, off]
        return StrCol(buf, off.ctypes.data)

    def arr(self, values, dtype) -> int:
        a = np.ascontiguousarray(values, dtype=dtype)
        if a.shape[0] == 0:
            a = np.zeros(1, dtype=dtype)
        self.refs.append(a)
        return a.ctypes.data


def fetch_expected_duration(t: M.Task, now: int, history=None):
    a, s = C.c_int64(), C.c_int64()
    p = t.duration_prediction
    lib().evo_fetch_expected_duration(p.value, p.std_dev, p.ttl, p.collected_at, t.expected_duration,
                                      t.expected_duration_std_dev, now, int(history is not None),
                                      M.duration_from_float(history[0]) if history else 0,
                                      M.duration_from_float(history[1]) if history else 0,
                                      C.addressof(a), C.addressof(s))
    return a.value, s.value


def tasks_struct(tasks: Sequence[M.Task], now: int, dependency_db: Optional[Dict[str, M.Task]] = None,
                 expected: Optional[Sequence[int]] = None):
    k = _Keep()
    t = Tasks()
    t.n = len(tasks)
    for f, get in (("id", lambda x: x.id), ("version", lambda x: x.version), ("project", lambda x: x.project),
                   ("build_variant", lambda x: x.build_variant), ("task_group", lambda x: x.task_group),
                   ("requester", lambda x: x.requester), ("activated_by", lambda x: x.activated_by),
                   ("distro_id", lambda x: x.distro_id), ("status", lambda x: x.status)):
        setattr(t, f, k.strcol([get(x) for x in tasks]))
    t.priority = k.arr([x.priority for x in tasks], np.int64)
    t.task_group_order = k.arr([x.task_group_order for x in tasks], np.int32)
    t.task_group_max_hosts = k.arr([x.task_group_max_hosts for x in tasks], np.int32)
    t.num_dependents = k.arr([x.num_dependents for x in tasks], np.int32)
    t.generate_task = k.arr([x.generate_task for x in tasks], np.uint8)
    t.override_dependencies = k.arr([x.override_dependencies for x in tasks], np.uint8)
    t.blocked = k.arr([x.blocked() for x in tasks], np.uint8)
    t.activated_time = k.arr([x.activated_time for x in tasks], np.int64)
    t.ingest_time = k.arr([x.ingest_time for x in tasks], np.int64)
    t.scheduled_time = k.arr([x.scheduled_time for x in tasks], np.int64)
    t.dependencies_met_time = k.arr([x.dependencies_met_time for x in tasks], np.int64)
    if expected is None:
        expected = [fetch_expected_duration(x, now)[0] for x in tasks]
    t.expected_ns = k.arr(expected, np.int64)
    dep_off, ids, want, found, dstat, dblk, dfin = [0], [], [], [], [], [], []
    db = dependency_db or {}
    for x in tasks:
        for d in x.depends_on:
            ids.append(d.task_id)
            want.append(d.status)
            dfin.append(d.finished_at)
            dt = db.get(d.task_id)
            found.append(dt is not None)
            dstat.append(dt.status if dt else "")
            dblk.append(dt.blocked() if dt else False)
        dep_off.append(len(ids))
    t.dep_off = k.arr(dep_off, np.int64)
    t.dep_task_id = k.strcol(ids)
    t.dep_status = k.strcol(want)
    t.dep_found = k.arr(found, np.uint8)
    t.dep_task_status = k.strcol(dstat)
    t.dep_task_blocked = k.arr(dblk, np.uint8)
    t.dep_finished_at = k.arr(dfin, np.int64)
    return t, k


def planner_settings(d: M.Distro) -> PlannerSettings:
    ps = d.planner_settings
    s = PlannerSettings()
    s.patch_factor, s.patch_time_in_queue_factor = ps.patch_factor, ps.patch_time_in_queue_factor
    s.commit_queue_factor, s.mainline_time_in_queue_factor = ps.commit_queue_factor, ps.mainline_time_in_queue_factor
    s.expected_runtime_factor, s.generate_task_factor = ps.expected_runtime_factor, ps.generate_task_factor
    s.stepback_task_factor, s.num_dependents_factor = ps.stepback_task_factor, float(ps.num_dependents_factor)
    s.target_time_ns = ps.target_time
    s.group_versions = int(ps.should_group_versions())
    s.has_container_pool = int(d.container_pool != "")
    s.includes_dependencies = int(d.dispatcher_settings.version == M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES)
    return s


def unit_value(d: M.Distro, tasks: Sequence[M.Task], now: int) -> M.SortingValueBreakdown:
    """unit.sortingValueBreakdown(ctx) for a unit holding `tasks` (planner.go:345-353)."""
    t, _k = tasks_struct(tasks, now)
    s = planner_settings(d)
    members = np.arange(len(tasks), dtype=np.int64)
    out = np.zeros(BD_N, dtype=np.int64)
    lib().evo_unit_value(C.byref(t), C.c_void_p(members.ctypes.data), C.c_int64(len(tasks)), C.byref(s),
                         C.c_int64(now), C.c_void_p(out.ctypes.data))
    return M.SortingValueBreakdown.from_row(out)


def plan(d: M.Distro, tasks: Sequence[M.Task], now: int):
    """PrepareTasksForPlanning(d, tasks).Export -> (order indices, breakdown rows, plan.Len())."""
    t, _k = tasks_struct(tasks, now)
    s = planner_settings(d)
    order = np.zeros(max(len(tasks), 1), dtype=np.int64)
    bd = np.zeros((max(len(tasks), 1), BD_N), dtype=np.int64)
    n_units = C.c_int64()
    n = lib().evo_plan(C.byref(t), C.byref(s), C.c_int64(now), C.c_void_p(order.ctypes.data),
                       C.c_void_p(bd.ctypes.data), C.byref(n_units))
    return order[:n].copy(), bd[:n].copy(), n_units.value


def _group_infos(tasks, rows) -> List[M.TaskGroupInfo]:
    out = []
    for r in rows:
        name = "" if int(r["name_task"]) < 0 else tasks[int(r["name_task"])].get_task_group_string()
        out.append(M.TaskGroupInfo(name, *[int(r[f]) for f in GROUP_FIELDS[1:]]))
    return out


def queue_info(distro_id: str, tasks: Sequence[M.Task], threshold: int, includes_dependencies: bool, now: int,
               dependency_db: Optional[Dict[str, M.Task]] = None, order: Optional[Sequence[int]] = None) -> M.DistroQueueInfo:
    t, _k = tasks_struct(tasks, now, dependency_db)
    order = np.ascontiguousarray(order if order is not None else np.arange(len(tasks)), dtype=np.int64)
    info = np.zeros(1, dtype=QINFO_DTYPE)
    groups = np.zeros(len(tasks) + 1, dtype=GROUP_DTYPE)
    buf = np.zeros(1, dtype=np.int64) if order.shape[0] == 0 else order
    n = lib().evo_get_distro_queue_info(C.byref(t), C.c_void_p(buf.ctypes.data), C.c_int64(order.shape[0]),
                                        distro_id.encode(), C.c_int64(threshold), C.c_int32(int(includes_dependencies)),
                                        C.c_int64(now), C.c_void_p(info.ctypes.data), C.c_void_p(groups.ctypes.data))
    q = info[0]
    return M.DistroQueueInfo(
        length=int(q["length"]), length_with_dependencies_met=int(q["length_with_dependencies_met"]),
        count_dep_filled_merge_queue_tasks=int(q["count_dep_filled_merge_queue_tasks"]),
        expected_duration=int(q["expected_duration"]), max_duration_threshold=int(q["max_duration_threshold"]),
        count_duration_over_threshold=int(q["count_duration_over_threshold"]),
        duration_over_threshold=int(q["duration_over_threshold"]),
        count_wait_over_threshold=int(q["count_wait_over_threshold"]),
        task_group_infos=_group_infos(tasks, groups[:n]), secondary_queue=bool(q["secondary_queue"]))


def deps_met(tasks: Sequence[M.Task], now: int, dependency_db=None) -> np.ndarray:
    t, _k = tasks_struct(tasks, now, dependency_db)
    out = np.zeros(max(len(tasks), 1), dtype=np.uint8)
    lib().evo_deps_met(C.byref(t), C.c_void_p(out.ctypes.data))
    return out[:len(tasks)].astype(bool)


def _satisfies_dependency(t: M.Task, dep_task: M.Task) -> bool:
    """Task.SatisfiesDependency, model/task/task.go:529-543."""
    for dep in t.depends_on:
        if dep.task_id == dep_task.id:
            if dep.status in (M.TASK_SUCCEEDED, ""):
                return dep_task.status == M.TASK_SUCCEEDED
            if dep.status == M.TASK_FAILED:
                return dep_task.status == M.TASK_FAILED
            if dep.status == M.ALL_STATUSES:
                return dep_task.status in (M.TASK_FAILED, M.TASK_SUCCEEDED) or dep_task.blocked()
    return False


def _deps_walk(t: M.Task, cache: Dict[str, M.Task], shortcut: bool) -> bool:
    """Task.DependenciesMet (task.go:632-671, shortcut=True) / Task.AllDependenciesSatisfied (task.go:795-821,
    shortcut=False) over a cache that already holds every task the collection has; a dependency the cache lacks
    is the lookup error both callers turn into "skip this task" (task_finder.go:86-101,181-186)."""
    if shortcut and t.has_dependencies_met():
        return True
    if not t.depends_on:
        return True
    deps = []
    for dep in t.depends_on:
        if dep.task_id not in cache:
            return False
        deps.append(cache[dep.task_id])
    return all(_satisfies_dependency(t, d) for d in deps)


def find_runnable(d: M.Distro, candidates: Sequence[M.Task], project_refs: Sequence[M.ProjectRef],
                  dependency_db: Optional[Dict[str, M.Task]] = None, finder: str = "legacy") -> List[M.Task]:
    """Restatement of LegacyFindRunnableTasks (scheduler/task_finder.go:40-106) and AlternateTaskFinder
    (:108-197; ParallelTaskFinder :199-317 filters identically) for one distro.  `candidates` stands for the
    tasks collection restricted to the distro: schedulableHostTasksQuery (model/task/db.go:671-689) is applied
    here, as task.FindHostSchedulable would (model/task/task.go:3342-3350)."""
    undispatched = [t for t in candidates
                    if t.activated and t.status == M.TASK_UNDISPATCHED and t.priority > M.DISABLED_TASK_PRIORITY
                    and t.execution_platform in ("", "host")
                    and (not t.unattainable_dependency or t.override_dependencies)]
    refs = {p.id: p for p in project_refs}
    cache = dict(dependency_db or {})
    cache.update({t.id: t for t in candidates})
    out = []
    for t in undispatched:
        ref = refs.get(t.project)
        if ref is None:  # "could not find project for task"
            continue
        if not ref.can_dispatch_task(t):  # model.ProjectCanDispatchTask, model/project_ref.go:3441-3462
            continue
        if d.valid_projects and ref.id not in d.valid_projects:
            continue
        if d.dispatcher_settings.version != M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES:
            if not _deps_walk(t, cache, shortcut=(finder == "legacy")):
                continue
        out.append(t)
    return out


def expected_durations_for_window(tasks: Sequence[M.Task], window_start: int, window_end: int):
    """Restatement of getExpectedDurationsForWindow (model/task/expected_duration.go:36-96) over finished-task
    documents: $match (completed status, not timed out, StartTime > start, FinishTime <= end), $group by display
    name within (project, build variant) with $avg and $stdDevPop of TimeTaken.  Exact rational arithmetic, one
    rounding per output -> {(project, bv, name): (count, mean, stddev)}; MongoDB's streaming doubles agree to ~1e-12."""
    import math
    from fractions import Fraction
    groups: Dict[tuple, List[int]] = {}
    for t in tasks:
        if t.status not in M.TASK_COMPLETED_STATUSES or t.timed_out:
            continue
        if not (t.start_time > window_start and t.finish_time <= window_end):
            continue
        groups.setdefault((t.project, t.build_variant, t.display_name), []).append(t.time_taken)
    out = {}
    for k, xs in groups.items():
        n, s = len(xs), sum(xs)
        m0 = s // n  # floor
        rem = s - n * m0
        s2 = sum((x - m0) ** 2 for x in xs)
        # the canonical roundings of include/evg_sched.h: double(s)/double(n); double(S2)/n minus (rem/n)^2, where
        # Python's int -> float conversions are the one round-to-nearest-even of the exact integers
        mean = float(s) / float(n)
        fr = float(rem) / float(n)
        var = max(float(s2) / float(n) - fr * fr, 0.0)
        exact_std = math.sqrt(Fraction(n * sum(x * x for x in xs) - s * s, n * n))  # reference value, for the tolerance test
        out[k] = (n, mean, math.sqrt(var), exact_std)
    return out


def hosts_struct(hosts: Sequence[M.Host], running: Dict[str, M.RunningTaskStats]):
    k = _Keep()
    h = Hosts()
    h.n = len(hosts)
    h.running_task = k.strcol([x.running_task for x in hosts])
    h.running_task_group = k.strcol([x.running_task_group for x in hosts])
    h.running_task_bv = k.strcol([x.running_task_build_variant for x in hosts])
    h.running_task_project = k.strcol([x.running_task_project for x in hosts])
    h.running_task_version = k.strcol([x.running_task_version for x in hosts])
    h.teardown_start_time = k.arr([x.task_group_teardown_start_time for x in hosts], np.int64)
    rts = [running.get(x.running_task) if x.running_task else None for x in hosts]
    h.rt_found = k.arr([bool(r and r.found) for r in rts], np.uint8)
    h.rt_expected_ns = k.arr([r.expected if r else 0 for r in rts], np.int64)
    h.rt_std_ns = k.arr([r.std_dev if r else 0 for r in rts], np.int64)
    h.rt_start_time = k.arr([r.start_time if r else ZERO for r in rts], np.int64)
    return h, k


def alloc_settings(data: M.HostAllocatorData, keep: _Keep) -> AllocSettings:
    d = data.distro
    hs = d.host_allocator_settings
    a = AllocSettings()
    for f, v in (("provider", d.provider), ("rounding_rule", hs.rounding_rule), ("feedback_rule", hs.feedback_rule)):
        b = v.encode()
        keep.refs.append(b)
        setattr(a, f, b)
    a.disabled, a.minimum_hosts, a.maximum_hosts = int(d.disabled), hs.minimum_hosts, hs.maximum_hosts
    a.has_pool = int(data.container_pool is not None)
    a.pool_max_containers = data.container_pool.max_containers if data.container_pool else 0
    a.parent_found = int(data.parent_distro_maximum_hosts is not None)
    a.parent_maximum_hosts = data.parent_distro_maximum_hosts or 0
    a.future_host_fraction = float(hs.future_host_fraction)
    return a


def _qinfo_rows(qi: M.DistroQueueInfo, keep: _Keep):
    info = np.zeros(1, dtype=QINFO_DTYPE)
    for f in QINFO_FIELDS[:-2]:
        info[0][f] = getattr(qi, f)
    info[0]["secondary_queue"] = int(qi.secondary_queue)
    info[0]["n_groups"] = len(qi.task_group_infos)
    groups = np.zeros(max(len(qi.task_group_infos), 1), dtype=GROUP_DTYPE)
    for i, g in enumerate(qi.task_group_infos):
        groups[i]["name_task"] = -1
        for f in GROUP_FIELDS[1:]:
            groups[i][f] = getattr(g, f)
    names = keep.strcol([g.name for g in qi.task_group_infos])
    keep.refs += [info, groups]
    return info, groups, names


def allocate(data: M.HostAllocatorData, now: int):
    """UtilizationBasedHostAllocator(ctx, &data) -> (new_hosts, free_hosts, status);
    mutates data.distro_queue_info.task_group_infos[].count_free/count_required."""
    h, k = hosts_struct(data.existing_hosts, data.running_tasks)
    a = alloc_settings(data, k)
    info, groups, names = _qinfo_rows(data.distro_queue_info, k)
    n, f = C.c_int64(), C.c_int64()
    st = lib().evo_allocate(C.byref(h), C.byref(a), C.c_void_p(info.ctypes.data), C.c_void_p(groups.ctypes.data),
                            C.byref(names), C.c_int64(now), C.byref(n), C.byref(f))
    for i, g in enumerate(data.distro_queue_info.task_group_infos):
        g.count_free, g.count_required = int(groups[i]["count_free"]), int(groups[i]["count_required"])
    return n.value, f.value, st


def calc_new_hosts_needed(short_ns, threshold, expected_free, n_long, n_overdue, n_mq, round_down=True) -> int:
    return int(lib().evo_calc_new_hosts_needed(short_ns, threshold, expected_free, n_long, n_overdue, n_mq, int(round_down)))


def calc_existing_free_hosts(hosts, running, fraction, threshold, now):
    h, _k = hosts_struct(hosts, running)
    out = C.c_int64()
    st = lib().evo_calc_existing_free_hosts(C.addressof(h), float(fraction), threshold, now, C.addressof(out))
    return out.value, st


def group_by_task_group(hosts: Sequence[M.Host], infos: Sequence[M.TaskGroupInfo]):
    """groupByTaskGroup -> {name: (host indices, info or None)} (allocator.go:223-260)."""
    h, k = hosts_struct(hosts, {})
    names = k.strcol([g.name for g in infos])
    bucket = np.zeros(max(len(hosts), 1), dtype=np.int64)
    n = lib().evo_group_by_task_group(C.byref(h), C.byref(names), C.c_int64(len(infos)), C.c_void_p(bucket.ctypes.data))
    out = {}
    for g in infos:
        out[g.name] = ([], g)
    for i, hh in enumerate(hosts):
        name = hh.get_task_group_string() if (hh.running_task != "" and hh.running_task_group != "") else ""
        code = int(bucket[i])
        if code >= 0 or code == -1:
            want = "" if code == -1 else infos[code].name
            assert want == name
        out.setdefault(name, ([], None))[0].append(i)
    assert len(out) == n
    return out


# ---------------------------------------------------------------------------
# synthetic SoA -> reference-shaped strings (parity at size, CPU baseline)
# ---------------------------------------------------------------------------
_REQ = ("gitter_request", "patch_request", "github_merge_request")


class SoAJob:
    """A batch of distros rebuilt as reference-shaped columns from the SoA the
    CUDA path consumes, so both sides see the same queue."""

    def __init__(self, soa, table, hosts=None, distros: Optional[Sequence[int]] = None):
        from evergreen_b200 import _lib as L  # constants only
        k = self.keep = _Keep()
        sel = list(range(table.n_distros)) if distros is None else list(distros)
        self.sel = sel
        toff = table.task_off
        ranges = [(int(toff[d]), int(toff[d + 1])) for d in sel]
        n = sum(b - a for a, b in ranges)
        self.task_off = np.zeros(len(sel) + 1, dtype=np.int64)
        np.cumsum([b - a for a, b in ranges], out=self.task_off[1:])
        gidx = np.concatenate([np.arange(a, b) for a, b in ranges]) if n else np.zeros(0, dtype=np.int64)
        dno = np.concatenate([np.full(b - a, d, dtype=np.int64) for d, (a, b) in zip(sel, ranges)]) if n else np.zeros(0, dtype=np.int64)
        local = gidx - toff[dno] if n else gidx
        fl = soa.flags[gidx]
        gid = soa.group_id[gidx]
        vid = soa.version_id[gidx]
        t = self.tasks = Tasks()
        t.n = n
        ids = [f"d{d}t{i}" for d, i in zip(dno.tolist(), local.tolist())]
        vers = [f"d{d}v{v}" for d, v in zip(dno.tolist(), vid.tolist())]
        t.id = k.strcol(ids)
        t.version = k.strcol(vers)
        t.project = k.strcol(["p"] * n)
        t.build_variant = k.strcol(["bv"] * n)
        t.task_group = k.strcol([("" if g < 0 else f"tg{g}") for g in gid.tolist()])
        t.requester = k.strcol([_REQ[c] for c in (fl & 3).tolist()])
        t.activated_by = k.strcol([("stepback" if f & L.EVG_TF_STEPBACK else "") for f in fl.tolist()])
        t.distro_id = k.strcol([("elsewhere" if f & L.EVG_TF_OTHER_DISTRO else f"d{d}") for f, d in zip(fl.tolist(), dno.tolist())])
        t.status = k.strcol(["undispatched"] * n)
        t.priority = k.arr(soa.priority[gidx], np.int64)
        t.task_group_order = k.arr(soa.task_group_order[gidx], np.int32)
        goff = table.group_off
        gmax = np.where(gid >= 0, table.group_max_hosts[np.clip(goff[dno] + gid, 0, max(table.group_max_hosts.shape[0] - 1, 0))]
                        if table.group_max_hosts.shape[0] else 0, 0) if n else np.zeros(0)
        t.task_group_max_hosts = k.arr(gmax, np.int32)
        t.num_dependents = k.arr(soa.num_dependents[gidx], np.int32)
        t.generate_task = k.arr((fl & L.EVG_TF_GENERATE) != 0, np.uint8)
        met = (fl & L.EVG_TF_DEPS_MET) != 0
        # in-queue dependency edges, rebuilt as DependsOn ids
        dep_off = [0]
        dep_ids: List[str] = []
        found: List[int] = []
        has_edges = soa.dep_idx is not None
        for pos, (g, d) in enumerate(zip(gidx.tolist(), dno.tolist())):
            if has_edges:
                for e in range(int(soa.dep_off[g]), int(soa.dep_off[g + 1])):
                    dep_ids.append(f"d{d}t{int(soa.dep_idx[e])}")
                    found.append(1)
            if not met[pos] and dep_off[-1] == len(dep_ids):
                dep_ids.append("not-in-queue")  # an unmet dependency outside the queue
                found.append(0)
            dep_off.append(len(dep_ids))
        dep_cnt = np.diff(np.array(dep_off, dtype=np.int64))
        # the SoA's deps-met bit and wait basis are already resolved: OverrideDependencies makes every met task with
        # dependencies take the HasDependenciesMet short-circuit (task.go:3393), so the oracle does not re-stamp
        # DependenciesMetTime (task.go:653) on them
        t.override_dependencies = k.arr(met & (dep_cnt > 0), np.uint8)
        t.blocked = k.arr(np.zeros(n), np.uint8)
        t.activated_time = k.arr(soa.queue_basis_ns[gidx], np.int64)
        t.ingest_time = k.arr(np.full(n, ZERO), np.int64)
        t.scheduled_time = k.arr(soa.wait_basis_ns[gidx], np.int64)
        t.dependencies_met_time = k.arr(np.full(n, ZERO), np.int64)
        t.expected_ns = k.arr(soa.expected_ns[gidx], np.int64)
        t.dep_off = k.arr(dep_off, np.int64)
        t.dep_task_id = k.strcol(dep_ids)
        t.dep_status = k.strcol([""] * len(dep_ids))
        t.dep_found = k.arr(np.zeros(len(dep_ids)), np.uint8)  # edges resolve in-queue; the extra one is missing
        t.dep_task_status = k.strcol([""] * len(dep_ids))
        t.dep_task_blocked = k.arr(np.zeros(len(dep_ids)), np.uint8)
        t.dep_finished_at = None
        # settings
        self.ps = (PlannerSettings * max(len(sel), 1))()
        self.distro_ids = (C.c_char_p * max(len(sel), 1))()
        for j, d in enumerate(sel):
            c = table.cfg[d]
            s = self.ps[j]
            for f in ("patch_factor", "patch_time_in_queue_factor", "commit_queue_factor", "mainline_time_in_queue_factor",
                      "expected_runtime_factor", "generate_task_factor", "stepback_task_factor"):
                setattr(s, f, int(c[f]))
            s.num_dependents_factor = float(c["num_dependents_factor"])
            s.target_time_ns = int(c["target_time_ns"])
            s.group_versions = int(c["group_versions"])
            s.includes_dependencies = int(c["includes_dependencies"])
            b = f"d{d}".encode()
            k.refs.append(b)
            self.distro_ids[j] = b
        # hosts
        self.hosts = None
        if hosts is not None:
            hoff = hosts.host_off
            hr = [(int(hoff[d]), int(hoff[d + 1])) for d in sel]
            hn = sum(b - a for a, b in hr)
            self.host_off = np.zeros(len(sel) + 1, dtype=np.int64)
            np.cumsum([b - a for a, b in hr], out=self.host_off[1:])
            hidx = np.concatenate([np.arange(a, b) for a, b in hr]) if hn else np.zeros(0, dtype=np.int64)
            hd = np.concatenate([np.full(b - a, d, dtype=np.int64) for d, (a, b) in zip(sel, hr)]) if hn else np.zeros(0, dtype=np.int64)
            hf = hosts.flags[hidx]
            hg = hosts.group_id[hidx]
            # version string of each group = version of any task in it
            gver = {}
            for pos, (d, g, v) in enumerate(zip(dno.tolist(), gid.tolist(), vers)):
                if g >= 0:
                    gver.setdefault((d, g), v)
            h = self.hosts = Hosts()
            h.n = hn
            run = (hf & L.EVG_HF_RUNNING) != 0
            h.running_task = k.strcol([(f"rt{i}" if r else "") for i, r in enumerate(run.tolist())])
            rg, rbv, rp, rv = [], [], [], []
            for d, g, r in zip(hd.tolist(), hg.tolist(), run.tolist()):
                if not r or g == L.EVG_HG_NONE:
                    rg.append(""); rbv.append(""); rp.append(""); rv.append("")
                elif g >= 0:
                    rg.append(f"tg{g}"); rbv.append("bv"); rp.append("p"); rv.append(gver.get((d, g), "?"))
                else:
                    rg.append("gone"); rbv.append("bv"); rp.append("p"); rv.append("old")
            h.running_task_group, h.running_task_bv = k.strcol(rg), k.strcol(rbv)
            h.running_task_project, h.running_task_version = k.strcol(rp), k.strcol(rv)
            h.teardown_start_time = k.arr(np.where((hf & L.EVG_HF_TEARDOWN) != 0, 1, ZERO), np.int64)
            h.rt_found = k.arr((hf & L.EVG_HF_RT_FOUND) != 0, np.uint8)
            h.rt_expected_ns = k.arr(hosts.expected_ns[hidx], np.int64)
            h.rt_std_ns = k.arr(hosts.std_ns[hidx], np.int64)
            h.rt_start_time = k.arr(hosts.start_ns[hidx], np.int64)
            self.alloc = (AllocSettings * max(len(sel), 1))()
            prov = {L.EVG_PROVIDER_STATIC: b"static", L.EVG_PROVIDER_EPHEMERAL: b"ec2-fleet", L.EVG_PROVIDER_DOCKER: b"docker"}
            for j, d in enumerate(sel):
                c = hosts.cfg[d]
                a = self.alloc[j]
                a.provider = prov[int(c["provider"])]
                a.rounding_rule = b"round-up" if int(c["round_up"]) else b"round-down"
                a.feedback_rule = b"waits-over-thresh-feedback" if int(c["waits_over_thresh_feedback"]) else b"no-feedback"
                a.disabled, a.minimum_hosts, a.maximum_hosts = int(c["disabled"]), int(c["minimum_hosts"]), int(c["maximum_hosts"])
                a.has_pool, a.pool_max_containers = int(c["has_pool"]), int(c["pool_max_containers"])
                a.parent_found, a.parent_maximum_hosts = int(c["parent_found"]), int(c["parent_maximum_hosts"])
                a.future_host_fraction = float(c["future_host_fraction"])

    def run(self, now: int, threads: int = 1):
        """plan -> queue info -> allocator for every selected distro on `threads` host threads."""
        n, D = int(self.tasks.n), len(self.sel)
        order = np.zeros(max(n, 1), dtype=np.int32)
        tv = np.zeros(max(n, 1), dtype=np.int64)
        info = np.zeros(max(D, 1), dtype=QINFO_DTYPE)
        new = np.zeros(max(D, 1), dtype=np.int64)
        free = np.zeros(max(D, 1), dtype=np.int64)
        st = np.zeros(max(D, 1), dtype=np.int32)
        have_hosts = self.hosts is not None
        groups = np.zeros(n + D + 1, dtype=GROUP_DTYPE)
        bd = np.zeros((max(n, 1), BD_N), dtype=np.int64)
        lib().evo_job_batch(C.byref(self.tasks), C.c_void_p(self.task_off.ctypes.data),
                            C.byref(self.hosts) if have_hosts else None,
                            C.c_void_p(self.host_off.ctypes.data) if have_hosts else None,
                            self.ps, self.alloc if have_hosts else None, self.distro_ids, C.c_int64(D), C.c_int64(now),
                            C.c_int32(threads), C.c_void_p(order.ctypes.data), C.c_void_p(tv.ctypes.data),
                            C.c_void_p(info.ctypes.data), C.c_void_p(new.ctypes.data), C.c_void_p(free.ctypes.data),
                            C.c_void_p(st.ctypes.data), C.c_void_p(groups.ctypes.data),
                            C.c_void_p(bd.ctypes.data))
        return {"order": order[:n], "total_value": tv[:n], "info": info[:D], "new_hosts": new[:D],
                "free_hosts": free[:D], "status": st[:D], "task_off": self.task_off, "groups": groups,
                "breakdown": bd[:n]}

    def groups_by_id(self, result, j: int, soa_group_id: np.ndarray):
        """TaskGroupInfos of selected distro j keyed by the SoA group id (-1 = the "" bucket)."""
        a = int(self.task_off[j])
        out = {}
        for g in range(int(result["info"][j]["n_groups"])):
            row = result["groups"][a + j + g]
            nt = int(row["name_task"])
            out[-1 if nt < 0 else int(soa_group_id[a + nt])] = row
        return out
