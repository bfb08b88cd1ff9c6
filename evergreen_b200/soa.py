"""SoA tables (numpy) that cross the C-ABI, and the marshalling of
reference-shaped structs (evergreen_b200.model) into them.

This is what the Go shim does on the reference side of the boundary
(INTEGRATION.md): intern the string keys the planner hashes
(task-group string, version, task id -> dense distro-local ids), resolve the
per-task inputs the reference fetches lazily (expected duration, dependency
state) and lay everything out column-wise.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import ctypes as C

import numpy as np

from . import _lib as L
from . import model as M


@dataclass
class TaskSoA:
    """evg_task_soa (include/evg_sched.h). 48 B per task."""
    priority: np.ndarray
    expected_ns: np.ndarray
    queue_basis_ns: np.ndarray
    wait_basis_ns: np.ndarray
    num_dependents: np.ndarray
    task_group_order: np.ndarray
    group_id: np.ndarray
    version_id: np.ndarray
    flags: np.ndarray
    dep_off: Optional[np.ndarray] = None
    dep_idx: Optional[np.ndarray] = None

    COLUMNS = (("priority", np.int32), ("expected_ns", np.int64), ("queue_basis_ns", np.int64),
               ("wait_basis_ns", np.int64), ("num_dependents", np.int32), ("task_group_order", np.int32),
               ("group_id", np.int32), ("version_id", np.int32), ("flags", np.uint32))

    @property
    def n_tasks(self) -> int:
        return int(self.priority.shape[0])

    @property
    def n_edges(self) -> int:
        return 0 if self.dep_idx is None else int(self.dep_idx.shape[0])

    def normalize(self) -> "TaskSoA":
        for name, dt in self.COLUMNS:
            setattr(self, name, np.ascontiguousarray(getattr(self, name), dtype=dt))
        if self.dep_idx is not None and self.dep_idx.shape[0] > 0:
            self.dep_off = np.ascontiguousarray(self.dep_off, dtype=np.int64)
            self.dep_idx = np.ascontiguousarray(self.dep_idx, dtype=np.int32)
        else:
            self.dep_off, self.dep_idx = None, None
        return self

    def struct(self) -> L.TaskSoAStruct:
        s = L.TaskSoAStruct()
        s.n_tasks, s.n_edges = self.n_tasks, self.n_edges
        for name, _ in self.COLUMNS:
            setattr(s, name, L.ptr(getattr(self, name)))
        s.dep_off, s.dep_idx = L.ptr(self.dep_off), L.ptr(self.dep_idx)
        return s

    def nbytes(self) -> int:
        n = sum(getattr(self, name).nbytes for name, _ in self.COLUMNS)
        if self.dep_idx is not None:
            n += self.dep_off.nbytes + self.dep_idx.nbytes
        return n


@dataclass
class DistroTable:
    """evg_distro_table."""
    task_off: np.ndarray
    group_off: np.ndarray
    cfg: np.ndarray              # L.DISTRO_CFG_DTYPE
    group_max_hosts: np.ndarray

    @property
    def n_distros(self) -> int:
        return int(self.cfg.shape[0])

    @property
    def n_groups(self) -> int:
        return int(self.group_off[-1]) if self.group_off.shape[0] else 0

    def normalize(self) -> "DistroTable":
        self.task_off = np.ascontiguousarray(self.task_off, dtype=np.int64)
        self.group_off = np.ascontiguousarray(self.group_off, dtype=np.int64)
        self.cfg = np.ascontiguousarray(self.cfg, dtype=L.DISTRO_CFG_DTYPE)
        self.group_max_hosts = np.ascontiguousarray(self.group_max_hosts, dtype=np.int32)
        return self

    def struct(self) -> L.DistroTableStruct:
        s = L.DistroTableStruct()
        s.n_distros = self.n_distros
        s.task_off, s.group_off = L.ptr(self.task_off), L.ptr(self.group_off)
        s.cfg = L.ptr(self.cfg) if self.n_distros else None
        s.group_max_hosts = L.ptr(self.group_max_hosts) if self.group_max_hosts.shape[0] else None
        return s

    def nbytes(self) -> int:
        return self.task_off.nbytes + self.group_off.nbytes + self.cfg.nbytes + self.group_max_hosts.nbytes


@dataclass
class HostSoA:
    """evg_host_soa + host_off + evg_alloc_cfg[]. 32 B per host."""
    flags: np.ndarray
    group_id: np.ndarray
    expected_ns: np.ndarray
    std_ns: np.ndarray
    start_ns: np.ndarray
    host_off: np.ndarray
    cfg: np.ndarray              # L.ALLOC_CFG_DTYPE

    COLUMNS = (("flags", np.uint32), ("group_id", np.int32), ("expected_ns", np.int64), ("std_ns", np.int64),
               ("start_ns", np.int64))

    @property
    def n_hosts(self) -> int:
        return int(self.flags.shape[0])

    def normalize(self) -> "HostSoA":
        for name, dt in self.COLUMNS:
            setattr(self, name, np.ascontiguousarray(getattr(self, name), dtype=dt))
        self.host_off = np.ascontiguousarray(self.host_off, dtype=np.int64)
        self.cfg = np.ascontiguousarray(self.cfg, dtype=L.ALLOC_CFG_DTYPE)
        return self

    def struct(self) -> L.HostSoAStruct:
        s = L.HostSoAStruct()
        s.n_hosts = self.n_hosts
        for name, _ in self.COLUMNS:
            setattr(s, name, L.ptr(getattr(self, name)) if self.n_hosts else None)
        return s

    def nbytes(self) -> int:
        return sum(getattr(self, name).nbytes for name, _ in self.COLUMNS) + self.host_off.nbytes + self.cfg.nbytes


@dataclass
class PlanOutput:
    order: np.ndarray          # int32 [T]
    total_value: np.ndarray    # int64 [T]
    info: np.ndarray           # QUEUE_INFO_DTYPE [D]
    group_info: np.ndarray     # GROUP_INFO_DTYPE [G]
    breakdown: Optional[np.ndarray] = None  # int64 [T, 13]

    def nbytes(self) -> int:
        n = self.order.nbytes + self.total_value.nbytes + self.info.nbytes + self.group_info.nbytes
        return n + (self.breakdown.nbytes if self.breakdown is not None else 0)


@dataclass
class AllocOutput:
    result: np.ndarray         # ALLOC_RESULT_DTYPE [D]
    status: np.ndarray         # int32 [D]

    def nbytes(self) -> int:
        return self.result.nbytes + self.status.nbytes


def _empty_tasks() -> TaskSoA:
    return TaskSoA(**{name: np.zeros(0, dtype=dt) for name, dt in TaskSoA.COLUMNS})


@dataclass
class TaskEdit:
    """evg_task_edit: rows leave, rows join, surviving tasks gain in-queue dependencies (include/evg_sched.h).
    `group_off`, `group_max_hosts` and `cfg` describe the new distro table (None: the old one's); apply_edit builds it."""
    remove_rows: np.ndarray                       # int64, strictly ascending rows of the current table
    insert: TaskSoA                               # rows appended after their distro's survivors, ids in the new id space
    insert_off: np.ndarray                        # int64 [D+1]: CSR of `insert` over distros
    add_edge_task: np.ndarray                     # int64, ascending composed row of a surviving task
    add_edge_dep: np.ndarray                      # int32, new distro-local index of its new dependency
    group_remap: Optional[np.ndarray] = None      # int32 per old group slot: new distro-local id, -1 = no survivor in it
    version_remap: Optional[np.ndarray] = None    # int32 per old (distro, version), CSR by the old n_versions
    group_off: Optional[np.ndarray] = None
    group_max_hosts: Optional[np.ndarray] = None
    cfg: Optional[np.ndarray] = None

    def normalize(self) -> "TaskEdit":
        self.remove_rows = np.ascontiguousarray(self.remove_rows, dtype=np.int64)
        self.insert = (self.insert if self.insert is not None else _empty_tasks()).normalize()
        self.insert_off = np.ascontiguousarray(self.insert_off, dtype=np.int64)
        self.add_edge_task = np.ascontiguousarray(self.add_edge_task, dtype=np.int64)
        self.add_edge_dep = np.ascontiguousarray(self.add_edge_dep, dtype=np.int32)
        if self.group_remap is not None:
            self.group_remap = np.ascontiguousarray(self.group_remap, dtype=np.int32)
        if self.version_remap is not None:
            self.version_remap = np.ascontiguousarray(self.version_remap, dtype=np.int32)
        return self

    def struct(self):
        """-> (TaskEditStruct, the inserted rows' struct it points to: keep both alive for the call)."""
        ins = self.insert.struct()
        p = lambda a: L.ptr(a) if a is not None and a.shape[0] else None  # noqa: E731
        s = L.TaskEditStruct(int(self.remove_rows.shape[0]), p(self.remove_rows), C.pointer(ins), L.ptr(self.insert_off),
                             int(self.add_edge_task.shape[0]), p(self.add_edge_task), p(self.add_edge_dep),
                             L.ptr(self.group_remap), L.ptr(self.version_remap))
        return s, ins

    def nbytes(self) -> int:
        """What the edit moves to the device (the new distro table aside)."""
        n = self.remove_rows.nbytes + self.insert.nbytes() + self.insert_off.nbytes + self.add_edge_task.nbytes + self.add_edge_dep.nbytes
        return n + sum(a.nbytes for a in (self.group_remap, self.version_remap) if a is not None)


def apply_edit(tasks: TaskSoA, distros: DistroTable, edit: TaskEdit):
    """The composed table of evg_edit_tasks, in numpy: -> (TaskSoA, DistroTable).  Distro d's queue is its surviving
    rows in their previous order, then its inserted rows; a survivor keeps (or remaps) its group and version ids and its
    edges to survivors (re-indexed, in order), then gains its added edges; inserted rows bring their own edges."""
    edit.normalize()
    D, T0 = distros.n_distros, tasks.n_tasks
    toff = distros.task_off
    ins = edit.insert
    keep = np.ones(T0, dtype=bool)
    keep[edit.remove_rows] = False
    distro_of = np.repeat(np.arange(D, dtype=np.int64), np.diff(toff))
    surv = np.nonzero(keep)[0]
    surv_d = distro_of[surv]
    n_surv = np.bincount(surv_d, minlength=D).astype(np.int64)
    n_ins = np.diff(edit.insert_off)
    new_off = np.concatenate([[0], np.cumsum(n_surv + n_ins)]).astype(np.int64)
    surv_first = np.concatenate([[0], np.cumsum(n_surv)])
    surv_new = new_off[surv_d] + np.arange(surv.shape[0]) - surv_first[surv_d]
    ins_d = np.repeat(np.arange(D, dtype=np.int64), n_ins)
    ins_new = new_off[ins_d] + n_surv[ins_d] + np.arange(ins.n_tasks) - edit.insert_off[ins_d]
    Tn = int(new_off[-1])
    cols = {}
    for name, dt in TaskSoA.COLUMNS:
        col = np.zeros(Tn, dtype=dt)
        col[surv_new] = getattr(tasks, name)[surv]
        col[ins_new] = getattr(ins, name)
        cols[name] = col
    if edit.group_remap is not None:
        g = tasks.group_id[surv].astype(np.int64)
        m = g >= 0
        g[m] = edit.group_remap[distros.group_off[surv_d[m]] + g[m]]
        if np.any(g[m] < 0):
            raise ValueError("group_remap maps the task group of a surviving task to -1")
        cols["group_id"][surv_new] = g
    if edit.version_remap is not None:
        vbase = np.concatenate([[0], np.cumsum(distros.cfg["n_versions"].astype(np.int64))])
        cols["version_id"][surv_new] = edit.version_remap[vbase[surv_d] + tasks.version_id[surv]]
    # edges: (owner composed row, dependency) from three sources; a stable sort by owner keeps each source's order and
    # a survivor's old edges ahead of its added ones
    owners, deps = [], []
    if tasks.n_edges:
        new_local = np.full(T0, -1, dtype=np.int64)
        new_local[surv] = surv_new - new_off[surv_d]
        deg = np.diff(tasks.dep_off)
        own = np.repeat(np.arange(T0, dtype=np.int64), deg)
        tgt = toff[distro_of[own]] + tasks.dep_idx
        live = keep[own] & keep[tgt]
        old_to_new = np.full(T0, -1, dtype=np.int64)
        old_to_new[surv] = surv_new
        owners.append(old_to_new[own[live]])
        deps.append(new_local[tgt[live]])
    owners.append(edit.add_edge_task)
    deps.append(edit.add_edge_dep.astype(np.int64))
    if ins.n_edges:
        owners.append(np.repeat(ins_new, np.diff(ins.dep_off)))
        deps.append(ins.dep_idx.astype(np.int64))
    owner = np.concatenate(owners) if owners else np.zeros(0, np.int64)
    dep = np.concatenate(deps) if deps else np.zeros(0, np.int64)
    o = np.argsort(owner, kind="stable")
    dep_off = np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=Tn))]).astype(np.int64)
    new_tasks = TaskSoA(**cols, dep_off=dep_off, dep_idx=dep[o].astype(np.int32)).normalize()
    new_distros = DistroTable(new_off, distros.group_off if edit.group_off is None else edit.group_off,
                              distros.cfg if edit.cfg is None else edit.cfg,
                              distros.group_max_hosts if edit.group_max_hosts is None else edit.group_max_hosts)
    return new_tasks, DistroTable(**{k: np.array(v, copy=True) for k, v in vars(new_distros).items()}).normalize()


# ---------------------------------------------------------------------------
# marshalling reference-shaped structs -> SoA
# ---------------------------------------------------------------------------

def planner_cfg_row(d: M.Distro, includes_dependencies: bool, n_versions: int) -> tuple:
    ps = d.planner_settings
    return (ps.patch_factor, ps.patch_time_in_queue_factor, ps.commit_queue_factor,
            ps.mainline_time_in_queue_factor, ps.expected_runtime_factor, ps.generate_task_factor,
            ps.stepback_task_factor, float(ps.num_dependents_factor), d.get_target_time(),
            int(ps.should_group_versions()), int(includes_dependencies), n_versions, 0)


def requester_class(r: str) -> int:
    if M.is_github_merge_queue_requester(r):
        return L.EVG_TF_REQ_MERGE_QUEUE
    if M.is_patch_requester(r):
        return L.EVG_TF_REQ_PATCH
    return L.EVG_TF_REQ_OTHER


def satisfies_dependency(dep: M.Dependency, dep_task: M.Task) -> bool:
    """Task.SatisfiesDependency (model/task/task.go:529-543)."""
    if dep.status in (M.TASK_SUCCEEDED, ""):
        return dep_task.status == M.TASK_SUCCEEDED
    if dep.status == M.TASK_FAILED:
        return dep_task.status == M.TASK_FAILED
    if dep.status == M.ALL_STATUSES:
        return dep_task.status in (M.TASK_FAILED, M.TASK_SUCCEEDED) or dep_task.blocked()
    return False


def dependencies_met(t: M.Task, in_queue: Dict[str, M.Task], db: Optional[Dict[str, M.Task]],
                     now: Optional[int] = None) -> bool:
    """Task.DependenciesMet (model/task/task.go:632-671) against the in-queue
    cache first, then `db` (the tasks collection lookup); a missing dependency
    is the lookup error checkDependenciesMet turns into false (scheduler.go:161-168).
    With `now`, a fresh evaluation that comes out met stamps DependenciesMetTime on the task like the reference
    does (setDependenciesMetTime, task.go:653,673-684): the latest non-zero FinishedAt of its dependencies, else now."""
    if t.has_dependencies_met():
        return True
    for dep in t.depends_on:
        dep_task = in_queue.get(dep.task_id)
        if dep_task is None and db is not None:
            dep_task = db.get(dep.task_id)
        if dep_task is None:
            return False
        if not satisfies_dependency(dep, dep_task):
            return False
    if now is not None:
        best = M.ZERO_TIME
        for dep in t.depends_on:
            if not M.is_zero_time(dep.finished_at) and dep.finished_at > best:
                best = dep.finished_at
        t.dependencies_met_time = now if M.is_zero_time(best) else best
    return True


@dataclass
class MarshalledDistro:
    """Key tables the shim keeps to translate results back to strings."""
    group_names: List[str] = field(default_factory=list)
    versions: List[str] = field(default_factory=list)


def marshal_tasks(batch: Sequence[tuple], now: int, dependency_db: Optional[Dict[str, M.Task]] = None,
                  duration_history: Optional[dict] = None, resolve_deps: bool = False, resolve_durations: bool = True,
                  intern: bool = True):
    """[(Distro, [Task])] -> (TaskSoA, DistroTable, [MarshalledDistro]).

    Per task this resolves FetchExpectedDuration (PopulateCaches, setup_funcs.go:20-67), which writes the task's
    DurationPrediction back like the reference.  resolve_durations=False leaves the tasks untouched and uploads
    Task.ExpectedDuration as it is, for callers that resolve the durations on the device (evg_resolve_durations).  Task.DependenciesMet
    (scheduler.go:161-168) is the DEVICE's job: the product path pairs these columns with marshal_deps() and
    Engine.upload_with_deps(), which sets the EVG_TF_DEPS_MET bit and the stamped wait basis on the GPU.
    resolve_deps=True evaluates it here instead (host restatement, kept for tests and for callers of the plain
    one-shot entry points that want self-contained columns).  intern=False skips the string work (task groups,
    versions, in-queue edges) for callers that let the device intern the strings (evg_upload_strings,
    evg_edit_strings): group_id is then -1, version_id 0, there are no edges, no groups and no key tables."""
    cols = {name: [] for name, _ in TaskSoA.COLUMNS}
    dep_off, dep_idx = [0], []
    task_off, group_off, cfg_rows, gmax, keys = [0], [0], [], [], []
    for d, tasks in batch:
        if len(tasks) > L.MAX_TASKS_PER_DISTRO:
            raise ValueError(f"distro {d.id!r}: {len(tasks)} tasks exceed {L.MAX_TASKS_PER_DISTRO}")
        incl = d.dispatcher_settings.version == M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES  # scheduler.go:28
        index = {t.id: i for i, t in enumerate(tasks)} if intern else {}
        by_id = {t.id: t for t in tasks}
        groups: Dict[str, int] = {}
        versions: Dict[str, int] = {}
        md = MarshalledDistro()
        for t in tasks:
            if resolve_durations:
                hist = None if duration_history is None else duration_history.get((t.project, t.build_variant, t.display_name))
                avg, _ = M.fetch_expected_duration(t, now, hist)
            else:
                avg = t.expected_duration
            gid, vid = -1, 0
            if intern and t.task_group != "":
                name = t.get_task_group_string()
                gid = groups.get(name)
                if gid is None:
                    gid = groups[name] = len(groups)
                    md.group_names.append(name)
                    gmax.append(t.task_group_max_hosts)
                elif gmax[group_off[-1] + gid] != t.task_group_max_hosts:
                    # TaskGroupInfo.MaxHosts is the value of the group's first task in PLAN order (scheduler.go:87-90);
                    # a per-group table can only carry one value, so members must agree (they do: it is a project setting)
                    raise ValueError(f"task group {name!r}: TaskGroupMaxHosts differs between members "
                                     f"({gmax[group_off[-1] + gid]} vs {t.task_group_max_hosts} on {t.id!r})")
            if intern:
                vid = versions.get(t.version)
                if vid is None:
                    vid = versions[t.version] = len(versions)
                    md.versions.append(t.version)
            qb = t.activated_time if t.activated_time != M.ZERO_TIME else t.ingest_time  # planner.go:318-322
            # checkDependenciesMet runs first (scheduler.go:82-98) and, on a fresh evaluation, stamps DependenciesMetTime
            # on the task (task.go:653); the wait is measured after that (scheduler.go:119-123)
            deps_met = dependencies_met(t, by_id, dependency_db, now) if resolve_deps else False
            wb = max(t.scheduled_time, t.dependencies_met_time)  # ZERO_TIME sorts first
            fl = requester_class(t.requester)
            if t.generate_task:
                fl |= L.EVG_TF_GENERATE
            if t.activated_by == M.STEPBACK_TASK_ACTIVATOR:
                fl |= L.EVG_TF_STEPBACK
            if deps_met:
                fl |= L.EVG_TF_DEPS_MET
            if t.distro_id != d.id:
                fl |= L.EVG_TF_OTHER_DISTRO
            if not -2 ** 31 <= t.priority < 2 ** 31 or not -2 ** 31 <= t.num_dependents < 2 ** 31:
                # evg_task_soa carries both as int32; Go's Task.Priority is an int64 whose valid range ends at
                # evergreen.MaxTaskPriority (100, globals.go:185), so a value out here is a corrupt document
                raise ValueError(f"task {t.id!r}: priority {t.priority} / num_dependents {t.num_dependents} outside int32")
            cols["priority"].append(t.priority)
            cols["expected_ns"].append(avg)
            cols["queue_basis_ns"].append(qb)
            cols["wait_basis_ns"].append(wb)
            cols["num_dependents"].append(t.num_dependents)
            cols["task_group_order"].append(t.task_group_order)
            cols["group_id"].append(gid)
            cols["version_id"].append(vid)
            cols["flags"].append(fl)
            for dep in t.depends_on if intern else ():  # only dependencies that are in this queue join units (planner.go:453)
                j = index.get(dep.task_id)
                if j is not None:
                    dep_idx.append(j)
            dep_off.append(len(dep_idx))
        task_off.append(task_off[-1] + len(tasks))
        group_off.append(group_off[-1] + len(groups))
        cfg_rows.append(planner_cfg_row(d, incl, len(versions)))
        keys.append(md)
    soa = TaskSoA(**{name: np.array(cols[name], dtype=dt) for name, dt in TaskSoA.COLUMNS},
                  dep_off=np.array(dep_off, dtype=np.int64), dep_idx=np.array(dep_idx, dtype=np.int32)).normalize()
    table = DistroTable(np.array(task_off, dtype=np.int64), np.array(group_off, dtype=np.int64),
                        np.array(cfg_rows, dtype=L.DISTRO_CFG_DTYPE), np.array(gmax, dtype=np.int32)).normalize()
    return soa, table, keys


def pack_strings(strings: Sequence):
    """[str or bytes] -> (uint8 bytes, int64 offsets[n+1]): an evg_str_col (a str is encoded as UTF-8)."""
    enc = [x.encode() if isinstance(x, str) else bytes(x) for x in strings]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    if enc:
        np.cumsum([len(b) for b in enc], out=off[1:])
    return np.frombuffer(b"".join(enc), dtype=np.uint8).copy() if enc else np.zeros(0, np.uint8), off


@dataclass
class StringCols:
    """evg_string_cols (include/evg_sched.h), packed once: each task's id, version, task-group key ("" without a task
    group) and TaskGroupMaxHosts, and its DependsOn ids, concatenated distro by distro.  evg_intern_columns,
    evg_intern_batch and evg_upload_strings all read this."""
    task_off: np.ndarray
    id: tuple          # pack_strings of Task.Id
    version: tuple     # ... of Task.Version
    group_key: tuple   # ... of Task.GetTaskGroupString(), "" when TaskGroup == ""
    group_max_hosts: np.ndarray
    dep_off: np.ndarray
    dep_id: tuple      # ... of Dependency.TaskId, dep_off[-1] strings

    @classmethod
    def pack(cls, task_off, ids, versions, group_keys, group_max_hosts, dep_off, dep_ids) -> "StringCols":
        return cls(np.ascontiguousarray(task_off, np.int64), pack_strings(ids), pack_strings(versions), pack_strings(group_keys),
                   np.ascontiguousarray(group_max_hosts, np.int32), np.ascontiguousarray(dep_off, np.int64), pack_strings(dep_ids))

    @property
    def n_tasks(self) -> int:
        return int(self.dep_off.shape[0]) - 1

    @property
    def n_distros(self) -> int:
        return int(self.task_off.shape[0]) - 1

    def struct(self) -> L.StringColsStruct:
        col = lambda c: L.StrColStruct(L.ptr(c[0]) if c[0].shape[0] else None, L.ptr(c[1]))  # noqa: E731
        return L.StringColsStruct(self.n_tasks, self.n_distros, L.ptr(self.task_off), col(self.id), col(self.version),
                                  col(self.group_key), L.ptr(self.group_max_hosts) if self.n_tasks else None, L.ptr(self.dep_off),
                                  col(self.dep_id))

    def intern_out(self):
        """Arrays for every evg_intern_out field, sized for this batch -> (dict, InternOutStruct over them)."""
        T, D, E = self.n_tasks, self.n_distros, int(self.dep_off[-1])
        out = dict(group_id=np.empty(T, np.int32), version_id=np.empty(T, np.int32), group_off=np.zeros(D + 1, np.int64),
                   n_versions=np.zeros(D, np.int32), group_max_hosts=np.empty(max(T, 1), np.int32),
                   group_first=np.empty(max(T, 1), np.int64), dep_off=np.zeros(T + 1, np.int64), dep_idx=np.empty(max(E, 1), np.int32))
        return out, L.InternOutStruct(*[L.ptr(out[k]) for k in INTERN_OUT_FIELDS])

    def trim(self, out: dict) -> dict:
        """An intern_out dict after the call: the group tables and edges cut to the counts the offsets give."""
        G, En = int(out["group_off"][-1]), int(out["dep_off"][-1])
        out["group_max_hosts"], out["group_first"], out["dep_idx"] = out["group_max_hosts"][:G], out["group_first"][:G], out["dep_idx"][:En]
        return out


INTERN_OUT_FIELDS = ("group_id", "version_id", "group_off", "n_versions", "group_max_hosts", "group_first", "dep_off", "dep_idx")


def string_cols(batch: Sequence[tuple]) -> StringCols:
    """The strings of a tick, [(distro, [task])], packed as evg_string_cols."""
    tasks = [t for _, ts in batch for t in ts]
    task_off = np.zeros(len(batch) + 1, dtype=np.int64)
    if batch:
        np.cumsum([len(ts) for _, ts in batch], out=task_off[1:])
    dep_off = np.zeros(len(tasks) + 1, dtype=np.int64)
    if tasks:
        np.cumsum([len(t.depends_on) for t in tasks], out=dep_off[1:])
    return StringCols.pack(task_off, [t.id for t in tasks], [t.version for t in tasks],
                           [t.get_task_group_string() if t.task_group != "" else "" for t in tasks],
                           np.array([t.task_group_max_hosts for t in tasks], dtype=np.int32), dep_off,
                           [dep.task_id for t in tasks for dep in t.depends_on])


def intern_columns(batch: Sequence[tuple], threads: int = 0):
    """evg_intern_columns over a tick: the string work of marshal_tasks (task-group keys and versions to dense ids in
    first-appearance order, dependency ids to queue indices) in the library's C++ instead of Python dicts.
    -> dict(group_id, version_id, group_off, n_versions, group_max_hosts, group_first, dep_off, dep_idx)."""
    lib = L.load()
    sc = string_cols(batch)
    out, outs = sc.intern_out()
    L.check(lib.evg_intern_columns(C.byref(sc.struct()), C.byref(outs), int(threads)))
    return sc.trim(out)


@dataclass
class StringEdit:
    """evg_string_edit (include/evg_sched.h): rows leave and join a tick whose strings the device keeps.  The inserted
    rows bring their numeric columns (their ids and edges come from their strings, so `insert`'s group_id, version_id
    and edges are not sent) and their strings; the strings' task_off is the inserted rows' CSR over distros."""
    remove_rows: np.ndarray   # int64, strictly ascending rows of the resident table
    insert: TaskSoA
    strings: StringCols

    @property
    def insert_off(self) -> np.ndarray:
        return self.strings.task_off

    def struct(self):
        """-> (StringEditStruct, the structs it points to: keep both alive for the call)."""
        self.remove_rows = np.ascontiguousarray(self.remove_rows, dtype=np.int64)
        ins = self.insert.normalize().struct()
        ins.n_edges, ins.group_id, ins.version_id, ins.dep_off, ins.dep_idx = 0, None, None, None, None
        st = self.strings.struct()
        R = int(self.remove_rows.shape[0])
        s = L.StringEditStruct(R, L.ptr(self.remove_rows) if R else None, C.pointer(ins), L.ptr(self.insert_off), C.pointer(st))
        return s, (ins, st)

    def nbytes(self) -> int:
        """What the edit moves to the device: the removed rows, the inserted rows' seven numeric columns and strings."""
        sc = self.strings
        n = self.remove_rows.nbytes + sum(getattr(self.insert, name).nbytes for name in
                                          ("priority", "expected_ns", "queue_basis_ns", "wait_basis_ns", "num_dependents",
                                           "task_group_order", "flags"))
        n += sc.task_off.nbytes + sc.group_max_hosts.nbytes + sc.dep_off.nbytes
        return n + sum(c[0].nbytes + c[1].nbytes for c in (sc.id, sc.version, sc.group_key, sc.dep_id))


def _gather_strings(cols: Sequence[tuple], rows: np.ndarray) -> tuple:
    """Strings `rows` of the concatenation of the string columns `cols`, in that order -> (bytes, offsets)."""
    data = np.concatenate([c[0] for c in cols]) if cols else np.zeros(0, np.uint8)
    base = np.cumsum([0] + [c[0].shape[0] for c in cols])[:-1]
    start = np.concatenate([c[1][:-1] + b for c, b in zip(cols, base)]).astype(np.int64)
    lens = np.concatenate([np.diff(c[1]) for c in cols]).astype(np.int64)
    ln = lens[rows]
    off = np.concatenate([[0], np.cumsum(ln)]).astype(np.int64)
    idx = np.repeat(start[rows] - off[:-1], ln) + np.arange(int(off[-1]), dtype=np.int64)
    return np.ascontiguousarray(data[idx], np.uint8), off


def compose_strings(old: StringCols, edit: StringEdit) -> StringCols:
    """The composed string table of evg_edit_strings, in numpy: distro d's rows are its rows of `old` that
    edit.remove_rows does not name, in their order, then its rows of edit.strings."""
    ins = edit.strings
    T0, I, D = old.n_tasks, ins.n_tasks, old.n_distros
    keep = np.ones(T0, dtype=bool)
    keep[np.asarray(edit.remove_rows, np.int64)] = False
    distro = np.concatenate([np.repeat(np.arange(D), np.diff(old.task_off)), np.repeat(np.arange(D), np.diff(ins.task_off))])
    src = np.nonzero(np.concatenate([keep, np.ones(I, dtype=bool)]))[0]
    rows = src[np.argsort(distro[src], kind="stable")]  # old rows (< T0) sit before inserted ones within a distro
    task_off = np.concatenate([[0], np.cumsum(np.bincount(distro[src], minlength=D))]).astype(np.int64)
    # the DependsOn ids of each composed row: its range of the concatenated dep_off
    dstart = np.concatenate([old.dep_off[:-1], ins.dep_off[:-1] + old.dep_off[-1]]).astype(np.int64)
    dlen = np.concatenate([np.diff(old.dep_off), np.diff(ins.dep_off)]).astype(np.int64)[rows]
    dep_off = np.concatenate([[0], np.cumsum(dlen)]).astype(np.int64)
    edges = np.repeat(dstart[rows] - dep_off[:-1], dlen) + np.arange(int(dep_off[-1]), dtype=np.int64)
    return StringCols(task_off, _gather_strings([old.id, ins.id], rows), _gather_strings([old.version, ins.version], rows),
                      _gather_strings([old.group_key, ins.group_key], rows),
                      np.ascontiguousarray(np.concatenate([old.group_max_hosts, ins.group_max_hosts])[rows], np.int32), dep_off,
                      _gather_strings([old.dep_id, ins.dep_id], edges))


def provider_class(provider: str) -> int:
    if provider == M.PROVIDER_DOCKER:
        return L.EVG_PROVIDER_DOCKER
    if provider in M.PROVIDER_SPAWNABLE:
        return L.EVG_PROVIDER_EPHEMERAL
    return L.EVG_PROVIDER_STATIC


def alloc_cfg_row(data: M.HostAllocatorData) -> tuple:
    d = data.distro
    hs = d.host_allocator_settings
    pool = data.container_pool
    return (float(hs.future_host_fraction), provider_class(d.provider), int(d.disabled), hs.minimum_hosts,
            hs.maximum_hosts, int(hs.rounding_rule == M.HOST_ALLOCATOR_ROUND_UP),
            int(hs.feedback_rule == M.HOST_ALLOCATOR_WAITS_OVER_THRESH_FEEDBACK),
            int(pool is not None), pool.max_containers if pool else 0,
            int(data.parent_distro_maximum_hosts is not None),
            data.parent_distro_maximum_hosts if data.parent_distro_maximum_hosts is not None else 0)


def marshal_hosts(datas: Sequence[M.HostAllocatorData], group_names: Sequence[Sequence[str]],
                  running_tasks: Optional[Dict[str, M.Task]] = None) -> HostSoA:
    """[HostAllocatorData] -> HostSoA.  `group_names[d]` is the distro's group
    table (slot order of its TaskGroupInfos); hosts are bucketed like
    groupByTaskGroup (utilization_based_host_allocator.go:223-260).  `running_tasks` (task id -> Task): the documents
    task.Find(ByIds) returned (allocator.go:337); a host whose running task is one of them is found, with its StartTime
    and its ExpectedDuration / StdDev as stored (evg_resolve_durations replaces those on the device).  Other hosts
    read HostAllocatorData.running_tasks."""
    fl, gid, exp, std, start, off, rows = [], [], [], [], [], [0], []
    for data, names in zip(datas, group_names):
        lookup = {n: i for i, n in enumerate(names)}
        for h in data.existing_hosts:
            f = 0
            g = L.EVG_HG_NONE
            e = s = 0
            st = M.ZERO_TIME
            if h.running_task != "":
                f |= L.EVG_HF_RUNNING
                doc = running_tasks.get(h.running_task) if running_tasks is not None else None
                rt = data.running_tasks.get(h.running_task) if doc is None else \
                    M.RunningTaskStats(True, doc.expected_duration, doc.expected_duration_std_dev, doc.start_time)
                if rt is not None and rt.found:
                    f |= L.EVG_HF_RT_FOUND
                    e, s, st = rt.expected, rt.std_dev, rt.start_time
                if h.running_task_group != "":
                    g = lookup.get(h.get_task_group_string(), L.EVG_HG_UNQUEUED)
            if h.task_group_teardown_start_time != M.ZERO_TIME:
                f |= L.EVG_HF_TEARDOWN
            fl.append(f); gid.append(g); exp.append(e); std.append(s); start.append(st)
        off.append(len(fl))
        rows.append(alloc_cfg_row(data))
    return HostSoA(np.array(fl, dtype=np.uint32), np.array(gid, dtype=np.int32), np.array(exp, dtype=np.int64),
                   np.array(std, dtype=np.int64), np.array(start, dtype=np.int64), np.array(off, dtype=np.int64),
                   np.array(rows, dtype=L.ALLOC_CFG_DTYPE)).normalize()


def marshal_host_job(datas: Sequence[M.HostAllocatorData], n_provisioning: Sequence[int]) -> np.ndarray:
    """[HostAllocatorData] + len(ProvisioningHosts()) per distro -> HOST_JOB_CFG rows (evg_host_job_cfg): what
    hostAllocatorJob.Run reads besides the allocator's inputs (units/host_allocator.go:169-184, 330-333).  The billing
    rule reads the distro itself: the up hosts' embedded distro document is that distro."""
    from .scheduler import uses_hourly_billing
    if len(n_provisioning) != len(datas):
        raise ValueError("one provisioning count per distro")
    rows = np.zeros(len(datas), dtype=L.HOST_JOB_CFG_DTYPE)
    for i, (data, n) in enumerate(zip(datas, n_provisioning)):
        d = data.distro
        rows[i] = (int(n), int(d.single_task_distro),
                   int(d.host_allocator_settings.hosts_overallocated_rule == M.HOSTS_OVERALLOCATED_TERMINATE),
                   int(uses_hourly_billing(d)), 0)
    return rows


@dataclass
class IdleHostTable:
    """evg_idle_host_soa + idle_off: the idle hosts of every distro, grouped by distro in the job's query order.
    ``ids`` keeps each row's host id for the shim's follow-up (SetDecommissioned / a termination job)."""
    cols: Dict[str, np.ndarray]   # L.IDLE_HOST_COLUMNS, int64
    flags: np.ndarray             # uint32 EVG_IH_*
    idle_off: np.ndarray          # int64, n_distros + 1
    ids: List[str] = field(default_factory=list)

    @property
    def n_hosts(self) -> int:
        return int(self.flags.shape[0])

    @property
    def n_distros(self) -> int:
        return int(self.idle_off.shape[0]) - 1

    def struct(self) -> L.IdleHostSoAStruct:
        s = L.IdleHostSoAStruct()
        s.n_hosts, s.n_distros = self.n_hosts, self.n_distros
        for name in L.IDLE_HOST_COLUMNS:
            setattr(s, name, L.ptr(self.cols[name]) if self.n_hosts else None)
        s.flags = L.ptr(self.flags) if self.n_hosts else None
        return s


def idle_host_flags(h: M.Host, default_ami: Optional[str] = None) -> int:
    """The EVG_IH_* bits of one host, resolved from the host document and its lookups.  ``default_ami``: the distro
    document's GetDefaultAMI() (the idle-host job); None leaves EVG_IH_OUTDATED_AMI clear (the drawdown job)."""
    m = h.bootstrap_method
    f = ((L.EVG_IH_RUNNING_TASK_GROUP if h.running_task_group else 0) | (L.EVG_IH_LAST_TASK if h.last_task else 0)
         | (L.EVG_IH_STATUS_RUNNING if h.status == M.HOST_RUNNING else 0)
         | (L.EVG_IH_USER_DATA if m == M.BOOTSTRAP_METHOD_USER_DATA else 0)
         | (L.EVG_IH_LEGACY_BOOTSTRAP if m in ("", M.BOOTSTRAP_METHOD_LEGACY_SSH) else 0)  # LegacyBootstrap (distro.go:842-844)
         | (L.EVG_IH_NEEDS_NEW_AGENT if h.needs_new_agent else 0)
         | (L.EVG_IH_NEEDS_NEW_AGENT_MONITOR if h.needs_new_agent_monitor else 0)
         | (L.EVG_IH_OUTDATED_AMI if default_ami is not None and h.ami != default_ami else 0)
         | (L.EVG_IH_PAYMENT_NOT_DUE if h.time_til_next_payment > 5 * M.MINUTE else 0)  # maxTimeTilNextPayment
         | (L.EVG_IH_CLOUD_MANAGER_FAILED if h.cloud_manager_error else 0))
    if h.last_group:  # isAssignedSingleHostTaskGroup's LastGroup branch (units/host_monitoring_idle_termination.go:239-251)
        f |= L.EVG_IH_TASK_LOOKUP_FAILED if h.last_task_single_host_task_group is None else (
            L.EVG_IH_SINGLE_HOST_TASK_GROUP if h.last_task_single_host_task_group else 0)
    return f


_IDLE_HOST_TIMES = (("creation_ns", "creation_time"), ("start_ns", "start_time"), ("provision_ns", "provision_time"),
                    ("agent_start_ns", "agent_start_time"), ("last_communication_ns", "last_communication_time"),
                    ("last_task_completed_ns", "last_task_completed_time"),
                    ("teardown_start_ns", "task_group_teardown_start_time"), ("acceptable_idle_ns", "acceptable_host_idle_time"))


def marshal_idle_hosts(groups: Sequence[Sequence[M.Host]], default_amis: Optional[Sequence[str]] = None) -> IdleHostTable:
    """Idle hosts per distro, in the query's order -> the idle-host table.  ``default_amis``: each distro's
    GetDefaultAMI() for the idle-host job, None for the drawdown job.  A time outside the int64 nanosecond range is
    rejected, not clamped: the device would compare a different instant."""
    if default_amis is not None and len(default_amis) != len(groups):
        raise ValueError("one default AMI per distro")
    hosts = [h for g in groups for h in g]
    cols = {}
    for col, attr in _IDLE_HOST_TIMES:
        vals = [getattr(h, attr) for h in hosts]
        for h, v in zip(hosts, vals):
            if not -(2 ** 63) <= v < 2 ** 63:
                raise ValueError(f"host {h.id!r}: {attr} = {v} is outside the int64 nanosecond range")
        cols[col] = np.array(vals, dtype=np.int64)
    flags = np.array([idle_host_flags(h, None if default_amis is None else default_amis[d])
                      for d, g in enumerate(groups) for h in g], dtype=np.uint32)
    off = np.zeros(len(groups) + 1, np.int64)
    off[1:] = np.cumsum([len(g) for g in groups])
    return IdleHostTable(cols, flags, off, [h.id for h in hosts])


@dataclass
class EstHostTable:
    """evg_est_host_soa + est_host_off: the start-time estimator's hosts of every distro, in query order."""
    kind: np.ndarray          # uint8 EVG_EH_*
    expected_ns: np.ndarray   # int64
    dispatch_ns: np.ndarray   # int64
    est_host_off: np.ndarray  # int64, n_distros + 1

    @property
    def n_hosts(self) -> int:
        return int(self.kind.shape[0])

    @property
    def n_distros(self) -> int:
        return int(self.est_host_off.shape[0]) - 1

    def struct(self) -> L.EstHostSoAStruct:
        n = self.n_hosts
        return L.EstHostSoAStruct(n, *[L.ptr(a) if n else None for a in (self.kind, self.expected_ns, self.dispatch_ns)])


TASK_LOOKUP_ERROR = object()  # a running_tasks value: task.FindOneIdAndExecution returned an error
_EST_KIND = {M.HOST_UNINITIALIZED: L.EVG_EH_UNINITIALIZED, M.HOST_STARTING: L.EVG_EH_STARTING, M.HOST_PROVISIONING: L.EVG_EH_PROVISIONING}


def marshal_estimate_hosts(hosts_by_distro: Sequence[Sequence[M.Host]], running_tasks: Dict[str, object]) -> EstHostTable:
    """The hosts host.Find(ByDistroIDs(d)) returned for each distro, in query order -> the estimator's host table, as
    createSimulatorModel reads them (model/task_start_estimation.go:129-159).  running_tasks[h.running_task] is the
    running task's document (expected_duration, dispatch_time); absent or None: no document, the host is
    EVG_EH_IGNORED; TASK_LOOKUP_ERROR: the distro's rows end before that host."""
    kind, exp, disp, off = [], [], [], [0]
    for hosts in hosts_by_distro:
        for h in hosts:
            k, e, t = _EST_KIND.get(h.status, L.EVG_EH_IGNORED), 0, M.ZERO_TIME
            if h.status == M.HOST_RUNNING:
                k = L.EVG_EH_FREE
                if h.running_task != "":
                    doc = running_tasks.get(h.running_task)
                    if doc is TASK_LOOKUP_ERROR:
                        break
                    if doc is None:
                        k = L.EVG_EH_IGNORED
                    else:
                        k, e, t = L.EVG_EH_RUNNING, doc.expected_duration, doc.dispatch_time
            kind.append(k)
            exp.append(e)
            disp.append(t)
        off.append(len(kind))
    return EstHostTable(np.array(kind, dtype=np.uint8), np.array(exp, dtype=np.int64), np.array(disp, dtype=np.int64),
                        np.array(off, dtype=np.int64))


def queue_info_rows(infos: Sequence[M.DistroQueueInfo]):
    """[DistroQueueInfo] -> (QUEUE_INFO rows, GROUP_INFO rows, group_off, names per distro).
    Later duplicates of a name win, like the map built at allocator.go:243-246."""
    qrows = np.zeros(len(infos), dtype=L.QUEUE_INFO_DTYPE)
    grows, goff, names_all = [], [0], []
    for i, qi in enumerate(infos):
        q = qrows[i]
        q["length"] = qi.length
        q["length_with_dependencies_met"] = qi.length_with_dependencies_met
        q["count_dep_filled_merge_queue_tasks"] = qi.count_dep_filled_merge_queue_tasks
        q["expected_duration"] = qi.expected_duration
        q["max_duration_threshold"] = qi.max_duration_threshold
        q["count_duration_over_threshold"] = qi.count_duration_over_threshold
        q["duration_over_threshold"] = qi.duration_over_threshold
        q["count_wait_over_threshold"] = qi.count_wait_over_threshold
        q["secondary_queue"] = int(qi.secondary_queue)
        by_name = {}
        for g in qi.task_group_infos:
            by_name[g.name] = g
        names = []
        for name, g in by_name.items():
            row = tuple(getattr(g, f) for f in L.GROUP_INFO_FIELDS)
            if name == "":
                q["has_ungrouped"] = 1
                q["ungrouped"] = row
            else:
                names.append(name)
                grows.append(row)
        goff.append(len(grows))
        names_all.append(names)
    return qrows, np.array(grows, dtype=L.GROUP_INFO_DTYPE).reshape(-1), np.array(goff, dtype=np.int64), names_all


# ---------------------------------------------------------------------------
# dependency filter tables (evg_deps_in)
# ---------------------------------------------------------------------------

def _task_state(t: M.Task) -> int:
    st = 0 if t.status == M.TASK_SUCCEEDED else 1 if t.status == M.TASK_FAILED else 2
    return st | (L.EVG_TS_BLOCKED if t.blocked() else 0)


def _want(status: str) -> int:
    if status in (M.TASK_SUCCEEDED, ""):
        return L.EVG_WANT_SUCCESS
    if status == M.TASK_FAILED:
        return L.EVG_WANT_FAILED
    if status == M.ALL_STATUSES:
        return L.EVG_WANT_ANY
    return L.EVG_WANT_OTHER


@dataclass
class DepsTable:
    """evg_deps_in: every direct dependency of every task of the tick (all distros concatenated)."""
    dep_off: np.ndarray
    dep_kind: np.ndarray
    dep_ref: np.ndarray
    dep_want: np.ndarray
    task_state: np.ndarray
    task_pre: np.ndarray
    ext_state: np.ndarray

    @property
    def n_tasks(self) -> int:
        return int(self.task_state.shape[0])

    def struct(self) -> L.DepsInStruct:
        s = L.DepsInStruct()
        s.n_tasks, s.n_deps, s.n_ext = self.n_tasks, int(self.dep_ref.shape[0]), int(self.ext_state.shape[0])
        s.dep_off = L.ptr(self.dep_off)
        for f in ("dep_kind", "dep_ref", "dep_want"):
            setattr(s, f, L.ptr(getattr(self, f)) if s.n_deps else None)
        s.task_state, s.task_pre = L.ptr(self.task_state), L.ptr(self.task_pre)
        s.ext_state = L.ptr(self.ext_state) if s.n_ext else None
        return s


def marshal_dep_finished(batch: Sequence[tuple]) -> np.ndarray:
    """Dependency.FinishedAt of every dependency, in marshal_deps' order (what setDependenciesMetTime reads)."""
    return np.array([d.finished_at for _, tasks in batch for t in tasks for d in t.depends_on], dtype=np.int64)


def marshal_deps(batch: Sequence[tuple], dependency_db: Optional[Dict[str, M.Task]] = None,
                 ext_index: Optional[Dict[str, int]] = None) -> DepsTable:
    """[(Distro, [Task])] -> DepsTable.  A dependency resolves against the distro's own queue first (the
    depCache of scheduler.go:61-64), then against `dependency_db` (the tasks collection), else it is MISSING.
    `ext_index`, when given, is filled with the external id of every task id the table's external rows stand for."""
    dep_off, kind, ref, want, tstate, pre, ext_state = [0], [], [], [], [], [], []
    ext_index = {} if ext_index is None else ext_index
    ext_index.clear()
    db = dependency_db or {}
    base = 0
    for _, tasks in batch:
        index = {t.id: i for i, t in enumerate(tasks)}
        for t in tasks:
            tstate.append(_task_state(t))
            pre.append((L.EVG_TP_OVERRIDE if t.override_dependencies else 0) |
                       (0 if M.is_zero_time(t.dependencies_met_time) else L.EVG_TP_MET_TIME))
            for d in t.depends_on:
                want.append(_want(d.status))
                j = index.get(d.task_id)
                if j is not None:
                    kind.append(L.EVG_DEP_IN_QUEUE); ref.append(base + j)
                elif d.task_id in db:
                    k = ext_index.get(d.task_id)
                    if k is None:
                        k = ext_index[d.task_id] = len(ext_state)
                        ext_state.append(_task_state(db[d.task_id]))
                    kind.append(L.EVG_DEP_EXTERNAL); ref.append(k)
                else:
                    kind.append(L.EVG_DEP_MISSING); ref.append(0)
            dep_off.append(len(ref))
        base += len(tasks)
    return DepsTable(np.array(dep_off, np.int64), np.array(kind, np.uint8), np.array(ref, np.int32),
                     np.array(want, np.uint8), np.array(tstate, np.uint8), np.array(pre, np.uint8),
                     np.array(ext_state, np.uint8))


def _task_pre(t: M.Task) -> int:
    return (L.EVG_TP_OVERRIDE if t.override_dependencies else 0) | (0 if M.is_zero_time(t.dependencies_met_time) else L.EVG_TP_MET_TIME)


def deps_verdicts(deps: DepsTable, dep_finished: Optional[np.ndarray], now: int):
    """Task.DependenciesMet and the DependenciesMetTime stamp of every row of an evg_deps_in table, in numpy: what
    evg_upload_with_deps computes on the device (k_deps_met) -> (met uint8, stamp int64, EVG_TIME_ZERO = none)."""
    T = deps.n_tasks
    E = int(deps.dep_ref.shape[0])
    deg = np.diff(deps.dep_off)
    owner = np.repeat(np.arange(T, dtype=np.int64), deg)
    kind, ref = deps.dep_kind, deps.dep_ref.astype(np.int64)
    st = np.full(E, 2, dtype=np.uint8)
    inq, ext = kind == L.EVG_DEP_IN_QUEUE, kind == L.EVG_DEP_EXTERNAL
    st[inq] = deps.task_state[ref[inq]]
    st[ext] = deps.ext_state[ref[ext]]
    status = st & 3
    want = deps.dep_want
    ok = np.where(want == L.EVG_WANT_SUCCESS, status == 0,
                  np.where(want == L.EVG_WANT_FAILED, status == 1,
                           np.where(want == L.EVG_WANT_ANY, (status < 2) | ((st & L.EVG_TS_BLOCKED) != 0), False)))
    ok &= inq | ext
    row_ok = np.bincount(owner[~ok], minlength=T) == 0
    shortcut = (deps.task_pre & (L.EVG_TP_OVERRIDE | L.EVG_TP_MET_TIME)) != 0
    met = (row_ok | shortcut).astype(np.uint8)
    best = np.full(T, L.EVG_TIME_ZERO, dtype=np.int64)
    if dep_finished is not None and E:
        f = np.asarray(dep_finished, dtype=np.int64)
        live = (f != L.EVG_TIME_ZERO) & (f != 0)
        np.maximum.at(best, owner[live], f[live])
    fresh = row_ok & ~shortcut & (deg > 0)
    stamp = np.where(fresh, np.where(best == L.EVG_TIME_ZERO, np.int64(now), best), np.int64(L.EVG_TIME_ZERO)).astype(np.int64)
    return met, stamp


@dataclass
class DepsEdit:
    """evg_deps_edit: what changed in a resident tick's dependency table between two ticks (include/evg_sched.h)."""
    depart_ext: np.ndarray                          # int32 [n_remove]: external id a removed row becomes, -1 = none
    ext_state: np.ndarray                           # uint8 [n_ext]: the new external table, EVG_TS_*
    insert: DepsTable                               # the inserted rows' own entries (its ext_state is not read)
    add_row: np.ndarray                             # int64, ascending new global row of a surviving task
    add_kind: np.ndarray                            # uint8 EVG_DEP_*
    add_ref: np.ndarray                             # int32: new global row or new external id
    add_want: np.ndarray                            # uint8 EVG_WANT_*
    set_row: np.ndarray                             # int64: surviving tasks whose task_state / task_pre change
    set_state: np.ndarray                           # uint8
    set_pre: np.ndarray                             # uint8
    depart_finished: Optional[np.ndarray] = None    # int64 [n_remove]: FinishedAt of the entries that pointed there
    ext_finished: Optional[np.ndarray] = None       # int64 [n_ext]: FinishedAt of every entry on that id
    insert_finished: Optional[np.ndarray] = None    # int64 per inserted entry
    add_finished: Optional[np.ndarray] = None       # int64 per added entry

    def normalize(self) -> "DepsEdit":
        for f, dt in (("depart_ext", np.int32), ("ext_state", np.uint8), ("add_row", np.int64), ("add_kind", np.uint8),
                      ("add_ref", np.int32), ("add_want", np.uint8), ("set_row", np.int64), ("set_state", np.uint8),
                      ("set_pre", np.uint8)):
            setattr(self, f, np.ascontiguousarray(getattr(self, f), dtype=dt))
        for f in ("depart_finished", "ext_finished", "insert_finished", "add_finished"):
            if getattr(self, f) is not None:
                setattr(self, f, np.ascontiguousarray(getattr(self, f), dtype=np.int64))
        return self

    def struct(self):
        """-> (DepsEditStruct, the inserted rows' struct it points to: keep both alive for the call)."""
        self.normalize()
        ins = self.insert.struct()
        p = lambda a: L.ptr(a) if a is not None and a.shape[0] else None  # noqa: E731
        s = L.DepsEditStruct(p(self.depart_ext), p(self.depart_finished), int(self.ext_state.shape[0]), p(self.ext_state),
                             p(self.ext_finished), C.pointer(ins), p(self.insert_finished), int(self.add_row.shape[0]),
                             p(self.add_row), p(self.add_kind), p(self.add_ref), p(self.add_want), p(self.add_finished),
                             int(self.set_row.shape[0]), p(self.set_row), p(self.set_state), p(self.set_pre))
        return s, ins

    def nbytes(self) -> int:
        arrays = [getattr(self, f) for f in ("depart_ext", "ext_state", "add_row", "add_kind", "add_ref", "add_want", "set_row",
                                            "set_state", "set_pre", "depart_finished", "ext_finished", "insert_finished",
                                            "add_finished")]
        ins = self.insert
        arrays += [ins.dep_off, ins.dep_kind, ins.dep_ref, ins.dep_want, ins.task_state, ins.task_pre]
        return sum(a.nbytes for a in arrays if a is not None)


def apply_deps_edit(deps: DepsTable, task_off: np.ndarray, edit: TaskEdit, x: DepsEdit,
                    dep_finished: Optional[np.ndarray] = None, stamp: Optional[np.ndarray] = None):
    """The composed dependency table of evg_edit_tasks_with_deps, in numpy -> (DepsTable, FinishedAt per entry).
    `deps` / `dep_finished` are the previous tick's table over the previous distro offsets `task_off`, `stamp` its last
    evaluation's stamps (written back into task_pre as EVG_TP_MET_TIME); of `edit` only the removed rows and the
    inserted counts are read.  Raises ValueError where the device reports EVG_ERR_INVALID."""
    edit.normalize()
    x.normalize()
    T0, E0 = deps.n_tasks, int(deps.dep_ref.shape[0])
    Xn = int(x.ext_state.shape[0])
    fin0 = np.full(E0, L.EVG_TIME_ZERO, np.int64) if dep_finished is None or E0 == 0 else np.asarray(dep_finished, np.int64)
    D = int(task_off.shape[0]) - 1
    distro_of = np.repeat(np.arange(D, dtype=np.int64), np.diff(task_off))
    keep = np.ones(T0, dtype=bool)
    keep[edit.remove_rows] = False
    pos = np.cumsum(keep) - keep                       # survivors before each previous row
    n_ins = np.diff(edit.insert_off)
    ins_before = np.concatenate([[0], np.cumsum(n_ins)]).astype(np.int64)
    n_surv = np.bincount(distro_of[keep], minlength=D).astype(np.int64)
    new_off = np.concatenate([[0], np.cumsum(n_surv + n_ins)]).astype(np.int64)
    Tn = int(new_off[-1])
    new_row = np.where(keep, pos + ins_before[distro_of], -1)
    ins_d = np.repeat(np.arange(D, dtype=np.int64), n_ins)
    ins_new = new_off[ins_d] + n_surv[ins_d] + np.arange(ins_d.shape[0]) - edit.insert_off[ins_d]
    # the survivors' previous entries, rewritten
    own = np.repeat(np.arange(T0, dtype=np.int64), np.diff(deps.dep_off))
    live = keep[own]
    kind, ref = deps.dep_kind[live].copy(), deps.dep_ref[live].astype(np.int64)
    want, fin = deps.dep_want[live].copy(), fin0[live].copy()
    inq = kind == L.EVG_DEP_IN_QUEUE
    if np.any(inq & ((ref < 0) | (ref >= T0))):
        raise ValueError("an in-queue ref of the previous dependency table is outside it")
    if np.any((kind == L.EVG_DEP_EXTERNAL) & ((ref < 0) | (ref >= Xn))):
        raise ValueError("a surviving task's external ref is outside the new external table")
    gone = inq.copy()
    gone[inq] = ~keep[ref[inq]]
    stay = inq & ~gone
    ref[stay] = new_row[ref[stay]]
    k = ref[gone] - pos[ref[gone]]                    # index in remove_rows
    ref[gone] = x.depart_ext[k]
    kind[gone] = L.EVG_DEP_EXTERNAL
    if np.any(ref[gone] < 0):
        raise ValueError("a surviving task depends on a removed row whose depart_ext is -1")
    if x.depart_finished is not None:
        fin[gone] = x.depart_finished[k]
    ins = x.insert
    EI = int(ins.dep_ref.shape[0])
    zero = lambda n: np.full(n, L.EVG_TIME_ZERO, np.int64)  # noqa: E731
    owner = np.concatenate([new_row[own[live]], x.add_row, np.repeat(ins_new, np.diff(ins.dep_off))]).astype(np.int64)
    kind = np.concatenate([kind, x.add_kind, ins.dep_kind]).astype(np.uint8)
    ref = np.concatenate([ref, x.add_ref, ins.dep_ref]).astype(np.int32)
    want = np.concatenate([want, x.add_want, ins.dep_want]).astype(np.uint8)
    fin = np.concatenate([fin, zero(x.add_row.shape[0]) if x.add_finished is None else x.add_finished,
                          zero(EI) if x.insert_finished is None else x.insert_finished]).astype(np.int64)
    if x.ext_finished is not None:
        e = kind == L.EVG_DEP_EXTERNAL
        fin[e] = x.ext_finished[ref[e]]
    o = np.argsort(owner, kind="stable")
    dep_off = np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=Tn))]).astype(np.int64)
    state = np.zeros(Tn, np.uint8)
    pre = np.zeros(Tn, np.uint8)
    st = np.full(T0, L.EVG_TIME_ZERO, np.int64) if stamp is None else np.asarray(stamp, np.int64)
    sv = np.nonzero(keep)[0]
    state[new_row[sv]] = deps.task_state[sv]
    pre[new_row[sv]] = deps.task_pre[sv] | np.where((st[sv] != L.EVG_TIME_ZERO) & (st[sv] != 0), L.EVG_TP_MET_TIME, 0).astype(np.uint8)
    state[ins_new] = ins.task_state
    pre[ins_new] = ins.task_pre
    state[x.set_row] = x.set_state
    pre[x.set_row] = x.set_pre
    return DepsTable(dep_off, kind[o], ref[o], want[o], state, pre, x.ext_state.copy()), fin[o]


class DepsShim:
    """What a shim keeps to send a tick's dependency changes as an evg_deps_edit instead of the whole table: the
    external id of every task id the resident table's external rows stand for (ids only grow until the next full
    upload), and per queued task its entries (dependency id, wanted status, FinishedAt) and its task_state / task_pre
    as the device holds them after the last tick's stamps were written back."""

    def __init__(self, dependency_db: Optional[Dict[str, M.Task]] = None):
        self.db = dependency_db or {}
        self.ext: Dict[str, int] = {}
        self.entries: Dict[str, list] = {}
        self.rows: Dict[str, tuple] = {}

    def upload(self, batch: Sequence[tuple]):
        """A full upload of `batch`: -> (DepsTable, FinishedAt per entry), and the id map starts over from it."""
        pairs = [(b[0], b[1]) for b in batch]
        return marshal_deps(pairs, self.db, self.ext), marshal_dep_finished(pairs)

    def remember(self, batch: Sequence[tuple]) -> None:
        """After the tick's stamps were written back onto the Task objects."""
        self.entries = {}
        for _, ts in batch:
            q = {t.id for t in ts}
            for t in ts:  # the last element: the entry resolved to MISSING, which an edit keeps
                self.entries[t.id] = [(d.task_id, d.status, d.finished_at, d.task_id not in q and d.task_id not in self.db)
                                      for d in t.depends_on]
        self.rows = {t.id: (_task_state(t), _task_pre(t)) for _, ts in batch for t in ts}

    def _ext_id(self, task_id: str) -> int:
        k = self.ext.get(task_id)
        if k is None:
            k = self.ext[task_id] = len(self.ext)
        return k

    def edit(self, prev_ids: Sequence[Sequence[str]], batch: Sequence[tuple], remove_rows: np.ndarray) -> Optional[DepsEdit]:
        """The DepsEdit from the remembered tick (`prev_ids`: its task ids per distro in resident order) to `batch` in
        canonical order (survivors in their previous order, then arrivals) with `remove_rows` (ascending previous rows)
        gone.  Departures become external ids; their FinishedAt comes from the survivors' entries on them.  None when
        an edit cannot express the change: a survivor whose entries are not its previous ones plus new ones at the end,
        a kept entry whose FinishedAt or resolution (queue, collection, missing) changed otherwise."""
        flat_prev = [i for ids in prev_ids for i in ids]
        gone_ids = [flat_prev[int(r)] for r in remove_rows]
        gone_k = {i: k for k, i in enumerate(gone_ids)}
        depart_fin = np.full(len(gone_ids), L.EVG_TIME_ZERO, np.int64)
        depart_seen = np.zeros(len(gone_ids), dtype=bool)
        base = 0
        queue_of = []
        for _, ts in batch:
            queue_of.append({t.id: base + j for j, t in enumerate(ts)})
            base += len(ts)
        add = ([], [], [], [], [])
        sets = ([], [], [])
        ins_off, ikind, iref, iwant, ifin, istate, ipre = [0], [], [], [], [], [], []

        def resolve(dep_id: str, q: dict):
            j = q.get(dep_id)
            if j is not None:
                return L.EVG_DEP_IN_QUEUE, j
            if dep_id in self.db:
                return L.EVG_DEP_EXTERNAL, self._ext_id(dep_id)
            return L.EVG_DEP_MISSING, 0

        for d, (_, ts) in enumerate(batch):
            q = queue_of[d]
            prev_q = set(prev_ids[d])
            n_prev = len(prev_q) - sum(1 for i in prev_ids[d] if i in gone_k)
            for j, t in enumerate(ts):
                row = q[t.id]
                cur = [(x.task_id, x.status, x.finished_at) for x in t.depends_on]
                if j >= n_prev:  # an arrival brings its own entries
                    for dep_id, status, f in cur:
                        kd, rf = resolve(dep_id, q)
                        ikind.append(kd); iref.append(rf); iwant.append(_want(status)); ifin.append(f)
                    ins_off.append(len(iref))
                    istate.append(_task_state(t)); ipre.append(_task_pre(t))
                    continue
                old = self.entries.get(t.id)
                if old is None or len(cur) < len(old):
                    return None
                for (dep_id, status, f), (o_id, o_status, o_f, o_missing) in zip(cur, old):
                    if (dep_id, status) != (o_id, o_status):
                        return None
                    k = gone_k.get(dep_id)
                    if k is not None:  # departs now: every entry on it must agree on its FinishedAt
                        if depart_seen[k] and depart_fin[k] != f:
                            return None
                        depart_seen[k], depart_fin[k] = True, f
                        continue
                    if f != o_f:
                        return None
                    if (dep_id in prev_q) != (dep_id in q) or (o_missing and dep_id in self.db):
                        return None  # the dependency joined the queue, or a missing one turned up
                for dep_id, status, f in cur[len(old):]:
                    kd, rf = resolve(dep_id, q)
                    add[0].append(row); add[1].append(kd); add[2].append(rf); add[3].append(_want(status)); add[4].append(f)
                now = (_task_state(t), _task_pre(t))
                if now != self.rows.get(t.id):
                    sets[0].append(row); sets[1].append(now[0]); sets[2].append(now[1])
        depart_ext = np.array([self._ext_id(i) if depart_seen[k] else -1 for k, i in enumerate(gone_ids)], np.int32)
        ext_state = np.full(len(self.ext), 2, np.uint8)  # an id no longer in the collection satisfies nothing, as MISSING
        for i, k in self.ext.items():
            if i in self.db:
                ext_state[k] = _task_state(self.db[i])
        insert = DepsTable(np.array(ins_off, np.int64), np.array(ikind, np.uint8), np.array(iref, np.int32),
                           np.array(iwant, np.uint8), np.array(istate, np.uint8), np.array(ipre, np.uint8), np.zeros(0, np.uint8))
        return DepsEdit(depart_ext, ext_state, insert, np.array(add[0], np.int64), np.array(add[1], np.uint8),
                        np.array(add[2], np.int32), np.array(add[3], np.uint8), np.array(sets[0], np.int64),
                        np.array(sets[1], np.uint8), np.array(sets[2], np.uint8), depart_finished=depart_fin,
                        insert_finished=np.array(ifin, np.int64), add_finished=np.array(add[4], np.int64)).normalize()


@dataclass
class RunnableTable:
    """evg_runnable_in: every candidate task of every distro, plus the project-ref cache and the per-distro rules."""
    task_off: np.ndarray
    sched: np.ndarray
    project: np.ndarray
    project_flags: np.ndarray
    valid_off: np.ndarray
    valid_idx: np.ndarray
    finder: np.ndarray
    deps: Optional[DepsTable]
    pipe: Optional["PipelineTable"] = None  # what the pipeline finder reads besides (evg_pipeline_in); None: no pipeline distro

    @property
    def n_tasks(self) -> int:
        return int(self.sched.shape[0])

    @property
    def n_distros(self) -> int:
        return int(self.finder.shape[0])

    def struct(self):
        """-> (RunnableInStruct, keepalive): the nested evg_deps_in must outlive the call."""
        s = L.RunnableInStruct()
        s.n_tasks, s.n_distros, s.n_projects = self.n_tasks, self.n_distros, int(self.project_flags.shape[0])
        s.task_off, s.valid_off, s.finder = L.ptr(self.task_off), L.ptr(self.valid_off), L.ptr(self.finder)
        s.sched = L.ptr(self.sched) if s.n_tasks else None
        s.project = L.ptr(self.project) if s.n_tasks else None
        s.project_flags = L.ptr(self.project_flags) if s.n_projects else None
        s.valid_idx = L.ptr(self.valid_idx) if self.valid_idx.shape[0] else None
        keep = None
        if self.deps is not None:
            keep = self.deps.struct()
            s.deps = C.pointer(keep)
        return s, keep


def sched_bits(t: M.Task) -> int:
    """The EVG_SQ_* byte of one task: the fields of schedulableHostTasksQuery (model/task/db.go:671-689) and the
    requester classes ProjectCanDispatchTask looks at."""
    b = 0
    if t.activated:
        b |= L.EVG_SQ_ACTIVATED
    if t.status == M.TASK_UNDISPATCHED:
        b |= L.EVG_SQ_UNDISPATCHED
    if t.priority > M.DISABLED_TASK_PRIORITY:
        b |= L.EVG_SQ_PRIORITY_OK
    if t.execution_platform in ("", "host"):
        b |= L.EVG_SQ_HOST_PLATFORM
    if t.unattainable_dependency:
        b |= L.EVG_SQ_UNATTAINABLE
    if t.override_dependencies:
        b |= L.EVG_SQ_OVERRIDE_DEPS
    if t.requester == M.GITHUB_PR_REQUESTER:
        b |= L.EVG_SQ_GITHUB_PR
    if M.is_patch_requester(t.requester):
        b |= L.EVG_SQ_PATCH_REQUEST
    return b


def project_bits(p: M.ProjectRef) -> int:
    return ((L.EVG_PF_ENABLED if p.enabled else 0) | (L.EVG_PF_HIDDEN if p.hidden else 0) |
            (L.EVG_PF_DISPATCHING_DISABLED if p.dispatching_disabled else 0) |
            (L.EVG_PF_PATCHING_DISABLED if p.patching_disabled else 0))


@dataclass
class PipelineTable:
    """evg_pipeline_in: interned status strings of the candidates, of their dependency entries and of the external
    dependency documents, the "has an unattainable depends_on entry" bits, and the raw project_ref bits."""
    n_status: int
    dep_status: np.ndarray         # int32 per evg_deps_in entry: Dependency.Status
    task_status: np.ndarray        # int32 per candidate: Task.Status
    ext_status: np.ndarray         # int32 per external row
    task_unattainable: np.ndarray  # uint8 per candidate
    ext_unattainable: np.ndarray   # uint8 per external row
    project_raw: np.ndarray        # uint8 EVG_PR_* per project row

    def struct(self) -> L.PipelineInStruct:
        s = L.PipelineInStruct()
        s.n_status = int(self.n_status)
        nz = lambda a: L.ptr(a) if a.shape[0] else None  # noqa: E731
        s.dep_status, s.task_status, s.ext_status = nz(self.dep_status), nz(self.task_status), nz(self.ext_status)
        s.task_unattainable, s.ext_unattainable = nz(self.task_unattainable), nz(self.ext_unattainable)
        s.project_raw = nz(self.project_raw)
        return s


def project_raw_bits(p: M.ProjectRef) -> int:
    """EVG_PR_* of the project_ref DOCUMENT as stored (model/project_ref.go:52-59): enabled is bool,omitempty (stored only
    when true), dispatching_disabled and patching_disabled are *bool,omitempty (stored only when set)."""
    return ((L.EVG_PR_ENABLED if p.enabled else 0) | (L.EVG_PR_DISPATCHING_DISABLED if p.dispatching_disabled is True else 0) |
            (L.EVG_PR_PATCHING_FALSE if p.patching_disabled is False else 0))


def marshal_pipeline(batch: Sequence[tuple], project_refs: Sequence[M.ProjectRef],
                     dependency_db: Optional[Dict[str, M.Task]] = None) -> PipelineTable:
    """The evg_pipeline_in of a batch, in marshal_deps' order (its entries and external rows resolve the same way: the
    distro's own candidates first, then `dependency_db`).  Status strings are interned with the reserved ids first."""
    ids: Dict[str, int] = {M.TASK_SUCCEEDED: L.EVG_STATUS_SUCCESS, M.TASK_FAILED: L.EVG_STATUS_FAILED,
                           M.ALL_STATUSES: L.EVG_STATUS_ANY}
    intern = lambda x: ids.setdefault(x, len(ids))  # noqa: E731
    unatt = lambda t: int(any(d.unattainable for d in t.depends_on))  # noqa: E731
    db = dependency_db or {}
    dep_status, task_status, task_un, ext_status, ext_un = [], [], [], [], []
    ext_seen = set()
    for _, tasks in batch:
        index = {t.id for t in tasks}
        for t in tasks:
            task_status.append(intern(t.status))
            task_un.append(unatt(t))
            for d in t.depends_on:
                dep_status.append(intern(d.status))
                if d.task_id not in index and d.task_id in db and d.task_id not in ext_seen:
                    ext_seen.add(d.task_id)
                    ext_status.append(intern(db[d.task_id].status))
                    ext_un.append(unatt(db[d.task_id]))
    return PipelineTable(len(ids), np.array(dep_status, np.int32), np.array(task_status, np.int32),
                         np.array(ext_status, np.int32), np.array(task_un, np.uint8), np.array(ext_un, np.uint8),
                         np.array([project_raw_bits(p) for p in project_refs], np.uint8))


def marshal_runnable(batch: Sequence[tuple], project_refs: Sequence[M.ProjectRef], finder: str = "legacy",
                     dependency_db: Optional[Dict[str, M.Task]] = None) -> RunnableTable:
    """[(Distro, [candidate Task])] + the project-ref cache (getProjectRefCache, task_finder.go:46) -> RunnableTable.
    `finder`: "legacy" (LegacyFindRunnableTasks), "alternate" (AlternateTaskFinder / ParallelTaskFinder) or "pipeline"
    (RunnableTasksPipeline: `project_refs` are then the raw project_ref documents, and the table carries a
    PipelineTable)."""
    prow = {p.id: i for i, p in enumerate(project_refs)}
    flavour = {"legacy": L.EVG_FINDER_LEGACY, "alternate": L.EVG_FINDER_ALTERNATE, "parallel": L.EVG_FINDER_ALTERNATE,
               "pipeline": L.EVG_FINDER_PIPELINE}[finder]
    no_deps = L.EVG_FINDER_PIPELINE_NO_DEPS if finder == "pipeline" else L.EVG_FINDER_NO_DEPS
    task_off, valid_off, valid_idx, fnd, sched, proj = [0], [0], [], [], [], []
    for d, tasks in batch:
        for t in tasks:
            sched.append(sched_bits(t))
            proj.append(prow.get(t.project, -1))
        task_off.append(len(sched))
        valid_idx.extend(prow.get(name, -1) for name in d.valid_projects)
        valid_off.append(len(valid_idx))
        fnd.append(no_deps if d.dispatcher_settings.version == M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES else flavour)
    deps = marshal_deps(batch, dependency_db) if any(f != no_deps for f in fnd) else None
    pipe = marshal_pipeline(batch, project_refs, dependency_db) if finder == "pipeline" else None
    return RunnableTable(np.array(task_off, np.int64), np.array(sched, np.uint8), np.array(proj, np.int32),
                         np.array([project_bits(p) for p in project_refs], np.uint8), np.array(valid_off, np.int64),
                         np.array(valid_idx, np.int32), np.array(fnd, np.uint8), deps, pipe)


# ---------------------------------------------------------------------------
# alias queues (evg_alias_in)
# ---------------------------------------------------------------------------

SQ_BASE = L.EVG_SQ_ACTIVATED | L.EVG_SQ_UNDISPATCHED | L.EVG_SQ_PRIORITY_OK | L.EVG_SQ_HOST_PLATFORM


@dataclass
class AliasTable:
    """evg_alias_in: the tick's schedulable tasks, each once, and what decides the alias queues they join.
    tasks.group_id / version_id are table-global; tasks.dep_idx are row indices; `deps` covers the same rows."""
    tasks: TaskSoA
    group_max_hosts: np.ndarray   # per global group
    n_versions: int
    sched: np.ndarray             # uint8 EVG_SQ_*
    task_group_max_hosts: np.ndarray
    primary: np.ndarray           # distro index of Task.DistroId, -1
    secondary_off: np.ndarray     # CSR of Task.SecondaryDistros as name indices (-1: a name no distro has)
    secondary_idx: np.ndarray
    dest_off: np.ndarray          # CSR over names: the distros e with the name in {e} U e.Aliases
    dest_idx: np.ndarray
    deps: DepsTable
    dep_finished: np.ndarray

    @property
    def n_tasks(self) -> int:
        return self.tasks.n_tasks

    @property
    def n_names(self) -> int:
        return int(self.dest_off.shape[0]) - 1

    def normalize(self) -> "AliasTable":
        self.tasks.normalize()
        for f, dt in (("group_max_hosts", np.int32), ("sched", np.uint8), ("task_group_max_hosts", np.int32), ("primary", np.int32),
                      ("secondary_off", np.int64), ("secondary_idx", np.int32), ("dest_off", np.int64), ("dest_idx", np.int32),
                      ("dep_finished", np.int64)):
            setattr(self, f, np.ascontiguousarray(getattr(self, f), dtype=dt))
        return self

    def struct(self):
        """-> (AliasInStruct, keepalive)."""
        s = L.AliasInStruct()
        s.tasks = self.tasks.struct()
        s.n_groups, s.n_versions = int(self.group_max_hosts.shape[0]), int(self.n_versions)
        nz = lambda a: L.ptr(a) if a.shape[0] else None  # noqa: E731
        s.group_max_hosts, s.sched, s.task_group_max_hosts, s.primary = (nz(self.group_max_hosts), nz(self.sched),
                                                                         nz(self.task_group_max_hosts), nz(self.primary))
        s.secondary_off, s.secondary_idx = L.ptr(self.secondary_off), nz(self.secondary_idx)
        s.n_names = self.n_names
        s.dest_off, s.dest_idx = L.ptr(self.dest_off), nz(self.dest_idx)
        keep = self.deps.struct()
        s.deps = C.pointer(keep)
        s.dep_finished_ns = nz(self.dep_finished)
        return s, keep


def alias_name_table(distros: Sequence[M.Distro]):
    """(name -> index, dest_off, dest_idx): every name some distro's applicable set {e} U e.Aliases holds
    (FindApplicableDistroIDs, model/distro/aliases.go:14-27), and per name the distros whose set holds it."""
    dests: Dict[str, List[int]] = {}
    for i, d in enumerate(distros):
        for name in [d.id] + list(d.aliases):
            lst = dests.setdefault(name, [])
            if not lst or lst[-1] != i:
                lst.append(i)
    index = {name: k for k, name in enumerate(dests)}
    dest_off = np.zeros(len(dests) + 1, np.int64)
    if dests:
        np.cumsum([len(v) for v in dests.values()], out=dest_off[1:])
    dest_idx = np.array([i for v in dests.values() for i in v], np.int32)
    return index, dest_off, dest_idx


def marshal_aliases(distros: Sequence[M.Distro], tasks: Sequence[M.Task], now: int,
                    dependency_db: Optional[Dict[str, M.Task]] = None, duration_history: Optional[dict] = None):
    """The alias side of a tick: every distro and the tick's schedulable tasks, each task ONCE -> (AliasTable, planner cfg
    rows of the distros, MarshalledDistro of the whole table: global group names and versions).  Task groups and
    versions are interned once over the table, dependencies resolve against the table first, then `dependency_db`."""
    whole = M.Distro(id="")
    soa, table, keys = marshal_tasks([(whole, list(tasks))], now, dependency_db, duration_history)
    soa.flags &= np.uint32(~L.EVG_TF_OTHER_DISTRO & 0xFFFFFFFF)  # set per queue on the device
    index, dest_off, dest_idx = alias_name_table(distros)
    where = {d.id: i for i, d in enumerate(distros)}
    sec_off = np.zeros(len(tasks) + 1, np.int64)
    if len(tasks):
        np.cumsum([len(t.secondary_distros) for t in tasks], out=sec_off[1:])
    pairs = [(whole, list(tasks))]
    at = AliasTable(soa, table.group_max_hosts, int(table.cfg["n_versions"][0]),
                    np.array([sched_bits(t) for t in tasks], np.uint8), np.array([t.task_group_max_hosts for t in tasks], np.int32),
                    np.array([where.get(t.distro_id, -1) for t in tasks], np.int32), sec_off,
                    np.array([index.get(n, -1) for t in tasks for n in t.secondary_distros], np.int32), dest_off, dest_idx,
                    marshal_deps(pairs, dependency_db), marshal_dep_finished(pairs)).normalize()
    cfg = np.array([planner_cfg_row(d, d.dispatcher_settings.version == M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES, 0)
                    for d in distros], dtype=L.DISTRO_CFG_DTYPE)
    return at, cfg, keys[0]


def alias_queues(at: AliasTable, n_distros: int) -> List[np.ndarray]:
    """FindHostSchedulableForAlias restated over an AliasTable: per distro, the source rows of its alias queue in
    ascending order (a row once, however many of its names reach the distro)."""
    ok = ((at.sched & SQ_BASE) == SQ_BASE) & (((at.sched & L.EVG_SQ_UNATTAINABLE) == 0) | ((at.sched & L.EVG_SQ_OVERRIDE_DEPS) != 0))
    ok &= at.task_group_max_hosts != 1
    queues: List[set] = [set() for _ in range(n_distros)]
    for t in np.nonzero(ok)[0]:
        for name in at.secondary_idx[at.secondary_off[t]:at.secondary_off[t + 1]]:
            if name >= 0:
                for e in at.dest_idx[at.dest_off[name]:at.dest_off[name + 1]]:
                    queues[int(e)].add(int(t))
    return [np.array(sorted(q), dtype=np.int64) for q in queues]


def compose_aliases(at: AliasTable, cfg: np.ndarray):
    """The alias tick as a fresh evg_upload_with_deps would take it, built on the host (the route evg_plan_aliases
    replaces): (TaskSoA, DistroTable, DepsTable, dep_finished, source_row, group_source).  Each queue lists its rows in
    ascending source row with group and version ids renumbered in first-appearance order and its in-queue edges
    re-indexed; the dependency table refers to every other task as an external one (its state is the task's own)."""
    D = int(cfg.shape[0])
    queues = alias_queues(at, D)
    t = at.tasks
    rows = np.concatenate(queues) if D else np.zeros(0, np.int64)
    cols = {name: getattr(t, name)[rows].copy() for name, _ in TaskSoA.COLUMNS}
    task_off, group_off, gmax, gsrc, nver = [0], [0], [], [], []
    dep_off, dep_idx = [0], []
    k = 0
    for e, q in enumerate(queues):
        place = {int(u): i for i, u in enumerate(q)}
        groups: Dict[int, int] = {}
        versions: Dict[int, int] = {}
        for u in q:
            g = int(t.group_id[u])
            if g >= 0:
                if g not in groups:
                    groups[g] = len(groups)
                    gmax.append(int(at.group_max_hosts[g]))
                    gsrc.append(g)
                cols["group_id"][k] = groups[g]
            v = int(t.version_id[u])
            cols["version_id"][k] = versions.setdefault(v, len(versions))
            fl = int(t.flags[u]) & ~L.EVG_TF_OTHER_DISTRO
            cols["flags"][k] = fl | (L.EVG_TF_OTHER_DISTRO if int(at.primary[u]) != e else 0)
            if t.n_edges:
                for x in t.dep_idx[t.dep_off[u]:t.dep_off[u + 1]]:
                    if int(x) in place:
                        dep_idx.append(place[int(x)])
            dep_off.append(len(dep_idx))
            k += 1
        task_off.append(k)
        group_off.append(len(gmax))
        nver.append(len(versions))
    c = cfg.copy()
    c["n_versions"] = nver
    soa = TaskSoA(**cols, dep_off=np.array(dep_off, np.int64), dep_idx=np.array(dep_idx, np.int32)).normalize()
    table = DistroTable(np.array(task_off, np.int64), np.array(group_off, np.int64), c, np.array(gmax, np.int32)).normalize()
    d = at.deps
    T = at.n_tasks
    kind = d.dep_kind.copy()
    ref = np.where(kind == L.EVG_DEP_IN_QUEUE, d.dep_ref, np.where(kind == L.EVG_DEP_EXTERNAL, d.dep_ref + T, d.dep_ref)).astype(np.int32)
    kind[kind == L.EVG_DEP_IN_QUEUE] = L.EVG_DEP_EXTERNAL
    lens = (d.dep_off[1:] - d.dep_off[:-1])[rows] if T else np.zeros(0, np.int64)
    take = np.concatenate([np.arange(d.dep_off[u], d.dep_off[u + 1]) for u in rows]).astype(np.int64) if lens.sum() else np.zeros(0, np.int64)
    deps = DepsTable(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), kind[take], ref[take], d.dep_want[take],
                     d.task_state[rows], d.task_pre[rows], np.concatenate([d.task_state, d.ext_state]).astype(np.uint8))
    fin = at.dep_finished[take] if at.dep_finished.shape[0] else np.zeros(0, np.int64)
    return soa, table, deps, fin, rows.astype(np.int32), np.array(gsrc, np.int32)


@dataclass
class DurationRows:
    """evg_duration_rows: finished tasks, the interned group-by key of each, and the aggregation window."""
    key: np.ndarray
    time_taken_ns: np.ndarray
    start_ns: np.ndarray
    finish_ns: np.ndarray
    flags: np.ndarray
    n_keys: int
    window_start_ns: int
    window_end_ns: int

    @property
    def n_rows(self) -> int:
        return int(self.key.shape[0])

    def struct(self) -> L.DurationRowsStruct:
        s = L.DurationRowsStruct()
        s.n_rows, s.n_keys, s._reserved = self.n_rows, int(self.n_keys), 0
        for f in ("key", "time_taken_ns", "start_ns", "finish_ns", "flags"):
            setattr(s, f, L.ptr(getattr(self, f)) if s.n_rows else None)
        s.window_start_ns, s.window_end_ns = int(self.window_start_ns), int(self.window_end_ns)
        return s


def marshal_durations(tasks: Sequence[M.Task], window_start: int, window_end: int):
    """Finished tasks -> (DurationRows, keys): keys[i] = (project, build_variant, display_name) of key row i, in
    first-appearance order.  The $match of expected_duration.go:37-55 is evaluated on the device from the flags
    and the two timestamps; here a row only says what the task document says."""
    index: Dict[tuple, int] = {}
    key, taken, start, finish, flags = [], [], [], [], []
    for t in tasks:
        k = (t.project, t.build_variant, t.display_name)
        key.append(index.setdefault(k, len(index)))
        taken.append(t.time_taken); start.append(t.start_time); finish.append(t.finish_time)
        flags.append((L.EVG_DR_COMPLETED if t.status in M.TASK_COMPLETED_STATUSES else 0) |
                     (L.EVG_DR_TIMED_OUT if t.timed_out else 0))
    rows = DurationRows(np.array(key, np.int32), np.array(taken, np.int64), np.array(start, np.int64),
                        np.array(finish, np.int64), np.array(flags, np.uint8), len(index), window_start, window_end)
    return rows, list(index)


@dataclass
class DurationHistory:
    """The history half of evg_duration_in: finished tasks whose keys are numbered pair-major -- the keys of
    (project, build variant) pair p are pair_key_off[p] .. pair_key_off[p+1] -- and the key code of a task."""
    rows: DurationRows
    pair_key_off: np.ndarray
    keys: List[tuple]          # (project, build_variant, display_name) of each key
    pairs: Dict[tuple, int]    # (project, build_variant) -> pair index
    index: Dict[tuple, int]    # (project, build_variant, display_name) -> key

    @property
    def n_pairs(self) -> int:
        return int(self.pair_key_off.shape[0]) - 1

    def code(self, project: str, build_variant: str, display_name: str) -> int:
        """The evg_duration_cache.key of a task: its key; EVG_DK_PAIR(p) for DisplayName "" (the window query then has
        no name filter, expected_duration.go:54-56); EVG_DK_NONE when no finished task has it."""
        if display_name == "":
            p = self.pairs.get((project, build_variant))
            return L.EVG_DK_NONE if p is None else L.EVG_DK_PAIR(p)
        return self.index.get((project, build_variant, display_name), L.EVG_DK_NONE)

    def __call__(self, t: M.Task) -> int:
        return self.code(t.project, t.build_variant, t.display_name)


def marshal_duration_history(finished: Sequence[M.Task], tasks: Sequence[M.Task], now: int):
    """Finished tasks -> (DurationHistory, key code of each of `tasks`).  The window is the reference's
    (now - 1 week, now] (task.go:3543-3544).  Pairs are numbered in first-appearance order, a pair's names likewise."""
    pairs: Dict[tuple, int] = {}
    names: List[Dict[str, int]] = []
    for t in finished:
        p = pairs.setdefault((t.project, t.build_variant), len(pairs))
        if p == len(names):
            names.append({})
        names[p].setdefault(t.display_name, len(names[p]))
    off = np.zeros(len(pairs) + 1, np.int64)
    if pairs:
        np.cumsum([len(n) for n in names], out=off[1:])
    keys: List[tuple] = []
    for (proj, bv), p in pairs.items():
        keys.extend((proj, bv, n) for n in names[p])
    index = {k: i for i, k in enumerate(keys)}
    key, taken, start, finish, flags = [], [], [], [], []
    for t in finished:
        key.append(index[(t.project, t.build_variant, t.display_name)])
        taken.append(t.time_taken); start.append(t.start_time); finish.append(t.finish_time)
        flags.append((L.EVG_DR_COMPLETED if t.status in M.TASK_COMPLETED_STATUSES else 0) |
                     (L.EVG_DR_TIMED_OUT if t.timed_out else 0))
    rows = DurationRows(np.array(key, np.int32), np.array(taken, np.int64), np.array(start, np.int64),
                        np.array(finish, np.int64), np.array(flags, np.uint8), len(keys), now - 7 * 24 * M.HOUR, now)
    hist = DurationHistory(rows, off, keys, pairs, index)
    return hist, np.array([hist(t) for t in tasks], np.int32)


@dataclass
class DurationCache:
    """evg_duration_cache: what FetchExpectedDuration reads of each listed row.  rows None = every resident row."""
    value_ns: np.ndarray
    std_ns: np.ndarray
    ttl_ns: np.ndarray
    collected_ns: np.ndarray
    expected_ns: np.ndarray
    expected_std_ns: np.ndarray
    key: np.ndarray
    rows: Optional[np.ndarray] = None

    @property
    def n_rows(self) -> int:
        return int(self.key.shape[0])

    def normalize(self) -> "DurationCache":
        for f in L.DURATION_CACHE_COLUMNS:
            setattr(self, f, np.ascontiguousarray(getattr(self, f), dtype=np.int64))
        self.key = np.ascontiguousarray(self.key, dtype=np.int32)
        if self.rows is not None:
            self.rows = np.ascontiguousarray(self.rows, dtype=np.int64)
        return self

    def struct(self) -> L.DurationCacheStruct:
        s = L.DurationCacheStruct()
        s.n_rows = self.n_rows
        # NULL means "every resident row": an explicit list keeps a pointer even when it lists nothing
        self._rows_arg = None if self.rows is None else (self.rows if self.n_rows else np.zeros(1, np.int64))
        s.rows = L.ptr(self._rows_arg)
        for f in L.DURATION_CACHE_COLUMNS + ("key",):
            setattr(s, f, L.ptr(getattr(self, f)) if self.n_rows else None)
        return s

    def nbytes(self) -> int:
        return sum(getattr(self, f).nbytes for f in L.DURATION_CACHE_COLUMNS + ("key",)) + \
            (self.rows.nbytes if self.rows is not None else 0)


def _cache_of(tasks: Sequence[M.Task], codes, rows) -> DurationCache:
    ps = [t.duration_prediction for t in tasks]
    return DurationCache(np.array([p.value for p in ps], np.int64), np.array([p.std_dev for p in ps], np.int64),
                         np.array([p.ttl for p in ps], np.int64), np.array([p.collected_at for p in ps], np.int64),
                         np.array([t.expected_duration for t in tasks], np.int64),
                         np.array([t.expected_duration_std_dev for t in tasks], np.int64),
                         np.array(codes, np.int32), rows).normalize()


def marshal_duration_cache(tasks: Sequence[M.Task], lookup, rows=None) -> DurationCache:
    """The cache fields of the tick's tasks (resident order) for evg_resolve_durations; `lookup` maps a task to its key
    code (a DurationHistory).  `rows` lists the resident rows to resolve (ascending), None = all.  Reads only: the
    tasks are not touched."""
    if rows is not None:
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        tasks = [tasks[int(r)] for r in rows]
    return _cache_of(tasks, [lookup(t) for t in tasks], rows)


def marshal_running_cache(datas: Sequence[M.HostAllocatorData], running_tasks: Dict[str, M.Task], lookup):
    """The host counterpart: the running task of every host (marshal_hosts order) that `running_tasks` holds ->
    (DurationCache over those host rows, the Task of each listed row).  Hosts without such a task are not listed and
    keep what marshal_hosts gave them."""
    rows, docs = [], []
    r = 0
    for data in datas:
        for h in data.existing_hosts:
            t = running_tasks.get(h.running_task) if h.running_task != "" else None
            if t is not None:
                rows.append(r)
                docs.append(t)
            r += 1
    return _cache_of(docs, [lookup(t) for t in docs], np.array(rows, np.int64)), docs


def write_back_durations(tasks: Sequence[M.Task], out: dict) -> None:
    """What FetchExpectedDuration leaves on each Task (task.go:3519-3590): ExpectedDuration / StdDev and the
    DurationPrediction, from evg_download_durations' rows (`tasks` in listed-row order).  An unset TTL reads as
    predictionTTL, as it does on the device."""
    for i, t in enumerate(tasks):
        p = t.duration_prediction
        if p.ttl == 0:
            p.ttl = M.PREDICTION_TTL
        t.expected_duration, t.expected_duration_std_dev = int(out["avg_ns"][i]), int(out["std_ns"][i])
        p.value, p.std_dev, p.collected_at = int(out["value_ns"][i]), int(out["pred_std_ns"][i]), int(out["collected_ns"][i])


# ---------------------------------------------------------------------------------------------------------------
# legacy comparator prioritiser (scheduler/task_prioritizer.go, task_priority_cmp.go, setup_funcs.go:72-87)
@dataclass
class LegacyTable:
    """evg_legacy_soa + task_off + list_mode for a batch of distros."""
    priority: np.ndarray
    ingest_ns: np.ndarray
    expected_ns: np.ndarray
    num_dependents: np.ndarray
    revision_order: np.ndarray
    project_id: np.ndarray
    tg_rank: np.ndarray
    tg_pair_id: np.ndarray
    task_group_order: np.ndarray
    presort_rank: np.ndarray
    flags: np.ndarray
    task_off: np.ndarray
    list_mode: np.ndarray  # uint8 [3 * n_distros]: high priority, patch, repotracker

    COLUMNS = (("priority", np.int64), ("ingest_ns", np.int64), ("expected_ns", np.int64), ("num_dependents", np.int32),
               ("revision_order", np.int32), ("project_id", np.int32), ("tg_rank", np.int32), ("tg_pair_id", np.int32),
               ("task_group_order", np.int32), ("presort_rank", np.int32), ("flags", np.uint32))

    @property
    def n_tasks(self) -> int:
        return int(self.priority.shape[0])

    @property
    def n_distros(self) -> int:
        return int(self.task_off.shape[0]) - 1

    def struct(self) -> "L.LegacySoAStruct":
        s = L.LegacySoAStruct()
        s.n_tasks = self.n_tasks
        for name, _ in self.COLUMNS:
            setattr(s, name, L.ptr(getattr(self, name)))
        return s


def legacy_list_of(t: M.Task) -> int:
    """splitTasksByRequester (task_prioritizer.go:214-247): 0 high priority, 1 patch, 2 repotracker, 3 dropped."""
    if t.priority > M.MAX_TASK_PRIORITY:
        return 0
    if t.requester in M.SYSTEM_VERSION_REQUESTER_TYPES:
        return 2
    if M.is_patch_requester(t.requester):
        return 1
    return 3


def legacy_list_mode(tasks: Sequence[M.Task], expected: Sequence[int]) -> int:
    """Is the comparator chain a strict weak order on this list, and which byAge branch does it take
    (task_priority_cmp.go:73-95)?  Only tasks outside task groups reach byAge / byRuntime."""
    plain = [(t, e) for t, e in zip(tasks, expected) if t.task_group == ""]
    if any(e == 0 for _, e in plain) and any(e != 0 for _, e in plain):
        return L.EVG_LEGACY_MODE_LITERAL  # byRuntime ties a zero duration with everything (:109-111)
    commit = [t for t, _ in plain if t.requester in M.SYSTEM_VERSION_REQUESTER_TYPES]
    projects = [t.project for t in commit]
    if len(set(projects)) == len(projects):
        return L.EVG_LEGACY_MODE_INGEST      # no pair takes the revision-order branch
    if len(commit) == len(plain) and len(set(projects)) == 1:
        return L.EVG_LEGACY_MODE_REVISION    # every pair takes it
    return L.EVG_LEGACY_MODE_LITERAL


def marshal_legacy(batch: Sequence[tuple], now: Optional[int] = None, exact: bool = False) -> LegacyTable:
    """batch: (distro_id, tasks, versions) per distro; `versions` maps a version id to its Requester (what byCommitQueue
    reads of model.Version).  Resolves FetchExpectedDuration, interns the strings, decides each list's mode.
    exact=True marks a list that would be EVG_LEGACY_MODE_LITERAL (a format collision included) GO_STABLE instead, so
    the device replays Go's sort.Stable on it; INGEST and REVISION lists keep their key sort, which gives the same order
    for less."""
    cols = {name: [] for name, _ in LegacyTable.COLUMNS}
    task_off, modes = [0], []
    for _, tasks, versions in batch:
        versions = versions or {}
        expected = [M.fetch_expected_duration(t, now)[0] if now is not None else t.expected_duration for t in tasks]
        fmt = [f"{t.build_id}-{t.task_group}" for t in tasks]
        grouped = sorted({f for f, t in zip(fmt, tasks) if t.task_group != ""})
        rank = {f: k for k, f in enumerate(grouped)}
        pairs: Dict[tuple, int] = {}
        by_fmt: Dict[str, set] = {}
        for f, t in zip(fmt, tasks):
            if t.task_group != "":
                pairs.setdefault((t.task_group, t.build_id), len(pairs))
                by_fmt.setdefault(f, set()).add((t.task_group, t.build_id))
        collision = any(len(v) > 1 for v in by_fmt.values())
        keys = sorted(range(len(tasks)), key=lambda k: f"{fmt[k]}-{tasks[k].id}", reverse=True)
        presort = [0] * len(tasks)
        for pos, k in enumerate(keys):
            presort[k] = pos
        projects: Dict[str, int] = {}
        lists = [legacy_list_of(t) for t in tasks]
        for k, t in enumerate(tasks):
            if not -(2 ** 63) <= t.priority < 2 ** 63:
                raise ValueError(f"task {t.id!r}: priority {t.priority} is outside int64")
            rq = (L.EVG_LF_REQ_SYSTEM if t.requester in M.SYSTEM_VERSION_REQUESTER_TYPES else
                  L.EVG_LF_REQ_PATCH if M.is_patch_requester(t.requester) else L.EVG_LF_REQ_OTHER)
            fl = rq | (L.EVG_LF_GENERATE if t.generate_task else 0)
            if versions.get(t.version, "") == M.GITHUB_MERGE_REQUESTER:
                fl |= L.EVG_LF_MERGE_QUEUE_VERSION
            cols["priority"].append(t.priority); cols["ingest_ns"].append(t.ingest_time); cols["expected_ns"].append(expected[k])
            cols["num_dependents"].append(t.num_dependents); cols["revision_order"].append(t.revision_order_number)
            cols["project_id"].append(projects.setdefault(t.project, len(projects)))
            cols["tg_rank"].append(rank[fmt[k]] if t.task_group != "" else -1)
            cols["tg_pair_id"].append(pairs[(t.task_group, t.build_id)] if t.task_group != "" else -1)
            cols["task_group_order"].append(t.task_group_order); cols["presort_rank"].append(presort[k]); cols["flags"].append(fl)
        for lst in (0, 1, 2):
            sel = [k for k in range(len(tasks)) if lists[k] == lst]
            m = legacy_list_mode([tasks[k] for k in sel], [expected[k] for k in sel])
            m = L.EVG_LEGACY_MODE_LITERAL if collision else m
            modes.append(L.EVG_LEGACY_MODE_GO_STABLE if exact and m == L.EVG_LEGACY_MODE_LITERAL else m)
        task_off.append(task_off[-1] + len(tasks))
    return LegacyTable(**{name: np.array(cols[name], dtype=dt) for name, dt in LegacyTable.COLUMNS},
                       task_off=np.array(task_off, dtype=np.int64), list_mode=np.array(modes, dtype=np.uint8))


# ---------------------------------------------------------------------------------------------------------------
# DAG dispatcher input (model/task_queue_service_dependency.go:153-252)
def dag_input_from_queues(queues: Sequence[M.TaskQueue]):
    """Persisted TaskQueue documents -> the evg_dag_in of evg_dag_rebuild_batch, as rebuild() reads them:
    (item_off, group_off, dep_off, dep_item, group_id, group_index, per queue the compositeGroupID of each dense group).
    A dependency id that is not in the queue becomes -1 (addEdge returns without a line, :118-150)."""
    item_off, group_off, dep_off, dep_item, group_id, group_index, names = [0], [0], [0], [], [], [], []
    for q in queues:
        pos = {it.id: k for k, it in enumerate(q.queue)}
        groups: Dict[str, int] = {}
        for it in q.queue:
            for dep in it.dependencies:
                dep_item.append(pos.get(dep, -1))
            dep_off.append(len(dep_item))
            if it.group:
                gid = f"{it.group}_{it.build_variant}_{it.project}_{it.version}"  # compositeGroupID
                group_id.append(groups.setdefault(gid, len(groups)))
            else:
                group_id.append(-1)
            group_index.append(it.group_index)
        names.append(list(groups))
        item_off.append(item_off[-1] + len(q.queue))
        group_off.append(group_off[-1] + len(groups))
    a = lambda x, t: np.ascontiguousarray(np.array(x, dtype=t))  # noqa: E731
    return (a(item_off, np.int64), a(group_off, np.int64), a(dep_off, np.int64), a(dep_item, np.int32), a(group_id, np.int32),
            a(group_index, np.int32), names)


def persisted_dag_input(soa: TaskSoA, table: DistroTable, order: np.ndarray, cap: int = 0):
    """Host restatement of what evg_rebuild_dispatchers builds on the device: the evg_dag_in of every distro's persisted
    queue (the first min(length, cap) ranks, cap 0 = EVG_PERSISTED_QUEUE_CAP) from marshalled columns and the rank order
    (order[task_off[d] + r] = distro-local task at rank r; only the persisted ranks are read).
    -> (item_off, group_off, dep_off, dep_item, group_id, group_index, group_slot): item k of distro d is rank k; a
    resident edge becomes the rank of its dependency, -1 past the cap; the group slots that occur are numbered densely in
    order of first appearance, group_slot[group_off[d] + g] holding the slot of dense group g."""
    cap = cap or L.EVG_PERSISTED_QUEUE_CAP
    toff = np.asarray(table.task_off, dtype=np.int64)
    D = table.n_distros
    lens = np.minimum(np.diff(toff), cap)
    item_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    N = int(item_off[-1])
    d_of = np.repeat(np.arange(D, dtype=np.int64), lens)
    r = np.arange(N, dtype=np.int64) - item_off[d_of]
    task = toff[d_of] + np.asarray(order, dtype=np.int64)[toff[d_of] + r]
    rank_of = np.full(soa.n_tasks, -1, dtype=np.int32)
    rank_of[task] = r
    if soa.n_edges:
        deg = soa.dep_off[task + 1] - soa.dep_off[task]
        dep_off = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        e = np.repeat(soa.dep_off[task] - dep_off[:-1], deg) + np.arange(int(dep_off[-1]), dtype=np.int64)
        dep_item = rank_of[np.repeat(toff[d_of], deg) + soa.dep_idx[e]].astype(np.int32)
    else:
        dep_off, dep_item = np.zeros(N + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)
    slot = soa.group_id[task].astype(np.int64)
    grouped = np.nonzero(slot >= 0)[0]
    key = np.asarray(table.group_off, dtype=np.int64)[d_of[grouped]] + slot[grouped]
    _, first_at, inv = np.unique(key, return_index=True, return_inverse=True)
    head = grouped[first_at]                    # the item that first holds each occurring slot
    flag = np.zeros(N + 1, dtype=np.int64)
    flag[head] = 1
    pos = np.concatenate([[0], np.cumsum(flag[:N])])
    group_id = np.full(N, -1, dtype=np.int32)
    group_id[grouped] = pos[head[inv.ravel()]] - pos[item_off[d_of[grouped]]]
    group_off = pos[item_off].astype(np.int64)
    group_slot = np.zeros(int(group_off[-1]), dtype=np.int32)
    group_slot[pos[head]] = slot[head]
    return (item_off, group_off, dep_off, dep_item, group_id, soa.task_group_order[task].astype(np.int32), group_slot)


# ---------------------------------------------------------------------------------------------------------------
# FindNextTask's inputs (model/task_queue_service_dependency.go:258-469): evg_next_db and evg_next_req
def marshal_next_db(item_ids: Sequence[Sequence[str]], group_names: Sequence[Sequence[str]], db: dict) -> dict:
    """A database snapshot -> the columns of evg_next_db over the dispatchers' items (`item_ids[d]`: distro d's item ids
    in queue order) and groups (`group_names[d]`: the compositeGroupID of each dense group).  `db`:
      tasks: {id: {"start", "finish", "ingest": ns (M.ZERO_TIME = Go's zero time), "status", "version",
                   "est_generated": int or None, "deps_met": True / False / None for an error}}; a missing id = no document
      versions: {id: ProjectStorageMethod}; running_hosts: {compositeGroupID: count, -1 = error}, missing = 0
      generate_limit, pending_generate, max_large_parser, num_large_parser: ints, -1 = the query failed.
    The two start-time bits are evaluated as the reference writes them: !utility.IsZeroTime(StartTime) (:334) and
    StartTime != utility.ZeroTime, a comparison with time.Unix(0, 0) that Go's zero time fails (:657)."""
    flags, est, ingest = [], [], []
    tasks, versions = db.get("tasks", {}), db.get("versions", {})
    for ids in item_ids:
        for i in ids:
            doc = tasks.get(i)
            f = 0
            if doc is not None:
                f |= L.EVG_ND_FOUND
                if not M.is_zero_time(doc.get("start", 0)):
                    f |= L.EVG_ND_STARTED
                if doc.get("start", 0) != 0:
                    f |= L.EVG_ND_STARTED_GROUP
                if not M.is_zero_time(doc.get("finish", 0)) and doc.get("status", "") != M.TASK_SUCCEEDED:
                    f |= L.EVG_ND_FINISHED_NOT_SUCCEEDED
                if doc.get("version", "") in versions:
                    f |= L.EVG_ND_VERSION_FOUND
                    if versions[doc.get("version", "")] == "s3":
                        f |= L.EVG_ND_VERSION_S3
                met = doc.get("deps_met", True)
                f |= L.EVG_ND_DEPS_ERR if met is None else (L.EVG_ND_DEPS_MET_NOW if met else 0)
            flags.append(f)
            est.append(int((doc or {}).get("est_generated") or 0))
            t = (doc or {}).get("ingest", 0)
            ingest.append(0 if t == M.ZERO_TIME else t)  # only compared with After(amiUpdatedTime), itself after the epoch
    hosts = db.get("running_hosts", {})
    return {"flags": np.array(flags, dtype=np.uint8), "est_generated": np.array(est, dtype=np.int32),
            "ingest_ns": np.array(ingest, dtype=np.int64),
            "running_hosts": np.array([hosts.get(n, 0) for names in group_names for n in names], dtype=np.int32),
            "generate_limit": int(db.get("generate_limit", 0)), "pending_generate": int(db.get("pending_generate", 0)),
            "max_large_parser": int(db.get("max_large_parser", 0)), "num_large_parser": int(db.get("num_large_parser", 0))}


def marshal_next_requests(group_names: Sequence[Sequence[str]], requests):
    """`requests[d]`: distro d's (TaskSpec or None, amiUpdatedTime) in serving order -> (req_off, group, ami_updated_ns):
    the spec's compositeGroupID resolved to the dispatcher's dense group id, -1 for spec.Group == "" or an id that is
    none of the dispatcher's groups (:268-274); a zero amiUpdatedTime becomes 0."""
    req_off, group, ami = [0], [], []
    for names, reqs in zip(group_names, requests):
        dense = {n: g for g, n in enumerate(names)}
        for spec, t in reqs:
            group.append(dense.get(spec.composite_group_id(), -1) if spec is not None and spec.group else -1)
            ami.append(0 if M.is_zero_time(t) else t)
        req_off.append(len(group))
    return np.array(req_off, dtype=np.int64), np.array(group, dtype=np.int32), np.array(ami, dtype=np.int64)
