"""Host-side mirror of the reference `scheduler` package's plug points, backed by
libevgsched.so (CUDA, sm_90a).  Same names, argument meaning and error
behaviour as the Go interfaces this path sits behind:

* ``PrioritizeTasks`` / ``TaskPlanner``      scheduler/scheduler.go:25-51
* ``GetDistroQueueInfo``                      scheduler/scheduler.go:56-159
* ``HostAllocator`` / ``GetHostAllocator``    scheduler/host_allocator.go:15-32
* ``UtilizationBasedHostAllocator``           scheduler/utilization_based_host_allocator.go:26-130
* ``PlanDistro`` (planner half, DB-free)      scheduler/wrapper.go:30-130

plus the batched entry the GPU wants (one call per 15 s tick instead of one
amboy job per distro, units/crons.go:303-332).  Nothing here computes scores,
orders or host counts on the CPU; the host code only marshals and un-marshals.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L
from . import model as M
from . import soa as S

RUNNER_NAME = "scheduler"  # scheduler/scheduler.go:53
# new plug names a maintainer registers next to the existing ones
# (globals.go:1080-1100: ValidTaskPlannerVersions / ValidHostAllocators)
PLANNER_VERSION_GPU_TUNABLE = "gpu-tunable"
HOST_ALLOCATOR_GPU_UTILIZATION = "gpu-utilization"


class AllocatorError(Exception):
    """The `error` UtilizationBasedHostAllocator returns for data problems."""
    MESSAGES = {
        L.EVG_ALLOC_ERR_FUTURE_FRACTION: "future host factor must be between 0 and 1",   # allocator.go:302-304, NaN and < 0 too
        L.EVG_ALLOC_ERR_POOL_SIZE: "unable to plan hosts for distro due to pool size",     # allocator.go:200-202
        L.EVG_ALLOC_ERR_PARENT_MISSING: "error finding parent distros",                    # allocator.go:151-158
    }

    def __init__(self, status: int, distro_id: str = ""):
        super().__init__(f"error calculating hosts for distro {distro_id}: {self.MESSAGES.get(status, status)}")
        self.status = status


class Engine:
    """One evg_ctx: device buffers + stream.  Thread-compatible (one tick at a time).

    Result arrays live in pinned host buffers owned by the engine and are REUSED by the next
    call: copy what must outlive the next tick."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self.lib = L.load()
        h = C.c_void_p()
        L.check(self.lib.evg_init(int(device), C.c_void_p(stream) if stream else None, C.byref(h)))
        self.ctx = h
        self._n_tasks = self._n_distros = self._n_groups = 0
        self._n_disp = (0, 0)  # items and groups of the last rebuild_dispatchers()
        self._has_hosts = False
        self._n_dur = (0, 0)  # task and host rows of the last resolve_durations
        self._pinned = {}  # name -> (address, capacity in bytes): result buffers reused across ticks

    def close(self) -> None:
        if getattr(self, "ctx", None):
            for addr, _ in self._pinned.values():
                self.lib.evg_host_free(C.c_void_p(addr))
            self._pinned = {}
            self.lib.evg_shutdown(self.ctx)
            self.ctx = None

    def _out(self, name: str, shape, dtype) -> np.ndarray:
        """A result array in pinned host memory (evg_host_alloc), cached by name and grown on demand.
        The returned view is only valid until the next call that produces the same result."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
        nbytes = max(n * dtype.itemsize, 1)
        addr, cap = self._pinned.get(name, (0, 0))
        if cap < nbytes:
            if addr:
                self.lib.evg_host_free(C.c_void_p(addr))
            cap = nbytes + nbytes // 8
            addr = self.lib.evg_host_alloc(cap)
            if not addr:
                raise L.EvgError(L.EVG_ERR_NOMEM, L.last_error())
            self._pinned[name] = (addr, cap)
        buf = (C.c_uint8 * nbytes).from_address(addr)
        return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)

    def _plan_output(self, T: int, D: int, G: int, breakdown: bool) -> S.PlanOutput:
        info = self._out("info", D, L.QUEUE_INFO_DTYPE)
        ginfo = self._out("group_info", G, L.GROUP_INFO_DTYPE)
        return S.PlanOutput(self._out("order", T, np.int32), self._out("total_value", T, np.int64), info, ginfo,
                            self._out("breakdown", (T, L.EVG_BD_N), np.int64) if breakdown else None)

    def _alloc_output(self, D: int) -> S.AllocOutput:
        return S.AllocOutput(self._out("result", D, L.ALLOC_RESULT_DTYPE), self._out("status", D, np.int32))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- resident API ------------------------------------------------------
    def upload(self, tasks: S.TaskSoA, distros: S.DistroTable, hosts: Optional[S.HostSoA] = None) -> None:
        ts, ds = tasks.struct(), distros.struct()
        if hosts is not None:
            hs = hosts.struct()
            L.check(self.lib.evg_upload(self.ctx, C.byref(ts), C.byref(ds), C.byref(hs), L.ptr(hosts.host_off),
                                        L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None))
        else:
            L.check(self.lib.evg_upload(self.ctx, C.byref(ts), C.byref(ds), None, None, None))
        self._n_tasks, self._n_distros, self._n_groups = tasks.n_tasks, distros.n_distros, distros.n_groups
        self._has_hosts = hosts is not None

    def upload_with_deps(self, tasks: S.TaskSoA, distros: S.DistroTable, hosts: Optional[S.HostSoA], deps: "S.DepsTable",
                         dep_finished: Optional[np.ndarray], now: int) -> None:
        """evg_upload_with_deps: the device evaluates Task.DependenciesMet and writes the deps-met bit and the stamped
        wait basis of the resident columns itself."""
        ts, ds, dp = tasks.struct(), distros.struct(), deps.struct()
        fin = None
        if dep_finished is not None and dep_finished.shape[0]:
            fin = np.ascontiguousarray(dep_finished, dtype=np.int64)
        if hosts is not None:
            hs = hosts.struct()
            L.check(self.lib.evg_upload_with_deps(self.ctx, C.byref(ts), C.byref(ds), C.byref(hs), L.ptr(hosts.host_off),
                                                  L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None, C.byref(dp), L.ptr(fin), int(now)))
        else:
            L.check(self.lib.evg_upload_with_deps(self.ctx, C.byref(ts), C.byref(ds), None, None, None, C.byref(dp), L.ptr(fin), int(now)))
        self._n_tasks, self._n_distros, self._n_groups = tasks.n_tasks, distros.n_distros, distros.n_groups
        self._has_hosts = hosts is not None

    def download_deps(self):
        """(met, met_time): the device's Task.DependenciesMet verdicts and DependenciesMetTime stamps of the resident tick."""
        met = self._out("deps_met", self._n_tasks, np.uint8)
        stamp = self._out("deps_stamp", self._n_tasks, np.int64)
        L.check(self.lib.evg_download_deps(self.ctx, L.ptr(met) if self._n_tasks else None, L.ptr(stamp) if self._n_tasks else None))
        return met, stamp

    def upload_device(self, cols: dict, n_tasks: int, distros: S.DistroTable, hosts: Optional[S.HostSoA] = None,
                      n_edges: int = 0) -> None:
        """evg_upload_device: the task columns already live in device memory.  `cols` maps the evg_task_soa column
        names to device addresses (16-byte aligned, readable 8 rows past the end); nothing is copied, the caller
        keeps the memory alive until the next upload."""
        ts = L.TaskSoAStruct(int(n_tasks), int(n_edges), *[cols.get(name) for name, _ in S.TaskSoA.COLUMNS],
                             cols.get("dep_off"), cols.get("dep_idx"))
        ds = distros.struct()
        if hosts is not None:
            hs = hosts.struct()
            L.check(self.lib.evg_upload_device(self.ctx, C.byref(ts), C.byref(ds), C.byref(hs), L.ptr(hosts.host_off),
                                               L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None))
        else:
            L.check(self.lib.evg_upload_device(self.ctx, C.byref(ts), C.byref(ds), None, None, None))
        self._n_tasks, self._n_distros, self._n_groups = int(n_tasks), distros.n_distros, distros.n_groups
        self._has_hosts = hosts is not None

    def update_tasks(self, rows: np.ndarray, values: S.TaskSoA) -> None:
        """evg_update_tasks: the per-task scalars of `rows` (task slots of the resident table) take the values of
        `values`' rows; group / version / dependency structure stays.  48 B per changed row cross PCIe."""
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        values = values.normalize()
        if values.n_tasks != rows.shape[0]:
            raise ValueError("one value row per updated task slot")
        vs = values.struct()
        L.check(self.lib.evg_update_tasks(self.ctx, int(rows.shape[0]), L.ptr(rows), C.byref(vs)))

    def edit_tasks(self, edit: S.TaskEdit, distros: S.DistroTable, hosts: Optional[S.HostSoA] = None) -> None:
        """evg_edit_tasks: rows leave and join the resident queues on the device; `distros` is the new distro table
        (soa.apply_edit builds it).  The context then holds the tick a fresh upload of the composed table would."""
        es, keep = edit.normalize().struct()
        ds = distros.struct()
        hargs = (None, None, None)
        if hosts is not None:
            hs = hosts.struct()
            hargs = (C.byref(hs), L.ptr(hosts.host_off), L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None)
        L.check(self.lib.evg_edit_tasks(self.ctx, C.byref(es), C.byref(ds), *hargs))
        del keep
        self._n_tasks, self._n_distros, self._n_groups = int(distros.task_off[-1]), distros.n_distros, distros.n_groups
        self._has_hosts = hosts is not None

    def run(self, now: int, opts: int = 0) -> None:
        L.check(self.lib.evg_run_resident(self.ctx, int(now), int(opts)))

    def download(self, want_breakdown: bool = False, want_alloc: Optional[bool] = None):
        T, D, G = self._n_tasks, self._n_distros, self._n_groups
        po = self._plan_output(T, D, G, want_breakdown)
        ps = L.PlanOutStruct(L.ptr(po.order), L.ptr(po.total_value),
                             L.ptr(po.breakdown) if want_breakdown else None, L.ptr(po.info), L.ptr(po.group_info))
        ao = None
        if want_alloc is None:
            want_alloc = self._has_hosts
        if want_alloc:
            ao = self._alloc_output(D)
            as_ = L.AllocOutStruct(L.ptr(ao.result), L.ptr(ao.status))
            L.check(self.lib.evg_download(self.ctx, C.byref(ps), C.byref(as_)))
        else:
            L.check(self.lib.evg_download(self.ctx, C.byref(ps), None))
        return po, ao

    def download_queue(self, cap: int = 0, task_off=None):
        """evg_download_queue: (item_off, items) -- the TaskQueueItem rows of the first min(length, cap) ranks of every
        distro (cap 0 = the reference's 10 000), projected on the device; only those rows cross PCIe."""
        D = self._n_distros
        item_off = self._out("queue_item_off", D + 1, np.int64)
        cap_eff = cap or L.EVG_PERSISTED_QUEUE_CAP
        n = self._n_tasks if task_off is None else int(np.minimum(np.diff(task_off), cap_eff).sum())
        items = self._out("queue_items", max(n, 1), L.QUEUE_ITEM_DTYPE)
        L.check(self.lib.evg_download_queue(self.ctx, int(cap), L.ptr(item_off), L.ptr(items), int(max(n, 1))))
        return item_off, items[: int(item_off[D])]

    def bind_result_buffer(self, device_ptr: int, capacity_rows: int) -> None:
        """The allocator kernel writes evg_alloc_result rows straight into this device buffer
        (the all-gather send buffer, evergreen_b200.dist)."""
        L.check(self.lib.evg_bind_result_buffer(self.ctx, C.c_void_p(device_ptr) if device_ptr else None, int(capacity_rows)))

    def device_result_ptr(self) -> int:
        return int(self.lib.evg_device_result_ptr(self.ctx) or 0)

    def last_launch_count(self) -> int:
        return int(self.lib.evg_last_launch_count(self.ctx))

    def last_timing_ms(self) -> Tuple[float, float]:
        a, b = C.c_float(), C.c_float()
        L.check(self.lib.evg_last_timing_ms(self.ctx, C.byref(a), C.byref(b)))
        return a.value, b.value

    def general_timing_ms(self) -> Tuple[float, float]:
        """(k_gtask ms, segmented sort ms) of the last resident run; raises when it had no general-path distro."""
        a, b = C.c_float(), C.c_float()
        L.check(self.lib.evg_general_timing_ms(self.ctx, C.byref(a), C.byref(b)))
        return float(a.value), float(b.value)

    def kernel_timing_ms(self, n: int):
        """Per-run device time of the dominant kernel (k_plan_smem<1024,12>) for the last n resident runs."""
        buf = (C.c_float * max(n, 1))()
        L.check(self.lib.evg_kernel_timing_ms(self.ctx, buf, int(n)))
        return [buf[k] for k in range(n)]

    # -- one-shot batch API (host buffers in, host buffers out) ---------------
    def plan_batch(self, tasks: S.TaskSoA, distros: S.DistroTable, now: int, breakdown: bool = False) -> S.PlanOutput:
        T, D, G = tasks.n_tasks, distros.n_distros, distros.n_groups
        po = self._plan_output(T, D, G, breakdown)
        ps = L.PlanOutStruct(L.ptr(po.order), L.ptr(po.total_value), L.ptr(po.breakdown) if breakdown else None,
                             L.ptr(po.info), L.ptr(po.group_info))
        ts, ds = tasks.struct(), distros.struct()
        L.check(self.lib.evg_plan_batch(self.ctx, C.byref(ts), C.byref(ds), int(now),
                                        L.EVG_OPT_BREAKDOWN if breakdown else 0, C.byref(ps)))
        self._n_tasks, self._n_distros, self._n_groups, self._has_hosts = T, D, G, False
        return po

    def plan_and_alloc_batch(self, tasks: S.TaskSoA, distros: S.DistroTable, hosts: S.HostSoA, now: int,
                             breakdown: bool = False):
        T, D, G = tasks.n_tasks, distros.n_distros, distros.n_groups
        po = self._plan_output(T, D, G, breakdown)
        ao = self._alloc_output(D)
        ps = L.PlanOutStruct(L.ptr(po.order), L.ptr(po.total_value), L.ptr(po.breakdown) if breakdown else None,
                             L.ptr(po.info), L.ptr(po.group_info))
        as_ = L.AllocOutStruct(L.ptr(ao.result), L.ptr(ao.status))
        ts, ds, hs = tasks.struct(), distros.struct(), hosts.struct()
        L.check(self.lib.evg_plan_and_alloc_batch(self.ctx, C.byref(ts), C.byref(ds), C.byref(hs), L.ptr(hosts.host_off),
                                                  L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None, int(now),
                                                  L.EVG_OPT_BREAKDOWN if breakdown else 0, C.byref(ps), C.byref(as_)))
        self._n_tasks, self._n_distros, self._n_groups, self._has_hosts = T, D, G, True
        return po, ao

    def deps_met_batch(self, deps: "S.DepsTable") -> np.ndarray:
        """Task.DependenciesMet for every task of the tick on the device (evg_deps_met_batch)."""
        met = self._out("deps_met", deps.n_tasks, np.uint8)
        st = deps.struct()
        L.check(self.lib.evg_deps_met_batch(self.ctx, C.byref(st), L.ptr(met) if deps.n_tasks else None))
        return met

    def find_runnable_batch(self, table: "S.RunnableTable"):
        """The task finders' filter for every distro at once (evg_find_runnable_batch):
        -> (runnable [n_tasks] distro-local indices compacted per distro, -1 padded; count [n_distros])."""
        runnable = self._out("runnable", table.n_tasks, np.int32)
        count = self._out("runnable_count", table.n_distros, np.int64)
        st, keep = table.struct()
        outs = (L.ptr(runnable) if table.n_tasks else None, L.ptr(count) if table.n_distros else None)
        if table.pipe is None:
            L.check(self.lib.evg_find_runnable_batch(self.ctx, C.byref(st), *outs))
        else:  # evg_find_runnable_ex: the pipeline finder's tables ride along
            ps = table.pipe.struct()
            L.check(self.lib.evg_find_runnable_ex(self.ctx, C.byref(st), C.byref(ps), *outs))
        del keep
        return runnable, count

    def plan_from_finder(self, table: "S.RunnableTable", candidates: S.TaskSoA, distros: S.DistroTable,
                         hosts: Optional[S.HostSoA], dep_finished: Optional[np.ndarray], now: int):
        """evg_plan_from_finder: finder -> dependency predicate -> compaction -> resident planner inputs on the device.
        -> (runnable, count) as find_runnable_batch; the context then holds the tick of the KEPT tasks (run / download)."""
        if table.deps is None:
            raise ValueError("plan_from_finder needs the candidates' dependency table")
        runnable = self._out("runnable", table.n_tasks, np.int32)
        count = self._out("runnable_count", table.n_distros, np.int64)
        st, keep = table.struct()
        ts, ds = candidates.normalize().struct(), distros.struct()
        fin = None if dep_finished is None else np.ascontiguousarray(dep_finished, dtype=np.int64)
        hargs = (None, None, None)
        if hosts is not None:
            hs = hosts.struct()
            hargs = (C.byref(hs), L.ptr(hosts.host_off), L.ptr(hosts.cfg) if hosts.cfg.shape[0] else None)
        rest = (*hargs, L.ptr(fin) if fin is not None and fin.shape[0] else None, int(now),
                L.ptr(runnable) if table.n_tasks else None, L.ptr(count) if table.n_distros else None)
        if table.pipe is None:
            L.check(self.lib.evg_plan_from_finder(self.ctx, C.byref(st), C.byref(ts), C.byref(ds), *rest))
        else:  # evg_plan_from_finder_ex
            ps = table.pipe.struct()
            L.check(self.lib.evg_plan_from_finder_ex(self.ctx, C.byref(st), C.byref(ps), C.byref(ts), C.byref(ds), *rest))
        del keep
        self._n_tasks, self._n_distros, self._n_groups = int(count.sum()), distros.n_distros, distros.n_groups
        self._has_hosts = hosts is not None
        return runnable, count

    def plan_aliases(self, table: "S.AliasTable", cfg: np.ndarray, now: int):
        """evg_plan_aliases: every distro's alias queue built on the device from the tick's schedulable tasks, each
        given once; the context then holds the alias queues as its tick (run / download, planner only).
        -> (task_off, group_off, n_versions) of the alias queues."""
        D = int(cfg.shape[0])
        cfg = np.ascontiguousarray(cfg, dtype=L.DISTRO_CFG_DTYPE)
        task_off, group_off = np.zeros(D + 1, np.int64), np.zeros(D + 1, np.int64)
        n_versions = np.zeros(max(D, 1), np.int32)
        st, keep = table.normalize().struct()
        out = L.AliasOutStruct(L.ptr(task_off), L.ptr(group_off), L.ptr(n_versions))
        L.check(self.lib.evg_plan_aliases(self.ctx, C.byref(st), L.ptr(cfg) if D else None, D, int(now), C.byref(out)))
        del keep
        self._n_tasks, self._n_distros, self._n_groups = int(task_off[D]), D, int(group_off[D])
        self._has_hosts = False
        return task_off, group_off, n_versions[:D]

    def download_alias_map(self):
        """evg_download_alias_map: (source row of every resident row, global group id of every group slot)."""
        src = self._out("alias_source_row", self._n_tasks, np.int32)
        gsrc = self._out("alias_group_source", self._n_groups, np.int32)
        L.check(self.lib.evg_download_alias_map(self.ctx, L.ptr(src) if self._n_tasks else None,
                                                L.ptr(gsrc) if self._n_groups else None))
        return src, gsrc

    def expected_durations_batch(self, rows: "S.DurationRows") -> np.ndarray:
        """{$avg, $stdDevPop} of TimeTaken per key (evg_expected_durations_batch) -> DURATION_STAT_DTYPE[n_keys]."""
        out = self._out("duration_stats", rows.n_keys, L.DURATION_STAT_DTYPE)
        st = rows.struct()
        L.check(self.lib.evg_expected_durations_batch(self.ctx, C.byref(st), L.ptr(out) if rows.n_keys else None))
        return out

    def resolve_durations(self, history: Optional["S.DurationHistory"], now: int, tasks: Optional["S.DurationCache"] = None,
                          hosts: Optional["S.DurationCache"] = None) -> None:
        """evg_resolve_durations: Task.FetchExpectedDuration for the listed rows of the resident tick, against the
        weekly statistics of `history`, written into the resident expected_ns (tasks) and expected_ns / std_ns (hosts)
        on the device.  None leaves that side as uploaded."""
        keep = []
        din = L.DurationInStruct()
        if history is not None:
            hs = history.rows.struct()
            keep.append(hs)
            din.history = C.pointer(hs)
            din.n_pairs = history.n_pairs
            off = np.ascontiguousarray(history.pair_key_off, dtype=np.int64)
            keep.append(off)
            din.pair_key_off = L.ptr(off)
        for name, cache in (("tasks", tasks), ("hosts", hosts)):
            if cache is not None:
                cs = cache.normalize().struct()
                keep.append(cs)
                setattr(din, name, C.pointer(cs))
        L.check(self.lib.evg_resolve_durations(self.ctx, C.byref(din), int(now)))
        self._n_dur = (tasks.n_rows if tasks is not None else 0, hosts.n_rows if hosts is not None else 0)
        del keep

    def download_durations(self):
        """evg_download_durations -> (tasks, hosts): dicts of avg_ns, std_ns, value_ns, pred_std_ns, collected_ns and
        source (EVG_DS_*) per listed row of the last resolve_durations."""
        res = []
        for side, n in zip(("tasks", "hosts"), self._n_dur):
            res.append({f: self._out(f"dur_{side}_{f}", n, np.uint8 if f == "source" else np.int64) for f in L.DURATION_OUT_FIELDS})
        outs = [L.DurationOutStruct(*[L.ptr(d[f]) if d[f].shape[0] else None for f in L.DURATION_OUT_FIELDS]) for d in res]
        L.check(self.lib.evg_download_durations(self.ctx, C.byref(outs[0]), C.byref(outs[1])))
        return res[0], res[1]

    def prioritize_legacy_batch(self, table: "S.LegacyTable"):
        """evg_prioritize_legacy_batch: (order, count, status) of CmpBasedTaskPrioritizer over every distro of the table."""
        T, D = table.n_tasks, table.n_distros
        order = self._out("legacy_order", T, np.int32)
        count = self._out("legacy_count", D, np.int64)
        status = self._out("legacy_status", D, np.int32)
        ts = table.struct()
        L.check(self.lib.evg_prioritize_legacy_batch(self.ctx, C.byref(ts), L.ptr(table.task_off), L.ptr(table.list_mode), D,
                                                     L.ptr(order) if T else None, L.ptr(count), L.ptr(status)))
        return order, count, status

    def dag_rebuild_batch(self, item_off, group_off, dep_off, dep_item, group_id, group_index):
        """evg_dag_rebuild_batch -> (sorted, n_sorted, n_cycles, unit_items, unit_off)."""
        D = int(item_off.shape[0]) - 1
        N, E, G = int(item_off[-1]), int(dep_off[-1]) if dep_off.shape[0] else 0, int(group_off[-1])
        st = L.DagInStruct(N, E, L.ptr(dep_off), L.ptr(dep_item) if E else None, L.ptr(group_id) if N else None,
                           L.ptr(group_index) if N else None)
        sorted_ = self._out("dag_sorted", max(N, 1), np.int32)
        n_sorted, n_cycles = self._out("dag_nsorted", D, np.int32), self._out("dag_ncycles", D, np.int32)
        unit_items, unit_off = self._out("dag_unit_items", max(N, 1), np.int32), self._out("dag_unit_off", G + D, np.int32)
        L.check(self.lib.evg_dag_rebuild_batch(self.ctx, C.byref(st), L.ptr(item_off), L.ptr(group_off), D, L.ptr(sorted_) if N else None,
                                               L.ptr(n_sorted), L.ptr(n_cycles), L.ptr(unit_items) if N else None, L.ptr(unit_off)))
        return sorted_[:N], n_sorted, n_cycles, unit_items[:N], unit_off

    def rebuild_dispatchers(self, cap: int = 0):
        """evg_rebuild_dispatchers: the DAG dispatcher of every distro's persisted queue (the first min(length, cap) ranks,
        cap 0 = the reference's 10 000), built on the device from the resident tick after run().  -> dict of
        L.DISPATCH_OUT_FIELDS: item_off, sorted, n_sorted, n_cycles, group_off, group_slot, unit_items, unit_off, laid
        out as dag_rebuild_batch's results; group_slot maps each dense group back to the tick's group slot."""
        T, D, G = self._n_tasks, self._n_distros, self._n_groups
        o = {"item_off": self._out("disp_item_off", D + 1, np.int64), "group_off": self._out("disp_group_off", D + 1, np.int64)}
        for f, n in (("sorted", T), ("unit_items", T), ("group_slot", G), ("unit_off", G + D), ("n_sorted", D), ("n_cycles", D)):
            o[f] = self._out(f"disp_{f}", max(n, 1), np.int32)
        st = L.DispatchOutStruct(*[L.ptr(o[f]) for f in L.DISPATCH_OUT_FIELDS])
        L.check(self.lib.evg_rebuild_dispatchers(self.ctx, int(cap), max(T, 1), max(G, 1), C.byref(st)))
        N, G2 = int(o["item_off"][D]), int(o["group_off"][D])
        self._n_disp = (N, G2)
        return {"item_off": o["item_off"], "sorted": o["sorted"][:N], "n_sorted": o["n_sorted"][:D], "n_cycles": o["n_cycles"][:D],
                "group_off": o["group_off"], "group_slot": o["group_slot"][:G2], "unit_items": o["unit_items"][:N],
                "unit_off": o["unit_off"][:G2 + D]}

    @staticmethod
    def _next_args(db: dict, req, n_items: int, n_groups: int):
        """The evg_next_db / evg_next_req / evg_next_out of one call (soa.marshal_next_db, soa.marshal_next_requests)."""
        req_off, group, ami = (np.ascontiguousarray(a, dtype=t) for a, t in zip(req, (np.int64, np.int32, np.int64)))
        R = int(group.shape[0])
        cols = {f: np.ascontiguousarray(db[f]) for f in ("flags", "est_generated", "ingest_ns", "running_hosts")}
        dbs = L.NextDbStruct(n_items, n_groups, *[L.ptr(cols[f]) if cols[f].shape[0] else None
                                                  for f in ("flags", "est_generated", "ingest_ns", "running_hosts")],
                             db["generate_limit"], db["pending_generate"], db["max_large_parser"], db["num_large_parser"])
        rs = L.NextReqStruct(R, L.ptr(req_off), L.ptr(group) if R else None, L.ptr(ami) if R else None)
        item, outcome = np.full(R, -1, np.int32), np.zeros(R, np.int32)
        os_ = L.NextOutStruct(L.ptr(item) if R else None, L.ptr(outcome) if R else None)
        return dbs, rs, os_, item, outcome, (req_off, group, ami, cols)

    @staticmethod
    def _next_state(n_items: int, n_groups: int, state: Optional[dict] = None):
        st = {"item_bits": np.zeros(max(n_items, 1), np.uint8), "group_deleted": np.zeros(max(n_groups, 1), np.uint8),
              "group_running": np.zeros(max(n_groups, 1), np.int32)}
        if state is not None:
            for k in st:
                st[k][:state[k].shape[0]] = state[k]
        return st, L.NextStateStruct(*[L.ptr(st[k]) for k in ("item_bits", "group_deleted", "group_running")])

    def find_next_batch(self, disp: dict, db: dict, req, state: Optional[dict] = None):
        """evg_find_next_batch: FindNextTask for every request of every distro over host-marshalled dispatchers (`disp`:
        arrays named L.NEXT_DISPATCHER_FIELDS).  `state`: dict of item_bits / group_deleted / group_running, None = what a
        rebuild leaves.  -> (item per request, outcome per request, the state after the call)."""
        D = int(disp["item_off"].shape[0]) - 1
        N, G = int(disp["item_off"][-1]), int(disp["group_off"][-1])
        arrs = {f: np.ascontiguousarray(disp[f]) for f in L.NEXT_DISPATCHER_FIELDS}
        ds = L.NextDispatchersStruct(D, 0, *[L.ptr(arrs[f]) if arrs[f].shape[0] else None for f in L.NEXT_DISPATCHER_FIELDS])
        dbs, rs, os_, item, outcome, keep = self._next_args(db, req, N, G)
        st_in, si = self._next_state(N, G, state)
        st_out, so = self._next_state(N, G)
        L.check(self.lib.evg_find_next_batch(self.ctx, C.byref(ds), C.byref(dbs), C.byref(rs), C.byref(si), C.byref(so), C.byref(os_)))
        del keep
        return item, outcome, {"item_bits": st_out["item_bits"][:N], "group_deleted": st_out["group_deleted"][:G],
                               "group_running": st_out["group_running"][:G]}

    def find_next_tasks(self, db: dict, req):
        """evg_find_next_tasks: the same on the dispatchers the last rebuild_dispatchers() built, whose state stays on
        the device.  -> (item per request: the rank evg_download_queue returns, outcome per request)."""
        dbs, rs, os_, item, outcome, keep = self._next_args(db, req, *self._n_disp)
        L.check(self.lib.evg_find_next_tasks(self.ctx, C.byref(dbs), C.byref(rs), C.byref(os_)))
        del keep
        return item, outcome

    def download_dispatch_state(self) -> dict:
        """evg_download_dispatch_state: item_bits (EVG_NS_*), group_deleted and group_running of the chained dispatchers."""
        N, G = self._n_disp
        st, ss = self._next_state(N, G)
        L.check(self.lib.evg_download_dispatch_state(self.ctx, C.byref(ss)))
        return {"item_bits": st["item_bits"][:N], "group_deleted": st["group_deleted"][:G], "group_running": st["group_running"][:G]}

    def host_job(self, cfg: np.ndarray, spawned: Optional[np.ndarray] = None) -> dict:
        """evg_host_job: hostAllocatorJob.Run past the allocator for every distro of the resident tick after run(),
        on the device.  `cfg`: HOST_JOB_CFG rows (soa.marshal_host_job); `spawned`: len(hostsSpawned) per distro, None
        = max(n_hosts, 0).  -> dict of n_hosts, n_hosts_free, status (EVG_ALLOC_*) and report (HOST_REPORT rows)."""
        D = self._n_distros
        cfg = np.ascontiguousarray(cfg, dtype=L.HOST_JOB_CFG_DTYPE)
        if cfg.shape[0] != D or (spawned is not None and len(spawned) != D):
            raise ValueError("one job setting and spawned count per distro of the resident tick")
        sp = None if spawned is None else np.ascontiguousarray(spawned, dtype=np.int32)
        o = {"n_hosts": self._out("job_n_hosts", max(D, 1), np.int64), "n_hosts_free": self._out("job_n_free", max(D, 1), np.int64),
             "status": self._out("job_status", max(D, 1), np.int32), "report": self._out("job_report", max(D, 1), L.HOST_REPORT_DTYPE)}
        st = L.HostJobOutStruct(*[L.ptr(o[f]) for f in ("n_hosts", "n_hosts_free", "status", "report")])
        cfg_arg = cfg if D else np.zeros(1, L.HOST_JOB_CFG_DTYPE)
        L.check(self.lib.evg_host_job(self.ctx, L.ptr(cfg_arg), L.ptr(sp) if sp is not None and D else None, C.byref(st)))
        return {k: v[:D] for k, v in o.items()}

    def host_drawdown(self, table: S.IdleHostTable, existing_hosts, now: int, new_cap_target=None, queue_length_dm=None) -> dict:
        """evg_host_drawdown: hostDrawdownJob.Run for every distro of `table`, on the device.  `new_cap_target` (int64,
        EVG_NO_DRAWDOWN = no job) and `queue_length_dm` both None: chained on the resident tick's last host_job, whose
        distros are the table's.  -> dict of hosts (HOST_VERDICT rows) and distros (DRAWDOWN_DISTRO rows)."""
        D, H = table.n_distros, table.n_hosts
        if (new_cap_target is None) != (queue_length_dm is None):
            raise ValueError("new_cap_target and queue_length_dm: both or neither")
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.int64) for a in (existing_hosts, new_cap_target, queue_length_dm)]
        if any(a is not None and a.shape != (D,) for a in arrs):
            raise ValueError("one existing count, cap and queue length per distro of the table")
        arrs = [None if a is None else (a if D else np.zeros(1, np.int64)) for a in arrs]
        o = {"hosts": np.zeros(max(H, 1), L.HOST_VERDICT_DTYPE), "distros": np.zeros(max(D, 1), L.DRAWDOWN_DISTRO_DTYPE)}
        ins = L.DrawdownInStruct(*[L.ptr(a) for a in arrs])
        st = L.HostTermOutStruct(L.ptr(o["hosts"]), L.ptr(o["distros"]))
        L.check(self.lib.evg_host_drawdown(self.ctx, C.byref(table.struct()), L.ptr(table.idle_off), C.byref(ins), int(now), C.byref(st)))
        return {"hosts": o["hosts"][:H], "distros": o["distros"][:D]}

    def idle_hosts(self, table: S.IdleHostTable, cfg: np.ndarray, now: int) -> dict:
        """evg_idle_hosts: idleHostJob.Run for every distro of `table`, on the device.  `cfg`: IDLE_CFG rows.
        -> dict of hosts (HOST_VERDICT rows) and distros (IDLE_DISTRO rows)."""
        D, H = table.n_distros, table.n_hosts
        cfg = np.ascontiguousarray(cfg, dtype=L.IDLE_CFG_DTYPE)
        if cfg.shape != (D,):
            raise ValueError("one setting per distro of the table")
        o = {"hosts": np.zeros(max(H, 1), L.HOST_VERDICT_DTYPE), "distros": np.zeros(max(D, 1), L.IDLE_DISTRO_DTYPE)}
        st = L.HostTermOutStruct(L.ptr(o["hosts"]), L.ptr(o["distros"]))
        L.check(self.lib.evg_idle_hosts(self.ctx, C.byref(table.struct()), L.ptr(table.idle_off),
                                        L.ptr(cfg if D else np.zeros(1, L.IDLE_CFG_DTYPE)), int(now), C.byref(st)))
        return {"hosts": o["hosts"][:H], "distros": o["distros"][:D]}

    def estimate_start_times(self, table: S.EstHostTable, now: int, cap: int = 0, task_off=None):
        """evg_estimate_start_times: GetEstimatedStartTime for every persisted rank of every distro of the resident tick
        after run(), on the device.  `table`: soa.marshal_estimate_hosts over the tick's distros; `cap`, `task_off` as
        download_queue.  -> (item_off, start_ns, hosts_used): start_ns[item_off[d] + r] is the estimate of rank r of
        distro d (-1: no hosts), hosts_used[d] the size of its host pool."""
        D = self._n_distros
        if table.n_distros != D:
            raise ValueError("one host list per distro of the resident tick")
        item_off = self._out("est_item_off", D + 1, np.int64)
        n = self._n_tasks if task_off is None else int(np.minimum(np.diff(task_off), cap or L.EVG_PERSISTED_QUEUE_CAP).sum())
        start = self._out("est_start", max(n, 1), np.int64)
        used = self._out("est_hosts_used", max(D, 1), np.int32)
        L.check(self.lib.evg_estimate_start_times(self.ctx, int(cap), C.byref(table.struct()), L.ptr(table.est_host_off), int(now),
                                                  L.ptr(item_off), L.ptr(start), int(max(n, 1)), L.ptr(used)))
        return item_off, start[: int(item_off[D])], used[:D]

    def estimate_start_batch(self, durations, item_off, table: S.EstHostTable, now: int):
        """evg_estimate_start_batch: the same for caller-supplied queues -- durations[item_off[d] .. item_off[d+1]) are
        the ExpectedDuration of distro d's queue items in order.  Needs no tick.  -> (start_ns, hosts_used)."""
        item_off = np.ascontiguousarray(item_off, dtype=np.int64)
        durations = np.ascontiguousarray(durations, dtype=np.int64)
        D = item_off.shape[0] - 1
        if table.n_distros != D or D < 0:
            raise ValueError("one host list per queue")
        n = int(durations.shape[0])
        start = np.zeros(max(n, 1), np.int64)
        used = np.zeros(max(D, 1), np.int32)
        L.check(self.lib.evg_estimate_start_batch(self.ctx, L.ptr(durations) if n else None, L.ptr(item_off), D, C.byref(table.struct()),
                                                  L.ptr(table.est_host_off), int(now), L.ptr(start), L.ptr(used)))
        return start[:n], used[:D]

    def alloc_batch(self, hosts: S.HostSoA, qinfo: np.ndarray, ginfo: np.ndarray, group_off: np.ndarray, now: int):
        D = int(qinfo.shape[0])
        ao = self._alloc_output(D)
        as_ = L.AllocOutStruct(L.ptr(ao.result), L.ptr(ao.status))
        hs = hosts.struct()
        qinfo = np.ascontiguousarray(qinfo, dtype=L.QUEUE_INFO_DTYPE)
        ginfo = np.ascontiguousarray(ginfo, dtype=L.GROUP_INFO_DTYPE)
        group_off = np.ascontiguousarray(group_off, dtype=np.int64)
        L.check(self.lib.evg_alloc_batch(self.ctx, C.byref(hs), L.ptr(hosts.host_off),
                                         L.ptr(hosts.cfg) if D else None, L.ptr(qinfo) if D else None,
                                         L.ptr(ginfo) if ginfo.shape[0] else None, L.ptr(group_off), D, int(now),
                                         C.byref(as_)))
        return ao, ginfo


_default_engine: Optional[Engine] = None


def default_engine() -> Engine:
    global _default_engine
    if _default_engine is None:
        _default_engine = Engine(0)
    return _default_engine


# ---------------------------------------------------------------------------
# reference-shaped API
# ---------------------------------------------------------------------------

@dataclass
class TaskPlannerOptions:  # scheduler/scheduler.go:18-23
    id: str = ""
    is_secondary_queue: bool = False
    includes_dependencies: bool = False
    started_at: int = M.ZERO_TIME


def _queue_info_from_rows(q, groups, names: Sequence[str]) -> M.DistroQueueInfo:
    infos: List[M.TaskGroupInfo] = []
    if int(q["has_ungrouped"]):
        u = q["ungrouped"]
        infos.append(M.TaskGroupInfo("", *[int(u[f]) for f in L.GROUP_INFO_FIELDS]))
    for name, g in zip(names, groups):
        infos.append(M.TaskGroupInfo(name, *[int(g[f]) for f in L.GROUP_INFO_FIELDS]))
    return M.DistroQueueInfo(
        length=int(q["length"]), length_with_dependencies_met=int(q["length_with_dependencies_met"]),
        count_dep_filled_merge_queue_tasks=int(q["count_dep_filled_merge_queue_tasks"]),
        expected_duration=int(q["expected_duration"]), max_duration_threshold=int(q["max_duration_threshold"]),
        count_duration_over_threshold=int(q["count_duration_over_threshold"]),
        duration_over_threshold=int(q["duration_over_threshold"]),
        count_wait_over_threshold=int(q["count_wait_over_threshold"]), task_group_infos=infos,
        secondary_queue=bool(q["secondary_queue"]))


def _upload_with_device_deps(eng: Engine, batch, soa, table, hosts, now: int, dependency_db) -> None:
    """Upload a marshalled tick and let the device evaluate Task.DependenciesMet (scheduler.go:161-168) for it; the
    DependenciesMetTime stamps it made are written back on the Task objects, like tasks[i] = task (scheduler.go:137)."""
    pairs = [(d, t) for d, t in ((b[0], b[1]) for b in batch)]
    eng.upload_with_deps(soa, table, hosts, S.marshal_deps(pairs, dependency_db), S.marshal_dep_finished(pairs), now)
    _, stamp = eng.download_deps()
    k = 0
    for _, tasks in pairs:
        for t in tasks:
            if int(stamp[k]) != M.ZERO_TIME:
                t.dependencies_met_time = int(stamp[k])
            k += 1


def _resolve_durations_on_device(eng: Engine, tasks: Sequence[M.Task], finished_tasks: Sequence[M.Task], now: int,
                                 datas: Optional[Sequence[M.HostAllocatorData]] = None,
                                 running_tasks: Optional[Dict[str, M.Task]] = None) -> None:
    """PopulateCaches' FetchExpectedDuration for every task of the resident tick (and the running task of every host
    that `running_tasks` holds) on the device, then the fields the reference leaves on those Task objects."""
    docs = list(running_tasks.values()) if running_tasks is not None else []
    hist, _ = S.marshal_duration_history(finished_tasks, (), now)
    tcache = S.marshal_duration_cache(tasks, hist)
    hcache, hdocs = (None, [])
    if running_tasks is not None and datas is not None and docs:
        hcache, hdocs = S.marshal_running_cache(datas, running_tasks, hist)
    eng.resolve_durations(hist, now, tcache, hcache)
    tout, hout = eng.download_durations()
    S.write_back_durations(tasks, tout)
    # a task several hosts run is resolved once per host, with the same inputs and result: write it back once
    seen = set()
    for i, t in enumerate(hdocs):
        if id(t) not in seen:
            seen.add(id(t))
            S.write_back_durations([t], {f: hout[f][i:i + 1] for f in L.DURATION_OUT_FIELDS})


def plan_distros(batch: Sequence[Tuple[M.Distro, List[M.Task]]], now: int, *, engine: Optional[Engine] = None,
                 dependency_db: Optional[Dict[str, M.Task]] = None, breakdown: bool = True,
                 secondary: bool = False, finished_tasks: Optional[Sequence[M.Task]] = None):
    """Batched runTunablePlanner minus persistence (scheduler/scheduler.go:34-51):
    returns, per distro, (ranked [Task] with SortingValueBreakdown stamped,
    DistroQueueInfo).  `finished_tasks`: the task history getExpectedDurationsForWindow reads; when given, every
    task's expected duration is resolved on the device against it (evg_resolve_durations) instead of on the host, and
    written back onto the Task objects as FetchExpectedDuration does."""
    eng = engine or default_engine()
    soa, table, keys = S.marshal_tasks(batch, now, dependency_db, resolve_durations=finished_tasks is None)
    _upload_with_device_deps(eng, batch, soa, table, None, now, dependency_db)
    if finished_tasks is not None:
        _resolve_durations_on_device(eng, [t for _, ts in batch for t in ts], finished_tasks, now)
    return _ranked_results(eng, batch, table, keys, now, breakdown, secondary)


def _ranked_results(eng: Engine, batch, table, keys, now: int, breakdown: bool, secondary: bool):
    """Run the resident tick and turn its outputs into plan_distros' result: per distro (ranked [Task], DistroQueueInfo)."""
    eng.run(now, L.EVG_OPT_BREAKDOWN if breakdown else 0)
    po, _ = eng.download(want_breakdown=breakdown, want_alloc=False)
    out = []
    for d, (distro, tasks) in enumerate(batch):
        a, b = int(table.task_off[d]), int(table.task_off[d + 1])
        ga, gb = int(table.group_off[d]), int(table.group_off[d + 1])
        ranked = []
        for r in range(a, b):
            t = tasks[int(po.order[r])]
            if breakdown:
                t.sorting_value_breakdown = M.SortingValueBreakdown.from_row(po.breakdown[r])  # planner.go:475
            else:
                t.sorting_value_breakdown = M.SortingValueBreakdown(total_value=int(po.total_value[r]))
            ranked.append(t)
        info = _queue_info_from_rows(po.info[d], po.group_info[ga:gb], keys[d].group_names)
        info.secondary_queue = secondary  # scheduler.go:44
        out.append((ranked, info))
    return out


class ResidentTick:
    """The tick-to-tick cache a shim keeps so that only changes cross PCIe: the last batch's marshalled columns, each
    distro's task ids in resident order and a map from task id to row.  plan() takes the next Go-level batch, derives
    the edit (tasks dispatched or gone, arrivals, the in-queue dependencies survivors gained, group and version ids
    remapped to what marshal_tasks assigns on the composed order) and the evg_update_tasks rows of changed scalars, runs
    the tick and returns what plan_distros returns.  A change an edit cannot express (another distro list, a survivor
    that moved task group or lost a dependency that stays queued) uploads the batch instead.

    Canonical input order: survivors in their previous order, then arrivals in batch order (input order reaches the
    output only through the tie policy, and the reference's is arbitrary).  Task.DependenciesMet is evaluated on the host
    for every task of the batch (soa.dependencies_met), so the inserted rows carry their bit and survivors whose verdict
    changed are updated.  The engine must not run other ticks between two plan() calls."""

    SCALARS = ("priority", "expected_ns", "queue_basis_ns", "wait_basis_ns", "num_dependents", "task_group_order", "flags")

    def __init__(self, engine: Optional[Engine] = None, dependency_db: Optional[Dict[str, M.Task]] = None):
        self.engine = engine  # None: default_engine() at the first plan()
        self.dependency_db = dependency_db
        self.distro_ids: Optional[List[str]] = None
        self.ids: List[List[str]] = []   # per distro: task ids in resident order
        self.row: Dict[str, int] = {}    # task id -> row of the resident table
        self.soa = self.table = self.keys = None
        self.last = None                 # (edit, update rows) of the last plan(), None when it uploaded
        self.ranked: List[List[str]] = []  # per distro: task ids in the last plan()'s rank order
        self._disp = None                # (item_off, group names per dense group) of the dispatchers being served

    def canonical(self, batch):
        """The batch in canonical order: survivors in their previous order, then arrivals in batch order."""
        if self.distro_ids is None or [d.id for d, _ in batch] != self.distro_ids:
            return [(d, list(ts)) for d, ts in batch]
        out = []
        for (d, ts), prev in zip(batch, self.ids):
            by_id = {t.id: t for t in ts}
            seen = set(prev)
            out.append((d, [by_id[i] for i in prev if i in by_id] + [t for t in ts if t.id not in seen]))
        return out

    def diff(self, canon, soa: S.TaskSoA, table: S.DistroTable, keys):
        """(edit, update rows, update values) that take the resident tick to the marshalled `canon`, or None when an
        edit cannot express the change."""
        if self.distro_ids is None or [d.id for d, _ in canon] != self.distro_ids:
            return None
        old, ot = self.soa, self.table
        remove, n_surv, new_pos = [], [], {}
        for d, ((_, ts), prev) in enumerate(zip(canon, self.ids)):
            ids = {t.id for t in ts}
            gone = [i for i in prev if i not in ids]
            remove.extend(self.row[i] for i in gone)
            n_surv.append(len(prev) - len(gone))
            for k, t in enumerate(ts):
                new_pos[(d, t.id)] = k
        D = table.n_distros
        toff = table.task_off
        n_surv = np.array(n_surv, dtype=np.int64)
        ins_rows = np.concatenate([np.arange(toff[d] + n_surv[d], toff[d + 1]) for d in range(D)] or [np.zeros(0, np.int64)]).astype(np.int64)
        ins_n = np.diff(toff) - n_surv
        cols = {name: getattr(soa, name)[ins_rows] for name, _ in S.TaskSoA.COLUMNS}
        dep_off = dep_idx = None
        if soa.n_edges:
            deg = soa.dep_off[ins_rows + 1] - soa.dep_off[ins_rows]
            dep_off = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
            dep_idx = np.concatenate([soa.dep_idx[soa.dep_off[r]:soa.dep_off[r + 1]] for r in ins_rows] or [np.zeros(0, np.int32)])
        # remaps by name: the ids marshal_tasks gave the composed order
        gremap, vremap = [], []
        for d in range(D):
            gnew = {n: g for g, n in enumerate(keys[d].group_names)}
            vnew = {n: v for v, n in enumerate(keys[d].versions)}
            gremap.extend(gnew.get(n, -1) for n in self.keys[d].group_names)
            vremap.extend(vnew.get(n, -1) for n in self.keys[d].versions)
        # edges survivors gained: their marshalled edges minus the old edges that survive (as a multiset, in order)
        add_task, add_dep = [], []
        for d, prev in enumerate(self.ids):
            a0 = int(ot.task_off[d])
            for k_old, tid in enumerate(prev):
                k_new = new_pos.get((d, tid))
                if k_new is None:
                    continue
                r_old, r_new = a0 + k_old, int(toff[d]) + k_new
                want = soa.dep_idx[soa.dep_off[r_new]:soa.dep_off[r_new + 1]].tolist() if soa.n_edges else []
                kept = []
                if old.n_edges:
                    for j in old.dep_idx[old.dep_off[r_old]:old.dep_off[r_old + 1]].tolist():
                        p = new_pos.get((d, prev[j]))
                        if p is not None:
                            kept.append(p)
                rest = list(want)
                for p in kept:
                    if p not in rest:
                        return None  # the survivor lost a dependency that is still queued
                    rest.remove(p)
                add_task.extend([r_new] * len(rest))
                add_dep.extend(rest)
        edit = S.TaskEdit(np.sort(np.array(remove, dtype=np.int64)), S.TaskSoA(**cols, dep_off=dep_off, dep_idx=dep_idx),
                          np.concatenate([[0], np.cumsum(ins_n)]).astype(np.int64), np.array(add_task, dtype=np.int64),
                          np.array(add_dep, dtype=np.int32), np.array(gremap, dtype=np.int32), np.array(vremap, dtype=np.int32),
                          table.group_off, table.group_max_hosts, table.cfg).normalize()
        if edit.group_remap.shape[0] == 0:
            edit.group_remap = None
        try:
            composed, _ = S.apply_edit(old, ot, edit)
        except ValueError:
            return None
        if not (np.array_equal(composed.group_id, soa.group_id) and np.array_equal(composed.version_id, soa.version_id)):
            return None  # a survivor changed task group or version
        changed = np.zeros(soa.n_tasks, dtype=bool)
        for name in self.SCALARS:
            changed |= getattr(composed, name) != getattr(soa, name)
        rows = np.nonzero(changed)[0].astype(np.int64)
        values = S.TaskSoA(**{name: getattr(soa, name)[rows] for name, _ in S.TaskSoA.COLUMNS})
        return edit, rows, values

    def plan(self, batch: Sequence[Tuple[M.Distro, List[M.Task]]], now: int, *, breakdown: bool = True, secondary: bool = False):
        """One tick: what plan_distros returns for the batch in canonical order (self.canonical)."""
        eng = self.engine = self.engine or default_engine()
        canon = self.canonical(batch)
        soa, table, keys = S.marshal_tasks(canon, now, self.dependency_db, resolve_deps=True)
        change = self.diff(canon, soa, table, keys)
        if change is None:
            eng.upload(soa, table)
        else:
            edit, rows, values = change
            eng.edit_tasks(edit, table)
            if rows.shape[0]:
                eng.update_tasks(rows, values)
        self.last = None if change is None else change[:2]
        self.remember(canon, soa, table, keys)
        res = _ranked_results(eng, canon, table, keys, now, breakdown, secondary)
        self.ranked = [[t.id for t in ranked] for ranked, _ in res]
        self._disp = None  # the run ended the last dispatchers
        return res

    def dispatchers(self, cap: int = 0):
        """The DAG dispatcher of every distro's persisted queue of the last plan(), built on the device from the tick
        (dispatchers_from_tick): what rebuild_dag_dispatchers returns for the queues persist_task_queues would save."""
        return dispatchers_from_tick(self.ranked, [k.group_names for k in self.keys], cap=cap, engine=self.engine)

    def find_next_tasks(self, requests, db: dict, cap: int = 0, rebuild: bool = False):
        """FindNextTask for `requests[d]` = distro d's (TaskSpec or None, amiUpdatedTime) in serving order, on the
        dispatchers of the last plan()'s persisted queues (evg_find_next_tasks).  The first call after a plan(), or
        rebuild=True, builds them (evg_rebuild_dispatchers, which starts from IsDispatched == false); later calls serve
        against the state the earlier ones left on the device.  -> per distro the task id (None for nil) and EVG_NEXT_*
        outcome of each request."""
        eng = self.engine
        if rebuild or self._disp is None:
            r = eng.rebuild_dispatchers(cap)
            io, go = r["item_off"].copy(), r["group_off"].copy()
            self._disp = (io, [[self.keys[d].group_names[int(g)] for g in r["group_slot"][int(go[d]):int(go[d + 1])]]
                               for d in range(len(self.ranked))])
        io, names = self._disp
        ids = [self.ranked[d][:int(io[d + 1] - io[d])] for d in range(len(self.ranked))]
        item, outcome = eng.find_next_tasks(S.marshal_next_db(ids, names, db), S.marshal_next_requests(names, requests))
        return _next_results(ids, requests, item, outcome)

    def estimated_start_times(self, hosts_by_distro: Sequence[Sequence[M.Host]], running_tasks: Dict[str, object], now: int, cap: int = 0):
        """GetEstimatedStartTime for every persisted task of the last plan(), chained on the tick (evg_estimate_start_times):
        hosts_by_distro[d] are the up hosts of distro d in query order, running_tasks as soa.marshal_estimate_hosts takes
        them.  -> per distro {task id: estimate in ns} over its persisted ranks (-1: the distro has no hosts); a task
        that is not there is not queued, for which the reference returns -1."""
        io, start, _ = self.engine.estimate_start_times(S.marshal_estimate_hosts(hosts_by_distro, running_tasks), now, cap, self.table.task_off)
        return [dict(zip(ids, start[int(io[d]):int(io[d + 1])].tolist())) for d, ids in enumerate(self.ranked)]

    def remember(self, canon, soa: S.TaskSoA, table: S.DistroTable, keys) -> None:
        """Make the marshalled `canon` the resident tick the next diff starts from."""
        self.soa, self.table, self.keys = soa, table, keys
        self.distro_ids = [d.id for d, _ in canon]
        self.ids = [[t.id for t in ts] for _, ts in canon]
        self.row = {}
        for d, ids in enumerate(self.ids):
            a = int(table.task_off[d])
            self.row.update((i, a + k) for k, i in enumerate(ids))


def persist_task_queues(batch: Sequence[Tuple[M.Distro, List[M.Task]]], now: int, *, engine: Optional[Engine] = None,
                        dependency_db: Optional[Dict[str, M.Task]] = None, cap: int = 0) -> List[M.TaskQueue]:
    """Batched PersistTaskQueue minus the upsert (scheduler/task_queue_persister.go:14-42, TaskQueue.Save
    model/task_queue.go:216-219): plan every distro, then build each distro's TaskQueue document from the
    TaskQueueItem rows the device projected for the first min(length, 10 000) ranks -- only those rows are copied
    back -- plus the strings of the shim's own Task objects.  Tasks are stamped like the reference leaves them
    (ExpectedDuration scheduler.go:98, DependenciesMetTime task.go:653, ScheduledTime / DependenciesMetTime
    task.go:1164-1195 at `now`)."""
    eng = engine or default_engine()
    soa, table, keys = S.marshal_tasks(batch, now, dependency_db)
    _upload_with_device_deps(eng, batch, soa, table, None, now, dependency_db)
    eng.run(now)
    po, _ = eng.download(want_alloc=False)
    item_off, items = eng.download_queue(cap, table.task_off)
    out = []
    for d, (distro, tasks) in enumerate(batch):
        ga, gb = int(table.group_off[d]), int(table.group_off[d + 1])
        info = _queue_info_from_rows(po.info[d], po.group_info[ga:gb], keys[d].group_names)
        queue = []
        for row in items[int(item_off[d]):int(item_off[d + 1])]:
            t = tasks[int(row["task"])]
            t.expected_duration = int(row["expected_ns"])
            t.sorting_value_breakdown = M.SortingValueBreakdown(total_value=int(row["total_value"]))
            queue.append(M.TaskQueueItem(
                id=t.id, display_name=t.display_name, build_variant=t.build_variant,
                revision_order_number=t.revision_order_number, requester=t.requester, revision=t.revision, project=t.project,
                expected_duration=int(row["expected_ns"]), priority=int(row["priority"]),
                sorting_value_breakdown=t.sorting_value_breakdown, group=t.task_group,
                group_max_hosts=t.task_group_max_hosts, group_index=int(row["group_index"]), version=t.version,
                activated_by=t.activated_by, dependencies=[dep.task_id for dep in t.depends_on],
                dependencies_met=bool(int(row["flags"]) & L.EVG_QI_DEPS_MET)))
        for t in tasks:  # SetTasksScheduledAndDepsMetTime (model/task/task.go:1164-1195), every prioritised task
            if M.is_zero_time(t.scheduled_time):
                t.scheduled_time = now
            if t.has_dependencies_met() and M.is_zero_time(t.dependencies_met_time):
                t.dependencies_met_time = now
        out.append(M.TaskQueue(distro=distro.id, generated_at=now, queue=queue, distro_queue_info=info))
    return out


def PersistTaskQueue(distro: M.Distro, tasks: List[M.Task], *, now: int, engine: Optional[Engine] = None,
                     dependency_db: Optional[Dict[str, M.Task]] = None) -> M.TaskQueue:
    """scheduler.PersistTaskQueue for one distro; the caller upserts the returned document."""
    return persist_task_queues([(distro, tasks)], now, engine=engine, dependency_db=dependency_db)[0]


def PlanDistro(distro: M.Distro, find_tasks, *, now: int, engine: Optional[Engine] = None,
               dependency_db: Optional[Dict[str, M.Task]] = None, existing_queue_length: int = 0):
    """scheduler.PlanDistro (scheduler/wrapper.go:30-130) without its Mongo calls: a disabled distro is not planned
    -- its persisted queue is cleared when it has one (wrapper.go:45-78; returns (None, True iff cleared)) --
    otherwise the task finder runs and the queue is planned and projected (returns (TaskQueue, False)).
    Unscheduling of stale tasks (underwaterUnschedule, wrapper.go:41) is a database update and stays with the caller."""
    if distro.disabled:
        return None, existing_queue_length > 0
    tasks = list(find_tasks(distro))
    return PersistTaskQueue(distro, tasks, now=now, engine=engine, dependency_db=dependency_db), False


def hosts_to_request(distro: M.Distro, info: M.DistroQueueInfo, n_provisioning_hosts: int, allocate) -> Tuple[int, int]:
    """The allocator call of hostAllocatorJob.Run (units/host_allocator.go:180-196): a single-task distro spawns one
    host per queued task whose dependencies are met, minus the hosts already provisioning (:182-184); every other distro
    asks the HostAllocator (`allocate()` -> (new_hosts, free_hosts))."""
    if distro.single_task_distro:
        return info.length_with_dependencies_met - n_provisioning_hosts, 0
    return allocate()


# cloud/ec2_util.go:63-67
BY_THE_SECOND_BILLING_OS = ("linux", "windows")
COMMERCIAL_LINUX_DISTROS = ("suse",)


def uses_hourly_billing(d: M.Distro) -> bool:
    """cloud.UsesHourlyBilling (cloud/ec2_util.go:256-268): billed by the hour unless the arch names a by-the-second OS,
    and always for a commercial Linux distro."""
    by_the_second = any(a in d.arch for a in BY_THE_SECOND_BILLING_OS)
    commercial = any(c in d.id for c in COMMERCIAL_LINUX_DISTROS)
    return not by_the_second or commercial


def host_job_results(distros: Sequence[M.Distro], res: dict) -> list:
    """Engine.host_job's arrays -> [(n_hosts, n_hosts_free, HostAllocatorJobReport | None, DrawdownInfo | None)]: the
    report is None when the allocator's error ended the job (units/host_allocator.go:192-195)."""
    out = []
    for i, d in enumerate(distros):
        n, f = int(res["n_hosts"][i]), int(res["n_hosts_free"][i])
        if int(res["status"][i]) != L.EVG_ALLOC_OK:
            out.append((n, f, None, None))
            continue
        r = res["report"][i]
        rep = M.HostAllocatorJobReport(
            time_to_empty=int(r["time_to_empty_ns"]), time_to_empty_no_spawns=int(r["time_to_empty_no_spawns_ns"]),
            scheduled_duration=int(r["scheduled_duration_ns"]), hosts_avail=int(r["hosts_avail"]),
            hosts_spawned=int(r["hosts_spawned"]), overdue_in_groups=int(r["overdue_in_groups"]),
            free_in_groups=int(r["free_in_groups"]), required_in_groups=int(r["required_in_groups"]),
            host_queue_ratio=float(r["host_queue_ratio"]), no_spawns_ratio=float(r["no_spawns_ratio"]),
            drawdown=bool(r["drawdown"]), new_cap_target=int(r["new_cap_target"]), killable_hosts=int(r["killable_hosts"]))
        out.append((n, f, rep, M.DrawdownInfo(d.id, rep.new_cap_target) if rep.drawdown else None))
    return out


def host_allocator_jobs(batch: Sequence[Tuple[M.Distro, List[M.Task], M.HostAllocatorData]], now: int, *,
                        n_provisioning: Sequence[int], spawned: Optional[Sequence[int]] = None,
                        engine: Optional[Engine] = None, dependency_db: Optional[Dict[str, M.Task]] = None) -> list:
    """hostAllocatorJob.Run for every distro of one tick (units/host_allocator.go:152-337, 394-425): the planner and
    the allocator as plan_and_allocate runs them, then the single-task bypass, the time-to-empty report and the
    drawdown decision on the device.  `n_provisioning[d]` = len(ProvisioningHosts()); `spawned[d]` = len(hostsSpawned)
    (None: what CreateIntentHosts creates without a container pool, max(n_hosts, 0)).  Returns, per distro,
    (n_hosts, n_hosts_free, HostAllocatorJobReport or None when the allocator failed, DrawdownInfo or None)."""
    eng = engine or default_engine()
    datas = [h for _, _, h in batch]
    soa, table, keys = S.marshal_tasks([(d, t) for d, t, _ in batch], now, dependency_db)
    hosts = S.marshal_hosts(datas, [k.group_names for k in keys])
    _upload_with_device_deps(eng, batch, soa, table, hosts, now, dependency_db)
    eng.run(now)
    res = eng.host_job(S.marshal_host_job(datas, n_provisioning), None if spawned is None else np.asarray(spawned))
    return host_job_results([d for d, _, _ in batch], res)


MAX_TEARDOWN_GROUP_THRESHOLD = 4 * M.MINUTE  # evergreen.MaxTeardownGroupThreshold (globals.go:348)


def termination_reason(v) -> str:
    """getTerminationReason's text (units/host_monitoring_idle_termination.go:258-283) for an EVG_HT_TERM_* verdict."""
    ds = M.go_duration_string
    code = int(v["decision"])
    if code == L.EVG_HT_TERM_OUTDATED_AMI:
        return "host has an outdated AMI"
    if code == L.EVG_HT_TERM_COMMUNICATION:
        return (f"host is idle or unreachable, communication time {ds(int(v['communication_ns']))} is over threshold time "
                f"{ds(int(v['threshold_ns']))}")
    if code == L.EVG_HT_TERM_IDLE:
        return f"host is idle or unreachable, idle time {ds(int(v['idle_ns']))} is over threshold time {ds(int(v['threshold_ns']))}"
    assert code == L.EVG_HT_TERM_TEARDOWN, code
    return (f"time since the host's task group teardown start time {ds(int(v['since_teardown_ns']))} has exceeded the maximum "
            f"teardown threshold {ds(MAX_TEARDOWN_GROUP_THRESHOLD)}")


_HT_ERRORS = {L.EVG_HT_ERR_CLOUD_MANAGER: "getting cloud manager for host",  # what each job wraps its errors in
              L.EVG_HT_ERR_TASK_LOOKUP: "checking if host is running single host task group"}  # host_drawdown.go:140
_IDLE_ERRORS = dict(_HT_ERRORS)
_IDLE_ERRORS[L.EVG_HT_ERR_TASK_LOOKUP] = "getting information on idle host"  # host_monitoring_idle_termination.go:170


def host_drawdown_jobs(distro_ids: Sequence[str], idle_hosts: Sequence[Sequence[M.Host]], existing_host_counts: Sequence[int],
                       now: int, *, drawdown: Optional[Sequence[Optional[M.DrawdownInfo]]] = None,
                       queue_lengths: Optional[Sequence[int]] = None, engine: Optional[Engine] = None) -> list:
    """hostDrawdownJob.Run (units/host_drawdown.go:70-159) for every distro on the device.  `idle_hosts[d]`: the
    distro's IdleHostsWithDistroID, in order; `existing_host_counts[d]`: CountHostsCanOrWillRunTasksInDistro.
    Standalone: `drawdown[d]` is the job's DrawdownInfo (None: no job) and `queue_lengths[d]` the distro's
    LengthWithDependenciesMet.  Chained (both None): the drawdowns the engine's last host_allocator_jobs / host_job
    decided, with the tick's queue lengths.  Returns a HostDrawdownJob per distro, None where no job ran."""
    eng = engine or default_engine()
    table = S.marshal_idle_hosts(idle_hosts)
    cap = qlen = None
    if drawdown is not None or queue_lengths is not None:
        if drawdown is None or queue_lengths is None:
            raise ValueError("drawdown and queue_lengths: both or neither")
        cap = [L.EVG_NO_DRAWDOWN if x is None else int(x.new_cap_target) for x in drawdown]
        qlen = list(queue_lengths)
    res = eng.host_drawdown(table, existing_host_counts, now, cap, qlen)
    out, v = [], res["hosts"]
    for d, did in enumerate(distro_ids):
        r = res["distros"][d]
        if not r["ran"]:
            out.append(None)
            continue
        a, b = int(table.idle_off[d]), int(table.idle_off[d + 1])
        existing = int(existing_host_counts[d])
        job = M.HostDrawdownJob(did, existing - int(r["target"]), existing, b - a, int(r["target"]))
        for i in range(a, b):
            code = int(v[i]["decision"])
            if code == L.EVG_HT_DECOMMISSION:
                job.decommissioned_hosts.append(table.ids[i])
            elif code in _HT_ERRORS:
                job.errors.append((table.ids[i], _HT_ERRORS[code]))
        assert job.decommissioned == int(r["decommissioned"])
        out.append(job)
    return out


def idle_host_jobs(distros: Sequence[Optional[M.Distro]], idle_hosts: Sequence[Sequence[M.Host]], running_hosts_counts: Sequence[int],
                   now: int, *, acceptable_host_idle_time_seconds: int = 0, engine: Optional[Engine] = None) -> list:
    """idleHostJob.Run (units/host_monitoring_idle_termination.go:64-140) for every distro on the device.
    `distros[d]`: the distro document, None when it is missing from the collection (evaluated as the zero distro);
    `idle_hosts[d]`: its IdleEphemeralGroupedByDistroID hosts by ascending CreationTime; `running_hosts_counts[d]`: the
    aggregation's RunningHostsCount.  Returns an IdleHostJob per distro."""
    eng = engine or default_engine()
    zero = M.Distro()
    ds = [zero if d is None else d for d in distros]
    table = S.marshal_idle_hosts(idle_hosts, [d.default_ami for d in ds])
    cfg = np.zeros(len(ds), L.IDLE_CFG_DTYPE)
    for i, (d, n) in enumerate(zip(ds, running_hosts_counts)):
        idle = d.host_allocator_settings.acceptable_host_idle_time
        cfg[i] = (d.host_allocator_settings.minimum_hosts, int(n),
                  idle if idle != 0 else int(acceptable_host_idle_time_seconds) * M.SECOND)  # getIdleInfo (:197-200)
    res = eng.idle_hosts(table, cfg, now)
    out, v = [], res["hosts"]
    for d, did in enumerate(distros):
        a, b = int(table.idle_off[d]), int(table.idle_off[d + 1])
        job = M.IdleHostJob("" if did is None else did.id, b - a, int(res["distros"][d]["min_evaluate"]))
        for i in range(a, b):
            code = int(v[i]["decision"])
            if code >= L.EVG_HT_TERM_OUTDATED_AMI:
                job.terminated_hosts.append(table.ids[i])
                job.reasons.append(termination_reason(v[i]))
            elif code in _IDLE_ERRORS:
                job.errors.append((table.ids[i], _IDLE_ERRORS[code]))
        assert job.terminated == int(res["distros"][d]["terminated"])
        out.append(job)
    return out


def PrioritizeTasks(d: M.Distro, tasks: List[M.Task], opts: Optional[TaskPlannerOptions] = None, *, now: int,
                    engine: Optional[Engine] = None, dependency_db: Optional[Dict[str, M.Task]] = None):
    """scheduler.PrioritizeTasks (scheduler/scheduler.go:27-32) for one distro.
    Returns (plan, DistroQueueInfo); the reference persists the info instead
    of returning it (scheduler.go:43-48)."""
    opts = opts or TaskPlannerOptions()
    (plan, info), = plan_distros([(d, tasks)], now, engine=engine, dependency_db=dependency_db,
                                 secondary=opts.is_secondary_queue)
    info.plan_created_at = opts.started_at
    return plan, info


def GetDistroQueueInfo(distro: M.Distro, tasks: List[M.Task], max_duration_threshold: int,
                       opts: Optional[TaskPlannerOptions] = None, *, now: int, engine: Optional[Engine] = None,
                       dependency_db: Optional[Dict[str, M.Task]] = None) -> M.DistroQueueInfo:
    """scheduler.GetDistroQueueInfo (scheduler/scheduler.go:56-159).  Every
    quantity is a commutative sum, so the plan order does not matter."""
    opts = opts or TaskPlannerOptions()
    import copy
    d = copy.deepcopy(distro)
    d.planner_settings.target_time = max_duration_threshold
    d.dispatcher_settings.version = (M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES
                                     if opts.includes_dependencies else "")
    eng = engine or default_engine()
    soa, table, keys = S.marshal_tasks([(d, tasks)], now, dependency_db)
    _upload_with_device_deps(eng, [(d, tasks)], soa, table, None, now, dependency_db)
    eng.run(now)
    po, _ = eng.download(want_alloc=False)
    info = _queue_info_from_rows(po.info[0], po.group_info, keys[0].group_names)
    return info


def dependencies_met(batch: Sequence[Tuple[M.Distro, List[M.Task]]], *, engine: Optional[Engine] = None,
                     dependency_db: Optional[Dict[str, M.Task]] = None) -> List[List[bool]]:
    """Task.DependenciesMet (model/task/task.go:632-671) for every queued task, per distro: the predicate the
    task finders filter on and the bit the planner takes as EVG_TF_DEPS_MET."""
    eng = engine or default_engine()
    met = eng.deps_met_batch(S.marshal_deps(batch, dependency_db))
    out, a = [], 0
    for _, tasks in batch:
        out.append([bool(x) for x in met[a:a + len(tasks)]])
        a += len(tasks)
    return out


def find_runnable_tasks(batch: Sequence[Tuple[M.Distro, List[M.Task]]], project_refs: Sequence[M.ProjectRef], *,
                        finder: str = "legacy", dependency_db: Optional[Dict[str, M.Task]] = None,
                        engine: Optional[Engine] = None) -> List[List[M.Task]]:
    """LegacyFindRunnableTasks / AlternateTaskFinder / ParallelTaskFinder (scheduler/task_finder.go:40-317) or
    RunnableTasksPipeline (finder="pipeline", :34-36) for every distro of the tick: `batch` holds each distro's
    candidates (the rows the tasks collection has for it), the result the tasks each finder returns, in candidate order.
    The pipeline returns the candidates themselves here; pipeline_returned_tasks gives them as the aggregation decodes them."""
    eng = engine or default_engine()
    table = S.marshal_runnable(batch, project_refs, finder, dependency_db)
    runnable, count = eng.find_runnable_batch(table)
    out = []
    for i, (_, tasks) in enumerate(batch):
        a = int(table.task_off[i])
        out.append([tasks[int(j)] for j in runnable[a:a + int(count[i])]])
    return out


def plan_candidates(batch: Sequence[Tuple[M.Distro, List[M.Task]]], project_refs: Sequence[M.ProjectRef], now: int, *,
                    finder: str = "legacy", dependency_db: Optional[Dict[str, M.Task]] = None,
                    engine: Optional[Engine] = None):
    """The finder -> checkDependenciesMet -> PrioritizeTasks hand-over of scheduler.PlanDistro (wrapper.go:60-118,
    scheduler.go:56-168) without the host in the middle: `batch` holds every distro's CANDIDATES; the device filters them,
    evaluates their dependencies, compacts the planner's columns and plans (evg_plan_from_finder; finder="pipeline":
    evg_plan_from_finder_ex, which plans the kept tasks as pipeline_returned_tasks gives them).  Returns, per distro,
    (ranked kept tasks with TotalValue stamped, DistroQueueInfo)."""
    eng = engine or default_engine()
    table = S.marshal_runnable(batch, project_refs, finder, dependency_db)
    if table.deps is None:
        table.deps = S.marshal_deps(batch, dependency_db)
    soa, dtable, keys = S.marshal_tasks(batch, now, dependency_db)
    runnable, count = eng.plan_from_finder(table, soa, dtable, None, S.marshal_dep_finished(batch), now)
    eng.run(now)
    po, _ = eng.download(want_alloc=False)
    out, a_new = [], 0
    for d, (_, tasks) in enumerate(batch):
        a = int(table.task_off[d])
        kept = [tasks[int(j)] for j in runnable[a:a + int(count[d])]]
        ranked = []
        for r in range(a_new, a_new + len(kept)):
            t = kept[int(po.order[r])]
            t.sorting_value_breakdown = M.SortingValueBreakdown(total_value=int(po.total_value[r]))
            ranked.append(t)
        a_new += len(kept)
        ga, gb = int(dtable.group_off[d]), int(dtable.group_off[d + 1])
        out.append((ranked, _queue_info_from_rows(po.info[d], po.group_info[ga:gb], keys[d].group_names)))
    return out


def find_host_schedulable_for_alias(distro_id: str, tasks: Sequence[M.Task], distros: Sequence[M.Distro]) -> List[M.Task]:
    """task.FindHostSchedulableForAlias (model/task/task.go:3371-3386) over the tasks collection `tasks`, in its order:
    schedulableHostTasksQuery (model/task/db.go:671-689), TaskGroupMaxHosts != 1, and some SecondaryDistros name in
    FindApplicableDistroIDs(distro_id) = {distro_id} U Aliases (model/distro/aliases.go:14-27), looked up in `distros`."""
    d = next((x for x in distros if x.id == distro_id), None)
    if d is None:
        raise LookupError(f"error finding distro '{distro_id}'")  # aliases.go:20-22
    applicable = {d.id, *d.aliases}
    out = []
    for t in tasks:
        if not (t.activated and t.status == M.TASK_UNDISPATCHED and t.priority > M.DISABLED_TASK_PRIORITY and
                t.execution_platform in ("", "host")):
            continue
        if t.unattainable_dependency and not t.override_dependencies:
            continue
        if t.task_group_max_hosts == 1:  # single-host task groups stay out of alias queues (task.go:3379-3382)
            continue
        if any(name in applicable for name in t.secondary_distros):
            out.append(t)
    return out


def _plan_aliases(eng: Engine, distros, tasks, now: int, dependency_db):
    """evg_plan_aliases over the tick -> (task_off, group_off, source row of every resident row, group names per slot)."""
    table, cfg, keys = S.marshal_aliases(distros, tasks, now, dependency_db)
    task_off, group_off, _ = eng.plan_aliases(table, cfg, now)
    src, gsrc = (a.copy() for a in eng.download_alias_map())
    return task_off, group_off, src, [keys.group_names[int(g)] for g in gsrc]


def plan_alias_queues(distros: Sequence[M.Distro], tasks: Sequence[M.Task], now: int, *, engine: Optional[Engine] = None,
                      dependency_db: Optional[Dict[str, M.Task]] = None, breakdown: bool = False,
                      started_at: int = M.ZERO_TIME):
    """distroAliasSchedulerJob.Run for every distro at once, without Mongo (units/scheduler_alias.go:55-117): the tick's
    schedulable `tasks` (each once) fan out to the alias queues on the device (evg_plan_aliases), which are planned
    with IsSecondaryQueue (scheduler/scheduler.go:27-51).  Returns, per distro, (ranked [Task] with
    SortingValueBreakdown stamped -- shallow copies: a task in several queues has one TotalValue in each --
    DistroQueueInfo with secondary_queue and plan_created_at set)."""
    import copy
    eng = engine or default_engine()
    task_off, group_off, src, names = _plan_aliases(eng, distros, tasks, now, dependency_db)
    eng.run(now, L.EVG_OPT_BREAKDOWN if breakdown else 0)
    po, _ = eng.download(want_breakdown=breakdown, want_alloc=False)
    out = []
    for d in range(len(distros)):
        a, b = int(task_off[d]), int(task_off[d + 1])
        ga, gb = int(group_off[d]), int(group_off[d + 1])
        ranked = []
        for r in range(a, b):
            t = copy.copy(tasks[int(src[a + int(po.order[r])])])
            if breakdown:
                t.sorting_value_breakdown = M.SortingValueBreakdown.from_row(po.breakdown[r])
            else:
                t.sorting_value_breakdown = M.SortingValueBreakdown(total_value=int(po.total_value[r]))
            ranked.append(t)
        info = _queue_info_from_rows(po.info[d], po.group_info[ga:gb], names[ga:gb])
        info.secondary_queue = True  # scheduler.go:44
        info.plan_created_at = started_at
        out.append((ranked, info))
    return out


def persist_alias_task_queues(distros: Sequence[M.Distro], tasks: Sequence[M.Task], now: int, *, engine: Optional[Engine] = None,
                              dependency_db: Optional[Dict[str, M.Task]] = None, cap: int = 0) -> List[M.TaskQueue]:
    """persist_task_queues for the alias queues: every distro's secondary TaskQueue document (TaskQueue.collection() is
    the alias queues' collection) from the TaskQueueItem rows evg_download_queue projects on the device."""
    eng = engine or default_engine()
    task_off, group_off, src, names = _plan_aliases(eng, distros, tasks, now, dependency_db)
    eng.run(now)
    po, _ = eng.download(want_alloc=False)
    item_off, items = eng.download_queue(cap, task_off)
    out = []
    for d, distro in enumerate(distros):
        a, ga, gb = int(task_off[d]), int(group_off[d]), int(group_off[d + 1])
        info = _queue_info_from_rows(po.info[d], po.group_info[ga:gb], names[ga:gb])
        info.secondary_queue = True
        queue = []
        for row in items[int(item_off[d]):int(item_off[d + 1])]:
            t = tasks[int(src[a + int(row["task"])])]
            t.expected_duration = int(row["expected_ns"])
            queue.append(M.TaskQueueItem(
                id=t.id, display_name=t.display_name, build_variant=t.build_variant,
                revision_order_number=t.revision_order_number, requester=t.requester, revision=t.revision, project=t.project,
                expected_duration=int(row["expected_ns"]), priority=int(row["priority"]),
                sorting_value_breakdown=M.SortingValueBreakdown(total_value=int(row["total_value"])), group=t.task_group,
                group_max_hosts=t.task_group_max_hosts, group_index=int(row["group_index"]), version=t.version,
                activated_by=t.activated_by, dependencies=[dep.task_id for dep in t.depends_on],
                dependencies_met=bool(int(row["flags"]) & L.EVG_QI_DEPS_MET)))
        out.append(M.TaskQueue(distro=distro.id, generated_at=now, queue=queue, distro_queue_info=info))
    return out


def LegacyFindRunnableTasks(d: M.Distro, candidates: List[M.Task], project_refs: Sequence[M.ProjectRef], **kw) -> List[M.Task]:
    """scheduler/task_finder.go:40-106 for one distro."""
    return find_runnable_tasks([(d, candidates)], project_refs, finder="legacy", **kw)[0]


def AlternateTaskFinder(d: M.Distro, candidates: List[M.Task], project_refs: Sequence[M.ProjectRef], **kw) -> List[M.Task]:
    """scheduler/task_finder.go:108-197 for one distro."""
    return find_runnable_tasks([(d, candidates)], project_refs, finder="alternate", **kw)[0]


def ParallelTaskFinder(d: M.Distro, candidates: List[M.Task], project_refs: Sequence[M.ProjectRef], **kw) -> List[M.Task]:
    """scheduler/task_finder.go:199-317 for one distro (it filters as AlternateTaskFinder does)."""
    return find_runnable_tasks([(d, candidates)], project_refs, finder="parallel", **kw)[0]


def RunnableTasksPipeline(d: M.Distro, candidates: List[M.Task], project_refs: Sequence[M.ProjectRef], **kw) -> List[M.Task]:
    """scheduler/task_finder.go:34-36 (task.FindHostRunnable, model/task/db.go:887-1066) for one distro, the tasks as
    the aggregation returns them (pipeline_returned_tasks).  `project_refs` are the raw project_ref documents; the
    distro's ValidProjects must be those of its stored document ([] when there is none)."""
    return pipeline_returned_tasks(d, find_runnable_tasks([(d, candidates)], project_refs, finder="pipeline", **kw)[0])


def GetTaskFinder(version: str):
    """scheduler/task_finder.go:19-32: the finder of FinderSettings.Version; an unknown name falls back to legacy."""
    return {"parallel": ParallelTaskFinder, "legacy": LegacyFindRunnableTasks, "pipeline": RunnableTasksPipeline,
            "alternate": AlternateTaskFinder}.get(version, LegacyFindRunnableTasks)


def pipeline_returned_tasks(d: M.Distro, kept: Sequence[M.Task]) -> List[M.Task]:
    """The pipeline finder's kept tasks as PlanDistro receives them (copies):
    - with removeDeps (the distro is not revised-with-dependencies): DependsOn is empty.  $first: $$ROOT after
      $unwind depends_on leaves one sub-document, which mgo skips when it decodes into []Dependency;
    - otherwise: every DependsOn entry without Unattainable ($project of db.go:916-921)."""
    import copy
    out = []
    remove_deps = d.dispatcher_settings.version != M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES
    for t in kept:
        c = copy.copy(t)
        c.depends_on = [] if remove_deps else [M.Dependency(x.task_id, x.status, False, x.finished_at) for x in t.depends_on]
        out.append(c)
    return out


def get_expected_durations_for_window(tasks: Sequence[M.Task], window_start: int, window_end: int, *,
                                      engine: Optional[Engine] = None) -> Dict[tuple, Tuple[float, float]]:
    """getExpectedDurationsForWindow (model/task/expected_duration.go:36-96) for every (project, build variant) at
    once: {(project, build_variant, display_name): (exp_dur ns, std_dev ns)} over the finished tasks given; keys
    whose rows all fail the $match are absent, as they are from the aggregation's result."""
    eng = engine or default_engine()
    rows, keys = S.marshal_durations(tasks, window_start, window_end)
    stats = eng.expected_durations_batch(rows)
    return {k: (float(stats["mean_ns"][i]), float(stats["stddev_ns"][i])) for i, k in enumerate(keys) if stats["count"][i] > 0}


def allocate_distros(datas: Sequence[M.HostAllocatorData], now: int, *, engine: Optional[Engine] = None):
    """Batched UtilizationBasedHostAllocator: [(new_hosts, free_hosts, status)].
    Mutates each DistroQueueInfo.TaskGroupInfos[i].CountFree/CountRequired like
    the reference (utilization_based_host_allocator.go:107-110)."""
    eng = engine or default_engine()
    qrows, grows, goff, names = S.queue_info_rows([d.distro_queue_info for d in datas])
    hosts = S.marshal_hosts(datas, names)
    ao, ginfo = eng.alloc_batch(hosts, qrows, grows, goff, now)
    out = []
    for i, data in enumerate(datas):
        st = int(ao.status[i])
        if st == L.EVG_ALLOC_OK:
            lookup = {n: k for k, n in enumerate(names[i])}
            for g in data.distro_queue_info.task_group_infos:
                k = lookup.get(g.name)
                if k is not None:
                    row = ginfo[int(goff[i]) + k]
                    g.count_free, g.count_required = int(row["count_free"]), int(row["count_required"])
        out.append((int(ao.result[i]["new_hosts"]), int(ao.result[i]["free_hosts"]), st))
    return out


def UtilizationBasedHostAllocator(data: M.HostAllocatorData, *, now: int, engine: Optional[Engine] = None):
    """HostAllocator (scheduler/host_allocator.go:15): (newHostsNeeded, estimatedFreeHosts) or raises."""
    (n, f, st), = allocate_distros([data], now, engine=engine)
    if st != L.EVG_ALLOC_OK:
        raise AllocatorError(st, data.distro.id)
    return n, f


HostAllocator = Callable[..., Tuple[int, int]]


def GetHostAllocator(name: str) -> HostAllocator:
    """scheduler.GetHostAllocator (scheduler/host_allocator.go:25-32): every name resolves to the utilization allocator."""
    return UtilizationBasedHostAllocator


def plan_and_allocate(batch: Sequence[Tuple[M.Distro, List[M.Task], M.HostAllocatorData]], now: int, *,
                      engine: Optional[Engine] = None, dependency_db: Optional[Dict[str, M.Task]] = None,
                      finished_tasks: Optional[Sequence[M.Task]] = None, running_tasks: Optional[Dict[str, M.Task]] = None):
    """The fused tick: distroSchedulerJob + hostAllocatorJob for every distro
    (units/scheduler.go:57-87, units/host_allocator.go:76-196) in one call; the
    queue info stays on the device between the two halves.  `finished_tasks` as for plan_distros; `running_tasks`
    (task id -> Task, the documents task.Find(ByIds) returns for the hosts' running tasks, allocator.go:337) have their
    expected durations resolved on the device too (allocator.go:357-359) and written back.  Both need
    finished_tasks; None keeps the host's resolution."""
    if running_tasks is not None and finished_tasks is None:
        raise ValueError("running_tasks are resolved against finished_tasks")
    eng = engine or default_engine()
    datas = [h for _, _, h in batch]
    soa, table, keys = S.marshal_tasks([(d, t) for d, t, _ in batch], now, dependency_db,
                                       resolve_durations=finished_tasks is None)
    hosts = S.marshal_hosts(datas, [k.group_names for k in keys], running_tasks)
    _upload_with_device_deps(eng, batch, soa, table, hosts, now, dependency_db)
    if finished_tasks is not None:
        _resolve_durations_on_device(eng, [t for _, ts, _ in batch for t in ts], finished_tasks, now, datas, running_tasks)
    eng.run(now)
    po, ao = eng.download()
    out = []
    for i, (distro, tasks, _) in enumerate(batch):
        a, b = int(table.task_off[i]), int(table.task_off[i + 1])
        ga, gb = int(table.group_off[i]), int(table.group_off[i + 1])
        ranked = [tasks[int(po.order[r])] for r in range(a, b)]
        info = _queue_info_from_rows(po.info[i], po.group_info[ga:gb], keys[i].group_names)
        out.append((ranked, info, int(ao.result[i]["new_hosts"]), int(ao.result[i]["free_hosts"]), int(ao.status[i])))
    return out


# ---------------------------------------------------------------------------------------------------------------
class NotDecomposableError(Exception):
    """The legacy comparator chain is not a strict weak order on some list of the distro (commit builds of several
    projects in one list, zero and non-zero expected durations mixed, two task groups whose "BuildId-TaskGroup"
    strings are equal): the reference's result then depends on the exact steps of Go's sort.Stable, which the default
    prioritiser does not reproduce.  The order it did compute is attached.  CmpBasedTaskPrioritizer(exact=True)
    replays sort.Stable on such lists and never raises this."""

    def __init__(self, distro_id: str, tasks):
        super().__init__(f"distro {distro_id!r}: the comparator chain is not a strict weak order on this queue")
        self.tasks = tasks


class CmpBasedTaskPrioritizer:
    """scheduler.TaskPrioritizer (scheduler/task_prioritizer.go:20-25) implemented by the legacy comparator
    prioritiser on the GPU.  PrioritizeTasks returns (tasks in run order, orderingLogic, error) like the reference;
    orderingLogic -- the reference's map of per-comparison reason strings -- is always empty here.
    exact=True: lists on which the chain is not a strict weak order are sorted by a replay of Go's sort.Stable
    (EVG_LEGACY_MODE_GO_STABLE), so every queue gets the reference's order and PrioritizeTasks never returns
    NotDecomposableError."""

    def __init__(self, runtime_id: str = "", engine: Optional[Engine] = None, now: Optional[int] = None, exact: bool = False):
        self.runtime_id = runtime_id
        self.engine = engine
        self.now = now
        self.exact = exact

    def prioritize_batch(self, batch):
        """(distro_id, tasks, versions) per distro -> list of (sorted tasks, status)."""
        eng = self.engine or default_engine()
        table = S.marshal_legacy(batch, self.now, exact=self.exact)
        order, count, status = eng.prioritize_legacy_batch(table)
        out = []
        for d, (_, tasks, _) in enumerate(batch):
            a = int(table.task_off[d])
            out.append(([tasks[int(i)] for i in order[a:a + int(count[d])]], int(status[d])))
        return out

    def PrioritizeTasks(self, distro_id: str, tasks, versions=None):
        (sorted_tasks, status), = self.prioritize_batch([(distro_id, list(tasks), versions)])
        if status != L.EVG_LEGACY_OK:
            return None, None, NotDecomposableError(distro_id, sorted_tasks)
        return sorted_tasks, {}, None


# ---------------------------------------------------------------------------------------------------------------
def estimated_start_times(queues: Sequence[Optional[M.TaskQueue]], hosts_by_distro: Sequence[Sequence[M.Host]],
                          running_tasks: Dict[str, object], now: int, *, engine: Optional[Engine] = None) -> List[List[int]]:
    """model.GetEstimatedStartTime (model/task_start_estimation.go:99-122) for every item of every queue in one call
    (evg_estimate_start_batch): queues[d] is a distro's TaskQueue document (None: there is none), hosts_by_distro[d] its
    up hosts in query order; running_tasks as soa.marshal_estimate_hosts takes them.  -> per queue the estimate in ns of
    each item, -1 without hosts."""
    eng = engine or default_engine()
    durations = [[it.expected_duration for it in q.queue] if q is not None else [] for q in queues]
    off = np.zeros(len(queues) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in durations])
    start, _ = eng.estimate_start_batch(np.array([v for x in durations for v in x], dtype=np.int64), off,
                                        S.marshal_estimate_hosts(hosts_by_distro, running_tasks), now)
    return [start[int(off[d]):int(off[d + 1])].tolist() for d in range(len(queues))]


def get_estimated_start_time(task: M.Task, queue: Optional[M.TaskQueue], hosts: Sequence[M.Host], running_tasks: Dict[str, object],
                             now: int, *, engine: Optional[Engine] = None) -> int:
    """model.GetEstimatedStartTime for one task: `queue` is the task's distro's queue (None: no document), `hosts` the
    distro's up hosts.  -1 when there is no queue or the task is not in it (:104-116), neither of which reaches the
    device."""
    if queue is None:
        return -1
    pos = next((i for i, it in enumerate(queue.queue) if it.id == task.id), -1)
    if pos == -1:
        return -1
    return estimated_start_times([queue], [hosts], running_tasks, now, engine=engine)[0][pos]


def rebuild_dag_dispatchers(queues: Sequence[M.TaskQueue], *, engine: Optional[Engine] = None):
    """basicCachedDAGDispatcherImpl.rebuild for a batch of persisted queues (model/task_queue_service_dependency.go:
    153-252).  Per queue: (sorted item ids with None for each dependency cycle's placeholder, number of cycles,
    {composite group id: [item ids by GroupIndex]})."""
    eng = engine or default_engine()
    io, go, dep_off, dep_item, group_id, group_index, names = S.dag_input_from_queues(queues)
    srt, n_sorted, n_cycles, unit_items, unit_off = eng.dag_rebuild_batch(io, go, dep_off, dep_item, group_id, group_index)
    out = []
    for d, q in enumerate(queues):
        b = int(io[d])
        order = [None if int(i) < 0 else q.queue[int(i)].id for i in srt[b:b + int(n_sorted[d])]]
        u = int(go[d]) + d
        units = {name: [q.queue[int(i)].id for i in unit_items[b + int(unit_off[u + g]):b + int(unit_off[u + g + 1])]]
                 for g, name in enumerate(names[d])}
        out.append((order, int(n_cycles[d]), units))
    return out


def dispatchers_from_tick(ranked_ids: Sequence[Sequence[str]], group_names: Sequence[Sequence[str]], *, cap: int = 0,
                          engine: Optional[Engine] = None):
    """What rebuild_dag_dispatchers returns for the queues PersistTaskQueue would save from the engine's resident tick
    (after run()), built on the device: the queues never cross PCIe (evg_rebuild_dispatchers).  `ranked_ids[d]` holds
    distro d's task ids in rank order (at least its persisted head: what plan_distros / ResidentTick.plan /
    plan_alias_queues return), `group_names[d]` the name of each of its group slots (marshal_tasks' keys[d].group_names:
    Task.GetTaskGroupString has compositeGroupID's format)."""
    eng = engine or default_engine()
    r = eng.rebuild_dispatchers(cap)
    io, go = r["item_off"], r["group_off"]
    out = []
    for d, (ids, names) in enumerate(zip(ranked_ids, group_names)):
        b, u = int(io[d]), int(go[d]) + d
        order = [None if int(i) < 0 else ids[int(i)] for i in r["sorted"][b:b + int(r["n_sorted"][d])]]
        units = {names[int(r["group_slot"][int(go[d]) + g])]:
                 [ids[int(i)] for i in r["unit_items"][b + int(r["unit_off"][u + g]):b + int(r["unit_off"][u + g + 1])]]
                 for g in range(int(go[d + 1] - go[d]))}
        out.append((order, int(r["n_cycles"][d]), units))
    return out


def alias_dispatchers(distros: Sequence[M.Distro], tasks: Sequence[M.Task], now: int, *, engine: Optional[Engine] = None,
                      dependency_db: Optional[Dict[str, M.Task]] = None, cap: int = 0):
    """The DAG dispatcher of every distro's alias queue: evg_plan_aliases, the run, then evg_rebuild_dispatchers on the
    secondary queues persist_alias_task_queues would save.  Per distro what rebuild_dag_dispatchers returns for them."""
    eng = engine or default_engine()
    task_off, group_off, src, names = _plan_aliases(eng, distros, tasks, now, dependency_db)
    eng.run(now)
    po, _ = eng.download(want_alloc=False)
    ranked = [[tasks[int(src[int(task_off[d]) + int(i)])].id for i in po.order[int(task_off[d]):int(task_off[d + 1])]]
              for d in range(len(distros))]
    return dispatchers_from_tick(ranked, [names[int(group_off[d]):int(group_off[d + 1])] for d in range(len(distros))],
                                 cap=cap, engine=eng)


# ---------------------------------------------------------------------------------------------------------------
def _next_results(ids, requests, item, outcome):
    out, r = [], 0
    for d, reqs in enumerate(requests):
        out.append([(ids[d][int(item[r + k])] if item[r + k] >= 0 else None, int(outcome[r + k])) for k in range(len(reqs))])
        r += len(reqs)
    return out


def next_dispatchers(queues: Sequence[M.TaskQueue], *, engine: Optional[Engine] = None):
    """The evg_next_dispatchers of a batch of persisted queues: evg_dag_rebuild_batch's arrays plus GroupMaxHosts,
    DependenciesMet and the dense group id of every item.  -> (disp, compositeGroupID of each dense group per queue,
    the state a rebuild leaves: both IsDispatched copies from the persisted IsDispatched)."""
    eng = engine or default_engine()
    io, go, dep_off, dep_item, group_id, group_index, names = S.dag_input_from_queues(queues)
    srt, n_sorted, n_cycles, unit_items, unit_off = eng.dag_rebuild_batch(io, go, dep_off, dep_item, group_id, group_index)
    items = [it for q in queues for it in q.queue]
    disp = {"item_off": io, "group_off": go, "sorted": srt.copy(), "n_sorted": n_sorted.copy(), "unit_items": unit_items.copy(),
            "unit_off": unit_off.copy(), "group_id": group_id,
            "group_max_hosts": np.array([it.group_max_hosts for it in items], dtype=np.int32),
            "dependencies_met": np.array([it.dependencies_met for it in items], dtype=np.uint8)}
    # a persisted IsDispatched sets the node's bit and, for an item rebuild copies into a unit, the copy's
    state = {"item_bits": np.array([(L.EVG_NS_NODE | (L.EVG_NS_UNIT if g >= 0 else 0)) if it.is_dispatched else 0
                                    for it, g in zip(items, group_id)], dtype=np.uint8),
             "group_deleted": np.zeros(int(go[-1]), np.uint8), "group_running": np.zeros(int(go[-1]), np.int32)}
    return disp, names, state


def find_next_tasks(queues: Sequence[M.TaskQueue], requests, db: dict, *, engine: Optional[Engine] = None, built=None):
    """basicCachedDAGDispatcherImpl.FindNextTask (model/task_queue_service_dependency.go:258-469) for a batch of
    persisted queues: `requests[d]` = queue d's (TaskSpec or None, amiUpdatedTime) in serving order, against one frozen
    database snapshot `db` (soa.marshal_next_db).  `built`: (disp, names, state) from next_dispatchers or an earlier call,
    None = rebuild from the queues.  -> (per queue the (task id or None, EVG_NEXT_* outcome) of each request, `built`
    with the state the call left)."""
    eng = engine or default_engine()
    disp, names, state = built or next_dispatchers(queues, engine=eng)
    ids = [[it.id for it in q.queue] for q in queues]
    item, outcome, state = eng.find_next_batch(disp, S.marshal_next_db(ids, names, db), S.marshal_next_requests(names, requests), state)
    return _next_results(ids, requests, item, outcome), (disp, names, state)


class DAGDispatchService:
    """One distro's basicCachedDAGDispatcherImpl on the GPU: built from its persisted TaskQueue, FindNextTask(spec,
    amiUpdatedTime, db) serves one request per call like the reference, rebuild() starts over (Refresh's TTL is the
    caller's, :75-94).  last_outcome is the EVG_NEXT_* code of the last request."""

    def __init__(self, queue: M.TaskQueue, engine: Optional[Engine] = None):
        self.engine = engine
        self.rebuild(queue)

    def rebuild(self, queue: M.TaskQueue) -> None:
        self.queue = queue
        self.built = next_dispatchers([queue], engine=self.engine or default_engine())
        self.last_outcome = L.EVG_NEXT_NONE

    def FindNextTask(self, spec: Optional[M.TaskSpec], ami_updated_time: int, db: dict) -> Optional[M.TaskQueueItem]:
        res, self.built = find_next_tasks([self.queue], [[(spec, ami_updated_time)]], db, engine=self.engine, built=self.built)
        (tid, self.last_outcome), = res[0]
        return None if tid is None else next(it for it in self.queue.queue if it.id == tid)
