"""ctypes binding of libevgsched.so (include/evg_sched.h).

The library is the product; this module only loads it and mirrors its structs.
There is no fallback: if the shared object is missing, or no sm_90 device is
usable, every compute call raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libevgsched.so")

EVG_TIME_ZERO = -(2 ** 63)

EVG_OK = 0
EVG_ERR_INVALID, EVG_ERR_CUDA, EVG_ERR_NOMEM, EVG_ERR_STATE, EVG_ERR_INTERNAL = -1, -2, -3, -4, -5
EVG_ALLOC_OK, EVG_ALLOC_ERR_FUTURE_FRACTION, EVG_ALLOC_ERR_POOL_SIZE, EVG_ALLOC_ERR_PARENT_MISSING = 0, 1, 2, 3

EVG_TF_REQ_OTHER, EVG_TF_REQ_PATCH, EVG_TF_REQ_MERGE_QUEUE = 0, 1, 2
EVG_TF_GENERATE, EVG_TF_STEPBACK, EVG_TF_DEPS_MET, EVG_TF_OTHER_DISTRO = 0x4, 0x8, 0x10, 0x20
EVG_HF_RUNNING, EVG_HF_TEARDOWN, EVG_HF_RT_FOUND = 0x1, 0x2, 0x4
EVG_HG_NONE, EVG_HG_UNQUEUED = -1, -2
EVG_PROVIDER_STATIC, EVG_PROVIDER_EPHEMERAL, EVG_PROVIDER_DOCKER = 0, 1, 2
EVG_OPT_BREAKDOWN = 0x1
EVG_OPT_QUEUE_BREAKDOWN = 0x2
EVG_BD_N = 13
(EVG_BD_TASK_GROUP_LENGTH, EVG_BD_TOTAL_VALUE, EVG_BD_P_INITIAL, EVG_BD_P_TASK_GROUP, EVG_BD_P_GENERATOR,
 EVG_BD_P_COMMIT_QUEUE, EVG_BD_R_COMMIT_QUEUE, EVG_BD_R_NUM_DEPENDENTS, EVG_BD_R_ESTIMATED_RUNTIME,
 EVG_BD_R_MAINLINE_WAIT, EVG_BD_R_STEPBACK, EVG_BD_R_PATCH, EVG_BD_R_PATCH_WAIT) = range(13)
MAX_TASKS_PER_DISTRO = (1 << 21) - 1

# numpy mirrors of the POD structs (all naturally aligned, no padding)
DISTRO_CFG_DTYPE = np.dtype([
    ("patch_factor", "<i8"), ("patch_time_in_queue_factor", "<i8"), ("commit_queue_factor", "<i8"),
    ("mainline_time_in_queue_factor", "<i8"), ("expected_runtime_factor", "<i8"),
    ("generate_task_factor", "<i8"), ("stepback_task_factor", "<i8"), ("num_dependents_factor", "<f8"),
    ("target_time_ns", "<i8"), ("group_versions", "<i4"), ("includes_dependencies", "<i4"),
    ("n_versions", "<i4"), ("_reserved", "<i4")])
GROUP_INFO_FIELDS = ("count", "count_free", "count_required", "max_hosts", "expected_duration",
                     "count_duration_over_threshold", "count_wait_over_threshold",
                     "count_dep_filled_merge_queue_tasks", "duration_over_threshold")
GROUP_INFO_DTYPE = np.dtype([(f, "<i8") for f in GROUP_INFO_FIELDS])
QUEUE_INFO_DTYPE = np.dtype([
    ("length", "<i8"), ("length_with_dependencies_met", "<i8"), ("count_dep_filled_merge_queue_tasks", "<i8"),
    ("expected_duration", "<i8"), ("max_duration_threshold", "<i8"), ("count_duration_over_threshold", "<i8"),
    ("duration_over_threshold", "<i8"), ("count_wait_over_threshold", "<i8"), ("secondary_queue", "<i8"),
    ("has_ungrouped", "<i8"), ("ungrouped", GROUP_INFO_DTYPE)])
ALLOC_CFG_DTYPE = np.dtype([
    ("future_host_fraction", "<f8"), ("provider", "<i4"), ("disabled", "<i4"), ("minimum_hosts", "<i4"),
    ("maximum_hosts", "<i4"), ("round_up", "<i4"), ("waits_over_thresh_feedback", "<i4"), ("has_pool", "<i4"),
    ("pool_max_containers", "<i4"), ("parent_found", "<i4"), ("parent_maximum_hosts", "<i4")])
ALLOC_RESULT_DTYPE = np.dtype([("new_hosts", "<i4"), ("free_hosts", "<i4"), ("deficit_ns", "<i8")])
QUEUE_ITEM_DTYPE = np.dtype([("task", "<i4"), ("group_index", "<i4"), ("group_max_hosts", "<i4"), ("flags", "<u4"),
                             ("priority", "<i8"), ("expected_ns", "<i8"), ("total_value", "<i8")])
EVG_QI_DEPS_MET = 0x1
EVG_PERSISTED_QUEUE_CAP = 10000
assert QUEUE_ITEM_DTYPE.itemsize == 40
assert DISTRO_CFG_DTYPE.itemsize == 88 and GROUP_INFO_DTYPE.itemsize == 72
assert QUEUE_INFO_DTYPE.itemsize == 152 and ALLOC_CFG_DTYPE.itemsize == 48 and ALLOC_RESULT_DTYPE.itemsize == 16


class StrColStruct(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("off", C.c_void_p)]


class StringColsStruct(C.Structure):
    _fields_ = [("n_tasks", C.c_int64), ("n_distros", C.c_int32), ("task_off", C.c_void_p), ("id", StrColStruct),
                ("version", StrColStruct), ("group_key", StrColStruct), ("group_max_hosts", C.c_void_p),
                ("dep_off", C.c_void_p), ("dep_id", StrColStruct)]


class InternOutStruct(C.Structure):
    _fields_ = [("group_id", C.c_void_p), ("version_id", C.c_void_p), ("group_off", C.c_void_p), ("n_versions", C.c_void_p),
                ("group_max_hosts", C.c_void_p), ("group_first", C.c_void_p), ("dep_off", C.c_void_p), ("dep_idx", C.c_void_p)]


class QueueIndexOutStruct(C.Structure):
    _fields_ = [("min_position", C.c_void_p), ("dup_item", C.c_void_p), ("dup_off", C.c_void_p), ("dup_queue", C.c_void_p),
                ("n_dups", C.c_int64)]


class TaskSoAStruct(C.Structure):
    _fields_ = [("n_tasks", C.c_int64), ("n_edges", C.c_int64),
                ("priority", C.c_void_p), ("expected_ns", C.c_void_p), ("queue_basis_ns", C.c_void_p),
                ("wait_basis_ns", C.c_void_p), ("num_dependents", C.c_void_p), ("task_group_order", C.c_void_p),
                ("group_id", C.c_void_p), ("version_id", C.c_void_p), ("flags", C.c_void_p),
                ("dep_off", C.c_void_p), ("dep_idx", C.c_void_p)]


class DistroTableStruct(C.Structure):
    _fields_ = [("n_distros", C.c_int32), ("_reserved", C.c_int32), ("task_off", C.c_void_p),
                ("group_off", C.c_void_p), ("cfg", C.c_void_p), ("group_max_hosts", C.c_void_p)]


class TaskEditStruct(C.Structure):
    _fields_ = [("n_remove", C.c_int64), ("remove_rows", C.c_void_p), ("insert", C.POINTER(TaskSoAStruct)),
                ("insert_off", C.c_void_p), ("n_add_edges", C.c_int64), ("add_edge_task", C.c_void_p),
                ("add_edge_dep", C.c_void_p), ("group_remap", C.c_void_p), ("version_remap", C.c_void_p)]


class StringEditStruct(C.Structure):
    _fields_ = [("n_remove", C.c_int64), ("remove_rows", C.c_void_p), ("insert", C.POINTER(TaskSoAStruct)),
                ("insert_off", C.c_void_p), ("strings", C.POINTER(StringColsStruct))]


class PlanOutStruct(C.Structure):
    _fields_ = [("order", C.c_void_p), ("total_value", C.c_void_p), ("breakdown", C.c_void_p),
                ("info", C.c_void_p), ("group_info", C.c_void_p)]


class HostSoAStruct(C.Structure):
    _fields_ = [("n_hosts", C.c_int64), ("flags", C.c_void_p), ("group_id", C.c_void_p),
                ("expected_ns", C.c_void_p), ("std_ns", C.c_void_p), ("start_ns", C.c_void_p)]


class DepsInStruct(C.Structure):
    _fields_ = [("n_tasks", C.c_int64), ("n_deps", C.c_int64), ("dep_off", C.c_void_p), ("dep_kind", C.c_void_p),
                ("dep_ref", C.c_void_p), ("dep_want", C.c_void_p), ("task_state", C.c_void_p), ("task_pre", C.c_void_p),
                ("ext_state", C.c_void_p), ("n_ext", C.c_int64)]


class DepsEditStruct(C.Structure):
    _fields_ = [("depart_ext", C.c_void_p), ("depart_finished_ns", C.c_void_p), ("n_ext", C.c_int64), ("ext_state", C.c_void_p),
                ("ext_finished_ns", C.c_void_p), ("insert", C.POINTER(DepsInStruct)), ("insert_finished_ns", C.c_void_p),
                ("n_add", C.c_int64), ("add_row", C.c_void_p), ("add_kind", C.c_void_p), ("add_ref", C.c_void_p),
                ("add_want", C.c_void_p), ("add_finished_ns", C.c_void_p), ("n_set", C.c_int64), ("set_row", C.c_void_p),
                ("set_state", C.c_void_p), ("set_pre", C.c_void_p)]


EVG_DEP_IN_QUEUE, EVG_DEP_EXTERNAL, EVG_DEP_MISSING = 0, 1, 2
EVG_WANT_SUCCESS, EVG_WANT_FAILED, EVG_WANT_ANY, EVG_WANT_OTHER = 0, 1, 2, 3
EVG_TS_BLOCKED = 0x4
EVG_TP_OVERRIDE, EVG_TP_MET_TIME = 0x1, 0x2


class RunnableInStruct(C.Structure):
    _fields_ = [("n_tasks", C.c_int64), ("n_distros", C.c_int32), ("n_projects", C.c_int32), ("task_off", C.c_void_p),
                ("sched", C.c_void_p), ("project", C.c_void_p), ("project_flags", C.c_void_p), ("valid_off", C.c_void_p),
                ("valid_idx", C.c_void_p), ("finder", C.c_void_p), ("deps", C.POINTER(DepsInStruct))]


class AliasInStruct(C.Structure):
    _fields_ = [("tasks", TaskSoAStruct), ("n_groups", C.c_int32), ("n_versions", C.c_int32), ("group_max_hosts", C.c_void_p),
                ("sched", C.c_void_p), ("task_group_max_hosts", C.c_void_p), ("primary", C.c_void_p),
                ("secondary_off", C.c_void_p), ("secondary_idx", C.c_void_p), ("n_names", C.c_int32), ("_reserved", C.c_int32),
                ("dest_off", C.c_void_p), ("dest_idx", C.c_void_p), ("deps", C.POINTER(DepsInStruct)),
                ("dep_finished_ns", C.c_void_p)]


class AliasOutStruct(C.Structure):
    _fields_ = [("task_off", C.c_void_p), ("group_off", C.c_void_p), ("n_versions", C.c_void_p)]


EVG_SQ_ACTIVATED, EVG_SQ_UNDISPATCHED, EVG_SQ_PRIORITY_OK, EVG_SQ_HOST_PLATFORM = 0x01, 0x02, 0x04, 0x08
EVG_SQ_UNATTAINABLE, EVG_SQ_OVERRIDE_DEPS, EVG_SQ_GITHUB_PR, EVG_SQ_PATCH_REQUEST = 0x10, 0x20, 0x40, 0x80
EVG_PF_ENABLED, EVG_PF_HIDDEN, EVG_PF_DISPATCHING_DISABLED, EVG_PF_PATCHING_DISABLED = 0x1, 0x2, 0x4, 0x8
EVG_FINDER_NO_DEPS, EVG_FINDER_LEGACY, EVG_FINDER_ALTERNATE = 0, 1, 2
EVG_FINDER_PIPELINE, EVG_FINDER_PIPELINE_NO_DEPS = 3, 4
EVG_STATUS_SUCCESS, EVG_STATUS_FAILED, EVG_STATUS_ANY = 0, 1, 2
EVG_PR_ENABLED, EVG_PR_DISPATCHING_DISABLED, EVG_PR_PATCHING_FALSE = 0x1, 0x2, 0x4


class PipelineInStruct(C.Structure):
    _fields_ = [("n_status", C.c_int32), ("_reserved", C.c_int32), ("dep_status", C.c_void_p), ("task_status", C.c_void_p),
                ("ext_status", C.c_void_p), ("task_unattainable", C.c_void_p), ("ext_unattainable", C.c_void_p),
                ("project_raw", C.c_void_p)]


class DurationRowsStruct(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_keys", C.c_int32), ("_reserved", C.c_int32), ("key", C.c_void_p),
                ("time_taken_ns", C.c_void_p), ("start_ns", C.c_void_p), ("finish_ns", C.c_void_p), ("flags", C.c_void_p),
                ("window_start_ns", C.c_int64), ("window_end_ns", C.c_int64)]


EVG_DR_COMPLETED, EVG_DR_TIMED_OUT = 0x1, 0x2
DURATION_STAT_DTYPE = np.dtype([("count", np.int64), ("mean_ns", np.float64), ("stddev_ns", np.float64)])
EVG_DK_NONE = -1


def EVG_DK_PAIR(p: int) -> int:
    return -2 - p


EVG_DS_FRESH, EVG_DS_BACKFILL, EVG_DS_HISTORY, EVG_DS_PREVIOUS, EVG_DS_DEFAULT = 0, 1, 2, 3, 4
DURATION_CACHE_COLUMNS = ("value_ns", "std_ns", "ttl_ns", "collected_ns", "expected_ns", "expected_std_ns")


class DurationCacheStruct(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("rows", C.c_void_p), ("value_ns", C.c_void_p), ("std_ns", C.c_void_p),
                ("ttl_ns", C.c_void_p), ("collected_ns", C.c_void_p), ("expected_ns", C.c_void_p),
                ("expected_std_ns", C.c_void_p), ("key", C.c_void_p)]


class DurationInStruct(C.Structure):
    _fields_ = [("history", C.POINTER(DurationRowsStruct)), ("n_pairs", C.c_int32), ("_reserved", C.c_int32),
                ("pair_key_off", C.c_void_p), ("tasks", C.POINTER(DurationCacheStruct)),
                ("hosts", C.POINTER(DurationCacheStruct))]


DURATION_OUT_FIELDS = ("avg_ns", "std_ns", "value_ns", "pred_std_ns", "collected_ns", "source")


class DurationOutStruct(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in DURATION_OUT_FIELDS]


class LegacySoAStruct(C.Structure):
    _fields_ = [("n_tasks", C.c_int64), ("priority", C.c_void_p), ("ingest_ns", C.c_void_p), ("expected_ns", C.c_void_p),
                ("num_dependents", C.c_void_p), ("revision_order", C.c_void_p), ("project_id", C.c_void_p),
                ("tg_rank", C.c_void_p), ("tg_pair_id", C.c_void_p), ("task_group_order", C.c_void_p),
                ("presort_rank", C.c_void_p), ("flags", C.c_void_p)]


EVG_LF_REQ_SYSTEM, EVG_LF_REQ_PATCH, EVG_LF_REQ_OTHER, EVG_LF_GENERATE, EVG_LF_MERGE_QUEUE_VERSION = 0, 1, 2, 0x4, 0x8
EVG_LEGACY_MODE_INGEST, EVG_LEGACY_MODE_REVISION, EVG_LEGACY_MODE_LITERAL, EVG_LEGACY_MODE_GO_STABLE = 0, 1, 2, 3
EVG_LEGACY_OK, EVG_LEGACY_NOT_DECOMPOSABLE = 0, 1


class DagInStruct(C.Structure):
    _fields_ = [("n_items", C.c_int64), ("n_deps", C.c_int64), ("dep_off", C.c_void_p), ("dep_item", C.c_void_p),
                ("group_id", C.c_void_p), ("group_index", C.c_void_p)]


DISPATCH_OUT_FIELDS = ("item_off", "sorted", "n_sorted", "n_cycles", "group_off", "group_slot", "unit_items", "unit_off")


class DispatchOutStruct(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in DISPATCH_OUT_FIELDS]


# FindNextTask (evg_find_next_batch / evg_find_next_tasks)
(EVG_ND_FOUND, EVG_ND_STARTED, EVG_ND_STARTED_GROUP, EVG_ND_FINISHED_NOT_SUCCEEDED, EVG_ND_VERSION_FOUND, EVG_ND_VERSION_S3,
 EVG_ND_DEPS_MET_NOW, EVG_ND_DEPS_ERR) = (1 << k for k in range(8))
EVG_NEXT_NONE, EVG_NEXT_FOUND, EVG_NEXT_GAVE_UP = 0, 1, 2
EVG_NS_NODE, EVG_NS_UNIT = 1, 2


class NextDbStruct(C.Structure):
    _fields_ = [("n_items", C.c_int64), ("n_groups", C.c_int64), ("flags", C.c_void_p), ("est_generated", C.c_void_p),
                ("ingest_ns", C.c_void_p), ("running_hosts", C.c_void_p), ("generate_limit", C.c_int32),
                ("pending_generate", C.c_int32), ("max_large_parser", C.c_int32), ("num_large_parser", C.c_int32)]


class NextReqStruct(C.Structure):
    _fields_ = [("n_requests", C.c_int64), ("req_off", C.c_void_p), ("group", C.c_void_p), ("ami_updated_ns", C.c_void_p)]


class NextOutStruct(C.Structure):
    _fields_ = [("item", C.c_void_p), ("outcome", C.c_void_p)]


class NextStateStruct(C.Structure):
    _fields_ = [("item_bits", C.c_void_p), ("group_deleted", C.c_void_p), ("group_running", C.c_void_p)]


NEXT_DISPATCHER_FIELDS = ("item_off", "group_off", "sorted", "n_sorted", "unit_items", "unit_off", "group_id", "group_max_hosts",
                          "dependencies_met")


class NextDispatchersStruct(C.Structure):
    _fields_ = [("n_distros", C.c_int32), ("_reserved", C.c_int32)] + [(f, C.c_void_p) for f in NEXT_DISPATCHER_FIELDS]


assert (C.sizeof(NextDbStruct), C.sizeof(NextReqStruct), C.sizeof(NextOutStruct), C.sizeof(NextStateStruct),
        C.sizeof(NextDispatchersStruct)) == (64, 32, 16, 24, 80)


class AllocOutStruct(C.Structure):
    _fields_ = [("result", C.c_void_p), ("status", C.c_void_p)]


HOST_JOB_CFG_DTYPE = np.dtype([("n_provisioning", "<i8"), ("single_task_distro", "<i4"),
                               ("terminate_when_overallocated", "<i4"), ("hourly_billing", "<i4"), ("_reserved", "<i4")])
HOST_REPORT_FIELDS = ("time_to_empty_ns", "time_to_empty_no_spawns_ns", "scheduled_duration_ns", "hosts_avail", "hosts_spawned",
                      "overdue_in_groups", "free_in_groups", "required_in_groups", "new_cap_target", "killable_hosts",
                      "host_queue_ratio", "no_spawns_ratio", "drawdown")
HOST_REPORT_DTYPE = np.dtype([(f, "<i8") for f in HOST_REPORT_FIELDS[:10]] + [
    ("host_queue_ratio", "<f4"), ("no_spawns_ratio", "<f4"), ("drawdown", "<i4"), ("_reserved", "<i4")])
assert HOST_JOB_CFG_DTYPE.itemsize == 24 and HOST_REPORT_DTYPE.itemsize == 96


class HostJobOutStruct(C.Structure):
    _fields_ = [("n_hosts", C.c_void_p), ("n_hosts_free", C.c_void_p), ("status", C.c_void_p), ("report", C.c_void_p)]


# the idle-host table of evg_host_drawdown / evg_idle_hosts
(EVG_IH_RUNNING_TASK_GROUP, EVG_IH_LAST_TASK, EVG_IH_STATUS_RUNNING, EVG_IH_USER_DATA, EVG_IH_LEGACY_BOOTSTRAP,
 EVG_IH_NEEDS_NEW_AGENT, EVG_IH_NEEDS_NEW_AGENT_MONITOR, EVG_IH_OUTDATED_AMI, EVG_IH_SINGLE_HOST_TASK_GROUP,
 EVG_IH_TASK_LOOKUP_FAILED, EVG_IH_PAYMENT_NOT_DUE, EVG_IH_CLOUD_MANAGER_FAILED) = (1 << k for k in range(12))
(EVG_HT_NOT_CHECKED, EVG_HT_KEPT, EVG_HT_EXEMPT_AGENT, EVG_HT_EXEMPT_PAYMENT, EVG_HT_ERR_CLOUD_MANAGER, EVG_HT_ERR_TASK_LOOKUP,
 EVG_HT_DECOMMISSION, EVG_HT_TERM_OUTDATED_AMI, EVG_HT_TERM_COMMUNICATION, EVG_HT_TERM_IDLE, EVG_HT_TERM_TEARDOWN) = range(11)
EVG_NO_DRAWDOWN = -(2 ** 63)
IDLE_HOST_COLUMNS = ("creation_ns", "start_ns", "provision_ns", "agent_start_ns", "last_communication_ns",
                     "last_task_completed_ns", "teardown_start_ns", "acceptable_idle_ns")
HOST_VERDICT_DTYPE = np.dtype([("idle_ns", "<i8"), ("communication_ns", "<i8"), ("threshold_ns", "<i8"),
                               ("since_teardown_ns", "<i8"), ("decision", "<i4"), ("_reserved", "<i4")])
DRAWDOWN_DISTRO_DTYPE = np.dtype([("target", "<i8"), ("decommissioned", "<i8"), ("ran", "<i4"), ("_reserved", "<i4")])
IDLE_CFG_DTYPE = np.dtype([("minimum_hosts", "<i8"), ("running_hosts_count", "<i8"), ("acceptable_idle_ns", "<i8")])
IDLE_DISTRO_DTYPE = np.dtype([("min_evaluate", "<i8"), ("terminated", "<i8")])
assert (HOST_VERDICT_DTYPE.itemsize, DRAWDOWN_DISTRO_DTYPE.itemsize, IDLE_CFG_DTYPE.itemsize, IDLE_DISTRO_DTYPE.itemsize) == (40, 24, 24, 16)


class IdleHostSoAStruct(C.Structure):
    _fields_ = [("n_hosts", C.c_int64), ("n_distros", C.c_int32), ("_reserved", C.c_int32)] + [
        (f, C.c_void_p) for f in IDLE_HOST_COLUMNS + ("flags",)]


class DrawdownInStruct(C.Structure):
    _fields_ = [("existing_hosts", C.c_void_p), ("new_cap_target", C.c_void_p), ("queue_length_dm", C.c_void_p)]


class HostTermOutStruct(C.Structure):  # evg_host_drawdown_out and evg_idle_hosts_out
    _fields_ = [("hosts", C.c_void_p), ("distros", C.c_void_p)]


# the start-time estimator's host table (evg_estimate_start_times / evg_estimate_start_batch)
EVG_EH_UNINITIALIZED, EVG_EH_STARTING, EVG_EH_PROVISIONING, EVG_EH_FREE, EVG_EH_RUNNING, EVG_EH_IGNORED = range(6)
EVG_EST_ONCHIP_HOSTS = 1024


class EstHostSoAStruct(C.Structure):
    _fields_ = [("n_hosts", C.c_int64), ("kind", C.c_void_p), ("expected_ns", C.c_void_p), ("dispatch_ns", C.c_void_p)]


assert C.sizeof(EstHostSoAStruct) == 32


class EvgError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libevgsched error {code}: {msg}")
        self.code = code


# every symbol include/evg_sched.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "evg_init": (C.c_int, [C.c_int, _P, C.POINTER(_P)]),
    "evg_shutdown": (None, [_P]),
    "evg_last_error": (C.c_char_p, []),
    "evg_abi_version": (C.c_int, []),
    "evg_host_alloc": (_P, [C.c_uint64]),
    "evg_host_free": (None, [_P]),
    "evg_plan_batch": (C.c_int, [_P, _P, _P, C.c_int64, C.c_uint32, _P]),
    "evg_alloc_batch": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int64, _P]),
    "evg_plan_and_alloc_batch": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int64, C.c_uint32, _P, _P]),
    "evg_upload": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "evg_upload_device": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "evg_update_tasks": (C.c_int, [_P, C.c_int64, _P, _P]),
    "evg_edit_tasks": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "evg_edit_tasks_with_deps": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int64]),
    "evg_plan_from_finder": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, _P, _P]),
    "evg_plan_from_finder_ex": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, _P, _P]),
    "evg_plan_aliases": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int64, _P]),
    "evg_download_alias_map": (C.c_int, [_P, _P, _P]),
    "evg_intern_columns": (C.c_int, [_P, _P, C.c_int32]),
    "evg_intern_batch": (C.c_int, [_P, _P, _P]),
    "evg_upload_strings": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "evg_edit_strings": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "evg_queue_index_batch": (C.c_int, [_P, _P, _P, C.c_int32, _P]),
    "evg_run_resident": (C.c_int, [_P, C.c_int64, C.c_uint32]),
    "evg_download": (C.c_int, [_P, _P, _P]),
    "evg_download_queue": (C.c_int, [_P, C.c_int32, _P, _P, C.c_int64]),
    "evg_download_queue_breakdown": (C.c_int, [_P, C.c_int32, _P, _P, C.c_int64]),
    "evg_device_result_ptr": (_P, [_P]),
    "evg_bind_result_buffer": (C.c_int, [_P, _P, C.c_int64]),
    "evg_last_launch_count": (C.c_int64, [_P]),
    "evg_last_timing_ms": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "evg_kernel_timing_ms": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int32]),
    "evg_general_timing_ms": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "evg_deps_met_batch": (C.c_int, [_P, _P, _P]),
    "evg_upload_with_deps": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int64]),
    "evg_download_deps": (C.c_int, [_P, _P, _P]),
    "evg_find_runnable_batch": (C.c_int, [_P, _P, _P, _P]),
    "evg_find_runnable_ex": (C.c_int, [_P, _P, _P, _P, _P]),
    "evg_expected_durations_batch": (C.c_int, [_P, _P, _P]),
    "evg_resolve_durations": (C.c_int, [_P, _P, C.c_int64]),
    "evg_download_durations": (C.c_int, [_P, _P, _P]),
    "evg_prioritize_legacy_batch": (C.c_int, [_P, _P, _P, _P, C.c_int32, _P, _P, _P]),
    "evg_dag_rebuild_batch": (C.c_int, [_P, _P, _P, _P, C.c_int32, _P, _P, _P, _P, _P]),
    "evg_rebuild_dispatchers": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int64, _P]),
    "evg_find_next_batch": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "evg_find_next_tasks": (C.c_int, [_P, _P, _P, _P]),
    "evg_download_dispatch_state": (C.c_int, [_P, _P]),
    "evg_host_job": (C.c_int, [_P, _P, _P, _P]),
    "evg_host_drawdown": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P]),
    "evg_idle_hosts": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P]),
    "evg_estimate_start_times": (C.c_int, [_P, C.c_int32, _P, _P, C.c_int64, _P, _P, C.c_int64, _P]),
    "evg_estimate_start_batch": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P, C.c_int64, _P, _P]),
    "evg_plan_distro": (C.c_int, [_P, _P, _P, C.c_int32, _P, C.c_int64, C.c_uint32, _P]),
    "evg_alloc_distro": (C.c_int, [_P, _P, _P, _P, _P, C.c_int32, C.c_int64, _P, _P]),
}

_lib = None


def load() -> C.CDLL:
    """Load libevgsched.so (built in-tree by __graft_entry__.build()). Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). evergreen_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    if lib.evg_abi_version() != 1:
        raise ImportError("libevgsched.so ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    return (load().evg_last_error() or b"").decode("utf-8", "replace")


def check(rc: int) -> None:
    if rc != EVG_OK:
        raise EvgError(rc, last_error())


def ptr(a) -> int:
    """Address of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "columns must be C-contiguous"
    return a.ctypes.data
