"""Host-side mirror of the reference structs the scheduler hot path reads.

Only the fields the path touches are kept (SURVEY.md §8a row A20):
``task.Task`` (model/task/task.go:83-350), ``distro.Distro`` with
``PlannerSettings`` / ``HostAllocatorSettings`` (model/distro/distro.go:267-300),
``host.Host`` (model/host/host.go:79-88), ``model.TaskGroupInfo`` /
``model.DistroQueueInfo`` (model/task_queue.go:22-75),
``task.SortingValueBreakdown`` (model/task/task.go:3990-4038) and
``evergreen.ContainerPool`` (config_containerpools.go:11-22).

Times are int nanoseconds since the Unix epoch; ``ZERO_TIME`` stands for Go's
zero ``time.Time`` (year 1).  Durations are int nanoseconds (``time.Duration``).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Tuple

ZERO_TIME = -(2 ** 63)

NANOSECOND = 1
MICROSECOND = 1000
MILLISECOND = 1000 * MICROSECOND
SECOND = 1000 * MILLISECOND
MINUTE = 60 * SECOND
HOUR = 60 * MINUTE

# globals.go:753-759
PATCH_VERSION_REQUESTER = "patch_request"
GITHUB_PR_REQUESTER = "github_pull_request"
REPOTRACKER_VERSION_REQUESTER = "gitter_request"
GITHUB_MERGE_REQUESTER = "github_merge_request"
GIT_TAG_REQUESTER = "git_tag_request"
TRIGGER_REQUESTER = "trigger_request"
AD_HOC_REQUESTER = "ad_hoc"
# globals.go:766-772
SYSTEM_VERSION_REQUESTER_TYPES = (REPOTRACKER_VERSION_REQUESTER, TRIGGER_REQUESTER, GIT_TAG_REQUESTER, AD_HOC_REQUESTER)
MAX_TASK_PRIORITY = 100  # globals.go:185
# globals.go:219
STEPBACK_TASK_ACTIVATOR = "stepback"
# globals.go:52-71
TASK_UNDISPATCHED = "undispatched"
TASK_SUCCEEDED = "success"
TASK_FAILED = "failed"
ALL_STATUSES = "*"  # model/task/task.go:491
TASK_COMPLETED_STATUSES = (TASK_SUCCEEDED, TASK_FAILED)  # globals.go TaskCompletedStatuses
# globals.go:264
DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES = "revised-with-dependencies"
# globals.go:267-268
MAX_DURATION_PER_DISTRO_HOST = 30 * MINUTE
MAX_DURATION_PER_DISTRO_HOST_WITH_CONTAINERS = 2 * MINUTE
# model/task/task.go:64,67
DEFAULT_TASK_DURATION = 10 * MINUTE
PREDICTION_TTL = 8 * HOUR
# globals.go:309-314
HOST_ALLOCATOR_ROUND_DOWN = "round-down"
HOST_ALLOCATOR_ROUND_UP = "round-up"
HOST_ALLOCATOR_ROUND_DEFAULT = ""
HOST_ALLOCATOR_WAITS_OVER_THRESH_FEEDBACK = "waits-over-thresh-feedback"
HOST_ALLOCATOR_NO_FEEDBACK = "no-feedback"
# globals.go:671-676
PROVIDER_EC2_ONDEMAND = "ec2-ondemand"
PROVIDER_EC2_FLEET = "ec2-fleet"
PROVIDER_DOCKER = "docker"
PROVIDER_STATIC = "static"
PROVIDER_MOCK = "mock"
PROVIDER_SPAWNABLE = (PROVIDER_EC2_ONDEMAND, PROVIDER_EC2_FLEET, PROVIDER_MOCK, PROVIDER_DOCKER)  # globals.go:723-728
HOSTS_OVERALLOCATED_TERMINATE = "terminate-hosts-when-overallocated"  # globals.go:317
# model/task_queue.go:216-219
PERSISTED_QUEUE_CAP = 10000
# model/task_queue.go:17-20: the collections TaskQueue.Save writes to
TASK_QUEUES_COLLECTION = "task_queues"
TASK_SECONDARY_QUEUES_COLLECTION = "task_alias_queues"
DISABLED_TASK_PRIORITY = -1  # globals.go:187
HOST_RUNNING = "running"  # globals.go:24
HOST_UNINITIALIZED = "initializing"  # globals.go:26
HOST_STARTING = "starting"  # globals.go:35
HOST_PROVISIONING = "provisioning"  # globals.go:36
# globals.go:975-984: the statuses host.ByDistroIDs returns (model/host/db.go:628-635)
UP_HOST_STATUS = (HOST_RUNNING, HOST_UNINITIALIZED, "building", HOST_STARTING, HOST_PROVISIONING, "provision failed", "stopping", "stopped")
# model/distro/distro.go:319-321
BOOTSTRAP_METHOD_LEGACY_SSH = "legacy-ssh"
BOOTSTRAP_METHOD_USER_DATA = "user-data"


def is_github_merge_queue_requester(r: str) -> bool:  # globals.go:1195-1197
    return r == GITHUB_MERGE_REQUESTER


def is_patch_requester(r: str) -> bool:  # globals.go:1179-1185
    return r in (PATCH_VERSION_REQUESTER, GITHUB_PR_REQUESTER, GITHUB_MERGE_REQUESTER)


def is_zero_time(t: int) -> bool:
    """utility.IsZeroTime: true for Go's zero time and for the Unix epoch."""
    return t == ZERO_TIME or t == 0


@dataclass
class Dependency:  # model/task/task.go Dependency
    task_id: str
    status: str = ""
    unattainable: bool = False
    finished_at: int = ZERO_TIME


@dataclass
class CachedDurationValue:  # util/cached_value.go:87-93
    value: int = 0
    std_dev: int = 0
    ttl: int = 0
    collected_at: int = ZERO_TIME


@dataclass
class Task:
    id: str = ""
    version: str = ""
    project: str = ""
    build_variant: str = ""
    revision: str = ""               # TaskQueueItem.Revision (task_queue_persister.go:28)
    build_id: str = ""               # legacy prioritiser only (task_priority_cmp.go:149-174, setup_funcs.go:72-87)
    revision_order_number: int = 0   # legacy prioritiser only (task_priority_cmp.go:75-84)
    display_name: str = ""
    task_group: str = ""
    task_group_max_hosts: int = 0
    task_group_order: int = 0
    priority: int = 0
    requester: str = ""
    activated_by: str = ""
    generate_task: bool = False
    depends_on: List[Dependency] = field(default_factory=list)
    override_dependencies: bool = False
    num_dependents: int = 0
    activated_time: int = ZERO_TIME
    ingest_time: int = ZERO_TIME
    scheduled_time: int = ZERO_TIME
    dependencies_met_time: int = ZERO_TIME
    start_time: int = ZERO_TIME
    dispatch_time: int = ZERO_TIME   # the start-time estimator reads it of a host's running task (task_start_estimation.go:156)
    distro_id: str = ""
    secondary_distros: List[str] = field(default_factory=list)  # Task.SecondaryDistros: the alias queues it may join
    status: str = TASK_UNDISPATCHED
    # finished-task history (expected_duration.go:36-55)
    finish_time: int = ZERO_TIME
    time_taken: int = 0
    timed_out: bool = False  # Details.TimedOut
    # what the task finders' base query reads (schedulableHostTasksQuery, model/task/db.go:671-689)
    activated: bool = True
    execution_platform: str = ""           # "" (field absent) or "host" pass ByExecutionPlatform(host), db.go:647-663
    unattainable_dependency: bool = False  # the cached UnattainableDependency field
    expected_duration: int = 0
    expected_duration_std_dev: int = 0
    duration_prediction: CachedDurationValue = field(default_factory=CachedDurationValue)
    # outputs stamped by the planner (scheduler.go:98, planner.go:475)
    wait_since_dependencies_met: int = 0
    sorting_value_breakdown: Optional["SortingValueBreakdown"] = None

    def get_task_group_string(self) -> str:  # model/task/task.go:417-419
        return f"{self.task_group}_{self.build_variant}_{self.project}_{self.version}"

    def blocked(self) -> bool:  # model/task/task.go:3649-3660
        if self.override_dependencies:
            return False
        return any(d.unattainable for d in self.depends_on)

    def has_dependencies_met(self) -> bool:  # model/task/task.go:3393-3395
        return (not self.depends_on) or self.override_dependencies or not is_zero_time(self.dependencies_met_time)


@dataclass
class PlannerSettings:  # model/distro/distro.go:286-300
    version: str = "tunable"
    target_time: int = 0
    group_versions: Optional[bool] = None
    patch_factor: int = 0
    patch_time_in_queue_factor: int = 0
    commit_queue_factor: int = 0
    mainline_time_in_queue_factor: int = 0
    expected_runtime_factor: int = 0
    generate_task_factor: int = 0
    num_dependents_factor: float = 0.0
    stepback_task_factor: int = 0

    def should_group_versions(self) -> bool:  # distro.go:349-351
        return bool(self.group_versions)


@dataclass
class HostAllocatorSettings:  # model/distro/distro.go:267-280
    version: str = "utilization"
    minimum_hosts: int = 0
    maximum_hosts: int = 0
    rounding_rule: str = ""
    feedback_rule: str = ""
    hosts_overallocated_rule: str = ""
    acceptable_host_idle_time: int = 0
    future_host_fraction: float = 0.0


@dataclass
class DispatcherSettings:
    version: str = "revised-with-dependencies"


@dataclass
class ContainerPool:  # config_containerpools.go:11-22
    id: str = ""
    distro: str = ""
    max_containers: int = 0


@dataclass
class ProjectRef:  # the fields ProjectCanDispatchTask reads (model/project_ref.go:3441-3462)
    id: str = ""
    enabled: bool = False
    hidden: Optional[bool] = None
    dispatching_disabled: Optional[bool] = None
    patching_disabled: Optional[bool] = None

    def can_dispatch_task(self, t: "Task") -> bool:
        if not self.enabled and not (t.requester == GITHUB_PR_REQUESTER and bool(self.hidden)):
            return False
        if self.dispatching_disabled:
            return False
        if is_patch_requester(t.requester) and self.patching_disabled:
            return False
        return True


@dataclass
class Distro:
    id: str = ""
    provider: str = ""
    disabled: bool = False
    container_pool: str = ""
    single_task_distro: bool = False
    planner_settings: PlannerSettings = field(default_factory=PlannerSettings)
    host_allocator_settings: HostAllocatorSettings = field(default_factory=HostAllocatorSettings)
    dispatcher_settings: DispatcherSettings = field(default_factory=lambda: DispatcherSettings(version=""))
    valid_projects: List[str] = field(default_factory=list)
    aliases: List[str] = field(default_factory=list)  # Distro.Aliases (FindApplicableDistroIDs, model/distro/aliases.go:14-27)
    arch: str = ""  # Distro.Arch (cloud.UsesHourlyBilling reads it, cloud/ec2_util.go:256-268)
    default_ami: str = ""  # Distro.GetDefaultAMI() (model/distro/distro.go:112-127)

    def max_duration_per_host(self) -> int:  # distro.go:422-432
        if self.container_pool != "":
            return MAX_DURATION_PER_DISTRO_HOST_WITH_CONTAINERS
        return MAX_DURATION_PER_DISTRO_HOST

    def get_target_time(self) -> int:  # distro.go:434-440
        if self.planner_settings.target_time == 0:
            return self.max_duration_per_host()
        return self.planner_settings.target_time

    def is_ephemeral(self) -> bool:  # distro.go:478-480
        return self.provider in PROVIDER_SPAWNABLE


@dataclass
class Host:  # model/host/host.go:38-...
    id: str = ""
    running_task: str = ""
    running_task_group: str = ""
    running_task_build_variant: str = ""
    running_task_project: str = ""
    running_task_version: str = ""
    task_group_teardown_start_time: int = ZERO_TIME
    # what the drawdown and idle-host jobs read (units/host_drawdown.go, units/host_monitoring_idle_termination.go)
    status: str = ""
    creation_time: int = ZERO_TIME
    start_time: int = ZERO_TIME
    provision_time: int = ZERO_TIME
    agent_start_time: int = ZERO_TIME
    last_communication_time: int = ZERO_TIME
    last_task_completed_time: int = ZERO_TIME
    last_task: str = ""
    last_group: str = ""
    needs_new_agent: bool = False
    needs_new_agent_monitor: bool = False
    bootstrap_method: str = ""           # h.Distro.BootstrapSettings.Method (the embedded distro document)
    acceptable_host_idle_time: int = 0   # h.Distro.HostAllocatorSettings.AcceptableHostIdleTime
    ami: str = ""                        # h.GetAMI()
    # resolved lookups the jobs perform against MongoDB and the cloud provider
    last_task_single_host_task_group: Optional[bool] = False  # the last task IsPartOfSingleHostTaskGroup and succeeded;
                                                               # None: task.FindOneId failed or found nothing
    time_til_next_payment: int = 0       # manager.TimeTilNextPayment(h)
    cloud_manager_error: bool = False    # cloud.GetManagerOptions / GetManager returned an error

    def is_free(self) -> bool:  # host.go:214-221
        return self.running_task == "" and self.task_group_teardown_start_time == ZERO_TIME

    def get_task_group_string(self) -> str:  # host.go:663-665
        return (f"{self.running_task_group}_{self.running_task_build_variant}_"
                f"{self.running_task_project}_{self.running_task_version}")


@dataclass
class TaskGroupInfo:  # model/task_queue.go:22-47
    name: str = ""
    count: int = 0
    count_free: int = 0
    count_required: int = 0
    max_hosts: int = 0
    expected_duration: int = 0
    count_duration_over_threshold: int = 0
    count_wait_over_threshold: int = 0
    count_dep_filled_merge_queue_tasks: int = 0
    duration_over_threshold: int = 0


@dataclass
class DistroQueueInfo:  # model/task_queue.go:49-75
    length: int = 0
    length_with_dependencies_met: int = 0
    count_dep_filled_merge_queue_tasks: int = 0
    expected_duration: int = 0
    max_duration_threshold: int = 0
    plan_created_at: int = ZERO_TIME
    count_duration_over_threshold: int = 0
    duration_over_threshold: int = 0
    count_wait_over_threshold: int = 0
    task_group_infos: List[TaskGroupInfo] = field(default_factory=list)
    secondary_queue: bool = False


@dataclass
class TaskQueueItem:  # model/task_queue.go:131-153
    id: str = ""
    is_dispatched: bool = False
    display_name: str = ""
    group: str = ""
    group_max_hosts: int = 0
    group_index: int = 0
    version: str = ""
    build_variant: str = ""
    revision_order_number: int = 0
    requester: str = ""
    revision: str = ""
    project: str = ""
    expected_duration: int = 0
    priority: int = 0
    sorting_value_breakdown: Optional["SortingValueBreakdown"] = None
    dependencies: List[str] = field(default_factory=list)
    dependencies_met: bool = False
    activated_by: str = ""


@dataclass
class TaskSpec:  # model/task_queue.go:184-190: the task group the host last ran, as FindNextTask receives it
    group: str = ""
    build_variant: str = ""
    project: str = ""
    version: str = ""
    group_max_hosts: int = 0

    def composite_group_id(self) -> str:  # compositeGroupID, model/task_queue_service_dependency.go:700-702
        return f"{self.group}_{self.build_variant}_{self.project}_{self.version}"


@dataclass
class TaskQueue:  # model/task_queue.go:117-123
    distro: str = ""
    generated_at: int = ZERO_TIME
    queue: List[TaskQueueItem] = field(default_factory=list)
    distro_queue_info: Optional["DistroQueueInfo"] = None

    def collection(self) -> str:  # TaskQueue.Save routes on DistroQueueInfo.GetQueueCollection (model/task_queue.go:108-115)
        if self.distro_queue_info is not None and self.distro_queue_info.secondary_queue:
            return TASK_SECONDARY_QUEUES_COLLECTION
        return TASK_QUEUES_COLLECTION


@dataclass
class DuplicateEnqueuedTasksResult:  # model/task_queue.go:500-503
    task_id: str = ""
    distro_ids: List[str] = field(default_factory=list)


@dataclass
class SortingValueBreakdown:  # model/task/task.go:3990-4038 (flattened)
    task_group_length: int = 0
    total_value: int = 0
    # PriorityBreakdown
    initial_priority_impact: int = 0
    task_group_impact: int = 0
    generator_task_impact: int = 0
    priority_commit_queue_impact: int = 0
    # RankValueBreakdown
    rank_commit_queue_impact: int = 0
    num_dependents_impact: int = 0
    estimated_runtime_impact: int = 0
    mainline_wait_time_impact: int = 0
    stepback_impact: int = 0
    patch_impact: int = 0
    patch_wait_time_impact: int = 0

    FIELDS = ("task_group_length", "total_value", "initial_priority_impact", "task_group_impact",
              "generator_task_impact", "priority_commit_queue_impact", "rank_commit_queue_impact",
              "num_dependents_impact", "estimated_runtime_impact", "mainline_wait_time_impact",
              "stepback_impact", "patch_impact", "patch_wait_time_impact")

    @classmethod
    def from_row(cls, row) -> "SortingValueBreakdown":
        return cls(*[int(x) for x in row])

    def row(self):
        return [getattr(self, f) for f in self.FIELDS]


@dataclass
class RunningTaskStats:
    """What task.Find(ByIds) + FetchExpectedDuration yield for a host's running
    task (utilization_based_host_allocator.go:337,357-361)."""
    found: bool = True
    expected: int = 0
    std_dev: int = 0
    start_time: int = ZERO_TIME


@dataclass
class HostAllocatorData:  # scheduler/host_allocator.go:17-23
    distro: Distro
    existing_hosts: List[Host]
    distro_queue_info: DistroQueueInfo
    uses_containers: bool = False
    container_pool: Optional[ContainerPool] = None
    # resolved lookups the reference performs against MongoDB
    running_tasks: dict = field(default_factory=dict)         # task id -> RunningTaskStats
    parent_distro_maximum_hosts: Optional[int] = None         # distro.FindOneId(pool.Distro) (allocator.go:151-160)


@dataclass
class HostAllocatorJobReport:
    """The distro-scheduler-report hostAllocatorJob.Run computes after spawning (units/host_allocator.go:257-326), with
    the drawdown decision of setTargetAndTerminate (:328-337, 394-425).  Ratios are float32 values, as Go computes them;
    new_cap_target and killable_hosts are 0 when setTargetAndTerminate is not called."""
    time_to_empty: int = 0
    time_to_empty_no_spawns: int = 0
    scheduled_duration: int = 0
    hosts_avail: int = 0
    hosts_spawned: int = 0
    overdue_in_groups: int = 0
    free_in_groups: int = 0
    required_in_groups: int = 0
    host_queue_ratio: float = 0.0
    no_spawns_ratio: float = 0.0
    drawdown: bool = False
    new_cap_target: int = 0
    killable_hosts: int = 0


@dataclass
class DrawdownInfo:  # units/host_drawdown.go:33-36
    distro_id: str = ""
    new_cap_target: int = 0


@dataclass
class HostDrawdownJob:
    """What hostDrawdownJob.Run does for one distro (units/host_drawdown.go:70-118): the hosts it decommissions, in
    order, the errors it logs per host, and the counts of its closing log line."""
    distro_id: str = ""
    new_cap_target: int = 0
    existing_host_count: int = 0
    num_idle_hosts: int = 0
    drawdown_target: int = 0
    decommissioned_hosts: List[str] = field(default_factory=list)
    errors: List[Tuple[str, str]] = field(default_factory=list)  # (host id, what failed)

    @property
    def decommissioned(self) -> int:
        return len(self.decommissioned_hosts)


@dataclass
class IdleHostJob:
    """What idleHostJob.Run does for one distro (units/host_monitoring_idle_termination.go:128-140): the hosts it
    terminates with getTerminationReason's reason, in order, the errors it adds per host, and its counts."""
    distro_id: str = ""
    num_idle_hosts: int = 0
    min_hosts_to_evaluate: int = 0
    terminated_hosts: List[str] = field(default_factory=list)
    reasons: List[str] = field(default_factory=list)
    errors: List[Tuple[str, str]] = field(default_factory=list)

    @property
    def terminated(self) -> int:
        return len(self.terminated_hosts)


def _frac(u: int, prec: int) -> Tuple[int, str]:  # time.fmtFrac
    q, r = divmod(u, 10 ** prec)
    digits = f"{r:0{prec}d}".rstrip("0") if prec else ""
    return q, "." + digits if digits else ""


def go_duration_string(d: int) -> str:
    """time.Duration.String (go/src/time/time.go): "72h3m0.5s", "1.5µs", "0s"."""
    u = -d if d < 0 else d
    if u == 0:
        return "0s"
    if u < SECOND:
        if u < MICROSECOND:
            prec, unit = 0, "ns"
        elif u < MILLISECOND:
            prec, unit = 3, "µs"
        else:
            prec, unit = 6, "ms"
        q, frac = _frac(u, prec)
        text = f"{q}{frac}{unit}"
    else:
        secs, frac = _frac(u, 9)
        text = f"{secs % 60}{frac}s"
        mins = secs // 60
        if mins > 0:
            text = f"{mins % 60}m" + text
            if mins // 60 > 0:
                text = f"{mins // 60}h" + text
    return "-" + text if d < 0 else text


def duration_from_float(x: float) -> int:
    """time.Duration(float64) under DESIGN.md §3 (iv): truncation toward zero, a value beyond the int64 range saturated
    at its end, NaN -> 0 (the device's __double2ll_rz).  Go leaves the out-of-range conversion implementation-defined."""
    if x != x:
        return 0
    if x >= 2.0 ** 63:
        return 2 ** 63 - 1
    if x < -2.0 ** 63:
        return -2 ** 63
    return int(x)


def fetch_expected_duration(t: Task, now: int, history=None):
    """Decision logic of Task.FetchExpectedDuration (model/task/task.go:3519-3590)
    with CachedDurationValue.Get (util/cached_value.go:125-145).  ``history`` is
    the result of the weekly $avg/$stdDevPop aggregate (None = no rows).  The
    TTL jitter (task.go:3521) is not modelled: an unset TTL reads as 8 h.
    Returns (average, std_dev) and writes them back like the reference."""
    p = t.duration_prediction
    if p.ttl == 0:
        p.ttl = PREDICTION_TTL
    if p.value == 0 and t.expected_duration != 0:
        p.value = t.expected_duration
        p.collected_at = now - MINUTE
        return t.expected_duration, t.expected_duration_std_dev
    age = (2 ** 63 - 1) if p.collected_at == ZERO_TIME else now - p.collected_at
    if age < p.ttl:
        avg, std = p.value, p.std_dev
    else:
        if history is None:
            avg, std = (DEFAULT_TASK_DURATION, 0) if p.value == 0 else (p.value, p.std_dev)
        elif duration_from_float(history[0]) == 0:
            avg, std = DEFAULT_TASK_DURATION, 0
        else:
            avg, std = duration_from_float(history[0]), duration_from_float(history[1])
        p.value, p.std_dev, p.collected_at = avg, std, now
    t.expected_duration, t.expected_duration_std_dev = avg, std
    return avg, std
