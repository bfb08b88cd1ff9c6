/*
 * evg_sched.h -- C-ABI of libevgsched.so: the H100 (sm_90a) implementation of
 * Evergreen's scheduler hot path (scheduler.PlanDistro: tunable planner +
 * DistroQueueInfo + utilization host allocator), batched over distros.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch/CUDA types.
 * A Go maintainer binds it with cgo from package `scheduler` (INTEGRATION.md
 * shows the stub); the Python mirror in evergreen_b200/ binds it with ctypes.
 * Every entry point cites the reference interface it replaces; paths are
 * relative to the evergreen-ci/evergreen checkout.
 *
 * Layout: all distros of one scheduler tick are concatenated.  Distro d owns
 * tasks  [task_off[d],  task_off[d+1]),  hosts [host_off[d], host_off[d+1]) and
 * task-group slots [group_off[d], group_off[d+1]).  Indices inside a distro
 * (dep_idx, group_id, version_id, order[]) are distro-local.
 *
 * Determinism: `now_ns` replaces every time.Now()/time.Since on the path
 * (planner.go:318-322, scheduler.go:123, utilization_based_host_allocator.go:360).
 * Ties the reference leaves to map order / unstable sort are broken by the
 * canonical policy of DESIGN.md §3 (units: TotalValue desc, then the unit's
 * anchor -- the smallest input index among the tasks whose own key the unit is
 * filed under -- asc; tasks in a unit: the TaskList.Less chain, then input
 * index asc).
 *
 * There is no CPU fallback: every compute entry point fails with
 * EVG_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef EVG_SCHED_H
#define EVG_SCHED_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EVG_ABI_VERSION 1

/* Go's zero time.Time (year 1).  0 is the Unix epoch, which time.Time.IsZero
 * reports as NON-zero; other values are ns since the Unix epoch. */
#define EVG_TIME_ZERO INT64_MIN

/* library status codes (negative = failure; message via evg_last_error()) */
enum {
  EVG_OK = 0,
  EVG_ERR_INVALID = -1, /* bad argument / inconsistent offsets */
  EVG_ERR_CUDA = -2,    /* no usable sm_90 device, or a CUDA call failed */
  EVG_ERR_NOMEM = -3,   /* device or pinned allocation failed */
  EVG_ERR_STATE = -4    /* the resident tick cannot serve the call: there is none, or it lacks what the call needs
                           (its own columns, editability, hosts, dependency verdicts, alias map, resolved durations,
                           an allocator run since it was set, an evg_host_job on its current run) */
};

/* per-distro allocator status: the data errors UtilizationBasedHostAllocator
 * returns as `error` (utilization_based_host_allocator.go:151-160,200-202,302-304) */
enum {
  EVG_ALLOC_OK = 0,
  EVG_ALLOC_ERR_FUTURE_FRACTION = 1, /* future_host_fraction above 1 ("future host factor cannot be greater than 1"), below 0 or NaN */
  EVG_ALLOC_ERR_POOL_SIZE = 2,       /* "unable to plan hosts ... due to pool size" (maxHosts < 1) */
  EVG_ALLOC_ERR_PARENT_MISSING = 3   /* container pool parent distro not found */
};

/* evg_task_soa.flags */
#define EVG_TF_REQ_MASK 0x3u       /* requester class */
#define EVG_TF_REQ_OTHER 0u        /*   anything else -> mainline branch (planner.go:234) */
#define EVG_TF_REQ_PATCH 1u        /*   IsPatchRequester && !merge queue (globals.go:1179) */
#define EVG_TF_REQ_MERGE_QUEUE 2u  /*   IsGithubMergeQueueRequester (globals.go:1195) */
#define EVG_TF_GENERATE 0x4u       /* Task.GenerateTask */
#define EVG_TF_STEPBACK 0x8u       /* Task.ActivatedBy == "stepback" (globals.go:219) */
#define EVG_TF_DEPS_MET 0x10u      /* Task.DependenciesMet(...) (model/task/task.go:632) */
#define EVG_TF_OTHER_DISTRO 0x20u  /* Task.DistroId != distro id (scheduler.go:75) */

/* Task records, SoA (replaces []task.Task, model/task/task.go:83-350; the
 * fields are those SURVEY.md §8a row A20 lists).  48 B per task. */
typedef struct {
  int64_t n_tasks;
  int64_t n_edges;
  const int32_t* priority;         /* Task.Priority (int64 in Go; the shim saturates to int32) */
  const int64_t* expected_ns;      /* Task.FetchExpectedDuration(ctx).Average (task.go:3519) */
  const int64_t* queue_basis_ns;   /* ActivatedTime if !IsZero, else IngestTime if !IsZero, else EVG_TIME_ZERO (planner.go:318-322) */
  const int64_t* wait_basis_ns;    /* later of ScheduledTime, DependenciesMetTime (scheduler.go:119-122); EVG_TIME_ZERO if both zero */
  const int32_t* num_dependents;   /* Task.NumDependents */
  const int32_t* task_group_order; /* Task.TaskGroupOrder */
  const int32_t* group_id;         /* distro-local dense id of Task.GetTaskGroupString() (task.go:417); -1 when TaskGroup == "" */
  const int32_t* version_id;       /* distro-local dense id of Task.Version */
  const uint32_t* flags;           /* EVG_TF_* */
  /* Task.DependsOn restricted to dependencies that are themselves in this
   * distro's queue (planner.go:449-456), CSR over tasks; NULL when n_edges==0 */
  const int64_t* dep_off;          /* n_tasks + 1 */
  const int32_t* dep_idx;          /* distro-local index of the dependency */
} evg_task_soa;

/* distro.PlannerSettings (model/distro/distro.go:286-300), raw: the <=0 -> 1
 * clamp of the factor getters (distro.go:353-408) happens on the device. */
typedef struct {
  int64_t patch_factor;
  int64_t patch_time_in_queue_factor;
  int64_t commit_queue_factor;
  int64_t mainline_time_in_queue_factor;
  int64_t expected_runtime_factor;
  int64_t generate_task_factor;
  int64_t stepback_task_factor;
  double num_dependents_factor;
  int64_t target_time_ns;        /* d.GetTargetTime() (distro.go:434-440), resolved by the shim */
  int32_t group_versions;        /* PlannerSettings.ShouldGroupVersions() */
  int32_t includes_dependencies; /* DispatcherSettings.Version == "revised-with-dependencies" (scheduler.go:28) */
  int32_t n_versions;            /* number of distinct version ids in this distro */
  int32_t _reserved;
} evg_distro_cfg;

typedef struct {
  int32_t n_distros;
  int32_t _reserved;
  const int64_t* task_off;        /* n_distros + 1 */
  const int64_t* group_off;       /* n_distros + 1 */
  const evg_distro_cfg* cfg;      /* n_distros */
  const int32_t* group_max_hosts; /* per group slot: Task.TaskGroupMaxHosts of the group (scheduler.go:87-90) */
} evg_distro_table;

/* model.TaskGroupInfo without the name (model/task_queue.go:22-47); the name
 * of slot group_off[d]+g is the shim's string for group id g. 72 B. */
typedef struct {
  int64_t count;
  int64_t count_free;      /* written by the allocator (allocator.go:107-110); 0 when the distro's status is an error */
  int64_t count_required;  /* written by the allocator; 0 when the distro's status is an error */
  int64_t max_hosts;
  int64_t expected_duration;
  int64_t count_duration_over_threshold;
  int64_t count_wait_over_threshold;
  int64_t count_dep_filled_merge_queue_tasks;
  int64_t duration_over_threshold;
} evg_group_info;

/* model.DistroQueueInfo (model/task_queue.go:49-75).  `ungrouped` is the
 * TaskGroupInfo named "" (standalone tasks); it exists in TaskGroupInfos only
 * when has_ungrouped != 0. */
typedef struct {
  int64_t length;
  int64_t length_with_dependencies_met;
  int64_t count_dep_filled_merge_queue_tasks;
  int64_t expected_duration;
  int64_t max_duration_threshold;
  int64_t count_duration_over_threshold;
  int64_t duration_over_threshold;
  int64_t count_wait_over_threshold;
  int64_t secondary_queue; /* any task.DistroId != distro (scheduler.go:75-77); callers overwrite it (scheduler.go:44) */
  int64_t has_ungrouped;
  evg_group_info ungrouped;
} evg_queue_info;

/* task.SortingValueBreakdown flattened to 13 int64 (model/task/task.go:3990-4038) */
enum {
  EVG_BD_TASK_GROUP_LENGTH = 0, EVG_BD_TOTAL_VALUE,
  EVG_BD_P_INITIAL, EVG_BD_P_TASK_GROUP, EVG_BD_P_GENERATOR, EVG_BD_P_COMMIT_QUEUE,
  EVG_BD_R_COMMIT_QUEUE, EVG_BD_R_NUM_DEPENDENTS, EVG_BD_R_ESTIMATED_RUNTIME,
  EVG_BD_R_MAINLINE_WAIT, EVG_BD_R_STEPBACK, EVG_BD_R_PATCH, EVG_BD_R_PATCH_WAIT,
  EVG_BD_N
};

/* Planner outputs (replaces the []task.Task PrioritizeTasks returns,
 * scheduler.go:27, and the DistroQueueInfo of scheduler.go:43). */
typedef struct {
  int32_t* order;             /* [n_tasks] slot task_off[d]+r = distro-local index of the task ranked r (TaskPlan.Export, planner.go:462-481) */
  int64_t* total_value;       /* [n_tasks] SortingValueBreakdown.TotalValue of the unit the task was emitted from, rank order */
  int64_t* breakdown;         /* [n_tasks * EVG_BD_N] full breakdown in rank order, or NULL */
  evg_queue_info* info;       /* [n_distros] */
  evg_group_info* group_info; /* [group_off[n_distros]] */
} evg_plan_out;

/* evg_host_soa.flags */
#define EVG_HF_RUNNING 0x1u    /* Host.RunningTask != "" */
#define EVG_HF_TEARDOWN 0x2u   /* !Host.TaskGroupTeardownStartTime.IsZero() (host.go:219-221) */
#define EVG_HF_RT_FOUND 0x4u   /* the running task was returned by task.Find(ByIds) (allocator.go:337) */

/* host bucket codes for evg_host_soa.group_id (groupByTaskGroup, allocator.go:223-260) */
#define EVG_HG_NONE (-1)       /* name "" : no running task or no running task group */
#define EVG_HG_UNQUEUED (-2)   /* a named group with no TaskGroupInfo in the queue */

/* Existing hosts, SoA (replaces HostAllocatorData.ExistingHosts []host.Host,
 * host_allocator.go:17-23, model/host/host.go:79-88).  32 B per host. */
typedef struct {
  int64_t n_hosts;
  const uint32_t* flags;      /* EVG_HF_* */
  const int32_t* group_id;    /* EVG_HG_* or the distro-local task-group id of Host.GetTaskGroupString() (host.go:663) */
  const int64_t* expected_ns; /* running task FetchExpectedDuration().Average (allocator.go:357-358) */
  const int64_t* std_ns;      /* ... .StdDev (allocator.go:359) */
  const int64_t* start_ns;    /* running task StartTime (allocator.go:360), EVG_TIME_ZERO if unset */
} evg_host_soa;

enum { EVG_PROVIDER_STATIC = 0, /* not in evergreen.ProviderSpawnable (globals.go:723-728) */
       EVG_PROVIDER_EPHEMERAL = 1, /* ec2-ondemand, ec2-fleet, mock */
       EVG_PROVIDER_DOCKER = 2 };

/* distro.HostAllocatorSettings + the rest of HostAllocatorData that is not
 * hosts or queue info (model/distro/distro.go:267-280, host_allocator.go:17-23) */
typedef struct {
  double future_host_fraction;       /* outside [0, 1] (NaN included): EVG_ALLOC_ERR_FUTURE_FRACTION */
  int32_t provider;                   /* EVG_PROVIDER_* */
  int32_t disabled;                   /* Distro.Disabled */
  int32_t minimum_hosts;
  int32_t maximum_hosts;
  int32_t round_up;                   /* RoundingRule == "round-up" (allocator.go:174-177) */
  int32_t waits_over_thresh_feedback; /* FeedbackRule == "waits-over-thresh-feedback" (allocator.go:179-182) */
  int32_t has_pool;                   /* HostAllocatorData.ContainerPool != nil */
  int32_t pool_max_containers;        /* ContainerPool.MaxContainers */
  int32_t parent_found;               /* distro.FindOneId(pool.Distro) succeeded (allocator.go:151-158) */
  int32_t parent_maximum_hosts;       /* parent HostAllocatorSettings.MaximumHosts (allocator.go:159) */
} evg_alloc_cfg;

/* Allocator outputs (replaces the (int, int, error) of HostAllocator,
 * host_allocator.go:15).  `result` is the same data packed for the
 * multi-GPU all-gather: 16 B per distro.  Both counts fit their int32 fields:
 * new_hosts <= max(length_with_dependencies_met, minimum_hosts) and
 * 0 <= free_hosts <= the distro's host count.  The fraction is rejected
 * outside [0, 1], so every soon-to-be-free term lies in [0, 1] or, with a
 * threshold of 0, is NaN; a NaN sum floors to 0 (DESIGN.md §3 (iv)). */
typedef struct {
  int32_t new_hosts;   /* numNewHostsToRequest */
  int32_t free_hosts;  /* numFreeApprox (or len(freeHosts) on the early returns) */
  int64_t deficit_ns;  /* auxiliary: max(0, expected_duration - free_hosts*threshold), int64 with wrap: host-time the free pool cannot absorb */
} evg_alloc_result;

typedef struct {
  evg_alloc_result* result; /* [n_distros] */
  int32_t* status;          /* [n_distros] EVG_ALLOC_* */
} evg_alloc_out;

/* option bits */
#define EVG_OPT_BREAKDOWN 0x1u /* materialise evg_plan_out.breakdown */

typedef struct evg_ctx evg_ctx;

/* ---- lifecycle ---------------------------------------------------------- */

/* Bind a context to CUDA device `device`.  `stream` is a cudaStream_t the
 * kernels are launched on (e.g. the caller's torch stream) or NULL for a
 * private stream.  Replaces nothing in the reference (process bootstrap). */
int evg_init(int device, void* stream, evg_ctx** out);
void evg_shutdown(evg_ctx* ctx);
/* thread-local message for the last failing call on this thread */
const char* evg_last_error(void);
int evg_abi_version(void);

/* Pinned host buffers for the SoA columns (the Go shim fills C-allocated
 * memory so no Go pointer is retained across the call). */
void* evg_host_alloc(uint64_t bytes);
void evg_host_free(void* p);

/* ---- one-shot batch entry points: HOST pointers, H2D + kernels + D2H ---- */

/* Tunable planner + queue info for every distro of the tick.
 * Replaces: scheduler.PrioritizeTasks / runTunablePlanner minus persistence
 * (scheduler/scheduler.go:27-51): PrepareTasksForPlanning(...).Export
 * (planner.go:431-481) and GetDistroQueueInfo (scheduler.go:56-159). */
int evg_plan_batch(evg_ctx* ctx, const evg_task_soa* tasks, const evg_distro_table* distros,
                   int64_t now_ns, uint32_t opts, evg_plan_out* out);

/* Utilization host allocator for every distro, from queue infos the caller
 * already has (the reference reads them back from MongoDB,
 * units/host_allocator.go:152).  `groups` is in/out: count_free and
 * count_required are written like the reference mutates TaskGroupInfos.
 * Replaces: scheduler.UtilizationBasedHostAllocator
 * (scheduler/utilization_based_host_allocator.go:26-130) behind the
 * HostAllocator plug point (scheduler/host_allocator.go:15,25-32).
 * EVG_ERR_INVALID for a group_off that does not start at 0 or decreases, or a host_off that also misses n_hosts. */
int evg_alloc_batch(evg_ctx* ctx, const evg_host_soa* hosts, const int64_t* host_off,
                    const evg_alloc_cfg* cfg, const evg_queue_info* info, evg_group_info* groups,
                    const int64_t* group_off, int32_t n_distros, int64_t now_ns, evg_alloc_out* out);

/* Fused planner + allocator: the queue info never leaves the device.
 * Replaces: distroSchedulerJob.Run + hostAllocatorJob.Run for all distros of
 * one tick (units/scheduler.go:57-87, units/host_allocator.go:76-196). */
int evg_plan_and_alloc_batch(evg_ctx* ctx, const evg_task_soa* tasks, const evg_distro_table* distros,
                             const evg_host_soa* hosts, const int64_t* host_off,
                             const evg_alloc_cfg* acfg, int64_t now_ns, uint32_t opts,
                             evg_plan_out* plan_out, evg_alloc_out* alloc_out);

/* ---- resident API: inputs stay in HBM between ticks --------------------- */

/* Copy a tick's inputs into context-owned device buffers (hosts/host_off/acfg
 * may be NULL for planner-only use). */
int evg_upload(evg_ctx* ctx, const evg_task_soa* tasks, const evg_distro_table* distros,
               const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg);
/* Tick-to-tick update of the resident task table: row rows[i] (a task slot of the resident table, 0 <= rows[i] <
 * n_tasks) gets priority, num_dependents, task_group_order, flags, expected_ns, queue_basis_ns and wait_basis_ns of row i
 * of `values` (values->n_tasks == n_rows; its group / version / dependency columns are not read: a task keeps its
 * distro, its task group, its version and its in-queue dependency edges -- a tick that adds or removes tasks calls
 * evg_edit_tasks first).  48 bytes cross PCIe per changed row instead of the whole table.  Allowed on any tick in the
 * context's own columns: after evg_upload, evg_upload_with_deps, evg_edit_tasks, evg_plan_from_finder(_ex),
 * evg_plan_aliases, evg_plan_batch and evg_plan_and_alloc_batch; EVG_ERR_STATE without a tick or after
 * evg_upload_device (the caller owns those columns and edits them in place).  Drops the dependency verdicts of
 * evg_upload_with_deps.  Replaces nothing in the reference: there the scheduler re-reads every task document each tick
 * (scheduler/task_finder.go:40-197). */
int evg_update_tasks(evg_ctx* ctx, int64_t n_rows, const int64_t* rows, const evg_task_soa* values);

/* A change in queue membership between two ticks: rows leave, rows join, surviving tasks gain in-queue dependencies.
 * Host pointers. */
typedef struct {
  int64_t n_remove;
  const int64_t* remove_rows;   /* strictly ascending rows of the current resident table */
  const evg_task_soa* insert;   /* rows appended to their distro's queue after its survivors; n_tasks = rows inserted
                                   (NULL = none).  Group / version ids are in the new id space; dep_off / dep_idx are the
                                   rows' own in-queue edges as NEW distro-local indices */
  const int64_t* insert_off;    /* n_distros + 1: CSR of `insert` over distros */
  int64_t n_add_edges;          /* in-queue dependencies a SURVIVING task gains */
  const int64_t* add_edge_task; /* ascending NEW global row of a surviving task */
  const int32_t* add_edge_dep;  /* NEW distro-local index of the dependency (a survivor or an inserted row) */
  const int32_t* group_remap;   /* NULL = ids kept; else per OLD group slot: the new distro-local id, -1 = no survivor is in it */
  const int32_t* version_remap; /* NULL = ids kept; else per OLD (distro, version id), CSR by the old n_versions */
} evg_task_edit;

/* Tick-to-tick membership change of the resident task table, applied on the device: afterwards the context holds
 * exactly the tick a fresh evg_upload of the COMPOSED table would hold (outputs, evg_download_queue and the breakdown
 * match it bit for bit).  The composed table:
 *   - distro d's queue is its surviving rows in their previous order, then insert rows insert_off[d] .. insert_off[d+1];
 *   - a survivor keeps its group and version ids, or takes group_remap / version_remap of them;
 *   - a survivor's edges are its old edges whose dependency survived (re-indexed, in their old order), then its added
 *     edges in the order given; an inserted row's edges are its own;
 *   - `distros` is the new distro table: the same n_distros, task_off = old count - removed + inserted for every
 *     distro; cfg, group_off, group_max_hosts and n_versions may change as long as every id in use stays in range.
 * `hosts`, `host_off`, `acfg` as for evg_upload (NULL: planner only).  Only the edit crosses PCIe: the survivors are
 * gathered from the resident columns into a second column set the first edit allocates, which then becomes the
 * resident one.  A survivor cannot LOSE an in-queue dependency that stays in the queue (upload again for that), and
 * dependencies are not re-evaluated: pass EVG_TF_DEPS_MET for inserted rows and flip it for survivors with
 * evg_update_tasks.  Any device-side dependency state of evg_upload_with_deps is dropped.
 * Allowed after evg_upload, evg_upload_with_deps, evg_plan_from_finder(_ex), evg_edit_tasks and evg_plan_aliases;
 * EVG_ERR_STATE otherwise (no table, borrowed columns of evg_upload_device, the tick a one-shot call left).
 * EVG_ERR_INVALID for an edit the
 * host can reject (remove rows not strictly ascending or out of range, counts that disagree, another n_distros, an
 * added edge on a task that is not a survivor) leaves the previous tick resident and runnable; an id found out of range
 * on the device (or a survivor whose task group maps to -1) leaves no resident tick, as for evg_upload.
 * Replaces nothing in the reference: there the scheduler re-reads every task document each tick
 * (scheduler/task_finder.go:40-197). */
int evg_edit_tasks(evg_ctx* ctx, const evg_task_edit* edit, const evg_distro_table* distros,
                   const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg);

/* Like evg_upload, but the task columns already live in DEVICE memory (the finder's output, a generator kernel, a
 * previous tick edited in place): `tasks` holds device pointers, which the context borrows until the next upload or
 * evg_shutdown -- nothing is copied.  Every column must be 16-byte aligned and readable 8 elements past its last
 * row (the kernels read whole 128-bit vectors / TMA tiles).  `distros`, `hosts`, `host_off`, `acfg` are host
 * pointers as in evg_upload.  Replaces nothing in the reference (there the tasks are already in the process). */
int evg_upload_device(evg_ctx* ctx, const evg_task_soa* device_tasks, const evg_distro_table* distros,
                      const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg);
/* Launch the fused path on the resident inputs; asynchronous on the context
 * stream.  Safe to call repeatedly (each call recomputes from the inputs). */
int evg_run_resident(evg_ctx* ctx, int64_t now_ns, uint32_t opts);
/* Wait for the stream and copy results out; either pointer may be NULL. */
int evg_download(evg_ctx* ctx, evg_plan_out* plan_out, evg_alloc_out* alloc_out);
/* ---- the persisted queue (SURVEY.md §8 f.4) ---- */

#define EVG_QI_DEPS_MET 0x1u /* TaskQueueItem.DependenciesMet = Task.HasDependenciesMet() after GetDistroQueueInfo
                                stamped the task (scheduler.go:98,137; model/task/task.go:653,3393) */
/* The numeric half of model.TaskQueueItem (model/task_queue.go:131-153) for one persisted rank; the string half
 * (Id, DisplayName, BuildVariant, Requester, Revision, Project, Group, Version, ActivatedBy, Dependencies) is read by
 * the shim from its own []task.Task at index `task`.  40 B. */
typedef struct {
  int32_t task;            /* distro-local index of the task at this rank */
  int32_t group_index;     /* GroupIndex = Task.TaskGroupOrder */
  int32_t group_max_hosts; /* GroupMaxHosts = Task.TaskGroupMaxHosts (0 outside task groups) */
  uint32_t flags;          /* EVG_QI_* */
  int64_t priority;        /* Priority */
  int64_t expected_ns;     /* ExpectedDuration as GetDistroQueueInfo left it (scheduler.go:98) */
  int64_t total_value;     /* SortingValueBreakdown.TotalValue of the unit the task was emitted from (planner.go:475) */
} evg_queue_item;
#define EVG_PERSISTED_QUEUE_CAP 10000 /* TaskQueue.Save keeps the first 10 000 items (model/task_queue.go:216-219) */

/* After evg_run_resident: project the head of every distro's ranked queue -- the first min(length, cap) ranks, cap = 0
 * meaning EVG_PERSISTED_QUEUE_CAP -- into TaskQueueItem rows on the device and copy only those to the host.
 * item_off (n_distros + 1) receives the offsets of each distro's rows in `items`; `items_capacity` rows must be
 * available (sum over distros of min(length, cap); -EVG_ERR_INVALID with the needed count in evg_last_error otherwise).
 * Replaces: the TaskQueueItem projection and truncation of PersistTaskQueue / TaskQueue.Save
 * (scheduler/task_queue_persister.go:14-42, model/task_queue.go:216-219).  The upsert stays with the caller. */
int evg_download_queue(evg_ctx* ctx, int32_t cap, int64_t* item_off, evg_queue_item* items, int64_t items_capacity);

/* Device pointer to the resident evg_alloc_result[n_distros] vector, the
 * send buffer of the per-distro all-gather (SURVEY.md §8e). */
void* evg_device_result_ptr(evg_ctx* ctx);
/* Make the allocator kernel write its evg_alloc_result[] rows straight into a
 * caller-owned DEVICE buffer (e.g. the NCCL send buffer of the all-gather),
 * `capacity` rows long; NULL restores the context-owned buffer. */
int evg_bind_result_buffer(evg_ctx* ctx, void* device_ptr, int64_t capacity);
/* Number of kernels the context launched since the last call that reset the count; 0 for a NULL ctx.  These calls
 * reset it to 0 before their first launch: evg_run_resident (so evg_plan_batch, evg_plan_distro and the
 * evg_plan_and_alloc_batch it runs), evg_plan_and_alloc_batch's pipelined large ticks, evg_alloc_batch / evg_alloc_distro,
 * evg_deps_met_batch, evg_find_runnable_batch / _ex, evg_plan_from_finder / _ex, evg_edit_tasks, evg_plan_aliases,
 * evg_expected_durations_batch, evg_prioritize_legacy_batch, evg_dag_rebuild_batch, evg_rebuild_dispatchers,
 * evg_host_job, evg_host_drawdown, evg_idle_hosts, evg_find_next_batch, evg_find_next_tasks, evg_estimate_start_times and evg_estimate_start_batch.  Every other call adds the kernels it launches: the uploads (their range check), evg_update_tasks,
 * evg_download_queue and evg_resolve_durations. */
int64_t evg_last_launch_count(evg_ctx* ctx);
/* Device time in ms of the last evg_run_resident, from CUDA events on the context
 * stream (valid after a sync / download): total_ms spans the whole tick; sort_ms is
 * the general path's segmented radix sort when the tick had a distro above 12288
 * tasks, otherwise the k_plan_smem<1024,12> launch (see evg_kernel_timing_ms). */
int evg_last_timing_ms(evg_ctx* ctx, float* total_ms, float* sort_ms);

/* Device time in ms of the dominant kernel of on-chip ticks -- k_plan_cta<512,10240>, the on-chip planner of distros
 * with 5121..10240 tasks (or k_plan_smem<1024,12> when the tick has none) -- for each of the last `n`
 * evg_run_resident calls that launched it (n <= 128), from CUDA events recorded around that launch on its stream. */
int evg_kernel_timing_ms(evg_ctx* ctx, float* out_ms, int32_t n);

/* The general path's two big stages in the last evg_run_resident (ms, CUDA events on its stream): the per-task
 * pass k_gtask (reads every input column once) and the segmented radix sort (all passes). */
int evg_general_timing_ms(evg_ctx* ctx, float* task_pass_ms, float* sort_ms);

/* ---- dependency filter (SURVEY.md §8f.1: the next row after the planner/allocator path) ---- */

/* evg_deps_in.dep_kind */
#define EVG_DEP_IN_QUEUE 0  /* dep_ref = index (in this call's task table) of the dependency; its state is task_state[dep_ref] */
#define EVG_DEP_EXTERNAL 1  /* dep_ref indexes ext_state[] (the dependency was fetched from the tasks collection) */
#define EVG_DEP_MISSING 2   /* lookup failed: never met (checkDependenciesMet, scheduler/scheduler.go:161-168) */
/* evg_deps_in.dep_want: Dependency.Status */
#define EVG_WANT_SUCCESS 0  /* "success" or "" (model/task/task.go:533-534) */
#define EVG_WANT_FAILED 1   /* "failed" */
#define EVG_WANT_ANY 2      /* "*" AllStatuses: failed, succeeded or blocked (task.go:537-538) */
#define EVG_WANT_OTHER 3    /* any other string: never satisfied */
/* task_state / ext_state bits */
#define EVG_TS_STATUS_MASK 0x3u /* 0 "success", 1 "failed", 2 anything else */
#define EVG_TS_BLOCKED 0x4u     /* Task.Blocked() (task.go:3649-3660) */
/* task_pre bits: Task.HasDependenciesMet short-circuits (task.go:3393-3395) */
#define EVG_TP_OVERRIDE 0x1u    /* OverrideDependencies */
#define EVG_TP_MET_TIME 0x2u    /* !utility.IsZeroTime(DependenciesMetTime) */

/* All DIRECT dependencies of every task, CSR over tasks. */
typedef struct {
  int64_t n_tasks;
  int64_t n_deps;
  const int64_t* dep_off;   /* n_tasks + 1 */
  const uint8_t* dep_kind;  /* EVG_DEP_* */
  const int32_t* dep_ref;
  const uint8_t* dep_want;  /* EVG_WANT_* */
  const uint8_t* task_state;/* n_tasks, EVG_TS_* of the in-queue tasks themselves */
  const uint8_t* task_pre;  /* n_tasks, EVG_TP_* */
  const uint8_t* ext_state; /* n_ext, EVG_TS_* */
  int64_t n_ext;
} evg_deps_in;

/* met[t] = Task.DependenciesMet(ctx, depCache) for every task (model/task/task.go:632-671 with
 * SatisfiesDependency :529-543): the bit evg_task_soa.flags carries as EVG_TF_DEPS_MET and the predicate the
 * task finders filter on (scheduler/task_finder.go:40-197).  Host pointers in and out.
 * EVG_ERR_INVALID for a dep_ref out of range or a dep_off that does not start at 0, end at n_deps and never decrease:
 * the host checks its ends, k_deps_met every row before it reads the row's entries. */
int evg_deps_met_batch(evg_ctx* ctx, const evg_deps_in* in, uint8_t* met);

/* evg_upload with the dependency predicate evaluated ON THE DEVICE and wired into the planner's inputs: after the
 * copy, Task.DependenciesMet runs for every task (same tables as evg_deps_met_batch, over the same n_tasks tasks) and
 *   - the EVG_TF_DEPS_MET bit of the resident flags column is set from its verdict (the caller's bit is ignored);
 *   - a task whose dependencies were evaluated afresh and found met is stamped like Task.setDependenciesMetTime does
 *     (model/task/task.go:653,673-684): the latest non-zero dep_finished_ns[] (Dependency.FinishedAt, per dependency,
 *     NULL = unknown) of its dependencies, else now_ns; its resident wait basis becomes the later of the caller's
 *     wait_basis_ns (ScheduledTime) and that stamp (scheduler.go:119-122).
 * Neither the bit nor the stamp visits the host; evg_download_deps returns them for the write-back the reference does
 * (UpdateOne of DependenciesMetTime, task.go:659-666).  `deps` is checked as by evg_deps_met_batch; a table rejected on
 * the device leaves no resident tick.
 * Replaces: checkDependenciesMet inside GetDistroQueueInfo (scheduler/scheduler.go:82-98,161-168). */
int evg_upload_with_deps(evg_ctx* ctx, const evg_task_soa* tasks, const evg_distro_table* distros,
                         const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg,
                         const evg_deps_in* deps, const int64_t* dep_finished_ns, int64_t now_ns);
/* met[t] = Task.DependenciesMet; met_time_ns[t] = the stamp (EVG_TIME_ZERO when nothing was stamped).  Either may be NULL.
 * EVG_ERR_STATE without a tick; EVG_OK for a tick of no rows; then EVG_ERR_STATE unless the tick's verdicts are
 * evg_upload_with_deps' (evg_deps_met_batch and evg_update_tasks drop them; evg_resolve_durations and
 * evg_rebuild_dispatchers keep them). */
int evg_download_deps(evg_ctx* ctx, uint8_t* met, int64_t* met_time_ns);

/* ---- runnable-task filter: the task finders (SURVEY.md §8f.1) ------------- */

/* evg_runnable_in.sched: what schedulableHostTasksQuery (model/task/db.go:671-689) and ProjectCanDispatchTask read of a task */
#define EVG_SQ_ACTIVATED 0x01u      /* Activated */
#define EVG_SQ_UNDISPATCHED 0x02u   /* Status == "undispatched" */
#define EVG_SQ_PRIORITY_OK 0x04u    /* Priority > DisabledTaskPriority (-1) */
#define EVG_SQ_HOST_PLATFORM 0x08u  /* ByExecutionPlatform(host): field absent or "host" (db.go:647-663) */
#define EVG_SQ_UNATTAINABLE 0x10u   /* UnattainableDependency */
#define EVG_SQ_OVERRIDE_DEPS 0x20u  /* OverrideDependencies */
#define EVG_SQ_GITHUB_PR 0x40u      /* Requester == "github_pull_request" */
#define EVG_SQ_PATCH_REQUEST 0x80u  /* Task.IsPatchRequest() (model/task/task.go:545-547) */
/* evg_runnable_in.project_flags: ProjectRef fields ProjectCanDispatchTask reads (model/project_ref.go:3441-3462) */
#define EVG_PF_ENABLED 0x1u
#define EVG_PF_HIDDEN 0x2u
#define EVG_PF_DISPATCHING_DISABLED 0x4u
#define EVG_PF_PATCHING_DISABLED 0x8u
/* evg_runnable_in.finder, per distro */
#define EVG_FINDER_NO_DEPS 0    /* DispatcherSettings.Version == "revised-with-dependencies": dependencies are not filtered (task_finder.go:85) */
#define EVG_FINDER_LEGACY 1     /* LegacyFindRunnableTasks: Task.DependenciesMet, with the HasDependenciesMet short-circuit */
#define EVG_FINDER_ALTERNATE 2  /* AlternateTaskFinder / ParallelTaskFinder: Task.AllDependenciesSatisfied (task.go:795-821), no short-circuit */
/* RunnableTasksPipeline (task.FindHostRunnable, model/task/db.go:887-1066): only through the *_ex entry points, which
 * take an evg_pipeline_in.  Project gating reads the RAW project_ref document (evg_pipeline_in.project_raw), not the
 * merged ref of project_flags: enabled stored true, dispatching_disabled not true, and a PatchRequesters task needs
 * patching_disabled stored false (no hidden-project exemption). */
#define EVG_FINDER_PIPELINE 3          /* removeDeps: the $graphLookup dependency filter (db.go:923-996) */
#define EVG_FINDER_PIPELINE_NO_DEPS 4  /* DispatcherSettings.Version == "revised-with-dependencies" on the pipeline finder */

/* Every candidate task of every distro (the rows task.FindHostSchedulable would be asked about), concatenated. */
typedef struct {
  int64_t n_tasks;
  int32_t n_distros;
  int32_t n_projects;
  const int64_t* task_off;      /* n_distros + 1 */
  const uint8_t* sched;         /* n_tasks, EVG_SQ_* */
  const int32_t* project;       /* n_tasks: row of project_flags, or -1 when the project-ref cache has no such project */
  const uint8_t* project_flags; /* n_projects, EVG_PF_* */
  const int64_t* valid_off;     /* n_distros + 1: CSR of Distro.ValidProjects as project rows (-1 = a name no ref has) */
  const int32_t* valid_idx;
  const uint8_t* finder;        /* n_distros, EVG_FINDER_* */
  const evg_deps_in* deps;      /* direct dependencies of the same n_tasks tasks; NULL when every finder is NO_DEPS */
} evg_runnable_in;

/* LegacyFindRunnableTasks / AlternateTaskFinder / ParallelTaskFinder (scheduler/task_finder.go:40-317) over all
 * distros at once: runnable[task_off[d] .. task_off[d] + count[d]) holds the distro-local indices of the tasks
 * the finder returns for distro d, in input order (the reference appends in query order); the rest of the
 * distro's slots are -1.  Host pointers.  EVG_ERR_INVALID for a task_off that does not start at 0, end at n_tasks and
 * never decrease, a valid_off that does not start at 0 or decreases, a project row out of range, or in->deps rejected
 * as by evg_deps_met_batch. */
int evg_find_runnable_batch(evg_ctx* ctx, const evg_runnable_in* in, int32_t* runnable, int64_t* count);

/* The finder's output feeds the planner without leaving the device.  `in` describes every CANDIDATE task of every
 * distro as for evg_find_runnable_batch (in->deps is required: the planner's EVG_TF_DEPS_MET bit comes from it);
 * `candidates` holds the same rows' planner columns (flags without EVG_TF_DEPS_MET, wait_basis_ns = ScheduledTime,
 * in-queue dependency edges between candidates as distro-local candidate indices); `distros` is the distro table over
 * the candidates (task_off == in->task_off; group / version ids may name groups no kept task is in).  On the device:
 * k_deps_met (both predicates, DependenciesMetTime stamps from dep_finished_ns, as evg_upload_with_deps) -> the finders
 * -> EVG_TF_DEPS_MET and the stamped wait basis applied to the candidates' columns -> the compaction evg_edit_tasks
 * uses, with the dropped candidates removed and nothing inserted: the kept rows in their order, and the dependency
 * edges whose two ends were kept, re-indexed.  The kept table becomes the context's resident tick, in its own columns:
 * call evg_run_resident / evg_download next (evg_update_tasks and evg_edit_tasks may follow, as after evg_upload); ranks
 * refer to the compacted queues, and `runnable` (n_tasks, may be NULL) / `count` (n_distros) map them back exactly as
 * evg_find_runnable_batch reports them.  The only values the host reads in between are the n_distros counts (the
 * routing needs queue lengths).  EVG_ERR_INVALID for `in` rejected as by evg_find_runnable_batch, a candidate dep_off
 * that does not start at 0, end at n_edges and never decrease, a dep_idx outside its distro's candidates, or a
 * distros->group_off / host_off rejected as by evg_upload.
 * Replaces: the finder + checkDependenciesMet + PrioritizeTasks hand-over inside scheduler.PlanDistro
 * (scheduler/wrapper.go:60-118, scheduler/scheduler.go:56-168), where the filtered []task.Task is rebuilt on the host. */
int evg_plan_from_finder(evg_ctx* ctx, const evg_runnable_in* in, const evg_task_soa* candidates, const evg_distro_table* distros,
                         const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg,
                         const int64_t* dep_finished_ns, int64_t now_ns, int32_t* runnable, int64_t* count);

/* ---- the pipeline finder (RunnableTasksPipeline, scheduler/task_finder.go:34-36) ---- */

/* Status strings are interned by the shim; these ids are reserved. */
#define EVG_STATUS_SUCCESS 0 /* "success" */
#define EVG_STATUS_FAILED 1  /* "failed" */
#define EVG_STATUS_ANY 2     /* "*" (a Dependency.Status only) */
/* evg_pipeline_in.project_raw: the raw project_ref document the $lookup joins (db.go:998-1028) */
#define EVG_PR_ENABLED 0x1u              /* enabled stored true */
#define EVG_PR_DISPATCHING_DISABLED 0x2u /* dispatching_disabled stored true */
#define EVG_PR_PATCHING_FALSE 0x4u       /* patching_disabled stored false (unset is NOT false: *bool,omitempty) */

/* What the pipeline finder reads that evg_runnable_in cannot express.  The dependency documents are the entries of
 * in->deps: an EVG_DEP_IN_QUEUE entry's document is candidate dep_ref, an EVG_DEP_EXTERNAL one ext row dep_ref (any
 * document of the tasks collection, not only the queue's), and EVG_DEP_MISSING means no document has that id.
 * in->deps->dep_want, task_state, task_pre and ext_state are not read by the pipeline's own filter. */
typedef struct {
  int32_t n_status;                 /* interned status strings: ids 0 .. n_status-1, n_status >= 3 */
  int32_t _reserved;
  const int32_t* dep_status;        /* deps->n_deps: Dependency.Status */
  const int32_t* task_status;       /* n_tasks: Task.Status of each candidate */
  const int32_t* ext_status;        /* deps->n_ext: Task.Status of each external document */
  const uint8_t* task_unattainable; /* n_tasks: 1 when some entry of the candidate's own depends_on has unattainable: true */
  const uint8_t* ext_unattainable;  /* deps->n_ext: the same for each external document */
  const uint8_t* project_raw;       /* n_projects: EVG_PR_* of the raw project_ref document of each project row */
} evg_pipeline_in;

/* evg_find_runnable_batch with the pipeline finder available to any distro.  For an EVG_FINDER_PIPELINE distro a
 * candidate passes schedulableHostTasksQuery and ValidProjects as the other finders, the raw project gating above, and
 * the dependency filter: every DependsOn entry whose document EXISTS is satisfied -- its Status equals the document's
 * Status exactly, or it is "*" and the document is "success" / "failed" or has an unattainable depends_on entry --
 * entries without a document are ignored, a candidate whose entries ALL lack a document is dropped, one without
 * DependsOn is kept; OverrideDependencies and DependenciesMetTime do not help.  EVG_FINDER_PIPELINE_NO_DEPS distros
 * apply the gating without the dependency filter.  Output order: candidate order, as for the other finders.
 * pipe == NULL behaves exactly like evg_find_runnable_batch.  EVG_ERR_INVALID: a pipeline code with pipe == NULL, a
 * pipeline distro without in->deps, a status id outside [0, n_status), n_status < 3, and what evg_find_runnable_batch
 * rejects (k_pl_deps checks the rows of in->deps->dep_off as k_deps_met does).  Host pointers. */
int evg_find_runnable_ex(evg_ctx* ctx, const evg_runnable_in* in, const evg_pipeline_in* pipe, int32_t* runnable,
                         int64_t* count);

/* evg_plan_from_finder with the pipeline finder available (pipe == NULL: exactly evg_plan_from_finder).  What the
 * planner receives is what PlanDistro hands PrioritizeTasks after the aggregation's decode:
 *   - EVG_FINDER_PIPELINE: a kept task's DependsOn decodes empty ($unwind leaves one sub-document, which mgo skips), so
 *     its in-queue edges are dropped and EVG_TF_DEPS_MET is set without a DependenciesMetTime stamp;
 *   - EVG_FINDER_PIPELINE_NO_DEPS: DependenciesMet and its stamp are evaluated after the finder, with the Blocked()
 *     state of a dependency that is a KEPT candidate of the same distro ignored ($project strips
 *     depends_on.unattainable from the returned tasks, db.go:916-921, and they form the depCache, scheduler.go:61-64).
 * Everything else as evg_plan_from_finder; the candidate edges of EVG_FINDER_PIPELINE rows are not read. */
int evg_plan_from_finder_ex(evg_ctx* ctx, const evg_runnable_in* in, const evg_pipeline_in* pipe, const evg_task_soa* candidates,
                            const evg_distro_table* distros, const evg_host_soa* hosts, const int64_t* host_off,
                            const evg_alloc_cfg* acfg, const int64_t* dep_finished_ns, int64_t now_ns, int32_t* runnable,
                            int64_t* count);

/* ---- alias queues: the secondary queue of every distro (SURVEY.md §8 row A21) ---- */

/* The tick's schedulable tasks, each ONCE (not once per queue it may join).  Host pointers. */
typedef struct {
  /* planner columns of the n_tasks source rows: group_id / version_id are TABLE-GLOBAL dense ids (what
   * evg_intern_columns gives for the table as one distro), flags without EVG_TF_DEPS_MET and EVG_TF_OTHER_DISTRO (both
   * are set on the device), wait_basis_ns = ScheduledTime as for evg_upload_with_deps; dep_off / dep_idx are the entries
   * of Task.DependsOn that are rows of this table, as row indices, in DependsOn order with duplicates */
  evg_task_soa tasks;
  int32_t n_groups;                    /* global task groups */
  int32_t n_versions;                  /* global versions */
  const int32_t* group_max_hosts;      /* n_groups: TaskGroupMaxHosts of the group */
  const uint8_t* sched;                /* n_tasks: EVG_SQ_* (the schedulableHostTasksQuery bits) */
  const int32_t* task_group_max_hosts; /* n_tasks: raw Task.TaskGroupMaxHosts (== 1 keeps a task out, task group or not) */
  const int32_t* primary;              /* n_tasks: distro index of Task.DistroId, -1 when it is not in the distro table */
  const int64_t* secondary_off;        /* n_tasks + 1: CSR of Task.SecondaryDistros over the rows */
  const int32_t* secondary_idx;        /* name index of each entry, -1 for a name no distro has */
  int32_t n_names;
  int32_t _reserved;
  const int64_t* dest_off;             /* n_names + 1: CSR over names of the distros e whose {e} U e.Aliases holds the name */
  const int32_t* dest_idx;             /* distro index */
  const evg_deps_in* deps;             /* direct dependencies of the same n_tasks rows (required) */
  const int64_t* dep_finished_ns;      /* per deps entry: Dependency.FinishedAt (NULL = unknown) */
} evg_alias_in;

typedef struct {
  int64_t* task_off;   /* n_distros + 1: offsets of the alias queues in the resident tick */
  int64_t* group_off;  /* n_distros + 1: their task-group slots */
  int32_t* n_versions; /* n_distros */
} evg_alias_out;

/* task.FindHostSchedulableForAlias + scheduler.PrioritizeTasks(..., IsSecondaryQueue) for every distro at once.  Task t
 * is in distro e's alias queue iff t passes schedulableHostTasksQuery (ACTIVATED, UNDISPATCHED, PRIORITY_OK,
 * HOST_PLATFORM, and not UNATTAINABLE unless OVERRIDE_DEPS), task_group_max_hosts != 1, and some name of t's
 * SecondaryDistros is e or one of e's aliases -- once, however many names match.  Each alias queue lists its tasks in
 * ascending source row; its task groups and versions get dense ids in first-appearance order, as evg_intern_columns
 * assigns them; a task's in-queue edges are its dependencies that are in the same alias queue.  Task.DependenciesMet and
 * the DependenciesMetTime stamp are evaluated once per row (as evg_upload_with_deps does) and serve every queue the row
 * joins; EVG_TF_OTHER_DISTRO is set per queue (primary[t] != e).  cfg[e] is alias distro e's planner settings (its
 * n_versions is ignored: the device counts them).  The alias queues become the context's resident tick, planner only
 * (no hosts): evg_run_resident, evg_download, evg_download_queue, evg_update_tasks and evg_edit_tasks work on it as
 * after evg_upload; evg_download_alias_map maps its rows back to source rows.
 * What crosses PCIe: the source table once (host to device); in between, the host reads one count, then the queue,
 * group, version and edge offsets of every distro and the group_max_hosts of every alias group slot -- O(n_distros +
 * alias groups) values, nothing per task.
 * EVG_ERR_INVALID, previous tick still resident and runnable: negative sizes, null arrays, sizes that disagree, a CSR
 * (secondary_off, dest_off, tasks.dep_off) that does not start at 0, end at its entry count and never decrease, a
 * dest_idx outside [0, n_distros).  EVG_ERR_INVALID with no resident tick: deps rejected as by evg_deps_met_batch, an
 * id found out of range on the device (secondary_idx, primary, group_id, version_id, dep_idx, dep_ref), more than
 * 2^31-2 (queue, task) pairs, or an alias queue above 2^21-1 tasks.
 * Replaces: distroAliasSchedulerJob.Run for every distro (units/scheduler_alias.go:55-117): FindHostSchedulableForAlias
 * (model/task/task.go:3371-3386, model/distro/aliases.go:14-27) and PrioritizeTasks (scheduler/scheduler.go:27-51). */
int evg_plan_aliases(evg_ctx* ctx, const evg_alias_in* in, const evg_distro_cfg* cfg, int32_t n_distros, int64_t now_ns,
                     evg_alias_out* out);
/* After evg_plan_aliases (and evg_update_tasks, evg_resolve_durations, evg_rebuild_dispatchers): source_row[r] = the source row of resident row r (task_off[n_distros]
 * entries), group_source[s] = the global group id of alias group slot s (group_off[n_distros] entries).  Either may be
 * NULL.  EVG_ERR_STATE once another call replaced the tick's rows. */
int evg_download_alias_map(evg_ctx* ctx, int32_t* source_row, int32_t* group_source);

/* ---- host-side string interning for the marshaller ------------------------ */

/* A column of n strings: bytes[off[i] .. off[i+1]) is string i (not NUL-terminated). */
typedef struct {
  const char* bytes;
  const int64_t* off; /* n + 1 */
} evg_str_col;

/* The strings of a tick's tasks, concatenated distro by distro like evg_task_soa. */
typedef struct {
  int64_t n_tasks;
  int32_t n_distros;
  const int64_t* task_off;          /* n_distros + 1 */
  evg_str_col id;                   /* Task.Id */
  evg_str_col version;              /* Task.Version */
  evg_str_col group_key;            /* Task.GetTaskGroupString() (model/task/task.go:417-419); "" when Task.TaskGroup == "" */
  const int32_t* group_max_hosts;   /* Task.TaskGroupMaxHosts, n_tasks */
  const int64_t* dep_off;           /* n_tasks + 1: CSR over Task.DependsOn */
  evg_str_col dep_id;               /* Dependency.TaskId, dep_off[n_tasks] strings */
} evg_string_cols;

/* What the planner's columns need of those strings; every array is caller-allocated. */
typedef struct {
  int32_t* group_id;        /* n_tasks: dense per distro in first-appearance order, -1 without a task group */
  int32_t* version_id;      /* n_tasks: dense per distro in first-appearance order */
  int64_t* group_off;       /* n_distros + 1 */
  int32_t* n_versions;      /* n_distros */
  int32_t* group_max_hosts; /* capacity n_tasks: one per group slot, group_off[n_distros] used */
  int64_t* group_first;     /* capacity n_tasks: row of each group's first member (its name is group_key there) */
  int64_t* dep_off;         /* n_tasks + 1: in-queue dependency edges (planner.go:449-456) */
  int32_t* dep_idx;         /* capacity dep_off_in[n_tasks]: distro-local index of the dependency; targets outside the queue are dropped */
} evg_intern_out;

/* String work of marshalling a tick (scheduler.PrioritizeTasks builds the same maps while it walks a queue:
 * planner.go:431-456 files units under exactly these strings): group keys and versions to dense ids, dependency ids
 * to queue indices, per distro, `threads` distros at a time (<= 0: hardware concurrency).  Host only: no context.
 * EVG_ERR_INVALID when members of one task group disagree on TaskGroupMaxHosts (evg_last_error names the row), for a
 * task_off that does not start at 0, end at n_tasks and never decrease, and for a dep_off that does not start at 0 or
 * decreases. */
int evg_intern_columns(const evg_string_cols* in, evg_intern_out* out, int32_t threads);

/* ---- expected-duration statistics (SURVEY.md §8f.2) ----------------------- */

/* evg_duration_rows.flags */
#define EVG_DR_COMPLETED 0x1u  /* Status in evergreen.TaskCompletedStatuses (expected_duration.go:41-43) */
#define EVG_DR_TIMED_OUT 0x2u  /* Details.TimedOut == true (excluded, :44-46) */

/* Finished tasks (one row each) of any number of (project, build variant) windows at once; `key` interns the
 * group-by key -- (project, build variant, display name) -- so one call replaces one aggregation per pair. */
typedef struct {
  int64_t n_rows;
  int32_t n_keys;
  int32_t _reserved;
  const int32_t* key;            /* n_rows: 0 .. n_keys-1 */
  const int64_t* time_taken_ns;  /* n_rows: Task.TimeTaken */
  const int64_t* start_ns;       /* n_rows: Task.StartTime (UnixNano) */
  const int64_t* finish_ns;      /* n_rows: Task.FinishTime */
  const uint8_t* flags;          /* n_rows: EVG_DR_* */
  int64_t window_start_ns;       /* $match: StartTime > window_start && FinishTime <= window_end (:47-52) */
  int64_t window_end_ns;
} evg_duration_rows;

/* One group of the $group stage (expected_duration.go:66-76): {$avg, $stdDevPop} of TimeTaken.  count == 0 means the
 * aggregation returns no document for the key.  mean_ns = double(sum) / double(count); stddev_ns = sqrt(variance)
 * with the variance accumulated EXACTLY in integers around floor(mean) and rounded once at the end (MongoDB's
 * streaming Welford update differs from it in the last few ulps; the reference's own test allows 0.01 minutes). */
typedef struct {
  int64_t count;
  double mean_ns;
  double stddev_ns;
} evg_duration_stat;

/* getExpectedDurationsForWindow (model/task/expected_duration.go:36-96) for every key at once.  Host pointers. */
int evg_expected_durations_batch(evg_ctx* ctx, const evg_duration_rows* in, evg_duration_stat* out);

/* ---- the duration cache of a resident tick (SURVEY.md §8 rows A3/A4) ------- */

/* evg_duration_cache.key: the history key of (Project, BuildVariant, DisplayName), or one of these */
#define EVG_DK_NONE (-1)          /* no history row has the key: the window query returns no document */
#define EVG_DK_PAIR(p) (-2 - (p)) /* DisplayName == "": no name filter, the rows of (Project, BuildVariant) pair p grouped by
                                     name (expected_duration.go:54-56): one document exactly when ONE key of the pair matched */
/* evg_duration_out.source: which branch of Task.FetchExpectedDuration decided the row; every source but FRESH is persisted */
#define EVG_DS_FRESH 0     /* CachedDurationValue.Get: since(CollectedAt) < TTL, the cached value (cached_value.go:127-129) */
#define EVG_DS_BACKFILL 1  /* Value == 0 && ExpectedDuration != 0 (task.go:3524-3538) */
#define EVG_DS_HISTORY 2   /* stale, one document with a non-zero truncated $avg (task.go:3564-3569) */
#define EVG_DS_PREVIOUS 3  /* stale, not exactly one document, previous Value != 0 (task.go:3556-3562) */
#define EVG_DS_DEFAULT 4   /* stale: defaultTaskDuration (10 min, 0), no document and Value == 0 or a $avg truncating to 0 */

/* What FetchExpectedDuration reads of one task, for the listed rows of a resident table.  Host pointers. */
typedef struct {
  int64_t n_rows;
  const int64_t* rows;            /* strictly ascending resident rows (tasks or hosts); NULL = every row in order (a non-NULL list may be empty) */
  const int64_t* value_ns;        /* DurationPrediction.Value */
  const int64_t* std_ns;          /* DurationPrediction.StdDev */
  const int64_t* ttl_ns;          /* DurationPrediction.TTL; 0 = predictionTTL (8 h) -- a shim that wants
                                     utility.JitterInterval (task.go:3520-3522) passes its own draw instead */
  const int64_t* collected_ns;    /* DurationPrediction.CollectedAt, EVG_TIME_ZERO = zero time */
  const int64_t* expected_ns;     /* Task.ExpectedDuration */
  const int64_t* expected_std_ns; /* Task.ExpectedDurationStdDev */
  const int32_t* key;             /* history key, EVG_DK_NONE or EVG_DK_PAIR(p) */
} evg_duration_cache;

typedef struct {
  const evg_duration_rows* history; /* finished tasks; keys numbered pair-major (the keys of pair p are
                                       pair_key_off[p] .. pair_key_off[p+1]); window (now - 1 week, now]
                                       (taskCompletionEstimateWindow, task.go:3543-3544); NULL = no rows */
  int32_t n_pairs;
  int32_t _reserved;
  const int64_t* pair_key_off;      /* n_pairs + 1 */
  const evg_duration_cache* tasks;  /* rows of the resident task table; NULL leaves expected_ns as uploaded */
  const evg_duration_cache* hosts;  /* running tasks of the resident hosts; NULL leaves expected_ns / std_ns */
} evg_duration_in;

/* Per listed row, in listed-row order.  Any pointer may be NULL. */
typedef struct {
  int64_t* avg_ns;       /* the DurationStats returned = Task.ExpectedDuration afterwards */
  int64_t* std_ns;       /* ... .StdDev = Task.ExpectedDurationStdDev afterwards */
  int64_t* value_ns;     /* DurationPrediction after the call; persisted as ExpectedDuration (task.go:900) */
  int64_t* pred_std_ns;  /* ... StdDev; persisted as ExpectedDurationStdDev (task.go:901), even for BACKFILL */
  int64_t* collected_ns; /* ... CollectedAt */
  uint8_t* source;       /* EVG_DS_* */
} evg_duration_out;

/* Task.FetchExpectedDuration (model/task/task.go:3519-3590 with CachedDurationValue.Get, util/cached_value.go:125-145,
 * and getExpectedDurationsForWindow, expected_duration.go:36-96) for listed rows of the resident tick, the clock frozen
 * at now_ns.  The statistics of every key are computed on the device, decided per row, and the result written into
 * the resident planner column expected_ns (tasks) and the allocator columns expected_ns / std_ns (hosts); nothing
 * goes back to the host but the error word.  Allowed whenever the context holds its own resident tick (after evg_upload,
 * evg_upload_with_deps, evg_edit_tasks, evg_plan_from_finder(_ex) and evg_plan_aliases); the tick keeps everything else
 * (dependency verdicts, the alias map, evg_update_tasks / evg_edit_tasks afterwards).  EVG_ERR_STATE: no tick, borrowed
 * columns (evg_upload_device), the tick a one-shot call left, hosts != NULL on a tick without hosts.  EVG_ERR_INVALID with the tick untouched: rows out
 * of range or not strictly ascending, n_rows != the resident count when rows == NULL, a pair_key_off that does not start
 * at 0, end at n_keys and never decrease, null columns, and -- found on the device -- a key or pair out of range.
 * Replaces: PopulateCaches -> Task.FetchExpectedDuration (scheduler/setup_funcs.go:20-67) and the running-task
 * durations of the host allocator (utilization_based_host_allocator.go:357-359). */
int evg_resolve_durations(evg_ctx* ctx, const evg_duration_in* in, int64_t now_ns);
/* After evg_resolve_durations: its per-row results, listed-row order; either pointer may be NULL.  EVG_ERR_STATE once
 * another call replaced the tick's rows, or when the last evg_resolve_durations was rejected on the device. */
int evg_download_durations(evg_ctx* ctx, evg_duration_out* tasks, evg_duration_out* hosts);

/* ---- legacy comparator prioritiser (SURVEY.md §8 row L) ---------------------- */

/* evg_legacy_soa.flags */
#define EVG_LF_REQ_MASK 0x3u
#define EVG_LF_REQ_SYSTEM 0u              /* Requester in evergreen.SystemVersionRequesterTypes (globals.go:766-772): repotracker list, "commit build" */
#define EVG_LF_REQ_PATCH 1u               /* evergreen.IsPatchRequester (globals.go:1179-1185): patch list */
#define EVG_LF_REQ_OTHER 2u               /* anything else: logged and dropped (task_prioritizer.go:232-240) */
#define EVG_LF_GENERATE 0x4u              /* Task.GenerateTask */
#define EVG_LF_MERGE_QUEUE_VERSION 0x8u   /* versions[Task.Version].Requester == github_merge_request (byCommitQueue) */
/* byAge (task_priority_cmp.go:73-95) of one list, decided by the shim when it marshals the list */
#define EVG_LEGACY_MODE_INGEST 0    /* no two commit builds of the list share a project: IngestTime ascending */
#define EVG_LEGACY_MODE_REVISION 1  /* every non-group task is a commit build of ONE project: RevisionOrderNumber descending */
#define EVG_LEGACY_MODE_LITERAL 2   /* neither (or zero and non-zero expected durations mixed, or two (TaskGroup, BuildId)
                                       pairs format to one string): the chain is not a strict weak order on this list */
#define EVG_LEGACY_MODE_GO_STABLE 3 /* any list: sorted exactly as Go's sort.Stable sorts it -- from the groupTaskGroups
                                       presort, with the literal first-definitive chain, the same insertion sorts of
                                       20-blocks, symMerge probes and rotations -- so the result is the reference's order on
                                       any input.  Costs more than INGEST / REVISION, which give the same order where they apply */
/* per-distro status */
#define EVG_LEGACY_OK 0
#define EVG_LEGACY_NOT_DECOMPOSABLE 1 /* some list was EVG_LEGACY_MODE_LITERAL: no order is common to all stable sorts there;
                                         the list was sorted by the nearest transitive key (byAge by IngestTime only),
                                         which need not be the order Go's sort.Stable produces.  A distro whose lists
                                         are all INGEST, REVISION or GO_STABLE is EVG_LEGACY_OK */

/* What CmpBasedTaskPrioritizer reads of []task.Task and map[string]model.Version, SoA over the concatenated distros
 * (scheduler/task_prioritizer.go:80-278, task_priority_cmp.go:25-208, setup_funcs.go:72-87).  Strings are interned
 * by the shim; ranks are per distro. */
typedef struct {
  int64_t n_tasks;
  const int64_t* priority;         /* Task.Priority (int64: the > MaxTaskPriority split and byPriority) */
  const int64_t* ingest_ns;        /* Task.IngestTime */
  const int64_t* expected_ns;      /* Task.FetchExpectedDuration(ctx).Average */
  const int32_t* num_dependents;
  const int32_t* revision_order;   /* Task.RevisionOrderNumber */
  const int32_t* project_id;       /* interned Task.Project */
  const int32_t* tg_rank;          /* rank of "BuildId-TaskGroup" among the distro's distinct such strings, ascending byte order; -1 when TaskGroup == "" */
  const int32_t* tg_pair_id;       /* dense id of the (TaskGroup, BuildId) pair; -1 when TaskGroup == "" */
  const int32_t* task_group_order;
  const int32_t* presort_rank;     /* position of "BuildId-TaskGroup-Id" in DESCENDING byte order inside the distro (groupTaskGroups) */
  const uint32_t* flags;           /* EVG_LF_* */
} evg_legacy_soa;

/* CmpBasedTaskPrioritizer.PrioritizeTasks for every distro of the tick.  list_mode[3*d + {0,1,2}] is the
 * EVG_LEGACY_MODE_* of distro d's high-priority / patch / repotracker list.  order[task_off[d] .. +count[d]) receives
 * the distro-local indices of the prioritised tasks (dropped tasks leave -1 in the remaining slots).  Host pointers.
 * Replaces: the TaskPrioritizer interface (scheduler/task_prioritizer.go:20-25) minus the orderingLogic reasons. */
int evg_prioritize_legacy_batch(evg_ctx* ctx, const evg_legacy_soa* tasks, const int64_t* task_off, const uint8_t* list_mode,
                                int32_t n_distros, int32_t* order, int64_t* count, int32_t* status);

/* ---- DAG dispatcher rebuild (SURVEY.md §8 f.3) ------------------------------ */

/* The persisted queues of a batch of distros, concatenated in queue order (item k of distro d has queueIndex k). */
typedef struct {
  int64_t n_items;
  int64_t n_deps;
  const int64_t* dep_off;      /* n_items + 1: CSR of TaskQueueItem.Dependencies */
  const int32_t* dep_item;     /* n_deps: distro-local index of the item with that id, -1 when it is not in this queue */
  const int32_t* group_id;     /* n_items: distro-local dense id of compositeGroupID(Group, BuildVariant, Project, Version), -1 when Group == "" */
  const int32_t* group_index;  /* n_items: TaskQueueItem.GroupIndex */
} evg_dag_in;

/* basicCachedDAGDispatcherImpl.rebuild for every distro (model/task_queue_service_dependency.go:153-252).
 * sorted[item_off[d] .. + n_sorted[d]) = d.sorted as distro-local item indices: topo.SortStabilized over the edges
 *   dependency -> item with ties in queue order; -1 stands for the nil gonum leaves for a dependency cycle (one per
 *   cyclic component, n_cycles[d] of them); the rest of the distro's slots are -2.
 * unit_items[item_off[d] ..] = the items that have a group, bucketed by group id and stably sorted by GroupIndex inside
 *   each bucket (d.taskGroups[...].tasks); group g of distro d is unit_items[item_off[d] + unit_off[u + g] ..
 *   item_off[d] + unit_off[u + g + 1]) with u = group_off[d] + d (each distro has one closing entry).
 * Host pointers.  group_off (n_distros + 1) counts the groups of each distro.  EVG_ERR_INVALID for an item_off or
 * in->dep_off that does not start at 0, end at n_items / n_deps and never decrease, or a group_off that does not start
 * at 0 or decreases. */
int evg_dag_rebuild_batch(evg_ctx* ctx, const evg_dag_in* in, const int64_t* item_off, const int64_t* group_off, int32_t n_distros,
                          int32_t* sorted, int32_t* n_sorted, int32_t* n_cycles, int32_t* unit_items, int32_t* unit_off);

/* What evg_rebuild_dispatchers writes.  Host pointers; the arrays are laid out as evg_dag_rebuild_batch's. */
typedef struct {
  int64_t* item_off;   /* n_distros + 1: items of distro d = min(length_d, cap), exactly evg_download_queue's item_off */
  int32_t* sorted;     /* items_capacity: d.sorted as item (queue) indices, -1 per cyclic component, -2 tail */
  int32_t* n_sorted;   /* n_distros */
  int32_t* n_cycles;   /* n_distros */
  int64_t* group_off;  /* n_distros + 1: the task groups that occur in each persisted queue */
  int32_t* group_slot; /* groups_capacity: group_slot[group_off[d] + g] = the tick's distro-local group id of DAG group g
                          of distro d (its name is the shim's string for that slot) */
  int32_t* unit_items; /* items_capacity */
  int32_t* unit_off;   /* groups_capacity + n_distros, over group_off above */
} evg_dispatch_out;

/* basicCachedDAGDispatcherImpl.rebuild (model/task_queue_service_dependency.go:153-252) over the queue PersistTaskQueue
 * would save (scheduler/task_queue_persister.go:17-41, TaskQueue.Save model/task_queue.go:216-219) for every distro of
 * the resident tick, built on the device from the tick itself.  Item k of distro d is rank k, the row
 * evg_download_queue returns, for k < min(length_d, cap), cap = 0 meaning EVG_PERSISTED_QUEUE_CAP; same precondition as
 * evg_download_queue (after evg_run_resident), on a tick from any entry point that leaves one.
 *   - edges: a resident edge t -> j is a DAG edge when both rank below the cap (addEdge drops a dependency that is not in
 *     the persisted queue, :118-150); parallel edges and self-edges as in evg_dag_rebuild_batch;
 *   - groups: the tick's group slots of distro d that occur among its items, numbered densely in order of first
 *     appearance (compositeGroupID, :700-702, has Task.GetTaskGroupString's format, model/task/task.go:417-419).
 * Every output equals what evg_dag_rebuild_batch returns for that queue marshalled on the host.  The tick is left as it
 * was (outputs, dependency verdicts, alias map, durations, evg_edit_tasks afterwards).
 * EVG_ERR_INVALID with nothing launched: cap < 0, a null pointer the call needs, items_capacity below the items or
 * groups_capacity below sum over d of min(group slots of d, items of d) (the tick's group slot count always suffices);
 * evg_last_error reports both needed sizes.  EVG_ERR_STATE: no resident tick.
 * Replaces: the evg_download_queue -> dependency-id resolution -> compositeGroupID interning -> evg_dag_rebuild_batch
 * round trip a shim would make to hand FindNextTask d.sorted and d.taskGroups (:475-476, :527-543). */
int evg_rebuild_dispatchers(evg_ctx* ctx, int32_t cap, int64_t items_capacity, int64_t groups_capacity, evg_dispatch_out* out);

/* ---- DAG dispatcher: FindNextTask (SURVEY.md §8 f.3) ------------------------- */

/* evg_next_db.flags: what FindNextTask reads of an item's task document and version, resolved by the shim */
#define EVG_ND_FOUND 0x01u         /* task.FindOneId returned a document (:312, :433, :630); error or nil: clear */
#define EVG_ND_STARTED 0x02u       /* !utility.IsZeroTime(StartTime) (:334): false for Go's zero time and the Unix epoch */
#define EVG_ND_STARTED_GROUP 0x04u /* StartTime != utility.ZeroTime (:657): a struct comparison with time.Unix(0, 0) */
#define EVG_ND_FINISHED_NOT_SUCCEEDED 0x08u /* !IsZeroTime(FinishTime) && Status != "success" (:696-698) */
#define EVG_ND_VERSION_FOUND 0x10u /* VersionFindOne returned a document (:554-576) */
#define EVG_ND_VERSION_S3 0x20u    /* its ProjectStorageMethod is S3 (:578) */
#define EVG_ND_DEPS_MET_NOW 0x40u  /* nextTaskFromDB.DependenciesMet (:373, :662), e.g. from evg_deps_met_batch */
#define EVG_ND_DEPS_ERR 0x80u      /* ... returned an error: the item is skipped */

/* One frozen snapshot of the database for one call.  Per-item columns run over the concatenated items of every
 * dispatcher (item_off), running_hosts over their groups (group_off).  64 B. */
typedef struct {
  int64_t n_items;
  int64_t n_groups;
  const uint8_t* flags;          /* n_items: EVG_ND_* */
  const int32_t* est_generated;  /* n_items: EstimatedNumGeneratedTasks, 0 for nil (:340) */
  const int64_t* ingest_ns;      /* n_items: IngestTime (:392) */
  const int32_t* running_hosts;  /* n_groups: host.NumHostsByTaskSpec (:412, model/host/db.go:521-533); -1: error, which
                                    includes an empty variant / project / version */
  int32_t generate_limit;        /* TaskLimits.MaxPendingGeneratedTasks (:339) */
  int32_t pending_generate;      /* task.GetPendingGenerateTasks (:342); -1: the query failed */
  int32_t max_large_parser;      /* getMaxConcurrentLargeParserProjTasks, degraded mode resolved (:605-612); <= 0: no rule */
  int32_t num_large_parser;      /* task.CountLargeParserProjectTasks (:579); -1: the count failed */
} evg_next_db;

/* The requests of one call: distro d's are req_off[d] .. req_off[d+1], served in that order.  32 B. */
typedef struct {
  int64_t n_requests;
  const int64_t* req_off;        /* n_distros + 1 */
  const int32_t* group;          /* per request: the dense group id compositeGroupID(spec) resolves to in its distro (:268-274);
                                    -1 when spec.Group == "" or the id is none of the dispatcher's groups */
  const int64_t* ami_updated_ns; /* per request: amiUpdatedTime, 0 for a zero time (:392) */
} evg_next_req;

#define EVG_NEXT_NONE 0    /* the walk over d.sorted ended: FindNextTask returned nil at :468 */
#define EVG_NEXT_FOUND 1   /* item = the queue index (rank, the row evg_download_queue returns) of the TaskQueueItem */
#define EVG_NEXT_GAVE_UP 2 /* nil on a database miss: no task document, no version, a failed host count */
typedef struct {
  int32_t* item;    /* per request; -1 for nil */
  int32_t* outcome; /* per request: EVG_NEXT_* */
} evg_next_out;

/* Dispatcher state.  item_bits: the two IsDispatched copies the reference keeps per item. */
#define EVG_NS_NODE 0x1u /* the node's item (d.nodeItemMap; set at :496 and :515) */
#define EVG_NS_UNIT 0x2u /* the copy in schedulableUnit.tasks (:172-183; set at :681; all getTaskGroup and nextTaskGroupTask read) */
typedef struct {
  uint8_t* item_bits;      /* n_items */
  uint8_t* group_deleted;  /* n_groups: the unit left d.taskGroups (:653, :685) */
  int32_t* group_running;  /* n_groups: the unit's cached runningHosts (:411-427); 0 after a rebuild */
} evg_next_state;

/* A batch of dispatchers as evg_dag_rebuild_batch returns them, plus what FindNextTask reads of each item.  80 B. */
typedef struct {
  int32_t n_distros;
  int32_t _reserved;
  const int64_t* item_off;         /* n_distros + 1 */
  const int64_t* group_off;        /* n_distros + 1 */
  const int32_t* sorted;           /* evg_dag_rebuild_batch's outputs ... */
  const int32_t* n_sorted;
  const int32_t* unit_items;
  const int32_t* unit_off;
  const int32_t* group_id;         /* n_items: as evg_dag_in.group_id */
  const int32_t* group_max_hosts;  /* n_items: TaskQueueItem.GroupMaxHosts */
  const uint8_t* dependencies_met; /* n_items: TaskQueueItem.DependenciesMet */
} evg_next_dispatchers;

/* basicCachedDAGDispatcherImpl.FindNextTask (model/task_queue_service_dependency.go:258-469, with tryMarkItemDispatched
 * :486-498, tryMarkNextTaskGroupTaskDispatched :500-519, getTaskGroup :524-538, checkMaxConcurrentLargeParserProjectTasks
 * :549-603, nextTaskGroupTask :614-692, isBlockedSingleHostTaskGroup :696-698) for every request of every distro.
 *
 * The snapshot is frozen for the call.  The requests of one distro are served in the order given, each against the
 * state the earlier ones left.  With one request per distro this is the reference exactly; with several it is the
 * reference under requests that arrive before the database writes of the earlier ones land, which the reference accepts
 * ("a best-effort attempt ... not a foolproof operation", :428-430).  Nothing raises running_hosts inside a call.  Within a call state only
 * accumulates (bits get set, units get deleted, a cached runningHosts stops moving once it reaches maxHosts), and the
 * serving kernel relies on it: a unit found unable to yield under the snapshot is not scanned again in that call.  A
 * caller that clears bits does so between calls (state_in, or a rebuild), never between the requests of one call.
 *
 * Stateless form, host pointers: state_in (NULL: every bit clear, nothing deleted, runningHosts 0; an item persisted with
 * IsDispatched has both bits set) is not changed; state_out receives the state after the last request.  Ends the
 * resident tick (it stages into the dispatcher buffers evg_find_next_tasks serves from).
 * EVG_ERR_INVALID with nothing launched: a null pointer the call needs, offsets check_offsets rejects (item_off, group_off,
 * req_off), db sizes that differ from item_off / group_off, a request group outside [-1, groups of its distro), a
 * negative est_generated, a snapshot scalar below -1 (generate_limit and max_large_parser may be any value <= 0). */
int evg_find_next_batch(evg_ctx* ctx, const evg_next_dispatchers* disp, const evg_next_db* db, const evg_next_req* req,
                        const evg_next_state* state_in, evg_next_state* state_out, evg_next_out* out);

/* The same on the dispatchers the last successful evg_rebuild_dispatchers built from the resident tick; their state
 * stays on the device between calls and starts from IsDispatched == false at every rebuild.  GroupMaxHosts,
 * DependenciesMet and the dense group id of every item were gathered into the dispatchers' own buffers by the rebuild, as
 * the Go dispatcher holds the items as persisted: evg_update_tasks or evg_resolve_durations in between do not reach them.
 * Only reads the tick.  db->n_items / n_groups and req_off are over that rebuild's item_off / group_off.
 * EVG_ERR_STATE: no resident tick, or no evg_rebuild_dispatchers on it since the last evg_run_resident.
 * Replaces: copying sorted / unit_items back per distro and walking them in Go for the agents' next-task endpoint
 * (rest/route/host_agent.go:350-368). */
int evg_find_next_tasks(evg_ctx* ctx, const evg_next_db* db, const evg_next_req* req, evg_next_out* out);

/* The chained dispatchers' state (same precondition as evg_find_next_tasks); any pointer may be NULL. */
int evg_download_dispatch_state(evg_ctx* ctx, evg_next_state* state);

/* ---- the host allocator job's decisions (SURVEY.md §8 row A21) ---------------- */

/* What hostAllocatorJob.Run reads besides HostAllocatorData, per distro, resolved by the shim.  24 B. */
typedef struct {
  int64_t n_provisioning;               /* len(existingHosts.ProvisioningHosts()) (units/host_allocator.go:169); not in the host SoA */
  int32_t single_task_distro;           /* Distro.SingleTaskDistro (:182) */
  int32_t terminate_when_overallocated; /* resolved HostsOverallocatedRule == "terminate-hosts-when-overallocated" (:330) */
  int32_t hourly_billing;               /* cloud.UsesHourlyBilling(&upHosts[0].Distro) (:333, cloud/ec2_util.go:256-268) */
  int32_t _reserved;
} evg_host_job_cfg;

/* The distro-scheduler-report of one distro (units/host_allocator.go:257-337, 394-425).  96 B. */
typedef struct {
  int64_t time_to_empty_ns;           /* timeToEmpty (:304-321) */
  int64_t time_to_empty_no_spawns_ns; /* timeToEmptyNoSpawns */
  int64_t scheduled_duration_ns;      /* scheduledDuration (:287) */
  int64_t hosts_avail;                /* hostsAvail (:294) */
  int64_t hosts_spawned;              /* len(hostsSpawned) the report used (:233, :292) */
  int64_t overdue_in_groups;          /* totalOverdueInTaskGroups (:273) */
  int64_t free_in_groups;             /* freeInTaskGroups (:277) */
  int64_t required_in_groups;         /* requiredInTaskGroups (:278) */
  int64_t new_cap_target;             /* DrawdownInfo.NewCapTarget (:399-405); 0 when setTargetAndTerminate is not called */
  int64_t killable_hosts;             /* killableHosts (:396-400); 0 when setTargetAndTerminate is not called */
  float host_queue_ratio;             /* hostQueueRatio (:324), float32 as Go computes it */
  float no_spawns_ratio;              /* noSpawnsRatio (:326) */
  int32_t drawdown;                   /* 1: the job enqueues a host drawdown job (killableHosts > lowCountFloor, :408) */
  int32_t _reserved;
} evg_host_report;

/* Host pointers, n_distros entries each. */
typedef struct {
  int64_t* n_hosts;         /* nHosts handed to CreateIntentHosts (:184, :191) */
  int64_t* n_hosts_free;    /* nHostsFree (:191); 0 for a single-task distro */
  int32_t* status;          /* EVG_ALLOC_*: the allocator's error ends the job (:192-195) */
  evg_host_report* report;  /* all zero when status != EVG_ALLOC_OK */
} evg_host_job_out;

/* hostAllocatorJob.Run after the allocator (units/host_allocator.go:180-196, 253-337, 394-425) for every distro of the
 * resident tick, on the device, from the queue infos, group infos and allocator results evg_run_resident left there
 * (the result rows are read wherever evg_bind_result_buffer put them).  The tick is only read: calling it twice gives
 * the same answer, and every call allowed before it stays allowed.
 *   - single-task distro (:182-184): n_hosts = LengthWithDependenciesMet - n_provisioning (may be negative), n_hosts_free
 *     = 0, status EVG_ALLOC_OK; its group slots count CountFree = CountRequired = 0 (the reference never runs the
 *     allocator for it, whatever k_alloc wrote on the device);
 *   - any other distro: new_hosts, free_hosts and status of the allocator run; a status other than EVG_ALLOC_OK ends the
 *     job there (:192-195) and the report is zero;
 *   - spawned[d] = len(hostsSpawned) (:233); spawned == NULL means max(n_hosts, 0), what CreateIntentHosts creates
 *     without a container pool (scheduler/scheduler.go:172-215); a pool distro's shim calls again with the count
 *     MakeContainersAndParents returned;
 *   - report (:257-326): sums over the distro's group slots (its named TaskGroupInfos; the ungrouped info is excluded),
 *     int64 arithmetic with wrap, timeToEmpty truncated toward zero, 2532000 h when its host count is <= 0, both times
 *     0 when scheduledDuration <= 0; the ratios are float32(int64) rounded to nearest-even and divided IEEE-correctly
 *     (MaxDurationThreshold 0 gives +Inf or NaN, as Go does);
 *   - drawdown (:328-337, 394-425): when terminate_when_overallocated, the provider is not EVG_PROVIDER_STATIC
 *     (evergreen.ProviderSpawnable), hostQueueRatio < 0.25f, the distro has up hosts (its hosts in the host SoA) and
 *     !hourly_billing: killable = n_up when the ratio is 0, else int(float32(n_up) * (1 - ratio)) truncated (saturated
 *     at the int64 range, which only a negative MaxDurationThreshold can reach; Go leaves that conversion
 *     implementation-defined), new_cap_target = n_up - killable floored at MinimumHosts; drawdown = killable > 0.
 * What the library does not model and the shim applies itself: a disabled distro returns before this phase (:144-146);
 * the intent-host cap (:212-229) and a CreateIntentHosts error (:233-237) end the job before the report, so the shim
 * discards that distro's report; choosing the hosts to decommission is the drawdown job's (units/host_drawdown.go,
 * evg_host_drawdown below, which can read this call's reports where they are).
 * EVG_ERR_INVALID with nothing launched: null cfg or out (or a null array of out), a negative n_provisioning.
 * EVG_ERR_STATE: no resident tick, a tick without hosts, or no evg_run_resident on it since it was set (the one-shot
 * evg_plan_and_alloc_batch counts as one).  The first call allocates the call's own small buffers.
 * Replaces: the single-task bypass, the time-to-empty report and the drawdown decision of hostAllocatorJob.Run. */
int evg_host_job(evg_ctx* ctx, const evg_host_job_cfg* cfg, const int32_t* spawned, evg_host_job_out* out);

/* ---- host termination: the drawdown job and the idle-host job ------------- */

/* One idle-host table serves both jobs.  Rows are grouped by distro through an idle_off CSR (n_distros + 1 entries);
 * within a distro they come in the order the job's query returned them: IdleHostsWithDistroID's natural order for the
 * drawdown job (model/host/db.go:274-286, 373-381), IdleEphemeralGroupedByDistroID's ascending CreationTime for the
 * idle-host job (db.go:211-255).  Both queries return only ephemeral hosts with no running task that are not container
 * parents, so IdleTime's running-task branch, the running-task branch of isAssignedSingleHostTaskGroup and the
 * !IsEphemeral exemption of checkTerminationExemptions cannot be reached and are not modelled.
 * Times are int64 ns since the Unix epoch, EVG_TIME_ZERO for Go's zero time. */
enum {
  EVG_IH_RUNNING_TASK_GROUP = 1 << 0,      /* RunningTaskGroup != "" */
  EVG_IH_LAST_TASK = 1 << 1,               /* LastTask != "" */
  EVG_IH_STATUS_RUNNING = 1 << 2,          /* Status == evergreen.HostRunning */
  EVG_IH_USER_DATA = 1 << 3,               /* the embedded distro's bootstrap method is user-data */
  EVG_IH_LEGACY_BOOTSTRAP = 1 << 4,        /* the embedded distro's LegacyBootstrap() */
  EVG_IH_NEEDS_NEW_AGENT = 1 << 5,         /* NeedsNewAgent */
  EVG_IH_NEEDS_NEW_AGENT_MONITOR = 1 << 6, /* NeedsNewAgentMonitor */
  EVG_IH_OUTDATED_AMI = 1 << 7,            /* h.GetAMI() != d.GetDefaultAMI() against the distro document (idle job only) */
  EVG_IH_SINGLE_HOST_TASK_GROUP = 1 << 8,  /* isAssignedSingleHostTaskGroup through LastGroup: the last task is
                                              IsPartOfSingleHostTaskGroup and succeeded */
  EVG_IH_TASK_LOOKUP_FAILED = 1 << 9,      /* LastGroup != "" and the last task was not found, or the lookup failed */
  EVG_IH_PAYMENT_NOT_DUE = 1 << 10,        /* TimeTilNextPayment(h) > maxTimeTilNextPayment (5 min) */
  EVG_IH_CLOUD_MANAGER_FAILED = 1 << 11    /* GetManagerOptions or GetManager returned an error */
};

typedef struct {
  int64_t n_hosts;
  int32_t n_distros;
  int32_t _reserved;
  const int64_t* creation_ns;
  const int64_t* start_ns;
  const int64_t* provision_ns;
  const int64_t* agent_start_ns;
  const int64_t* last_communication_ns;
  const int64_t* last_task_completed_ns;
  const int64_t* teardown_start_ns;    /* TaskGroupTeardownStartTime */
  const int64_t* acceptable_idle_ns;   /* the host's embedded Distro.HostAllocatorSettings.AcceptableHostIdleTime */
  const uint32_t* flags;               /* EVG_IH_* */
} evg_idle_host_soa;

/* What the job decided for one row.  EVG_HT_NOT_CHECKED: past its distro's drawdown target, a distro without a drawdown,
 * or not among the idle job's evaluated hosts; nothing else of the row is written then (all zero). */
enum {
  EVG_HT_NOT_CHECKED = 0,
  EVG_HT_KEPT = 1,                 /* checked, no action */
  EVG_HT_EXEMPT_AGENT = 2,         /* checkTerminationExemptions: waiting for an agent */
  EVG_HT_EXEMPT_PAYMENT = 3,       /* checkTerminationExemptions: the next payment is more than 5 min away */
  EVG_HT_ERR_CLOUD_MANAGER = 4,    /* checkTerminationExemptions' error: the job reports it and leaves the host */
  EVG_HT_ERR_TASK_LOOKUP = 5,      /* isAssignedSingleHostTaskGroup's error: the job reports it and leaves the host */
  EVG_HT_DECOMMISSION = 6,         /* the drawdown job decommissions the host */
  EVG_HT_TERM_OUTDATED_AMI = 7,    /* the idle job terminates it, one code per reason of getTerminationReason, in its order */
  EVG_HT_TERM_COMMUNICATION = 8,
  EVG_HT_TERM_IDLE = 9,
  EVG_HT_TERM_TEARDOWN = 10
};

/* One row's verdict and the durations the job's messages print.  40 B. */
typedef struct {
  int64_t idle_ns;            /* IdleTime() */
  int64_t communication_ns;   /* GetElapsedCommunicationTime() */
  int64_t threshold_ns;       /* the idle threshold the job compares against (drawdown: 5 s, 10 min or the embedded
                                 distro's value; idle job: the distro's, 5 min or doubled); 0 when the job decided
                                 before it got to one (an exemption, a lookup error, a teardown or single-host task group
                                 that keeps a host from the drawdown) */
  int64_t since_teardown_ns;  /* time.Since(TaskGroupTeardownStartTime), INT64_MAX for Go's zero time */
  int32_t decision;           /* EVG_HT_* */
  int32_t _reserved;
} evg_host_verdict;

#define EVG_NO_DRAWDOWN INT64_MIN /* new_cap_target: no drawdown job for this distro */

/* evg_host_drawdown's per-distro inputs (n_distros entries each).  new_cap_target and queue_length_dm are both NULL
 * (chained) or both given (standalone). */
typedef struct {
  const int64_t* existing_hosts;   /* CountHostsCanOrWillRunTasksInDistro (units/host_drawdown.go:77) */
  const int64_t* new_cap_target;   /* DrawdownInfo.NewCapTarget, EVG_NO_DRAWDOWN = no job */
  const int64_t* queue_length_dm;  /* the distro's DistroQueueInfo.LengthWithDependenciesMet (:87, :141) */
} evg_drawdown_in;

/* Per distro.  24 B. */
typedef struct {
  int64_t target;          /* drawdownTarget = existing - NewCapTarget (:91), possibly <= 0; 0 when the job did not run */
  int64_t decommissioned;  /* j.Decommissioned */
  int32_t ran;             /* 1: the distro had a drawdown job */
  int32_t _reserved;
} evg_drawdown_distro;

typedef struct {
  evg_host_verdict* hosts;        /* n_hosts entries */
  evg_drawdown_distro* distros;   /* n_distros entries */
} evg_host_drawdown_out;

/* hostDrawdownJob.Run / checkAndDecommission (units/host_drawdown.go:70-159) for every distro, on the device, at a
 * frozen now_ns.  Per checked host, in order: checkTerminationExemptions (waiting for an agent with communication or
 * idle time < 10 min: exempt; a cloud manager error; the next payment more than 5 min away: exempt); tearing down and
 * not past 4 min: kept; a single-host task group: kept (a lookup error is reported and the host kept); then the
 * threshold is 5 s, 10 min in a running task group, the embedded distro's acceptable_idle_ns when LastTaskCompletedTime
 * is not zero and queue_length_dm > 0; IdleTime > threshold decommissions.  The loop stops before any host once the
 * target is <= 0 and the target drops only on a decommission, so a row is checked iff fewer than `target` rows before
 * it in its distro would be decommissioned; later rows are EVG_HT_NOT_CHECKED and report no error.
 *   - chained (new_cap_target and queue_length_dm NULL): the distros the last evg_host_job on the resident tick's run
 *     flagged drawdown = 1, with its new_cap_target and the tick's LengthWithDependenciesMet, none of which leaves the
 *     device; hosts->n_distros must be the tick's.
 *   - standalone: explicit values, as a separate drawdown job fed a DrawdownInfo; needs no tick and touches none.
 * The tick is only read.  EVG_ERR_INVALID with nothing launched: a null hosts, idle_off, in, existing_hosts or out (or a
 * null array of out or of hosts with n_hosts > 0), a bad idle_off, a negative n_hosts, n_distros, existing_hosts or
 * queue_length_dm, new_cap_target and queue_length_dm not both NULL or both given, or a chained call whose n_distros is
 * not the tick's.  EVG_ERR_STATE (chained only): no resident tick, or no evg_host_job on its current run.  The first
 * call allocates the call's own buffers.
 * Replaces: the per-host loop of hostDrawdownJob (the shim calls SetDecommissioned for each EVG_HT_DECOMMISSION row). */
int evg_host_drawdown(evg_ctx* ctx, const evg_idle_host_soa* hosts, const int64_t* idle_off, const evg_drawdown_in* in,
                      int64_t now_ns, evg_host_drawdown_out* out);

/* evg_idle_hosts' per-distro settings.  24 B. */
typedef struct {
  int64_t minimum_hosts;        /* Distro.HostAllocatorSettings.MinimumHosts; 0 for a distro missing from the collection */
  int64_t running_hosts_count;  /* IdleHostsByDistroID.RunningHostsCount */
  int64_t acceptable_idle_ns;   /* the distro's AcceptableHostIdleTime, or SchedulerConfig.AcceptableHostIdleTimeSeconds
                                   when that is 0 (units/host_monitoring_idle_termination.go:197-200) */
} evg_idle_cfg;

/* Per distro.  16 B. */
typedef struct {
  int64_t min_evaluate;  /* getMinNumHostsToEvaluate (:143-156) */
  int64_t terminated;    /* j.Terminated for the distro */
} evg_idle_distro;

typedef struct {
  evg_host_verdict* hosts;     /* n_hosts entries */
  evg_idle_distro* distros;    /* n_distros entries */
} evg_idle_hosts_out;

/* idleHostJob.Run / checkAndTerminateHost / getIdleInfo / getTerminationReason
 * (units/host_monitoring_idle_termination.go:64-283) for every distro, on the device, at a frozen now_ns.  Row i of a
 * distro is evaluated iff i < min_evaluate = clamp(running_hosts_count - minimum_hosts, 0, n_idle) or it has an
 * outdated AMI.  An evaluated host: the exemptions (as evg_host_drawdown; a cloud manager error is reported), then a
 * task lookup error (reported, not terminated), then the threshold: acceptable_idle_ns, 5 min in a single-host task
 * group, else doubled (int64 wrap) in a running task group; then the first reason that holds: an outdated AMI with
 * IdleTime > 0 outside a single-host task group; communication time >= threshold and not tearing down; IdleTime > 0 and
 * >= threshold; more than 4 min since the teardown start while tearing down.  No reason: EVG_HT_KEPT.
 * A distro missing from the distro collection is decommissioned by the shim (:92-110); its idle rows are still
 * evaluated, as the Go loop does, with a zero-value distro: minimum_hosts 0, the scheduler config's idle time and
 * EVG_IH_OUTDATED_AMI set iff the host's AMI is not "".
 * Needs no tick and leaves any tick as it was.  EVG_ERR_INVALID with nothing launched: a null hosts, idle_off, cfg or
 * out (or a null array of out or of hosts with n_hosts > 0), a bad idle_off, a negative n_hosts, n_distros,
 * minimum_hosts or running_hosts_count.  The first call allocates the call's own buffers.
 * Replaces: the per-host loop of idleHostJob (the shim enqueues a termination job for each EVG_HT_TERM_* row). */
int evg_idle_hosts(evg_ctx* ctx, const evg_idle_host_soa* hosts, const int64_t* idle_off, const evg_idle_cfg* cfg,
                   int64_t now_ns, evg_idle_hosts_out* out);

/* ---- task start-time estimates (model/task_start_estimation.go) ----------- */

/* evg_est_host_soa.kind: what createSimulatorModel makes of a host (model/task_start_estimation.go:129-159) */
enum {
  EVG_EH_UNINITIALIZED = 0, /* Status == evergreen.HostUninitialized: timeToCompletion 4 min (:131-132) */
  EVG_EH_STARTING = 1,      /* HostStarting: 3 min (:133-134) */
  EVG_EH_PROVISIONING = 2,  /* HostProvisioning: 1 min (:135-136) */
  EVG_EH_FREE = 3,          /* HostRunning with RunningTask == "": 0 (:138-139) */
  EVG_EH_RUNNING = 4,       /* HostRunning with a task: ExpectedDuration - time.Since(DispatchTime) (:156-157) */
  EVG_EH_IGNORED = 5        /* contributes no host: any other status, or the running task has no document (:148-154) */
};
/* A pool of at most this many hosts is simulated in shared memory, a larger one in global memory; same results. */
#define EVG_EST_ONCHIP_HOSTS 1024

/* The hosts host.Find(ByDistroIDs(distro)) returns (model/task_start_estimation.go:117, model/host/db.go:628-635), per
 * distro in query order, SoA; replaces the []host.Host and the task.FindOneIdAndExecution of each running host
 * (:141).  A lookup ERROR makes the reference return the pool built so far (:142-147): the shim ends the distro's rows
 * before that host.  32 B. */
typedef struct {
  int64_t n_hosts;
  const uint8_t* kind;        /* EVG_EH_* */
  const int64_t* expected_ns; /* EVG_EH_RUNNING: the running task's stored ExpectedDuration field (:157); else not read */
  const int64_t* dispatch_ns; /* EVG_EH_RUNNING: its DispatchTime, EVG_TIME_ZERO for Go's zero time; else not read */
} evg_est_host_soa;

/* GetEstimatedStartTime (model/task_start_estimation.go:99-122) for EVERY persisted position of every distro of the
 * resident tick, after evg_run_resident: createSimulatorModel (:124-163) on the device, the pool sorted once (:60), then
 * one run of dispatchNextTask (:69-96) per distro, whose state after position p is what a fresh simulate(p) returns
 * (:53-67).  `cap` and `item_off` (n_distros + 1, written) are evg_download_queue's, so start_ns[k] is the estimate of
 * the queue item evg_download_queue returns as items[k]: the queue is the resident expected_ns column read through the
 * rank order, which never leaves the device.  est_host_off (n_distros + 1) is the CSR of `hosts` over the tick's
 * distros.  time.Since is taken at now_ns and saturates; everything else is int64 arithmetic that wraps, as in Go.
 * A distro without items has no estimates; one without hosts (none given, or all EVG_EH_IGNORED) gets -1 for every item
 * (:54-59).  -1 is also a value a run can reach, so hosts_used[d] (n_distros) reports the pool size of each distro.
 * Only reads the tick: every call allowed before it stays allowed, the dispatchers of evg_rebuild_dispatchers included,
 * and calling it again (another now_ns, other hosts) recomputes from the same queue.  The first call allocates its own
 * buffers.  EVG_ERR_INVALID with nothing launched and the tick still runnable: a null pointer the call needs, a negative
 * cap or n_hosts, an est_host_off check_offsets rejects, a kind above EVG_EH_IGNORED (evg_last_error names the row),
 * items_capacity below the rows needed (with the count in evg_last_error, item_off already written).  EVG_ERR_STATE:
 * no resident tick.
 * Replaces: LoadTaskQueue, the position scan's simulator set-up and the O(position x hosts) replay per task asked about
 * (graphql/task_resolver.go:360-371 calls it once per task); the id-to-position lookup stays with the shim. */
int evg_estimate_start_times(evg_ctx* ctx, int32_t cap, const evg_est_host_soa* hosts, const int64_t* est_host_off,
                             int64_t now_ns, int64_t* item_off, int64_t* start_ns, int64_t items_capacity,
                             int32_t* hosts_used);

/* The same for caller-supplied queues (a queue loaded from the task_queues collection, a secondary queue):
 * durations[item_off[d] .. item_off[d+1]) are TaskQueueItem.ExpectedDuration of distro d's items in queue order (:126-128).
 * Host pointers.  Needs no tick and leaves any tick as it was.  EVG_ERR_INVALID with nothing launched: as above, a
 * negative n_distros, an item_off check_offsets rejects.
 * Replaces: createSimulatorModel(...).simulate(pos) (:121) for every pos of every queue. */
int evg_estimate_start_batch(evg_ctx* ctx, const int64_t* durations, const int64_t* item_off, int32_t n_distros,
                             const evg_est_host_soa* hosts, const int64_t* est_host_off, int64_t now_ns, int64_t* start_ns,
                             int32_t* hosts_used);

/* ---- single-distro wrappers: the per-job drop-in ------------------------- */

/* One distro: PrioritizeTasks for `d` (scheduler/scheduler.go:27). */
int evg_plan_distro(evg_ctx* ctx, const evg_task_soa* tasks, const evg_distro_cfg* cfg,
                    int32_t n_groups, const int32_t* group_max_hosts, int64_t now_ns, uint32_t opts,
                    evg_plan_out* out);
/* One distro: UtilizationBasedHostAllocator(ctx, &HostAllocatorData{...})
 * (scheduler/utilization_based_host_allocator.go:26). */
int evg_alloc_distro(evg_ctx* ctx, const evg_host_soa* hosts, const evg_alloc_cfg* cfg,
                     const evg_queue_info* info, evg_group_info* groups, int32_t n_groups,
                     int64_t now_ns, evg_alloc_result* result, int32_t* status);

#ifdef __cplusplus
}
#endif
#endif /* EVG_SCHED_H */
