"""tests/golden/host_allocator_job.json (make_host_allocator_job_golden.py) as model objects: the tick of each case
and the job inputs it states.  Shared by the CPU tests and the GPU tests."""
from evergreen_b200 import model as M
import golden_loader as G

CASES = G.load("host_allocator_job.json")
NOW = CASES["now"]
GROUP_KEYS = ("bv", "p", "v")  # a case's task group "g" is Task.GetTaskGroupString() "g_bv_p_v"


def distro(c: dict) -> M.Distro:
    d = c["distro"]
    hs = d["HostAllocatorSettings"]
    return M.Distro(id=d["Id"], provider=d["Provider"], arch=d["Arch"], single_task_distro=d["SingleTaskDistro"],
                    planner_settings=M.PlannerSettings(target_time=d["TargetTime"]),
                    host_allocator_settings=M.HostAllocatorSettings(
                        minimum_hosts=hs["MinimumHosts"], maximum_hosts=hs["MaximumHosts"],
                        future_host_fraction=float(hs["FutureHostFraction"]),
                        hosts_overallocated_rule=hs["HostsOverallocatedRule"]))


def tasks(c: dict):
    out = []
    for t in c["tasks"]:
        task = M.Task(id=t["Id"], expected_duration=t["ExpectedDuration"],
                      depends_on=[M.Dependency(task_id=x) for x in t.get("DependsOn", [])])
        if "TaskGroup" in t:
            task.task_group, task.task_group_max_hosts = t["TaskGroup"], t["TaskGroupMaxHosts"]
            task.build_variant, task.project, task.version = GROUP_KEYS
        if "ScheduledAgo" in t:
            task.scheduled_time = NOW - t["ScheduledAgo"]
        out.append(task)
    return out


def allocator_data(c: dict) -> M.HostAllocatorData:
    hosts = []
    for h in c["hosts"]:
        host = M.Host(id=h["Id"], running_task=h.get("RunningTask", ""))
        if "RunningTaskGroup" in h:
            host.running_task_group = h["RunningTaskGroup"]
            host.running_task_build_variant, host.running_task_project, host.running_task_version = GROUP_KEYS
        hosts.append(host)
    running = {r["Id"]: M.RunningTaskStats(True, r["ExpectedDuration"], 0, NOW - r["StartAgo"]) for r in c.get("running_tasks", [])}
    return M.HostAllocatorData(distro=distro(c), existing_hosts=hosts, distro_queue_info=M.DistroQueueInfo(),
                               running_tasks=running)


def batch_entry(c: dict):
    """(Distro, tasks, HostAllocatorData) of the case's tick, as scheduler.host_allocator_jobs takes it."""
    data = allocator_data(c)
    return data.distro, tasks(c), data


def job_input(c: dict):
    """-> (DistroQueueInfo as the job reads it, (nHosts, nHostsFree, status))."""
    j = c["job_input"]
    q = j["queue_info"]
    groups = [M.TaskGroupInfo(name="_".join((g["Name"],) + GROUP_KEYS), count=g["Count"], count_free=g["CountFree"],
                              count_required=g["CountRequired"], expected_duration=g["ExpectedDuration"],
                              count_duration_over_threshold=g["CountDurationOverThreshold"],
                              count_wait_over_threshold=g["CountWaitOverThreshold"],
                              duration_over_threshold=g["DurationOverThreshold"]) for g in q["TaskGroupInfos"]]
    info = M.DistroQueueInfo(length_with_dependencies_met=q["LengthWithDependenciesMet"], expected_duration=q["ExpectedDuration"],
                             max_duration_threshold=q["MaxDurationThreshold"],
                             count_duration_over_threshold=q["CountDurationOverThreshold"],
                             duration_over_threshold=q["DurationOverThreshold"], task_group_infos=groups)
    return info, (j["n_hosts"], j["n_hosts_free"], j["status"])


def threshold(c: dict) -> int:
    """MaxDurationThreshold the case's planner runs with: raw_threshold when the case sets one (0 cannot come from
    Distro.GetTargetTime, distro.go:434-440), else the distro's."""
    return c.get("raw_threshold", c["distro"]["TargetTime"])
