"""Line-by-line restatement of the drawdown job (units/host_drawdown.go:70-159) and the idle-host job
(units/host_monitoring_idle_termination.go:64-342) with the host predicates they call (model/host/host.go), over
model objects at a frozen `now`.  Test infrastructure only: the product never imports it.

Each job returns its model record (HostDrawdownJob / IdleHostJob) and one verdict per idle host, as the device writes
them: (decision, idle, communication, threshold, since teardown), all zero for a host the job does not check."""
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler as S

I64_MAX, I64_MIN = 2 ** 63 - 1, -(2 ** 63)
MAX_TEARDOWN_GROUP_THRESHOLD = 4 * M.MINUTE           # globals.go:348
MAX_AGENT_UNRESPONSIVE_INTERVAL = 5 * M.MINUTE        # host.go:624
MAX_AGENT_MONITOR_UNRESPONSIVE_INTERVAL = 5 * M.MINUTE  # host.go:634
IDLE_WAITING_FOR_AGENT_CUTOFF = 10 * M.MINUTE         # host_monitoring_idle_termination.go:24
MAX_TIME_TIL_NEXT_PAYMENT = 5 * M.MINUTE              # :27
IDLE_TIME_DRAWDOWN_CUTOFF = 5 * M.SECOND              # host_drawdown.go:23
IDLE_TASK_GROUP_DRAWDOWN_CUTOFF = 10 * M.MINUTE       # host_drawdown.go:24
SINGLE_HOST_TASK_GROUP_IDLE_CUTOFF = 5 * M.MINUTE     # host_monitoring_idle_termination.go:206
NOT_CHECKED = (L.EVG_HT_NOT_CHECKED, 0, 0, 0, 0)


def since(now, t):
    """time.Since(t) at a frozen now: Time.Sub saturates; Go's zero time lies before every int64 instant."""
    if t == M.ZERO_TIME:
        return I64_MAX
    return max(I64_MIN, min(I64_MAX, now - t))


def wrap(x):
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


def is_tearing_down(h):  # host.go:219-221
    return h.task_group_teardown_start_time != M.ZERO_TIME


def teardown_time_exceeded_max(h, now):  # host.go:2241-2243
    return since(now, h.task_group_teardown_start_time) > MAX_TEARDOWN_GROUP_THRESHOLD


def idle_time(h, now):  # host.go:671-706 (the idle queries return no host with a running task)
    if is_tearing_down(h):
        if teardown_time_exceeded_max(h, now):
            return since(now, h.task_group_teardown_start_time)
        return 0
    if h.last_task != "":
        return since(now, h.last_task_completed_time)
    if h.bootstrap_method == M.BOOTSTRAP_METHOD_USER_DATA:
        if h.agent_start_time != M.ZERO_TIME and h.agent_start_time > 0:  # After(utility.ZeroTime)
            return since(now, h.agent_start_time)
    elif h.status == M.HOST_RUNNING:
        return since(now, h.provision_time)
    return 0


def get_elapsed_communication_time(h, now):  # host.go:2220-2238
    if is_tearing_down(h):
        return 0
    if h.last_communication_time > h.creation_time:
        return since(now, h.last_communication_time)
    if h.start_time > h.creation_time:
        return since(now, h.start_time)
    if h.last_communication_time != M.ZERO_TIME:
        return since(now, h.last_communication_time)
    return since(now, h.creation_time)


def legacy_bootstrap(h):  # distro.go:842-844, on the host's embedded distro
    return h.bootstrap_method in ("", M.BOOTSTRAP_METHOD_LEGACY_SSH)


def is_waiting_for_agent(h, now):  # host.go:2006-2026
    if legacy_bootstrap(h) and h.needs_new_agent:
        return True
    if not legacy_bootstrap(h) and h.needs_new_agent_monitor:
        return True
    if M.is_zero_time(h.last_communication_time):
        return True
    interval = MAX_AGENT_UNRESPONSIVE_INTERVAL if legacy_bootstrap(h) else MAX_AGENT_MONITOR_UNRESPONSIVE_INTERVAL
    cutoff = now - interval  # Go's Time.Add cannot leave its range here; below every int64 instant nothing is Before it
    return h.last_communication_time < cutoff


def is_assigned_single_host_task_group(h):  # host_monitoring_idle_termination.go:228-256 -> (bool, error)
    if h.last_group != "":
        if h.last_task_single_host_task_group is None:
            return False, "host's last task group task not found"
        return bool(h.last_task_single_host_task_group), None
    return False, None


def check_termination_exemptions(h, now):  # :287-338 -> (exit early, error, decision)
    idle = idle_time(h, now)
    comm = get_elapsed_communication_time(h, now)
    if is_waiting_for_agent(h, now) and (comm < IDLE_WAITING_FOR_AGENT_CUTOFF or idle < IDLE_WAITING_FOR_AGENT_CUTOFF):
        return True, None, L.EVG_HT_EXEMPT_AGENT
    if h.cloud_manager_error:
        return True, "getting cloud manager for host", L.EVG_HT_ERR_CLOUD_MANAGER
    if h.time_til_next_payment > MAX_TIME_TIL_NEXT_PAYMENT:
        return True, None, L.EVG_HT_EXEMPT_PAYMENT
    return False, None, None


def verdict(h, now, code, threshold=0):
    return (code, idle_time(h, now), get_elapsed_communication_time(h, now), threshold,
            since(now, h.task_group_teardown_start_time))


def check_and_decommission(h, now, queue_len, state):  # host_drawdown.go:127-159 -> (verdict, error)
    exit_early, err, code = check_termination_exemptions(h, now)
    if exit_early or err is not None:
        return verdict(h, now, code), err
    if is_tearing_down(h) and not teardown_time_exceeded_max(h, now):
        return verdict(h, now, L.EVG_HT_KEPT), None
    single, err = is_assigned_single_host_task_group(h)
    if err is not None:
        return verdict(h, now, L.EVG_HT_ERR_TASK_LOOKUP), "checking if host is running single host task group"
    if single:
        return verdict(h, now, L.EVG_HT_KEPT), None
    idle = idle_time(h, now)
    threshold = IDLE_TIME_DRAWDOWN_CUTOFF
    if h.running_task_group != "":
        threshold = IDLE_TASK_GROUP_DRAWDOWN_CUTOFF
    if h.last_task_completed_time != M.ZERO_TIME and queue_len > 0:
        threshold = h.acceptable_host_idle_time
    if idle > threshold:
        state["target"] -= 1
        return verdict(h, now, L.EVG_HT_DECOMMISSION, threshold), None
    return verdict(h, now, L.EVG_HT_KEPT, threshold), None


def drawdown_job(distro_id, idle_hosts, existing_host_count, new_cap_target, queue_len, now):
    """hostDrawdownJob.Run (host_drawdown.go:70-118)."""
    target = existing_host_count - new_cap_target  # :91
    job = M.HostDrawdownJob(distro_id, new_cap_target, existing_host_count, len(idle_hosts), target)
    state = {"target": target}
    verdicts = [NOT_CHECKED] * len(idle_hosts)
    for i, h in enumerate(idle_hosts):
        if state["target"] <= 0:
            break
        verdicts[i], err = check_and_decommission(h, now, queue_len, state)
        if verdicts[i][0] == L.EVG_HT_DECOMMISSION:
            job.decommissioned_hosts.append(h.id)
        if err is not None:
            job.errors.append((h.id, err))
    return job, verdicts


def get_min_num_hosts_to_evaluate(n_idle, running_hosts_count, minimum_hosts):  # :143-156
    max_hosts_to_terminate = running_hosts_count - minimum_hosts
    if max_hosts_to_terminate <= 0:
        return 0
    if n_idle > max_hosts_to_terminate:
        return max_hosts_to_terminate
    return n_idle


def host_has_outdated_ami(h, d):  # :340-342
    return h.ami != d.default_ami


def check_and_terminate_host(h, d, now, sched_idle_seconds):  # :158-226, 258-283 -> (verdict, error, reason)
    exit_early, err, code = check_termination_exemptions(h, now)
    if exit_early:
        return verdict(h, now, code), err, ""
    threshold = d.host_allocator_settings.acceptable_host_idle_time  # getIdleInfo
    if threshold == 0:
        threshold = sched_idle_seconds * M.SECOND
    single, err = is_assigned_single_host_task_group(h)
    if err is not None:
        return verdict(h, now, L.EVG_HT_ERR_TASK_LOOKUP), "getting information on idle host", ""
    if single:
        threshold = SINGLE_HOST_TASK_GROUP_IDLE_CUTOFF
    elif h.running_task_group != "":
        threshold = wrap(threshold * 2)
    idle, comm = idle_time(h, now), get_elapsed_communication_time(h, now)
    tearing, since_td = is_tearing_down(h), since(now, h.task_group_teardown_start_time)
    ds = M.go_duration_string
    if host_has_outdated_ami(h, d) and idle > 0 and not single:
        code, reason = L.EVG_HT_TERM_OUTDATED_AMI, "host has an outdated AMI"
    elif comm >= threshold and not tearing:
        code = L.EVG_HT_TERM_COMMUNICATION
        reason = f"host is idle or unreachable, communication time {ds(comm)} is over threshold time {ds(threshold)}"
    elif idle > 0 and idle >= threshold:
        code = L.EVG_HT_TERM_IDLE
        reason = f"host is idle or unreachable, idle time {ds(idle)} is over threshold time {ds(threshold)}"
    elif since_td > MAX_TEARDOWN_GROUP_THRESHOLD and tearing:
        code = L.EVG_HT_TERM_TEARDOWN
        reason = (f"time since the host's task group teardown start time {ds(since_td)} has exceeded the maximum "
                  f"teardown threshold {ds(MAX_TEARDOWN_GROUP_THRESHOLD)}")
    else:
        code, reason = L.EVG_HT_KEPT, ""
    return verdict(h, now, code, threshold), None, reason


def idle_job(d, idle_hosts, running_hosts_count, now, sched_idle_seconds=0):
    """idleHostJob.Run's loop for one distro (:128-140); `d` None: missing from the collection, the zero distro."""
    dd = d if d is not None else M.Distro()
    min_num = get_min_num_hosts_to_evaluate(len(idle_hosts), running_hosts_count, dd.host_allocator_settings.minimum_hosts)
    job = M.IdleHostJob(dd.id, len(idle_hosts), min_num)
    verdicts = [NOT_CHECKED] * len(idle_hosts)
    evaluated = 0
    for i, h in enumerate(idle_hosts):
        if evaluated >= min_num and not host_has_outdated_ami(h, dd):
            continue
        evaluated += 1
        verdicts[i], err, reason = check_and_terminate_host(h, dd, now, sched_idle_seconds)
        if reason:
            job.terminated_hosts.append(h.id)
            job.reasons.append(reason)
        if err is not None:
            job.errors.append((h.id, err))
    return job, verdicts


assert S.MAX_TEARDOWN_GROUP_THRESHOLD == MAX_TEARDOWN_GROUP_THRESHOLD
