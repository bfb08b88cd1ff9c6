"""Restatement of hostAllocatorJob.Run past the allocator (units/host_allocator.go:180-337, 394-425) over model
objects, with numpy float32 for the ratios as Go computes them.  Independent of the library: it reads the
DistroQueueInfo the planner produced (with the CountFree / CountRequired the allocator wrote) and the allocator's
(nHosts, nHostsFree, status), and returns what the job decides."""
from typing import Optional

import numpy as np

from evergreen_b200 import model as M

MAX_POSSIBLE_TIME = 2532000 * M.HOUR  # maxPossibleHours * time.Hour (:309)
LOW_RATIO_THRESH = np.float32(0.25)   # :329
INT64_MAX = 2 ** 63 - 1


def w64(x: int) -> int:
    """Go int / time.Duration arithmetic: two's-complement wrap at 64 bits."""
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


def f32(x: int) -> np.float32:
    """float32(int64): one rounding to nearest-even (numpy casts int64 -> float32 directly, not through float64)."""
    return np.array([x], dtype=np.int64).astype(np.float32)[0]


def go_div(a: int, b: int) -> int:
    """Go integer division, truncated toward zero (b > 0 here)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def f32_to_int(x: np.float32) -> int:
    """int(float32) truncated; out of the int64 range it saturates (Go leaves that implementation-defined)."""
    v = float(x)
    if v >= 2.0 ** 63:
        return INT64_MAX
    if v < -2.0 ** 63:
        return -2 ** 63
    return int(v)


def uses_hourly_billing(d: M.Distro) -> bool:
    """cloud.UsesHourlyBilling (cloud/ec2_util.go:256-268)."""
    by_the_second = any(a in d.arch for a in ("linux", "windows"))
    commercial = any(c in d.id for c in ("suse",))
    return not by_the_second or commercial


def host_allocator_job(distro: M.Distro, info: M.DistroQueueInfo, n_up: int, n_provisioning: int, alloc,
                       spawned: Optional[int] = None) -> dict:
    """-> {n_hosts, n_hosts_free, status, report: dict of the evg_host_report fields (ratios as np.float32)}.
    `alloc` = (nHosts, nHostsFree, status) the allocator returned (not read for a single-task distro)."""
    report = {"time_to_empty_ns": 0, "time_to_empty_no_spawns_ns": 0, "scheduled_duration_ns": 0, "hosts_avail": 0,
              "hosts_spawned": 0, "overdue_in_groups": 0, "free_in_groups": 0, "required_in_groups": 0,
              "host_queue_ratio": np.float32(0), "no_spawns_ratio": np.float32(0), "drawdown": 0, "new_cap_target": 0,
              "killable_hosts": 0}
    single = distro.single_task_distro
    if single:  # :182-184
        n_hosts, n_free, status = w64(info.length_with_dependencies_met - n_provisioning), 0, 0
    else:       # :186-195
        n_hosts, n_free, status = alloc
        if status != 0:
            return {"n_hosts": n_hosts, "n_hosts_free": n_free, "status": status, "report": report}
    n_spawned = max(n_hosts, 0) if spawned is None else spawned  # len(hostsSpawned) (:233)
    overdue = n_over = d_over = expected = free = required = 0
    for g in info.task_group_infos:  # :271-280
        if g.name != "":
            overdue = w64(overdue + g.count_wait_over_threshold)
            n_over = w64(n_over + g.count_duration_over_threshold)
            d_over = w64(d_over + g.duration_over_threshold)
            expected = w64(expected + g.expected_duration)
            if not single:  # the reference never ran the allocator: the infos hold the planner's zeros
                free = w64(free + g.count_free)
                required = w64(required + g.count_required)
    corrected_expected = w64(info.expected_duration - expected)              # :283
    corrected_over = w64(info.duration_over_threshold - d_over)              # :285
    sched = w64(corrected_expected - corrected_over)                         # :287
    over_no_groups = w64(info.count_duration_over_threshold - n_over)        # :289
    corrected_spawned = w64(n_spawned - required)                            # :292
    avail = w64(w64(w64(n_free - free) + corrected_spawned) - over_no_groups)  # :294
    tte = tte_ns = 0
    if sched > 0:  # :304-321
        avail_ns = w64(avail - corrected_spawned)
        if avail <= 0:
            tte = tte_ns = MAX_POSSIBLE_TIME
        elif avail_ns <= 0:
            tte, tte_ns = go_div(sched, avail), MAX_POSSIBLE_TIME
        else:
            tte, tte_ns = go_div(sched, avail), go_div(sched, avail_ns)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = f32(tte) / f32(info.max_duration_threshold)        # :324
        ratio_ns = f32(tte_ns) / f32(info.max_duration_threshold)  # :326
    report.update(time_to_empty_ns=tte, time_to_empty_no_spawns_ns=tte_ns, scheduled_duration_ns=sched, hosts_avail=avail,
                  hosts_spawned=n_spawned, overdue_in_groups=overdue, free_in_groups=free, required_in_groups=required,
                  host_queue_ratio=ratio, no_spawns_ratio=ratio_ns)
    terminate = distro.host_allocator_settings.hosts_overallocated_rule == M.HOSTS_OVERALLOCATED_TERMINATE  # :330
    if terminate and distro.provider in M.PROVIDER_SPAWNABLE and ratio < LOW_RATIO_THRESH and n_up > 0 \
            and not uses_hourly_billing(distro):  # :331-335
        killable, cap = n_up, 0  # setTargetAndTerminate :394-425
        if ratio != 0:
            with np.errstate(over="ignore"):
                killable = f32_to_int(f32(n_up) * (np.float32(1) - ratio))
            cap = n_up - killable
        if cap < distro.host_allocator_settings.minimum_hosts:
            cap = distro.host_allocator_settings.minimum_hosts
        report.update(killable_hosts=killable, new_cap_target=cap, drawdown=int(killable > 0))
    return {"n_hosts": n_hosts, "n_hosts_free": n_free, "status": status, "report": report}


def float_bits(x) -> int:
    return int(np.array([x], dtype=np.float32).view(np.uint32)[0])


def same_float(a, b) -> bool:
    """Bit-equal float32 values; two NaNs match whatever their payloads (Go's NaN bits depend on the CPU)."""
    a, b = np.float32(a), np.float32(b)
    if np.isnan(a) or np.isnan(b):
        return bool(np.isnan(a) and np.isnan(b))
    return float_bits(a) == float_bits(b)
