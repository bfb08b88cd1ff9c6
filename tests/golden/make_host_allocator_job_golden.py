#!/usr/bin/env python3
"""Generate tests/golden/host_allocator_job.json: hostAllocatorJob.Run past the allocator
(units/host_allocator.go:180-337, 394-425).

The first case is the reference's TestSingleTaskDistroHostAllocatorJob (units/host_allocator_test.go:20-77).
Every other case exercises one branch of the job, named in `branches` with the Go lines it takes.  Each case is a
tick small enough to follow by hand: the distro, its queued tasks, its up hosts, what the reference reads besides
them (provisioning hosts, hosts spawned), and:

  job_input  what the job reads after the allocator: the DistroQueueInfo fields, the named TaskGroupInfos with the
             CountFree / CountRequired the allocator wrote, and (nHosts, nHostsFree, error status);
  expect     the job's decisions, worked out below line by line from job_input (`why` shows the arithmetic).

Float32 values are the Go expressions float32(int64) / float32(int64) etc., evaluated here with numpy float32
scalars one operation at a time (int64 -> float32 rounds to nearest-even); the json keeps their bit patterns.
Most cases give the distro MaximumHosts 0 so that UtilizationBasedHostAllocator returns at its first check
(utilization_based_host_allocator.go:39-48): nHosts = 0 and nHostsFree = the free hosts.
"""
import json
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_allocator_job.json")
NOW = 1_800_000_000 * 10 ** 9
MIN = 60 * 10 ** 9
T = 30 * MIN                      # MaxDurationThreshold of most cases (distro.go:434-440 default)
MAXT = 2532000 * 3600 * 10 ** 9   # maxPossibleHours * time.Hour (host_allocator.go:309-313)


def f32(x: int) -> np.float32:
    """float32(int64), round to nearest-even (numpy casts int64 -> float32 directly)."""
    return np.array([x], dtype=np.int64).astype(np.float32)[0]


def bits(x: np.float32) -> str:
    return "0x%08x" % int(np.array([x], dtype=np.float32).view(np.uint32)[0])


def distro(name, **kw):
    d = {"Id": name, "Provider": "ec2-fleet", "Arch": "linux_amd64", "SingleTaskDistro": False, "TargetTime": T,
         "HostAllocatorSettings": {"MinimumHosts": 0, "MaximumHosts": 0, "FutureHostFraction": 0.0,
                                   "HostsOverallocatedRule": "terminate-hosts-when-overallocated"}}
    for k, v in kw.items():
        if k in ("MinimumHosts", "MaximumHosts", "FutureHostFraction", "HostsOverallocatedRule"):
            d["HostAllocatorSettings"][k] = v
        else:
            d[k] = v
    return d


def free_hosts(n):
    return [{"Id": f"h{i}"} for i in range(n)]


def report(tte=0, tte_ns=0, sched=0, avail=0, spawned=0, overdue=0, free=0, required=0, ratio=np.float32(0),
           ratio_ns=np.float32(0), drawdown=0, cap=0, killable=0):
    return {"time_to_empty_ns": tte, "time_to_empty_no_spawns_ns": tte_ns, "scheduled_duration_ns": sched,
            "hosts_avail": avail, "hosts_spawned": spawned, "overdue_in_groups": overdue, "free_in_groups": free,
            "required_in_groups": required, "host_queue_ratio": bits(ratio), "no_spawns_ratio": bits(ratio_ns),
            "drawdown": drawdown, "new_cap_target": cap, "killable_hosts": killable}


def qinfo(lwdm, expected, over_n=0, over_d=0, thr=T, groups=()):
    return {"LengthWithDependenciesMet": lwdm, "ExpectedDuration": expected, "CountDurationOverThreshold": over_n,
            "DurationOverThreshold": over_d, "MaxDurationThreshold": thr, "TaskGroupInfos": list(groups)}


cases = []

# ---- units/host_allocator_test.go:20-77: 3 queued tasks, 2 with dependencies met, 1 provisioning host
r = f32(30 * MIN) / f32(T)
r_ns = f32(MAXT) / f32(T)
cases.append({
    "name": "TestSingleTaskDistroHostAllocatorJob", "ref": "units/host_allocator_test.go:20-77",
    "branches": ["single-task bypass :182-184"],
    "distro": distro("d", SingleTaskDistro=True),
    "tasks": [{"Id": "t1", "ExpectedDuration": 10 * MIN}, {"Id": "t2", "ExpectedDuration": 10 * MIN},
              {"Id": "t3", "ExpectedDuration": 10 * MIN, "DependsOn": ["missing"]}],
    "hosts": [], "n_provisioning": 1, "spawned": None,
    "job_input": {"queue_info": qinfo(2, 30 * MIN), "n_hosts": 1, "n_hosts_free": 0, "status": 0},
    "expect": {"n_hosts": 1, "n_hosts_free": 0, "status": 0,
               "report": report(tte=30 * MIN, tte_ns=MAXT, sched=30 * MIN, avail=1, spawned=1, ratio=r, ratio_ns=r_ns)},
    "why": "nHosts = LengthWithDependenciesMet 2 - 1 provisioning = 1 (the test then finds 2 active hosts); "
           "spawned max(1,0) = 1; ExpectedDuration counts all 3 tasks (the distro does not include dependencies, "
           "scheduler.go:77-112): sched = 30m; hostsAvail = 0 + 1 - 0 = 1, noSpawns = 0 -> tte = 30m / 1, "
           "ttens = max; ratio = f32(30m)/f32(30m) = 1: no drawdown"})

# ---- scheduledDuration <= 0 (:304-306), then ratio exactly 0: killableHosts = numUpHosts, NewCapTarget 0 (:396-397)
cases.append({
    "name": "scheduled_duration_not_positive", "ref": "units/host_allocator.go:283-306,396-397,403-405",
    "branches": ["scheduledDuration <= 0 :304-306", "hostQueueRatio == 0 :396-397"],
    "distro": distro("d-sched"),
    "tasks": [{"Id": "t1", "ExpectedDuration": 40 * MIN}],
    "hosts": free_hosts(2), "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(1, 40 * MIN, 1, 40 * MIN), "n_hosts": 0, "n_hosts_free": 2, "status": 0},
    "expect": {"n_hosts": 0, "n_hosts_free": 2, "status": 0,
               "report": report(avail=1, drawdown=1, cap=0, killable=2)},
    "why": "the only task is over the threshold: sched = (40m - 0) - (40m - 0) = 0 -> both times 0, ratio 0/f32(30m) = 0; "
           "hostsAvail = (2 - 0) + 0 - 1 = 1; terminate, ec2-fleet, 0 < 0.25, 2 up hosts, by-the-second: "
           "killable = 2, NewCapTarget 0 (MinimumHosts 0)"})

# ---- hostsAvail <= 0 (:311-313)
r = f32(MAXT) / f32(T)
cases.append({
    "name": "hosts_avail_not_positive", "ref": "units/host_allocator.go:294,311-313",
    "branches": ["hostsAvail <= 0 :311-313"],
    "distro": distro("d-avail"),
    "tasks": [{"Id": "t1", "ExpectedDuration": 10 * MIN}],
    "hosts": [], "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(1, 10 * MIN), "n_hosts": 0, "n_hosts_free": 0, "status": 0},
    "expect": {"n_hosts": 0, "n_hosts_free": 0, "status": 0,
               "report": report(tte=MAXT, tte_ns=MAXT, sched=10 * MIN, avail=0, ratio=r, ratio_ns=r)},
    "why": "no hosts, none spawned: hostsAvail = 0 -> both times 2532000h; ratio = f32(9115200000000000000)/f32(30m)"})

# ---- only hostsAvailNoSpawns <= 0 (:314-316); also no up hosts (:332 len(upHosts) > 0)
r = f32(5 * MIN) / f32(T)
r_ns = f32(MAXT) / f32(T)
cases.append({
    "name": "only_no_spawns_not_positive", "ref": "units/host_allocator.go:292-294,314-316,332",
    "branches": ["hostsAvailNoSpawns <= 0 :314-316", "no up hosts :332"],
    "distro": distro("d-nospawn"),
    "tasks": [{"Id": "t1", "ExpectedDuration": 10 * MIN}],
    "hosts": [], "n_provisioning": 0, "spawned": 2,
    "job_input": {"queue_info": qinfo(1, 10 * MIN), "n_hosts": 0, "n_hosts_free": 0, "status": 0},
    "expect": {"n_hosts": 0, "n_hosts_free": 0, "status": 0,
               "report": report(tte=5 * MIN, tte_ns=MAXT, sched=10 * MIN, avail=2, spawned=2, ratio=r, ratio_ns=r_ns)},
    "why": "2 hosts spawned: correctedHostsSpawned 2, hostsAvail 2, noSpawns 0 -> tte = 10m/2 = 5m, ttens = max; "
           "ratio f32(5m)/f32(30m) ~ 0.167 < 0.25 but no up hosts: no drawdown"})


def truncation_case(name, ref, branches, tte, n_up, why, expect_fn, **dkw):
    """One standalone task of n_up * tte on n_up free hosts: hostsAvail = noSpawns = n_up, both times = tte."""
    r = f32(tte) / f32(T)
    return {"name": name, "ref": ref, "branches": branches, "distro": distro("d-" + name, **dkw),
            "tasks": [{"Id": "t1", "ExpectedDuration": n_up * tte}], "hosts": free_hosts(n_up), "n_provisioning": 0,
            "spawned": None,
            "job_input": {"queue_info": qinfo(1, n_up * tte), "n_hosts": 0, "n_hosts_free": n_up, "status": 0},
            "expect": {"n_hosts": 0, "n_hosts_free": n_up, "status": 0,
                       "report": dict(report(tte=tte, tte_ns=tte, sched=n_up * tte, avail=n_up, ratio=r, ratio_ns=r),
                                      **expect_fn(r))},
            "why": why}


# ratio in (0, 0.25): killable = int(float32(4) * (1 - r)), truncated (:399-400)
r01 = f32(180 * 10 ** 9) / f32(T)
k01 = int(np.float32(4) * (np.float32(1) - r01))  # f32 product 3.6, truncated
assert k01 == 3
cases.append(truncation_case(
    "ratio_below_quarter", "units/host_allocator.go:324,332-335,398-401", ["0 < hostQueueRatio < 0.25 :399-400"],
    180 * 10 ** 9, 4, "12m on 4 free hosts: tte = 3m, ratio ~ 0.1; killable = int(4 * 0.9 (float32)) = int(3.6) = 3, "
                      "NewCapTarget 4 - 3 = 1", lambda r: {"drawdown": 1, "killable_hosts": 3, "new_cap_target": 1}))
# ratio exactly 0.25f: not < lowRatioThresh (:329,332)
rq = f32(450 * 10 ** 9) / f32(T)
assert rq == np.float32(0.25)
cases.append(truncation_case(
    "ratio_exactly_quarter", "units/host_allocator.go:329,332", ["hostQueueRatio == 0.25 :332"], 450 * 10 ** 9, 1,
    "7.5m on 1 free host: f32(7.5m) / f32(30m) is exactly 0.25 (a power-of-two ratio): no drawdown", lambda r: {}))
# MinimumHosts floor (:403-405)
cases.append(truncation_case(
    "min_hosts_floor", "units/host_allocator.go:399-405", ["NewCapTarget < MinimumHosts :403-405"], 180 * 10 ** 9, 4,
    "as ratio_below_quarter: killable 3, NewCapTarget 4 - 3 = 1 < MinimumHosts 3 -> 3",
    lambda r: {"drawdown": 1, "killable_hosts": 3, "new_cap_target": 3}, MinimumHosts=3))
# killableHosts == 0: no drawdown job (:407-408), NewCapTarget still computed
r02 = f32(360 * 10 ** 9) / f32(T)
assert int(np.float32(1) * (np.float32(1) - r02)) == 0
cases.append(truncation_case(
    "killable_zero", "units/host_allocator.go:399-408", ["killableHosts == 0 :408"], 360 * 10 ** 9, 1,
    "6m on 1 free host: ratio ~ 0.2; killable = int(1 * 0.8) = 0, NewCapTarget 1 - 0 = 1; 0 > lowCountFloor fails",
    lambda r: {"drawdown": 0, "killable_hosts": 0, "new_cap_target": 1}))
# the drawdown conditions one at a time (:330-334): the ratio_below_quarter tick otherwise
cases.append(truncation_case(
    "terminate_off", "units/host_allocator.go:330,332", ["HostsOverallocatedRule != terminate :330"], 180 * 10 ** 9, 4,
    "ratio ~ 0.1 but the rule is unset: no drawdown", lambda r: {}, HostsOverallocatedRule=""))
cases.append(truncation_case(
    "static_provider", "units/host_allocator.go:331-332", ["provider not in ProviderSpawnable :331"], 180 * 10 ** 9, 4,
    "ratio ~ 0.1 but a static distro cannot be terminated: no drawdown", lambda r: {}, Provider="static"))
cases.append(truncation_case(
    "hourly_billing_arch", "units/host_allocator.go:333-334, cloud/ec2_util.go:256-268", ["UsesHourlyBilling :333-334"],
    180 * 10 ** 9, 4, "ratio ~ 0.1 but Arch osx_amd64 names no by-the-second OS: billed hourly, no drawdown",
    lambda r: {}, Arch="osx_amd64"))
cases.append(truncation_case(
    "hourly_billing_commercial_linux", "units/host_allocator.go:333-334, cloud/ec2_util.go:256-268",
    ["UsesHourlyBilling :333-334"], 180 * 10 ** 9, 4,
    "ratio ~ 0.1, Arch linux_amd64 but the id names suse: commercial Linux is billed hourly, no drawdown",
    lambda r: {}, Id="suse15-small"))

# ---- MaxDurationThreshold 0: float32(0) / float32(0) is NaN (:324-326), and NaN < 0.25 is false
nan = np.float32(np.nan)
cases.append({
    "name": "max_duration_threshold_zero", "ref": "units/host_allocator.go:324-326,332",
    "branches": ["MaxDurationThreshold == 0 :324-326"],
    "distro": distro("d-zero"), "raw_threshold": 0,
    "tasks": [{"Id": "t1", "ExpectedDuration": 10 * MIN}],
    "hosts": free_hosts(1), "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(1, 10 * MIN, 1, 10 * MIN, thr=0), "n_hosts": 0, "n_hosts_free": 1, "status": 0},
    "expect": {"n_hosts": 0, "n_hosts_free": 1, "status": 0,
               "report": report(avail=0, ratio=nan, ratio_ns=nan)},
    "why": "with a 0 threshold every task is over it: sched 0, both times 0, hostsAvail = 1 - 1 = 0; "
           "ratio = 0/0 = NaN (any NaN bit pattern); NaN < 0.25 is false: no drawdown"})

# ---- int64 -> float32 rounds once, to nearest-even: 2^60 + 2^36 + 1 -> 2^60 + 2^37 (via float64 it would tie to 2^60)
big = 2 ** 60 + 2 ** 36 + 1
rb = f32(big) / f32(2 ** 61)
assert bits(rb) == "0x3f000001"
cases.append({
    "name": "int64_to_float32_rounding", "ref": "units/host_allocator.go:318-319,324",
    "branches": ["float32(int64) rounding :324"],
    "distro": distro("d-round", TargetTime=2 ** 61),
    "tasks": [{"Id": "t1", "ExpectedDuration": big}],
    "hosts": free_hosts(1), "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(1, big, thr=2 ** 61), "n_hosts": 0, "n_hosts_free": 1, "status": 0},
    "expect": {"n_hosts": 0, "n_hosts_free": 1, "status": 0,
               "report": report(tte=big, tte_ns=big, sched=big, avail=1, ratio=rb, ratio_ns=rb)},
    "why": "tte = 2^60+2^36+1 on 1 host; float32 of it is 2^60+2^37 (above the half-way point), / 2^61 = 0.5 + 2^-24 "
           "(0x3f000001); rounding through float64 first would give 0.5"})

# ---- task groups: the allocator really runs (MaximumHosts 100, FutureHostFraction 1)
# group g: 2 tasks of 40m (both over the threshold), one scheduled 2h ago (waiting over it), the other 5m ago,
# TaskGroupMaxHosts 5;
# one up host runs a task of g that started 30m ago and is expected to take 30m; one free host; one standalone task of 10m.
# allocator: bucket g: soon-free term = clamp((30m - 0)/30m) = 1 -> expected free 1; required = floor(0/30m - 1 + 2) = 1
#            (utilization_based_host_allocator.go:135-220, 262-301, 324-394); bucket "": 1 free host, required
#            floor(10m/30m - 1) < 0 -> 0, free 1; nHosts = 0 + 1 = 1 (<= LengthWithDependenciesMet 3 - 1 free), nHostsFree = 2.
G_TASKS = [{"Id": "g1", "ExpectedDuration": 40 * MIN, "TaskGroup": "g", "TaskGroupMaxHosts": 5, "ScheduledAgo": 120 * MIN},
           {"Id": "g2", "ExpectedDuration": 40 * MIN, "TaskGroup": "g", "TaskGroupMaxHosts": 5, "ScheduledAgo": 5 * MIN},
           {"Id": "s1", "ExpectedDuration": 10 * MIN, "ScheduledAgo": 5 * MIN}]
G_HOSTS = [{"Id": "h0", "RunningTask": "rt", "RunningTaskGroup": "g"}, {"Id": "h1"}]
G_RUNNING = [{"Id": "rt", "ExpectedDuration": 30 * MIN, "StartAgo": 30 * MIN}]
G_INFO = {"Name": "g", "Count": 2, "ExpectedDuration": 80 * MIN, "CountDurationOverThreshold": 2,
          "DurationOverThreshold": 80 * MIN, "CountWaitOverThreshold": 1, "CountFree": 1, "CountRequired": 1}
r = f32(10 * MIN) / f32(T)
cases.append({
    "name": "task_groups", "ref": "units/host_allocator.go:271-294,304-320",
    "branches": ["task groups contribute free, required and overdue :271-280"],
    "distro": distro("d-groups", MaximumHosts=100, FutureHostFraction=1.0),
    "tasks": G_TASKS, "hosts": G_HOSTS, "running_tasks": G_RUNNING, "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(3, 90 * MIN, 2, 80 * MIN, groups=[G_INFO]), "n_hosts": 1, "n_hosts_free": 2, "status": 0},
    "expect": {"n_hosts": 1, "n_hosts_free": 2, "status": 0,
               "report": report(tte=10 * MIN, tte_ns=10 * MIN, sched=10 * MIN, avail=1, spawned=1, overdue=1, free=1,
                                required=1, ratio=r, ratio_ns=r)},
    "why": "groups: overdue 1, over 2 / 80m, expected 80m, free 1, required 1; sched = (90m - 80m) - (80m - 80m) = 10m; "
           "spawned max(1,0) = 1, corrected 1 - 1 = 0; hostsAvail = (2 - 1) + 0 - (2 - 2) = 1 = noSpawns; "
           "tte = ttens = 10m; ratio f32(10m)/f32(30m) ~ 0.333: no drawdown"})

# ---- the same tick as a single-task distro: its group counters are the planner's zeros (:182-184 skips the allocator)
r = f32(200 * 10 ** 9) / f32(T)
r_ns = f32(MAXT) / f32(T)
assert int(np.float32(2) * (np.float32(1) - r)) == 1
g_single = dict(G_INFO, CountFree=0, CountRequired=0)
cases.append({
    "name": "single_task_distro_with_groups", "ref": "units/host_allocator.go:182-184,271-320,396-405",
    "branches": ["single-task distro with task groups :182-184,271-280"],
    "distro": distro("d-groups-single", MaximumHosts=100, FutureHostFraction=1.0, SingleTaskDistro=True),
    "tasks": G_TASKS, "hosts": G_HOSTS, "running_tasks": G_RUNNING, "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(3, 90 * MIN, 2, 80 * MIN, groups=[g_single]), "n_hosts": 3, "n_hosts_free": 0, "status": 0},
    "expect": {"n_hosts": 3, "n_hosts_free": 0, "status": 0,
               "report": report(tte=200 * 10 ** 9, tte_ns=MAXT, sched=10 * MIN, avail=3, spawned=3, overdue=1,
                                ratio=r, ratio_ns=r_ns, drawdown=1, killable=1, cap=1)},
    "why": "nHosts = 3 - 0; free and required in groups 0; sched 10m; spawned 3, corrected 3; hostsAvail = 0 + 3 - 0 = 3, "
           "noSpawns 0 -> tte = 600s/3 = 200s, ttens = max; ratio ~ 0.111 < 0.25, 2 up hosts: "
           "killable = int(2 * 0.889) = 1, NewCapTarget 2 - 1 = 1"})

# ---- an allocator error ends the job (:191-195): FutureHostFraction > 1 (utilization_based_host_allocator.go:302-304)
cases.append({
    "name": "allocator_error", "ref": "units/host_allocator.go:191-195",
    "branches": ["allocator error :192-195"],
    "distro": distro("d-err", MaximumHosts=100, FutureHostFraction=1.5),
    "tasks": [{"Id": "t1", "ExpectedDuration": 10 * MIN}],
    "hosts": free_hosts(1), "n_provisioning": 0, "spawned": None,
    "job_input": {"queue_info": qinfo(1, 10 * MIN), "n_hosts": 0, "n_hosts_free": 1, "status": 1},
    "expect": {"n_hosts": 0, "n_hosts_free": 1, "status": 1, "report": report()},
    "why": "the allocator returns (0, len(freeHosts) = 1, error): no report, no drawdown"})

json.dump({"generated_from": "units/host_allocator.go, units/host_allocator_test.go", "now": NOW, "cases": cases},
          open(OUT, "w"), indent=1, sort_keys=True)
print(f"{len(cases)} cases -> {OUT}")
