#!/usr/bin/env python3
"""Generate tests/golden/host_termination.json: the drawdown job (units/host_drawdown.go:70-159) and the idle-host
job (units/host_monitoring_idle_termination.go:64-342) on small hand-checkable inputs.

Cases named `reference:` are the reference's own tests, encoded as the job sees them: the idle hosts its query returns
(hosts running a task are not among them), in query order.  The tests' `time.Now()` offsets become offsets from the
instant they insert their documents, 1 ms before the job's frozen clock NOW: two drawdown tests rely on some time
passing between the two (a host idle for exactly the 5 s cutoff is not over it).  The mock cloud manager's TimeTilNextPayment is 0
for these hosts, and the mock environment's scheduler config has AcceptableHostIdleTimeSeconds 0.  `expect.hosts` are
the ids the test asserts (compared as a set); `expect.count` the count it asserts.

Cases named `branch:` take one branch each, worked out by hand in `why`; `expect.decisions` gives the EVG_HT_* code
and, where the job compares one, the threshold of every host.  Together they take every decision code and every
threshold rule (`rules`).
"""
import json
import os

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_termination.json")
NOW = 1_800_000_000 * 10 ** 9
S = 10 ** 9
MIN = 60 * S
ZERO = -(2 ** 63)


INSERT = NOW - 10 ** 6  # the reference tests insert their documents, then run the job: here 1 ms later


def ago(d):
    return NOW - d


def at(d):  # the reference tests' time.Now().Add(-d), taken when they insert their documents
    return INSERT - d


def host(hid, **kw):
    return dict(id=hid, **kw)


def running(hid, **kw):  # a running, provisioned host of the reference tests
    return host(hid, status="running", **kw)


def drawdown(name, source, distros, expect, why="", rules=()):
    return dict(name=name, source=source, job="drawdown", distros=distros, expect=expect, why=why, rules=list(rules))


def idle(name, source, distros, expect, why="", rules=(), sched_idle_seconds=0):
    return dict(name=name, source=source, job="idle", sched_idle_seconds=sched_idle_seconds, distros=distros, expect=expect,
                why=why, rules=list(rules))


def dd(did, idle_hosts, existing, cap, qlen=0):
    return dict(id=did, idle_hosts=idle_hosts, existing_hosts=existing, new_cap_target=cap, queue_length_dm=qlen)


def idistro(did, idle_hosts, running_count, minimum=0, idle_ns=0, default_ami="", missing=False):
    return dict(id=did, idle_hosts=idle_hosts, running_hosts_count=running_count, minimum_hosts=minimum,
                acceptable_idle_ns=idle_ns, default_ami=default_ami, missing=missing)


R_DD = "units/host_drawdown_test.go TestHostDrawdown/"
R_IT = "units/host_monitoring_idle_termination_test.go "

CASES = [
    # ---------------------------------------------------------------- reference: TestHostDrawdown (9 cases)
    drawdown("reference: DecommissionsHostsDownToCap", R_DD + "DecommissionsHostsDownToCap",
             [dd("d", [running("h3", creation_time=at(30 * MIN)), running("h4", creation_time=at(30 * MIN)),
                       running("h5", creation_time=at(20 * MIN))], 5, 3)],
             {"hosts": ["h3", "h4"], "count": 2},
             "5 hosts can run tasks, cap 3: target 2; h1 and h2 run tasks and are not idle"),
    drawdown("reference: IgnoresSingleHostTaskGroupHosts", R_DD + "IgnoresSingleHostTaskGroupHosts",
             [dd("d", [running("h2", creation_time=at(30 * MIN), last_group="dummy_task_group2", last_task="dummy_task_name2",
                               last_task_single_host_task_group=True)], 2, 0)],
             {"hosts": [], "count": 0}, "h1 runs a task; h2's last task is a succeeded single-host task group task"),
    drawdown("reference: IgnoresHostRunningTask", R_DD + "IgnoresHostRunningTask", [dd("d", [], 1, 0)],
             {"hosts": [], "count": 0}, "the only host runs a task, so no host is idle"),
    drawdown("reference: IgnoresHostThatRecentlyRanTaskGroup", R_DD + "IgnoresHostThatRecentlyRanTaskGroup",
             [dd("d", [running("h1", creation_time=at(30 * MIN), last_task="dummy_task_group1", last_group="dummy_task_group1",
                               last_task_completed_time=at(MIN), last_task_single_host_task_group=None)], 1, 0)],
             {"hosts": [], "count": 0}, "the last task id names no task: the lookup fails and the host is kept"),
    drawdown("reference: DecommissionsIdleMultiHostTaskGroupHost", R_DD + "DecommissionsIdleMultiHostTaskGroupHost",
             [dd("d", [running("h1", creation_time=at(30 * MIN), last_task="dummy_task_name1",
                               last_task_completed_time=at(20 * MIN))], 1, 0)],
             {"hosts": ["h1"], "count": 1}),
    drawdown("reference: HandlesHostInTeardown", R_DD + "HandlesHostInTeardown",
             [dd("d", [running("recent", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               task_group_teardown_start_time=INSERT),
                       running("old", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               task_group_teardown_start_time=at(30 * MIN))], 2, 0)],
             {"hosts": ["old"], "count": 1}),
    drawdown("reference: HandlesIdleHostsWithTaskQueue", R_DD + "HandlesIdleHostsWithTaskQueue",
             [dd("d", [running("active", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               last_task_completed_time=at(5 * S), last_task="dummy_task_name1", acceptable_host_idle_time=90 * S),
                       running("stale", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               acceptable_host_idle_time=90 * S)], 2, 0, 1)],
             {"hosts": ["stale"], "count": 1}),
    drawdown("reference: HandlesIdleHostsWithTaskQueueWithNoDependenceMet", R_DD + "HandlesIdleHostsWithTaskQueueWithNoDependenceMet",
             [dd("d", [running("active", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               last_task_completed_time=at(5 * S), last_task="dummy_task_name1", acceptable_host_idle_time=90 * S),
                       running("stale", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               acceptable_host_idle_time=90 * S)], 2, 0, 0)],
             {"hosts": ["active", "stale"], "count": 2}),
    drawdown("reference: HandlesIdleHostsWithNoQueue", R_DD + "HandlesIdleHostsWithNoQueue",
             [dd("d", [running("active", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               last_task_completed_time=at(5 * S), last_task="dummy_task_name1", acceptable_host_idle_time=90 * S),
                       running("stale", creation_time=at(30 * MIN), last_communication_time=at(MIN),
                               acceptable_host_idle_time=90 * S)], 2, 0, 0)],
             {"hosts": ["active", "stale"], "count": 2}),
    # ---------------------------------------------------------------- reference: TestFlaggingIdleHosts (12 subtests)
    idle("reference: HostsCurrentlyRunningTasksShouldNeverBeFlagged", R_IT + "TestFlaggingIdleHosts/HostsCurrentlyRunningTasksShouldNeverBeFlagged",
         [idistro("distro1", [], 1, idle_ns=4 * MIN)], {"hosts": [], "count": 0}),
    idle("reference: EvenWithLastCommunicationTimeGreaterThanTenMinutes", R_IT + "TestFlaggingIdleHosts/EvenWithLastCommunicationTimeGreaterThanTenMinutes",
         [idistro("distro1", [], 1, idle_ns=4 * MIN)], {"hosts": [], "count": 0}),
    idle("reference: HostInBetweenSingleHostTaskGroupTasksShouldHaveExtraIdleTime",
         R_IT + "TestFlaggingIdleHosts/HostInBetweenSingleHostTaskGroupTasksShouldHaveExtraIdleTime",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT, last_task="t1", last_group="tg1",
                                      last_task_completed_time=at(3 * MIN), last_task_single_host_task_group=True)], 1, idle_ns=4 * MIN)],
         {"hosts": [], "count": 0}),
    idle("reference: HostInBetweenSingleHostTaskGroupTasksButIsLongIdleShouldBeIdleTerminated",
         R_IT + "TestFlaggingIdleHosts/HostInBetweenSingleHostTaskGroupTasksButIsLongIdleShouldBeIdleTerminated",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT, last_task="t1", last_group="tg1",
                                      last_task_completed_time=at(20 * MIN), last_task_single_host_task_group=True)], 1, idle_ns=4 * MIN)],
         {"hosts": ["host1"], "count": 1}),
    idle("reference: HostRunningTaskWithOutdatedAMIShouldNotBeIdleTerminated",
         R_IT + "TestFlaggingIdleHosts/HostRunningTaskWithOutdatedAMIShouldNotBeIdleTerminated",
         [idistro("distro1", [], 1, idle_ns=4 * MIN, default_ami="ami-newer")], {"hosts": [], "count": 0}),
    idle("reference: RecentlyActiveButCurrentlyIdleHostWithOutdatedAMIShouldBeIdleTerminated",
         R_IT + "TestFlaggingIdleHosts/RecentlyActiveButCurrentlyIdleHostWithOutdatedAMIShouldBeIdleTerminated",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT, last_task="t1",
                                      last_task_completed_time=at(S), ami="ami-older")], 1, idle_ns=4 * MIN, default_ami="ami-newer")],
         {"hosts": ["host1"], "count": 1}),
    idle("reference: HostWithOutdatedAMIInBetweenSingleHostTaskGroupTasksShouldNotBeIdleTerminated",
         R_IT + "TestFlaggingIdleHosts/HostWithOutdatedAMIInBetweenSingleHostTaskGroupTasksShouldNotBeIdleTerminated",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT, last_task="t1", last_group="tg1",
                                      last_task_completed_time=at(3 * MIN), ami="ami-older", last_task_single_host_task_group=True)],
                  1, idle_ns=4 * MIN, default_ami="ami-newer")],
         {"hosts": [], "count": 0}),
    idle("reference: HostsNotRunningTasksShouldBeFlaggedIfTheyHaveBeenIdleLongerThanIdleThreshold",
         R_IT + "TestFlaggingIdleHosts/HostsNotRunningTasksShouldBeFlaggedIfTheyHaveBeenIdleLongerThanIdleThreshold",
         [idistro("distro1", [running("host1", last_task="t1", last_task_completed_time=at(20 * MIN), last_communication_time=INSERT),
                              running("host2", last_task="t2", last_task_completed_time=at(2 * MIN), last_communication_time=INSERT)],
                  2, idle_ns=4 * MIN)],
         {"hosts": ["host1"], "count": 1}),
    idle("reference: HostsThatRecentlyRanTaskShouldBeFlaggedIfTheyHaveBeenIdleLongerThanIdleThreshold",
         R_IT + "TestFlaggingIdleHosts/HostsThatRecentlyRanTaskShouldBeFlaggedIfTheyHaveBeenIdleLongerThanIdleThreshold",
         [idistro("distro1", [running("host1", last_task="t1", last_task_completed_time=at(20 * MIN), last_communication_time=INSERT),
                              running("host2", last_task="t2", last_task_completed_time=at(2 * MIN), last_communication_time=INSERT)],
                  2, idle_ns=4 * MIN)],
         {"hosts": ["host1"], "count": 1}),
    idle("reference: LegacyHostsThatNeedNewAgentsShouldNotBeMarkedIdle",
         R_IT + "TestFlaggingIdleHosts/LegacyHostsThatNeedNewAgentsShouldNotBeMarkedIdle",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT, needs_new_agent=True,
                                      bootstrap_method="legacy-ssh")], 1, idle_ns=4 * MIN)],
         {"hosts": [], "count": 0}),
    idle("reference: NonLegacyHostsThatNeedNewAgentMonitorsShouldNotBeMarkedIdle",
         R_IT + "TestFlaggingIdleHosts/NonLegacyHostsThatNeedNewAgentMonitorsShouldNotBeMarkedIdle",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=at(5 * MIN),
                                      needs_new_agent_monitor=True, bootstrap_method="ssh")], 1, idle_ns=4 * MIN)],
         {"hosts": [], "count": 0}),
    idle("reference: NonLegacyHostsThatDoNotNeedNewAgentMonitorsShouldBeMarkedIdle",
         R_IT + "TestFlaggingIdleHosts/NonLegacyHostsThatDoNotNeedNewAgentMonitorsShouldBeMarkedIdle",
         [idistro("distro1", [running("host1", creation_time=at(24 * 60 * MIN), last_communication_time=at(MIN),
                                      needs_new_agent=True, bootstrap_method="ssh")], 1, idle_ns=4 * MIN)],
         {"hosts": ["host1"], "count": 1}),
    # ---------------------------------------------------------------- reference: the other idle-host tests
    idle("reference: AddSomeHostsWithReferencedDistrosThatDoNotExistInTheDistroCollection",
         R_IT + "TestFlaggingIdleHostsWithMissingDistroIDs/AddSomeHostsWithReferencedDistrosThatDoNotExistInTheDistroCollection",
         [idistro("distro2", [running("host1", creation_time=at(10 * MIN), last_communication_time=INSERT)], 1, minimum=1),
          idistro("distro1", [running("host2", creation_time=at(20 * MIN), last_communication_time=INSERT)], 1, minimum=2),
          idistro("distroZ", [running("host3", creation_time=at(30 * MIN), last_communication_time=INSERT)], 1, missing=True),
          idistro("distroA", [running("host4", creation_time=at(30 * MIN), last_communication_time=INSERT)], 1, missing=True),
          idistro("distroC", [running("host5", creation_time=at(20 * MIN), last_communication_time=INSERT)], 1, missing=True)],
         {"hosts": ["host3", "host4", "host5"], "count": 3},
         "the missing distros' hosts are evaluated with the zero distro: threshold 0 s, so communication time 0 >= 0"),
    idle("reference: NeitherHostShouldBeFlaggedAsIdleAsMinimumHostsIsTwo",
         R_IT + "TestFlaggingIdleHostsWhenNonZeroMinimumHosts/NeitherHostShouldBeFlaggedAsIdleAsMinimumHostsIsTwo",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT),
                              running("host2", creation_time=at(20 * MIN), last_communication_time=INSERT)], 2, minimum=2)],
         {"hosts": [], "count": 0, "min_evaluate": [0]}),
    idle("reference: MinimumHostsIsTwo;OneHostIsRunningItsTaskAndTwoHostsAreIdle",
         R_IT + "TestFlaggingIdleHostsWhenNonZeroMinimumHosts/MinimumHostsIsTwo;OneHostIsRunningItsTaskAndTwoHostsAreIdle",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT),
                              running("host2", creation_time=at(20 * MIN), last_communication_time=INSERT)], 3, minimum=2)],
         {"hosts": ["host1"], "count": 1, "min_evaluate": [1]}),
    idle("reference: TestTearingDownIsNotConsideredIdle", R_IT + "TestTearingDownIsNotConsideredIdle",
         [idistro("distro1", [running("host1", creation_time=at(30 * MIN), last_communication_time=INSERT),
                              running("host2", creation_time=at(30 * MIN), last_communication_time=INSERT, task_group_teardown_start_time=INSERT),
                              running("host3", creation_time=at(30 * MIN), last_communication_time=INSERT,
                                      task_group_teardown_start_time=at(20 * MIN)),
                              running("host4", creation_time=at(30 * MIN), last_communication_time=at(20 * MIN),
                                      task_group_teardown_start_time=INSERT)], 4)],
         {"hosts": ["host1", "host3"], "count": 2}),
    idle("reference: TestPopulateIdleHostJobsCalculations", R_IT + "TestPopulateIdleHostJobsCalculations",
         [idistro("distro1", [running("host4", creation_time=at(40 * MIN), last_communication_time=INSERT),
                              running("host1", creation_time=at(20 * MIN), last_communication_time=INSERT),
                              running("host2", creation_time=at(10 * MIN), last_communication_time=INSERT)], 4, minimum=3),
          idistro("distro2", [running("host5", creation_time=at(50 * MIN), last_communication_time=INSERT),
                              running("host3", creation_time=at(30 * MIN), last_communication_time=INSERT)], 2)],
         {"min_evaluate": [1, 2]}, "only the counts are asserted: 4 running - 3 minimum = 1 of 3 idle; 2 - 0 = 2 of 2"),
] + [
    idle(f"reference: TestGetNumHostsToEvaluate minimum {m}", R_IT + "TestGetNumHostsToEvaluate",
         [idistro("d1", [host("h1"), host("h2"), host("h3")], 5, minimum=m)], {"min_evaluate": [want]})
    for m, want in ((0, 3), (4, 1), (5, 0))
] + [
    # ---------------------------------------------------------------- branch cases: the drawdown job
    drawdown("branch: drawdown exemptions and lookup error",
             "host_drawdown.go:128-145, host_monitoring_idle_termination.go:287-338",
             [dd("d", [running("agent", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), needs_new_agent=True),
                       running("cloud", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), cloud_manager_error=True),
                       running("payment", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), time_til_next_payment=6 * MIN),
                       running("lookup", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_group="g", last_task="t",
                               last_task_completed_time=ago(MIN), last_task_single_host_task_group=None),
                       running("teardown", creation_time=ago(30 * MIN), last_communication_time=ago(MIN),
                               task_group_teardown_start_time=ago(4 * MIN))], 10, 0)],
             {"decisions": {"agent": ["EVG_HT_EXEMPT_AGENT", 0], "cloud": ["EVG_HT_ERR_CLOUD_MANAGER", 0],
                            "payment": ["EVG_HT_EXEMPT_PAYMENT", 0], "lookup": ["EVG_HT_ERR_TASK_LOOKUP", 0],
                            "teardown": ["EVG_HT_KEPT", 0]}, "hosts": [], "count": 0},
             "agent: legacy bootstrap needing an agent, communication 1 min < 10 min; cloud: the manager lookup fails; "
             "payment: 6 min > 5 min; lookup: LastGroup set and the task lookup fails; teardown: exactly 4 min is not past "
             "MaxTeardownGroupThreshold"),
    drawdown("branch: drawdown thresholds", "host_drawdown.go:147-158",
             [dd("d", [running("tg-kept", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), running_task_group="g",
                               bootstrap_method="user-data", agent_start_time=ago(10 * MIN)),
                       running("tg-over", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), running_task_group="g",
                               bootstrap_method="user-data", agent_start_time=ago(10 * MIN + 1)),
                       running("own-kept", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_task="t",
                               last_task_completed_time=ago(90 * S), acceptable_host_idle_time=90 * S),
                       running("cutoff-kept", creation_time=ago(30 * MIN), last_communication_time=ago(MIN),
                               bootstrap_method="user-data", agent_start_time=ago(5 * S)),
                       running("cutoff-over", creation_time=ago(30 * MIN), last_communication_time=ago(MIN),
                               bootstrap_method="user-data", agent_start_time=ago(5 * S + 1))], 10, 0, 3)],
             {"decisions": {"tg-kept": ["EVG_HT_KEPT", 10 * MIN], "tg-over": ["EVG_HT_DECOMMISSION", 10 * MIN],
                            "own-kept": ["EVG_HT_KEPT", 90 * S], "cutoff-kept": ["EVG_HT_KEPT", 5 * S],
                            "cutoff-over": ["EVG_HT_DECOMMISSION", 5 * S]},
              "hosts": ["tg-over", "cutoff-over"], "count": 2},
             "3 tasks have their dependencies met.  tg-*: user-data hosts idle since their agent started, in a running task "
             "group without a completed task: 10 min cutoff, kept at exactly 10 min, decommissioned 1 ns later; own-kept: "
             "a completed task, so the embedded distro's 90 s applies and 90 s is not over it; cutoff-*: the 5 s cutoff, "
             "kept at exactly 5 s",
             rules=("drawdown: 5 s", "drawdown: 10 min in a running task group", "drawdown: acceptable idle time")),
    drawdown("branch: drawdown target", "host_drawdown.go:91-97, 149-151",
             [dd("cap", [running("a", creation_time=ago(30 * MIN), last_communication_time=ago(MIN)),
                         running("b", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), needs_new_agent=True),
                         running("c", creation_time=ago(30 * MIN), last_communication_time=ago(MIN)),
                         running("d", creation_time=ago(30 * MIN), last_communication_time=ago(MIN))], 4, 2),
              dd("negative", [running("e", creation_time=ago(30 * MIN), last_communication_time=ago(MIN))], 2, 3),
              dd("none", [running("f", creation_time=ago(30 * MIN), last_communication_time=ago(MIN))], 2, None),
              dd("tg", [running("g", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), running_task_group="x")], 1, 0)],
             {"decisions": {"a": ["EVG_HT_DECOMMISSION", 5 * S], "b": ["EVG_HT_EXEMPT_AGENT", 0], "c": ["EVG_HT_DECOMMISSION", 5 * S],
                            "d": ["EVG_HT_NOT_CHECKED", 0], "e": ["EVG_HT_NOT_CHECKED", 0], "f": ["EVG_HT_NOT_CHECKED", 0],
                            "g": ["EVG_HT_DECOMMISSION", 10 * MIN]},
              "hosts": ["a", "c", "g"], "count": 3,
              "distros": [{"target": 2, "decommissioned": 2, "ran": 1}, {"target": -1, "decommissioned": 0, "ran": 1},
                          {"target": 0, "decommissioned": 0, "ran": 0}, {"target": 1, "decommissioned": 1, "ran": 1}]},
             "cap: target 4 - 2 = 2, a and c (b is exempt) reach it, so d is never checked; negative: target 2 - 3 = -1 "
             "stops before any host; none: no drawdown job; tg: provisioned long ago (idle = since Go's zero time) in a "
             "running task group, 10 min cutoff",
             rules=("drawdown: 5 s", "drawdown: 10 min in a running task group")),
    # ---------------------------------------------------------------- branch cases: the idle-host job
    idle("branch: idle exemptions, lookup error and teardown", "host_monitoring_idle_termination.go:158-283",
         [idistro("d", [running("cloud", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), cloud_manager_error=True),
                        running("payment", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), time_til_next_payment=6 * MIN),
                        running("lookup", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_group="g",
                                last_task="t", last_task_completed_time=ago(MIN), last_task_single_host_task_group=None),
                        running("teardown", creation_time=ago(30 * MIN), last_communication_time=ago(MIN),
                                task_group_teardown_start_time=ago(5 * MIN)),
                        running("agent", creation_time=ago(30 * MIN), last_communication_time=0, last_task="t",
                                last_task_completed_time=ago(MIN))], 5, idle_ns=10 * MIN)],
         {"decisions": {"cloud": ["EVG_HT_ERR_CLOUD_MANAGER", 0], "payment": ["EVG_HT_EXEMPT_PAYMENT", 0],
                        "lookup": ["EVG_HT_ERR_TASK_LOOKUP", 0], "teardown": ["EVG_HT_TERM_TEARDOWN", 10 * MIN],
                        "agent": ["EVG_HT_EXEMPT_AGENT", 0]}, "hosts": ["teardown"], "count": 1},
         "cloud: the manager lookup fails; payment: 6 min > 5 min; lookup: LastGroup set and the task lookup fails; "
         "teardown: idle = 5 min (its teardown is past 4 min) < 10 min, communication 0 while tearing down, and 5 min > "
         "4 min since the teardown start; agent: a Unix-epoch LastCommunicationTime is zero to utility.IsZeroTime, so "
         "the host waits for an agent, and its idle time 1 min < 10 min",
         rules=("idle: the distro's idle time",)),
    idle("branch: idle thresholds and reasons", "host_monitoring_idle_termination.go:194-226, 258-283",
         [idistro("d", [running("doubled-kept", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), running_task_group="g",
                                last_task="t", last_task_completed_time=ago(7 * MIN)),
                        running("single-idle", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_group="g",
                                last_task="t", last_task_completed_time=ago(5 * MIN), last_task_single_host_task_group=True),
                        running("comm", creation_time=ago(30 * MIN), last_communication_time=ago(4 * MIN), last_task="t",
                                last_task_completed_time=ago(MIN)),
                        running("ami", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_task="t",
                                last_task_completed_time=ago(1), ami="old"),
                        running("beyond", creation_time=ago(30 * MIN), last_communication_time=ago(MIN), last_task="t",
                                last_task_completed_time=ago(20 * MIN))], 3, idle_ns=4 * MIN)],
         {"decisions": {"doubled-kept": ["EVG_HT_KEPT", 8 * MIN], "single-idle": ["EVG_HT_TERM_IDLE", 5 * MIN],
                        "comm": ["EVG_HT_TERM_COMMUNICATION", 4 * MIN], "ami": ["EVG_HT_TERM_OUTDATED_AMI", 4 * MIN],
                        "beyond": ["EVG_HT_NOT_CHECKED", 0]},
          "hosts": ["single-idle", "comm", "ami"], "count": 3, "min_evaluate": [3]},
         "3 running, minimum 0: the first 3 rows are evaluated and then only outdated AMIs (ami: 1 ns idle); doubled: 7 min < "
         "2 x 4 min; single-idle: 5 min >= the 5 min single-host cutoff; comm: 4 min >= 4 min; beyond is the 5th row",
         rules=("idle: doubled in a running task group", "idle: 5 min in a single-host task group", "idle: the distro's idle time")),
    idle("branch: idle missing distro and the scheduler's idle time", "host_monitoring_idle_termination.go:92-110, 197-200",
         [idistro("gone", [running("m", creation_time=ago(30 * MIN), last_communication_time=ago(3 * MIN))], 1, missing=True)],
         {"decisions": {"m": ["EVG_HT_TERM_COMMUNICATION", 2 * MIN]}, "hosts": ["m"], "count": 1},
         "a missing distro evaluates with MinimumHosts 0 and AcceptableHostIdleTime 0, so the scheduler config's 120 s "
         "applies: communication 3 min >= 2 min", rules=("idle: the scheduler config's idle time",), sched_idle_seconds=120),
]

RULES = ("drawdown: 5 s", "drawdown: 10 min in a running task group", "drawdown: acceptable idle time",
         "idle: the distro's idle time", "idle: the scheduler config's idle time", "idle: 5 min in a single-host task group",
         "idle: doubled in a running task group")


def main():
    with open(OUT, "w") as f:
        json.dump({"now": NOW, "rules": list(RULES), "cases": CASES}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
