"""The drawdown and idle-host jobs without a GPU: the layout of their structs, the restatement on every golden case,
the golden's coverage, the idle-host table soa.marshal_idle_hosts builds, and Go's Duration.String."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import host_termination_cases as HT
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN = M.MINUTE


def test_struct_layout(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
#define F(s, f) printf(" %zu", offsetof(s, f));
int main(void) {
  printf("%zu", sizeof(evg_idle_host_soa));
  F(evg_idle_host_soa, n_hosts) F(evg_idle_host_soa, n_distros) F(evg_idle_host_soa, creation_ns) F(evg_idle_host_soa, start_ns)
  F(evg_idle_host_soa, provision_ns) F(evg_idle_host_soa, agent_start_ns) F(evg_idle_host_soa, last_communication_ns)
  F(evg_idle_host_soa, last_task_completed_ns) F(evg_idle_host_soa, teardown_start_ns) F(evg_idle_host_soa, acceptable_idle_ns)
  F(evg_idle_host_soa, flags)
  printf("\n%zu", sizeof(evg_host_verdict));
  F(evg_host_verdict, idle_ns) F(evg_host_verdict, communication_ns) F(evg_host_verdict, threshold_ns)
  F(evg_host_verdict, since_teardown_ns) F(evg_host_verdict, decision)
  printf("\n%zu", sizeof(evg_drawdown_distro));
  F(evg_drawdown_distro, target) F(evg_drawdown_distro, decommissioned) F(evg_drawdown_distro, ran)
  printf("\n%zu", sizeof(evg_idle_cfg));
  F(evg_idle_cfg, minimum_hosts) F(evg_idle_cfg, running_hosts_count) F(evg_idle_cfg, acceptable_idle_ns)
  printf("\n%zu", sizeof(evg_idle_distro));
  F(evg_idle_distro, min_evaluate) F(evg_idle_distro, terminated)
  printf("\n%zu", sizeof(evg_drawdown_in));
  F(evg_drawdown_in, existing_hosts) F(evg_drawdown_in, new_cap_target) F(evg_drawdown_in, queue_length_dm)
  printf("\n%zu", sizeof(evg_host_drawdown_out));
  F(evg_host_drawdown_out, hosts) F(evg_host_drawdown_out, distros)
  printf("\n%zu", sizeof(evg_idle_hosts_out));
  F(evg_idle_hosts_out, hosts) F(evg_idle_hosts_out, distros)
  printf("\n%d %d %d %d %lld\n", EVG_IH_CLOUD_MANAGER_FAILED, EVG_IH_OUTDATED_AMI, EVG_HT_TERM_TEARDOWN, EVG_HT_DECOMMISSION,
         (long long)EVG_NO_DRAWDOWN);
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    out = [[int(x) for x in line.split()] for line in subprocess.check_output([str(exe)]).decode().strip().split("\n")]

    def of(dt):
        return [dt.itemsize] + [dt.fields[f][1] for f in dt.names if f != "_reserved"]

    def of_struct(st):
        return [ctypes.sizeof(st)] + [getattr(st, f).offset for f, _ in st._fields_ if f != "_reserved"]

    assert out[0] == of_struct(L.IdleHostSoAStruct)
    assert out[1] == of(L.HOST_VERDICT_DTYPE)
    assert out[2] == of(L.DRAWDOWN_DISTRO_DTYPE)
    assert out[3] == of(L.IDLE_CFG_DTYPE)
    assert out[4] == of(L.IDLE_DISTRO_DTYPE)
    assert out[5] == of_struct(L.DrawdownInStruct)
    assert out[6] == out[7] == of_struct(L.HostTermOutStruct)
    assert out[8] == [L.EVG_IH_CLOUD_MANAGER_FAILED, L.EVG_IH_OUTDATED_AMI, L.EVG_HT_TERM_TEARDOWN, L.EVG_HT_DECOMMISSION,
                      L.EVG_NO_DRAWDOWN]


@pytest.mark.parametrize("name", sorted(HT.CASES))
def test_restatement_on_golden(name):
    c = HT.CASES[name]
    jobs, verdicts = HT.run_oracle(c)
    e = c["expect"]
    ran = [j for j in jobs if j is not None]
    if "hosts" in e:
        assert sorted(h for j in ran for h in HT.picked(j)) == sorted(e["hosts"])
    if "count" in e:
        assert sum(len(HT.picked(j)) for j in ran) == e["count"]
    if "min_evaluate" in e:
        assert [j.min_hosts_to_evaluate for j in jobs] == e["min_evaluate"]
    if "distros" in e:
        for j, d, want in zip(jobs, c["distros"], e["distros"]):
            got = ({"target": 0, "decommissioned": 0, "ran": 0} if j is None else
                   {"target": j.drawdown_target, "decommissioned": j.decommissioned, "ran": 1})
            assert got == want, d["id"]
    ids = [h["id"] for d in c["distros"] for h in d["idle_hosts"]]
    for hid, (code, threshold) in e.get("decisions", {}).items():
        v = verdicts[ids.index(hid)]
        assert (v[0], v[3]) == (HT.code(code), threshold), hid


def test_golden_covers_every_decision_and_threshold_rule():
    codes = {HT.code(code) for c in HT.CASES.values() for code, _ in c["expect"].get("decisions", {}).values()}
    assert codes == set(range(L.EVG_HT_TERM_TEARDOWN + 1))
    rules = {r for c in HT.CASES.values() for r in c["rules"]}
    assert rules == set(HT.GOLDEN["rules"])
    names = [c["source"] for c in HT.CASES.values() if c["name"].startswith("reference:")]
    assert sum("TestHostDrawdown/" in s for s in names) == 9
    assert sum("TestFlaggingIdleHosts/" in s for s in names) == 12
    for t in ("WithMissingDistroIDs", "WhenNonZeroMinimumHosts", "TestTearingDownIsNotConsideredIdle",
              "TestPopulateIdleHostJobsCalculations", "TestGetNumHostsToEvaluate"):
        assert any(t in s for s in names), t


def test_marshal_idle_hosts_round_trips():
    groups = [[M.Host(id="a", status="running", creation_time=5, start_time=6, provision_time=7, agent_start_time=8,
                      last_communication_time=9, last_task_completed_time=10, task_group_teardown_start_time=11,
                      acceptable_host_idle_time=12, running_task_group="g", last_task="t", bootstrap_method="user-data",
                      needs_new_agent=True, needs_new_agent_monitor=True, ami="x", last_group="g",
                      last_task_single_host_task_group=True, time_til_next_payment=5 * MIN + 1, cloud_manager_error=True)],
              [],
              [M.Host(id="b", bootstrap_method="legacy-ssh", last_group="g", last_task_single_host_task_group=None,
                      time_til_next_payment=5 * MIN), M.Host(id="c")]]
    t = soa.marshal_idle_hosts(groups, ["y", "", ""])
    assert (t.n_hosts, t.n_distros, t.ids, t.idle_off.tolist()) == (3, 3, ["a", "b", "c"], [0, 1, 1, 3])
    assert [t.cols[c][0] for c in L.IDLE_HOST_COLUMNS] == list(range(5, 13))
    assert t.cols["creation_ns"][1] == M.ZERO_TIME
    assert t.flags.tolist() == [
        L.EVG_IH_RUNNING_TASK_GROUP | L.EVG_IH_LAST_TASK | L.EVG_IH_STATUS_RUNNING | L.EVG_IH_USER_DATA | L.EVG_IH_NEEDS_NEW_AGENT
        | L.EVG_IH_NEEDS_NEW_AGENT_MONITOR | L.EVG_IH_OUTDATED_AMI | L.EVG_IH_SINGLE_HOST_TASK_GROUP | L.EVG_IH_PAYMENT_NOT_DUE
        | L.EVG_IH_CLOUD_MANAGER_FAILED,
        L.EVG_IH_LEGACY_BOOTSTRAP | L.EVG_IH_TASK_LOOKUP_FAILED,
        L.EVG_IH_LEGACY_BOOTSTRAP]
    s = t.struct()
    assert (s.n_hosts, s.n_distros, s.flags) == (3, 3, t.flags.ctypes.data)
    assert soa.marshal_idle_hosts(groups).flags[0] & L.EVG_IH_OUTDATED_AMI == 0  # the drawdown job does not read AMIs
    empty = soa.marshal_idle_hosts([])
    assert (empty.n_hosts, empty.n_distros, empty.idle_off.tolist(), empty.struct().creation_ns) == (0, 0, [0], None)


@pytest.mark.parametrize("field,value", [("creation_time", 2 ** 63), ("last_communication_time", -(2 ** 63) - 1),
                                         ("acceptable_host_idle_time", 2 ** 64)])
def test_marshal_idle_hosts_rejects_times_outside_int64(field, value):
    with pytest.raises(ValueError, match=field):
        soa.marshal_idle_hosts([[M.Host(id="h", **{field: value})]])


@pytest.mark.parametrize("d,want", [
    (0, "0s"), (1, "1ns"), (1100, "1.1µs"), (1500, "1.5µs"), (2_200_000, "2.2ms"), (1_500_000_000, "1.5s"),
    (4 * MIN, "4m0s"), (M.HOUR + 15 * MIN + 30 * M.SECOND + 918_273_645, "1h15m30.918273645s"), (-1_500_000_000, "-1.5s"),
    (-1, "-1ns"), (2 ** 63 - 1, "2562047h47m16.854775807s"), (-(2 ** 63), "-2562047h47m16.854775808s")])
def test_go_duration_string(d, want):
    assert M.go_duration_string(d) == want
