"""The host allocator job's decisions without a GPU: the layout of the evg_host_job structs, the restatement
oracle_host_job on every golden case, each case's stated job inputs against the CPU oracle's planner and allocator
run on its tick, and the job settings soa.marshal_host_job builds."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import host_job_cases as HC
import oracle_host_job as OJ
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler as S
from evergreen_b200 import soa
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = HC.CASES["cases"]


def test_struct_layout(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(evg_host_job_cfg), offsetof(evg_host_job_cfg, n_provisioning),
         offsetof(evg_host_job_cfg, single_task_distro), offsetof(evg_host_job_cfg, terminate_when_overallocated),
         offsetof(evg_host_job_cfg, hourly_billing));
  printf("%zu", sizeof(evg_host_report));
#define F(f) printf(" %zu", offsetof(evg_host_report, f));
  F(time_to_empty_ns) F(time_to_empty_no_spawns_ns) F(scheduled_duration_ns) F(hosts_avail) F(hosts_spawned)
  F(overdue_in_groups) F(free_in_groups) F(required_in_groups) F(new_cap_target) F(killable_hosts)
  F(host_queue_ratio) F(no_spawns_ratio) F(drawdown)
  printf("\n%zu %zu %zu %zu %zu\n", sizeof(evg_host_job_out), offsetof(evg_host_job_out, n_hosts),
         offsetof(evg_host_job_out, n_hosts_free), offsetof(evg_host_job_out, status), offsetof(evg_host_job_out, report));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    out = [[int(x) for x in line.split()] for line in subprocess.check_output([str(exe)]).decode().strip().split("\n")]
    cd, rd = L.HOST_JOB_CFG_DTYPE, L.HOST_REPORT_DTYPE
    assert out[0] == [cd.itemsize] + [cd.fields[f][1] for f in ("n_provisioning", "single_task_distro",
                                                                 "terminate_when_overallocated", "hourly_billing")]
    assert out[1] == [rd.itemsize] + [rd.fields[f][1] for f in L.HOST_REPORT_FIELDS]
    S_ = L.HostJobOutStruct
    assert out[2] == [ctypes.sizeof(S_)] + [getattr(S_, f).offset for f in ("n_hosts", "n_hosts_free", "status", "report")]


def assert_job(got: dict, expect: dict, where: str):
    assert (got["n_hosts"], got["n_hosts_free"], got["status"]) == (expect["n_hosts"], expect["n_hosts_free"], expect["status"]), where
    for f in L.HOST_REPORT_FIELDS:
        want = expect["report"][f]
        if f in ("host_queue_ratio", "no_spawns_ratio"):
            want = np.array([int(want, 16)], dtype=np.uint32).view(np.float32)[0] if isinstance(want, str) else want
            assert OJ.same_float(got["report"][f], want), (where, f, got["report"][f], want)
        else:
            assert int(got["report"][f]) == int(want), (where, f, got["report"][f], want)


def test_golden_covers_every_branch():
    assert CASES[0]["name"] == "TestSingleTaskDistroHostAllocatorJob" and CASES[0]["expect"]["n_hosts"] == 1
    branches = " ".join(b for c in CASES for b in c["branches"])
    for b in ("scheduledDuration <= 0", "hostsAvail <= 0", "hostsAvailNoSpawns <= 0", "hostQueueRatio == 0 ",
              "0 < hostQueueRatio < 0.25", "hostQueueRatio == 0.25", "MinimumHosts", "killableHosts == 0",
              "HostsOverallocatedRule", "ProviderSpawnable", "UsesHourlyBilling", "no up hosts", "MaxDurationThreshold == 0",
              "float32(int64)", "task groups contribute", "single-task distro with task groups", "allocator error"):
        assert b in branches, b


@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_restatement_on_golden(c):
    info, alloc = HC.job_input(c)
    data = HC.allocator_data(c)
    got = OJ.host_allocator_job(data.distro, info, len(data.existing_hosts), c["n_provisioning"], alloc, c["spawned"])
    assert_job(got, c["expect"], c["name"])


@pytest.mark.parametrize("c", CASES, ids=lambda c: c["name"])
def test_golden_inputs_match_the_oracle_tick(c):
    """The job inputs each case states are what the CPU oracle's GetDistroQueueInfo and UtilizationBasedHostAllocator
    compute from the case's tick."""
    distro, tasks, data = HC.batch_entry(c)
    info = O.queue_info(distro.id, tasks, HC.threshold(c), False, HC.NOW)
    data.distro_queue_info = info
    n, f, st = O.allocate(data, HC.NOW)
    want, alloc = HC.job_input(c)
    if not distro.single_task_distro:
        assert (n, f, st) == alloc
    for k in ("length_with_dependencies_met", "expected_duration", "max_duration_threshold", "count_duration_over_threshold",
              "duration_over_threshold"):
        assert getattr(info, k) == getattr(want, k), k
    named = [g for g in info.task_group_infos if g.name != ""]
    assert len(named) == len(want.task_group_infos)
    for g, w in zip(named, want.task_group_infos):
        for k in ("name", "expected_duration", "count_duration_over_threshold", "duration_over_threshold",
                  "count_wait_over_threshold"):
            assert getattr(g, k) == getattr(w, k), k
        if not distro.single_task_distro:
            assert (g.count_free, g.count_required) == (w.count_free, w.count_required)


def test_marshal_host_job():
    datas = [HC.allocator_data(c) for c in CASES]
    prov = list(range(len(datas)))
    rows = soa.marshal_host_job(datas, prov)
    assert rows.dtype == L.HOST_JOB_CFG_DTYPE and rows.shape == (len(datas),)
    for r, d, p in zip(rows, datas, prov):
        assert int(r["n_provisioning"]) == p
        assert bool(r["single_task_distro"]) == d.distro.single_task_distro
        assert bool(r["terminate_when_overallocated"]) == (d.distro.host_allocator_settings.hosts_overallocated_rule ==
                                                           M.HOSTS_OVERALLOCATED_TERMINATE)
        assert bool(r["hourly_billing"]) == OJ.uses_hourly_billing(d.distro)
    with pytest.raises(ValueError):
        soa.marshal_host_job(datas, prov[:-1])


@pytest.mark.parametrize("arch,did,hourly", [("linux_amd64", "ubuntu", False), ("windows-64", "win", False),
                                             ("osx", "mac", True), ("", "x", True), ("linux_arm64", "suse15", True),
                                             ("windows", "opensuse-ish", True)])
def test_uses_hourly_billing(arch, did, hourly):
    d = M.Distro(id=did, arch=arch)
    assert S.uses_hourly_billing(d) == hourly == OJ.uses_hourly_billing(d)


def test_restatement_wraps_and_saturates():
    """int64 wrap of the group sums and the saturating float32 -> int conversion a negative threshold reaches."""
    d = M.Distro(id="d", provider=M.PROVIDER_EC2_FLEET, arch="linux",
                 host_allocator_settings=M.HostAllocatorSettings(hosts_overallocated_rule=M.HOSTS_OVERALLOCATED_TERMINATE))
    big = 2 ** 62
    g = [M.TaskGroupInfo(name=f"g{i}", expected_duration=big) for i in range(4)]
    info = M.DistroQueueInfo(expected_duration=0, max_duration_threshold=-1, task_group_infos=g)
    got = OJ.host_allocator_job(d, info, 3, 0, (0, 5, 0))
    assert got["report"]["scheduled_duration_ns"] == 0  # 0 - (4 * 2^62 wrapped to 0)
    info = M.DistroQueueInfo(expected_duration=3 * 10 ** 18, max_duration_threshold=-1)
    got = OJ.host_allocator_job(d, info, 4, 0, (0, 1, 0))  # float32(4) * (1 + 3e18) is past the int64 range
    r = got["report"]
    assert r["time_to_empty_ns"] == 3 * 10 ** 18 and r["host_queue_ratio"] < 0
    assert r["killable_hosts"] == 2 ** 63 - 1 and r["drawdown"] == 1 and r["new_cap_target"] == 0
