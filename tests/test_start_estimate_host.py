"""The start-time estimator's host side without a GPU: marshal_estimate_hosts against the CPU restatement of
createSimulatorModel (every status, a task without a document, the failed-lookup cut-off), the new struct and constants
against the header, and the two answers get_estimated_start_time gives without reaching the device."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from oracle import oracle_estimate as OE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = json.load(open(os.path.join(ROOT, "tests", "golden", "task_start_estimation.json")))["models"]
MINUTE = 60 * 10 ** 9


def model_inputs(m):
    hosts = [M.Host(id=f"h{i}", status=h["status"], running_task=h["running_task"]) for i, h in enumerate(m["hosts"])]
    running = {k: S.TASK_LOOKUP_ERROR if v == "error" else None if v is None else M.Task(id=k, **v) for k, v in m["running"].items()}
    return hosts, running


def pool_of(table, now, d=0):
    """timeToCompletion of each row of distro d that contributes a host, as k_es_host computes it."""
    fixed = {L.EVG_EH_UNINITIALIZED: 4 * MINUTE, L.EVG_EH_STARTING: 3 * MINUTE, L.EVG_EH_PROVISIONING: MINUTE, L.EVG_EH_FREE: 0}
    out = []
    for i in range(int(table.est_host_off[d]), int(table.est_host_off[d + 1])):
        k = int(table.kind[i])
        if k == L.EVG_EH_RUNNING:
            out.append(OE.wrap(int(table.expected_ns[i]) - OE.since(now, int(table.dispatch_ns[i]))))
        elif k != L.EVG_EH_IGNORED:
            out.append(fixed[k])
    return out


@pytest.mark.parametrize("m", MODELS, ids=[m["name"] for m in MODELS])
def test_marshal_estimate_hosts_builds_the_reference_pool(m):
    hosts, running = model_inputs(m)
    table = S.marshal_estimate_hosts([hosts], running)
    assert pool_of(table, m["now"]) == m["expect"]
    oracle_running = {k: OE.LOOKUP_ERROR if v is S.TASK_LOOKUP_ERROR else v for k, v in running.items()}
    assert pool_of(table, m["now"]) == OE.create_simulator_model(m["queue"], hosts, oracle_running, m["now"]).hosts


def test_marshal_estimate_hosts_rows():
    now = 1_000 * MINUTE
    t = M.Task(id="t", expected_duration=5 * MINUTE, dispatch_time=now - MINUTE)
    d0 = [M.Host(status=M.HOST_UNINITIALIZED), M.Host(status=M.HOST_STARTING), M.Host(status=M.HOST_PROVISIONING),
          M.Host(status=M.HOST_RUNNING), M.Host(status=M.HOST_RUNNING, running_task="t"), M.Host(status="building"),
          M.Host(status=M.HOST_RUNNING, running_task="gone"), M.Host(status=M.HOST_RUNNING, running_task="none")]
    d1 = []
    d2 = [M.Host(status=M.HOST_RUNNING), M.Host(status=M.HOST_RUNNING, running_task="err"), M.Host(status=M.HOST_RUNNING)]
    d3 = [M.Host(status=M.HOST_STARTING, running_task="t")]  # only a running host's task is looked up
    table = S.marshal_estimate_hosts([d0, d1, d2, d3], {"t": t, "none": None, "err": S.TASK_LOOKUP_ERROR})
    assert table.est_host_off.tolist() == [0, 8, 8, 9, 10]  # the failed lookup ends distro 2 after its first host
    assert table.kind.tolist() == [L.EVG_EH_UNINITIALIZED, L.EVG_EH_STARTING, L.EVG_EH_PROVISIONING, L.EVG_EH_FREE, L.EVG_EH_RUNNING,
                                   L.EVG_EH_IGNORED, L.EVG_EH_IGNORED, L.EVG_EH_IGNORED, L.EVG_EH_FREE, L.EVG_EH_STARTING]
    assert table.expected_ns[4] == 5 * MINUTE and table.dispatch_ns[4] == now - MINUTE
    assert (table.kind.dtype, table.expected_ns.dtype, table.dispatch_ns.dtype, table.est_host_off.dtype) == (np.uint8, np.int64, np.int64, np.int64)
    assert (table.n_hosts, table.n_distros) == (10, 4)
    assert pool_of(table, now) == [4 * MINUTE, 3 * MINUTE, MINUTE, 0, 4 * MINUTE]
    assert set(M.UP_HOST_STATUS) >= {M.HOST_RUNNING, M.HOST_UNINITIALIZED, M.HOST_STARTING, M.HOST_PROVISIONING}


def test_struct_and_constants_match_the_header():
    src = open(os.path.join(ROOT, "include", "evg_sched.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct \{([^}]*)\} evg_est_host_soa;", src).group(1), flags=re.S)
    assert re.findall(r"(\w+);", body) == [f for f, _ in L.EstHostSoAStruct._fields_]
    assert C.sizeof(L.EstHostSoAStruct) == 32 and all(C.sizeof(t) == 8 for _, t in L.EstHostSoAStruct._fields_)
    enum = re.sub(r"/\*.*?\*/", "", re.search(r"enum \{\s*(EVG_EH_UNINITIALIZED.*?)\};", src, flags=re.S).group(1), flags=re.S)
    assert {k: int(v) for k, v in re.findall(r"(EVG_EH_\w+) = (\d+)", enum)} == {
        n: getattr(L, n) for n in ("EVG_EH_UNINITIALIZED", "EVG_EH_STARTING", "EVG_EH_PROVISIONING", "EVG_EH_FREE", "EVG_EH_RUNNING",
                                   "EVG_EH_IGNORED")}
    assert int(re.search(r"#define EVG_EST_ONCHIP_HOSTS (\d+)", src).group(1)) == L.EVG_EST_ONCHIP_HOSTS
    for name in ("evg_estimate_start_times", "evg_estimate_start_batch"):
        decl = re.search(name + r"\(([^;]*)\);", re.sub(r"/\*.*?\*/", "", src, flags=re.S)).group(1)
        assert len(decl.split(",")) == len(L.SYMBOLS[name][1]), name


def test_get_estimated_start_time_without_a_queue_or_a_position():
    class NoDevice:  # neither answer may reach the device
        def __getattr__(self, name):
            raise AssertionError(name)
    task = M.Task(id="t")
    hosts = [M.Host(status=M.HOST_RUNNING)]
    assert scheduler.get_estimated_start_time(task, None, hosts, {}, 0, engine=NoDevice()) == -1
    queue = M.TaskQueue(distro="d", queue=[M.TaskQueueItem(id="a", expected_duration=MINUTE)])
    assert scheduler.get_estimated_start_time(task, queue, hosts, {}, 0, engine=NoDevice()) == -1
