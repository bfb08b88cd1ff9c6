"""tests/golden/host_termination.json as model objects, and the restatement run on a case.  Shared by the CPU and GPU
tests of the drawdown and idle-host jobs."""
import json
import os

import oracle_host_termination as OT
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_termination.json")
GOLDEN = json.load(open(PATH))
NOW = GOLDEN["now"]
CASES = {c["name"]: c for c in GOLDEN["cases"]}


def hosts_of(d):
    return [M.Host(**h) for h in d["idle_hosts"]]


def distro_of(d):
    """The distro document of an idle-job distro, None when it is missing from the collection."""
    if d["missing"]:
        return None
    return M.Distro(id=d["id"], default_ami=d["default_ami"], host_allocator_settings=M.HostAllocatorSettings(
        minimum_hosts=d["minimum_hosts"], acceptable_host_idle_time=d["acceptable_idle_ns"]))


def run_oracle(case):
    """-> (per-distro job records, None where no drawdown ran; verdicts of every row in table order)."""
    jobs, verdicts = [], []
    for d in case["distros"]:
        hs = hosts_of(d)
        if case["job"] == "drawdown":
            if d["new_cap_target"] is None:
                job, v = None, [OT.NOT_CHECKED] * len(hs)
            else:
                job, v = OT.drawdown_job(d["id"], hs, d["existing_hosts"], d["new_cap_target"], d["queue_length_dm"], NOW)
        else:
            job, v = OT.idle_job(distro_of(d), hs, d["running_hosts_count"], NOW, case["sched_idle_seconds"])
        jobs.append(job)
        verdicts += v
    return jobs, verdicts


def picked(job):
    return job.decommissioned_hosts if isinstance(job, M.HostDrawdownJob) else job.terminated_hosts


def code(name):
    return getattr(L, name)
