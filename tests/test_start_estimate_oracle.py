"""The start-time estimator without a GPU: the CPU restatement (oracle_estimate) replays every call sequence of
tests/golden/task_start_estimation.json on one simulator object, builds every golden host pool, and its one-run form
(fresh_estimates, what the device computes) equals a fresh object's simulate(p) for every p."""
import json
import os
import types

import numpy as np
import pytest

from oracle import oracle_estimate as OE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "task_start_estimation.json")))
CASES, MODELS = GOLDEN["cases"], GOLDEN["models"]
REFERENCE_TESTS = {"TestNoHosts", "TestNoTasks", "TestManyFreeHosts", "TestSingleFreeHost", "TestSingleOccupiedHost", "TestMultipleHosts",
                   "TestMultipleHostsUnordered", "TestRunningHosts", "TestEvenDistribution"}


def ids(cases):
    return [c["name"] for c in cases]


def fresh_by_object(durations, pool):
    """simulate(p) of a NEW simulator for every p."""
    return [OE.Simulator(durations, pool).simulate(p) for p in range(len(durations))]


def test_the_goldens_hold_the_reference_tests_and_one_trap_per_consequence():
    names = set(ids(CASES))
    assert REFERENCE_TESTS <= names
    assert all(not c["derived"] for c in CASES if c["name"] in REFERENCE_TESTS)
    assert sorted(int(n.split(":")[0].split()[1]) for n in names if n.startswith("trap ")) == list(range(1, 8))
    assert "TestCreateModel" in ids(MODELS)


@pytest.mark.parametrize("case", CASES, ids=ids(CASES))
def test_the_object_replays_the_call_sequence(case):
    s = OE.Simulator(case["tasks"], case["hosts"])
    for pos, want in case["calls"]:
        assert s.simulate(pos) == want, pos


@pytest.mark.parametrize("case", CASES, ids=ids(CASES))
def test_one_run_gives_every_fresh_answer(case):
    got = OE.fresh_estimates(case["tasks"], case["hosts"])
    assert got == fresh_by_object(case["tasks"], case["hosts"])
    if "fresh" in case:
        assert got == case["fresh"]


def test_a_golden_pins_the_difference_between_the_object_and_a_fresh_run():
    case = next(c for c in CASES if c["name"] == "TestMultipleHostsUnordered")
    assert case["calls"][2] == [2, 5 * 10 ** 9] and case["fresh"][2] == 6 * 10 ** 9
    differing = [c["name"] for c in CASES if c.get("fresh") and [e for _, e in c["calls"]] != [c["fresh"][p] for p, _ in c["calls"]]]
    assert len(differing) >= 5 and "TestMultipleHostsUnordered" in differing


@pytest.mark.parametrize("seed", range(8))
def test_prefix_property_on_random_pools_and_queues(seed):
    rng = np.random.default_rng(7100 + seed)
    for _ in range(40):
        m, n = int(rng.integers(0, 12)), int(rng.integers(0, 40))
        span = [10, 10 ** 9, 2 ** 62][int(rng.integers(0, 3))]
        pool = rng.integers(-span, span, m).tolist()
        durations = rng.integers(-span // 4, span, n).tolist()
        if rng.random() < 0.3:
            durations = [durations[0]] * n if n else []
        assert OE.fresh_estimates(durations, pool) == fresh_by_object(durations, pool)


def as_hosts(rows):
    return [types.SimpleNamespace(**r) for r in rows]


def as_running(docs):
    return {k: OE.LOOKUP_ERROR if v == "error" else None if v is None else types.SimpleNamespace(**v) for k, v in docs.items()}


@pytest.mark.parametrize("model", MODELS, ids=ids(MODELS))
def test_create_simulator_model(model):
    s = OE.create_simulator_model(model["queue"], as_hosts(model["hosts"]), as_running(model["running"]), model["now"])
    assert s.hosts == model["expect"] and s.tasks == model["queue"]


def test_get_estimated_start_time_positions():
    m = next(x for x in MODELS if x["name"] == "TestCreateModel")
    hosts, running = as_hosts(m["hosts"]), as_running(m["running"])
    args = (m["queue"], hosts, running, m["now"])
    assert OE.get_estimated_start_time("a", None, *args) == -1
    assert OE.get_estimated_start_time("zz", ["a", "b"], *args) == -1
    assert OE.get_estimated_start_time("a", ["a", "b"], *args) == 60 * 10 ** 9       # the soonest host: 1 min
    assert OE.get_estimated_start_time("b", ["a", "b"], *args) == 3 * 60 * 10 ** 9   # then the starting host: 3 min
