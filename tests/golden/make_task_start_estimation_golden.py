"""Writes task_start_estimation.json: the task start-time estimator's tests as data.  Data only: the reference tests
(model/task_start_estimation_test.go) are transcribed, the derived cases are worked out by hand from
model/task_start_estimation.go:53-163; nothing here runs an implementation.

`cases`: a simulator set up with `hosts` (timeToCompletion of each host, as the test assigns them: NOT sorted) and
`tasks` (durations, queue order), then `calls`: [pos, expected return] of each simulate(pos) in order, ON THE SAME
OBJECT -- every call sorts the pool again and continues from the position and elapsed time the last one left.
`fresh` (where given): what a NEW simulator returns for simulate(p), per p -- one sort, then no other; this is what
GetEstimatedStartTime computes (:121) and it differs from `calls` once an insertion has left the pool unsorted.
`models`: createSimulatorModel at a frozen `now`: hosts in query order (status, running_task), `running`: task id ->
{expected_duration, dispatch_time}, null = no document, "error" = the lookup failed; `expect`: the pool built.
All values are int64 nanoseconds.  `derived`: false for a reference test transcribed whole."""
import json
import os

S = 10 ** 9
M = 60 * S
MAX, MIN = 2 ** 63 - 1, -(2 ** 63)
NOW = 1_700_000_000 * S
SRC = "model/task_start_estimation_test.go"


def calls(*expected):
    return [[p, e] for p, e in enumerate(expected)]


CASES = [
    {"name": "TestNoHosts", "source": SRC + ":66-71", "derived": False,
     "hosts": [], "tasks": [M, M], "calls": [[1, -1]], "fresh": [-1, -1]},
    {"name": "TestNoTasks", "source": SRC + ":73-78", "derived": False,
     "hosts": [0, 0], "tasks": [], "calls": [[0, -1]], "fresh": []},
    {"name": "TestManyFreeHosts", "source": SRC + ":80-87", "derived": False,
     "hosts": [0, 0], "tasks": [M, M], "calls": [[1, 0]], "fresh": [0, 0]},
    {"name": "TestSingleFreeHost", "source": SRC + ":89-102", "derived": False,
     "hosts": [0], "tasks": [M, 2 * M, 3 * M, 4 * M], "calls": calls(0, M, 3 * M, 6 * M), "fresh": [0, M, 3 * M, 6 * M]},
    {"name": "TestSingleOccupiedHost", "source": SRC + ":104-117", "derived": False,
     "hosts": [7 * M], "tasks": [M, 2 * M, 3 * M, 4 * M], "calls": calls(7 * M, 8 * M, 10 * M, 13 * M),
     "fresh": [7 * M, 8 * M, 10 * M, 13 * M]},
    {"name": "TestMultipleHosts", "source": SRC + ":119-132", "derived": False,
     # fresh: 1 s is below the first host left and is appended -> [5, 15, 1]; nothing sorts it again, so position 1
     # fast-forwards 5 s, not 1 s, and the pool goes [10, -4, 5], [-14, -5, 15]: elapsed 15 s, then back to 1 s
     "hosts": [5 * S, 0, 15 * S], "tasks": [S, 5 * S, 15 * S, 30 * S], "calls": calls(0, S, 5 * S, 6 * S),
     "fresh": [0, 5 * S, 15 * S, S]},
    {"name": "TestMultipleHostsUnordered", "source": SRC + ":134-147", "derived": False,
     # the pool is [1 s, 0 s, 10 s] after position 1; the object sorts it for simulate(2) (fast-forward 0: 5 s), a fresh
     # run does not (fast-forward 1 s: 6 s, then -1 s: 5 s)
     "hosts": [5 * S, 0, 15 * S], "tasks": [5 * S, S, 30 * S, 15 * S], "calls": calls(0, 5 * S, 5 * S, 6 * S),
     "fresh": [0, 5 * S, 6 * S, 5 * S]},
    {"name": "TestRunningHosts", "source": SRC + ":149-162", "derived": False,
     "hosts": [25 * S, 10 * S, 15 * S], "tasks": [30 * S, 15 * S, 10 * S, 5 * S], "calls": calls(10 * S, 15 * S, 25 * S, 30 * S),
     "fresh": [10 * S, 15 * S, 30 * S, 40 * S]},
    {"name": "TestEvenDistribution", "source": SRC + ":164-179", "derived": False,
     "hosts": [10 * S] * 5, "tasks": [10 * S] * 14, "calls": calls(*[(i // 5 + 1) * 10 * S for i in range(14)])},
    {"name": "trap 1: a duration below the first host left is appended, so the first element is not the minimum", "source": ":84-95",
     "derived": True,
     # 5 s against [10, 20]: no pair matches, appended -> [10, 20, 5].  Fresh: fast-forward 10 s, [10, -5, 5], then 10 s
     # again.  The object sorts to [5, 10, 20] and fast-forwards 5 s twice.
     "hosts": [0, 10 * S, 20 * S], "tasks": [5 * S, 5 * S, 5 * S], "calls": calls(0, 5 * S, 10 * S), "fresh": [0, 10 * S, 20 * S]},
    {"name": "trap 2: the value is inserted in FRONT of hosts[i], an element that may be smaller", "source": ":86-88",
     "derived": True,
     # 5 s against [2, 8, 9]: pair 0 matches, inserted at 0 -> [5, 2, 8, 9].  Fresh fast-forwards 5 s; the sorted
     # object 2 s.
     "hosts": [0, 2 * S, 8 * S, 9 * S], "tasks": [5 * S, S], "calls": calls(0, 2 * S), "fresh": [0, 5 * S]},
    {"name": "trap 3: with one or two hosts the pair test never runs and the value is always appended", "source": ":84-85, :92",
     "derived": True,
     # sorted [1, 3]: 10 s appended -> [2, 10]; 0 s appended -> [8, 0]; fresh fast-forwards 8 s, the object sorts and
     # fast-forwards 0
     "hosts": [3 * S, S], "tasks": [10 * S, 0, 2 * S], "calls": calls(S, 3 * S, 3 * S), "fresh": [S, 3 * S, 11 * S]},
    {"name": "trap 4: the scan reaches the last pair of the hosts left (i = count - 3); i = count - 2 appends", "source": ":84-92",
     "derived": True,
     # 25 s against [10, 20, 30]: pair 1 (20, 30) is the last one and matches -> [10, 25, 20, 30].  Fresh: [15, 10, 20]
     # takes 15 s at 1 -> [15, 15, 10, 20]; fast-forward 15 s.  The object: sorted [10, 15, 20] takes 15 s at 0, then
     # [10, 15, 15, 20] fast-forwards 10 s.
     "hosts": [0, 10 * S, 20 * S, 30 * S], "tasks": [25 * S, 15 * S, 0], "calls": calls(0, 10 * S, 20 * S), "fresh": [0, 10 * S, 25 * S]},
    {"name": "trap 5: an overrun host has a negative timeToCompletion and the elapsed time goes down", "source": ":72-73, :157",
     "derived": True,
     "hosts": [-5 * S, 3 * S], "tasks": [S, S], "calls": calls(-5 * S, -4 * S), "fresh": [-5 * S, 3 * S]},
    {"name": "trap 6: -1 is a value a run can reach, not only 'no estimate'", "source": ":54-59, :66", "derived": True,
     "hosts": [-1], "tasks": [7, 7], "calls": calls(-1, 6), "fresh": [-1, 6]},
    {"name": "trap 7: the elapsed time wraps as int64", "source": ":73, :76", "derived": True,
     # [MAX, MAX]: elapsed MAX, pool [0, MAX]; fast-forward 0, pool [MAX, 1]; fresh adds MAX again: -2.  The object
     # sorts to [1, MAX] and adds 1: MIN.
     "hosts": [MAX, MAX], "tasks": [MAX, 1, 1], "calls": calls(MAX, MAX, MIN), "fresh": [MAX, MAX, -2]},
]


def host(status, running_task=""):
    return {"status": status, "running_task": running_task}


MODELS = [
    {"name": "TestCreateModel", "source": SRC + ":32-64", "derived": False, "now": NOW,
     # the test reads the clock and allows 100 ms; at a frozen clock the values are exact
     "hosts": [host("running", "t1"), host("running", "t2"), host("starting")],
     "running": {"t1": {"expected_duration": 5 * M, "dispatch_time": NOW - 4 * M},
                 "t2": {"expected_duration": 30 * M, "dispatch_time": NOW - 10 * M}},
     "queue": [60 * M, M], "expect": [M, 20 * M, 3 * M]},
    {"name": "every status, an overrun task, a task without a document, then a failed lookup", "source": ":129-159", "derived": True,
     "now": NOW,
     # "building" is up (UpHostStatus) but no case of the switch; the host running "gone" is skipped (:148-154); the
     # lookup of "err" fails and the pool built so far is returned: the free host behind it is never reached (:142-147)
     "hosts": [host("initializing"), host("starting"), host("provisioning"), host("running"), host("running", "t1"),
               host("running", "gone"), host("building"), host("running", "late"), host("running", "err"), host("running")],
     "running": {"t1": {"expected_duration": 5 * M, "dispatch_time": NOW - 4 * M},
                 "late": {"expected_duration": M, "dispatch_time": NOW - 10 * M}, "gone": None, "err": "error"},
     "queue": [M], "expect": [4 * M, 3 * M, M, 0, M, -9 * M]},
    {"name": "a running task that was never dispatched: time.Since of the zero time saturates", "source": ":156-157", "derived": True,
     "now": NOW,
     "hosts": [host("running", "t0")], "running": {"t0": {"expected_duration": 10 * M, "dispatch_time": MIN}},
     "queue": [M], "expect": [10 * M - MAX]},
]

if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "task_start_estimation.json")
    with open(out, "w") as f:
        json.dump({"cases": CASES, "models": MODELS}, f, indent=1)
        f.write("\n")
