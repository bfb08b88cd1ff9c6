"""Writes queue_index.json: saved task queues with what FindMinimumQueuePositionForTask and FindDuplicateEnqueuedTasks
(model/task_queue.go:407-435, 505-547) return for them.  Data only: expected values are written by hand from the
reference's code and tests; nothing here runs an implementation.

Case layout: "queues": [{"distro", "items": [[id, is_dispatched], ...]}] in collection order; "duplicates": [{"task_id",
"distros"}] -- compared as sets of ids, each with its distros as a set, the way TestFindDuplicateEnqueuedTasks compares
them (assert.Subset both ways); "positions": {id: FindMinimumQueuePositionForTask}, -1 for an id no queue holds;
"resolver": {id: the GraphQL minQueuePosition field}, where a negative position is shown as 0
(graphql/task_resolver.go:570-581).  `derived`: false for a case of TestFindDuplicateEnqueuedTasks transcribed whole
(model/task_queue_test.go:223-280, whose queues hold items with Id set and every other field zero), true for a case
written here for minQueuePosition, which the reference's tests do not reach."""
import json
import os

SOURCE = "model/task_queue_test.go:223-280"


def q(distro, *ids, dispatched=()):
    return {"distro": distro, "items": [[i, k in dispatched] for k, i in enumerate(ids)]}


def resolver(positions):
    return {k: max(v, 0) for k, v in positions.items()}


CASES = [
    {"name": "MatchesDuplicatesAcrossDifferentQueues", "source": SOURCE, "derived": False,
     "queues": [q("d1", "task1", "task2", "task3"), q("d2", "task1", "task3", "task4", "task5", "task6"), q("d3", "task3")],
     "duplicates": [{"task_id": "task1", "distros": ["d1", "d2"]}, {"task_id": "task3", "distros": ["d1", "d2", "d3"]}]},
    {"name": "DoesNotMatchDuplicatesWithinSameQueue", "source": SOURCE, "derived": False,
     "queues": [q("d1", "task1", "task1", "task2")], "duplicates": []},
    {"name": "DoesNotMatchEmptyQueues", "source": SOURCE, "derived": False, "queues": [q("d1")], "duplicates": []},
    {"name": "DoesNotMatchAllUnique", "source": SOURCE, "derived": False,
     "queues": [q("d1", "task1", "task2"), q("d2", "task3", "task4")], "duplicates": []},
    # ---- derived: minQueuePosition
    {"name": "PositionsAcrossQueuesAndAnAbsentId", "source": "model/task_queue.go:407-435", "derived": True,
     # task3 sits at index 2, 1 and 0: the smallest wins; task7 is in no queue
     "queues": [q("d1", "task1", "task2", "task3"), q("d2", "task1", "task3", "task4", "task5", "task6"), q("d3", "task3")],
     "positions": {"task1": 1, "task2": 2, "task3": 1, "task4": 3, "task5": 4, "task6": 5, "task7": -1},
     "duplicates": [{"task_id": "task1", "distros": ["d1", "d2"]}, {"task_id": "task3", "distros": ["d1", "d2", "d3"]}]},
    {"name": "RepeatedIdInOneQueueCountsAtItsFirstIndex", "source": "model/task_queue.go:407-435, 505-547", "derived": True,
     # a twice in d1 only: no duplicate; b twice in d1 and once in d2: a duplicate of {d1, d2}
     "queues": [q("d1", "x", "a", "b", "a", "b"), q("d2", "y", "z", "w", "b")],
     "positions": {"a": 2, "b": 3, "x": 1, "y": 1, "z": 2, "w": 3},
     "duplicates": [{"task_id": "b", "distros": ["d1", "d2"]}]},
    {"name": "DispatchedItemsStillCount", "source": "model/task_queue.go:414-425", "derived": True,
     # the pipeline has no IsDispatched filter: t1, dispatched at index 0 of d1, is at position 1
     "queues": [q("d1", "t1", "t2", dispatched=(0,)), q("d2", "t2", "t3", "t1", dispatched=(0, 2))],
     "positions": {"t1": 1, "t2": 1, "t3": 2},
     "duplicates": [{"task_id": "t1", "distros": ["d1", "d2"]}, {"task_id": "t2", "distros": ["d1", "d2"]}]},
    {"name": "EmptyStringIsAnOrdinaryId", "source": "model/task_queue.go:407-435, 505-547", "derived": True,
     "queues": [q("d1"), q("d2", "a", ""), q("d3"), q("d4", "", "b")],
     "positions": {"": 1, "a": 1, "b": 2, "c": -1},
     "duplicates": [{"task_id": "", "distros": ["d2", "d4"]}]},
    {"name": "IdsDifferingInTheLastByteOrInLength", "source": "model/task_queue.go:407-435, 505-547", "derived": True,
     "queues": [q("d1", "abc", "abcd", "abd"), q("d2", "ab", "abd", "abc", "abce")],
     "positions": {"abc": 1, "abcd": 2, "abd": 2, "ab": 1, "abce": 4, "abcde": -1, "a": -1},
     "duplicates": [{"task_id": "abc", "distros": ["d1", "d2"]}, {"task_id": "abd", "distros": ["d1", "d2"]}]},
]
for c in CASES:
    if "positions" in c:
        c["resolver"] = resolver(c["positions"])

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "queue_index.json")
    with open(path, "w") as f:
        json.dump({"cases": CASES}, f, indent=1)
        f.write("\n")
