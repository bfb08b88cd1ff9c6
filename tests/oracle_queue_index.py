"""The two aggregations over the task_queues collection, restated stage by stage over plain documents -- the test
oracle of evg_queue_index_batch and of scheduler's host mirror, and independent of both.

A document is {"distro": str, "queue": [{"_id": str, "is_dispatched": bool}, ...]}, a TaskQueue as it is saved.

* min_queue_position: FindMinimumQueuePositionForTask (model/task_queue.go:407-435): $match on queue._id, $unwind
  with includeArrayIndex, $match again, $sort by index, $limit 1; index + 1, or -1 without a result.
* duplicate_enqueued_tasks: FindDuplicateEnqueuedTasks (:505-547): $unwind queue, $group by queue._id with $addToSet of
  distro and a $sum count, $project the set's $size, $match count > 1 and size > 1.
"""
from typing import Dict, List, Sequence


def docs_of(queues) -> List[dict]:
    """model.TaskQueue objects as saved documents."""
    return [{"distro": q.distro, "queue": [{"_id": it.id, "is_dispatched": it.is_dispatched} for it in q.queue]} for q in queues]


def _unwind(docs, index_field=None):
    for doc in docs:
        for k, item in enumerate(doc["queue"]):  # $unwind drops a document whose array is empty
            out = dict(doc, queue=item)
            if index_field:
                out[index_field] = k
            yield out


def min_queue_position(docs: Sequence[dict], task_id: str) -> int:
    matched = [d for d in docs if any(it["_id"] == task_id for it in d["queue"])]   # $match {queue._id: id}
    unwound = list(_unwind(matched, "index"))                                        # $unwind, includeArrayIndex
    unwound = [d for d in unwound if d["queue"]["_id"] == task_id]                   # $match {queue._id: id}
    unwound.sort(key=lambda d: d["index"])                                           # $sort {index: 1}
    results = unwound[:1]                                                            # $limit 1
    return results[0]["index"] + 1 if results else -1


def resolver_position(docs: Sequence[dict], task_id: str) -> int:
    """GraphQL's minQueuePosition (graphql/task_resolver.go:570-581): a negative result is shown as 0."""
    p = min_queue_position(docs, task_id)
    return 0 if p < 0 else p


def duplicate_enqueued_tasks(docs: Sequence[dict]) -> Dict[str, List[str]]:
    """{task id: its distros} -- a dict, the ids in the order $group first met them (the aggregation promises no order,
    and neither does $addToSet; callers compare them as sets unless they pin an order themselves)."""
    groups: Dict[str, dict] = {}
    for d in _unwind(docs):                                                          # $unwind queue
        g = groups.setdefault(d["queue"]["_id"], {"distros": [], "count": 0})         # $group {_id: queue._id}
        if d["distro"] not in g["distros"]:                                           #   distros: $addToSet distro
            g["distros"].append(d["distro"])
        g["count"] += 1                                                               #   count: $sum 1
    projected = {k: dict(g, num_unique_distros=len(g["distros"])) for k, g in groups.items()}   # $project $size
    return {k: g["distros"] for k, g in projected.items() if g["count"] > 1 and g["num_unique_distros"] > 1}  # $match
