"""The cross-queue views without a GPU: the golden cases of queue_index.json through the stage-by-stage oracle and
through scheduler's host mirror (find_minimum_queue_position_for_task, find_duplicate_enqueued_tasks), the mirror equal
to the oracle on seeded random collections, and evg_queue_index_out's layout against its ctypes mirror."""
import ctypes
import os
import random
import subprocess

import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler

import golden_loader
import oracle_queue_index as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = golden_loader.load("queue_index.json")["cases"]


def queues_of(case):
    return [M.TaskQueue(distro=q["distro"], queue=[M.TaskQueueItem(id=i, is_dispatched=bool(disp)) for i, disp in q["items"]])
            for q in case["queues"]]


def as_sets(dups):
    """[(id, distros)] -> {id: frozenset(distros)}, the comparison TestFindDuplicateEnqueuedTasks makes."""
    out = {}
    for i, ds in dups:
        assert i not in out and len(set(ds)) == len(ds)
        out[i] = frozenset(ds)
    return out


def test_golden_file_covers_what_it_claims():
    names = {c["name"] for c in CASES}
    assert {"MatchesDuplicatesAcrossDifferentQueues", "DoesNotMatchDuplicatesWithinSameQueue", "DoesNotMatchEmptyQueues",
            "DoesNotMatchAllUnique"} <= names
    assert sum(not c["derived"] for c in CASES) == 4
    derived = [c for c in CASES if c["derived"]]
    assert derived and all("positions" in c and "resolver" in c for c in derived)
    assert any(v == -1 for c in derived for v in c["positions"].values())
    assert any("" in c["positions"] for c in derived)
    assert any(disp for c in derived for q in c["queues"] for _, disp in q["items"])


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_golden_through_the_oracle(name):
    case = next(c for c in CASES if c["name"] == name)
    docs = O.docs_of(queues_of(case))
    want = as_sets((d["task_id"], d["distros"]) for d in case["duplicates"])
    assert as_sets(O.duplicate_enqueued_tasks(docs).items()) == want
    for i, p in case.get("positions", {}).items():
        assert O.min_queue_position(docs, i) == p, i
        assert O.resolver_position(docs, i) == case["resolver"][i], i


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_golden_through_the_host_mirror(name):
    case = next(c for c in CASES if c["name"] == name)
    queues = queues_of(case)
    want = as_sets((d["task_id"], d["distros"]) for d in case["duplicates"])
    assert as_sets((r.task_id, r.distro_ids) for r in scheduler.find_duplicate_enqueued_tasks(queues)) == want
    for i, p in case.get("positions", {}).items():
        assert scheduler.find_minimum_queue_position_for_task(queues, i) == p, i


def random_collection(seed, n_queues=None, n_ids=None):
    """Queues drawn from a small id pool, so ids repeat within a queue and across queues; some queues empty, some
    items dispatched, ids that are prefixes of one another and ""."""
    rng = random.Random(seed)
    n_queues = n_queues or rng.randint(1, 12)
    n_ids = n_ids or rng.randint(1, 40)
    pool = [""] + [f"t{rng.randint(0, 3)}" * rng.randint(1, 3) + str(k) for k in range(n_ids)]
    queues = []
    for d in range(n_queues):
        n = 0 if rng.random() < 0.2 else rng.randint(1, 30)
        items = [M.TaskQueueItem(id=rng.choice(pool), is_dispatched=rng.random() < 0.2) for _ in range(n)]
        queues.append(M.TaskQueue(distro=f"distro-{d}", queue=items))
    return queues, pool + ["absent"]


@pytest.mark.parametrize("seed", range(40))
def test_mirror_equals_the_oracle_on_random_collections(seed):
    queues, ids = random_collection(seed)
    docs = O.docs_of(queues)
    for i in ids:
        assert scheduler.find_minimum_queue_position_for_task(queues, i) == O.min_queue_position(docs, i), i
    got = [(r.task_id, r.distro_ids) for r in scheduler.find_duplicate_enqueued_tasks(queues)]
    # the mirror's pinned order (first item, queues in collection order) is the order the oracle's $group meets them
    assert got == list(O.duplicate_enqueued_tasks(docs).items())


def test_random_collections_reach_every_case():
    seen = set()
    for seed in range(40):
        queues, _ = random_collection(seed)
        if any(not q.queue for q in queues):
            seen.add("empty queue")
        for q in queues:
            ids = [it.id for it in q.queue]
            if len(ids) != len(set(ids)):
                seen.add("repeat within a queue")
        if scheduler.find_duplicate_enqueued_tasks(queues):
            seen.add("duplicates")
    assert seen == {"empty queue", "repeat within a queue", "duplicates"}


def test_out_struct_layout_matches_the_ctypes_mirror(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(evg_queue_index_out), offsetof(evg_queue_index_out, min_position),
         offsetof(evg_queue_index_out, dup_item), offsetof(evg_queue_index_out, dup_off),
         offsetof(evg_queue_index_out, dup_queue), offsetof(evg_queue_index_out, n_dups));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    S = L.QueueIndexOutStruct
    assert got == [ctypes.sizeof(S), S.min_position.offset, S.dup_item.offset, S.dup_off.offset, S.dup_queue.offset,
                   S.n_dups.offset]
