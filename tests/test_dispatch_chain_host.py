"""The DAG dispatcher chained onto the resident tick, without a GPU: the layout of evg_dispatch_out, and the host
restatement soa.persisted_dag_input on oracle-planned ticks against the document route (TaskQueueItems of the persisted
queue marshalled as rebuild_dag_dispatchers does), then oracle_dag.rebuild on both."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from oracle import oracle as O
from oracle import oracle_dag as OD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOW = 1_700_000_000_000_000_000


def test_struct_layout(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(evg_dispatch_out), offsetof(evg_dispatch_out, item_off),
         offsetof(evg_dispatch_out, sorted), offsetof(evg_dispatch_out, n_sorted), offsetof(evg_dispatch_out, n_cycles),
         offsetof(evg_dispatch_out, group_off), offsetof(evg_dispatch_out, group_slot), offsetof(evg_dispatch_out, unit_items),
         offsetof(evg_dispatch_out, unit_off));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    out = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    S_ = L.DispatchOutStruct
    assert out == [ctypes.sizeof(S_)] + [getattr(S_, f).offset for f in L.DISPATCH_OUT_FIELDS]


def random_batch(rnd, sizes):
    """Distros of random tasks: task groups (some spread over versions), dependencies inside the queue in both
    directions (cycles), duplicates, self-edges, dependencies on other distros' tasks and on tasks that exist nowhere."""
    batch = []
    for d, n in enumerate(sizes):
        tasks = []
        for k in range(n):
            grp = rnd.random() < 0.35
            tasks.append(M.Task(id=f"d{d}t{k}", version=f"v{rnd.randrange(3)}", project="p", build_variant=f"bv{rnd.randrange(2)}",
                                task_group=f"g{rnd.randrange(5)}" if grp else "", task_group_order=rnd.randrange(-2, 9),
                                priority=rnd.randrange(0, 60), num_dependents=rnd.randrange(0, 4), distro_id=f"d{d}"))
        for k, t in enumerate(tasks):
            for _ in range(rnd.choice([0, 0, 0, 1, 2, 3])):
                t.depends_on.append(M.Dependency(f"d{d}t{rnd.randrange(n)}"))
            if rnd.random() < 0.05:
                t.depends_on.append(M.Dependency(f"d{d}t{k}"))  # a self-edge
            if rnd.random() < 0.05:
                t.depends_on.append(M.Dependency(f"d{(d + 1) % len(sizes)}t0"))  # another distro's queue
            if rnd.random() < 0.05:
                t.depends_on.append(M.Dependency("nowhere"))
            if t.depends_on and rnd.random() < 0.1:
                t.depends_on.append(t.depends_on[0])  # a parallel line
        # GroupMaxHosts is a per-group setting: members agree
        for t in tasks:
            t.task_group_max_hosts = 2 if t.task_group else 0
        batch.append((M.Distro(id=f"d{d}"), tasks))
    return batch


def oracle_order(batch):
    """Per distro the oracle planner's rank order (distro-local task per rank), concatenated."""
    return np.concatenate([O.plan(d, ts, NOW)[0] for d, ts in batch] or [np.zeros(0)]).astype(np.int32)


def persisted_queues(batch, order, toff, cap):
    out = []
    for d, (distro, ts) in enumerate(batch):
        a = int(toff[d])
        n = min(len(ts), cap or L.EVG_PERSISTED_QUEUE_CAP)
        q = []
        for r in range(n):
            t = ts[int(order[a + r])]
            q.append(M.TaskQueueItem(id=t.id, group=t.task_group, build_variant=t.build_variant, project=t.project,
                                     version=t.version, group_index=t.task_group_order,
                                     dependencies=[x.task_id for x in t.depends_on]))
        out.append(M.TaskQueue(distro=distro.id, queue=q))
    return out


def oracle_items(ids, lo, hi, dep_off, dep_item, group_id, group_index, names):
    """oracle_dag's item dicts for items [lo, hi) of a marshalled DAG input; -1 dependencies name no item."""
    items = []
    for j in range(lo, hi):
        g = int(group_id[j])
        items.append({"id": ids[j - lo], "group": names[g] if g >= 0 else "", "group_index": int(group_index[j]),
                      "dependencies": [ids[int(x)] if x >= 0 else "absent" for x in dep_item[dep_off[j]:dep_off[j + 1]]]})
    return items


@pytest.mark.parametrize("cap", [0, 1, 3, 7, 25, 60, 100_000])
@pytest.mark.parametrize("seed", [1, 2])
def test_restatement_matches_the_document_route(seed, cap):
    rnd = random.Random(seed * 100 + cap)
    batch = random_batch(rnd, [0, 1, 2, 9, 50, 140])
    soa, table, keys = S.marshal_tasks(batch, NOW, resolve_deps=True)
    order = oracle_order(batch)
    io, go, dep_off, dep_item, group_id, group_index, group_slot = S.persisted_dag_input(soa, table, order, cap)
    queues = persisted_queues(batch, order, table.task_off, cap)
    dio, dgo, ddep_off, ddep_item, dgroup_id, dgroup_index, dnames = S.dag_input_from_queues(queues)
    assert io.tolist() == dio.tolist() and go.tolist() == dgo.tolist()
    assert group_id.tolist() == dgroup_id.tolist() and group_index.tolist() == dgroup_index.tolist()
    for d in range(table.n_distros):
        assert [keys[d].group_names[int(s)] for s in group_slot[go[d]:go[d + 1]]] == dnames[d]
    truncated = False
    for j in range(int(io[-1])):
        mine = [int(x) for x in dep_item[dep_off[j]:dep_off[j + 1]] if x >= 0]
        theirs = [int(x) for x in ddep_item[ddep_off[j]:ddep_off[j + 1]] if x >= 0]
        assert mine == theirs, j  # the in-queue edges, in DependsOn order, duplicates kept
        truncated |= any(x < 0 for x in dep_item[dep_off[j]:dep_off[j + 1]])
    if cap in (1, 3, 7):
        assert truncated  # some dependency ranks past the cap
    for d, q in enumerate(queues):
        ids = [it.id for it in q.queue]
        a, b = int(io[d]), int(io[d + 1])
        want = OD.rebuild([{"id": it.id, "group": it.group, "build_variant": it.build_variant, "project": it.project,
                            "version": it.version, "group_index": it.group_index, "dependencies": it.dependencies} for it in q.queue])
        names = [keys[d].group_names[int(s)] for s in group_slot[go[d]:go[d + 1]]]
        got = OD.rebuild(oracle_items(ids, a, b, dep_off, dep_item, group_id, group_index, names))
        # the items carry the whole composite name as their group: oracle_dag appends three empty fields to it
        assert got[:2] == want[:2] and {k[:-3]: v for k, v in got[2].items()} == want[2]


def test_groups_only_past_the_cap_are_not_numbered():
    """A task group whose members all rank past the cap has no dense id; the others are numbered by first appearance."""
    ts = [M.Task(id=f"t{k}", task_group=("late" if k >= 4 else f"g{k % 2}"), task_group_max_hosts=1, version="v", priority=100 - k)
          for k in range(8)]
    batch = [(M.Distro(id="d"), ts)]
    soa, table, keys = S.marshal_tasks(batch, NOW, resolve_deps=True)
    order = np.arange(8, dtype=np.int32)
    io, go, _, _, group_id, _, group_slot = S.persisted_dag_input(soa, table, order, 4)
    assert io.tolist() == [0, 4] and go.tolist() == [0, 2]
    assert group_id.tolist() == [0, 1, 0, 1]
    assert [keys[0].group_names[int(s)] for s in group_slot] == ["g0___v", "g1___v"]  # Group_BuildVariant_Project_Version
