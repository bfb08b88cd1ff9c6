"""evg_queue_index_batch: FindMinimumQueuePositionForTask and FindDuplicateEnqueuedTasks for every id of the saved
queues at once, compared output for output with the stage-by-stage oracle (tests/oracle_queue_index.py): the golden
cases, seeded random collections (also with EVG_INTERN_HASH_BITS making every id collide), the persisted queues of
resident ticks with aliased tasks, the errors, and the launch count."""
import copy
import ctypes as C
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_entry_guard import launched_kernels
from test_host_logic import random_tasks
from test_queue_index_host import CASES, as_sets, queues_of

import oracle_queue_index as O

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000 * 10 ** 9


@pytest.fixture(scope="module")
def eng():
    e = scheduler.Engine(0)
    yield e
    e.close()


def flatten(docs):
    ids = [it["_id"] for d in docs for it in d["queue"]]
    item_off = np.concatenate([[0], np.cumsum([len(d["queue"]) for d in docs])]).astype(np.int64)
    return ids, item_off


def expected(docs):
    """What evg_queue_index_batch must return for these documents, from the oracle: every item's position, and the
    duplicated ids in the order of their first item with their queues ascending (distinct distros per document)."""
    ids, _ = flatten(docs)
    pos = {i: O.min_queue_position(docs, i) for i in dict.fromkeys(ids)}
    queue_of = {d["distro"]: q for q, d in enumerate(docs)}
    dups = O.duplicate_enqueued_tasks(docs)
    first = {}
    for k, i in enumerate(ids):
        first.setdefault(i, k)
    order = sorted(dups, key=lambda i: first[i])
    qs = [sorted(queue_of[d] for d in dups[i]) for i in order]
    return dict(min_position=np.array([pos[i] for i in ids], np.int32), dup_item=np.array([first[i] for i in order], np.int64),
                dup_off=np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int64),
                dup_queue=np.array([q for x in qs for q in x], np.int32))


def check(eng, docs):
    ids, item_off = flatten(docs)
    got = eng.queue_index(ids, item_off)
    want = expected(docs)
    for k in want:
        assert np.array_equal(got[k], want[k]), (k, got[k][:20], want[k][:20])
    return got


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_golden_cases(eng, name):
    case = next(c for c in CASES if c["name"] == name)
    docs = O.docs_of(queues_of(case))
    got = check(eng, docs)
    ids, _ = flatten(docs)
    off = got["dup_off"]
    dups = [(ids[int(i)], [docs[int(q)]["distro"] for q in got["dup_queue"][off[k]:off[k + 1]]]) for k, i in enumerate(got["dup_item"])]
    assert as_sets(dups) == as_sets((d["task_id"], d["distros"]) for d in case["duplicates"])
    pos = dict(zip(ids, got["min_position"].tolist()))
    for i, p in case.get("positions", {}).items():
        assert pos.get(i, -1) == p, i  # an id no queue holds has no item: -1


def random_docs(seed, n_queues, mean_len, n_ids):
    """Queues over a pool of n_ids ids (many duplicates, repeats within a queue), a fifth of them empty; ids of ~60
    bytes that differ in their last bytes or only in length, and ""."""
    rng = random.Random(seed)
    pool = [""] + [f"evergreen_ubuntu2204_compile_patch_{rng.randrange(10 ** 6):06x}_{k}" + "x" * rng.randrange(3)
                   for k in range(n_ids)]
    docs = []
    for d in range(n_queues):
        n = 0 if rng.random() < 0.2 else rng.randint(1, 2 * mean_len)
        docs.append({"distro": f"distro-{d}", "queue": [{"_id": rng.choice(pool), "is_dispatched": rng.random() < 0.1} for _ in range(n)]})
    return docs


SHAPES = [(1, 50, 20), (7, 30, 60), (40, 60, 900), (300, 8, 1500), (3, 700, 3000)]


@pytest.mark.parametrize("seed", range(len(SHAPES)))
def test_random_collections_equal_the_oracle(eng, seed):
    got = check(eng, random_docs(900 + seed, *SHAPES[seed]))
    assert seed == 0 or got["dup_item"].shape[0] > 0


@pytest.mark.parametrize("bits", ["0", "1", "4"])
def test_every_id_colliding(eng, monkeypatch, bits):
    monkeypatch.setenv("EVG_INTERN_HASH_BITS", bits)
    for seed, shape in enumerate([(7, 30, 60), (40, 20, 300)]):
        check(eng, random_docs(950 + seed, *shape))
    check(eng, O.docs_of(queues_of(next(c for c in CASES if c["name"] == "IdsDifferingInTheLastByteOrInLength"))))


def test_no_items(eng):
    for docs in ([], [{"distro": "d", "queue": []}] * 3):
        got = check(eng, docs)
        assert got["dup_off"].tolist() == [0]


# ---------------------------------------------------------------- resident ticks
def aliased_batch(seed, n_distros=6, n=300):
    """Go-level batch: each distro's own tasks, and about a tenth of all tasks also filed under 1-3 other distros, the
    same Task, as FindHostSchedulable files a task under every distro that aliases its DistroId."""
    rng = random.Random(seed)
    own, db = [], {}
    for d in range(n_distros):
        tasks, ext = random_tasks(rng, n)
        for t in tasks:
            t.id = f"d{d}-{t.id}"
            for dep in t.depends_on:
                if dep.task_id.startswith("t"):
                    dep.task_id = f"d{d}-{dep.task_id}"
        own.append(tasks)
        db.update(ext)
    lists = [list(ts) for ts in own]
    for d, ts in enumerate(own):
        for t in ts:
            if rng.random() < 0.1:
                for e in rng.sample([x for x in range(n_distros) if x != d], rng.randint(1, 3)):
                    lists[e].append(t)
    return [(M.Distro(id=f"distro{d}"), ts) for d, ts in enumerate(lists)], db


def test_resident_tick_with_aliased_tasks(eng):
    batch, db = aliased_batch(31)
    saved = copy.deepcopy((batch, db))  # persist_task_queues stamps its tasks, and so does plan()
    rt = scheduler.ResidentTick(eng, dependency_db=db)
    rt.plan(batch, NOW)
    # the persisted rows, their ids read from tasks[item.task]
    task_off = rt.table.task_off
    item_off, items = eng.download_queue(0, task_off)
    item_off, items = item_off.copy(), items.copy()
    ids = [rt.ids[d][int(items[k]["task"])] for d in range(len(batch)) for k in range(int(item_off[d]), int(item_off[d + 1]))]
    eng.run(NOW)
    before = [x.copy() for x in eng.download_queue(0, task_off)]
    got = eng.queue_index(ids, item_off)
    # the oracle over what persist_task_queues saves for the same batch
    queues = scheduler.persist_task_queues(saved[0], NOW, dependency_db=saved[1])
    docs = O.docs_of(queues)
    assert [it["_id"] for d in docs for it in d["queue"]] == ids
    want = expected(docs)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    assert want["dup_item"].shape[0] > 20
    # the tick is as it was: the queue downloads again unchanged, and a run gives what it gave before
    assert all(np.array_equal(a, b) for a, b in zip(eng.download_queue(0, task_off), before))
    eng.run(NOW)
    assert all(np.array_equal(a, b) for a, b in zip(eng.download_queue(0, task_off), before))
    # ResidentTick.queue_index keys both views by task id
    positions, dups = rt.queue_index()
    assert positions == {i: O.min_queue_position(docs, i) for i in ids}
    assert dups == O.duplicate_enqueued_tasks(docs)


def test_alias_queues_from_synth(eng):
    """An evg_plan_aliases tick (synth.make_aliases): each alias queue's persisted rows named by their source row."""
    w = synth.make(np.array([400, 30, 0, 900, 120]), 1601, tg_frac=0.1)
    at, cfg = synth.make_aliases(w, 1602, name_frac=0.6)
    task_off, _, _ = eng.plan_aliases(at, cfg, w.now)
    task_off = task_off.copy()
    eng.run(w.now)
    item_off, items = (x.copy() for x in eng.download_queue(0, task_off))
    src, _ = eng.download_alias_map()
    ids = [f"task-{int(src[int(task_off[d]) + int(items[k]['task'])])}" for d in range(task_off.shape[0] - 1)
           for k in range(int(item_off[d]), int(item_off[d + 1]))]
    docs = [{"distro": f"alias-{d}", "queue": [{"_id": i, "is_dispatched": False} for i in ids[int(item_off[d]):int(item_off[d + 1])]]}
            for d in range(task_off.shape[0] - 1)]
    got = check(eng, docs)
    assert got["dup_item"].shape[0] > 10


# ---------------------------------------------------------------- errors and launches
def raw(eng, data, off, item_off, n_queues):
    N = max(int(item_off[-1]) if item_off.shape[0] else 0, 1)
    bufs = [np.empty(N, np.int32), np.empty(N, np.int64), np.zeros(N + 1, np.int64), np.empty(N, np.int32)]
    st = L.QueueIndexOutStruct(*[L.ptr(b) for b in bufs], 0)
    col = L.StrColStruct(L.ptr(data), L.ptr(off))
    rc = eng.lib.evg_queue_index_batch(eng.ctx, C.byref(col), L.ptr(item_off), n_queues, C.byref(st))
    return rc, L.last_error() if rc else ""


def test_errors_leave_the_context_usable(eng):
    docs = random_docs(970, 7, 30, 60)
    ids, item_off = flatten(docs)
    data, off = S.pack_strings(ids)
    bad_item_off = item_off.copy()
    k = int(np.nonzero(np.diff(item_off))[0][0]) + 1
    bad_item_off[k] = bad_item_off[k + 1] + 1
    bad_off = off.copy()
    bad_off[5] = off[-1] + 1  # a string past its byte column; the last offset stays
    for args, name in [((data, off, bad_item_off, len(docs)), "item_off"), ((data, bad_off, item_off, len(docs)), "ids.off"),
                       ((data, off, item_off, -1), "negative sizes")]:
        rc, msg = raw(eng, *args)
        assert rc == L.EVG_ERR_INVALID and msg.startswith("evg_queue_index_batch") and name in msg, (name, msg)
        check(eng, docs)


def test_launch_count_matches_the_profiler():
    """torch.profiler can miss the first kernels of a window (as in test_gpu_onchip_sort.profiled): a torch kernel opens
    each window, and a list that differs from the context's count is taken again, a few times.  The call is pure, so
    every try launches the same kernels, and a count that is wrong fails every try."""
    import torch
    docs = random_docs(980, 40, 60, 900)
    ids, item_off = flatten(docs)
    packed = S.pack_strings(ids)
    eng = scheduler.Engine(0)  # a context of its own, as test_entry_guard gives every case
    try:
        def call():
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
            eng.queue_index(packed, item_off)

        for _ in range(6):
            names = launched_kernels(call)
            if eng.last_launch_count() == len(names):
                break
        assert names and eng.last_launch_count() == len(names), names
        assert names[0].startswith("k_qx_keys") and any(n.startswith("k_al_scatter") for n in names)
    finally:
        eng.close()
