"""The device sorts outside the planner, each against a plain sort of the same keys: the alias queues' radix sort at
every pass count, and the three segmented merge sorts (legacy prioritiser, DAG task-group buckets, start-estimate host
pools) at every run length.

Alias queues (evg_plan_aliases step 3).  Every (queue e, source row t) pair is the key e << 32 | t, written in
source-row order.  A stable LSD radix sort by the queue bits alone then lists every queue in ascending source row:
  bits   = the smallest b with 2^b >= D, capped at 31
  passes = ceil(bits / 8): 8-bit digits at shifts 32, 40, 48, 56; D = 1 runs no pass
  a pass = one k_al_hist, one scan_counts and one k_al_scatter over ceil(P / 2048) tiles of 2048 keys
So D = 2 .. 256 sorts in one pass, 257 .. 65 536 in two, 65 537 .. 2^24 in three.  Every case counts k_al_hist and
k_al_scatter in torch.profiler's kernel list.  The tables are crafted so that every row passes
FindHostSchedulableForAlias: the pairs are then exactly what secondary_idx and dest_idx name.  The reference is a
numpy dedupe of each row's destinations and np.lexsort((row, queue)).  The cases place queue ids where a dropped pass
or a wrong shift shows: ids that share their low byte, or their low two bytes, and differ above; every pair in queue
D - 1; rows in descending queue order, so every key moves; one name that fans a row out to hundreds of queues; a row
that names one distro twice, directly and through an alias; 90 % of the pairs in one queue; and tiles in which every
digit but one is empty.  The first-appearance group and version numbering per queue is checked against numpy too,
once at more than 1 048 576 pairs, where scan_counts' block sums take k_scan_sums' carry loop.
The fourth pass (shift 56) is not reached.  It needs D > 2^24, i.e. 16.8 M distro cfg rows and about 1.5 GB of host
cfg.  It is the same kernel at a higher shift, and passes two and three already show that the shift advances.

The segmented merge sorts (k_seg_merge_pass<LegacyOrder / DagGroupOrder / EsValueOrder>) are one kernel template with
three orders.  Runs of length L = 1, 2, 4, ... below the longest segment are merged pairwise, each element placed by
one binary search in its sibling run: a left run counts the sibling's elements that sort strictly before it, a right
run those that do not sort after it.  Edge branches: L >= n copies the segment, a run with no sibling (s0 >= n) is
copied, and s1 = min(s0 + L, n) shortens the last sibling.  The pass count comes from the longest segment, so one
shape set (the segments of SHAPE, with the longest one first, then last, and a call of many empty segments between
tiny ones) runs through all three:
  legacy      a numpy lexsort of the comparator chain per list, then mergeTasks' interleave (oracle_legacy)
  DAG groups  oracle_dag.rebuild
  estimates   the numpy restatement of test_gpu_start_estimate (fresh / expect)
"""
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle_dag as OD
from oracle import oracle_legacy as OL
from test_entry_guard import launched_kernels
from test_gpu_alias import plan_and_check
from test_gpu_legacy import _tq, mk_copy, random_queue
from test_gpu_start_estimate import expect, pools_of

I64_MIN, I64_MAX = -(2 ** 63), 2 ** 63 - 1
I32_MIN, I32_MAX = -(2 ** 31), 2 ** 31 - 1
NOW = synth.NOW_NS


@pytest.fixture(scope="module")
def fresh():
    """A second context: the host route of the alias queues is uploaded here."""
    eng = scheduler.Engine(0)
    yield eng
    eng.close()


# ================================================================ A. the alias queues' radix sort
def alias_passes(D):
    bits = 0
    while bits < 31 and (1 << bits) < D:
        bits += 1
    return (bits + 7) // 8


def base_rows(T, seed, groups=False):
    """T source rows' task columns, table-global ids, from a one-distro synth tick: (TaskSoA, group_max_hosts, n_versions,
    cfg row).  groups=False: no task group."""
    w = synth.make(np.array([T]), seed, tg_frac=0.2 if groups else 0.0, group_versions_frac=1.0 if groups else 0.0)
    t = w.tasks
    flags = t.flags & np.uint32(~(L.EVG_TF_DEPS_MET | L.EVG_TF_OTHER_DISTRO) & 0xFFFFFFFF)
    tasks = S.TaskSoA(t.priority, t.expected_ns, t.queue_basis_ns, t.wait_basis_ns, t.num_dependents, t.task_group_order, t.group_id,
                      t.version_id, flags, np.zeros(T + 1, np.int64), np.zeros(0, np.int32)).normalize()
    return tasks, w.distros.group_max_hosts.astype(np.int32), int(w.distros.cfg["n_versions"][0]), w.distros.cfg[:1]


def alias_table(base, D, sec_off, sec_idx, extra=(), seed=0):
    """An AliasTable whose every row passes FindHostSchedulableForAlias (all base bits, no unattainable dependency,
    TaskGroupMaxHosts 0, no dependency).  Names 0 .. D-1 are the distros' own ids; name D + j is an alias shared by the
    distros extra[j].  -> (AliasTable, cfg of D distros)."""
    tasks, gmax, n_versions, cfg = base
    T = tasks.n_tasks
    rng = np.random.default_rng(seed)
    dest_off = np.concatenate([[0], np.cumsum([1] * D + [len(x) for x in extra])]).astype(np.int64)
    dest_idx = np.concatenate([np.arange(D)] + [np.asarray(x) for x in extra]).astype(np.int32)
    deps = S.DepsTable(np.zeros(T + 1, np.int64), np.zeros(0, np.uint8), np.zeros(0, np.int32), np.zeros(0, np.uint8),
                       np.zeros(T, np.uint8), np.zeros(T, np.uint8), np.zeros(0, np.uint8))
    primary = np.where(rng.random(T) < 0.1, -1, rng.integers(0, D, T)).astype(np.int32)
    at = S.AliasTable(tasks, gmax, n_versions, np.full(T, S.SQ_BASE, np.uint8), np.zeros(T, np.int32), primary,
                      np.asarray(sec_off, np.int64), np.asarray(sec_idx, np.int32), dest_off, dest_idx, deps,
                      np.zeros(0, np.int64)).normalize()
    return at, np.repeat(cfg, D)


def one_name(q):
    """Row t names the own id of distro q[t]."""
    return np.arange(len(q) + 1, dtype=np.int64), np.asarray(q, np.int32)


def names_of(rows):
    """Row t names rows[t] (a list)."""
    return np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64), np.array([n for r in rows for n in r], np.int32)


def low_byte_queues(D, T):
    """Queue ids that share their low byte (c + 256 k) and, where D allows, their low two bytes (c + 65 536 k), in
    descending k: a pass that is dropped or reads the wrong shift leaves them in source order."""
    c = min(5, (D - 1) % 256)  # at least two ids c + 256 k below D once D > 256
    k1 = (D - 1 - c) // 256
    q = c + 256 * (k1 - np.arange(T) % (k1 + 1))
    k2 = (D - 1 - c) // 65536
    if k2 > 0:
        q[1::2] = c + 65536 * (k2 - (np.arange(T)[1::2] // 2) % (k2 + 1))
    return q


def alias_rows(kind, D, T, rng):
    """(sec_off, sec_idx, extra) of one key distribution over T rows and D distros."""
    if kind == "descending":           # every key moves
        return one_name(D - 1 - (np.arange(T) * D) // T) + ((),)
    if kind == "last":                 # every pair in queue D - 1
        return one_name(np.full(T, D - 1)) + ((),)
    if kind == "low_byte":
        return one_name(low_byte_queues(D, T)) + ((),)
    if kind == "hot":                  # 90 % of the pairs in one queue
        return one_name(np.where(rng.random(T) < 0.9, D // 2, rng.integers(0, D, T))) + ((),)
    if kind == "tiles":                # one queue per 2048-key tile: every other digit is empty across the tile
        return one_name(((np.arange(T) // 2048) * 40503 + 17) % D) + ((),)
    if kind == "random":               # 1-3 own ids per row
        return names_of([rng.integers(0, D, rng.integers(1, 4)).tolist() for _ in range(T)]) + ((),)
    if kind == "fan_out":              # one name shared by up to 700 distros, named by every 8th row
        wide = np.unique(np.linspace(0, D - 1, min(D, 700)).astype(np.int64))[::-1]
        rows = [[D] if t % 8 == 0 else [int(x)] for t, x in enumerate(rng.integers(0, D, T))]
        return names_of(rows) + ((wide,),)
    if kind == "dup":                  # e directly, through an alias holding e and one more distro, and e again
        e = rng.integers(0, D, T)
        other = rng.integers(0, D, T)
        extra = [[int(a), int(b)] if a != b else [int(a)] for a, b in zip(e, other)]
        return names_of([[int(x), D + t, int(x)] for t, x in enumerate(e)]) + (extra,)
    raise ValueError(kind)


def expected_pairs(at):
    """Each row's distinct destinations in secondary_idx / dest_idx order, then np.lexsort((row, queue))."""
    T = at.n_tasks
    row = np.repeat(np.arange(T, dtype=np.int64), np.diff(at.secondary_off))
    name = at.secondary_idx.astype(np.int64)
    row, name = row[name >= 0], name[name >= 0]
    cnt = at.dest_off[name + 1] - at.dest_off[name]
    row = np.repeat(row, cnt)
    queue = at.dest_idx[np.repeat(at.dest_off[name], cnt) + np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)].astype(np.int64)
    _, first = np.unique((queue << 32) | row, return_index=True)   # a destination counts once per row
    keep = np.sort(first)
    row, queue = row[keep], queue[keep]
    o = np.lexsort((row, queue))
    return queue[o], row[o]


def first_appearance(queue, ids, D):
    """Per queue, the distinct ids in first-appearance order over the sorted pairs: (ids in slot order, offsets)."""
    sel = np.nonzero(ids >= 0)[0]
    _, first = np.unique((queue[sel] << 32) | ids[sel].astype(np.int64), return_index=True)
    at = np.sort(sel[first])
    return ids[at], np.concatenate([[0], np.cumsum(np.bincount(queue[at], minlength=D))]).astype(np.int64)


def plan_and_count(engine, at, cfg):
    """evg_plan_aliases under torch.profiler -> (task_off, group_off, n_versions, kernel names).  As in
    test_gpu_onchip_sort.profiled, a torch kernel opens the window and the list must hold every kernel the context
    counted; a window that saw none of them is opened again, a few more times than there."""
    import torch

    def call():
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        out.append(engine.plan_aliases(at, cfg, NOW))

    for _ in range(6):
        out = []
        names = launched_kernels(call)
        if len(names) == engine.last_launch_count():
            task_off, group_off, n_versions = out[0]
            return task_off.copy(), group_off.copy(), n_versions.copy(), [n.split("(")[0] for n in names]
    raise AssertionError(f"the profiler saw {len(names)} kernels, the context counted {engine.last_launch_count()}: {names}")


def check_alias(engine, at, cfg, groups=False):
    D = int(cfg.shape[0])
    task_off, group_off, n_versions, kernels = plan_and_count(engine, at, cfg)
    p = alias_passes(D)
    assert kernels.count("k_al_hist") == p and kernels.count("k_al_scatter") == p, (D, p, kernels)
    queue, row = expected_pairs(at)
    assert np.array_equal(task_off, np.concatenate([[0], np.cumsum(np.bincount(queue, minlength=D))]))
    src, gsrc = engine.download_alias_map()
    assert src.shape == row.shape
    bad = np.nonzero(src != row)[0]
    assert bad.size == 0, (D, int(bad[0]), int(src[bad[0]]), int(row[bad[0]]))
    want_g, want_goff = first_appearance(queue, at.tasks.group_id[row], D)
    assert np.array_equal(group_off, want_goff) and np.array_equal(gsrc, want_g)
    _, want_voff = first_appearance(queue, at.tasks.version_id[row], D)
    assert np.array_equal(n_versions, np.diff(want_voff))
    if groups:
        assert gsrc.shape[0] > 0 and (np.diff(want_voff) > 1).any()
    return queue


D_CASES = [1, 2, 255, 256, 257, 4096, 65536, 65537, 100_000]
KINDS = ["descending", "last", "low_byte", "hot", "tiles", "random", "fan_out", "dup"]


def test_alias_routing_restated():
    assert [alias_passes(D) for D in D_CASES] == [0, 1, 1, 1, 2, 2, 2, 3, 3]
    assert alias_passes(2 ** 24) == 3 and alias_passes(2 ** 24 + 1) == 4 and alias_passes(2 ** 31) == 4
    # the key distributions are what their names say
    rng = np.random.default_rng(1)
    q = low_byte_queues(100_000, 4000)
    assert (q % 256 == 5).all() and len(set(q.tolist())) > 300 and (q == 65536 + 5).any() and (q < 100_000).all()
    for D in D_CASES[4:]:
        q = low_byte_queues(D, 6145)
        assert len(set(q.tolist())) > 1 and len(set((q % 256).tolist())) == 1 and (q < D).all()
    assert (np.diff(alias_rows("descending", 65537, 6145, rng)[1].astype(np.int64)) < 0).all()
    off, idx, extra = alias_rows("dup", 300, 50, rng)
    at, _ = alias_table(base_rows(50, 1), 300, off, idx, extra)
    queue, row = expected_pairs(at)
    assert len(queue) == sum(len(x) for x in extra)
    assert np.array_equal(np.bincount(row, minlength=50), [len(x) for x in extra])


@pytest.mark.gpu
@pytest.mark.parametrize("D", D_CASES)
def test_alias_sort_at_every_pass_count(engine, D):
    """Every key distribution over 3 * 2048 + 1 source rows, on both sides of every pass-count boundary."""
    rng = np.random.default_rng(9000 + D)
    base = base_rows(3 * 2048 + 1, 9001)
    for kind in KINDS:
        if kind == "low_byte" and D <= 256:
            continue
        off, idx, extra = alias_rows(kind, D, base[0].n_tasks, rng)
        at, cfg = alias_table(base, D, off, idx, extra, seed=D)
        queue = check_alias(engine, at, cfg)
        if kind == "low_byte":
            assert len(np.unique(queue)) > 1 and (np.unique(queue) % 256 == queue[0] % 256).all()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [257, 65537])
@pytest.mark.parametrize("P", [1, 2047, 2048, 2049, 3 * 2048 + 1, 300_000])
def test_alias_sort_at_every_tile_count(engine, D, P):
    """A last tile of 1, 2047, 2048 and 1 keys, and 147 tiles: descending and low-byte queues, at two and three passes."""
    rng = np.random.default_rng(9100 + P)
    base = base_rows(P, 9101)
    for kind in ("descending", "low_byte", "hot"):
        off, idx, extra = alias_rows(kind, D, P, rng)
        at, cfg = alias_table(base, D, off, idx, extra, seed=P)
        check_alias(engine, at, cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4096, 65537])
def test_alias_groups_and_versions_plan_like_a_fresh_upload(engine, fresh, D):
    """Task groups and versions numbered per queue in first appearance, then the composed tick planned against a fresh
    upload of the host route (soa.compose_aliases), at two and three passes."""
    rng = np.random.default_rng(9200 + D)
    base = base_rows(6000, 9201, groups=True)
    for kind in ("random", "low_byte"):
        off, idx, extra = alias_rows(kind, D, base[0].n_tasks, rng)
        at, cfg = alias_table(base, D, off, idx, extra, seed=D)
        check_alias(engine, at, cfg, groups=True)
        plan_and_check(engine, fresh, at, cfg, NOW)


@pytest.mark.gpu
def test_alias_scale_scans_take_the_carry_loop(engine):
    """2^20 + 2049 pairs: the group and version flags' scans have 1027 block sums, so k_scan_sums carries over two
    chunks.  Groups of consecutive rows are spread over 4096 queues (two passes)."""
    P = (1 << 20) + 2049
    base = base_rows(P, 9301, groups=True)
    rng = np.random.default_rng(9300)
    at, cfg = alias_table(base, 4096, *one_name(rng.integers(0, 4096, P)), seed=9302)
    assert (P + 1023) // 1024 > 1024
    check_alias(engine, at, cfg, groups=True)


# ================================================================ B. the segmented merge sorts
SHAPE = [0, 0, 1, 2, 3, 4, 5, 7, 8, 9, 255, 256, 257, 1023, 1024, 1025, 0, 4097, 0]


def shape_of(name, rng):
    """Segment lengths: SHAPE shuffled with its longest segment first or last, or many empty segments between tiny
    ones (one 256-thread block spans dozens of segments)."""
    if name == "sparse":
        return rng.choice([0, 0, 0, 0, 0, 1, 2, 3], 900).tolist()
    rest = [n for n in SHAPE if n != max(SHAPE)]
    rng.shuffle(rest)
    return [max(SHAPE)] + rest if name == "longest_first" else rest + [max(SHAPE)]


SHAPES = ["longest_first", "longest_last", "sparse"]


# ---------------------------------------------------------------- legacy prioritiser
def legacy_reference(table):
    """(order, count, status) of evg_prioritize_legacy_batch for lists in a decomposable mode: per distro a stable sort
    by (list, comparator chain, presort rank), then mergeTasks' interleave."""
    order = np.full(table.n_tasks, -1, np.int32)
    count = np.zeros(table.n_distros, np.int64)
    for d in range(table.n_distros):
        a, b = int(table.task_off[d]), int(table.task_off[d + 1])
        s = slice(a, b)
        prio, fl = table.priority[s], table.flags[s]
        req = fl & 3
        lst = np.where(prio > M.MAX_TASK_PRIORITY, 0, np.where(req == L.EVG_LF_REQ_SYSTEM, 2, np.where(req == L.EVG_LF_REQ_PATCH, 1, 3)))
        modes = table.list_mode[3 * d:3 * d + 3]
        assert (modes != L.EVG_LEGACY_MODE_LITERAL).all()
        revision = modes[np.minimum(lst, 2)] == L.EVG_LEGACY_MODE_REVISION
        grp = table.tg_rank[s] >= 0
        plain = ~grp
        z = np.zeros(b - a, np.int64)
        keys = (  # last key first, as np.lexsort takes them
            table.presort_rank[s],
            np.where(plain, ~table.expected_ns[s], z),                                   # byRuntime: longer first
            np.where(plain, np.where(revision, ~table.revision_order[s].astype(np.int64), table.ingest_ns[s]), z),  # byAge
            np.where(plain, (fl & L.EVG_LF_GENERATE) == 0, 0),                            # byGenerateTasks
            np.where(plain, ~table.num_dependents[s].astype(np.int64), z),                # byNumDeps
            np.where(plain, ~prio, z),                                                    # byPriority
            np.where(plain, (fl & L.EVG_LF_MERGE_QUEUE_VERSION) == 0, 0),                 # byCommitQueue
            np.where(grp, table.task_group_order[s], 0),                                  # byTaskGroupOrder: order in a group,
            np.where(grp, table.tg_rank[s], 0),                                           # then the group's rank,
            plain,                                                                        # group tasks first
            lst)
        o = np.lexsort(keys)
        by = [o[lst[o] == k].tolist() for k in range(3)]
        merged = OL.merge_tasks(by[0], by[2], by[1])
        order[a:a + len(merged)] = merged
        count[d] = len(merged)
    return order, count, np.zeros(table.n_distros, np.int32)


def legacy_table(lengths, rng):
    """Heavily tied comparators at their int64 / int32 extremes, task groups with tg_rank a function of tg_pair_id,
    a presort permutation per distro, INGEST and REVISION lists."""
    n = int(sum(lengths))
    grp = rng.random(n) < 0.25
    rank = rng.integers(0, 4, n)
    req = rng.choice(np.array([L.EVG_LF_REQ_SYSTEM, L.EVG_LF_REQ_PATCH, L.EVG_LF_REQ_OTHER], np.uint32), n, p=[0.45, 0.45, 0.1])
    flags = req | np.where(rng.random(n) < 0.2, L.EVG_LF_GENERATE, 0).astype(np.uint32) | \
        np.where(rng.random(n) < 0.2, L.EVG_LF_MERGE_QUEUE_VERSION, 0).astype(np.uint32)
    pick = lambda vals, dt: rng.choice(np.array(vals, dt), n)  # noqa: E731
    return S.LegacyTable(
        priority=pick([I64_MIN, -1, 100, 101, I64_MAX], np.int64), ingest_ns=pick([I64_MIN, 0, I64_MAX], np.int64),
        expected_ns=pick([I64_MIN, 1, I64_MAX], np.int64), num_dependents=pick([I32_MIN, 0, I32_MAX], np.int32),
        revision_order=pick([I32_MIN, 0, I32_MAX], np.int32), project_id=np.zeros(n, np.int32),
        tg_rank=np.where(grp, rank, -1).astype(np.int32), tg_pair_id=np.where(grp, 3 - rank, -1).astype(np.int32),
        task_group_order=np.where(grp, rng.integers(0, 3, n), 0).astype(np.int32),
        presort_rank=np.concatenate([rng.permutation(k) for k in lengths] + [np.zeros(0, np.int64)]).astype(np.int32), flags=flags,
        task_off=np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64),
        list_mode=rng.choice(np.array([L.EVG_LEGACY_MODE_INGEST, L.EVG_LEGACY_MODE_REVISION], np.uint8), 3 * len(lengths)))


def test_legacy_reference_equals_the_oracle():
    """The numpy restatement against oracle_legacy (literal comparators, Go's sort.Stable) on small decomposable queues,
    with the comparators' fields at their extremes."""
    rnd = np.random.default_rng(9400)
    versions = {f"v{k}": (M.GITHUB_MERGE_REQUESTER if k == 0 else M.PATCH_VERSION_REQUESTER) for k in range(6)}
    checked = 0
    for seed in range(40):
        batch = []
        for k, n in enumerate([0, 1, 2, 3, 9, 25, 60]):
            tasks = random_queue(random.Random(9400 + 97 * seed + k), n)
            for t in tasks:
                t.num_dependents = int(rnd.choice([I32_MIN, 0, 1, I32_MAX]))
                t.revision_order_number = int(rnd.choice([I32_MIN, 0, 7, I32_MAX]))
                t.ingest_time = int(rnd.choice([I64_MIN, NOW, I64_MAX]))
                t.expected_duration = int(rnd.choice([I64_MIN, -1, M.MINUTE, I64_MAX]))
                patch = t.requester not in M.SYSTEM_VERSION_REQUESTER_TYPES
                t.priority = int(rnd.choice([I64_MIN, -1, 100, 101, I64_MAX] if patch else [I64_MIN, -1, 100]))
            batch.append((f"d{k}", tasks, versions))
        table = S.marshal_legacy(batch, None)
        keep = [d for d in range(len(batch)) if (table.list_mode[3 * d:3 * d + 3] != L.EVG_LEGACY_MODE_LITERAL).all()]
        for d in keep:
            a, b = int(table.task_off[d]), int(table.task_off[d + 1])
            one = S.LegacyTable(**{f: getattr(table, f)[a:b] for f, _ in S.LegacyTable.COLUMNS},
                                task_off=np.array([0, b - a], np.int64), list_mode=table.list_mode[3 * d:3 * d + 3])
            order, count, _ = legacy_reference(one)
            tasks = batch[d][1]
            want = [t.id for t in OL.prioritize_tasks([mk_copy(t) for t in tasks], versions, None)]
            assert [tasks[int(i)].id for i in order[:int(count[0])]] == want, (seed, d)
            assert (order[int(count[0]):] == -1).all()
            checked += 1
    assert checked > 200


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_legacy_merge_sort_at_every_run_length(engine, shape):
    rng = np.random.default_rng(9500 + SHAPES.index(shape))
    table = legacy_table(shape_of(shape, rng), rng)
    order, count, status = (x.copy() for x in engine.prioritize_legacy_batch(table))
    want_order, want_count, want_status = legacy_reference(table)
    assert np.array_equal(count, want_count) and np.array_equal(status, want_status)
    bad = np.nonzero(order != want_order)[0]
    assert bad.size == 0, (shape, int(bad[0]), int(np.searchsorted(table.task_off, bad[0], "right") - 1))


# ---------------------------------------------------------------- DAG task-group buckets
GROUP_INDEX = [I32_MIN, I32_MIN + 1, -1, 0, 1, I32_MAX]


def dag_items(n, tag, rng):
    """Grouped and ungrouped items; four groups over six GroupIndex values, so most (group, index) pairs repeat and
    only stability orders them; a few in-queue dependencies."""
    items = []
    for k in range(n):
        deps = [f"{tag}-{int(rng.integers(n))}"] if rng.random() < 0.05 else []
        items.append({"id": f"{tag}-{k}", "group": f"g{int(rng.integers(4))}" if rng.random() < 0.7 else "", "build_variant": "bv",
                      "project": "p", "version": "v", "group_index": int(rng.choice(GROUP_INDEX)), "dependencies": deps})
    return items


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_dag_group_merge_sort_at_every_run_length(engine, shape):
    rng = np.random.default_rng(9600 + SHAPES.index(shape))
    batches = [dag_items(n, f"q{d}", rng) for d, n in enumerate(shape_of(shape, rng))]
    res = scheduler.rebuild_dag_dispatchers([_tq(b) for b in batches], engine=engine)
    for d, (items, (order, n_cycles, units)) in enumerate(zip(batches, res)):
        want_order, want_cycles, want_units = OD.rebuild(items)
        assert order == want_order and n_cycles == len(want_cycles), d
        assert units == want_units, d
    big = max(batches, key=len)
    assert len(big) < 1000 or len({(it["group"], it["group_index"]) for it in big if it["group"]}) == 4 * len(GROUP_INDEX)


# ---------------------------------------------------------------- start-estimate host pools
def est_hosts(pools, rng):
    """Host rows whose pools have the given sizes: free hosts (0), starting hosts (3 min), running hosts at the int64
    extremes or overrunning, and ignored rows between them, so that pool sizes differ from row counts.  Each pool's
    last value is a 3 h overrun, below every other value but I64_MIN: a run left unmerged moves it."""
    kind, expected, dispatch, off = [], [], [], [0]
    empties = 0
    for m in pools:
        k = rng.choice(np.array([L.EVG_EH_FREE, L.EVG_EH_STARTING, L.EVG_EH_RUNNING, L.EVG_EH_UNINITIALIZED, L.EVG_EH_PROVISIONING], np.uint8),
                       m, p=[0.3, 0.3, 0.3, 0.05, 0.05])
        n_ign = int(rng.integers(0, 3)) + m // 40 if m else 2 * (empties % 2)   # an empty pool: no row, or ignored rows only
        empties += m == 0
        if m:
            k[-1] = L.EVG_EH_RUNNING
        k = np.insert(k, rng.integers(0, m + 1, n_ign), L.EVG_EH_IGNORED)
        r = k.shape[0]
        # once I64_MIN is popped every later value wraps, and the pool's order no longer shows in the estimates: it goes
        # to the pools below 256 hosts only
        e = rng.choice(np.array([I64_MAX, M.MINUTE, 30 * M.MINUTE, 0] + ([I64_MIN] if m < 256 else []), np.int64), r)
        t = np.where(rng.random(r) < 0.5, NOW, NOW - rng.integers(0, 2, r) * M.HOUR).astype(np.int64)
        if m:
            last = np.nonzero(k != L.EVG_EH_IGNORED)[0][-1]
            e[last], t[last] = 0, NOW - 3 * M.HOUR   # an overrun of 3 h; every other overrun is 1 h at most
        kind.append(k)
        expected.append(e)
        dispatch.append(t)
        off.append(off[-1] + r)
    cat = lambda xs, dt: np.concatenate(xs + [np.zeros(0, dt)]).astype(dt)  # noqa: E731
    return S.EstHostTable(cat(kind, np.uint8), cat(expected, np.int64), cat(dispatch, np.int64), np.array(off, np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_estimate_pool_merge_sort_at_every_run_length(engine, shape):
    """Every listed queue holds more items than its pool, so every sorted value is popped into an estimate.  Empty pools
    (no row, or ignored rows only) sit between full ones; distros with hosts and no items are sorted but not simulated,
    one of them with a pool larger than any listed one."""
    rng = np.random.default_rng(9700 + SHAPES.index(shape))
    pools = shape_of(shape, rng)
    longest = max(pools)
    idle = [3, longest + 900, 40]                       # hosts, no items
    sizes = pools + idle
    table = est_hosts(sizes, rng)
    n_items = [m + 1 + int(rng.integers(0, 4)) for m in pools] + [0] * len(idle)
    queues = [np.where(rng.random(n) < 0.3, 3 * M.MINUTE, rng.integers(0, 2 * M.HOUR, n)).tolist() for n in n_items]
    off = np.concatenate([[0], np.cumsum(n_items)]).astype(np.int64)
    dur = np.array([v for q in queues for v in q], dtype=np.int64)
    start, used = (x.copy() for x in engine.estimate_start_batch(dur, off, table, NOW))
    p = pools_of(table, NOW)
    rows = np.diff(table.est_host_off)
    assert [len(x) for x in p] == sizes and (rows > np.array(sizes)).any()
    assert ((rows == 0) & (np.array(sizes) == 0)).any() and ((rows > 0) & (np.array(sizes) == 0)).any()
    vals = np.concatenate([np.array(x, np.int64) for x in p])
    assert {0, 3 * M.MINUTE, I64_MIN, I64_MAX} <= set(vals.tolist()) and (vals < 0).any()
    least = [x[-1] for x in p[:len(pools)] if x]
    assert all(v == -3 * M.HOUR for v in least) and -3 * M.HOUR == min(v for v in vals.tolist() if v != I64_MIN)
    want, want_used = expect(dur, off, p)
    assert np.array_equal(used, want_used)
    bad = np.nonzero(start != want)[0]
    assert bad.size == 0, (shape, int(bad[0]), int(np.searchsorted(off, bad[0], "right") - 1))
