"""EVG_LEGACY_MODE_GO_STABLE: the legacy prioritiser's replay of Go's sort.Stable on lists where the comparator chain
is not a strict weak order, against oracle/oracle_legacy.py (literal comparators + a port of sort.Stable) id for id.

The replay runs insertion sorts of 20-blocks, then per level waves of symMerge calls; a wave whose largest call spans
more than 1024 tasks rotates with a CTA per call, any other with a warp per call.  The list lengths below sit on both
sides of the 20-block and level edges (19 .. 41), of that rotation boundary (1024 / 1025: the first wave of the top
level) and reach a few tens of thousands."""
import random

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler as S
from evergreen_b200 import soa
from oracle import oracle_legacy as OL
from test_gpu_legacy import G, NOW, mk, random_queue

pytestmark = pytest.mark.gpu

VERSIONS = {f"v{k}": (M.GITHUB_MERGE_REQUESTER if k == 0 else M.PATCH_VERSION_REQUESTER) for k in range(6)}


def literal_queue(rnd, n, kind, tag="t"):
    """n tasks that all land in one list on which the chain is not a strict weak order, with many ties:
      repo       commit builds of three projects (byAge switches field pair by pair)
      patch      patch tasks whose expected durations mix zero and non-zero (byRuntime ties a zero with everything)
      high       high-priority commit builds of three projects and patch tasks
      collision  repotracker tasks in task groups whose "BuildId-TaskGroup" strings collide"""
    out = []
    for k in range(n):
        t = M.Task(id=f"{tag}_{k:06d}_{rnd.randrange(10 ** 6)}", version=f"v{rnd.randrange(6)}", build_id=f"b{rnd.randrange(4)}",
                   priority=rnd.choice([0, 0, 1, 5]), num_dependents=rnd.choice([0, 0, 0, 1, 3]), generate_task=rnd.random() < 0.05,
                   revision_order_number=rnd.randrange(6), ingest_time=NOW - rnd.randrange(6) * M.HOUR,
                   expected_duration=rnd.randrange(1, 5) * 10 * M.MINUTE, project=rnd.choice(["pa", "pb", "pc"]),
                   requester=M.REPOTRACKER_VERSION_REQUESTER)
        if kind == "patch":
            t.requester = rnd.choice([M.PATCH_VERSION_REQUESTER, M.GITHUB_PR_REQUESTER])
            t.expected_duration = 0 if rnd.random() < 0.3 else t.expected_duration
        elif kind == "high":
            t.priority = rnd.choice([101, 150, 150])
            t.requester = rnd.choice([M.REPOTRACKER_VERSION_REQUESTER, M.TRIGGER_REQUESTER, M.PATCH_VERSION_REQUESTER])
        elif kind == "collision" and rnd.random() < 0.4:
            t.build_id, t.task_group = rnd.choice([("a-b", "c"), ("a", "b-c"), ("a", "b"), ("b", "a")])
            t.task_group_order = rnd.randrange(1, 4)
        elif kind == "repo" and rnd.random() < 0.1:
            t.task_group, t.task_group_order = f"tg{rnd.randrange(2)}", rnd.randrange(1, 4)
        out.append(t)
    return pin_durations(out)


def pin_durations(tasks):
    """A fresh cached prediction per task, so FetchExpectedDuration returns expected_duration as it is -- zero included
    (without one, a zero resolves to the default duration)."""
    for t in tasks:
        t.duration_prediction = M.CachedDurationValue(value=t.expected_duration, ttl=M.HOUR, collected_at=NOW)
    return tasks


def ids(tasks):
    return [t.id for t in tasks]


def check_exact(engine, batch, *, discriminate=True):
    """Every distro of the batch through exact=True in one call, id for id against the oracle; with `discriminate`, the
    default (LITERAL) order differs from the oracle's on some distro, so the check tells a replay from a key sort."""
    exact = S.CmpBasedTaskPrioritizer(engine=engine, now=NOW, exact=True).prioritize_batch(batch)
    launches = engine.last_launch_count()
    want = [ids(OL.prioritize_tasks(list(tasks), versions, NOW)) for _, tasks, versions in batch]
    for d, ((got, status), w) in enumerate(zip(exact, want)):
        assert status == L.EVG_LEGACY_OK, d
        assert ids(got) == w, (d, len(w))
    if discriminate:
        approx = S.CmpBasedTaskPrioritizer(engine=engine, now=NOW).prioritize_batch(batch)
        assert any(ids(got) != w for (got, _), w in zip(approx, want))
    return launches


LENGTHS = [0, 1, 2, 19, 20, 21, 39, 40, 41, 300, 1024, 1025, 2500]


@pytest.mark.parametrize("kind", ["repo", "patch", "high", "collision"])
def test_one_list_at_every_length(engine, kind):
    """One distro per length, all its tasks in one LITERAL list, several distros per call."""
    rnd = random.Random(5000 + ["repo", "patch", "high", "collision"].index(kind))
    batch = [(f"d{n}", literal_queue(rnd, n, kind, f"d{n}"), VERSIONS) for n in LENGTHS]
    table = soa.marshal_legacy(batch, NOW, exact=True)
    modes = table.list_mode.reshape(-1, 3)
    assert (modes[LENGTHS.index(19):] == L.EVG_LEGACY_MODE_GO_STABLE).any(axis=1).all()
    check_exact(engine, batch)


@pytest.mark.parametrize("seed", range(4))
def test_mixed_queues_match_the_oracle(engine, seed):
    """Production-shaped queues: every list kind at once, commit builds of three projects (also in the high-priority
    list), zero and non-zero runtimes mixed, merge-queue versions; a few hundred and a few thousand tasks."""
    rnd = random.Random(5100 + seed)
    batch = [(f"d{k}", pin_durations(random_queue(rnd, n, one_project=False, zero_runtimes=k % 2 == 1)), VERSIONS)
             for k, n in enumerate([0, 3, 45, 400, 777, 3000, 1])]
    check_exact(engine, batch)


def test_a_long_list(engine):
    """One repotracker list of 30 000 tasks next to a short one.  The launches follow from the longest distro alone:
    k_legacy_init, 15 merge passes, k_gs_insertion, then per level (block 20 .. 20 480) k_gs_seed and ceil(log2(min(2
    block, 30 000))) waves -- 6, 7, ..., 15, 15 -- and k_legacy_interleave."""
    rnd = random.Random(5200)
    batch = [("big", literal_queue(rnd, 30_000, "repo", "big"), VERSIONS), ("small", literal_queue(rnd, 41, "patch", "s"), VERSIONS)]
    levels = [20 << k for k in range(11)]
    assert levels[-1] < 30_000 < 2 * levels[-1]
    waves = [(min(2 * b, 30_000) - 1).bit_length() for b in levels]
    assert waves == list(range(6, 16)) + [15]
    assert check_exact(engine, batch) == 1 + 15 + 1 + len(levels) + sum(waves) + 1


def test_reference_vectors_through_exact(engine):
    p = S.CmpBasedTaskPrioritizer(engine=engine, now=NOW, exact=True)
    for case in G["orders"]:
        got, reasons, err = p.PrioritizeTasks("distro", [mk(t) for t in case["tasks"]], case["versions"])
        assert err is None and reasons == {}
        if "want_order" in case:
            assert ids(got) == case["want_order"]
        for a, b in case.get("want_before", []):
            assert ids(got).index(a) < ids(got).index(b)
    for case in G["splits"]:
        tasks = [mk(t) for t in case["tasks"]]
        got, _, err = p.PrioritizeTasks("d", tasks, {})
        assert err is None and ids(got) == ids(OL.prioritize_tasks(list(tasks), {}, NOW))


def test_non_decomposable_queue_is_served(engine):
    """The three-project queue the default prioritiser reports NotDecomposableError on."""
    tasks = random_queue(random.Random(77), 300, one_project=False)
    got, reasons, err = S.CmpBasedTaskPrioritizer(engine=engine, now=NOW, exact=True).PrioritizeTasks("d", tasks, {})
    assert err is None and reasons == {}
    assert ids(got) == ids(OL.prioritize_tasks(list(tasks), {}, NOW))


def test_go_stable_on_decomposable_lists_equals_the_key_sort(engine):
    """INGEST and REVISION lists forced to GO_STABLE: the same order, and every distro OK."""
    rnd = random.Random(5300)
    batch = [(f"d{k}", random_queue(rnd, n), VERSIONS) for k, n in enumerate([0, 1, 2, 21, 41, 400, 1500, 3])]
    table = soa.marshal_legacy(batch, NOW)
    assert (table.list_mode != L.EVG_LEGACY_MODE_LITERAL).all()
    assert (table.list_mode == L.EVG_LEGACY_MODE_REVISION).any() and (table.list_mode == L.EVG_LEGACY_MODE_INGEST).any()
    want = [x.copy() for x in engine.prioritize_legacy_batch(table)]
    table.list_mode[:] = L.EVG_LEGACY_MODE_GO_STABLE
    got = [x.copy() for x in engine.prioritize_legacy_batch(table)]
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert (got[2] == L.EVG_LEGACY_OK).all()


def test_literal_distros_are_untouched_by_go_stable_neighbours(engine):
    """A call mixing LITERAL, GO_STABLE and key-mode distros gives the LITERAL distros the order and status of a call with
    them alone."""
    rnd = random.Random(5400)
    lit = [(f"l{k}", literal_queue(rnd, n, kind, f"l{k}"), VERSIONS) for k, (n, kind) in enumerate([(300, "repo"), (60, "patch"), (2000, "high")])]
    ex = [(f"e{k}", literal_queue(rnd, n, kind, f"e{k}"), VERSIONS) for k, (n, kind) in enumerate([(500, "repo"), (41, "collision")])]
    key = [(f"k{k}", random_queue(rnd, n), VERSIONS) for k, n in enumerate([50, 700])]
    alone = soa.marshal_legacy(lit, NOW)
    a_order, a_count, a_status = (x.copy() for x in engine.prioritize_legacy_batch(alone))
    assert (a_status == L.EVG_LEGACY_NOT_DECOMPOSABLE).all()
    batch = [ex[0], lit[0], key[0], lit[1], ex[1], lit[2], key[1]]
    mixed = soa.marshal_legacy(batch, NOW, exact=True)
    lit_at = [1, 3, 5]
    for d in lit_at:  # back to LITERAL for the distros of `lit`
        mixed.list_mode[3 * d:3 * d + 3] = alone.list_mode[3 * lit_at.index(d):3 * lit_at.index(d) + 3]
    assert (mixed.list_mode == L.EVG_LEGACY_MODE_GO_STABLE).any() and (mixed.list_mode == L.EVG_LEGACY_MODE_LITERAL).any()
    order, count, status = (x.copy() for x in engine.prioritize_legacy_batch(mixed))
    for j, d in enumerate(lit_at):
        a, b = int(mixed.task_off[d]), int(mixed.task_off[d + 1])
        a0, b0 = int(alone.task_off[j]), int(alone.task_off[j + 1])
        assert np.array_equal(order[a:b], a_order[a0:b0]) and count[d] == a_count[j] and status[d] == a_status[j]
    for d in (0, 4, 2, 6):
        a = int(mixed.task_off[d])
        tasks = batch[d][1]
        assert status[d] == L.EVG_LEGACY_OK
        assert [tasks[int(i)].id for i in order[a:a + int(count[d])]] == ids(OL.prioritize_tasks(list(tasks), VERSIONS, NOW))


def test_unknown_list_mode_is_rejected(engine):
    table = soa.marshal_legacy([("d", literal_queue(random.Random(1), 30, "repo"), VERSIONS)], NOW, exact=True)
    table.list_mode[2] = L.EVG_LEGACY_MODE_GO_STABLE + 1
    with pytest.raises(L.EvgError, match="unknown list mode 4"):
        engine.prioritize_legacy_batch(table)
