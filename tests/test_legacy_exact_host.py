"""soa.marshal_legacy(exact=True): the lists that would be EVG_LEGACY_MODE_LITERAL -- and only those -- become
EVG_LEGACY_MODE_GO_STABLE; no device needed."""
import random

import numpy as np

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa

NOW = 1_700_000_000 * M.SECOND


def queue(rnd, n):
    projects = rnd.choice([["p"], ["pa", "pb", "pc"]])
    zeros = rnd.random() < 0.3
    out = []
    for k in range(n):
        req = rnd.choice([M.REPOTRACKER_VERSION_REQUESTER, M.PATCH_VERSION_REQUESTER, M.TRIGGER_REQUESTER, "nonsense"])
        tg = rnd.random() < 0.2
        out.append(M.Task(id=f"t{k}", requester=req, project=rnd.choice(projects), priority=rnd.choice([0, 5, 101]),
                          build_id=rnd.choice(["a", "a-b"]), task_group=rnd.choice(["b-c", "c"]) if tg else "",
                          expected_duration=0 if zeros and rnd.random() < 0.5 else M.MINUTE))
    return out


def test_exact_marks_exactly_the_literal_lists():
    rnd = random.Random(3)
    batch = [(f"d{k}", queue(rnd, rnd.choice([0, 1, 2, 5, 30])), {}) for k in range(300)]
    plain = soa.marshal_legacy(batch, None)
    exact = soa.marshal_legacy(batch, None, exact=True)
    lit = plain.list_mode == L.EVG_LEGACY_MODE_LITERAL
    assert lit.any() and (~lit).any()
    assert np.array_equal(exact.list_mode, np.where(lit, L.EVG_LEGACY_MODE_GO_STABLE, plain.list_mode))
    for name, _ in soa.LegacyTable.COLUMNS:
        assert np.array_equal(getattr(plain, name), getattr(exact, name))
    assert np.array_equal(plain.task_off, exact.task_off)


def test_a_format_collision_is_go_stable():
    """Two (TaskGroup, BuildId) pairs that format to one "BuildId-TaskGroup" string, in an otherwise INGEST list."""
    tasks = [M.Task(id="x", requester=M.PATCH_VERSION_REQUESTER, build_id="a-b", task_group="c", expected_duration=M.MINUTE),
             M.Task(id="y", requester=M.PATCH_VERSION_REQUESTER, build_id="a", task_group="b-c", expected_duration=M.MINUTE)]
    assert soa.marshal_legacy([("d", tasks, {})], None).list_mode.tolist() == [L.EVG_LEGACY_MODE_LITERAL] * 3
    assert soa.marshal_legacy([("d", tasks, {})], None, exact=True).list_mode.tolist() == [L.EVG_LEGACY_MODE_GO_STABLE] * 3
    tasks[1].build_id = "z"
    assert soa.marshal_legacy([("d", tasks, {})], None, exact=True).list_mode.tolist() == [L.EVG_LEGACY_MODE_INGEST] * 3
