"""FindNextTask without a GPU: every golden sequence of tests/golden/dag_find_next_task.json through the CPU restatement
(oracle_dispatch), the marshalling of a database snapshot and of TaskSpecs into evg_next_db / evg_next_req against
hand-written columns, and the new structs against the header."""
import copy
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from oracle import oracle_dispatch as OX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "dag_find_next_task.json")))
CASES = GOLDEN["cases"]
for _c in CASES:  # a case over a shared fixture gets its own copy of the items and the db
    if "fixture" in _c:
        _f = copy.deepcopy(GOLDEN["fixtures"][_c["fixture"]])
        _c["items"], _c["db"] = _f["items"], dict(_f["db"], **_c["db_extra"])


def merge(db, update):
    """update's keys set in db, dict values merged key by key (a step's db_update: the writes a test makes between requests)."""
    for k, v in update.items():
        if isinstance(v, dict) and isinstance(db.get(k), dict):
            merge(db[k], v)
        else:
            db[k] = copy.deepcopy(v)


def replay(case, serve, state, rebuild):
    """Every step of a golden case through serve(spec, ami, db) -> (id, outcome), with rebuild(items) where the case
    rebuilds; an asserted property is checked on the id serve returned; state() after the last step."""
    db = copy.deepcopy(case["db"])
    items = {it["id"]: it for it in case["items"]}
    last = {}
    for k, st in enumerate(case["steps"]):
        merge(db, st.get("db_update", {}))
        if "rebuild" in st:
            base = {it["id"]: it for it in case["items"]}
            queue = [dict(base[i], dependencies_met=met) for i, met in st["rebuild"]]
            rebuild(copy.deepcopy(queue))
            items = {it["id"]: it for it in queue}
        got, outcome = serve(st["spec"], st["ami"], db)
        prop = st.get("property")
        if prop is None:
            assert (got, outcome) == (st["expect"], st["outcome"]), (case["name"], k)
            continue
        assert got is not None and outcome == 1, (case["name"], k)
        for f in ("group", "build_variant", "version"):
            assert f not in prop or items[got].get(f, "") == prop[f], (case["name"], k, f)
        if "increasing" in prop:
            assert int(got) > last.get(prop["increasing"], 0), (case["name"], k)
            last[prop["increasing"]] = int(got)
    if "final" in case:
        node, unit, groups = state()
        assert (node, unit) == (case["final"]["node"], case["final"]["unit"]), case["name"]
        assert {g: [int(a), int(b)] for g, (a, b) in groups.items()} == case["final"]["groups"], case["name"]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_through_the_oracle(case):
    d = OX.Dispatcher(copy.deepcopy(case["items"]))
    replay(case, lambda spec, ami, db: (d.find_next_task(spec, ami, db), d.last_outcome), d.state, d.rebuild)


def test_golden_covers_every_trap_and_names_its_sources():
    names = " ".join(c["name"] for c in CASES)
    for k in range(1, 10):
        assert re.search(rf"trap[ 0-9and]*\b{k}\b", names), k
    assert all(c["source"] for c in CASES)
    whole = {c["name"] for c in CASES if not c["derived"]}
    assert {"TestFindNextTask", "TestNextTaskForDefaultTaskSpec", "TestSingleHostTaskGroupsBlock", "TestIntraTaskGroupDependencies",
            "TestOutsideTasksWithTaskGroupDependencies", "TestNewSingleHostTaskGroupLimits"} <= whole
    assert sum(len(c["steps"]) for c in CASES if c["name"] == "TestFindNextTask") == 100


def test_rebuild_resets_the_state():
    case = next(c for c in CASES if c["name"].startswith("trap 3"))
    d = OX.Dispatcher(copy.deepcopy(case["items"]))
    db = {"tasks": {"x": {"start": 0, "finish": 0, "status": "", "version": "", "est_generated": None, "ingest": 0, "deps_met": True}}}
    assert d.find_next_task(None, 0, db) == "x" and d.find_next_task(None, 0, db) is None and d.last_outcome == OX.GAVE_UP
    d.rebuild(copy.deepcopy(case["items"]))
    assert d.find_next_task(None, 0, db) == "x"


def test_marshal_snapshot_and_requests():
    Z = M.ZERO_TIME
    names = [["g_bv_p_v", "h_bv_p_v"], []]
    db = {"tasks": {"a": {"start": Z, "finish": Z, "status": "failed", "version": "v1", "est_generated": 3, "ingest": 77, "deps_met": True},
                    "b": {"start": 0, "finish": 9, "status": "failed", "version": "v2", "est_generated": None, "ingest": Z, "deps_met": None},
                    "c": {"start": 5, "finish": 9, "status": "success", "version": "gone", "ingest": 0, "deps_met": False}},
          "versions": {"v1": "s3", "v2": "db"}, "running_hosts": {"h_bv_p_v": -1}, "generate_limit": 7, "num_large_parser": -1}
    cols = S.marshal_next_db([["a", "b"], ["missing", "c"]], names, db)
    F = L.EVG_ND_FOUND
    assert cols["flags"].tolist() == [
        F | L.EVG_ND_STARTED_GROUP | L.EVG_ND_VERSION_FOUND | L.EVG_ND_VERSION_S3 | L.EVG_ND_DEPS_MET_NOW,  # Go's zero time: only :657 sees a start
        F | L.EVG_ND_FINISHED_NOT_SUCCEEDED | L.EVG_ND_VERSION_FOUND | L.EVG_ND_DEPS_ERR,                   # the epoch: not started either way
        0,
        F | L.EVG_ND_STARTED | L.EVG_ND_STARTED_GROUP]
    assert cols["est_generated"].tolist() == [3, 0, 0, 0] and cols["ingest_ns"].tolist() == [77, 0, 0, 0]
    assert cols["running_hosts"].tolist() == [0, -1]
    assert (cols["generate_limit"], cols["pending_generate"], cols["max_large_parser"], cols["num_large_parser"]) == (7, 0, 0, -1)
    spec = M.TaskSpec("h", "bv", "p", "v")
    req_off, group, ami = S.marshal_next_requests(names, [[(None, Z), (spec, 0), (M.TaskSpec("", "bv", "p", "v"), 12),
                                                            (M.TaskSpec("nope", "bv", "p", "v"), 12)], [(spec, 3)]])
    assert req_off.tolist() == [0, 4, 5] and group.tolist() == [-1, 1, -1, -1, -1] and ami.tolist() == [0, 0, 12, 12, 3]


def test_structs_match_the_header():
    src = open(os.path.join(ROOT, "include", "evg_sched.h")).read()
    for name, cls in (("evg_next_db", L.NextDbStruct), ("evg_next_req", L.NextReqStruct), ("evg_next_out", L.NextOutStruct),
                      ("evg_next_state", L.NextStateStruct), ("evg_next_dispatchers", L.NextDispatchersStruct)):
        body = re.search(r"typedef struct \{([^}]*)\} " + name + ";", src).group(1)
        fields = re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
        assert fields == [f for f, _ in cls._fields_], name
        for f, t in cls._fields_:
            decl = re.search(r"([\w \*]+?)\b" + f + ";", re.sub(r"/\*.*?\*/", "", body, flags=re.S)).group(1)
            assert C.sizeof(t) == (8 if "*" in decl or "int64_t" in decl else 4), (name, f)
    for macro in ("EVG_ND_FOUND", "EVG_ND_STARTED", "EVG_ND_STARTED_GROUP", "EVG_ND_FINISHED_NOT_SUCCEEDED", "EVG_ND_VERSION_FOUND",
                  "EVG_ND_VERSION_S3", "EVG_ND_DEPS_MET_NOW", "EVG_ND_DEPS_ERR", "EVG_NEXT_NONE", "EVG_NEXT_FOUND", "EVG_NEXT_GAVE_UP",
                  "EVG_NS_NODE", "EVG_NS_UNIT"):
        assert int(re.search(rf"#define {macro} (0x[0-9a-fA-F]+|\d+)", src).group(1), 0) == getattr(L, macro), macro
    assert (OX.EXHAUSTED, OX.FOUND, OX.GAVE_UP) == (L.EVG_NEXT_NONE, L.EVG_NEXT_FOUND, L.EVG_NEXT_GAVE_UP)
