"""The pipeline task finder without a GPU: the stage-by-stage oracle on the golden cases and against the legacy
finder on the reference's fuzzy fixture, the evg_pipeline_in marshalling, the returned-task view and the struct
layouts of include/evg_sched.h."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import golden_loader as G
import oracle_pipeline as OP
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIPELINE = G.load("task_finder_pipeline.json")


def pipeline_case(case):
    """-> (Distro, [candidate Task], [ProjectRef as the raw documents])."""
    d = M.Distro(id=case.get("distro_id", ""), valid_projects=list(case.get("valid_projects", [])),
                 dispatcher_settings=M.DispatcherSettings(version=case.get("dispatcher_version", "")))
    return d, [G.make_task(t, 0, 0) for t in case["tasks"]], [M.ProjectRef(**r) for r in case["project_refs"]]


def check_case(case, got):
    ids = [t.id for t in got]
    if "expect_len" in case:
        assert len(ids) == case["expect_len"]
    if "expect_ids" in case:
        assert ids == case["expect_ids"]
    for tid, want in case.get("expect_depends_on", {}).items():
        t = next(x for x in got if x.id == tid)
        assert [[x.task_id, x.status, x.unattainable] for x in t.depends_on] == want


@pytest.mark.parametrize("case", PIPELINE["cases"], ids=lambda c: c["name"])
def test_pipeline_oracle_golden(case):
    d, tasks, refs = pipeline_case(case)
    got = OP.find_runnable(d, tasks, refs)
    check_case(case, got)
    # the host view of the kept candidates is what the oracle decodes
    view = scheduler.pipeline_returned_tasks(d, [next(t for t in tasks if t.id == g.id) for g in got])
    assert [(t.id, [(x.task_id, x.status, x.unattainable) for x in t.depends_on]) for t in view] == \
        [(t.id, [(x.task_id, x.status, x.unattainable) for x in t.depends_on]) for t in got]


def test_pipeline_differs_from_legacy_where_the_golden_file_says():
    """The derived cases are exactly where the legacy finder gives another answer (the reference's own cases agree)."""
    for case in PIPELINE["cases"]:
        d, tasks, refs = pipeline_case(case)
        pipe = [t.id for t in OP.find_runnable(d, tasks, refs)]
        legacy = [t.id for t in O.find_runnable(d, tasks, refs, finder="legacy")]
        if case["kind"] == "asserted":
            assert pipe == legacy, case["name"]
        elif case["name"].startswith("derived/returned"):
            continue
        else:
            assert pipe != legacy, case["name"]


@pytest.mark.parametrize("seed", range(20))
def test_pipeline_and_legacy_agree_on_fuzzy_tasks(seed):
    """TaskFinderComparisonSuite.TestFindRunnableHostsIsIdentical (task_finder_test.go:309-334) for the pipeline."""
    tasks = G.random_finder_tasks(random.Random(seed))
    refs = [M.ProjectRef(**r) for r in G.load("task_finder.json")["cases"][-1]["project_refs"]]
    a = sorted(t.id for t in O.find_runnable(M.Distro(), tasks, refs, finder="legacy"))
    b = sorted(t.id for t in OP.find_runnable(M.Distro(), tasks, refs))
    assert a == b


def test_marshal_runnable_pipeline_bits():
    refs = [M.ProjectRef(id="p", enabled=True), M.ProjectRef(id="q", enabled=False, dispatching_disabled=True,
                                                             patching_disabled=False),
            M.ProjectRef(id="r", enabled=True, patching_disabled=True, dispatching_disabled=False)]
    db = {"x": M.Task(id="x", status="started", depends_on=[M.Dependency("y", unattainable=True)]),
          "z": M.Task(id="z", status=M.TASK_FAILED)}
    d0 = M.Distro(id="d0")
    d1 = M.Distro(id="d1", dispatcher_settings=M.DispatcherSettings(version=M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
    a = M.Task(id="a", project="p", depends_on=[M.Dependency("b", "*"), M.Dependency("x", ""), M.Dependency("gone", "weird")])
    b = M.Task(id="b", project="q", status="", depends_on=[M.Dependency("z", M.TASK_FAILED, unattainable=True)])
    c = M.Task(id="c", project="r", status=M.TASK_SUCCEEDED, depends_on=[M.Dependency("x", M.TASK_SUCCEEDED)])
    table = S.marshal_runnable([(d0, [a, b]), (d1, [c])], refs, finder="pipeline", dependency_db=db)
    assert table.finder.tolist() == [L.EVG_FINDER_PIPELINE, L.EVG_FINDER_PIPELINE_NO_DEPS]
    assert table.deps is not None and table.deps.dep_kind.tolist() == [L.EVG_DEP_IN_QUEUE, L.EVG_DEP_EXTERNAL, L.EVG_DEP_MISSING,
                                                                        L.EVG_DEP_EXTERNAL, L.EVG_DEP_EXTERNAL]
    p = table.pipe
    # the reserved ids, then first appearance in marshalling order: "undispatched" 3 (a), "" 4 (a's entry on x),
    # "started" 5 (x, the first external document), "weird" 6 (the entry on a missing task)
    assert p.n_status == 7
    assert p.task_status.tolist() == [3, 4, L.EVG_STATUS_SUCCESS]
    assert p.dep_status.tolist() == [L.EVG_STATUS_ANY, 4, 6, L.EVG_STATUS_FAILED, L.EVG_STATUS_SUCCESS]
    assert p.ext_status.tolist() == [5, L.EVG_STATUS_FAILED]
    assert p.task_unattainable.tolist() == [0, 1, 0]  # b's own entry is unattainable
    assert p.ext_unattainable.tolist() == [1, 0]      # x has an unattainable entry, z none
    assert p.project_raw.tolist() == [L.EVG_PR_ENABLED, L.EVG_PR_DISPATCHING_DISABLED | L.EVG_PR_PATCHING_FALSE,
                                      L.EVG_PR_ENABLED]
    # the other finders marshal as before
    legacy = S.marshal_runnable([(d0, [a, b]), (d1, [c])], refs, finder="legacy", dependency_db=db)
    assert legacy.pipe is None and legacy.finder.tolist() == [L.EVG_FINDER_LEGACY, L.EVG_FINDER_NO_DEPS]


def test_get_task_finder_maps_every_name():
    assert scheduler.GetTaskFinder("legacy") is scheduler.LegacyFindRunnableTasks
    assert scheduler.GetTaskFinder("alternate") is scheduler.AlternateTaskFinder
    assert scheduler.GetTaskFinder("parallel") is scheduler.ParallelTaskFinder
    assert scheduler.GetTaskFinder("pipeline") is scheduler.RunnableTasksPipeline
    assert scheduler.GetTaskFinder("") is scheduler.LegacyFindRunnableTasks
    assert scheduler.GetTaskFinder("nonsense") is scheduler.LegacyFindRunnableTasks


def test_struct_layouts_match_the_header(tmp_path):
    c = tmp_path / "layout.c"
    c.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(evg_pipeline_in), offsetof(evg_pipeline_in, dep_status),
         offsetof(evg_pipeline_in, task_status), offsetof(evg_pipeline_in, ext_status),
         offsetof(evg_pipeline_in, task_unattainable), offsetof(evg_pipeline_in, ext_unattainable),
         offsetof(evg_pipeline_in, project_raw), sizeof(evg_runnable_in));
  printf("%d %d %d %d %d %d %d %d\\n", EVG_FINDER_PIPELINE, EVG_FINDER_PIPELINE_NO_DEPS, EVG_STATUS_SUCCESS, EVG_STATUS_FAILED,
         EVG_STATUS_ANY, EVG_PR_ENABLED, EVG_PR_DISPATCHING_DISABLED, EVG_PR_PATCHING_FALSE);
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    lines = subprocess.check_output([str(exe)], text=True).split("\n")
    S_ = L.PipelineInStruct
    assert [int(x) for x in lines[0].split()] == [
        ctypes.sizeof(S_), S_.dep_status.offset, S_.task_status.offset, S_.ext_status.offset, S_.task_unattainable.offset,
        S_.ext_unattainable.offset, S_.project_raw.offset, ctypes.sizeof(L.RunnableInStruct)]
    assert [int(x) for x in lines[1].split()] == [
        L.EVG_FINDER_PIPELINE, L.EVG_FINDER_PIPELINE_NO_DEPS, L.EVG_STATUS_SUCCESS, L.EVG_STATUS_FAILED, L.EVG_STATUS_ANY,
        L.EVG_PR_ENABLED, L.EVG_PR_DISPATCHING_DISABLED, L.EVG_PR_PATCHING_FALSE]


def test_pipeline_table_struct_pointers():
    p = S.PipelineTable(3, np.zeros(0, np.int32), np.zeros(2, np.int32), np.zeros(0, np.int32), np.zeros(2, np.uint8),
                        np.zeros(0, np.uint8), np.zeros(1, np.uint8))
    s = p.struct()
    assert s.n_status == 3 and s.dep_status is None and s.ext_status is None and s.task_status and s.project_raw
