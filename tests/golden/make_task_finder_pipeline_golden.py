#!/usr/bin/env python3
"""Write tests/golden/task_finder_pipeline.json: what the pipeline task finder (RunnableTasksPipeline ->
task.FindHostRunnable, scheduler/task_finder.go:34-36, model/task/db.go:887-1066) returns, transcribed by hand -- the Go
tests insert into MongoDB and cannot run here.

`asserted` cases are the TaskFinderSuite tests as TestDBTaskFinder runs them (scheduler/task_finder_test.go:41-47:
FindHostRunnable(ctx, d.Id, true)), with the exact expectation of the Go test.  The suite's distro has the id "", so the
aggregation never reads a distro document and skips filterInvalidDistros (db.go:893-903,1050-1052): ValidProjects
plays no part, and "other-project" still gives 3 because tasks 0 and 1 name a project without a project_ref.

`derived` cases are not asserted by any Go test: each follows from the aggregation and the mgo decoder at the lines
given in `ref`.  `expect_ids` are in candidate order (the library's canonical order; $group leaves it unspecified).
`expect_depends_on` gives, per returned id, DependsOn as the decoded task holds it: [task_id, status, unattainable].

Task / project-ref dicts use the field names of evergreen_b200.model; Go zero values apply to omitted fields.  A
project ref's omitted `dispatching_disabled` / `patching_disabled` are unset *bool fields (absent from the document).
"""
import json
import os

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "task_finder_pipeline.json")
F = "scheduler/task_finder_test.go"
DB = "model/task/db.go"
UND, OK, FAIL = "undispatched", "success", "failed"


def base_tasks():  # SetupTest :70-95
    ts = [dict(id=f"t{i}", status=UND, activated=True, project="exists") for i in range(6)]
    ts[5]["priority"] = -1
    return ts


def go_task(**kw):
    d = dict(status="", activated=False)
    d.update(kw)
    return d


def ready(**kw):  # a schedulable task of project "p"
    d = dict(status=UND, activated=True, project="p")
    d.update(kw)
    return d


refs_enabled = [dict(id="exists", enabled=True)]
deps = [go_task(id="td1"), go_task(id="td2")]
cases = []

# ---- TaskFinderSuite under TestDBTaskFinder
cases.append(dict(name="NoRunnableTasksReturnsEmptySlice", ref=f"{F}:113-118", kind="asserted",
                  tasks=[], project_refs=refs_enabled, expect_len=0))
t = base_tasks(); t[4]["activated"] = False
cases.append(dict(name="InactiveTasksNeverReturned", ref=f"{F}:120-129", kind="asserted",
                  tasks=t + deps, project_refs=refs_enabled, expect_len=4))
cases.append(dict(name="FilterTasksWhenValidProjectsSet/default", ref=f"{F}:131-136", kind="asserted",
                  tasks=base_tasks() + deps, project_refs=refs_enabled, expect_len=5))
cases.append(dict(name="FilterTasksWhenValidProjectsSet/listed", ref=f"{F}:138-146 ({DB}:893-903: distro id \"\")",
                  kind="asserted", tasks=base_tasks() + deps, project_refs=refs_enabled, valid_projects=[], expect_len=5))
t = base_tasks(); t[0]["project"] = "something_else"; t[1]["project"] = "something_else"
cases.append(dict(name="FilterTasksWhenValidProjectsSet/other-project", ref=f"{F}:148-156 (distro document cleared)",
                  kind="asserted", tasks=t + deps, project_refs=refs_enabled, valid_projects=[], expect_len=3,
                  expect_ids=["t2", "t3", "t4"]))
t = base_tasks()
td1 = go_task(id="td1", status=FAIL)
td2 = go_task(id="td2", status=UND, depends_on=[dict(task_id="none", status="*", unattainable=True)])
t[0]["depends_on"] = [dict(task_id="td1", status=FAIL)]
t[1]["depends_on"] = [dict(task_id="td1", status=OK)]
t[2]["depends_on"] = [dict(task_id="td2", status="*"), dict(task_id="td1", status="*")]
t[3]["depends_on"] = [dict(task_id="td1", status="*")]
cases.append(dict(name="TasksWithUnsatisfiedDependenciesNeverReturned", ref=f"{F}:159-191", kind="asserted",
                  tasks=t + [td1, td2], project_refs=refs_enabled, expect_len=4, expect_ids=["t0", "t2", "t3", "t4"]))
cases.append(dict(name="TasksWithDisabledProjectNeverReturned", ref=f"{F}:193-202", kind="asserted",
                  tasks=[], project_refs=[dict(id="exists", enabled=False)], expect_len=0))
cases.append(dict(name="TasksWithProjectDispatchingDisabledNeverReturned", ref=f"{F}:204-213", kind="asserted",
                  tasks=[], project_refs=[dict(id="exists", dispatching_disabled=True)], expect_len=0))

# ---- item 3: gating by the raw project_ref document
gate_refs = [dict(id="p", enabled=True), dict(id="hidden", enabled=False, hidden=True),
             dict(id="patch-false", enabled=True, patching_disabled=False),
             dict(id="dispatch-false", enabled=True, dispatching_disabled=False)]
cases.append(dict(
    name="derived/raw-project-gating", kind="derived",
    ref=f"{DB}:998-1048 (filterDisabledProjects, filterPatchingDisabledProjects); model/project_ref.go:52-59 (omitempty)",
    note="a patch / PR / merge-queue task of a project that never set patching_disabled is dropped; a hidden project "
         "gives a PR task no exemption; patching_disabled stored false admits patches; dispatching_disabled stored "
         "false does not block",
    tasks=[ready(id="mainline", requester="gitter_request"), ready(id="patch", requester="patch_request"),
           ready(id="pr", requester="github_pull_request"), ready(id="mq", requester="github_merge_request"),
           ready(id="hidden-pr", project="hidden", requester="github_pull_request"),
           ready(id="patch-ok", project="patch-false", requester="patch_request"),
           ready(id="dispatch-ok", project="dispatch-false"), ready(id="no-ref", project="nowhere")],
    project_refs=gate_refs, expect_ids=["mainline", "patch-ok", "dispatch-ok"]))

# ---- item 5: the satisfied_dependencies expression
cases.append(dict(
    name="derived/status-compare", kind="derived",
    ref=f"{DB}:967-987 (projectSatisfied)",
    note="statuses compare exactly (\"\" is not \"success\"); \"*\" accepts success / failed or a dependency with an "
         "unattainable depends_on entry, whatever its OverrideDependencies",
    tasks=[ready(id="empty-want-success-dep", depends_on=[dict(task_id="ds", status="")]),
           ready(id="empty-want-empty-dep", depends_on=[dict(task_id="de", status="")]),
           ready(id="star-overridden-blocked", depends_on=[dict(task_id="dob", status="*")]),
           ready(id="star-started", depends_on=[dict(task_id="dst", status="*")]),
           ready(id="other-status", depends_on=[dict(task_id="dst", status="started")]),
           go_task(id="ds", status=OK), go_task(id="de", status=""),
           go_task(id="dob", status="started", override_dependencies=True,
                   depends_on=[dict(task_id="gone", status=OK, unattainable=True)]),
           go_task(id="dst", status="started")],
    project_refs=[dict(id="p", enabled=True)],
    expect_ids=["empty-want-empty-dep", "star-overridden-blocked", "other-status"]))

# ---- item 6: which entries count
cases.append(dict(
    name="derived/missing-targets", kind="derived",
    ref=f"{DB}:923-960,989-996 ($graphLookup, the two $unwinds, matchIds, $group / $redact)",
    note="an entry without a document is ignored; a task whose entries all lack one is dropped; a task without "
         "DependsOn is kept; DependenciesMetTime and OverrideDependencies do not help",
    tasks=[ready(id="one-missing", depends_on=[dict(task_id="d-ok", status=OK), dict(task_id="ghost", status=OK)]),
           ready(id="all-missing", depends_on=[dict(task_id="ghost", status=OK), dict(task_id="ghost2", status=OK)]),
           ready(id="no-deps"),
           ready(id="met-time-unmet", dependencies_met_time=5, depends_on=[dict(task_id="d-fail", status=OK)]),
           ready(id="override-unmet", override_dependencies=True, depends_on=[dict(task_id="d-fail", status=OK)]),
           go_task(id="d-ok", status=OK), go_task(id="d-fail", status=FAIL)],
    project_refs=[dict(id="p", enabled=True)], expect_ids=["one-missing", "no-deps"]))

# ---- item 8: what the planner receives with removeDeps
cases.append(dict(
    name="derived/returned-depends-on-removeDeps", kind="derived",
    ref=f"{DB}:975-996 ($first: $$ROOT after $unwind); db/mgo/bson/decode.go:202,503-528",
    note="the returned task's depends_on is one sub-document, which mgo skips: DependsOn decodes empty",
    tasks=[ready(id="a", depends_on=[dict(task_id="d1", status=OK), dict(task_id="d2", status=FAIL)]), ready(id="b"),
           go_task(id="d1", status=OK), go_task(id="d2", status=FAIL)],
    project_refs=[dict(id="p", enabled=True)], expect_ids=["a", "b"], expect_depends_on={"a": [], "b": []}))

# ---- item 9: without removeDeps
cases.append(dict(
    name="derived/returned-depends-on-revised-with-dependencies", kind="derived",
    dispatcher_version="revised-with-dependencies",
    ref=f"{DB}:916-921 (removeFields), 1041-1051 (no dependency filter); scheduler/scheduler.go:61-64",
    note="no dependency filter; every returned task loses depends_on.unattainable, so a \"*\" dependency on a returned "
         "task never sees it blocked",
    tasks=[ready(id="up", status=UND, depends_on=[dict(task_id="gone", status=OK, unattainable=True)]),
           ready(id="down", depends_on=[dict(task_id="up", status="*")]),
           ready(id="unmet", depends_on=[dict(task_id="d-fail", status=OK)]),
           go_task(id="d-fail", status=FAIL)],
    project_refs=[dict(id="p", enabled=True)], expect_ids=["up", "down", "unmet"],
    expect_depends_on={"up": [["gone", OK, False]], "down": [["up", "*", False]], "unmet": [["d-fail", OK, False]]}))

json.dump(dict(source=F, cases=cases), open(OUT, "w"), indent=1)
print("wrote", OUT, len(cases), "cases")
