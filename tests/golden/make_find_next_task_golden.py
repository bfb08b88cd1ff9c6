"""Writes dag_find_next_task.json: request sequences for the DAG dispatcher's FindNextTask with the id (or nil) and the
outcome each request must return.  Data only.  Expected values are written by hand from the reference's code and tests
(model/task_queue_service_dependency.go:258-698, model/task_queue_service_test.go); nothing here runs an implementation.

Case layout: `fixture` names shared items and db under "fixtures" (`db_extra` is merged into that db); otherwise items (TaskQueueItem fields; omitted fields are Go zero values), db (the snapshot, see
oracle/oracle_dispatch.py), steps: each {"spec": TaskSpec fields or null, "ami": amiUpdatedTime ns (0 = zero time),
"db_update": merged key by key into db before the request (the reference's tests write to the database between
requests), "rebuild": the items service.rebuild() is called with before the request, as [id, DependenciesMet] pairs over the case's
items (refreshTaskQueue, :2026-2061: the tasks whose status is not a completed one, in insertion order, DependenciesMet =
Task.HasDependenciesMet after Task.DependenciesMet), "expect": item id or null, "outcome": 1 found / 0 the walk ended / 2 nil on a database miss;
where the reference test asserts a property instead of an id, "property": {"group", "build_variant", "version": the
returned item's fields, "not_nil": true, "increasing": a label -- the id as an integer exceeds that of the previous
step with the same label}}, and (optional) `final`: the state after the last step -- node and unit IsDispatched bits
per item, {group: [deleted, cached runningHosts]}.
`derived`: true for a case no reference test reaches or one cut down from a reference test, false for a reference test
transcribed whole.  Settings the reference's test environment leaves at their defaults are taken as 0 (no generate
limit; no large-parser limit unless the test sets one)."""
import json
import os

G = {"group": "g", "build_variant": "bv", "project": "p", "version": "v"}
GID = "g_bv_p_v"


def item(i, **kw):
    return dict({"id": i, "dependencies_met": True}, **kw)


def doc(**kw):
    return dict({"start": 0, "finish": 0, "status": "undispatched", "version": "v", "est_generated": None, "ingest": 0,
                 "deps_met": True}, **kw)


def step(expect, outcome=None, spec=None, ami=0, **kw):
    return dict({"spec": spec, "ami": ami, "expect": expect, "outcome": (1 if expect is not None else 0) if outcome is None else outcome}, **kw)


CASES = [
    {"name": "TestSingleHostTaskGroupsBlock", "source": "model/task_queue_service_test.go:1205-1258", "derived": False,
     # five items of one single-host group, DependenciesMet false as the test leaves it; task 0 finished and succeeded
     # (started: skipped), task 1 finished and failed: the unit is deleted and the request returns nil (:652-655)
     "items": [dict(G, id=str(i), group_max_hosts=1) for i in range(5)],
     "db": {"tasks": {"0": doc(start=880, finish=940, status="success"), "1": doc(start=940, finish=1000, status="failed"),
                      "2": doc(status=""), "3": doc(status=""), "4": doc(status="")}},
     "steps": [step(None, spec=G)],
     "final": {"node": [0] * 5, "unit": [0] * 5, "groups": {GID: [1, 0]}}},
    {"name": "after TestFindNextTaskForOutdatedHostAMI: the group path has no AMI rule", "source": "model/task_queue_service_test.go:1539-1593",
     "derived": True,
     # cut down to two tasks shaped like the ones the test inserts, and with the task-group task ALSO ingested after the
     # AMI update (the test's is ingested before): the standalone task is skipped (:392), the task-group task is handed
     # out because nothing on the group path compares its ingest time
     "items": [item("1"), item("2", group="e2e_core_task_group", build_variant="e2e_openshift_cloud_qa", project="ops-manager-kubernetes",
                               version="5d88953e2a60ed61eefe9561", group_max_hosts=5, group_index=2)],
     "db": {"tasks": {"1": doc(ingest=1060), "2": doc(ingest=1500)}},
     "steps": [step("2", ami=1000)],
     "final": {"node": [1, 1], "unit": [0, 1],
               "groups": {"e2e_core_task_group_e2e_openshift_cloud_qa_ops-manager-kubernetes_5d88953e2a60ed61eefe9561": [1, 0]}}},
    {"name": "trap 1 and 2: the branch is GroupMaxHosts, and an item has two IsDispatched copies", "source": ":305, :172-183, :496, :515, :681",
     "derived": True,
     # queue c, b, a; c depends on a, so d.sorted = b, a, c.  b has GroupMaxHosts 2 and no group: group path, no unit,
     # skipped.  a has a group and GroupMaxHosts 0: standalone path, which sets only the node's bit -- the unit's copy of
     # a stays clear and the unit hands a out again.
     "items": [item("c", **G, group_max_hosts=2, dependencies=["a"]), item("b", group_max_hosts=2), item("a", **G, group_max_hosts=0)],
     "db": {"tasks": {"a": doc(), "b": doc(), "c": doc()}},
     "steps": [step("a"), step("c"), step("a"), step(None)],
     "final": {"node": [1, 0, 1], "unit": [1, 0, 1], "groups": {GID: [1, 0]}}},
    {"name": "trap 3: marked before any database check", "source": ":309, :334", "derived": True,
     "items": [item("x"), item("y")],
     "db": {"tasks": {"x": doc(start=5), "y": doc()}},
     "steps": [step("y"), step(None, db_update={"tasks": {"x": doc(), "y": doc()}})],
     "final": {"node": [1, 1], "unit": [0, 0], "groups": {}}},
    {"name": "trap 4: skip and give up differ", "source": ":321-331, :365-371, :549-603", "derived": True,
     # w has no document: nil for the request.  x's version is missing: nil.  z's version is in S3 and the limit is
     # reached: skipped.  y's version is not in S3: handed out.
     "items": [item("w"), item("x"), item("z"), item("y")],
     "db": {"tasks": {"x": doc(version="vx"), "z": doc(version="vz"), "y": doc(version="vy")}, "versions": {"vz": "s3", "vy": "db"},
            "max_large_parser": 1, "num_large_parser": 5},
     "steps": [step(None, 2), step(None, 2), step("y"), step(None)],
     "final": {"node": [1, 1, 1, 1], "unit": [0, 0, 0, 0], "groups": {}}},
    {"name": "trap 5: runningHosts is cached once it reaches maxHosts", "source": ":411-427", "derived": True,
     "items": [item("g1", **G, group_max_hosts=1), item("g2", **G, group_max_hosts=1, group_index=1), item("s")],
     "db": {"tasks": {"g1": doc(), "g2": doc(), "s": doc()}, "running_hosts": {GID: 1}},
     "steps": [step("s"), step(None, db_update={"running_hosts": {GID: 0}})],
     "final": {"node": [0, 0, 1], "unit": [0, 0, 0], "groups": {GID: [0, 1]}}},
    {"name": "trap 5: a failed host count gives up", "source": ":413-425", "derived": True,
     "items": [item("g1", **G, group_max_hosts=1), item("s")],
     "db": {"tasks": {"g1": doc(), "s": doc()}, "running_hosts": {GID: -1}},
     "steps": [step(None, 2)],
     "final": {"node": [0, 0], "unit": [0, 0], "groups": {GID: [0, 0]}}},
    {"name": "trap 6: the unit is deleted at its last position", "source": ":684-686", "derived": True,
     # g1 has started and is skipped, g2 sits at the last position: handing it out deletes the unit with g1 never handed out
     "items": [item("g1", **G, group_max_hosts=2), item("g2", **G, group_max_hosts=2, group_index=1)],
     "db": {"tasks": {"g1": doc(start=5), "g2": doc()}},
     "steps": [step("g2", spec=G), step(None, spec=G)],
     "final": {"node": [0, 1], "unit": [0, 1], "groups": {GID: [1, 0]}}},
    {"name": "trap 7: the spec path checks neither runningHosts nor the AMI", "source": ":268-282", "derived": True,
     "items": [item("g1", **G, group_max_hosts=1), item("g2", **G, group_max_hosts=1, group_index=1)],
     "db": {"tasks": {"g1": doc(ingest=100), "g2": doc(ingest=100)}, "running_hosts": {GID: 5}},
     "steps": [step("g1", spec=G, ami=50), step(None, ami=50)],
     "final": {"node": [1, 0], "unit": [1, 0], "groups": {GID: [0, 5]}}},
    {"name": "trap 8: pending + estimated >= limit, both positive; After is strict", "source": ":341-363, :392", "derived": True,
     # x: 4 + 6 >= 10 skipped.  n: nil estimate, no rule.  e: ingested exactly at the AMI update: not After, handed out.
     "items": [item("x"), item("y"), item("n"), item("e")],
     "db": {"tasks": {"x": doc(est_generated=6), "y": doc(est_generated=5), "n": doc(), "e": doc(ingest=70)},
            "generate_limit": 10, "pending_generate": 4},
     "steps": [step("y"), step("n"), step("e", ami=70), step(None)],
     "final": {"node": [1, 1, 1, 1], "unit": [0, 0, 0, 0], "groups": {}}},
    {"name": "trap 8: a failed pending count skips, a limit of 0 disables the rule", "source": ":341-352", "derived": True,
     "items": [item("x"), item("y")],
     "db": {"tasks": {"x": doc(est_generated=6), "y": doc()}, "generate_limit": 10, "pending_generate": -1},
     "steps": [step("y"), step(None)],
     "final": {"node": [1, 1], "unit": [0, 0], "groups": {}}},
    {"name": "trap 9: a dependency cycle's placeholder is skipped", "source": ":290-292", "derived": True,
     "items": [item("a", dependencies=["b"]), item("b", dependencies=["a"]), item("c")],
     "db": {"tasks": {"a": doc(), "b": doc(), "c": doc()}},
     "steps": [step("c"), step(None)],
     "final": {"node": [0, 0, 1], "unit": [0, 0, 0], "groups": {}}},
    {"name": "the two zero-time tests", "source": ":334, :657", "derived": True,
     # Go's zero StartTime (-2^63 here): not started for the standalone path, started for nextTaskGroupTask
     "items": [item("g1", **G, group_max_hosts=2), item("s")],
     "db": {"tasks": {"g1": doc(start=-(2 ** 63)), "s": doc(start=-(2 ** 63))}},
     "steps": [step("s"), step(None)],
     "final": {"node": [0, 1], "unit": [0, 0], "groups": {GID: [0, 0]}}},
]

# ---- the reference's suite over SetupTest's fixture (model/task_queue_service_test.go:409-527)
V1, V2 = "version_1", "version_2"
SHAPES = [("", "variant_1", V1, 0), ("group_1", "variant_1", V1, 1), ("group_2", "variant_1", V1, 2), ("group_1", "variant_2", V1, 2),
          ("group_1", "variant_1", V2, 2)]
VERSIONS = {V1: "s3", V2: "", "5d8cd23da4cf4747f4210333": "", "5d88953e2a60ed61eefe9561": "", "version": "", "": ""}


def setup_deps(i):  # :428-439
    return [str(i + 5)] if i % 5 == 0 and (30 < i < 50 or 60 < i < 80) else []


def setup_items(done=()):
    """refreshTaskQueue over SetupTest's tasks once the ids in `done` have succeeded."""
    out = []
    for i in range(100):
        if str(i) in done:
            continue
        g, bv, v, mh = SHAPES[i % 5]
        out.append({"id": str(i), "group": g, "build_variant": bv, "version": v, "project": "project_1", "group_max_hosts": mh,
                    "dependencies": setup_deps(i), "dependencies_met": all(d in done for d in setup_deps(i))})
    return out


def setup_db(**kw):
    return dict({"tasks": {str(i): doc(status="", version=SHAPES[i % 5][2], deps_met=not setup_deps(i)) for i in range(100)},
                 "versions": VERSIONS}, **kw)


def spec_of(k):
    g, bv, v, _ = SHAPES[k]
    return {"group": g, "build_variant": bv, "version": v, "project": "project_1"}


def succeeded(i):
    return {"tasks": {i: {"status": "success"}}}


def find_next_task_steps():  # :1357-1537
    steps, prev = [], None

    def add(st):
        nonlocal prev
        if prev is not None:
            st["db_update"] = succeeded(prev)  # setTaskStatus(next.Id, TaskSucceeded) after every request
        steps.append(st)
        prev = st["expect"]
    for k, first in ((1, 1), (2, 2), (3, 3), (4, 4), (1, 26)):  # :1366-1433: five per unit through the TaskSpec
        for i in range(5):
            add(step(str(5 * i + first), spec=spec_of(k)))
    add(step("0"))  # :1446-1450
    # :1459-1525 assert the unit and increasing ids; the ids are the ones the test's comments list
    for k, ids in ((1, range(51, 100, 5)), (2, range(27, 100, 5)), (3, range(28, 100, 5)), (4, range(29, 100, 5))):
        for i in ids:
            g, bv, v, _ = SHAPES[k]
            st = step(str(i))
            st["property"] = {"group": g, "build_variant": bv, "version": v, "increasing": f"unit {k}"}
            add(st)
    done = {str(i) for i in range(100) if i % 5} | {"0"}
    for n, i in enumerate(["5", "10", "15", "20", "25", "30", "50", "45", "40", "35", "55", "60", "80", "75", "70", "65", "85", "90", "95"]):  # :1529
        st = step(i)
        add(st)
        if n:  # :1535 refreshTaskQueue after every one of these requests: a rebuild without the succeeded tasks
            st["rebuild"] = setup_items(done)
            st["db_update"]["tasks"].update({it["id"]: {"deps_met": True} for it in st["rebuild"]
                                             if it["dependencies_met"] and it["dependencies"]})  # Task.DependenciesMet now holds
        done.add(i)
    return steps


TG = {"group": "tg_compile_and_test", "build_variant": "archlinux", "version": "5d8cd23da4cf4747f4210333", "project": "genny", "group_max_hosts": 1}


def outside(i, order, met=True):
    return dict(TG, id=f"taskgroup_task{i}", group_index=order, dependencies=[], dependencies_met=met)


EXT5 = {"id": "external_task5", "build_variant": "archlinux", "version": V1, "project": "project_1", "dependencies": ["taskgroup_task3"]}


def intra(done):
    deps = {"task1": ["task2", "task4", "task3"], "task2": [], "task3": ["task2", "task4"], "task4": ["task2"]}
    return [dict(TG, id=t, dependencies=d, dependencies_met=all(x in done for x in d)) for t, d in deps.items() if t not in done]


def intra_update(done):
    return {"tasks": dict({t: {"status": "success"} for t in done}, **{it["id"]: {"deps_met": it["dependencies_met"]} for it in intra(done)})}


G1 = {"group": "group_1", "build_variant": "variant_1", "version": V1, "project": "project_1", "group_max_hosts": 1}
G1ID = "group_1_variant_1_project_1_version_1"
CASES += [
    {"name": "TestFindNextTask", "source": "model/task_queue_service_test.go:1357-1537 over SetupTest :409-527", "derived": False,
     "items": setup_items(), "db": setup_db(), "steps": find_next_task_steps()},
    {"name": "TestNextTaskForDefaultTaskSpec", "source": "model/task_queue_service_test.go:883-964", "derived": False,
     "items": setup_items(), "db": setup_db(),
     "steps": [step("0")] + [step(str(i)) for i in range(1, 100, 5)] + [step("2"), step("7"), step("12")]},
    {"name": "TestTaskGroupTasksRunningHostsVersusMaxHosts", "source": "model/task_queue_service_test.go:1595-1636", "derived": False,
     # one running host whose last task group is group_1_variant_1_project_1_version_1 (maxHosts 1)
     "items": setup_items(), "db": setup_db(running_hosts={G1ID: 1}), "steps": [step("0"), step("2"), step("7")]},
    {"name": "TestOutsideTasksWithTaskGroupDependencies", "source": "model/task_queue_service_test.go:37-192", "derived": False,
     "items": [outside(1, 4), outside(2, 1), outside(3, 3), outside(4, 2), dict(EXT5, dependencies_met=False)],
     "db": {"tasks": dict({f"taskgroup_task{i}": doc(version=TG["version"]) for i in (1, 2, 3, 4)}, external_task5=doc(version=V1, deps_met=False)),
            "versions": VERSIONS},
     "steps": [step("taskgroup_task2"), step("taskgroup_task4"), step("taskgroup_task3"),
               # :168-174: the collection holds t1, t3 (succeeded) and t5; the refresh queues t1 and t5
               step("taskgroup_task1", rebuild=[outside(1, 4), dict(EXT5, dependencies_met=True)],
                    db_update={"tasks": {"taskgroup_task3": {"status": "success"}, "external_task5": {"deps_met": True}}}),
               step("external_task5"), step(None), step(None), step(None)]},
    {"name": "TestIntraTaskGroupDependencies", "source": "model/task_queue_service_test.go:194-407", "derived": False,
     "items": intra(()), "db": {"tasks": {it["id"]: doc(version=TG["version"], deps_met=it["dependencies_met"]) for it in intra(())},
                                "versions": VERSIONS},
     "steps": [step("task2"), step(None), step(None), step(None),
               step("task4", rebuild=intra({"task2"}), db_update=intra_update({"task2"})), step(None), step(None),
               step("task3", rebuild=intra({"task2", "task4"}), db_update=intra_update({"task2", "task4"})), step(None),
               step("task1", rebuild=intra({"task2", "task3", "task4"}), db_update=intra_update({"task2", "task3", "task4"})), step(None)]},
    {"name": "TestSelfEdge", "source": "model/task_queue_service_test.go:659-684", "derived": False,
     "items": [{"id": "t0", "dependencies": ["t0"]}], "db": {"tasks": {"t0": doc(start=-(2 ** 63), finish=-(2 ** 63), deps_met=False)}},
     "steps": [step(None)]},
    {"name": "TestDependencyCycle", "source": "model/task_queue_service_test.go:686-714", "derived": False,
     # StartTime is not set: Go's zero time, which !utility.IsZeroTime (:334) reads as not started
     "items": [{"id": "t0", "dependencies": ["t1"]}, {"id": "t1", "dependencies": ["t0"]}, {"id": "t2", "dependencies_met": True}],
     "db": {"tasks": {"t0": doc(start=-(2 ** 63), deps_met=False), "t1": doc(start=-(2 ** 63), deps_met=False), "t2": doc(start=-(2 ** 63))}},
     "steps": [step("t2")]},
    {"name": "TestSingleHostTaskGroupOrdering", "source": "model/task_queue_service_test.go:1745-1801", "derived": False,
     "items": [dict(G1, id=str(i), group_index=gi, dependencies_met=True) for i, gi in enumerate([2, 0, 4, 1, 3])],
     "db": {"tasks": {str(i): doc(status="", version=V1) for i in range(5)}, "versions": VERSIONS},
     "steps": [step(i, spec=G1) for i in ["1", "3", "0", "4", "2"]]},
    {"name": "TestInProgressSingleHostTaskGroupLimits", "source": "model/task_queue_service_test.go:1803-1853", "derived": False,
     # degraded mode with a limit of 1, one started task of an S3 version counted: the TaskSpec path has no parser check
     "items": [{"id": "sample_s3_task", "version": V1, "project": "project_1", "dependencies_met": True}] +
              [dict(G1, id=str(i), dependencies_met=True) for i in range(5)],
     "db": {"tasks": dict({str(i): doc(status="", version=V1) for i in range(5)}, sample_s3_task=doc(status="started", version=V1, start=-(2 ** 63))),
            "versions": VERSIONS, "max_large_parser": 1, "num_large_parser": 1},
     "steps": [dict(step(str(i), spec=G1), property={"not_nil": True}) for i in range(5)]},
    {"name": "TestNewSingleHostTaskGroupLimits", "source": "model/task_queue_service_test.go:1855-1903", "derived": False,
     # the same fixture through the walk: every task is marked and then skipped by the parser limit (:365-371, :456-462)
     "items": [{"id": "sample_s3_task", "version": V1, "project": "project_1", "dependencies_met": True}] +
              [dict(G1, id=str(i), dependencies_met=True) for i in range(5)],
     "db": {"tasks": dict({str(i): doc(status="", version=V1) for i in range(5)}, sample_s3_task=doc(status="started", version=V1, start=-(2 ** 63))),
            "versions": VERSIONS, "max_large_parser": 1, "num_large_parser": 1},
     "steps": [step(None) for _ in range(5)],
     "final": {"node": [1] * 6, "unit": [0] + [1] * 5, "groups": {G1ID: [1, 0]}}},
]

FIXTURES = {"SetupTest": {"items": setup_items(), "db": setup_db()}}  # stored once; a case names it in `fixture`
for case in CASES:
    if case["items"] == FIXTURES["SetupTest"]["items"]:
        extra = {k: v for k, v in case["db"].items() if k not in FIXTURES["SetupTest"]["db"]}
        case.update(fixture="SetupTest", db_extra=extra)
        del case["items"], case["db"]
for case in CASES:  # a rebuild lists [id, DependenciesMet]: the item's other fields are those of the case's `items`
    for st in case["steps"]:
        if "rebuild" in st:
            st["rebuild"] = [[it["id"], it["dependencies_met"]] for it in st["rebuild"]]

if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "dag_find_next_task.json"), "w") as f:
        f.write('{"fixtures": ' + json.dumps(FIXTURES, separators=(",", ":")) + ',\n"cases": [\n' + ",\n".join(json.dumps(c, separators=(",", ":")) for c in CASES) + "\n]}\n")  # one case per line
