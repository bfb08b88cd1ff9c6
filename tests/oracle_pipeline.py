"""Restatement of RunnableTasksPipeline -> task.FindHostRunnable (scheduler/task_finder.go:34-36,
model/task/db.go:887-1066), stage by stage, over dict documents as MongoDB would hold them.

A field Go writes with omitempty is absent when zero; a missing value is the sentinel MISSING, which $eq treats as
equal only to another MISSING.  The documents returned are decoded back into evergreen_b200.model Tasks the way mgo
decodes them into []task.Task (model/task/db.go:1061): a depends_on that is a sub-document (what $unwind leaves) is
skipped and decodes empty, and a removed depends_on.unattainable decodes false.

$group leaves its output order unspecified; the library's canonical order is candidate order, which find_runnable
returns.  Only test code uses this module.
"""
import copy
from typing import Dict, List, Optional, Sequence

from evergreen_b200 import model as M

MISSING = object()
PATCH_REQUESTERS = (M.PATCH_VERSION_REQUESTER, M.GITHUB_PR_REQUESTER, M.GITHUB_MERGE_REQUESTER)  # globals.go:959-963
COMPLETED = (M.TASK_SUCCEEDED, M.TASK_FAILED)  # evergreen.TaskCompletedStatuses, globals.go:1139


def task_doc(t: M.Task) -> dict:
    """Task.MarshalBSON of the fields the aggregation reads.  depends_on has no omitempty and mgo writes a nil slice as
    [] (db/mgo/bson/encode.go:353-365), so it is always an array; Dependency.status / unattainable have no omitempty."""
    d = {"_id": t.id, "status": t.status, "activated": t.activated, "priority": t.priority, "project": t.project,
         "requester": t.requester, "unattainable_dependency": t.unattainable_dependency,
         "override_dependencies": t.override_dependencies,
         "depends_on": [{"_id": x.task_id, "status": x.status, "unattainable": x.unattainable} for x in t.depends_on]}
    if t.execution_platform:
        d["execution_platform"] = t.execution_platform
    return d


def project_doc(p: M.ProjectRef) -> dict:
    """The raw project_ref document: enabled is bool,omitempty; dispatching_disabled / patching_disabled are
    *bool,omitempty (model/project_ref.go:52-59)."""
    d = {"_id": p.id}
    if p.enabled:
        d["enabled"] = True
    if p.dispatching_disabled is not None:
        d["dispatching_disabled"] = p.dispatching_disabled
    if p.patching_disabled is not None:
        d["patching_disabled"] = p.patching_disabled
    return d


def get(doc, path: str):
    """A dotted path as an aggregation expression reads it: through arrays it collects the values it finds."""
    cur = doc
    for k in path.split("."):
        if isinstance(cur, list) and k.isdigit():  # a positional path ("project_ref.0.enabled")
            cur = cur[int(k)] if int(k) < len(cur) else MISSING
        elif isinstance(cur, list):
            vals = [x.get(k, MISSING) for x in cur if isinstance(x, dict)]
            cur = [v for v in vals if v is not MISSING]
        elif isinstance(cur, dict):
            cur = cur.get(k, MISSING)
        else:
            return MISSING
        if cur is MISSING:
            return MISSING
    return cur


def eq(a, b) -> bool:
    if a is MISSING or b is MISSING:
        return a is MISSING and b is MISSING
    return a == b


def unwind(docs, field):
    """$unwind with preserveNullAndEmptyArrays: an empty array or a missing field leaves the document without it."""
    out = []
    for d in docs:
        v = d.get(field, MISSING)
        if isinstance(v, list) and v:
            for x in v:
                e = dict(d)
                e[field] = x
                out.append(e)
        else:
            e = dict(d)
            e.pop(field, None)
            out.append(e)
    return out


def schedulable(d: dict) -> bool:
    """schedulableHostTasksQuery (model/task/db.go:671-689)."""
    return (d["activated"] is True and d["status"] == M.TASK_UNDISPATCHED and d["priority"] > M.DISABLED_TASK_PRIORITY
            and d.get("execution_platform", "host") == "host"
            and (not d["unattainable_dependency"] or d["override_dependencies"]))


def aggregate(distro: M.Distro, candidates: Sequence[dict], collection: Dict[str, dict],
              project_refs: Sequence[dict]) -> List[dict]:
    remove_deps = distro.dispatcher_settings.version != M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES
    # matchActivatedUndispatchedTasks (the candidates stand for the applicable-distro filter)
    docs = [copy.deepcopy(d) for d in candidates if schedulable(d)]
    # removeFields: depends_on.unattainable
    for d in docs:
        for x in d["depends_on"]:
            x.pop("unattainable", None)
    # graphLookupTaskDeps, maxDepth 0: the existing documents whose _id is among depends_on._id, from the collection
    for d in docs:
        want = {x["_id"] for x in d["depends_on"]}
        d["dependency"] = [copy.deepcopy(collection[i]) for i in sorted(want) if i in collection]
    # filterInvalidDistros, only with a distro id and a non-empty ValidProjects
    if distro.id != "" and distro.valid_projects:
        docs = [d for d in docs if d["project"] in distro.valid_projects]
    if remove_deps:
        docs = unwind(docs, "dependency")
        docs = unwind(docs, "depends_on")
        docs = [d for d in docs if eq(get(d, "depends_on._id"), get(d, "dependency._id"))]  # matchIds
        for d in docs:  # projectSatisfied ($or / $and stop at the first decisive arm)
            want, have = get(d, "depends_on.status"), get(d, "dependency.status")
            sat = eq(want, have)
            if not sat and eq(want, "*"):
                sat = have in COMPLETED
                if not sat:
                    un = get(d, "dependency.depends_on.unattainable")
                    assert isinstance(un, list), "$anyElementTrue needs an array"
                    sat = any(bool(x) for x in un)
            d["satisfied_dependencies"] = sat
        groups: Dict[str, dict] = {}  # regroupTasks
        for d in docs:
            g = groups.setdefault(d["_id"], {"_id": d["_id"], "satisfied_set": [], "root": d})
            if d["satisfied_dependencies"] not in g["satisfied_set"]:
                g["satisfied_set"].append(d["satisfied_dependencies"])
        docs = [g["root"] for g in groups.values() if all(g["satisfied_set"])]  # redact + replaceRoot
    refs = {p["_id"]: p for p in project_refs}
    for d in docs:  # joinProjectRef
        d["project_ref"] = [refs[d["project"]]] if d["project"] in refs else []
    docs = [d for d in docs if eq(get(d, "project_ref.0.enabled"), True)
            and not eq(get(d, "project_ref.0.dispatching_disabled"), True)]  # filterDisabledProjects
    docs = [d for d in docs if d["requester"] not in PATCH_REQUESTERS
            or eq(get(d, "project_ref.0.patching_disabled"), False)]  # filterPatchingDisabledProjects
    for d in docs:
        del d["project_ref"]
    return docs


def decode(doc: dict, original: M.Task) -> M.Task:
    """mgo's decode into task.Task of the fields the aggregation changed: depends_on."""
    t = copy.copy(original)
    deps = doc.get("depends_on", MISSING)
    if isinstance(deps, list):
        fin = {x.task_id: x.finished_at for x in original.depends_on}
        t.depends_on = [M.Dependency(task_id=x["_id"], status=x["status"], unattainable=bool(x.get("unattainable", False)),
                                     finished_at=fin.get(x["_id"], M.ZERO_TIME)) for x in deps]
    else:  # missing, or one sub-document where []Dependency is expected (db/mgo/bson/decode.go:503-528)
        t.depends_on = []
    return t


def find_runnable(distro: M.Distro, candidates: Sequence[M.Task], project_refs: Sequence[M.ProjectRef],
                  dependency_db: Optional[Dict[str, M.Task]] = None) -> List[M.Task]:
    """The tasks RunnableTasksPipeline returns for `distro`, decoded, in candidate order.  `candidates` stand for the
    distro's rows of the tasks collection; the collection the $graphLookup searches is `candidates` plus
    `dependency_db`."""
    collection = {t.id: task_doc(t) for t in (dependency_db or {}).values()}
    cand_docs = [task_doc(t) for t in candidates]
    collection.update({d["_id"]: d for d in cand_docs})
    out = aggregate(distro, cand_docs, collection, [project_doc(p) for p in project_refs])
    by_id = {d["_id"]: d for d in out}
    return [decode(by_id[t.id], t) for t in candidates if t.id in by_id]
