"""CPU restatement of the DAG dispatcher's FindNextTask (SURVEY.md §8 f.3) -- test infrastructure only.

Only tests/, __graft_entry__.smoke() and profiles/ may import this module.

Follows model/task_queue_service_dependency.go:258-469 (basicCachedDAGDispatcherImpl.FindNextTask) with
tryMarkItemDispatched :486-498, tryMarkNextTaskGroupTaskDispatched :500-519, getTaskGroup :524-538,
checkMaxConcurrentLargeParserProjectTasks :549-603, nextTaskGroupTask :614-692 and isBlockedSingleHostTaskGroup :696-698,
on top of oracle_dag.rebuild's d.sorted and d.taskGroups.  A restatement of behaviour, statement by statement where the
behaviour hangs on the order of statements; nothing is copied.

The dispatcher is an object with mutable state; every database read goes through `db`, a plain dict the caller may
change between requests (the reference's tests write to the database between FindNextTask calls):

  db["tasks"][id] = {"start": ns, "finish": ns, "status": str, "version": str, "est_generated": int or None,
                     "ingest": ns, "deps_met": True / False / None (None: DependenciesMet returned an error)}
                    a missing id is task.FindOneId's nil document (an error reads the same: the call returns nil)
  db["versions"][version id] = "s3" or anything else (ProjectStorageMethod); a missing id is a nil version
  db["running_hosts"][composite group id] = host.NumHostsByTaskSpec, -1 for its error; a missing id is 0
  db["generate_limit"], db["pending_generate"] (-1: GetPendingGenerateTasks failed),
  db["max_large_parser"] (already resolved for degraded mode), db["num_large_parser"] (-1: the count failed)

Times are ns since the Unix epoch; ZERO_TIME stands for Go's zero time.Time.  The reference tests a start time in two
ways: !utility.IsZeroTime(StartTime) (:334; false for Go's zero time and for the epoch) and StartTime != utility.ZeroTime
(:657; a struct comparison with time.Unix(0, 0), so Go's zero time counts as started).  Both are kept as written.

State the reference keeps and this keeps (the traps are numbered in DESIGN.md §4.14):
  * item["dispatched"]: the node's item, d.nodeItemMap (set by :496, :515);
  * unit["tasks"][i]["dispatched"]: the VALUE copy rebuild put into schedulableUnit.tasks (:172-183), set by :681 and
    read by getTaskGroup and nextTaskGroupTask only -- two bits per grouped item;
  * unit["running_hosts"] (cached, :411-427) and the deletion of the unit from d.taskGroups (:653, :685).
"""
from __future__ import annotations

from typing import Dict, List, Optional

from oracle import oracle_dag

ZERO_TIME = -(2 ** 63)
FOUND, EXHAUSTED, GAVE_UP = 1, 0, 2  # outcome of one request: an item / the walk ended / nil on a database miss


def is_zero_time(t: int) -> bool:  # utility.IsZeroTime: Go's zero time or the Unix epoch
    return t == ZERO_TIME or t == 0


def composite_group_id(group: str, variant: str, project: str, version: str) -> str:  # :700-702
    return f"{group}_{variant}_{project}_{version}"


class Dispatcher:
    """One basicCachedDAGDispatcherImpl.  `items`: TaskQueueItem-like dicts {id, group, build_variant, project, version,
    group_index, group_max_hosts, dependencies, dependencies_met, is_dispatched}."""

    def __init__(self, items: List[dict]):
        self.rebuild(items)

    def rebuild(self, items: List[dict]) -> None:  # :153-252
        order, self.cycles, units = oracle_dag.rebuild(items)
        self.items = [dict(it, dispatched=bool(it.get("is_dispatched", False))) for it in items]  # nodeItemMap
        self.by_id = {it["id"]: it for it in self.items}
        self.sorted = [None if i is None else self.by_id[i] for i in order]
        self.task_groups: Dict[str, dict] = {}
        for gid, ids in units.items():
            first = next(it for it in self.items if it.get("group", "") and self.group_of(it) == gid)
            self.task_groups[gid] = {"id": gid, "running_hosts": 0, "max_hosts": int(first.get("group_max_hosts", 0)),  # :172-180
                                     "tasks": [dict(self.by_id[i]) for i in ids]}  # value copies of the items
        self.units0 = dict(self.task_groups)  # every unit of this rebuild, deleted or not
        self.last_outcome = EXHAUSTED

    @staticmethod
    def group_of(it: dict) -> str:
        return composite_group_id(it.get("group", ""), it.get("build_variant", ""), it.get("project", ""), it.get("version", ""))

    # ---- state as the device keeps it, for comparison
    def state(self):
        """(node bit per item, unit-copy bit per item (0 for items outside every unit), {group id: (deleted, running_hosts)})."""
        unit_bit = {t["id"]: t["dispatched"] for u in self.units0.values() for t in u["tasks"]}
        return ([int(it["dispatched"]) for it in self.items], [int(unit_bit.get(it["id"], False)) for it in self.items],
                {g: (g not in self.task_groups, u["running_hosts"]) for g, u in self.units0.items()})

    # ---- the helpers
    def get_task_group(self, gid: str):  # :524-538
        unit = self.task_groups.get(gid)
        if unit is None:
            return None, False, False
        has = False
        for it in unit["tasks"]:
            if it.get("dependencies_met", False) and not it["dispatched"]:
                has = True
        return unit, True, has

    @staticmethod
    def parser_check(db: dict, doc: dict):  # :549-603 -> (should_continue, should_return) as the call sites use them
        mx = db.get("max_large_parser", 0)
        if mx <= 0:
            return False, False
        if doc["version"] not in db.get("versions", {}):  # error or nil version (:555-576)
            return False, True
        if db["versions"][doc["version"]] == "s3":
            n = db.get("num_large_parser", 0)
            if n < 0:       # the count failed (:580-589)
                return True, False
            if n >= mx:     # :590-600
                return True, False
        return False, False

    def next_task_group_task(self, unit: dict, db: dict) -> Optional[dict]:  # :614-692
        live = self.task_groups.get(unit["id"])
        # :615 compares the map's unit with the caller's copy; requests served one after another always pass a unit
        # that is still in the map, so this cannot fire here.  Kept because the reference has it.
        if live is None or len(live["tasks"]) != len(unit["tasks"]):
            return None
        for i, it in enumerate(unit["tasks"]):
            if it["dispatched"]:
                continue
            doc = db["tasks"].get(it["id"])
            if doc is None:  # :631-650
                return None
            if unit["max_hosts"] == 1 and not is_zero_time(doc["finish"]) and doc["status"] != "success":  # :652-655, :696-698
                del self.task_groups[unit["id"]]
                return None
            if doc["start"] != 0:  # :657 StartTime != utility.ZeroTime (time.Unix(0, 0))
                continue
            if doc["deps_met"] is None or not doc["deps_met"]:  # :662-677
                continue
            it["dispatched"] = True  # :681, the unit's copy
            if i == len(unit["tasks"]) - 1:  # :684-686
                del self.task_groups[unit["id"]]
            return it
        return None

    def try_mark_next_task_group_task(self, unit: dict, db: dict) -> Optional[dict]:  # :500-519
        nxt = self.next_task_group_task(unit, db)
        if nxt is not None:
            self.by_id[nxt["id"]]["dispatched"] = True  # :515, the node's item
        return nxt

    # ---- FindNextTask
    def find_next_task(self, spec: Optional[dict], ami_updated: int, db: dict) -> Optional[str]:
        """spec: {group, build_variant, project, version} or None.  Returns the item id or None; self.last_outcome tells
        a walk that ended (EXHAUSTED) from a nil on a database miss (GAVE_UP)."""
        self.last_outcome = FOUND
        if spec and spec.get("group", ""):  # :268-282
            unit, ok, _ = self.get_task_group(self.group_of(spec))
            if ok:
                nxt = self.try_mark_next_task_group_task(unit, db)
                if nxt is not None:
                    return nxt["id"]
        for item in list(self.sorted):  # getSortedCopy
            if item is None:  # a dependency cycle's placeholder (:290-292)
                continue
            if item.get("group_max_hosts", 0) == 0:  # :305: the branch is GroupMaxHosts, not Group
                if not item.get("dependencies_met", False):
                    continue
                if item["dispatched"]:  # tryMarkItemDispatched :486-498
                    continue
                item["dispatched"] = True  # marked BEFORE any database check
                doc = db["tasks"].get(item["id"])
                if doc is None:  # :313-332
                    self.last_outcome = GAVE_UP
                    return None
                if not is_zero_time(doc["start"]):  # :334
                    continue
                limit, est = db.get("generate_limit", 0), doc.get("est_generated") or 0
                if limit > 0 and est > 0:  # :341-363
                    pending = db.get("pending_generate", 0)
                    if pending < 0:
                        continue
                    if pending + est >= limit:
                        continue
                cont, ret = self.parser_check(db, doc)  # :365-371
                if ret:
                    self.last_outcome = GAVE_UP
                    return None
                if cont:
                    continue
                if doc["deps_met"] is None:  # :373-384
                    continue
                if not doc["deps_met"]:
                    continue
                if not is_zero_time(ami_updated) and doc["ingest"] > ami_updated:  # :392, strict After
                    continue
                return item["id"]
            gid = self.group_of(item)  # :405-409
            unit, _, has = self.get_task_group(gid)
            if not has:
                continue
            if unit["running_hosts"] < unit["max_hosts"]:  # :411
                n = db.get("running_hosts", {}).get(gid, 0)
                if n < 0:  # :413-425
                    self.last_outcome = GAVE_UP
                    return None
                unit["running_hosts"] = n  # :426-427 (the unit is the map's entry: setTaskGroup stores the same value)
                if unit["running_hosts"] < unit["max_hosts"]:
                    nxt = self.try_mark_next_task_group_task(unit, db)
                    if nxt is not None:
                        doc = db["tasks"].get(nxt["id"])
                        if doc is None:  # :433-455
                            self.last_outcome = GAVE_UP
                            return None
                        cont, ret = self.parser_check(db, doc)  # :456-462, after the mark
                        if ret:
                            self.last_outcome = GAVE_UP
                            return None
                        if cont:
                            continue
                        return nxt["id"]
        self.last_outcome = EXHAUSTED
        return None
