"""Seeded multi-tick Go-level scripts for the resident dependency table (evg_edit_tasks_with_deps): every tick
dispatches tasks (biased to the heads of the queues), finishes some of them `success` / `failed` (their dependents'
FinishedAt written as MarkDependenciesFinished does), leaves others dispatched or gone from the tasks collection, blocks
and unblocks external tasks, flips survivors' OverrideDependencies, lets survivors gain dependencies, and brings
arrivals that depend on survivors, on each other, on external tasks and on ids no collection holds, with wants "",
"failed", "*" and other strings.  Heads leave with their dependents often, so chains leave in one tick."""
import copy
import random

import numpy as np

from evergreen_b200 import model as M
from evergreen_b200 import soa as S

NOW = 1_700_000_000 * 10 ** 9
WANTS = ["", "", "success", "failed", "*", "*", "other"]


def _task(rng, tid, distro_id):
    t = M.Task(id=tid, version=f"v{rng.randrange(4)}", project="p", build_variant="bv", distro_id=distro_id,
               priority=rng.choice([0, 0, 5, 50]), requester=rng.choice(["gitter_request", "patch_request"]),
               num_dependents=rng.randrange(3), activated_time=NOW - rng.randrange(10 ** 13),
               scheduled_time=NOW - rng.randrange(10 ** 12), expected_duration=rng.randrange(1, 3600) * 10 ** 9)
    if rng.random() < 0.2:
        t.task_group, t.task_group_order, t.task_group_max_hosts = f"tg{rng.randrange(3)}", rng.randrange(1, 5), 2
    return t


def _blocked_doc(rng, tid, status):
    t = M.Task(id=tid, status=status)
    if rng.random() < 0.3:
        t.depends_on = [M.Dependency("gone", unattainable=True)]
    return t


class Script:
    """One script: `batch` is the current Go-level tick, `db` the tasks collection outside the queues."""

    def __init__(self, seed: int, sizes, dep_frac: float = 0.3):
        self.rng = rng = random.Random(seed)
        self.dep_frac = dep_frac
        self.db = {}
        self.n = 0
        for k in range(12):  # tasks of other queues and finished ones
            self.db[f"x{k}"] = _blocked_doc(rng, f"x{k}", rng.choice([M.TASK_SUCCEEDED, M.TASK_FAILED, "started"]))
        self.batch = []
        for k, n in enumerate(sizes):
            d = M.Distro(id=f"d{k}", dispatcher_settings=M.DispatcherSettings(M.DISPATCHER_VERSION_REVISED_WITH_DEPENDENCIES))
            d.planner_settings.group_versions = k % 3 == 2
            ts = [self._new(d.id) for _ in range(n)]
            for t in ts:
                self._depend(t, ts)
            self.batch.append((d, ts))

    def _new(self, distro_id):
        self.n += 1
        return _task(self.rng, f"t{self.n}", distro_id)

    def _depend(self, t, pool):
        rng = self.rng
        while rng.random() < self.dep_frac:
            u = rng.random()
            if u < 0.6 and len(pool) > 1:
                dep_id = rng.choice(pool).id
            elif u < 0.9:
                dep_id = rng.choice(sorted(self.db))
            else:
                dep_id = f"nowhere{rng.randrange(5)}"
            if dep_id != t.id:
                t.depends_on.append(M.Dependency(dep_id, status=rng.choice(WANTS)))

    def step(self, tick: int, dispatch: float = 0.15, arrive: float = 0.1):
        """The next Go-level batch (its tasks are copies: the previous batch's Task objects stay as they were)."""
        rng = self.rng
        fin_at = NOW + (tick + 1) * 10 ** 10
        out = []
        queued = [[copy.copy(t) for t in ts] for _, ts in self.batch]
        for ts in queued:
            for t in ts:
                t.depends_on = [copy.copy(x) for x in t.depends_on]
        departed = {}
        for (d, _), ts in zip(self.batch, queued):
            n = len(ts)
            keep = []
            for i, t in enumerate(ts):
                if rng.random() < 2 * dispatch * (1 - i / max(n, 1)):
                    departed[t.id] = t
                else:
                    keep.append(t)
            out.append((d, keep))
        # a departure finishes, stays dispatched, or leaves the collection
        finished = {}
        for tid, t in departed.items():
            u = rng.random()
            if u < 0.7:
                status = M.TASK_SUCCEEDED if rng.random() < 0.7 else M.TASK_FAILED
                self.db[tid] = _blocked_doc(rng, tid, status)
                finished[tid] = fin_at
            elif u < 0.9:
                self.db[tid] = _blocked_doc(rng, tid, "started")
        # external tasks change status or blocking (their dependents' FinishedAt is kept)
        for tid in sorted(self.db):
            if rng.random() < 0.1:
                self.db[tid] = _blocked_doc(rng, tid, rng.choice([M.TASK_SUCCEEDED, M.TASK_FAILED, "started"]))
        for d, keep in out:
            for t in keep:
                for x in t.depends_on:
                    if x.task_id in finished:  # MarkDependenciesFinished
                        x.finished_at = finished[x.task_id]
                if rng.random() < 0.05:
                    t.override_dependencies = not t.override_dependencies
                if t.depends_on and rng.random() < 0.05:
                    x = rng.choice(t.depends_on)
                    x.unattainable = not x.unattainable
                if rng.random() < 0.05:
                    t.priority += 3
        for k, (d, keep) in enumerate(out):
            arrivals = [self._new(d.id) for _ in range(int(arrive * len(self.batch[k][1])) + rng.randrange(3))]
            pool = keep + arrivals
            for t in arrivals:
                self._depend(t, pool)
            for t in keep:
                if rng.random() < 0.05:
                    self._depend(t, pool)
            rng.shuffle(keep)
            out[k] = (d, keep + arrivals)
        self.batch = out
        return out


def edit_rows(prev_ids, canon):
    """(remove_rows, insert_off) of the step from the tick with `prev_ids` to `canon` (canonical order)."""
    now = {t.id for _, ts in canon for t in ts}
    flat = [i for ids in prev_ids for i in ids]
    remove = np.array([r for r, i in enumerate(flat) if i not in now], dtype=np.int64)
    prev = set(flat)
    n_ins = [sum(1 for t in ts if t.id not in prev) for _, ts in canon]
    return remove, np.concatenate([[0], np.cumsum(n_ins)]).astype(np.int64)


def canonical(prev_ids, batch):
    out = []
    for (d, ts), prev in zip(batch, prev_ids):
        by_id = {t.id: t for t in ts}
        seen = set(prev)
        out.append((d, [by_id[i] for i in prev if i in by_id] + [t for t in ts if t.id not in seen]))
    return out


def write_back(canon, stamp):
    k = 0
    for _, ts in canon:
        for t in ts:
            if int(stamp[k]) != M.ZERO_TIME:
                t.dependencies_met_time = int(stamp[k])
            k += 1


def task_off(canon):
    return np.concatenate([[0], np.cumsum([len(ts) for _, ts in canon])]).astype(np.int64)


def ids_of(canon):
    return [[t.id for t in ts] for _, ts in canon]


def host_verdicts(canon, db):
    """soa.dependencies_met (the Go restatement) of every task, without stamping."""
    out = []
    for _, ts in canon:
        by_id = {t.id: t for t in ts}
        out.extend(S.dependencies_met(t, by_id, db) for t in ts)
    return np.array(out, dtype=np.uint8)
