"""evg_edit_strings against its definition: the edited context equals a second context fed evg_upload_strings of the
composed string table (soa.compose_strings), output for output; ResidentTick(device_strings=True) equals
ResidentTick(); the state and error rules."""
import copy
import ctypes as C
import dataclasses

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_entry_guard import launched_kernels
from test_gpu_intern import outputs, snap
from test_gpu_tick_state import CODES, NONE, OWN, OWN_HOSTS, PROBES

import edit_strings_scripts as X
import parity

pytestmark = pytest.mark.gpu

SIZES = (0, 1, 40, 700, 0, 300, 13, 2000)


def numeric(batch):
    return S.marshal_tasks(batch, X.NOW, intern=False)


def offsets(batch):
    return np.concatenate([[0], np.cumsum([len(ts) for _, ts in batch])]).astype(np.int64)


def hosts_for(n_distros, seed):
    return synth.make(np.full(n_distros, 4), seed, n_hosts=30).hosts


class Pair:
    """Context a edits its resident strings; context b uploads the composed table each tick."""

    def __init__(self, script: X.Script, hosts):
        self.a, self.b = scheduler.Engine(0), scheduler.Engine(0)
        self.script, self.hosts = script, hosts
        self.prev = script.batch
        self.old = S.string_cols(self.prev)
        soa, table, _ = numeric(self.prev)
        self.cfg = table.cfg
        self.mirror = soa  # the numeric columns a holds: what b uploads for the survivors
        for eng in (self.a, self.b):
            eng.upload_strings(soa, self.old, self.cfg, hosts)

    def close(self):
        self.a.close()
        self.b.close()

    def step(self, **kw):
        batch = self.script.next_batch(**kw)
        soa, table, _ = numeric(batch)
        edit = X.string_edit(self.prev, batch, offsets(self.prev), soa)
        composed = S.compose_strings(self.old, edit)
        keep = np.ones(self.mirror.n_tasks, dtype=bool)
        keep[edit.remove_rows] = False
        n_ins = np.diff(edit.insert_off)
        toff = offsets(batch)
        surv_new = np.concatenate([np.arange(toff[d], toff[d + 1] - n_ins[d]) for d in range(len(batch))]).astype(np.int64)
        for name, _ in S.TaskSoA.COLUMNS:
            getattr(soa, name)[surv_new] = getattr(self.mirror, name)[keep]
        got = self.a.edit_strings(edit, table.cfg, self.hosts, n_dep_ids=int(composed.dep_off[-1]))
        want = self.b.upload_strings(soa, composed, table.cfg, self.hosts)
        self.mirror = soa
        for k in S.INTERN_OUT_FIELDS:
            assert np.array_equal(got[k], want[k]), k
        self.prev, self.old = batch, composed
        return edit, want

    def same(self):
        task_off = offsets(self.prev)
        w = synth.Workload("s", X.NOW, None, S.DistroTable(task_off, np.zeros(1), self.cfg, np.zeros(0)), self.hosts)
        for opts in (0, L.EVG_OPT_BREAKDOWN):
            assert outputs(self.a, w, opts) == outputs(self.b, w, opts)
        for eng in (self.a, self.b):
            eng.run(X.NOW, L.EVG_OPT_QUEUE_BREAKDOWN)
        assert snap(self.a.download_queue_breakdown(0, task_off)) == snap(self.b.download_queue_breakdown(0, task_off))


@pytest.mark.parametrize("bits", [None, "0"])
def test_edits_equal_upload_of_the_composed_table(monkeypatch, bits):
    if bits is not None:
        monkeypatch.setenv("EVG_INTERN_HASH_BITS", bits)
    p = Pair(X.Script(501, SIZES), hosts_for(len(SIZES), 502))
    try:
        seen = set()
        for step in range(5):
            before = {(d, g) for d, (_, ts) in enumerate(p.prev) for t in ts for g in [t.get_task_group_string()] if t.task_group}
            edit, out = p.step(leave=0.2, arrive=0.2)
            after = {(d, g) for d, (_, ts) in enumerate(p.prev) for t in ts for g in [t.get_task_group_string()] if t.task_group}
            seen.add("group vanished") if before - after else None
            seen.add("group appeared") if after - before else None
            p.same()
            # update_tasks between two edits, on both contexts
            rng = np.random.default_rng(step)
            rows = np.sort(rng.choice(p.a._n_tasks, size=min(50, p.a._n_tasks), replace=False)).astype(np.int64)
            vals = S.TaskSoA(**{name: np.asarray(rng.integers(0, 1000, rows.shape[0]), dt) for name, dt in S.TaskSoA.COLUMNS})
            for eng in (p.a, p.b):
                eng.update_tasks(rows, vals)
            for name, _ in S.TaskSoA.COLUMNS:
                getattr(p.mirror, name)[rows] = getattr(vals, name)
            p.same()
        assert seen == {"group vanished", "group appeared"}
    finally:
        p.close()


def test_edges_follow_arrivals_and_departures():
    """A survivor gains the edge to an arrival it named before it existed and loses the edge to a departed task."""
    p = Pair(X.Script(511, (60, 30)), None)
    try:
        gained = lost = False
        for _ in range(6):
            prev_ids = [{t.id for t in ts} for _, ts in p.prev]
            edit, out = p.step(leave=0.3, arrive=0.3)
            ids = [{t.id for t in ts} for _, ts in p.prev]
            for d, (_, ts) in enumerate(p.prev):
                for t in ts:
                    if t.id in prev_ids[d]:
                        names = [x.task_id for x in t.depends_on]
                        gained |= any(n in ids[d] and n not in prev_ids[d] for n in names)
                        lost |= any(n in prev_ids[d] and n not in ids[d] for n in names)
            assert int(out["dep_off"][-1]) > 0
            p.same()
        assert gained and lost
        assert any(len(t.depends_on) != len({x.task_id for x in t.depends_on}) for _, ts in p.prev for t in ts)  # repeated ids
    finally:
        p.close()


def test_empty_edit_full_replacement_and_emptied_distros():
    p = Pair(X.Script(521, SIZES), hosts_for(len(SIZES), 522))
    try:
        edit, _ = p.step(leave=0.0, arrive=0.0)
        assert edit.remove_rows.shape[0] == 0 and edit.strings.n_tasks == 0
        p.same()
        p.step(replace_all=set(range(len(SIZES))))
        p.same()
        p.step(empty={2, 3, 7})
        p.same()
        p.step(empty=set(range(len(SIZES))))
        p.same()
        edit, _ = p.step(replace_all=set(range(len(SIZES))))  # onto an empty tick: every row is an inserted one
        assert p.a._n_tasks == edit.strings.n_tasks > 0 and edit.remove_rows.shape[0] == 0
        p.same()
    finally:
        p.close()


def test_intern_batch_and_queue_index_leave_the_strings():
    p = Pair(X.Script(531, SIZES), hosts_for(len(SIZES), 532))
    try:
        p.step()
        other = S.string_cols(X.Script(533, (3000, 50)).batch)  # larger than the tick: the staging buffers grow
        p.a.intern_batch(other)
        p.a.queue_index([f"id{i % 7}" for i in range(500)], np.array([0, 200, 500], np.int64))
        p.step()
        p.same()
    finally:
        p.close()


def test_launch_count_matches_the_profiler():
    p = Pair(X.Script(541, SIZES), None)
    try:
        batch = p.script.next_batch()
        soa, table, _ = numeric(batch)
        edit = X.string_edit(p.prev, batch, offsets(p.prev), soa)
        names = launched_kernels(lambda: p.a.edit_strings(edit, table.cfg))
        assert names and p.a.last_launch_count() == len(names), names
        assert {"k_sx_rows", "k_sx_edges", "k_sx_len", "k_sx_copy", "k_in_keys"} <= {n.split("(")[0] for n in names}
    finally:
        p.close()


# ---- state and errors ---------------------------------------------------------------------------------------------

def edit_call(eng, edit, cfg):
    """evg_edit_strings asked for the per-distro outputs only -> its return code."""
    es, keep = edit.struct()
    group_off, n_versions = np.zeros(cfg.shape[0] + 1, np.int64), np.zeros(max(cfg.shape[0], 1), np.int32)
    outs = L.InternOutStruct(None, None, L.ptr(group_off), L.ptr(n_versions), None, None, None, None)
    return eng.lib.evg_edit_strings(eng.ctx, C.byref(es), L.ptr(cfg), None, None, None, C.byref(outs))


@pytest.fixture(scope="module")
def world():
    script = X.Script(551, SIZES)
    prev = script.batch
    batch = script.next_batch()
    soa, table, _ = numeric(batch)
    return dict(prev=prev, batch=batch, soa=soa, cfg=table.cfg, hosts=hosts_for(len(SIZES), 552),
                edit=X.string_edit(prev, batch, offsets(prev), soa))


def bad_edits(world):
    """name -> (edit, 'host' or 'device')"""
    e = world["edit"]
    cases = {}
    r = e.remove_rows
    cases["unsorted"] = (dataclasses.replace(e, remove_rows=r[::-1].copy()), "host")
    cases["out of range"] = (dataclasses.replace(e, remove_rows=np.append(r, 10 ** 9)), "host")
    sc = e.strings
    shifted = sc.task_off.copy()
    shifted[-1] += 1  # does not end at the inserted row count
    cases["insert_off"] = (dataclasses.replace(e, strings=dataclasses.replace(sc, task_off=shifted)), "host")
    cases["n_distros"] = (dataclasses.replace(e, strings=dataclasses.replace(sc, task_off=sc.task_off[:-1].copy(),
                                                                             )), "host")
    dep_off = sc.dep_off.copy()
    dep_off[0] = 1
    cases["intern_check"] = (dataclasses.replace(e, strings=dataclasses.replace(sc, dep_off=dep_off)), "host")
    # a dep_off row inside the inserted columns that decreases: only the kernel that reads the row sees it
    dep_off = sc.dep_off.copy()
    k = int(np.nonzero(dep_off[2:] < dep_off[-1])[0][0]) + 1
    dep_off[k] = dep_off[k + 1] + 1
    cases["dep_off row"] = (dataclasses.replace(e, strings=dataclasses.replace(sc, dep_off=dep_off)), "device")
    id_off = sc.id[1].copy()
    id_off[3] = id_off[-1] + 1
    cases["string row"] = (dataclasses.replace(e, strings=dataclasses.replace(sc, id=(sc.id[0], id_off))), "device")
    return cases


def probe_states(world, edit):
    """PROBES, each on a fresh context whose evg_upload_strings tick `edit` was applied to (or rejected on)."""
    got = []
    for probe in PROBES.values():
        eng = scheduler.Engine(0)
        try:
            eng.upload_strings(numeric(world["prev"])[0], S.string_cols(world["prev"]), world["cfg"], world["hosts"])
            rc, msg = edit_call(eng, edit, world["cfg"]), L.last_error()
            got.append(probe(eng))
        finally:
            eng.close()
    return rc, msg, got


def test_host_and_device_rejections(world):
    rc, _, got = probe_states(world, world["edit"])
    assert rc == L.EVG_OK and got == [CODES[x] for x in OWN.split()]  # planner only: the edit passed no hosts
    for name, (edit, where) in bad_edits(world).items():
        rc, msg, got = probe_states(world, edit)
        assert rc == L.EVG_ERR_INVALID and "evg_edit_strings" in msg, (name, msg)
        assert got == [CODES[x] for x in (OWN_HOSTS if where == "host" else NONE).split()], name
        if where == "device":
            assert "composed row" in msg, msg
    # a survivor and an arrival of one task group that disagree on TaskGroupMaxHosts: the lowest composed row is named
    e = world["edit"]
    sc = e.strings
    old = S.string_cols(world["prev"])
    key = lambda c, i: bytes(c.group_key[0][c.group_key[1][i]:c.group_key[1][i + 1]])  # noqa: E731
    gone = set(e.remove_rows.tolist())
    d_old = np.repeat(np.arange(old.n_distros), np.diff(old.task_off))
    d_ins = np.repeat(np.arange(sc.n_distros), np.diff(sc.task_off))
    held = {(int(d_old[i]), key(old, i)) for i in range(old.n_tasks) if i not in gone}
    i = next(i for i in range(sc.n_tasks) if key(sc, i) and (int(d_ins[i]), key(sc, i)) in held)  # joins a survivor's group
    gmh = sc.group_max_hosts.copy()
    gmh[i] += 7
    eng = scheduler.Engine(0)
    try:
        eng.upload_strings(numeric(world["prev"])[0], S.string_cols(world["prev"]), world["cfg"], world["hosts"])
        bad = dataclasses.replace(e, strings=dataclasses.replace(sc, group_max_hosts=gmh))
        composed = S.compose_strings(S.string_cols(world["prev"]), bad)
        out, outs = composed.intern_out()
        assert L.load().evg_intern_columns(C.byref(composed.struct()), C.byref(outs), 1) == L.EVG_ERR_INVALID
        want = L.last_error()
        assert edit_call(eng, bad, world["cfg"]) == L.EVG_ERR_INVALID
        row = want.split("row ")[1].split(" ")[0].rstrip(":")
        assert f"row {row}:" in L.last_error(), (want, L.last_error())
        assert [probe(eng) for probe in PROBES.values()] == [CODES[x] for x in NONE.split()]
    finally:
        eng.close()


@pytest.mark.parametrize("before", ["upload", "edit_tasks", "plan_batch", "rejected_edit_then_upload", "edit_tasks_with_deps"])
def test_state_error_without_resident_strings(world, before):
    eng = scheduler.Engine(0)
    try:
        soa, table, _ = S.marshal_tasks(world["prev"], X.NOW)
        if before == "upload":
            eng.upload(soa, table, world["hosts"])
        elif before == "edit_tasks":
            eng.upload_strings(numeric(world["prev"])[0], S.string_cols(world["prev"]), world["cfg"], world["hosts"])
            empty = S.TaskEdit(np.zeros(0, np.int64), None, np.zeros(table.n_distros + 1, np.int64), np.zeros(0, np.int64),
                               np.zeros(0, np.int32))
            eng.edit_tasks(empty, table)
        elif before == "plan_batch":
            eng.plan_batch(soa, table, X.NOW)
        elif before == "edit_tasks_with_deps":
            # a string tick holds no dependency table, so evg_edit_tasks_with_deps refuses it and leaves the tick and its
            # strings; on a tick that holds one (ResidentTick's device_deps path), the call leaves no string table
            eng.upload_strings(numeric(world["prev"])[0], S.string_cols(world["prev"]), world["cfg"], world["hosts"])
            rc = eng.lib.evg_edit_tasks_with_deps(eng.ctx, C.byref(L.TaskEditStruct()), C.byref(L.DistroTableStruct()), None, None,
                                                  None, 0, None, None, C.byref(L.DepsEditStruct()), X.NOW)
            assert rc == L.EVG_ERR_STATE and "dependency table" in L.last_error()
            assert edit_call(eng, world["edit"], world["cfg"]) == L.EVG_OK
            script = X.Script(551, SIZES)
            script.next_batch()
            prev = script.batch
            batch = script.next_batch(leave=0.1, arrive=0.0)  # no arrival changes how a kept DependsOn id resolves
            rt = scheduler.ResidentTick(eng, device_deps=True)
            rt.plan(prev, X.NOW)
            rt.plan(batch, X.NOW)
            assert rt.last is not None  # the tick went through evg_edit_tasks_with_deps
        else:  # an edit rejected on the host keeps the strings; a later evg_upload drops them
            eng.upload_strings(numeric(world["prev"])[0], S.string_cols(world["prev"]), world["cfg"], world["hosts"])
            bad, _ = bad_edits(world)["unsorted"]
            assert edit_call(eng, bad, world["cfg"]) == L.EVG_ERR_INVALID
            assert edit_call(eng, world["edit"], world["cfg"]) == L.EVG_OK
            eng.upload(soa, table, world["hosts"])
        assert edit_call(eng, world["edit"], world["cfg"]) == L.EVG_ERR_STATE
        assert "string table" in L.last_error()
    finally:
        eng.close()


# ---- ResidentTick ---------------------------------------------------------------------------------------------------

def test_resident_tick_with_device_strings_equals_the_host_interned_one():
    script = X.Script(561, SIZES)
    batches = [script.batch] + [script.next_batch(leave=0.15, arrive=0.15) for _ in range(4)]
    batches.append([(d, ts) for d, ts in batches[-1][:-1]])  # another distro list: uploads again
    batches.append(script.next_batch())
    res = []
    for device_strings in (False, True):
        eng = scheduler.Engine(0)
        try:
            rt = scheduler.ResidentTick(eng, device_strings=device_strings)
            got = []
            copies = copy.deepcopy(batches)
            for k, batch in enumerate(copies):
                prev_ids = {t.id for t in copies[k - 1][3][1]} if k else set()
                surv = [t for t in batch[3][1] if t.id in prev_ids]
                if k == 2:  # a survivor gains a DependsOn id naming another queued task (generate.tasks does this)
                    surv[0].depends_on.append(M.Dependency(surv[1].id))
                if k == 4:  # a survivor moves to another version (and so to another task-group key)
                    surv[2].version = "v-moved"
                out = rt.plan(batch, X.NOW)
                got.append([([t.id for t in ranked], [dataclasses.astuple(t.sorting_value_breakdown) for t in ranked], info)
                            for ranked, info in out])
                if k == 3 and device_strings:  # an oracle-checked tick
                    soa, table, _ = S.marshal_tasks(rt.canonical(batch), X.NOW, resolve_deps=True)
                    eng.run(X.NOW, 0)
                    po, _ = eng.download(want_alloc=False)
                    parity.check_against_oracle(synth.Workload("rt", X.NOW, soa, table, None), po, None)
                # the default path sends the gained edge as an added edge; device strings must upload for it
                assert (rt.last is None) == (k in ((0, 2, 4, 5, 6) if device_strings else (0, 4, 5, 6))), k
            res.append(got)
        finally:
            eng.close()
    assert res[0] == res[1]
