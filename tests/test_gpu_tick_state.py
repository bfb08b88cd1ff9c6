"""What every entry point leaves of the resident tick, and what every call that reads the tick needs of it.  Each set-up
below runs on a fresh context and is followed by exactly one probe; the return code of every (set-up, probe) pair is
the literal table EXPECT.  The probes pass no output they would write through, so they report the state rules and
nothing else."""
import copy
import ctypes as C

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_edit import raw_edit
from test_gpu_finder_compaction import candidates

pytestmark = pytest.mark.gpu

CAP = 64  # room for every probe's outputs: each set-up has fewer distros, and the probes ask for one rank per queue


def _run_first(eng):
    """download_queue and rebuild_dispatchers read the last run's ranks: give them one on the tick under test."""
    eng.lib.evg_run_resident(eng.ctx, synth.NOW_NS, 0)


def _queue(eng):
    _run_first(eng)
    item_off, items = np.zeros(CAP + 1, np.int64), np.zeros(CAP, L.QUEUE_ITEM_DTYPE)
    return eng.lib.evg_download_queue(eng.ctx, 1, L.ptr(item_off), L.ptr(items), CAP)


def _dispatchers(eng):
    _run_first(eng)
    bufs = {f: np.zeros(2 * CAP + 2, np.int64 if f in ("item_off", "group_off") else np.int32) for f in L.DISPATCH_OUT_FIELDS}
    out = L.DispatchOutStruct(*[L.ptr(bufs[f]) for f in L.DISPATCH_OUT_FIELDS])
    return eng.lib.evg_rebuild_dispatchers(eng.ctx, 1, CAP, CAP, C.byref(out))


def _edit(eng):
    """An edit the host rejects once the state allows it (its distro table has n_distros -1): INVALID means allowed."""
    es, ds = L.TaskEditStruct(), L.DistroTableStruct()
    ds.n_distros = -1
    return eng.lib.evg_edit_tasks(eng.ctx, C.byref(es), C.byref(ds), None, None, None)


def _resolve(eng, hosts):
    """Nothing to resolve: OK whenever the state allows the call (with hosts: an empty host list)."""
    din = L.DurationInStruct()
    if hosts:
        rows = np.zeros(1, np.int64)
        cs = L.DurationCacheStruct()
        cs.rows = L.ptr(rows)
        din.hosts = C.pointer(cs)
    return eng.lib.evg_resolve_durations(eng.ctx, C.byref(din), synth.NOW_NS)


PROBES = {
    "run": lambda e: e.lib.evg_run_resident(e.ctx, synth.NOW_NS, 0),
    "download": lambda e: e.lib.evg_download(e.ctx, C.byref(L.PlanOutStruct()), None),
    "download_alloc": lambda e: e.lib.evg_download(e.ctx, None, C.byref(L.AllocOutStruct())),
    "download_queue": _queue,
    "rebuild_dispatchers": _dispatchers,
    "update_tasks": lambda e: e.lib.evg_update_tasks(e.ctx, 0, None, None),
    "edit_tasks": _edit,
    "resolve": lambda e: _resolve(e, False),
    "resolve_hosts": lambda e: _resolve(e, True),
    "download_deps": lambda e: e.lib.evg_download_deps(e.ctx, None, None),
    "download_durations": lambda e: e.lib.evg_download_durations(e.ctx, None, None),
    "download_alias_map": lambda e: e.lib.evg_download_alias_map(e.ctx, None, None),
}

# One column per probe, in PROBES order: "." EVG_OK, "S" EVG_ERR_STATE, "I" EVG_ERR_INVALID (evg_edit_tasks allowed).
OWN_HOSTS = ". . . . . . I . . S S S"
OWN = ". . S . . . I . S S S S"
FIXED_HOSTS = ". . . . . . S S S S S S"
FIXED = ". . S . . . S S S S S S"
NONE = "S S S S S S S S S S S S"
EXPECT = {
    # the tick each entry point leaves
    "upload": OWN_HOSTS,
    "upload_with_deps": ". . . . . . I . . . S S",
    "plan_from_finder": OWN_HOSTS,
    "edit_tasks": OWN_HOSTS,
    "plan_aliases": ". . S . . . I . S S S .",
    "upload_device": ". . . . . S S S S S S S",
    "plan_batch": FIXED,
    "plan_and_alloc_batch": FIXED_HOSTS,
    "plan_and_alloc_batch_pipelined": FIXED_HOSTS,
    "upload_empty": ". . S . . . I . S . S S",
    # an upload with hosts, then a call that ends the tick or changes what it holds
    "upload+deps_met_batch": OWN_HOSTS,
    "upload+find_runnable_batch": NONE,
    "upload+prioritize_legacy_batch": NONE,
    "upload+dag_rebuild_batch": NONE,
    "upload+expected_durations_batch": NONE,
    "upload+alloc_batch": NONE,
    "upload+update_tasks": OWN_HOSTS,
    "upload+resolve_durations": ". . . . . . I . . S . S",
    "upload+rebuild_dispatchers": OWN_HOSTS,
    "upload_with_deps+deps_met_batch": OWN_HOSTS,
    "upload_with_deps+update_tasks": OWN_HOSTS,
    "upload_with_deps+resolve_durations": ". . . . . . I . . . . S",
    "plan_aliases+edit_tasks": OWN,
    # set-ups whose last call fails
    "upload_bad_host_off": FIXED,
    "upload_bad_group_id": NONE,
    "edit_rejected_on_host": OWN_HOSTS,
    "edit_rejected_on_device": NONE,
    "plan_aliases_rejected_on_host": ". . S . . . I . S S S .",
    "resolve_bad_key": OWN_HOSTS,
    "resolve_rejected_on_host": ". . . . . . I . . S . S",
}
CODES = {".": L.EVG_OK, "S": L.EVG_ERR_STATE, "I": L.EVG_ERR_INVALID}


@pytest.fixture(scope="module")
def world():
    w, table, fin = candidates([300, 2000, 40], 1301, "mixed")
    at, cfg = synth.make_aliases(w, 1302, name_frac=0.7)
    soa, atab, _, _, _, _ = S.compose_aliases(at, cfg)
    off = np.array([0, 7, 30, 31], np.int64)
    cols = {name: np.zeros(int(off[-1]), dt) for name, dt in S.LegacyTable.COLUMNS}
    cols["tg_rank"][:], cols["tg_pair_id"][:] = -1, -1
    return dict(
        w=w, table=table, fin=fin, at=at, cfg=cfg, alias_w=synth.Workload("alias", w.now, soa, atab, None),
        dw=synth.make_duration_cache(w, 1303, n_rows=20_000, n_keys=300),
        plain=synth.make(np.array([100, 40, 700]), 1304, tg_frac=0.1, n_hosts=10),
        empty=synth.make(np.array([0, 0]), 1305),
        big=synth.make(np.full(8, 280_000), 1306, tg_frac=0.1, n_hosts=100),
        legacy=S.LegacyTable(**cols, task_off=off, list_mode=np.zeros(9, np.uint8)),
    )


def fails(code, fn):
    with pytest.raises(L.EvgError) as e:
        fn()
    assert e.value.code == code, str(e.value)


def upload(eng, W):
    w = W["w"]
    eng.upload(w.tasks, w.distros, w.hosts)


def upload_with_deps(eng, W):
    w = W["w"]
    eng.upload_with_deps(w.tasks, w.distros, w.hosts, W["table"].deps, W["fin"], w.now)


def plan_aliases(eng, W):
    eng.plan_aliases(W["at"], W["cfg"], W["w"].now)


def upload_device(eng, W):
    import torch
    w = W["plain"]
    cols = {name: torch.from_numpy(np.concatenate([getattr(w.tasks, name), np.zeros(8, dt)])).cuda() for name, dt in S.TaskSoA.COLUMNS}
    eng.upload_device({k: v.data_ptr() for k, v in cols.items()}, w.n_tasks, w.distros, w.hosts)
    torch.cuda.synchronize()
    return cols  # the context borrows these until the probe is done


def edit(eng, W, seed=1310):
    upload(eng, W)
    e = synth.next_tick(W["w"], seed)
    eng.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)


def alias_edit(eng, W):
    plan_aliases(eng, W)
    e = synth.next_tick(W["alias_w"], 1313)
    eng.edit_tasks(e.edit, e.workload.distros)


def alloc(eng, W):
    w = W["w"]
    upload(eng, W)
    eng.run(w.now)
    po, _ = eng.download()
    eng.alloc_batch(w.hosts, po.info.copy(), po.group_info.copy(), w.distros.group_off, w.now)


def dag(eng, W):
    upload(eng, W)
    item_off, group_off = np.array([0, 3, 5], np.int64), np.array([0, 1, 1], np.int64)
    eng.dag_rebuild_batch(item_off, group_off, np.array([0, 0, 1, 1, 2, 2], np.int64), np.array([0, 0], np.int32),
                          np.array([0, -1, 0, -1, -1], np.int32), np.array([0, 0, 1, 0, 0], np.int32))


def update(eng, W):
    w = W["w"]
    rows = np.array([0, 5, w.n_tasks - 1], np.int64)
    eng.update_tasks(rows, S.TaskSoA(**{name: getattr(w.tasks, name)[rows].copy() for name, _ in S.TaskSoA.COLUMNS}))


def resolve(eng, W):
    dw = W["dw"]
    eng.resolve_durations(dw.history, W["w"].now, dw.tasks, dw.hosts)


def dispatchers(eng, W):
    eng.run(W["w"].now)
    eng.rebuild_dispatchers(0)


def bad_host_off(eng, W):
    w = W["w"]
    h = copy.copy(w.hosts)
    h.host_off = w.hosts.host_off.copy()
    h.host_off[-1] += 1
    fails(L.EVG_ERR_INVALID, lambda: eng.upload(w.tasks, w.distros, h))


def bad_group_id(eng, W):
    w = W["w"]
    upload(eng, W)
    t = copy.copy(w.tasks)
    t.group_id = w.tasks.group_id.copy()
    t.group_id[0] = 1_000_000
    fails(L.EVG_ERR_INVALID, lambda: eng.upload(t, w.distros, w.hosts))


def edit_rejected_on_host(eng, W):
    upload(eng, W)
    e = synth.next_tick(W["w"], 1311)
    nd = e.workload.distros
    off = nd.task_off.copy()
    off[1:] += 1
    assert raw_edit(eng, e.edit, S.DistroTable(off, nd.group_off, nd.cfg, nd.group_max_hosts).normalize()) == L.EVG_ERR_INVALID


def edit_rejected_on_device(eng, W):
    upload(eng, W)
    e = synth.next_tick(W["w"], 1312)
    ed = copy.copy(e.edit)
    ed.group_remap = np.full(int(W["w"].distros.group_off[-1]), -1, np.int32)  # every surviving task group dissolves
    assert raw_edit(eng, ed, e.workload.distros) == L.EVG_ERR_INVALID


def plan_aliases_rejected_on_host(eng, W):
    plan_aliases(eng, W)
    at = copy.copy(W["at"])
    at.dest_idx = W["at"].dest_idx.copy()
    at.dest_idx[0] = W["cfg"].shape[0]
    fails(L.EVG_ERR_INVALID, lambda: eng.plan_aliases(at, W["cfg"], W["w"].now))


def resolve_bad_key(eng, W):
    upload(eng, W)
    resolve(eng, W)
    dw = W["dw"]
    tasks = copy.copy(dw.tasks)
    tasks.key = dw.tasks.key.copy()
    tasks.key[0] = dw.history.rows.n_keys
    fails(L.EVG_ERR_INVALID, lambda: eng.resolve_durations(dw.history, W["w"].now, tasks, dw.hosts))


def resolve_rejected_on_host(eng, W):
    upload(eng, W)
    resolve(eng, W)
    dw = W["dw"]
    short = S.DurationCache(*[getattr(dw.tasks, f)[:-1] for f in L.DURATION_CACHE_COLUMNS], dw.tasks.key[:-1])
    fails(L.EVG_ERR_INVALID, lambda: eng.resolve_durations(dw.history, W["w"].now, short))


def then(first, second):
    def run(eng, W):
        first(eng, W)
        return second(eng, W)
    return run


SETUPS = {
    "upload": upload,
    "upload_with_deps": upload_with_deps,
    "plan_from_finder": lambda eng, W: eng.plan_from_finder(W["table"], W["w"].tasks, W["w"].distros, W["w"].hosts, W["fin"], W["w"].now),
    "edit_tasks": edit,
    "plan_aliases": plan_aliases,
    "upload_device": upload_device,
    "plan_batch": lambda eng, W: eng.plan_batch(W["w"].tasks, W["w"].distros, W["w"].now),
    "plan_and_alloc_batch": lambda eng, W: eng.plan_and_alloc_batch(W["w"].tasks, W["w"].distros, W["w"].hosts, W["w"].now),
    "plan_and_alloc_batch_pipelined": lambda eng, W: eng.plan_and_alloc_batch(W["big"].tasks, W["big"].distros, W["big"].hosts,
                                                                                W["big"].now),
    "upload_empty": lambda eng, W: eng.upload(W["empty"].tasks, W["empty"].distros),
    "upload+deps_met_batch": then(upload, lambda eng, W: eng.deps_met_batch(W["table"].deps)),
    "upload+find_runnable_batch": then(upload, lambda eng, W: eng.find_runnable_batch(W["table"])),
    "upload+prioritize_legacy_batch": then(upload, lambda eng, W: eng.prioritize_legacy_batch(W["legacy"])),
    "upload+dag_rebuild_batch": dag,
    "upload+expected_durations_batch": then(upload, lambda eng, W: eng.expected_durations_batch(W["dw"].history.rows)),
    "upload+alloc_batch": alloc,
    "upload+update_tasks": then(upload, update),
    "upload+resolve_durations": then(upload, resolve),
    "upload+rebuild_dispatchers": then(upload, dispatchers),
    "upload_with_deps+deps_met_batch": then(upload_with_deps, lambda eng, W: eng.deps_met_batch(W["table"].deps)),
    "upload_with_deps+update_tasks": then(upload_with_deps, update),
    "upload_with_deps+resolve_durations": then(upload_with_deps, resolve),
    "plan_aliases+edit_tasks": alias_edit,
    "upload_bad_host_off": bad_host_off,
    "upload_bad_group_id": bad_group_id,
    "edit_rejected_on_host": edit_rejected_on_host,
    "edit_rejected_on_device": edit_rejected_on_device,
    "plan_aliases_rejected_on_host": plan_aliases_rejected_on_host,
    "resolve_bad_key": resolve_bad_key,
    "resolve_rejected_on_host": resolve_rejected_on_host,
}


def test_the_table_covers_every_setup_and_probe():
    assert set(SETUPS) == set(EXPECT)
    assert all(len(row.split()) == len(PROBES) for row in EXPECT.values())


@pytest.mark.parametrize("setup", sorted(SETUPS))
def test_state_rules(world, setup):
    got, want = {}, {}
    for k, (name, probe) in enumerate(PROBES.items()):
        eng = scheduler.Engine(0)
        try:
            keep = SETUPS[setup](eng, world)
            got[name] = probe(eng)
            del keep
        finally:
            eng.close()
        want[name] = CODES[EXPECT[setup].split()[k]]
    assert got == want
