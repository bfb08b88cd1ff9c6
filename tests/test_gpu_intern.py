"""evg_intern_batch and evg_upload_strings: evg_intern_columns on the device.  Every output of evg_intern_batch equals
the host's evg_intern_columns for the same strings, bit for bit, also when EVG_INTERN_HASH_BITS makes (nearly) every
string collide; a tick uploaded with evg_upload_strings behaves exactly like evg_upload of the host-interned table."""
import ctypes as C
import dataclasses
import os
import random
import sys

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_entry_guard import launched_kernels
from test_gpu_tick_state import CODES, NONE, OWN_HOSTS, PROBES
from test_host_logic import random_tasks

import parity

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
import intern_bench  # noqa: E402

pytestmark = pytest.mark.gpu


def host_intern(sc: S.StringCols):
    """evg_intern_columns on one thread (the lowest bad row is then the one it names) -> (rc, message, outputs)."""
    out, outs = sc.intern_out()
    rc = L.load().evg_intern_columns(C.byref(sc.struct()), C.byref(outs), 1)
    return rc, L.last_error() if rc else "", sc.trim(out) if rc == L.EVG_OK else None


def device_intern(eng, sc: S.StringCols):
    out, outs = sc.intern_out()
    rc = eng.lib.evg_intern_batch(eng.ctx, C.byref(sc.struct()), C.byref(outs))
    return rc, L.last_error() if rc else "", sc.trim(out) if rc == L.EVG_OK else None


def check_same(eng, sc: S.StringCols):
    rc, _, want = host_intern(sc)
    assert rc == L.EVG_OK, L.last_error()
    got = eng.intern_batch(sc)
    for k in S.INTERN_OUT_FIELDS:
        assert np.array_equal(got[k], want[k]), k
    return want


def pack(distros):
    """[[(id, version, group key, max hosts, [dependency ids])]] -> StringCols."""
    rows = [r for d in distros for r in d]
    task_off = np.concatenate([[0], np.cumsum([len(d) for d in distros])]).astype(np.int64)
    dep_off = np.concatenate([[0], np.cumsum([len(r[4]) for r in rows])]).astype(np.int64)
    return S.StringCols.pack(task_off, [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows],
                             np.array([r[3] for r in rows], np.int32), dep_off, [x for r in rows for x in r[4]])


def random_batch(seed=11):
    """The batches of test_host_logic.test_intern_columns_equals_the_python_marshaller."""
    rng = random.Random(seed)
    batch = []
    for d, n in enumerate([0, 1, 40, 700, 0, 2500, 13]):
        tasks, _ = random_tasks(rng, n)
        for t in tasks:
            t.id = f"d{d}-{t.id}"
            for dep in t.depends_on:
                if dep.task_id.startswith("t"):
                    dep.task_id = f"d{d}-{dep.task_id}"
        batch.append((M.Distro(id=f"d{d}"), tasks))
    return batch


def edge_batch():
    """Empty strings, "" groups beside named ones, repeated ids, every kind of dependency, prefixes, last-byte twins, NUL
    and non-ASCII bytes, strings above 4 KB, and strings of 0-7 bytes at every alignment of the byte columns."""
    long_a, long_b = "x" * 5000, "x" * 4999 + "y"
    d0 = [("a", "", "", 1, ["b", "missing", "a", "b", "b"]),      # forward, missing, itself, duplicated
          ("b", "v", "g", 2, ["a", "c1", ""]),                      # c1 lives in another distro
          ("a", "v", "g", 2, ["a"]),                                # a repeated id keeps its first index
          ("", "vv", "", 1, [""]),                                  # the empty id is a key like any other
          ("ab", "v\x00", "g\x00", 3, ["a\x00", "ab"]),             # NUL bytes
          ("abc", "v\x00", "gé", 4, ["abc", "ab", "abcd"]),         # prefixes; non-ASCII
          (long_a, long_b, long_a, 5, [long_b, long_a]),            # above 4 KB, differing in the last byte
          (long_b, long_a, long_b, 6, [long_a]),
          ("zz", "", "g", 2, ["é", "zz"])]
    d1 = [("c1", "v", "g", 9, ["a", "c1"]), ("é", "v", "", 0, ["é"])]
    d2 = [("only", "v", "", 0, ["only", "nothing"])]
    # 0-7 byte strings behind a pad of every length 0-7 so that each starts at every offset modulo 8
    d3 = []
    for pad in range(8):
        d3.append(("p" * pad, "q" * pad, "r" * pad if pad else "", 7, []))
        for n in range(8):
            s = "".join(chr(0x61 + (n * 3 + i) % 26) for i in range(n))
            d3.append((s, s, s, 7, [s, "p" * pad]))
    return pack([d0, [], d1, d2, d3, []])


@pytest.fixture(scope="module")
def eng():
    e = scheduler.Engine(0)
    yield e
    e.close()


@pytest.mark.parametrize("bits", [None, "0", "1", "8"])
def test_intern_batch_equals_the_host(eng, monkeypatch, bits):
    if bits is not None:
        monkeypatch.setenv("EVG_INTERN_HASH_BITS", bits)
    want = check_same(eng, S.string_cols(random_batch()))
    assert int(want["dep_off"][-1]) > 50 and int(want["group_off"][-1]) > 20
    want = check_same(eng, edge_batch())
    assert int(want["dep_off"][-1]) > 30 and int(want["group_off"][-1]) > 10
    check_same(eng, pack([]))
    check_same(eng, pack([[], [], []]))
    check_same(eng, pack([[("t", "v", "g", 1, ["t", "u"])]]))
    check_same(eng, pack([[("t", "v", "", 1, [])], [], [("t", "v", "", 1, [])]]))


def test_intern_batch_at_the_bench_shape(eng):
    T, ids, vers, gk, dep_off, tgt = intern_bench.make(100, 10_000)
    sc = S.StringCols.pack(np.arange(101, dtype=np.int64) * 10_000, ids, vers, gk, np.ones(T, np.int32), dep_off, tgt)
    want = check_same(eng, sc)
    assert int(want["dep_off"][-1]) > 60_000 and int(want["group_off"][-1]) > 10_000


def broken(sc: S.StringCols, **kw) -> S.StringCols:
    return dataclasses.replace(sc, **kw)


def test_intern_batch_errors_name_the_table_and_leave_the_context_usable(eng, monkeypatch):
    sc = edge_batch()
    T = sc.n_tasks
    dep_off = sc.dep_off.copy()
    dep_off[3], dep_off[4] = dep_off[4], dep_off[3]           # a row that decreases
    task_off = sc.task_off.copy()
    task_off[2] = task_off[3] + 1                              # distros out of order
    id_off = sc.id[1].copy()
    id_off[5] = id_off[-1] + 1                                 # a string past its byte column
    cases = {"dep_off": broken(sc, dep_off=dep_off), "task_off": broken(sc, task_off=task_off),
             "id.off": broken(sc, id=(sc.id[0], id_off))}
    for name, bad in cases.items():
        rc, msg, _ = device_intern(eng, bad)
        assert rc == L.EVG_ERR_INVALID and "evg_intern_batch" in msg and name in msg, (name, msg)
        check_same(eng, sc)
    # members of one task group that disagree on TaskGroupMaxHosts: the lowest such row is named, also when collisions
    # scramble which row claims the group's slot
    gmax = sc.group_max_hosts.copy()
    rows = [i for i in range(T) if sc.group_key[1][i + 1] > sc.group_key[1][i]]
    key = lambda i: bytes(sc.group_key[0][sc.group_key[1][i]:sc.group_key[1][i + 1]])  # noqa: E731
    twins = [i for i in rows if any(key(j) == key(i) for j in rows if j < i)]
    assert len(twins) >= 2
    for i in twins[-2:]:
        gmax[i] += 100
    bad = broken(sc, group_max_hosts=gmax)
    _, host_msg, _ = host_intern(bad)
    for bits in ("32", "0"):
        monkeypatch.setenv("EVG_INTERN_HASH_BITS", bits)
        rc, msg, _ = device_intern(eng, bad)
        assert rc == L.EVG_ERR_INVALID and f"row {twins[-2]}:" in msg and f"row {twins[-2]}:" in host_msg, (msg, host_msg)
        check_same(eng, sc)
    # a null column and negative sizes fail on the host
    st = sc.struct()
    st.dep_off = None
    out, outs = sc.intern_out()
    assert eng.lib.evg_intern_batch(eng.ctx, C.byref(st), C.byref(outs)) == L.EVG_ERR_INVALID
    st = sc.struct()
    st.n_tasks = -1
    assert eng.lib.evg_intern_batch(eng.ctx, C.byref(st), C.byref(outs)) == L.EVG_ERR_INVALID


# ---------------------------------------------------------------- evg_upload_strings
def string_tick(w: synth.Workload, seed: int):
    """The strings of synthetic tick w (its ids and in-queue edges spelled out, plus dependencies on other distros'
    tasks and on ids no task has) -> (StringCols, the host-interned workload evg_upload takes)."""
    rng = np.random.default_rng(seed)
    t, dt = w.tasks, w.distros
    D, T = dt.n_distros, t.n_tasks
    distro_of = np.repeat(np.arange(D), np.diff(dt.task_off))
    local = np.arange(T) - dt.task_off[distro_of]
    ids = [f"task_{d}_{i:07d}" for d, i in zip(distro_of.tolist(), local.tolist())]
    vers = [f"version_{v}" for v in t.version_id.tolist()]
    gk = [f"group_{g}_bv_proj" if g >= 0 else "" for g in t.group_id.tolist()]
    gmh = np.where(t.group_id >= 0, dt.group_max_hosts[np.maximum(dt.group_off[distro_of] + t.group_id, 0)] if dt.n_groups else 0,
                   rng.integers(0, 5, T)).astype(np.int32)
    deps, dep_off = [], [0]
    for r in range(T):
        d = int(distro_of[r])
        for e in range(int(t.dep_off[r]), int(t.dep_off[r + 1])) if t.n_edges else ():
            deps.append(ids[int(dt.task_off[d]) + int(t.dep_idx[e])])
        if rng.random() < 0.03:
            deps.append(f"task_{(d + 1) % D}_{0:07d}")  # another distro's task (or this one's when D == 1)
        if rng.random() < 0.03:
            deps.append(f"gone_{r}")
        dep_off.append(len(deps))
    sc = S.StringCols.pack(dt.task_off, ids, vers, gk, gmh, np.array(dep_off, np.int64), deps)
    rc, msg, h = host_intern(sc)
    assert rc == L.EVG_OK, msg
    cols = {name: getattr(t, name) for name, _ in S.TaskSoA.COLUMNS}
    cols["group_id"], cols["version_id"] = h["group_id"], h["version_id"]
    tasks = S.TaskSoA(**cols, dep_off=h["dep_off"], dep_idx=h["dep_idx"]).normalize()
    cfg = dt.cfg.copy()
    cfg["n_versions"] = h["n_versions"]
    distros = S.DistroTable(dt.task_off, h["group_off"], cfg, h["group_max_hosts"]).normalize()
    return sc, synth.Workload(w.name, w.now, tasks, distros, w.hosts)


def snap(x):
    if isinstance(x, np.ndarray):
        return x.tobytes(), x.dtype.str, x.shape
    if isinstance(x, dict):
        return {k: snap(v) for k, v in x.items()}
    if isinstance(x, (tuple, list)):
        return [snap(v) for v in x]
    if dataclasses.is_dataclass(x):
        return {f.name: snap(getattr(x, f.name)) for f in dataclasses.fields(x)}
    return x


def outputs(eng, w, opts):
    eng.run(w.now, opts)
    res = [eng.download(want_breakdown=bool(opts & L.EVG_OPT_BREAKDOWN)), eng.download_queue(0, w.distros.task_off)]
    res.append(eng.rebuild_dispatchers(0))
    if w.hosts is not None:
        res.append(eng.host_job(np.zeros(w.distros.n_distros, L.HOST_JOB_CFG_DTYPE)))
    return snap(res)


@pytest.fixture(scope="module")
def tick():
    w = synth.make(np.array([3000, 1, 0, 20, 500, 2500, 13_000, 900, 6000, 300]), 1501, zipf_priority=True, unmet_dep_frac=0.05,
                   met_dep_frac=0.02, tg_frac=0.1, group_versions_frac=0.3, includes_dependencies=True, n_hosts=40)
    return string_tick(w, 1502)


def test_upload_strings_is_upload_of_the_host_interned_table(tick, monkeypatch):
    monkeypatch.setenv("EVG_SPARSE_CLASS", "0")
    sc, wh = tick
    assert wh.tasks.n_edges > 0 and wh.distros.n_groups > 0 and wh.distros.cfg["group_versions"].any()
    a, b = scheduler.Engine(0), scheduler.Engine(0)
    try:
        a.upload(wh.tasks, wh.distros, wh.hosts)
        got = b.upload_strings(wh.tasks, sc, wh.distros.cfg, wh.hosts)
        want = host_intern(sc)[2]
        for k in S.INTERN_OUT_FIELDS:
            assert np.array_equal(got[k], want[k]), k
        for opts in (0, L.EVG_OPT_BREAKDOWN):
            assert outputs(a, wh, opts) == outputs(b, wh, opts)
        po, ao = b.download()
        parity.check_against_oracle(wh, po, ao)
        # the tick stays editable and updatable, and resolves durations, exactly as after evg_upload
        e = synth.next_tick(wh, 1503)
        for eng in (a, b):
            eng.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)
            eng.update_tasks(e.rows, e.values)
        assert outputs(a, e.workload, 0) == outputs(b, e.workload, 0)
        dw = synth.make_duration_cache(e.workload, 1504, n_rows=20_000, n_keys=300)
        for eng in (a, b):
            eng.resolve_durations(dw.history, e.workload.now, dw.tasks, dw.hosts)
        assert snap(a.download_durations()) == snap(b.download_durations())
        assert outputs(a, e.workload, L.EVG_OPT_BREAKDOWN) == outputs(b, e.workload, L.EVG_OPT_BREAKDOWN)
        # planner only, and a tick without tasks
        a.upload(wh.tasks, wh.distros)
        b.upload_strings(wh.tasks, sc, wh.distros.cfg)
        assert outputs(a, dataclasses.replace(wh, hosts=None), 0) == outputs(b, dataclasses.replace(wh, hosts=None), 0)
    finally:
        a.close()
        b.close()


def upload_strings_setup(kind, tick):
    sc, wh = tick

    def run(eng):
        if kind != "ok":
            eng.upload(wh.tasks, wh.distros, wh.hosts)
        bad = sc
        if kind == "host":
            bad = broken(sc, task_off=sc.task_off[::-1].copy())
        elif kind == "device":
            dep_off = sc.dep_off.copy()  # row k decreases; the ends stay, so only the kernel that reads the row sees it
            k = int(np.nonzero(dep_off[2:] < dep_off[-1])[0][0]) + 1
            dep_off[k] = dep_off[k + 1] + 1
            bad = broken(sc, dep_off=dep_off)
        try:
            eng.upload_strings(wh.tasks, bad, wh.distros.cfg, wh.hosts)
            assert kind == "ok"
        except L.EvgError as e:
            assert kind != "ok" and e.code == L.EVG_ERR_INVALID, str(e)
    return run


@pytest.mark.parametrize("kind,row", [("ok", OWN_HOSTS), ("host", OWN_HOSTS), ("device", NONE)])
def test_tick_state_after_upload_strings(tick, kind, row):
    """evg_upload_strings leaves evg_upload's tick; rejected on the host, the previous tick stays; on the device, none."""
    setup = upload_strings_setup(kind, tick)
    got = []
    for probe in PROBES.values():
        eng = scheduler.Engine(0)
        try:
            setup(eng)
            got.append(probe(eng))
        finally:
            eng.close()
    assert got == [CODES[x] for x in row.split()]


def test_launch_count_matches_the_profiler(tick):
    sc, wh = tick
    eng = scheduler.Engine(0)
    try:
        eng.upload(wh.tasks, wh.distros, wh.hosts)
        for fn in (lambda: eng.intern_batch(sc), lambda: eng.upload_strings(wh.tasks, sc, wh.distros.cfg, wh.hosts)):
            names = launched_kernels(fn)
            assert names and eng.last_launch_count() == len(names), names
            assert any(n.startswith("k_in_keys") for n in names)
    finally:
        eng.close()
