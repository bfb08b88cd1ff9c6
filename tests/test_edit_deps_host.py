"""The resident dependency table without a GPU: over seeded multi-tick scripts, soa.DepsShim's dependency edit composed
by soa.apply_deps_edit (what evg_edit_tasks_with_deps builds on the device) gives every task the DependenciesMet
verdict and DependenciesMetTime stamp a fresh soa.marshal_deps of the composed batch gives, and the Go restatement
soa.dependencies_met agrees; plus the rejected inputs, the struct layout and the exported symbol."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import edit_deps_scripts as X
from evergreen_b200 import _lib as L
from evergreen_b200 import soa as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_script(seed, sizes, ticks):
    """-> (ticks expressed as an edit, ticks uploaded); asserts equality at every tick."""
    sc = X.Script(seed, sizes)
    shim = S.DepsShim(sc.db)
    canon = [(d, list(ts)) for d, ts in sc.batch]
    deps, fin = shim.upload(canon)
    met, stamp = S.deps_verdicts(deps, fin, X.NOW)
    assert np.array_equal(met, X.host_verdicts(canon, sc.db))
    X.write_back(canon, stamp)
    shim.remember(canon)
    prev_ids, prev_off = X.ids_of(canon), X.task_off(canon)
    n_edit = n_upload = 0
    for tick in range(ticks):
        now = X.NOW + (tick + 1) * 10 ** 11
        canon = X.canonical(prev_ids, sc.step(tick))
        remove, ins_off = X.edit_rows(prev_ids, canon)
        dx = shim.edit(prev_ids, canon, remove)
        fresh, fresh_fin = S.marshal_deps(canon, sc.db), S.marshal_dep_finished(canon)
        if dx is None:
            n_upload += 1
            deps, fin = shim.upload(canon)
        else:
            n_edit += 1
            stub = S.TaskEdit(remove, None, ins_off, np.zeros(0, np.int64), np.zeros(0, np.int32))
            deps, fin = S.apply_deps_edit(deps, prev_off, stub, dx, fin, stamp)
        got_met, got_stamp = S.deps_verdicts(deps, fin, now)
        want_met, want_stamp = S.deps_verdicts(fresh, fresh_fin, now)
        assert np.array_equal(got_met, want_met), (seed, tick)
        assert np.array_equal(got_stamp, want_stamp), (seed, tick)
        assert np.array_equal(got_met, X.host_verdicts(canon, sc.db)), (seed, tick)
        # the tables differ only in external ids: the same entries per task, the same task_state / task_pre
        assert np.array_equal(deps.dep_off, fresh.dep_off) and np.array_equal(deps.dep_want, fresh.dep_want)
        assert np.array_equal(deps.task_state, fresh.task_state) and np.array_equal(deps.task_pre, fresh.task_pre)
        inq = fresh.dep_kind == L.EVG_DEP_IN_QUEUE
        assert np.array_equal(deps.dep_kind[inq], fresh.dep_kind[inq]) and np.array_equal(deps.dep_ref[inq], fresh.dep_ref[inq])
        X.write_back(canon, got_stamp)
        stamp = got_stamp
        shim.remember(canon)
        prev_ids, prev_off = X.ids_of(canon), X.task_off(canon)
    return n_edit, n_upload


@pytest.mark.parametrize("seed", range(6))
def test_scripts_compose_what_a_fresh_marshal_evaluates(seed):
    n_edit, _ = run_script(seed, [1, 7, 40, 90], ticks=8)
    assert n_edit >= 4


def test_a_longer_script_on_one_big_queue():
    n_edit, _ = run_script(99, [600], ticks=6)
    assert n_edit >= 3


def tiny():
    """Distro 0: rows 0 (no deps), 1 -> 0 in-queue, 2 -> external 0; distro 1: row 3 -> row 2 (another distro)."""
    deps = S.DepsTable(np.array([0, 0, 1, 2, 3], np.int64), np.array([0, 1, 0], np.uint8), np.array([0, 0, 2], np.int32),
                       np.zeros(3, np.uint8), np.full(4, 2, np.uint8), np.zeros(4, np.uint8), np.array([0], np.uint8))
    return deps, np.array([0, 3, 4], np.int64)


def empty_edit(n_remove, n_ext=1, **kw):
    e0 = np.zeros(0, np.int64)
    x = S.DepsEdit(np.full(n_remove, -1, np.int32), np.zeros(n_ext, np.uint8),
                   S.DepsTable(np.zeros(1, np.int64), *(np.zeros(0, t) for t in (np.uint8, np.int32, np.uint8, np.uint8, np.uint8, np.uint8))),
                   e0, np.zeros(0, np.uint8), np.zeros(0, np.int32), np.zeros(0, np.uint8), e0, np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    for k, v in kw.items():
        setattr(x, k, v)
    return x


def test_apply_deps_edit_by_hand():
    deps, toff = tiny()
    # row 0 leaves as external id 1 (finished at 77), row 3's in-queue ref to row 2 moves to row 1; the stamp of row 1 is
    # written back; the new external table has two ids
    edit = S.TaskEdit(np.array([0]), None, np.array([0, 0, 0]), np.zeros(0, np.int64), np.zeros(0, np.int32))
    x = empty_edit(1, n_ext=2, depart_ext=np.array([1], np.int32), depart_finished=np.array([77], np.int64))
    stamp = np.array([L.EVG_TIME_ZERO, 5, L.EVG_TIME_ZERO, L.EVG_TIME_ZERO], np.int64)
    got, fin = S.apply_deps_edit(deps, toff, edit, x, None, stamp)
    assert got.dep_off.tolist() == [0, 1, 2, 3]
    assert got.dep_kind.tolist() == [1, 1, 0] and got.dep_ref.tolist() == [1, 0, 1]
    assert fin.tolist() == [77, L.EVG_TIME_ZERO, L.EVG_TIME_ZERO]
    assert got.task_pre.tolist() == [L.EVG_TP_MET_TIME, 0, 0]


def test_apply_deps_edit_rejects_what_the_device_rejects():
    deps, toff = tiny()
    edit = S.TaskEdit(np.array([0]), None, np.array([0, 0, 0]), np.zeros(0, np.int64), np.zeros(0, np.int32))
    with pytest.raises(ValueError, match="depart_ext is -1"):
        S.apply_deps_edit(deps, toff, edit, empty_edit(1))
    with pytest.raises(ValueError, match="external ref"):
        S.apply_deps_edit(deps, toff, S.TaskEdit(np.array([3]), None, np.array([0, 0, 0]), np.zeros(0, np.int64),
                                                 np.zeros(0, np.int32)), empty_edit(1, n_ext=0))


def test_exports_the_new_symbol():
    assert "evg_edit_tasks_with_deps" in L.SYMBOLS
    header = open(os.path.join(ROOT, "include", "evg_sched.h")).read()
    assert "int evg_edit_tasks_with_deps(" in header


def test_deps_edit_struct_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "evg_sched.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(evg_deps_edit), offsetof(evg_deps_edit, n_ext), '
                   'offsetof(evg_deps_edit, insert), offsetof(evg_deps_edit, n_add), offsetof(evg_deps_edit, set_pre));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    S_ = L.DepsEditStruct
    assert got == [ctypes.sizeof(S_), S_.n_ext.offset, S_.insert.offset, S_.n_add.offset, S_.set_pre.offset]
