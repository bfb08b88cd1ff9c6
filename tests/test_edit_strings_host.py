"""Without a GPU: soa.compose_strings (the host mirror of evg_edit_strings' composed string table), the ctypes mirror of
evg_string_edit, and the call's argument guard."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S

import edit_strings_scripts as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same_cols(a: S.StringCols, b: S.StringCols):
    assert np.array_equal(a.task_off, b.task_off) and np.array_equal(a.dep_off, b.dep_off)
    assert np.array_equal(a.group_max_hosts, b.group_max_hosts)
    for name in ("id", "version", "group_key", "dep_id"):
        assert bytes(getattr(a, name)[0]) == bytes(getattr(b, name)[0]), name
        assert np.array_equal(getattr(a, name)[1], getattr(b, name)[1]), name


@pytest.mark.parametrize("seed", range(3))
def test_compose_then_intern_equals_marshal_of_the_composed_batch(seed):
    sc = X.Script(400 + seed)
    prev = sc.batch
    old = S.string_cols(prev)
    seen = set()
    for step in range(6):
        kw = dict(empty={4, 6} if step == 2 else (), replace_all={2} if step == 3 else ())
        batch = sc.next_batch(leave=0.0 if step == 4 else 0.15, arrive=0.0 if step == 4 else 0.15, **kw)
        toff = np.concatenate([[0], np.cumsum([len(ts) for _, ts in prev])])
        edit = X.string_edit(prev, batch, toff)
        composed = S.compose_strings(old, edit)
        same_cols(composed, S.string_cols(batch))
        soa, table, keys = S.marshal_tasks(batch, X.NOW)
        out, outs = composed.intern_out()
        assert L.load().evg_intern_columns(ctypes.byref(composed.struct()), ctypes.byref(outs), 2) == L.EVG_OK, L.last_error()
        out = composed.trim(out)
        assert np.array_equal(out["group_id"], soa.group_id) and np.array_equal(out["version_id"], soa.version_id)
        assert np.array_equal(out["group_off"], table.group_off) and np.array_equal(out["group_max_hosts"], table.group_max_hosts)
        assert out["n_versions"].tolist() == [len(k.versions) for k in keys]
        assert np.array_equal(out["dep_off"], soa.dep_off if soa.dep_off is not None else np.zeros(soa.n_tasks + 1, np.int64))
        if soa.dep_idx is not None:
            assert np.array_equal(out["dep_idx"], soa.dep_idx)
        if edit.remove_rows.shape[0] == 0 and edit.strings.n_tasks == 0:
            seen.add("empty edit")
        if any(len(ts) == 0 and len(o) > 0 for (_, ts), (_, o) in zip(batch, prev)):
            seen.add("emptied distro")
        prev, old = batch, composed
    assert seen == {"empty edit", "emptied distro"}


def test_marshal_without_interning_keeps_the_numeric_columns():
    batch = X.Script(7).batch
    full, _, _ = S.marshal_tasks(batch, X.NOW)
    bare, table, keys = S.marshal_tasks(batch, X.NOW, intern=False)
    for name in ("priority", "expected_ns", "queue_basis_ns", "wait_basis_ns", "num_dependents", "task_group_order", "flags"):
        assert np.array_equal(getattr(full, name), getattr(bare, name)), name
    assert (bare.group_id == -1).all() and (bare.version_id == 0).all() and bare.n_edges == 0
    assert table.n_groups == 0 and all(k.group_names == [] and k.versions == [] for k in keys)


def test_string_edit_struct_layout_matches_the_header(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(evg_string_edit), offsetof(evg_string_edit, n_remove),
         offsetof(evg_string_edit, remove_rows), offsetof(evg_string_edit, insert), offsetof(evg_string_edit, insert_off),
         offsetof(evg_string_edit, strings));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    St = L.StringEditStruct
    assert got == [ctypes.sizeof(St), St.n_remove.offset, St.remove_rows.offset, St.insert.offset, St.insert_off.offset,
                   St.strings.offset]


def test_struct_points_at_the_edit():
    batch = X.Script(8).batch
    nxt = X.Script(8)
    nxt.batch = batch
    new = nxt.next_batch()
    edit = X.string_edit(batch, new, np.concatenate([[0], np.cumsum([len(ts) for _, ts in batch])]))
    st, keep = edit.struct()
    assert st.n_remove == edit.remove_rows.shape[0] and st.insert_off == L.ptr(edit.strings.task_off)
    assert st.insert.contents.group_id is None and st.insert.contents.dep_off is None
    assert st.insert.contents.n_tasks == edit.strings.n_tasks == st.strings.contents.n_tasks
    assert edit.nbytes() > 0


def test_null_context_and_arguments_are_rejected():
    lib = L.load()
    assert lib.evg_edit_strings(None, None, None, None, None, None, None) == L.EVG_ERR_INVALID
    assert L.last_error() == "evg_edit_strings: null context"


def test_device_strings_cannot_be_combined_with_device_deps():
    with pytest.raises(ValueError):
        scheduler.ResidentTick(device_deps=True, device_strings=True)
