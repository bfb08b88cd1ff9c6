"""The alias side without a GPU: find_host_schedulable_for_alias rule by rule, the layout marshal_aliases gives the
device, the host restatement of the queues it builds, and the ctypes mirrors of evg_alias_in / evg_alias_out."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_alias import NOW, rule_tick

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ids(tasks):
    return [t.id for t in tasks]


def test_find_host_schedulable_for_alias_rule_by_rule():
    distros, tasks, _ = rule_tick()
    find = scheduler.find_host_schedulable_for_alias
    # t0 names d1 and a1 (an alias of d1 too): once; t1 names its own distro; t2/t3 single-host; t4-t8 fail the base
    # query; t9 is unattainable but overridden; t10 names nothing known; t14 names nothing
    assert ids(find("d0", tasks, distros)) == ["t0", "t1"]
    assert ids(find("d1", tasks, distros)) == ["t0", "t9", "t11", "t12", "t13", "t15", "t16"]
    assert ids(find("d2", tasks, distros)) == []
    assert ids(find("d3", tasks, distros)) == []
    with pytest.raises(LookupError):
        find("missing", tasks, distros)
    # the distro's own id applies without being listed among its aliases
    solo = [M.Distro(id="x")]
    assert ids(find("x", [M.Task(id="a", secondary_distros=["x"])], solo)) == ["a"]


def test_marshal_aliases_layout():
    distros, tasks, db = rule_tick()
    at, cfg, keys = S.marshal_aliases(distros, tasks, NOW, db)
    names = ["d0", "a1", "d1", "a2", "d2", "d3", "nobody-uses-this"]
    assert at.n_names == len(names)
    assert at.dest_off.tolist() == [0, 1, 3, 4, 5, 6, 7, 8]
    assert at.dest_idx.tolist() == [0, 0, 1, 1, 1, 2, 3, 3]
    assert at.secondary_off.tolist()[:3] == [0, 2, 3]
    assert at.secondary_idx.tolist()[:3] == [names.index("d1"), names.index("a1"), names.index("d0")]
    assert int(at.secondary_idx[at.secondary_off[10]]) == -1          # "zzz"
    assert at.primary.tolist()[11:13] == [0, 2] and int(at.primary[16]) == -1
    assert cfg.shape[0] == 4 and (cfg["n_versions"] == 0).all()
    # task groups and versions are interned once over the table: t11 and t12 share the group of "tg"
    assert int(at.tasks.group_id[11]) == int(at.tasks.group_id[12]) >= 0
    assert keys.group_names[int(at.tasks.group_id[11])] == "tg_bv_p_vx"
    assert int(at.group_max_hosts[int(at.tasks.group_id[11])]) == 3 and at.n_versions == len(keys.versions)
    assert at.task_group_max_hosts.tolist()[2:4] == [1, 1]
    assert not (at.tasks.flags & (L.EVG_TF_OTHER_DISTRO | L.EVG_TF_DEPS_MET)).any()
    assert at.sched[4] & L.EVG_SQ_ACTIVATED == 0 and at.sched[8] & L.EVG_SQ_UNATTAINABLE
    # edges: DependsOn entries that are rows of the table, as row indices, duplicates kept
    e = lambda i: at.tasks.dep_idx[at.tasks.dep_off[i]:at.tasks.dep_off[i + 1]].tolist()  # noqa: E731
    assert e(13) == [14, 9] and e(15) == [9, 9] and e(9) == []          # "done" is not a row of the table
    # dependencies: in-table ones refer to rows, the rest to the tasks collection
    d = at.deps
    assert d.dep_kind[d.dep_off[9]] == L.EVG_DEP_EXTERNAL and d.dep_ref[d.dep_off[13]] == 14


def test_alias_queues_restate_the_finder():
    distros, tasks, db = rule_tick()
    at, cfg, _ = S.marshal_aliases(distros, tasks, NOW, db)
    queues = S.alias_queues(at, len(distros))
    for d, q in zip(distros, queues):
        assert [tasks[int(i)].id for i in q] == ids(scheduler.find_host_schedulable_for_alias(d.id, tasks, distros))
    soa, table, deps, fin, src, gsrc = S.compose_aliases(at, cfg)
    assert table.task_off.tolist() == [0, 2, 9, 9, 9]
    assert src.tolist() == [0, 1, 0, 9, 11, 12, 13, 15, 16]
    assert (soa.flags[:2] & L.EVG_TF_OTHER_DISTRO == 0).all() and (soa.flags[2:] & L.EVG_TF_OTHER_DISTRO != 0).all()
    assert table.group_off.tolist() == [0, 0, 1, 1, 1] and gsrc.tolist() == [int(at.tasks.group_id[11])]
    assert soa.dep_idx.tolist() == [1, 1, 1]                            # t13 -> t9; t15 -> t9 twice
    assert deps.n_tasks == 9 and int(table.cfg["n_versions"][1]) == len({tasks[int(i)].version for i in src[2:]})


def test_synthetic_alias_tick_covers_the_rules():
    w = synth.make(np.array([1, 20, 700, 3000, 14000]), 11, tg_frac=0.2, met_dep_frac=0.05)
    at, cfg = synth.make_aliases(w, 12, big=13000)
    n = np.diff(at.secondary_off)
    assert n.max() >= 3 and (n == 0).any() and (at.secondary_idx == -1).any()
    assert (np.diff(at.dest_off)[w.distros.n_distros:] > 1).any()       # an alias name several distros share
    assert (at.task_group_max_hosts == 1).any() and ((at.task_group_max_hosts == 1) & (at.tasks.group_id < 0)).any()
    assert (at.sched & L.EVG_SQ_UNATTAINABLE).any() and ((at.sched & S.SQ_BASE) != S.SQ_BASE).any()
    queues = S.alias_queues(at, w.distros.n_distros)
    assert max(len(q) for q in queues) > 12288
    own = [np.isin(q, np.nonzero(at.primary == e)[0]).any() for e, q in enumerate(queues)]
    assert any(own)                                                      # a task in its own distro's alias queue


def test_struct_layouts_match_the_header(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(evg_alias_in), offsetof(evg_alias_in, n_groups),
         offsetof(evg_alias_in, secondary_idx), offsetof(evg_alias_in, n_names), offsetof(evg_alias_in, dest_off),
         offsetof(evg_alias_in, deps), offsetof(evg_alias_in, dep_finished_ns), sizeof(evg_alias_out));
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    A = L.AliasInStruct
    assert got == [ctypes.sizeof(A), A.n_groups.offset, A.secondary_idx.offset, A.n_names.offset, A.dest_off.offset,
                   A.deps.offset, A.dep_finished_ns.offset, ctypes.sizeof(L.AliasOutStruct)]
