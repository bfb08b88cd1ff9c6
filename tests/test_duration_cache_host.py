"""The duration cache without a GPU: the restatement of FetchExpectedDuration (tests/oracle_durations.py) on every
golden case and against the existing oracle, the marshalled key codes, and the new structs' layouts."""
import copy
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import golden_loader
import oracle_durations as OD
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from oracle import oracle as O

GOLD = golden_loader.load("duration_cache.json")
NOW = GOLD["now"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", GOLD["cases"], ids=[c["name"] for c in GOLD["cases"]])
def test_restatement_on_golden_case(case):
    t = OD.golden_task(case["task"])
    before = copy.deepcopy(t)
    got = OD.fetch_expected_duration(t, NOW, OD.golden_finished(case["finished"]))
    assert t == before, "the restatement must not touch the task"
    e = case["expect"]
    assert {k: got[k] for k in e} == e, case["ref"]
    assert got["persisted"] == (e["source"] != OD.FRESH)
    assert got["ttl"] == (case["task"]["prediction"]["ttl"] or M.PREDICTION_TTL)


def test_golden_covers_every_source():
    assert {c["expect"]["source"] for c in GOLD["cases"]} == {OD.FRESH, OD.BACKFILL, OD.HISTORY, OD.PREVIOUS, OD.DEFAULT}
    assert sum(c["kind"] == "asserted" for c in GOLD["cases"]) == 2


def _random_world(rng: random.Random, n_tasks: int, names=("a", "b", "c")):
    finished = []
    for i in range(rng.randrange(0, 40)):
        taken = rng.choice([0, 1, 7, 10 * M.MINUTE, 10 * M.MINUTE + rng.randrange(1000), rng.randrange(1, 3 * M.HOUR)])
        fin = NOW - rng.choice([0, 1, M.HOUR, 6 * 24 * M.HOUR, 7 * 24 * M.HOUR, 8 * 24 * M.HOUR])
        finished.append(M.Task(id=f"f{i}", project=rng.choice(["p", "q"]), build_variant=rng.choice(["x", "y"]),
                               display_name=rng.choice(names), status=rng.choice(["success", "failed", "started"]),
                               timed_out=rng.random() < 0.1, time_taken=taken, finish_time=fin,
                               start_time=fin - taken))
    tasks = []
    for i in range(n_tasks):
        pred = M.CachedDurationValue(
            value=rng.choice([0, 0, 7 * M.MINUTE, 1]), std_dev=rng.choice([0, 3 * M.MINUTE]),
            ttl=rng.choice([0, 0, M.HOUR, 1]),
            collected_at=rng.choice([M.ZERO_TIME, NOW, NOW + M.HOUR, NOW - M.HOUR, NOW - 8 * M.HOUR, NOW - 9 * M.HOUR]))
        tasks.append(M.Task(id=f"t{i}", project=rng.choice(["p", "q", "r"]), build_variant=rng.choice(["x", "y"]),
                            display_name=rng.choice(names), expected_duration=rng.choice([0, 0, 12 * M.MINUTE]),
                            expected_duration_std_dev=rng.choice([0, M.MINUTE]), duration_prediction=pred))
    return finished, tasks


@pytest.mark.parametrize("seed", range(6))
def test_restatement_agrees_with_the_oracle(seed):
    """Without empty display names the name-filtered query returns the key's own statistics: the restatement and
    O.fetch_expected_duration over O.expected_durations_for_window agree on every returned pair."""
    rng = random.Random(seed)
    finished, tasks = _random_world(rng, 300)
    stats = O.expected_durations_for_window(finished, NOW - OD.WINDOW, NOW)
    for t in tasks:
        got = OD.fetch_expected_duration(t, NOW, finished)
        st = stats.get((t.project, t.build_variant, t.display_name))
        want = O.fetch_expected_duration(copy.deepcopy(t), NOW, None if st is None else (st[1], st[2]))
        assert (got["avg"], got["std"]) == want, t
        # the host mirror writes the same DurationPrediction back
        m = copy.deepcopy(t)
        M.fetch_expected_duration(m, NOW, None if st is None else (st[1], st[2]))
        assert (m.duration_prediction.value, m.duration_prediction.std_dev, m.duration_prediction.collected_at) == \
            (got["value"], got["pred_std"], got["collected"])


def test_history_keys_are_pair_major():
    rng = random.Random(3)
    finished, tasks = _random_world(rng, 50, names=("a", "b", ""))
    tasks.append(M.Task(id="nokey", project="zz", build_variant="x", display_name="a"))
    tasks.append(M.Task(id="nopair", project="zz", build_variant="x", display_name=""))
    hist, codes = S.marshal_duration_history(finished, tasks, NOW)
    assert hist.rows.window_start_ns == NOW - OD.WINDOW and hist.rows.window_end_ns == NOW
    off = hist.pair_key_off
    assert off[0] == 0 and off[-1] == hist.rows.n_keys == len(hist.keys) and np.all(np.diff(off) >= 0)
    for (proj, bv), p in hist.pairs.items():
        ks = hist.keys[off[p]:off[p + 1]]
        assert ks and all(k[:2] == (proj, bv) for k in ks)
        assert len(set(ks)) == len(ks)
    for f, k in zip(finished, hist.rows.key):
        assert hist.keys[k] == (f.project, f.build_variant, f.display_name)
    for t, c in zip(tasks, codes):
        if t.display_name == "":
            p = hist.pairs.get((t.project, t.build_variant))
            assert c == (L.EVG_DK_NONE if p is None else L.EVG_DK_PAIR(p))
        else:
            k = (t.project, t.build_variant, t.display_name)
            assert c == (hist.keys.index(k) if k in hist.keys else L.EVG_DK_NONE)
    assert codes[-2] == L.EVG_DK_NONE and codes[-1] == L.EVG_DK_NONE


def test_marshal_duration_cache_reads_only():
    finished, tasks = _random_world(random.Random(5), 40)
    hist, codes = S.marshal_duration_history(finished, tasks, NOW)
    before = copy.deepcopy(tasks)
    c = S.marshal_duration_cache(tasks, hist, rows=[1, 4, 9])
    assert tasks == before
    assert c.rows.tolist() == [1, 4, 9] and c.key.tolist() == [codes[1], codes[4], codes[9]]
    assert c.value_ns.tolist() == [tasks[i].duration_prediction.value for i in (1, 4, 9)]
    assert c.collected_ns.tolist() == [tasks[i].duration_prediction.collected_at for i in (1, 4, 9)]
    full = S.marshal_duration_cache(tasks, hist)
    assert full.rows is None and full.n_rows == 40 and full.key.tolist() == codes.tolist()


def test_marshal_tasks_opt_out_leaves_tasks_alone():
    _, tasks = _random_world(random.Random(6), 30)
    before = copy.deepcopy(tasks)
    soa, _, _ = S.marshal_tasks([(M.Distro(id="d"), tasks)], NOW, resolve_durations=False)
    assert tasks == before
    assert soa.expected_ns.tolist() == [t.expected_duration for t in tasks]


def test_struct_layouts(tmp_path):
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "evg_sched.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(evg_duration_cache), offsetof(evg_duration_cache, rows),
         offsetof(evg_duration_cache, expected_std_ns), offsetof(evg_duration_cache, key), sizeof(evg_duration_in));
  printf("%zu %zu %zu %zu %zu %zu\n", offsetof(evg_duration_in, n_pairs), offsetof(evg_duration_in, pair_key_off),
         offsetof(evg_duration_in, tasks), offsetof(evg_duration_in, hosts), sizeof(evg_duration_out),
         offsetof(evg_duration_out, source));
  printf("%d %d %d %d %d %d %d\n", EVG_DK_NONE, EVG_DK_PAIR(0), EVG_DK_PAIR(5), EVG_DS_FRESH, EVG_DS_BACKFILL,
         EVG_DS_PREVIOUS, EVG_DS_DEFAULT);
  return 0;
}'''
    c = tmp_path / "t.c"
    c.write_text(prog)
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    out = [[int(x) for x in line.split()] for line in subprocess.check_output([str(exe)]).decode().strip().split("\n")]
    DC, DI, DO = L.DurationCacheStruct, L.DurationInStruct, L.DurationOutStruct
    assert out[0] == [ctypes.sizeof(DC), DC.rows.offset, DC.expected_std_ns.offset, DC.key.offset, ctypes.sizeof(DI)]
    assert out[1] == [DI.n_pairs.offset, DI.pair_key_off.offset, DI.tasks.offset, DI.hosts.offset, ctypes.sizeof(DO),
                      DO.source.offset]
    assert out[2] == [L.EVG_DK_NONE, L.EVG_DK_PAIR(0), L.EVG_DK_PAIR(5), L.EVG_DS_FRESH, L.EVG_DS_BACKFILL,
                      L.EVG_DS_PREVIOUS, L.EVG_DS_DEFAULT]
