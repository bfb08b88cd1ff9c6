"""The edge ticks of test_gpu_tick_report_edges land where their comments say, checked without a GPU against the CPU
oracle's planner and allocator and the restatement oracle_host_job: each crafted evg_host_job case reaches its branch,
ratio bits, ulp or saturation; the warp-sum layouts put wide distros on the stated lanes; every score-edge tick reaches
what it exists for."""
import numpy as np
import pytest

import oracle_host_job as OJ
import test_gpu_tick_report_edges as E
from evergreen_b200 import _lib as L
from oracle import oracle as O
from test_gpu_host_job import restate


def oracle_run(w):
    ref = O.SoAJob(w.tasks, w.distros, w.hosts).run(w.now, 8)
    return ref, E.oracle_plan(w, ref)


def test_crafted_cases_land():
    cases = E.EDGE_CASES
    w, job = E.crafted_tick(cases)
    ref, plan = oracle_run(w)
    assert (ref["status"] == L.EVG_ALLOC_OK).all()
    assert list(ref["free_hosts"]) == [c.n_up for c in cases]  # idle hosts are free hosts
    given = E.given_spawned(w, cases, job, plan)
    with_given = restate(*plan, w.distros.group_off, w.hosts, job, given)
    with_null = restate(*plan, w.distros.group_off, w.hosts, job, None)
    for d, c in enumerate(cases):
        r = with_null[d] if c.null else with_given[d]
        assert c.lands(r), (c.name, r)
        assert r["report"]["time_to_empty_ns"] >= 0  # sched > 0 and hosts_avail > 0 there: no quotient below zero
    ratios = [r["report"]["host_queue_ratio"] for r in with_given]
    # NaN, +Inf and -0.0 occur; -Inf cannot: the time to empty is never negative and float32(threshold) is never -0
    assert any(np.isnan(x) for x in ratios) and any(np.isposinf(x) for x in ratios)
    assert 0x80000000 in {OJ.float_bits(x) for x in ratios}
    assert {0x3E800000, 0x3E7FFFFF} <= {OJ.float_bits(x) for x in ratios}
    # the single-task distros' groups do need hosts in the allocator's rows: the job leaves them out
    goff = w.distros.group_off
    for d, c in enumerate(cases):
        if c.single:
            assert plan[0].group_info["count_required"][int(goff[d]):int(goff[d + 1])].sum() > 0, c.name


@pytest.mark.parametrize("name", list(E.LAYOUTS))
def test_warp_layouts_land(name):
    n, wide, singles, big = E.LAYOUTS[name]
    cases = E.layout_cases(name)
    w, job = E.crafted_tick(cases)
    slots = np.diff(w.distros.group_off)
    assert len(slots) == n
    is_wide = slots > 16  # kHostJobWarpGroups
    lanes = {d % 32 for d in np.nonzero(is_wide)[0]}
    assert 0 in lanes
    if n >= 32:
        assert 31 in lanes
    if n % 32:
        assert is_wide[n - n % 32:].any()  # the partial last warp holds a wide distro
    ref, plan = oracle_run(w)
    goff = w.distros.group_off
    for d in big:  # the wrap, on the path the distro's slot count picks
        _, job_sum = E.wrapped_group_sums(w, d)
        assert not -2 ** 63 <= job_sum <= E.I64_MAX
    for d in singles:
        if is_wide[d]:
            assert plan[0].group_info["count_required"][int(goff[d]):int(goff[d + 1])].sum() > 0
    if name == "n95":
        assert is_wide[:32].all()  # one warp of wide distros only
        assert {16, 17} <= set(slots.tolist()) and (slots > 32).sum() >= 3  # > 32 slots: lanes stride past one pass
        assert {bool(is_wide[d]) for d in big} == {True, False}  # wrapping sums on both paths
        assert any(is_wide[d] and d in singles for d in range(n)) and any(is_wide[d] and d not in singles for d in range(32, 64))


@pytest.mark.parametrize("route,kind,density", E.EDGE_TICKS)
def test_edge_ticks_reach_their_rows(route, kind, density):
    w, rows = E.report_edge_tick(route, kind, density)
    E.reaches(w, kind, rows)
