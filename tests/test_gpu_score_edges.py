"""The planner's tiered scorer outside synth.make's domain, on every route.

The hot kernels score a task with 32-bit arithmetic when the whole warp is inside its domain (evg_score.cuh
score32_bad), else with the 64-bit fast form, else with the literal Go arithmetic; each warp votes.  These ticks put
edge values (synth.sprinkle_edges) next to ordinary tasks, one per warp stretch or densely, so that mixed warps reach
every fallback, and compare each tick with the oracle: ranked order, TotalValue, queue info, allocator decisions and
the 13-field breakdown.  test_host_logic.py checks on the CPU that every tick built here really holds mixed warps."""
import copy

import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import soa, synth

pytestmark = pytest.mark.gpu

# k_plan_cta instances <THREADS, CAP> (evg_sched.cu kNT_* / kNCap*): a tile is 2 * THREADS task slots
CTA_CLASSES = ((384, 64), (1280, 128), (5120, 256), (10240, 512))
GTASK_TILE, GTASK_WARP = 2048, 128  # k_gtask: 2048-slot tiles, a warp scores 128 consecutive slots (4 per lane)


def cta_threads(n):
    return next(th for cap, th in CTA_CLASSES if n <= cap)


def _route_tick(route, seed):
    """The tick of one route, before any edge is sprinkled (see ROUTES)."""
    if route == "warp":  # <= 32 tasks: one warp per distro
        sizes = np.concatenate([[32, 31, 1, 2], synth.Rng(seed).integers(120, 1, 32)])
        return synth.make(sizes, seed, zipf_priority=True, tg_frac=0.08, group_versions_frac=0.2, met_dep_frac=0.01,
                          unmet_dep_frac=0.01, includes_dependencies=True, custom_factor_frac=0.3, n_hosts=150,
                          providers=(0.6, 0.2, 0.2))
    if route == "cta":  # every k_plan_cta instance, several distros each, every start residue mod 4
        sizes = np.array([65, 383, 384, 130, 1279, 1001, 1280, 385, 3003, 5120, 4097, 1282, 9001, 10240, 10239, 5119, 7002, 257])
        return synth.make(sizes, seed, zipf_priority=True, tg_frac=0.12, custom_factor_frac=0.3, n_hosts=150,
                          providers=(0.7, 0.2, 0.1))
    if route == "smem":  # GroupVersions, in-queue dependencies, the 10241..12288 class (with the sparse-class rule off)
        sizes = np.array([3000, 3001, 11000, 12288, 10241, 2000])
        w = synth.make(sizes, seed, zipf_priority=True, tg_frac=0.12, met_dep_frac=0.02, unmet_dep_frac=0.02,
                       includes_dependencies=True, custom_factor_frac=0.3, n_hosts=120)
        w.distros.cfg["group_versions"][[0, 4]] = 1
        return w
    if route == "general":  # > 12288 tasks: k_gtask, the unit kernels, the radix sort
        sizes = np.array([13001, 20003, 16002, 12289])
        w = synth.make(sizes, seed, zipf_priority=True, tg_frac=0.1, met_dep_frac=0.02, unmet_dep_frac=0.02,
                       includes_dependencies=True, custom_factor_frac=0.3, n_hosts=120)
        w.distros.cfg["group_versions"][2] = 1
        return w
    raise ValueError(route)


def vote_layout(route, n):
    """(warp stretch, tile, aligned) in task slots of a distro of n tasks on this route; aligned: slots count from the
    distro's first task rounded down to a multiple of four, as the TMA tiles and the vector loads do, else from it."""
    if route == "cta":
        return 32, 2 * cta_threads(n), True
    if route == "general":
        return GTASK_WARP, GTASK_TILE, True
    return 32, 32, False


def sparse_rows(w, route):
    """One edge row per warp stretch -- at its first lane, its last lane and a lane between, in turn -- plus the first
    and the last slot of every tile."""
    toff = w.distros.task_off
    rows = []
    for d in range(w.distros.n_distros):
        a, b = int(toff[d]), int(toff[d + 1])
        stretch, tile, aligned = vote_layout(route, b - a)
        a0 = a & ~3 if aligned else a
        for k, s in enumerate(range(a0, b, stretch)):
            rows.append(s + (0, stretch - 1, (7 * k + 3) % stretch)[k % 3])
        for s in range(a0, b, tile):
            rows += [s, s + tile - 1]
    rows = np.array(rows, dtype=np.int64)
    distro = np.searchsorted(toff, rows, side="right") - 1
    inside = (rows >= 0) & (rows < w.n_tasks)
    inside[inside] &= rows[inside] >= toff[distro[inside]]
    return rows[inside]


ROUTES = ("warp", "cta", "smem", "general")
KINDS = synth.ROW_KINDS
DENSITIES = ("sparse", "dense")


def edge_tick(route, kind, density):
    """One route's tick with `kind` sprinkled at `density`, the distro-level knobs dealt to its distros."""
    seed = 500 + 17 * ROUTES.index(route) + KINDS.index(kind)
    w = _route_tick(route, seed)
    kw = dict(positions=sparse_rows(w, route)) if density == "sparse" else dict(frac=0.3)
    synth.sprinkle_edges(w, seed, kinds=(kind,) + synth.DISTRO_KINDS, **kw)
    return w


def run(engine, w, breakdown=False):
    if w.hosts is not None:
        return engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now, breakdown=breakdown)
    return engine.plan_batch(w.tasks, w.distros, w.now, breakdown=breakdown), None


def check_tick(engine, w):
    """The oracle (with hosts), the size-independent properties, and the breakdown rerun field for field."""
    po, ao = run(engine, w)
    parity.check_against_oracle(w, po, ao)
    parity.check_properties(w, po, ao)
    order, tv = po.order.copy(), po.total_value.copy()
    pb, _ = run(engine, w, breakdown=True)
    assert np.array_equal(pb.order, order) and np.array_equal(pb.total_value, tv)
    ref = parity.check_against_oracle(w, pb, None)
    assert np.array_equal(pb.breakdown, ref["breakdown"])
    return tv


def value_ranges(w, tv):
    toff = w.distros.task_off
    return [int(tv[toff[d]:toff[d + 1]].max()) - int(tv[toff[d]:toff[d + 1]].min()) if toff[d + 1] > toff[d] else 0
            for d in range(w.distros.n_distros)]


@pytest.mark.parametrize("density", DENSITIES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("route", ROUTES)
def test_score_edges(engine, monkeypatch, route, kind, density):
    if route == "smem":
        monkeypatch.setenv("EVG_SPARSE_CLASS", "0")  # keep the 4097+ task classes on k_plan_smem
    w = edge_tick(route, kind, density)
    tv = check_tick(engine, w)
    ranges = value_ranges(w, tv)
    if kind == "u32" and route in ("warp", "cta"):
        # just past the u32 key of k_plan_cta, which hands such distros to k_plan_smem: a 33-bit range there (on the
        # other routes in-queue dependency units and GroupVersions fold the row into wider units)
        assert any(2 ** 32 <= r < 2 ** 33 for r in ranges), ranges
    if kind == "wrap":  # k_plan_cta punts, k_plan_smem sorts wide keys, the general path runs all eight passes
        assert int(tv.min()) < -2 ** 62 and max(ranges) >= 2 ** 63, ranges
    if kind == "thresh" and route == "general":  # in-domain values: one key word where no distro knob widens the range
        assert min(ranges) < 2 ** 32, ranges


def test_breakdown_of_tiny_distros_on_a_fresh_context():
    """A breakdown run plans the <= 32-task distros with k_plan_smem, which parks keys of value ranges beyond 32 bits in
    a scratch buffer.  A tick of tiny distros only, on a context that never held a larger tick, must have that buffer
    too (it used to be sized only when some distro was on-chip-sized: an illegal address on a fresh context)."""
    from evergreen_b200 import scheduler
    w = edge_tick("warp", "nd", "sparse")
    eng = scheduler.Engine(0)
    try:
        pb, _ = eng.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now, breakdown=True)
        ref = parity.check_against_oracle(w, pb, None)
        assert np.array_equal(pb.breakdown, ref["breakdown"])
        assert max(value_ranges(w, pb.total_value)) >= 2 ** 32
    finally:
        eng.close()


def test_update_tasks_moves_rows_across_the_domain(engine):
    """evg_update_tasks on a resident tick: rows move out of the 32-bit domain (edge values) and back in (their
    original values), on every route at once; each run equals a fresh upload of the edited table and the oracle."""
    sizes = np.array([20, 700, 3000, 9000, 14000, 1, 25000])
    w = synth.make(sizes, 231, zipf_priority=True, tg_frac=0.12, met_dep_frac=0.02, unmet_dep_frac=0.03,
                   includes_dependencies=True, custom_factor_frac=0.3, n_hosts=50)
    w.distros.cfg["generate_task_factor"] = 100  # what the `wrap` rows set: evg_update_tasks changes task rows only
    orig = copy.deepcopy(w.tasks)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    rng = np.random.default_rng(7)
    t = w.tasks
    edited = np.zeros(0, dtype=np.int64)
    for round_, kinds in enumerate((("nd", "exp"), ("tiq", "prio", "basis"), ("wrap", "thresh"))):
        back = edited[rng.uniform(size=edited.shape[0]) < 0.5]  # half of the edited rows return to their values
        for name, _ in t.COLUMNS:
            getattr(t, name)[back] = getattr(orig, name)[back]
        fresh = np.sort(rng.choice(t.n_tasks, size=t.n_tasks // 40, replace=False)).astype(np.int64)
        synth.sprinkle_edges(w, 600 + round_, kinds=kinds, positions=fresh)
        rows = np.union1d(back, fresh)
        edited = np.union1d(np.setdiff1d(edited, back), fresh)
        engine.update_tasks(rows, soa.TaskSoA(**{name: getattr(t, name)[rows].copy() for name, _ in t.COLUMNS}))
        engine.run(w.now)
        po, ao = copy.deepcopy(engine.download())
        parity.check_against_oracle(w, po, ao)
        fo, fa = engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now)
        for f in ("order", "total_value", "info", "group_info"):
            assert np.array_equal(getattr(po, f), getattr(fo, f)), (round_, f)
        assert np.array_equal(ao.result, fa.result)
        engine.upload(w.tasks, w.distros, w.hosts)  # resident again for the next round


def test_gbest_range_held_by_multi_member_units(engine):
    """k_gbest folds each general-path distro's value range over the work list.  Here only multi-member units hold the
    extremes: a few task groups at priority 2^31 - 1 set each distro's maximum, a few task groups at the lowest value
    its minimum (every lone task sits in between), and a GroupVersions distro whose lowest version unit is pinned
    to the lowest priority and factors.  Work-list warps are sparse and straddle distros."""
    sizes = np.array([13001, 14002, 12999, 15003])
    w = synth.make(sizes, 241, tg_frac=0.0, custom_factor_frac=0.0, n_hosts=60)
    t, dt = w.tasks, w.distros
    toff = dt.task_off
    t.priority[:] = 50
    t.flags[:] = (t.flags & ~np.uint32(L.EVG_TF_GENERATE | L.EVG_TF_STEPBACK)) | np.uint32(L.EVG_TF_DEPS_MET)
    group_off = [0]
    gid = np.full(t.n_tasks, -1, dtype=np.int32)
    tgo = np.zeros(t.n_tasks, dtype=np.int32)
    for d in range(dt.n_distros):
        a = int(toff[d])
        if d == 2:
            group_off.append(group_off[-1])
            continue
        # two groups of three at the top, two of two at the bottom, spread over the distro
        for g, (start, n, top) in enumerate(((37, 3, True), (5000, 3, True), (777, 2, False), (9000, 2, False))):
            rows = a + start + np.arange(n)
            gid[rows] = g
            tgo[rows] = np.arange(1, n + 1)
            t.version_id[rows] = t.version_id[rows[0]]
            if top:
                t.priority[rows] = 2 ** 31 - 1
            else:
                t.priority[rows] = -1
                t.expected_ns[rows] = 0
                t.num_dependents[rows] = 0
                t.queue_basis_ns[rows] = w.now - 2 * synth.WEEK_NS
                t.flags[rows] = np.uint32(L.EVG_TF_DEPS_MET)
        group_off.append(group_off[-1] + 4)
    t.group_id, t.task_group_order = gid, tgo
    dt.group_off = np.array(group_off, dtype=np.int64)
    dt.group_max_hosts = np.ones(group_off[-1], dtype=np.int32)
    # distro 2: GroupVersions; version 0's tasks carry the lowest priority and time, the factors clamp to 1
    a, b = int(toff[2]), int(toff[3])
    dt.cfg["group_versions"][2] = 1
    low = np.nonzero(t.version_id[a:b] == 0)[0] + a
    t.priority[low] = -2 ** 31
    t.expected_ns[low] = 0
    t.num_dependents[low] = 0
    t.queue_basis_ns[low] = w.now - 2 * synth.WEEK_NS
    t.flags[low] = np.uint32(L.EVG_TF_DEPS_MET)
    for f in ("patch_factor", "patch_time_in_queue_factor", "commit_queue_factor", "mainline_time_in_queue_factor",
              "expected_runtime_factor", "generate_task_factor", "stepback_task_factor"):
        dt.cfg[f][2] = -1
    t.normalize()
    dt.normalize()
    po, ao = run(engine, w)
    parity.check_against_oracle(w, po, ao)
    parity.check_properties(w, po, ao)
    for d in (0, 1, 3):  # the extremes are the units' values, not a lone task's
        a, b = int(toff[d]), int(toff[d + 1])
        top = set(np.nonzero(t.priority[a:b] == 2 ** 31 - 1)[0].tolist())
        bottom = set(np.nonzero(t.priority[a:b] == -1)[0].tolist())
        assert int(po.order[a]) in top and int(po.order[b - 1]) in bottom
        assert int(po.total_value[a]) > 2 ** 32
