"""The general path's radix sort (evg_plan_general.cuh: k_gsched, k_ghist, k_gdscan, k_gscatter, k_gemit) at every pass
count, both key widths, the digit shapes a tile can hold and every tile-count remainder of k_gdscan.

Each distro sorts the key Vmax - V in gen_npass(bits) = ceil(bits / 8) stable LSD passes, where bits is the bit length of
Vmax - Vmin; a second key word travels when bits > 32, and the result ends in buffer npass & 1.  The distros built here
hold lone tasks only (no task group, no GroupVersions, no in-queue edge, no merge-queue or generator flag), so every unit
has one member and the tie policy of DESIGN.md §3 reduces to the input index: the expected queue of values v is
order = lexsort((index, -v)) and TotalValue per rank v[order].  Every GPU test compares with that numpy reference bit for
bit, and with the oracle where the tick is small enough.

The values are crafted (`craft`) to a chosen width of Vmax - Vmin and, where a test needs it, a digit shape.  Every
distro shares one planner setting (PLANNER); a lone patch task's TotalValue is then (1 + priority) * rank + 1 with
rank = 2 + minutes in queue + RUNTIME_FACTOR * expected minutes, wrapped to int64 as Go's arithmetic wraps
(`lone_value`).  test_crafted_values_match_the_oracle checks that form against oracle.unit_value and every crafted
distro's width and digit shape against the oracle's planner, on the CPU.  Because the setting is shared, a resident
tick can move the same distros across widths with evg_update_tasks, which changes task rows only.
"""
import copy

import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa, synth

GTILE = 2048                  # kGTile: keys per sort tile; tiles start at (distro start & ~3) + k * 2048
RUNTIME_FACTOR = 256          # ExpectedRuntimeFactor: rank - 2 = 256 * expected minutes + minutes in queue (< 256)
PLANNER = dict(patch_factor=1, patch_time_in_queue_factor=1, commit_queue_factor=1, mainline_time_in_queue_factor=1,
               expected_runtime_factor=RUNTIME_FACTOR, generate_task_factor=1, stepback_task_factor=1)
RANK_MIN = 2 + RUNTIME_FACTOR  # one expected minute, no time in queue (a zero expected duration would mean "unknown")
RANK_MAX = 2 + RUNTIME_FACTOR * 140_000_000  # 1.4e8 expected minutes: 8.4e18 ns, inside int64
PRIO_BITS = 31                # priority <= 2^31 - 1
EXACT_BITS = 34               # widths a priority-0 distro reaches exactly: any rank delta below 2^34
NOW = synth.NOW_NS
WIDTHS = (0, 1, 8, 9, 16, 17, 24, 25, 32, 33, 40, 41, 48, 49, 56, 57, 63, 64)  # each side of every pass-count boundary


# ---------------------------------------------------------------- value crafting
def lone_value(prio, rank):
    """TotalValue (planner.go:209-300) of a lone patch task under PLANNER: (1 + prio) * rank + 1, wrapped to int64."""
    with np.errstate(over="ignore"):
        v = (np.asarray(prio, np.int64).astype(np.uint64) + np.uint64(1)) * np.asarray(rank, np.int64).astype(np.uint64)
        v = v + np.uint64(1)
    return np.atleast_1d(v).view(np.int64)


def rank_columns(rank):
    """(minutes in queue, expected minutes) that give `rank` under PLANNER."""
    rank = np.asarray(rank, np.int64)
    assert np.all(rank >= RANK_MIN) and np.all(rank <= RANK_MAX)
    return (rank - 2) % RUNTIME_FACTOR, (rank - 2) // RUNTIME_FACTOR


def width(v) -> int:
    """Bit length of Vmax - Vmin: what gen_bits computes."""
    v = np.asarray(v, np.int64)
    return (int(v.max()) - int(v.min())).bit_length() if v.size else 0


def sort_keys(v) -> np.ndarray:
    """Vmax - V as the sort sees it (uint64: the difference of two int64 is below 2^64)."""
    u = np.asarray(v, np.int64).view(np.uint64)
    return np.uint64(u[np.argmax(v)]) - u


def digits(v, j) -> np.ndarray:
    """Pass j's digit of every key."""
    return ((sort_keys(v) >> np.uint64(8 * j)) & np.uint64(255)).astype(np.int64)


def craft(n, b, rng, shape="dense", offset=0):
    """(priority, rank) of n lone tasks whose values span width b (offset: added to every rank of a priority-0 draw, so
    the values move without the width changing):
      dense    values spread over the whole range, the minimum and the maximum both present;
      levels3  three distinct values (the extremes and one between), dealt to the tasks at random: ties across tiles;
      all256   priority 0 and rank deltas (i mod 256) + 256 * r: every pass-0 digit in any 256 consecutive tasks;
      stride8 / stride16 / stride32
               rank deltas (priority 0) or values (priority >= 1, stride32) that are multiples of 2^s: the low s / 8 digits
               of every key are equal, so in those passes one digit's run is a whole tile;
      top      values k * 2^56 + 1 for k = 1 .. 256 in turn: keys that differ only in the top digit of the high word."""
    idx = np.arange(n)
    if b == 0:
        return np.zeros(n, np.int64), np.full(n, RANK_MIN + offset, np.int64)
    if shape == "top":  # (1 + 2^30 - 1) * (k * 2^26) + 1
        return np.full(n, 2 ** 30 - 1, np.int64), (1 + rng.permutation(n) % 256) << 26
    if shape == "stride32":  # (1 + p) * 2^32 + 1, 1 + p < 3 * 2^(b - 34)
        pmax = 3 << (b - 34)
        p = rng.integers(0, pmax, n)
        p[:2] = (0, pmax - 1)
        return p, np.full(n, 1 << 32, np.int64)
    if shape.startswith("stride") or shape == "all256" or b <= EXACT_BITS:
        s = int(shape[6:]) if shape.startswith("stride") else 0
        top = 0 if b == 0 else 1 if b == 1 else 3 << (b - 2)  # the range: [2^(b-1), 2^b)
        if shape == "all256":
            delta = idx % 256 + (rng.integers(0, (top >> 8) + 1, n) << 8)
            delta[0], delta[256] = 0, top
        else:
            delta = rng.integers(0, (top >> s) + 1, n) << s
            delta[:2] = (0, top)
        if shape == "levels3":
            delta = np.array([0, top, top // 3])[rng.integers(0, 3, n)]
            delta[:3] = (0, top, top // 3)
        return np.zeros(n, np.int64), RANK_MIN + offset + delta
    # wider: 1 + priority < 2^pb times rank <= R, R * 2^pb = 3 * 2^(b - 2); b = 64 wraps
    pb = min(PRIO_BITS, b - EXACT_BITS + 1)
    R = (3 << (b - 2)) >> pb
    p = rng.integers(0, 1 << pb, n)
    r = rng.integers(RANK_MIN, R + 1, n)
    p[:3] = ((1 << pb) - 1, 0, (1 << pb) - 1)
    r[:3] = (R, RANK_MIN, R // 2)
    if shape == "levels3":
        k = rng.integers(0, 3, n)
        k[:3] = (0, 1, 2)
        p, r = p[:3][k], r[:3][k]
    return p, r


def craft_checked(n, b, rng, shape="dense", offset=0):
    p, r = craft(n, b, rng, shape, offset)
    perm = np.arange(n) if shape == "all256" else rng.permutation(n)  # the extremes anywhere (all256 keeps its order)
    p, r = p[perm], r[perm]
    assert width(lone_value(p, r)) == b, (b, shape, width(lone_value(p, r)))
    return p, r


def lone_tick(parts, seed, *, units=False, edges=True, n_hosts=0):
    """One tick whose distro d takes the (priority, rank) columns parts[d] (synth.make draws the rest).  units: task
    groups and in-queue dependency edges as synth.make places them (values of multi-member units are the oracle's);
    edges=False keeps the task groups only.  n_hosts: hosts for the allocator, as synth.make spreads them."""
    sizes = np.array([len(p) for p, _ in parts], np.int64)
    deps = units and edges
    w = synth.make(sizes, seed, tg_frac=0.1 if units else 0.0, met_dep_frac=0.03 if deps else 0.0,
                   unmet_dep_frac=0.01 if deps else 0.0, includes_dependencies=deps, custom_factor_frac=0.0,
                   n_hosts=n_hosts)
    set_values(w.tasks, np.arange(w.n_tasks), np.concatenate([p for p, _ in parts]), np.concatenate([r for _, r in parts]),
               keep_deps_met=units)
    for f, x in PLANNER.items():
        w.distros.cfg[f] = x
    w.distros.cfg["num_dependents_factor"] = 0.0
    w.distros.normalize()
    return w


def set_values(t, rows, prio, rank, keep_deps_met=False):
    """Rows become lone patch tasks of these priorities and ranks (no dependents, no generator / stepback flag)."""
    q, m = rank_columns(rank)
    t.priority[rows] = prio
    t.expected_ns[rows] = m * M.MINUTE
    t.queue_basis_ns[rows] = NOW - q * M.MINUTE
    t.wait_basis_ns[rows] = NOW
    t.num_dependents[rows] = 0
    met = (t.flags[rows] & np.uint32(L.EVG_TF_DEPS_MET)) if keep_deps_met else np.uint32(L.EVG_TF_DEPS_MET)
    t.flags[rows] = np.uint32(L.EVG_TF_REQ_PATCH) | met
    t.normalize()


def tick_values(w):
    return lone_value(w.tasks.priority, (2 + (NOW - w.tasks.queue_basis_ns) // M.MINUTE
                                         + RUNTIME_FACTOR * (w.tasks.expected_ns // M.MINUTE)))


def place(specs, seed, *, units=False, edges=True, n_hosts=0):
    """Distros from specs (n, start residue mod 4 or None, width, shape) -- or (n, residue, (priority, rank)) for columns
    crafted elsewhere -- in order; a filler distro of 1-3 tasks (width 0, k_plan_warp) goes before a spec whose start
    would not have its residue.  units, edges, n_hosts: as lone_tick.  -> (tick, spec distro ids)."""
    rng = np.random.default_rng(seed)
    parts, ids, base = [], [], 0
    for n, res, *what in specs:
        if res is not None and base % 4 != res:
            k = (res - base) % 4
            parts.append(craft(k, 0, rng))
            base += k
        ids.append(len(parts))
        parts.append(what[0] if len(what) == 1 else craft_checked(n, what[0], rng, what[1]))
        assert len(parts[-1][0]) == n
        base += n
    return lone_tick(parts, seed, units=units, edges=edges, n_hosts=n_hosts), ids


def size_for(tiles, res, last):
    """Tasks of a distro that starts at residue `res` mod 4 and spans `tiles` sort tiles, the last holding `last` keys."""
    return GTILE * (tiles - 1) + last - res


def n_tiles(w, d):
    a, b = int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])
    return -(-(b - (a & ~3)) // GTILE)


# ---------------------------------------------------------------- the ticks
def every_width_tick(seed=71, units=False):
    rng = np.random.default_rng(seed)
    return lone_tick([craft_checked(12289 + 389 * k, b, rng) for k, b in enumerate(WIDTHS)], seed, units=units)


SHAPES = (  # (n, start residue, width, shape, what it aims at)
    (20480, 0, 20, "all256", "every pass-0 digit in every tile"),
    (16384, 1, 24, "stride8", "pass 0: one digit, a whole tile's run, digit 0"),
    (30000, 2, 32, "stride16", "passes 0-1: one digit per tile"),
    (14000, 3, 62, "stride32", "passes 0-3 (the low word): one digit"),
    (25000, 0, 64, "top", "keys that differ only in the top digit of the high word"),
    (size_for(7, 0, 1), 0, 9, "dense", "last tile of 1 key"),
    (size_for(8, 1, 4), 1, 33, "dense", "last tile of 4 keys"),
    (size_for(9, 2, 2047), 2, 17, "dense", "last tile of 2047 keys"),
    (size_for(10, 3, 2048), 3, 57, "dense", "last tile of 2048 keys"),
    (size_for(8, 3, 1), 3, 64, "dense", "last tile of 1 key"),
    (size_for(8, 2, 2048), 2, 8, "dense", "last tile of 2048 keys"),
)
LAST_TILES = {5: 1, 6: 4, 7: 2047, 8: 2048, 9: 1, 10: 2048}  # SHAPES row -> keys of its last tile


def shape_tick():
    return place([s[:4] for s in SHAPES], 83)


TIE_WIDTHS = (8, 32, 64)  # 1, 4 and 8 passes


def tie_tick():
    rng = np.random.default_rng(97)
    parts = []
    for k, b in enumerate(TIE_WIDTHS):
        p, r = craft(3, b, rng, "levels3")
        v = lone_value(p, r)
        pair = next(x for x in ((0, 1), (0, 2), (1, 2)) if width(v[list(x)]) == b)  # two levels that span the width
        for levels in (np.array(pair), np.arange(3)):
            pick = levels[rng.integers(0, levels.shape[0], 24001 + 1001 * k + levels.shape[0])]
            pick[:levels.shape[0]] = levels
            parts.append((p[pick], r[pick]))
    return lone_tick(parts, 97)


# k_gdscan: 7, 8, 9 tiles; 33..65 tiles split into four groups of ceil(nt / 4) tiles, walked 8 at a time: the groups'
# remainders mod 8 take every value (groups of 9 .. 17 tiles: 1 .. 7, 0, 1; the last group's: 6, 0, 3, 6), then 64, 65
GDSCAN_TILES = (7, 8, 9, 33, 38, 40, 44, 48, 52, 56, 60, 64, 65)
GDSCAN_WIDTHS = (12, 33, 20, 64, 9, 41, 25, 56, 17, 48, 63, 32, 1)


def gdscan_tick():
    rng = np.random.default_rng(5)
    specs = [(size_for(nt, k % 4, int(rng.integers(1, GTILE + 1))), k % 4, b, "dense")
             for k, (nt, b) in enumerate(zip(GDSCAN_TILES, GDSCAN_WIDTHS))]
    return place(specs, 5)


# ---------------------------------------------------------------- checks
def check_sorted(w, po, values, distros=None):
    """Bit for bit against the stable sort of the crafted values (~v orders like -v and cannot overflow)."""
    toff = w.distros.task_off
    for d in range(w.distros.n_distros) if distros is None else distros:
        a, b = int(toff[d]), int(toff[d + 1])
        v = values[a:b]
        order = np.lexsort((np.arange(b - a), ~v))
        k = parity.first_diff(po.order[a:b], order)
        assert k < 0, (f"distro {d} (width {width(v)}): rank {k} holds task {po.order[a + k]}, want {order[k]} "
                       f"(values {po.total_value[a + k]} / {v[order[k]]})")
        assert np.array_equal(po.total_value[a:b], v[order]), d


def gpu_widths(w, po):
    toff = w.distros.task_off
    return [width(po.total_value[toff[d]:toff[d + 1]]) for d in range(w.distros.n_distros)]


# ---------------------------------------------------------------- CPU: the crafting against the oracle
def test_crafted_values_match_the_oracle():
    """lone_value against oracle.unit_value, then every crafted distro's width and digit shape from the values the
    oracle's planner ranks (its TotalValue per rank must be the crafted value of the task it ranks there)."""
    from oracle import oracle as O
    rng = np.random.default_rng(3)
    d = M.Distro(id="d0", planner_settings=M.PlannerSettings(**PLANNER))
    samples = [craft(300, b, rng, s) for b, s in [(b, "dense") for b in WIDTHS] + [(20, "all256"), (32, "stride16"),
                                                                                 (62, "stride32"), (64, "top")]]
    pick = np.r_[0:3, 256, 299]  # the extremes and a value between them, the top of all256, one more
    p = np.concatenate([x[pick] for x, _ in samples])
    r = np.concatenate([x[pick] for _, x in samples])
    want = lone_value(p, r)
    assert np.any(want < 0)  # the wrapped values are among them
    q, m = rank_columns(r)
    for k in range(p.shape[0]):
        t = M.Task(id="t", version="v", project="p", build_variant="bv", priority=int(p[k]),
                   requester=M.PATCH_VERSION_REQUESTER, activated_time=NOW - int(q[k]) * M.MINUTE, scheduled_time=NOW,
                   expected_duration=int(m[k]) * M.MINUTE, distro_id="d0")
        assert O.unit_value(d, [t], NOW).total_value == int(want[k]), (k, int(p[k]), int(r[k]))

    def oracle_values(w):
        ref = O.SoAJob(w.tasks, w.distros, None).run(w.now, 8)
        v = tick_values(w)
        out = []
        for j in range(w.distros.n_distros):
            a, b = int(ref["task_off"][j]), int(ref["task_off"][j + 1])
            tv = ref["total_value"][a:b]
            assert np.array_equal(tv, v[int(w.distros.task_off[j]) + ref["order"][a:b]]), j
            out.append(tv)
        return out

    assert [width(v) for v in oracle_values(every_width_tick())] == list(WIDTHS)
    w, ids = shape_tick()
    vals = oracle_values(w)
    for row, d in enumerate(ids):
        n, res, b, shape, _ = SHAPES[row]
        v = vals[d]
        assert width(v) == b and int(w.distros.task_off[d]) % 4 == res, (row, width(v))
        if shape == "all256":  # in input order: every tile of the distro holds all 256 pass-0 digits
            dg = digits(tick_values(w)[w.distros.task_off[d]:w.distros.task_off[d + 1]], 0)
            a0 = int(w.distros.task_off[d]) & 3
            for s in range(-a0, n, GTILE):
                assert np.unique(dg[max(s, 0):s + GTILE]).shape[0] == 256, s
        if shape.startswith("stride"):
            low = int(shape[6:]) // 8
            assert all(np.all(digits(v, j) == 0) for j in range(low)) and len(np.unique(digits(v, low))) == 256
        if shape == "top":
            assert all(np.all(digits(v, j) == 0) for j in range(7)) and len(np.unique(digits(v, 7))) == 256
        if shape in ("all256", "stride8"):
            assert {0, 255} <= set(digits(v, 0 if shape == "all256" else 1).tolist())
        if row in LAST_TILES:
            nt = n_tiles(w, d)
            a = int(w.distros.task_off[d])
            assert n + (a & 3) - GTILE * (nt - 1) == LAST_TILES[row], row
    w = tie_tick()
    for j, v in enumerate(oracle_values(w)):
        assert width(v) == TIE_WIDTHS[j // 2] and len(np.unique(v)) == 2 + j % 2, j
    w, ids = gdscan_tick()
    assert [n_tiles(w, d) for d in ids] == list(GDSCAN_TILES)
    assert [int(w.distros.task_off[d]) % 4 for d in ids] == [k % 4 for k in range(len(ids))]
    assert [width(tick_values(w)[w.distros.task_off[d]:w.distros.task_off[d + 1]]) for d in ids] == list(GDSCAN_WIDTHS)


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_every_pass_count_in_one_tick(engine):
    """Widths 0 .. 64 (0 to 8 passes, one and two key words) share *maxpass and both buffers in one tick."""
    w = every_width_tick()
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    assert gpu_widths(w, po) == list(WIDTHS)
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
@pytest.mark.parametrize("b", WIDTHS)
def test_each_pass_count_alone(engine, b):
    """One distro per tick: *maxpass is the distro's own pass count."""
    rng = np.random.default_rng(1000 + b)
    w = lone_tick([craft_checked(13001 + 7 * b, b, rng)], 1000 + b)
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    assert gpu_widths(w, po) == [b]
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_digit_shapes_inside_tiles(engine):
    """One digit for a whole tile, all 256 digits in a tile, digits 0 and 255, keys that differ only in the top digit of
    the high word, and last tiles of 1, 4, 2047 and 2048 keys at every start residue."""
    w, ids = shape_tick()
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    widths = gpu_widths(w, po)
    assert [widths[d] for d in ids] == [s[2] for s in SHAPES]
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_ties_across_tiles(engine):
    """Two or three distinct values spread over 12+ tiles at 1, 4 and 8 passes: only the stability of every pass and
    k_gdscan's tile offsets keep equal keys in input order."""
    w = tie_tick()
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    assert gpu_widths(w, po) == [b for b in TIE_WIDTHS for _ in (2, 3)]
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_gdscan_tile_counts(engine):
    """Tile counts 7, 8, 9, every per-group remainder mod 8 of k_gdscan's unrolled walks, 64 and 65, at start residues
    0 to 3, with partial last tiles."""
    w, ids = gdscan_tick()
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    widths = gpu_widths(w, po)
    assert [widths[d] for d in ids] == list(GDSCAN_WIDTHS)
    check_sorted(w, po, tick_values(w))
    parity.check_properties(w, po)


@pytest.mark.gpu
def test_largest_distro(engine):
    """A distro of MAX_TASKS_PER_DISTRO tasks (1024 tiles, eight passes, two key words) next to a 13 000-task one at
    width 9."""
    rng = np.random.default_rng(11)
    w = lone_tick([craft_checked(L.MAX_TASKS_PER_DISTRO, 64, rng), craft_checked(13000, 9, rng)], 11)
    assert n_tiles(w, 0) == 1024
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    assert gpu_widths(w, po) == [64, 9]
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None, distros=[1])
    parity.check_properties(w, po)


@pytest.mark.gpu
def test_resident_tick_across_widths(engine):
    """Upload once, then evg_update_tasks moves the same distros through widths 64 -> 9 -> 0 -> 33 -> 1 with a run after
    each step: the high-word buffers are written only for wide distros and *maxpass is recomputed every run, so a stale
    high word or pass count would show.  Each run equals a fresh plan_batch on a second context and the reference."""
    from evergreen_b200 import scheduler
    seq = (64, 9, 0, 33, 1)
    rng = np.random.default_rng(13)
    sizes = (13001, 20003, 16002)
    w = lone_tick([craft_checked(n, seq[0], rng) for n in sizes], 13)
    t = w.tasks
    fresh = scheduler.Engine(0)
    try:
        engine.upload(t, w.distros)
        for step, b in enumerate(seq):
            if step:
                parts = [craft_checked(n, b, rng) for n in sizes]
                rows = np.arange(t.n_tasks, dtype=np.int64)
                set_values(t, rows, np.concatenate([p for p, _ in parts]), np.concatenate([r for _, r in parts]))
                engine.update_tasks(rows, soa.TaskSoA(**{name: getattr(t, name)[rows].copy() for name, _ in t.COLUMNS}))
            engine.run(w.now)
            po, _ = copy.deepcopy(engine.download())
            assert gpu_widths(w, po) == [b] * len(sizes), step
            check_sorted(w, po, tick_values(w))
            fo = fresh.plan_batch(t, w.distros, w.now)
            for f in ("order", "total_value", "info"):
                assert np.array_equal(getattr(po, f), getattr(fo, f)), (step, f)
    finally:
        fresh.close()


@pytest.mark.gpu
def test_every_pass_count_with_units(engine):
    """The every-width tick with task groups and in-queue dependency edges on top: the pre-arrangement k_gplace builds
    is no longer the identity, and multi-member units carry their own values.  Against the oracle."""
    w = every_width_tick(units=True)
    assert w.distros.n_groups > 0 and w.tasks.n_edges > 0
    po = engine.plan_batch(w.tasks, w.distros, w.now)
    parity.check_against_oracle(w, po, None)
    parity.check_properties(w, po)
    assert max(gpu_widths(w, po)) == 64
