"""The utilization host allocator on each of its kernels, at the boundaries that pick them and at its numeric edges,
bit for bit against the C++ oracle (parity.check_against_oracle: new_hosts, free_hosts, status, deficit_ns and every
group's count_free / count_required).

The route rule (run_alloc_range in evg_sched.cu), restated:
* a range of at least 4096 distros is split: k_alloc_groupless plans, one thread each, the distros that have no task
  group and at most 64 hosts, and k_alloc skips them;
* k_alloc is k_alloc<128> (a block per distro, buckets cached 512 groups at a time) when some distro of the TICK has
  more than 1024 task groups, else k_alloc<32> (a warp per distro, 128 groups at a time); it launches once, and not at
  all when the list it would walk is empty;
* when the range is the whole table and upload_hosts listed the distros against the resident table (an upload or an
  edit with hosts), k_alloc walks only the listed distros (task groups, or more than 64 hosts); the sub-ranges of the
  pipelined one-shot call run unlisted.  An edit without hosts leaves a tick without hosts, which the run does not
  allocate.
alloc_route() predicts the launches, and every GPU case checks the prediction against torch.profiler."""
import math
from collections import Counter

import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from oracle import oracle as O

NOW = synth.NOW_NS
I64_MAX, I64_MIN = 2 ** 63 - 1, -2 ** 63
SPLIT_DISTROS, GROUPLESS_HOSTS, WIDE_GROUPS = 4096, 64, 1024


def alloc_route(groups, hosts, *, max_groups=None, listed=False):
    """Counter of the allocator kernels one run_alloc_range launches over distros with these group and host counts.
    max_groups: the tick's largest group count (the range's by default); listed: whole-table range of a listed tick."""
    groups, hosts = np.asarray(groups), np.asarray(hosts)
    n = groups.shape[0]
    split = n >= SPLIT_DISTROS
    if max_groups is None:
        max_groups = int(groups.max()) if n else 0
    teams = int(((groups > 0) | (hosts > GROUPLESS_HOSTS)).sum()) if split and listed else n
    out = Counter()
    if teams:
        out["k_alloc<128>" if max_groups > WIDE_GROUPS else "k_alloc<32>"] += 1
    if split:
        out["k_alloc_groupless"] += 1
    return out


# ---------------------------------------------------------------------------------------------------- the generator
HOT = (0, 1, 31, 32, 63, 127, 128, 129, 255, 256, 383, 384, 511, 512, 513, 543, 1023, 1024, 1535, 1536)
THRESHOLDS = (1, -5 * M.MINUTE, 0, 3)
FRACTIONS = (0.0, -0.0, 1.0, math.nextafter(1.0, 2.0), -0.25, 5e-324, -5e-324, float("nan"), -1e300, 0.1)


def host_edges(rng, n):
    """(expected, stddev, start) for n running hosts: soon_free_term's edges -- Go's zero start (time.Since saturates),
    a start in the future, expected near +-2^63 (the subtraction wraps), stddev 0, -1 and 2^62 (3 * stddev wraps), and
    elapsed at kMaxDurationPerDistroHost and at expected + 3 * stddev, each +-1 ns."""
    k = rng.integers(n, 0, 11)
    exp = rng.integers(n, 10 * M.SECOND, 2 * M.HOUR)
    std = exp // 5
    start = NOW - rng.integers(n, 0, 3 * M.HOUR)
    cut = 30 * M.MINUTE + rng.integers(n, -1, 1)
    e3 = 35 * M.MINUTE + rng.integers(n, -1, 1)
    start = np.where(k == 0, M.ZERO_TIME, start)
    start = np.where(k == 1, NOW + M.HOUR, start)
    exp = np.where(k == 2, I64_MAX, np.where(k == 3, I64_MIN + 1, exp))
    std = np.where(k == 4, 0, np.where(k == 5, -1, np.where(k == 6, 2 ** 62, std)))
    exp, std, start = (np.where(k == 7, 10 * M.MINUTE, exp), np.where(k == 7, 400 * M.SECOND, std), np.where(k == 7, NOW - cut, start))
    exp, std, start = (np.where(k == 8, 20 * M.MINUTE, exp), np.where(k == 8, 5 * M.MINUTE, std), np.where(k == 8, NOW - e3, start))
    return exp, std, start


def make_tick(groups, hosts, seed, *, ungrouped=None, edges=True, hot_frac=0.5):
    """One tick: distro d has groups[d] task groups of one task each, ungrouped[d] standalone tasks (3 by default) and
    hosts[d] hosts -- running, free, in teardown and running with their task not found, interleaved; the running ones
    sit in the "" bucket, in a group (half of them in the HOT groups, at the allocator's stretch and lane boundaries)
    or in a group the queue does not have.  With `edges`, a seeded quarter of the distros take an edge threshold,
    fraction, pool or configuration, a tenth of the running hosts soon_free_term's edges, and the last 12 distros
    (of a tick of at least 24) the calcNewHostsNeeded quotients of CALC_EDGES."""
    rng = synth.Rng(seed)
    groups = np.asarray(groups, np.int64)
    hosts = np.asarray(hosts, np.int64)
    D = groups.shape[0]
    ung = np.full(D, 3, np.int64) if ungrouped is None else np.asarray(ungrouped, np.int64)
    sizes = groups + ung
    toff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    goff = np.concatenate([[0], np.cumsum(groups)]).astype(np.int64)
    T = int(toff[-1])
    dof = np.repeat(np.arange(D), sizes)
    local = np.arange(T) - toff[dof]
    gid = np.where(local < groups[dof], local, -1).astype(np.int32)
    u = rng.uniform(T)
    flags = np.where(u < 0.4, L.EVG_TF_REQ_PATCH, np.where(u < 0.45, L.EVG_TF_REQ_MERGE_QUEUE, L.EVG_TF_REQ_OTHER)).astype(np.uint32)
    flags |= np.where(rng.uniform(T) < 0.95, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
    tasks = S.TaskSoA(rng.integers(T, 0, 100).astype(np.int32), rng.integers(T, 10 * M.SECOND, 2 * M.HOUR),
                      NOW - rng.integers(T, 0, 72 * M.HOUR), NOW - rng.integers(T, 0, 3 * M.HOUR), np.zeros(T, np.int32),
                      np.where(gid >= 0, 1, 0).astype(np.int32), gid, np.zeros(T, np.int32), flags).normalize()
    cfg = np.zeros(D, L.DISTRO_CFG_DTYPE)
    cfg["target_time_ns"] = M.MAX_DURATION_PER_DISTRO_HOST
    cfg["n_versions"] = 1
    distros = S.DistroTable(toff, goff, cfg, rng.integers(int(goff[-1]), 1, 4).astype(np.int32)).normalize()

    hoff = np.concatenate([[0], np.cumsum(hosts)]).astype(np.int64)
    H = int(hoff[-1])
    hd = np.repeat(np.arange(D), hosts)
    k = rng.uniform(H)
    running = k < 0.6
    found = running & (k < 0.55)
    teardown = (k >= 0.9)
    hflags = (np.where(running, L.EVG_HF_RUNNING, 0) | np.where(found, L.EVG_HF_RT_FOUND, 0) |
              np.where(teardown, L.EVG_HF_TEARDOWN, 0)).astype(np.uint32)
    ng = groups[hd]
    hot = np.array(HOT, np.int64)
    pick_hot = hot[rng.integers(H, 0, len(HOT) - 1)]
    pick = np.where((rng.uniform(H) < hot_frac) & (pick_hot < ng), pick_hot, (rng.uniform(H) * np.maximum(ng, 1)).astype(np.int64))
    b = rng.uniform(H)
    hgid = np.where(running & (ng > 0) & (b < 0.6), pick, np.where(running & (b > 0.92), L.EVG_HG_UNQUEUED, L.EVG_HG_NONE))
    exp = rng.integers(H, 10 * M.SECOND, 2 * M.HOUR)
    std = exp // 5
    start = NOW - (rng.uniform(H) * 2.0 * exp).astype(np.int64)
    acfg = np.zeros(D, L.ALLOC_CFG_DTYPE)
    acfg["future_host_fraction"] = 0.4
    acfg["provider"] = L.EVG_PROVIDER_EPHEMERAL
    acfg["disabled"] = (rng.uniform(D) < 0.02).astype(np.int32)
    acfg["minimum_hosts"] = rng.integers(D, 0, 2)
    acfg["maximum_hosts"] = rng.integers(D, 10, 5000)
    acfg["round_up"] = (rng.uniform(D) < 0.3).astype(np.int32)
    acfg["waits_over_thresh_feedback"] = (rng.uniform(D) < 0.2).astype(np.int32)
    if edges:
        e = rng.uniform(H) < 0.1
        ee, es, est = host_edges(rng, H)
        exp, std, start = np.where(e, ee, exp), np.where(e, es, std), np.where(e, est, start)
        distro_edges(rng, distros, acfg, hosts)
    hs = S.HostSoA(hflags, hgid.astype(np.int32), np.where(found, exp, 0), np.where(found, std, 0),
                   np.where(running, start, M.ZERO_TIME), hoff, acfg).normalize()
    w = synth.Workload("alloc routes", NOW, tasks, distros, hs)
    if edges and D >= 24:
        calc_edges(w, range(D - 12, D))
    return w


# calcNewHostsNeeded (allocator.go:268-296) on the "" bucket of a distro whose three standalone tasks have these expected
# durations under this threshold, with no free host and no soon-to-be-free term, so x = short_ns / threshold exactly:
# 2; one ulp above 2; one ulp below 2; 1/3 (0 < x < 1 with no free host); 4/3 (rounding); and 2^63 (a finite x beyond
# int64: two short tasks of -2^62 under a threshold of -1).  Each with round-down and with round-up.
CALC_EDGES = ((2 ** 51, (2 ** 51, 2 ** 51, 0)), (2 ** 51, (2 ** 51, 2 ** 51, 1)), (2 ** 52, (2 ** 52, 2 ** 52 - 1, 0)),
              (3, (1, 0, 0)), (3, (2, 2, 0)), (-1, (-2 ** 62, -2 ** 62, 0)))


def calc_edges(w, ds):
    """Give distros ds, in turn, the CALC_EDGES cases x round-down / round-up (their first three standalone tasks, their
    threshold, hosts that run tasks the allocator cannot find, a plain ephemeral configuration)."""
    t, dt, h = w.tasks, w.distros, w.hosts
    for j, d in enumerate(ds):
        thr, exps = CALC_EDGES[(j // 2) % len(CALC_EDGES)]
        a = int(dt.task_off[d] + dt.group_off[d + 1] - dt.group_off[d])
        assert dt.task_off[d + 1] - a >= 3 and (t.group_id[a:a + 3] < 0).all()
        t.expected_ns[a:a + 3] = exps
        t.flags[a:a + 3] = L.EVG_TF_REQ_PATCH | L.EVG_TF_DEPS_MET
        dt.cfg["target_time_ns"][d] = thr
        h0, h1 = int(h.host_off[d]), int(h.host_off[d + 1])
        h.flags[h0:h1] = L.EVG_HF_RUNNING
        h.group_id[h0:h1] = L.EVG_HG_NONE
        c = h.cfg
        c[d] = 0
        c["future_host_fraction"][d] = 0.4
        c["provider"][d] = L.EVG_PROVIDER_EPHEMERAL
        c["maximum_hosts"][d] = 10 ** 6
        c["round_up"][d] = j % 2


def boundary_groups(n_groups, k_cache):
    """The groups at k_alloc's stretch edges: the last of each stretch and the first of the next, and lanes 0 and 31
    of the last stretch, for a distro of n_groups groups cached k_cache at a time."""
    out = set()
    for gb in range(k_cache, n_groups, k_cache):
        out |= {gb - 1, gb}
    last = (n_groups - 1) // k_cache * k_cache
    if last > 0:
        out |= {g for g in (last, last + 31) if g < n_groups}
    return sorted(out)


FULL_TERM_HOSTS = (3, 5, 8)  # running hosts per boundary group, in turn: bucket sums of 1.2, 2.0 and 3.2 at fraction 0.4


def place_boundary_hosts(w, d, k_cache):
    """Overwrite distro d's hosts: boundary group i gets FULL_TERM_HOSTS[i % 3] running hosts whose task is past its
    expected duration (term = the fraction, 0.4: floor(soon) of the bucket is 1, 2 or 3, and differs from its
    neighbour's), each group's hosts followed by one such host in the "" bucket, spread over the distro's host order
    among its other hosts.  The distro gets a plain configuration so that its status is OK."""
    h, dt = w.hosts, w.distros
    bg = boundary_groups(int(dt.group_off[d + 1] - dt.group_off[d]), k_cache)
    gids = [g for i, b in enumerate(bg) for g in [b] * FULL_TERM_HOSTS[i % 3] + [L.EVG_HG_NONE]]
    h0, h1 = int(h.host_off[d]), int(h.host_off[d + 1])
    assert h1 - h0 >= len(gids), (d, h1 - h0, len(gids))
    pos = h0 + np.round(np.linspace(0, h1 - h0 - 1, len(gids))).astype(np.int64)
    h.flags[pos] = L.EVG_HF_RUNNING | L.EVG_HF_RT_FOUND
    h.group_id[pos] = gids
    h.expected_ns[pos] = M.MINUTE
    h.std_ns[pos] = 0
    h.start_ns[pos] = NOW - 2 * M.MINUTE
    dt.cfg["target_time_ns"][d] = M.MAX_DURATION_PER_DISTRO_HOST
    c = h.cfg
    c[d] = 0
    c["future_host_fraction"][d] = 0.4
    c["provider"][d] = L.EVG_PROVIDER_EPHEMERAL
    c["maximum_hosts"][d] = 10 ** 6
    return bg


def full_term_hosts(w, d, g):
    """Running, found hosts of distro d in group g whose task is past its expected duration, stddev 0."""
    h = w.hosts
    h0, h1 = int(h.host_off[d]), int(h.host_off[d + 1])
    m = ((h.flags[h0:h1] & (L.EVG_HF_RUNNING | L.EVG_HF_RT_FOUND)) == (L.EVG_HF_RUNNING | L.EVG_HF_RT_FOUND))
    m &= (h.group_id[h0:h1] == g) & (h.std_ns[h0:h1] == 0) & (h.start_ns[h0:h1] + h.expected_ns[h0:h1] <= NOW)
    return int(m.sum())


def distro_edges(rng, distros, acfg, hosts):
    """A quarter of the distros, dealt in turn: a threshold of 1 ns, negative, 0 (through the C ABI) or 3 ns; an edge
    fraction; a container pool whose parent_maximum_hosts * pool_max_containers (* pool_max_containers again in
    isMaxHostsCapacity) nears or passes the int64 range, or is below 1; minimum / maximum hosts at the int32 extremes;
    a disabled distro; docker at or above maximum_hosts."""
    D = distros.n_distros
    cfg = distros.cfg
    chosen = np.nonzero(rng.uniform(D) < 0.25)[0]
    for j, d in enumerate(chosen.tolist()):
        kind = j % 5
        v = j // 5
        if kind == 0:
            cfg["target_time_ns"][d] = THRESHOLDS[v % len(THRESHOLDS)]
        elif kind == 1:
            acfg["future_host_fraction"][d] = FRACTIONS[v % len(FRACTIONS)]
        elif kind == 2:
            acfg["provider"][d] = L.EVG_PROVIDER_DOCKER
            acfg["has_pool"][d] = 1
            acfg["parent_found"][d] = int(v % 4 != 3)
            pm, pc = ((2 ** 31 - 1, 2 ** 31 - 1), (2 ** 31 - 1, 3), (0, 5), (-1, 5))[v % 4]
            acfg["parent_maximum_hosts"][d], acfg["pool_max_containers"][d] = pm, pc
        elif kind == 3:
            mn, mx = ((2 ** 31 - 1, 2 ** 31 - 1), (-2 ** 31, 2 ** 31 - 1), (5, -2 ** 31), (3, 0), (0, 2 ** 31 - 1))[v % 5]
            acfg["minimum_hosts"][d], acfg["maximum_hosts"][d] = mn, mx
            acfg["disabled"][d] = int(v % 3 == 1)
        else:
            acfg["provider"][d] = L.EVG_PROVIDER_DOCKER
            acfg["maximum_hosts"][d] = max(int(hosts[d]) - v % 2, 0)


# ---------------------------------------------------------------------------------------------------- FP64 host order
def _tree(terms):
    while len(terms) > 1:
        terms = [terms[i] + terms[i + 1] if i + 1 < len(terms) else terms[i] for i in range(0, len(terms), 2)]
    return terms[0] if terms else 0.0


def _seq(terms):
    s = 0.0
    for t in terms:
        s += t
    return s


def order_sensitive_terms(seed, n, threshold=9, fraction=0.3):
    """left values (expected - elapsed, in [0, threshold]) of n running hosts of one bucket whose soon-to-be-free terms
    fraction * (threshold - left) / threshold have a floor of their host-order sum that differs from the floor of the
    same terms summed in reverse, as a pairwise tree, and as 32 lane-strided partials folded by a tree."""
    rng = np.random.default_rng(seed)
    for _ in range(200_000):
        left = rng.integers(0, threshold + 1, n)
        terms = [fraction * (float(threshold - x) / float(threshold)) for x in left.tolist()]
        fwd = math.floor(_seq(terms))
        lanes = [_seq(terms[lane::32]) for lane in range(32)]
        others = (math.floor(_seq(terms[::-1])), math.floor(_tree(terms)), math.floor(_tree(lanes)))
        if all(o != fwd for o in others):
            return left
    raise AssertionError("no order-sensitive bucket found")


def order_tick(seed):
    """Distros whose only running bucket is an order-sensitive one: the "" bucket of a groupless distro (k_alloc_groupless
    with the split, else k_alloc), the "" bucket of a distro with task groups, and group 0, 31 and 129 of such distros.
    Threshold 9 ns and fraction 0.3: neither is dyadic, so the terms are inexact."""
    plan = [(0, None), (0, None), (200, None), (200, 0), (200, 31), (200, 129), (200, 129)]
    n_hosts = [40, 64, 64, 64, 64, 64, 500]
    w = make_tick([p[0] for p in plan], n_hosts, seed, edges=False)
    h = w.hosts
    for d, ((_, g), n) in enumerate(zip(plan, n_hosts)):
        a = int(h.host_off[d])
        left = order_sensitive_terms(seed + d, min(n, 64))
        m = len(left)
        elapsed = 10 * M.MINUTE
        h.flags[a:a + m] = L.EVG_HF_RUNNING | L.EVG_HF_RT_FOUND
        h.flags[a + m:a + n] = 0  # free
        h.group_id[a:a + n] = L.EVG_HG_NONE
        if g is not None:
            h.group_id[a:a + m] = g
        h.start_ns[a:a + m] = NOW - elapsed
        h.expected_ns[a:a + m] = elapsed + left
        h.std_ns[a:a + m] = 0
        w.distros.cfg["target_time_ns"][d] = 9
        h.cfg["future_host_fraction"][d] = 0.3
        h.cfg["maximum_hosts"][d] = 10 ** 6
        h.cfg["disabled"][d] = 0
    return w


# ---------------------------------------------------------------------------------------------------- host-only checks
def test_alloc_route_rule():
    g64 = np.zeros(SPLIT_DISTROS, np.int64)
    h = np.zeros(SPLIT_DISTROS, np.int64)
    assert alloc_route(g64, h) == Counter({"k_alloc<32>": 1, "k_alloc_groupless": 1})
    assert alloc_route(g64, h, listed=True) == Counter({"k_alloc_groupless": 1})
    h[7] = GROUPLESS_HOSTS + 1
    assert alloc_route(g64, h, listed=True) == Counter({"k_alloc<32>": 1, "k_alloc_groupless": 1})
    assert alloc_route(g64[1:], h[1:], listed=True) == Counter({"k_alloc<32>": 1})
    assert alloc_route([WIDE_GROUPS, 0], [0, 0]) == Counter({"k_alloc<32>": 1})
    assert alloc_route([WIDE_GROUPS + 1, 0], [0, 0]) == Counter({"k_alloc<128>": 1})
    assert alloc_route([0], [0], max_groups=WIDE_GROUPS + 1) == Counter({"k_alloc<128>": 1})


def test_order_sensitive_sums_differ_by_order():
    for seed, n in ((1, 40), (2, 64)):
        left = order_sensitive_terms(seed, n)
        terms = [0.3 * (float(9 - x) / 9.0) for x in left.tolist()]
        fwd = math.floor(_seq(terms))
        assert fwd != math.floor(_seq(terms[::-1])) and fwd != math.floor(_tree(terms))
        assert fwd != math.floor(_tree([_seq(terms[lane::32]) for lane in range(32)]))


def test_oracle_conversion_rule():
    """double -> int64 in calcNewHostsNeeded (DESIGN.md §3): NaN gives 0, beyond the int64 range saturates; both were
    undefined behaviour in the oracle (x86 gave INT64_MIN, which the n < 0 clamp turned into 0)."""
    assert O.calc_new_hosts_needed(0, 0, 0, 0, 0, 0, True) == 0                 # 0 / 0
    assert O.calc_new_hosts_needed(1, 0, 0, 0, 0, 0, True) == I64_MAX           # +Inf
    assert O.calc_new_hosts_needed(-1, 0, 0, 0, 0, 0, False) == 0               # -Inf
    assert O.calc_new_hosts_needed(I64_MAX, 1, 0, 0, 0, 0, True) == I64_MAX     # 2^63
    assert O.calc_new_hosts_needed(I64_MIN, -1, 0, 0, 0, 0, False) == I64_MAX
    assert O.calc_new_hosts_needed(2 ** 62, 1, 0, 0, 0, 0, True) == 2 ** 62     # in range: exact
    assert O.calc_new_hosts_needed(5 * 2 ** 50 + 1, 2 ** 50, 0, 0, 0, 0, True) == 5   # 5 + 1 ulp
    assert O.calc_new_hosts_needed(5 * 2 ** 50 + 1, 2 ** 50, 0, 0, 0, 0, False) == 6
    assert O.calc_new_hosts_needed(5 * 2 ** 50 - 1, 2 ** 50, 0, 0, 0, 0, True) == 4   # 5 - 1 ulp
    assert O.calc_new_hosts_needed(5 * 2 ** 50 - 1, 2 ** 50, 0, 0, 0, 0, False) == 5


def test_calc_edges_land_where_stated():
    """The quotients CALC_EDGES promises, in IEEE double as both sides compute them."""
    xs = [float(sum(e)) / float(t) for t, e in CALC_EDGES]
    assert xs[0] == 2.0 and xs[1] == math.nextafter(2.0, 3.0) and xs[2] == math.nextafter(2.0, 0.0)
    assert 0 < xs[3] < 1 and xs[4] != math.floor(xs[4]) and xs[5] >= 2.0 ** 63
    for x, want in zip(xs, ((2, 2), (2, 3), (1, 2), (1, 1), (1, 2), (I64_MAX, I64_MAX))):
        t, e = CALC_EDGES[xs.index(x)]
        assert (O.calc_new_hosts_needed(sum(e), t, 0, 0, 0, 0, True), O.calc_new_hosts_needed(sum(e), t, 0, 0, 0, 0, False)) == want


@pytest.mark.parametrize("fraction,ok", [(0.0, True), (-0.0, True), (1.0, True), (5e-324, True),
                                          (math.nextafter(1.0, 2.0), False), (-5e-324, False), (-0.25, False),
                                          (float("nan"), False), (-1e300, False)])
def test_oracle_fraction_rule(fraction, ok):
    """future_host_fraction outside [0, 1], NaN included, is EVG_ALLOC_ERR_FUTURE_FRACTION."""
    host = M.Host(id="h", running_task="t")
    _, st = O.calc_existing_free_hosts([host], {"t": M.RunningTaskStats(expected=M.MINUTE, start_time=NOW - M.MINUTE)},
                                       fraction, M.MAX_DURATION_PER_DISTRO_HOST, NOW)
    assert st == (L.EVG_ALLOC_OK if ok else L.EVG_ALLOC_ERR_FUTURE_FRACTION)


# ---------------------------------------------------------------------------------------------------- GPU cases
def profiled_alloc(eng, fn):
    """The allocator kernels fn launches, guarded against torch.profiler missing the first kernel of a window (as in
    test_gpu_host_termination.test_launch_counts): a torch kernel opens the window, and a list shorter than the
    context's launch count is taken again.  (It can be longer: the one-shot call's upload validates the ids before the
    context starts counting.)"""
    import torch
    from test_entry_guard import launched_kernels
    out = {}

    def call():
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        out["r"] = fn()
    for _ in range(6):
        names = launched_kernels(call)
        if len(names) >= eng.last_launch_count():
            break
    assert len(names) >= eng.last_launch_count(), names
    return out["r"], Counter(n.split("(")[0] for n in names if n.startswith("k_alloc"))


def one_shot(eng, w, want):
    (po, ao), got = profiled_alloc(eng, lambda: eng.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now))
    assert got == want
    parity.check_against_oracle(w, po, ao)
    return po, ao


def counts(w):
    return np.diff(w.distros.group_off), np.diff(w.hosts.host_off)


def small(n, seed):
    """n small distros: most without groups and with 0-3 hosts, some with 1-8 groups and 31-33 hosts."""
    r = synth.Rng(seed)
    g = np.where(r.uniform(n) < 0.1, r.integers(n, 1, 8), 0)
    h = np.where(g > 0, r.integers(n, 31, 33), r.integers(n, 0, 3))
    return g, h


@pytest.mark.gpu
@pytest.mark.parametrize("n", [SPLIT_DISTROS, SPLIT_DISTROS - 1])
def test_groupless_limit(engine, n):
    """Groupless distros of 64 and 65 hosts (and 0 .. 3, and 31 .. 33 with groups), with the split on and off."""
    g, h = small(n, 7000 + n)
    h[:8] = [64, 65, 64, 65, 63, 2000, 32, 33]
    g[:8] = 0
    w = make_tick(g, h, 7100 + n)
    one_shot(engine, w, alloc_route(*counts(w), listed=True))


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True], ids=["k_alloc32", "k_alloc128"])
def test_stretches(engine, wide):
    """k_alloc<32>: 128, 129, 257 and 1024 groups (largest 1024); k_alloc<128>: 1025, 512, 513 and 1537 groups.  In
    every distro of more than one stretch, place_boundary_hosts puts 3, 5 or 8 full-term running hosts in the last group
    of each stretch, the first of the next, and lanes 0 and 31 of the last stretch, with "" bucket hosts between them;
    the test asserts that placement and that each such bucket's floor(soon) reaches count_free.  Host counts 31, 32, 33
    and 2000, interleaved running, free, teardown and not-found."""
    big, k_cache = ([1025, 512, 513, 1537], 512) if wide else ([128, 129, 257, 1024], 128)
    g, h = small(60, 7200 + wide)
    g = np.concatenate([big, [0, 3, 0, 7], g])
    h = np.concatenate([[33, 31, 32, 2000] if wide else [32, 31, 33, 2000], [0, 33, 65, 1], h])
    w = make_tick(g, h, 7300 + wide)
    placed = {d: place_boundary_hosts(w, d, k_cache) for d in range(4) if big[d] > k_cache}
    # the placement the test stands on: every multi-stretch distro has full-term hosts on both sides of every stretch
    # edge and in lanes 0 and 31 of its last stretch where they exist
    assert sorted(placed) == ([0, 2, 3] if wide else [1, 2, 3])
    for d, bg in placed.items():
        assert {k_cache - 1, k_cache} <= set(bg)
        assert all(full_term_hosts(w, d, b) >= 3 for b in bg), d
    po, ao = one_shot(engine, w, alloc_route(*counts(w), listed=True))
    # floor(soon) of each boundary bucket is seen: count_free = floor(0.4 * hosts) (no free host is in a group bucket)
    for d, bg in placed.items():
        assert int(ao.status[d]) == L.EVG_ALLOC_OK
        got = [int(po.group_info["count_free"][int(w.distros.group_off[d]) + b]) for b in bg]
        assert all(c >= math.floor(_seq([0.4] * FULL_TERM_HOSTS[i % 3])) >= 1 for i, c in enumerate(got)), (d, got)


@pytest.mark.gpu
@pytest.mark.parametrize("lane", [5, 100], ids=["warp0", "warp3"])
def test_team_reduction(engine, lane):
    """k_alloc<128>: one group, owned by warp 0 or warp 3 of the team, fails the pool-size check (max_hosts < 1): the
    status must be the team's max, free_hosts the free count, and every group's outputs 0; a twin distro without the
    bad group checks the sums of all four warps."""
    g = np.array([1100, 1100, 0, 4])
    h = np.array([600, 600, 3, 40])
    w = make_tick(g, h, 7400 + lane, edges=False, hot_frac=0.0)
    w.distros.group_max_hosts[lane] = 0
    po, ao = one_shot(engine, w, alloc_route(*counts(w), listed=True))
    assert int(ao.status[0]) == L.EVG_ALLOC_ERR_POOL_SIZE and int(ao.status[1]) == L.EVG_ALLOC_OK
    assert not po.group_info["count_free"][:1100].any() and not po.group_info["count_required"][:1100].any()
    assert po.group_info["count_required"][1100:2200].any()


@pytest.mark.gpu
def test_host_order_sums(engine):
    """Buckets whose floor(sum) depends on the order of the FP64 additions, as the "" bucket and as group buckets, on
    k_alloc_groupless, k_alloc<32> and k_alloc<128>: only host order matches the oracle."""
    w = order_tick(7500)
    one_shot(engine, w, alloc_route(*counts(w), listed=True))
    # the same distros in a tick of 4096 (k_alloc_groupless takes the first two) and in a wide tick
    g, h = counts(w)
    sg, sh = small(SPLIT_DISTROS - len(g), 7501)
    for extra_g, extra_h in ((sg, sh), (np.array([1200]), np.array([5]))):
        big = make_tick(np.concatenate([g, extra_g]), np.concatenate([h, extra_h]), 7502, edges=False)
        _splice(big, w)
        one_shot(engine, big, alloc_route(*counts(big), listed=True))


def _splice(big, w):
    """Copy w's hosts and allocator / threshold config over the first distros of big (same host counts)."""
    n = w.distros.n_distros
    hb = int(w.hosts.host_off[-1])
    for name in ("flags", "group_id", "expected_ns", "std_ns", "start_ns"):
        getattr(big.hosts, name)[:hb] = getattr(w.hosts, name)
    big.hosts.cfg[:n] = w.hosts.cfg
    big.distros.cfg["target_time_ns"][:n] = w.distros.cfg["target_time_ns"]


@pytest.mark.gpu
def test_listed_and_unlisted_ticks(engine):
    """Upload with hosts (listed), an edit without hosts (no allocator), edits that give a groupless distro its first
    task group and take the last one away from another, with hosts (listed again) and without."""
    g, h = small(SPLIT_DISTROS + 10, 7600)
    g[:4], h[:4] = [0, 1, 300, 0], [70, 10, 2000, 64]
    w = make_tick(g, h, 7601)

    def resident(w, call, hosts):
        call()
        _, got = profiled_alloc(engine, lambda: engine.run(w.now))
        assert got == (alloc_route(*counts(w), listed=True) if hosts else Counter())
        po, ao = engine.download()
        assert (ao is not None) == hosts
        parity.check_against_oracle(w, po, ao)

    resident(w, lambda: engine.upload(w.tasks, w.distros, w.hosts), True)
    e = synth.next_tick(w, 7602, arrive=0.0, change=0.0)
    resident(e.workload, lambda: engine.edit_tasks(e.edit, e.workload.distros), False)
    w = e.workload
    for with_hosts in (True, False):
        ed, w2 = _group_edit(w, first=0 if with_hosts else 3, last=1)
        resident(w2, lambda: engine.edit_tasks(ed, w2.distros, w2.hosts if with_hosts else None), with_hosts)
        ed, w = _group_edit(w2, first=1, last=0 if with_hosts else 3)
        resident(w, lambda: engine.edit_tasks(ed, w.distros, w.hosts if with_hosts else None), with_hosts)


def _group_edit(w, first, last):
    """The edit in which groupless distro `first` gains a one-task group 0 and distro `last` loses every grouped task
    (its hosts in those groups become EVG_HG_UNQUEUED) -> (TaskEdit, the composed workload)."""
    t, dt = w.tasks, w.distros
    D = dt.n_distros
    goff = dt.group_off
    assert goff[first + 1] == goff[first] and goff[last + 1] > goff[last]
    toff = dt.task_off
    rows = np.arange(int(toff[last]), int(toff[last + 1]))
    remove = rows[t.group_id[rows] >= 0]
    ins = S.TaskSoA(np.array([50], np.int32), np.array([M.HOUR]), np.array([NOW - M.HOUR]), np.array([NOW - M.MINUTE]),
                    np.zeros(1, np.int32), np.ones(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                    np.array([L.EVG_TF_DEPS_MET | L.EVG_TF_REQ_PATCH], np.uint32)).normalize()
    ins_off = np.zeros(D + 1, np.int64)
    ins_off[first + 1:] = 1
    ng = np.diff(goff)
    remap = (np.arange(int(goff[-1])) - np.repeat(goff[:-1], ng)).astype(np.int32)
    remap[int(goff[last]):int(goff[last + 1])] = -1
    ng2 = ng.copy()
    ng2[first], ng2[last] = 1, 0
    goff2 = np.concatenate([[0], np.cumsum(ng2)]).astype(np.int64)
    keep = np.nonzero(remap >= 0)[0]
    gmax = np.zeros(int(goff2[-1]), np.int32)
    old_d = np.repeat(np.arange(D), ng)
    gmax[goff2[old_d[keep]] + remap[keep]] = dt.group_max_hosts[keep]
    gmax[int(goff2[first])] = 2
    ed = S.TaskEdit(remove.astype(np.int64), ins, ins_off, np.zeros(0, np.int64), np.zeros(0, np.int32), remap, None,
                    goff2, gmax, None).normalize()
    tasks, distros = S.apply_edit(t, dt, ed)
    h = w.hosts
    hg = h.group_id.copy()
    a, b = int(h.host_off[last]), int(h.host_off[last + 1])
    hg[a:b] = np.where(hg[a:b] >= 0, L.EVG_HG_UNQUEUED, hg[a:b])
    hosts = S.HostSoA(h.flags.copy(), hg, h.expected_ns.copy(), h.std_ns.copy(), h.start_ns.copy(), h.host_off.copy(),
                      h.cfg.copy()).normalize()
    return ed, synth.Workload(w.name, w.now, tasks, distros, hosts)


@pytest.mark.gpu
def test_pipelined_one_shot(engine):
    """A tick of 2^21 tasks takes the pipelined one-shot call: two chunks of 4096 distros each run their own
    unlisted k_alloc and k_alloc_groupless; the first distros of each chunk carry the boundary shapes.  Checked against
    the oracle on those distros and a sample of the rest, and against the resident run of the same tables."""
    D = 2 * SPLIT_DISTROS
    g, h = small(D, 7700)
    for base in (0, SPLIT_DISTROS):
        g[base:base + 6], h[base:base + 6] = [0, 0, 129, 300, 1, 0], [64, 65, 2000, 33, 31, 0]
    ung = np.maximum((1 << 21) // D - g, 0)
    for base in (0, SPLIT_DISTROS):  # each chunk holds exactly 2^20 tasks
        ung[base + 10] -= (g + ung)[base:base + SPLIT_DISTROS].sum() - (1 << 20)
    w = make_tick(g, h, 7701, ungrouped=ung)
    assert w.n_tasks == 1 << 21
    half = int(np.searchsorted(w.distros.task_off, w.n_tasks // 2))
    assert half == SPLIT_DISTROS
    want = alloc_route(g[:half], h[:half], max_groups=int(g.max())) + alloc_route(g[half:], h[half:], max_groups=int(g.max()))
    (po, ao), got = profiled_alloc(engine, lambda: engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now))
    assert got == want
    sel = sorted(set(range(6)) | set(range(half, half + 6)) | set(range(7, D, 97)) | set(range(D - 12, D)))
    parity.check_against_oracle(w, po, ao, distros=sel)
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now)
    po2, ao2 = engine.download()
    assert np.array_equal(ao.result, ao2.result) and np.array_equal(ao.status, ao2.status)
    assert np.array_equal(po.group_info, po2.group_info)
