"""Synthetic scheduler ticks in the shapes BASELINE.json names (SURVEY.md §8d).

Counter-based splitmix64 (the same generator a Go/C++ harness can reproduce):
value k of stream s under seed S is mix64(S + stream_salt(s) + (k+1)*GOLDEN).
Everything is produced column-wise with numpy straight into the SoA tables the
C-ABI takes; oracle.SoAJob rebuilds reference-shaped strings from the same
tables for the CPU side.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

from . import _lib as L
from . import model as M
from .soa import SQ_BASE, AliasTable, DepsTable, DistroTable, HostSoA, TaskEdit, TaskSoA, apply_edit

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
NOW_NS = 1_800_000_000 * 10 ** 9
SEED_BASE = 0xE5E60000


def mix64(z: np.ndarray) -> np.ndarray:
    z = z.astype(np.uint64, copy=True)
    with np.errstate(over="ignore"):
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z


class Rng:
    def __init__(self, seed: int):
        self.seed = np.uint64(seed)
        self.stream = 0

    def u64(self, n: int) -> np.ndarray:
        self.stream += 1
        with np.errstate(over="ignore"):
            salt = mix64(np.array([self.stream], dtype=np.uint64) * np.uint64(0xD1342543DE82EF95))[0]
            k = (np.arange(1, n + 1, dtype=np.uint64) * GOLDEN) + self.seed + salt
        return mix64(k)

    def uniform(self, n: int) -> np.ndarray:
        return (self.u64(n) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))

    def integers(self, n: int, lo: int, hi: int) -> np.ndarray:
        """uniform integers in [lo, hi]"""
        span = hi - lo + 1
        return (lo + (self.uniform(n) * span).astype(np.int64)).clip(lo, hi)


@dataclass
class Workload:
    name: str
    now: int
    tasks: TaskSoA
    distros: DistroTable
    hosts: Optional[HostSoA]

    @property
    def n_tasks(self) -> int:
        return self.tasks.n_tasks

    def algorithmic_bytes(self) -> int:
        """SURVEY.md §8d: 60*T + 4*E + 28*H + 96*G + 16*D (compulsory traffic only)."""
        H = self.hosts.n_hosts if self.hosts is not None else 0
        return (60 * self.tasks.n_tasks + 4 * self.tasks.n_edges + 28 * H + 96 * self.distros.n_groups +
                16 * self.distros.n_distros)


def _ranges(off: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """Concatenated index ranges [off[i], off[i+1]) for i in ids, in that order."""
    lens = (off[ids + 1] - off[ids]).astype(np.int64)
    if lens.sum() == 0:
        return np.zeros(0, dtype=np.int64)
    starts = np.repeat(off[ids], lens)
    within = np.arange(int(lens.sum()), dtype=np.int64) - np.repeat(np.cumsum(lens) - lens, lens)
    return starts + within


def take_distros(w: Workload, ids) -> Workload:
    """The sub-tick of the distros `ids` (in that order): what one rank of a distro-sharded job uploads.  Task groups,
    versions and in-queue dependency edges are distro-local, so rows move as they are."""
    ids = np.asarray(ids, dtype=np.int64)
    t, d, h = w.tasks, w.distros, w.hosts
    rows = _ranges(d.task_off, ids)
    cols = {name: getattr(t, name)[rows] for name, _ in t.COLUMNS}
    dep_off = dep_idx = None
    if t.n_edges:
        deg = (t.dep_off[rows + 1] - t.dep_off[rows]).astype(np.int64)
        dep_off = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        dep_idx = t.dep_idx[_ranges(t.dep_off, rows)] if deg.sum() else np.zeros(0, dtype=np.int32)
    tasks = TaskSoA(**cols, dep_off=dep_off, dep_idx=dep_idx).normalize()
    n = (d.task_off[ids + 1] - d.task_off[ids]).astype(np.int64)
    g = (d.group_off[ids + 1] - d.group_off[ids]).astype(np.int64)
    distros = DistroTable(np.concatenate([[0], np.cumsum(n)]).astype(np.int64), np.concatenate([[0], np.cumsum(g)]).astype(np.int64),
                          d.cfg[ids], d.group_max_hosts[_ranges(d.group_off, ids)]).normalize()
    hosts = None
    if h is not None:
        hr = _ranges(h.host_off, ids)
        hn = (h.host_off[ids + 1] - h.host_off[ids]).astype(np.int64)
        hosts = HostSoA(h.flags[hr], h.group_id[hr], h.expected_ns[hr], h.std_ns[hr], h.start_ns[hr],
                        np.concatenate([[0], np.cumsum(hn)]).astype(np.int64), h.cfg[ids]).normalize()
    return Workload(f"{w.name} [{len(ids)} of {d.n_distros} distros]", w.now, tasks, distros, hosts)


def _zipf_priorities(rng: Rng, n: int, s: float = 1.1, kmax: int = 100) -> np.ndarray:
    ranks = np.arange(1, kmax + 2, dtype=np.float64)
    w = ranks ** (-s)
    cdf = np.cumsum(w) / w.sum()
    return np.searchsorted(cdf, rng.uniform(n)).clip(0, kmax).astype(np.int32)


def make(sizes: np.ndarray, seed: int, *, name: str = "synthetic", now: int = NOW_NS, zipf_priority: bool = False,
         unmet_dep_frac: float = 0.0, met_dep_frac: float = 0.0, tg_frac: float = 0.10,
         group_versions_frac: float = 0.0, custom_factor_frac: float = 0.10, includes_dependencies: bool = False,
         n_hosts: int = 0, providers: Tuple[float, float, float] = (1.0, 0.0, 0.0)) -> Workload:
    """Build one tick. `sizes[d]` = tasks queued on distro d.
    providers = fractions (ephemeral, docker+pool, static)."""
    sizes = np.asarray(sizes, dtype=np.int64)
    D = int(sizes.shape[0])
    rng = Rng(seed)
    task_off = np.zeros(D + 1, dtype=np.int64)
    np.cumsum(sizes, out=task_off[1:])
    T = int(task_off[-1])
    distro_of = np.repeat(np.arange(D, dtype=np.int64), sizes)
    local = np.arange(T, dtype=np.int64) - task_off[distro_of]

    expected = rng.integers(T, 10 * M.SECOND, 2 * M.HOUR)
    queue_basis = now - rng.integers(T, 0, 72 * M.HOUR)
    wait_basis = now - rng.integers(T, 0, 3 * M.HOUR)
    u = rng.uniform(T)
    req = np.where(u < 0.40, L.EVG_TF_REQ_PATCH, np.where(u < 0.45, L.EVG_TF_REQ_MERGE_QUEUE, L.EVG_TF_REQ_OTHER))
    priority = _zipf_priorities(rng, T) if zipf_priority else np.zeros(T, dtype=np.int32)
    numdep = np.floor(np.log(np.maximum(rng.uniform(T), 1e-300)) / np.log(0.3)).astype(np.int32).clip(0, 10000)
    flags = req.astype(np.uint32)
    flags |= np.where(rng.uniform(T) < 0.01, L.EVG_TF_GENERATE, 0).astype(np.uint32)
    flags |= np.where(rng.uniform(T) < 0.01, L.EVG_TF_STEPBACK, 0).astype(np.uint32)
    flags |= np.where(rng.uniform(T) < 0.005, L.EVG_TF_OTHER_DISTRO, 0).astype(np.uint32)

    # versions: ~50 tasks per version per distro
    n_versions = np.maximum(1, sizes // 50).astype(np.int64)
    version = (rng.uniform(T) * n_versions[distro_of]).astype(np.int64).clip(0, None)
    version = np.minimum(version, n_versions[distro_of] - 1)

    # task groups: a random 10% of tasks, chunked into groups in order of appearance
    is_tg = rng.uniform(T) < tg_frac
    tg_idx = np.nonzero(is_tg)[0]
    gid = np.full(T, -1, dtype=np.int64)
    tgo = np.zeros(T, dtype=np.int32)
    group_off = np.zeros(D + 1, dtype=np.int64)
    group_max_hosts = np.zeros(0, dtype=np.int32)
    if tg_idx.shape[0]:
        n = tg_idx.shape[0]
        d_tg = distro_of[tg_idx]
        first_in_distro = np.ones(n, dtype=bool)
        first_in_distro[1:] = d_tg[1:] != d_tg[:-1]
        brk = (rng.uniform(n) < 0.2) | first_in_distro
        # position inside the run since the last break; force a break every 8 members
        start_pos = np.maximum.accumulate(np.where(brk, np.arange(n), 0))
        pos = np.arange(n) - start_pos
        brk |= (pos % 8 == 0)
        start_pos = np.maximum.accumulate(np.where(brk, np.arange(n), 0))
        pos = np.arange(n) - start_pos
        gglobal = np.cumsum(brk) - 1                    # global group number
        gfirst = np.zeros(D + 1, dtype=np.int64)        # groups before each distro
        counts = np.bincount(d_tg[brk], minlength=D)
        np.cumsum(counts, out=gfirst[1:])
        group_off = gfirst.copy()
        gid[tg_idx] = gglobal - gfirst[d_tg]
        tgo[tg_idx] = (pos + 1).astype(np.int32)
        version[tg_idx] = version[tg_idx[start_pos]]    # a group lives in one version
        group_max_hosts = rng.integers(int(gfirst[-1]), 1, 4).astype(np.int32)

    # dependency edges onto other in-queue tasks
    dep_off = None
    dep_idx = None
    deps_met = np.ones(T, dtype=bool)
    if unmet_dep_frac > 0 or met_dep_frac > 0:
        ud = rng.uniform(T)
        has_unmet = (ud < unmet_dep_frac) & (sizes[distro_of] > 1)
        has_met = (ud >= unmet_dep_frac) & (ud < unmet_dep_frac + met_dep_frac) & (sizes[distro_of] > 1)
        n_dep = np.where(has_unmet | has_met, 1 + (rng.uniform(T) < 0.2), 0).astype(np.int64)
        dep_off = np.zeros(T + 1, dtype=np.int64)
        np.cumsum(n_dep, out=dep_off[1:])
        E = int(dep_off[-1])
        owner = np.repeat(np.arange(T, dtype=np.int64), n_dep)
        tgt = (rng.uniform(E) * (sizes[distro_of[owner]] - 1)).astype(np.int64)
        tgt = np.minimum(tgt, sizes[distro_of[owner]] - 2)
        tgt = np.where(tgt >= local[owner], tgt + 1, tgt)  # never depend on yourself
        dep_idx = tgt.astype(np.int32)
        deps_met = ~has_unmet
    else:
        # a few tasks wait on something outside the queue
        deps_met = rng.uniform(T) >= 0.01
    flags |= np.where(deps_met, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)

    tasks = TaskSoA(priority, expected, queue_basis, wait_basis, numdep, tgo, gid.astype(np.int32),
                    version.astype(np.int32), flags, dep_off, dep_idx).normalize()

    cfg = np.zeros(D, dtype=L.DISTRO_CFG_DTYPE)
    custom = rng.uniform(D) < custom_factor_frac
    for f in ("patch_factor", "patch_time_in_queue_factor", "commit_queue_factor", "mainline_time_in_queue_factor",
              "expected_runtime_factor", "generate_task_factor", "stepback_task_factor"):
        cfg[f] = np.where(custom, rng.integers(D, 1, 100), 0)
    cfg["num_dependents_factor"] = np.where(custom, np.round(rng.uniform(D) * 100, 2), 0.0)
    prov_u = rng.uniform(D)
    provider = np.where(prov_u < providers[0], L.EVG_PROVIDER_EPHEMERAL,
                        np.where(prov_u < providers[0] + providers[1], L.EVG_PROVIDER_DOCKER, L.EVG_PROVIDER_STATIC))
    has_pool = provider == L.EVG_PROVIDER_DOCKER
    cfg["target_time_ns"] = np.where(has_pool, M.MAX_DURATION_PER_DISTRO_HOST_WITH_CONTAINERS, M.MAX_DURATION_PER_DISTRO_HOST)
    cfg["group_versions"] = (rng.uniform(D) < group_versions_frac).astype(np.int32)
    cfg["includes_dependencies"] = int(includes_dependencies)
    cfg["n_versions"] = n_versions.astype(np.int32)
    distros = DistroTable(task_off, group_off, cfg, group_max_hosts).normalize()

    hosts = None
    if n_hosts > 0:
        share = sizes.astype(np.float64) / max(1, sizes.sum())
        hcount = np.floor(share * n_hosts).astype(np.int64)
        hcount[: int(n_hosts - hcount.sum())] += 1 if D else 0
        host_off = np.zeros(D + 1, dtype=np.int64)
        np.cumsum(hcount, out=host_off[1:])
        H = int(host_off[-1])
        hd = np.repeat(np.arange(D, dtype=np.int64), hcount)
        running = rng.uniform(H) < 0.7
        found = running & (rng.uniform(H) < 0.98)
        teardown = (~running) & (rng.uniform(H) < 0.03)
        hflags = (np.where(running, L.EVG_HF_RUNNING, 0) | np.where(found, L.EVG_HF_RT_FOUND, 0) |
                  np.where(teardown, L.EVG_HF_TEARDOWN, 0)).astype(np.uint32)
        hexp = np.where(found, rng.integers(H, 10 * M.SECOND, 2 * M.HOUR), 0)
        hstd = np.where(found, hexp // 5, 0)
        elapsed = (rng.uniform(H) * 2.0 * hexp).astype(np.int64)
        hstart = np.where(found, now - elapsed, M.ZERO_TIME)
        ng = (group_off[1:] - group_off[:-1])[hd] if H else np.zeros(0, dtype=np.int64)
        in_group = running & (rng.uniform(H) < 0.05)
        pick = (rng.uniform(H) * np.maximum(ng, 1)).astype(np.int64)
        hgid = np.where(in_group, np.where((ng > 0) & (rng.uniform(H) < 0.8), np.minimum(pick, np.maximum(ng - 1, 0)),
                                           L.EVG_HG_UNQUEUED), L.EVG_HG_NONE).astype(np.int32)
        acfg = np.zeros(D, dtype=L.ALLOC_CFG_DTYPE)
        acfg["future_host_fraction"] = 0.4
        acfg["provider"] = provider
        acfg["disabled"] = (rng.uniform(D) < 0.02).astype(np.int32)
        acfg["minimum_hosts"] = rng.integers(D, 0, 2)
        acfg["maximum_hosts"] = rng.integers(D, 10, 500)
        acfg["round_up"] = (rng.uniform(D) < 0.1).astype(np.int32)
        acfg["waits_over_thresh_feedback"] = (rng.uniform(D) < 0.2).astype(np.int32)
        acfg["has_pool"] = has_pool.astype(np.int32)
        acfg["pool_max_containers"] = np.where(has_pool, 10, 0)
        acfg["parent_found"] = has_pool.astype(np.int32)
        acfg["parent_maximum_hosts"] = np.where(has_pool, rng.integers(D, 5, 50), 0)
        hosts = HostSoA(hflags, hgid, hexp, hstd, hstart, host_off, acfg).normalize()
    return Workload(name, now, tasks, distros, hosts)


# ---------------------------------------------------------------- edge values
# make() stays inside the domain of the kernels' 32-bit scorer (evg_score.cuh: factors below 2^14, priority and
# NumDependents below 2^15, time in queue and expected duration below 2^50 ns, a clock and bases at or after 1970).
# sprinkle_edges() overwrites rows of a tick with values at and beyond those limits -- and with the values production
# does produce: compile tasks with thousands of dependents, stale patches, admin priorities, clock skew, epoch-zero
# times, TotalValue wrapping int64 (DESIGN.md §3).
I64_MAX = 2 ** 63 - 1
FAST_LIMIT_NS = (1 << 15) * M.MINUTE  # evg_score.cuh kFastLimit: 2^15 minutes
WEEK_NS = 7 * 24 * M.HOUR
EDGE_SALT = 0x3DCE0D6E

EDGE_VALUES = {
    "nd": [-1, 32, 63, 64, 65, 2 ** 15 - 1, 2 ** 15, 2 ** 31 - 1],                    # NumDependents
    "prio": [-2 ** 31, -1, 2 ** 15 - 1, 2 ** 15, 2 ** 31 - 1],                        # priority
    "tiq": [2 ** 50 - 1, 2 ** 50, FAST_LIMIT_NS - 1, FAST_LIMIT_NS + 1, WEEK_NS - 1,  # time in queue (basis = now - tiq)
            WEEK_NS + 1, 0, FAST_LIMIT_NS],
    "basis": ["now+1", 0, -2 ** 63 + 1, M.ZERO_TIME],                                 # queue and wait basis
    # expected duration; 2^62 + 1 twice in a distro wraps its int64 expected-duration sums
    "exp": [2 ** 50 - 1, 2 ** 50, FAST_LIMIT_NS - 1, FAST_LIMIT_NS, FAST_LIMIT_NS + 1, -1, 0, 2 ** 62 + 1],
    "thresh": [-1, 0, 1],                                                             # offset from the distro's target time
    "u32": ["high", "low"],   # TotalValue 2^32 + 401 (merge queue, priority 2^31 - 1) and 2: a range of 33 bits
    "wrap": ["neg", "pos"],   # TotalValue wrapped to below -2^62 / above 2^62: a range beyond 2^63
}
ROW_KINDS = tuple(EDGE_VALUES)
# distro-level knobs, dealt to the distros in turn (None: left as make() drew it)
EDGE_FACTORS = [None, 2 ** 14 - 1, None, 0, None, -5, 2 ** 14]   # the seven integer factors (<= 0 clamps to 1)
EDGE_NDF = [None, 2.5, 7.0, 2.0 ** 27 + 0.5, 2 ** 14 - 1.0, 0.01]  # NumDependentsFactor; 2^27+.5: table entries pass 2^32 at n = 32
DISTRO_KINDS = ("factors", "ndf", "clock")
_INT_FACTORS = ("patch_factor", "patch_time_in_queue_factor", "commit_queue_factor", "mainline_time_in_queue_factor",
                "expected_runtime_factor", "generate_task_factor", "stepback_task_factor")


def _wrap64(x: int) -> int:
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


def _floor_minutes(d: int) -> int:
    """int64(math.Floor(time.Duration(d).Minutes())) for d >= 0 (the stdlib's two-term FP64 formula)."""
    return int(np.floor(float(d // M.MINUTE) + float(d % M.MINUTE) / (60 * 1e9)))


def _wrapping_expected(cfg, negative: bool) -> int:
    """An expected duration (whole minutes) at which a lone patch task of priority 2^31 - 1 with the generator flag, a
    saturated time in queue and no dependents has TotalValue (unitInfo.value, planner.go:209-300) in
    [-2^62 - 2^61, -2^62) (negative) or in [2^62 + 2^60, 2^63).  Each minute moves the wrapped value by
    2^31 * GenerateTaskFactor * ExpectedRuntimeFactor (2^37.6 or more), so some minute below 2^64 / that step
    (< 1.6e8 minutes, inside int64 nanoseconds) lands in the window."""
    f = {k: (int(cfg[k]) if int(cfg[k]) > 0 else 1) for k in _INT_FACTORS}
    prio = 2 ** 31 * f["generate_task_factor"]
    a = prio * (1 + f["patch_factor"] + f["patch_time_in_queue_factor"] * _floor_minutes(I64_MAX)) + 1
    step = prio * f["expected_runtime_factor"]
    lo, hi = (-2 ** 62 - 2 ** 61, -2 ** 62) if negative else (2 ** 62 + 2 ** 60, 2 ** 63)
    m = -(-((lo - a) % 2 ** 64) // step)
    assert lo <= _wrap64(a + step * m) < hi and m * M.MINUTE <= I64_MAX
    return m * M.MINUTE


def sprinkle_edges(w: Workload, seed: int, *, kinds, frac: Optional[float] = None, positions=None) -> dict:
    """Overwrite rows of `w` in place with edge values.  Row kinds (EDGE_VALUES) are dealt to the chosen rows in turn,
    each kind's values in turn; the distro kinds ("factors", "ndf", "clock") set distro d's knob to entry d of their
    list.  Rows: `positions` (global row indices), else a `frac` of all rows, else one in 32.  A stream of its own, so
    make() draws the same tick for every seed whether or not edges are sprinkled afterwards.  Group ids, versions and
    dependency edges are left alone: the tick stays valid.  Returns {kind: global rows it wrote}."""
    rng = Rng(seed ^ EDGE_SALT)
    t, dt = w.tasks, w.distros
    cfg = dt.cfg
    D = dt.n_distros
    kinds = tuple(kinds)
    unknown = [k for k in kinds if k not in EDGE_VALUES and k not in DISTRO_KINDS]
    if unknown:
        raise ValueError(f"unknown edge kinds {unknown}")
    now = int(w.now)
    for d in range(D):
        if "factors" in kinds and EDGE_FACTORS[d % len(EDGE_FACTORS)] is not None:
            for f in _INT_FACTORS:
                cfg[f][d] = EDGE_FACTORS[d % len(EDGE_FACTORS)]
        if "ndf" in kinds and EDGE_NDF[d % len(EDGE_NDF)] is not None:
            cfg["num_dependents_factor"][d] = EDGE_NDF[d % len(EDGE_NDF)]
        if "clock" in kinds and d % 3 == 2:
            cfg["target_time_ns"][d] = now + M.HOUR  # a threshold in the future: the literal time.Since comparison
    row_kinds = [k for k in kinds if k in EDGE_VALUES]
    out = {k: [] for k in row_kinds}
    if not row_kinds or t.n_tasks == 0:
        return {k: np.zeros(0, np.int64) for k in out}
    if positions is not None:
        rows = np.unique(np.asarray(positions, dtype=np.int64))
    else:
        rows = np.nonzero(rng.uniform(t.n_tasks) < (frac if frac is not None else 1.0 / 32))[0]
    distro_of = np.searchsorted(dt.task_off, rows, side="right") - 1
    aim = {}  # (distro, sign) -> expected duration that wraps TotalValue to that sign
    for j, (r, d) in enumerate(zip(rows.tolist(), distro_of.tolist())):
        kind = row_kinds[j % len(row_kinds)]
        vals = EDGE_VALUES[kind]
        v = vals[(j // len(row_kinds)) % len(vals)]
        if kind == "u32" and (t.group_id[r] >= 0 or cfg["group_versions"][d]):
            continue  # a lone task's value: a unit's would add its other members' terms
        out[kind].append(r)
        if kind == "nd":
            t.num_dependents[r] = v
        elif kind == "prio":
            t.priority[r] = v
        elif kind == "tiq":
            t.queue_basis_ns[r] = now - v
        elif kind == "basis":
            b = now + 1 if v == "now+1" else v
            t.queue_basis_ns[r] = b
            t.wait_basis_ns[r] = b
        elif kind == "exp":
            t.expected_ns[r] = v
        elif kind == "thresh":
            target = int(cfg["target_time_ns"][d])
            t.wait_basis_ns[r] = _wrap64(now - target + v)
            t.expected_ns[r] = target + v
            t.flags[r] |= L.EVG_TF_DEPS_MET
        elif kind == "u32":
            keep = int(t.flags[r]) & (L.EVG_TF_DEPS_MET | L.EVG_TF_OTHER_DISTRO)
            cfg["commit_queue_factor"][d] = 1
            cfg["num_dependents_factor"][d] = 0.0
            t.num_dependents[r] = 0
            t.expected_ns[r] = 0
            if v == "high":  # (1 + 2^31 - 1 + 200) * (1 + CommitQueueFactor) + 1
                t.priority[r] = 2 ** 31 - 1
                t.flags[r] = keep | L.EVG_TF_REQ_MERGE_QUEUE
            else:            # mainline, waited over a week: 1 * 1 + 1
                t.priority[r] = -1
                t.flags[r] = keep | L.EVG_TF_REQ_OTHER
                t.queue_basis_ns[r] = now - 2 * WEEK_NS
        elif kind == "wrap":
            # priority 2^31 - 1 times GenerateTaskFactor 100, times a rank that holds the saturated time.Since of a basis
            # at the start of int64: the product wraps; the expected duration aims the wrap at the wanted sign
            keep = int(t.flags[r]) & (L.EVG_TF_DEPS_MET | L.EVG_TF_OTHER_DISTRO)
            cfg["generate_task_factor"][d] = 100
            if (d, v) not in aim:
                aim[(d, v)] = _wrapping_expected(cfg[d], v == "neg")
            t.priority[r] = 2 ** 31 - 1
            t.flags[r] = keep | L.EVG_TF_REQ_PATCH | L.EVG_TF_GENERATE
            t.queue_basis_ns[r] = -2 ** 63 + 1
            t.num_dependents[r] = 0
            t.expected_ns[r] = aim[(d, v)]
    return {k: np.asarray(v, dtype=np.int64) for k, v in out.items()}


# ---------------------------------------------------------------- the next tick
EDIT_SALT = 0x7E11C0DE


@dataclass
class EditTick:
    edit: TaskEdit            # membership change (evg_edit_tasks)
    rows: np.ndarray          # composed rows whose scalars changed (evg_update_tasks)
    values: TaskSoA           # their new values
    workload: Workload        # the composed tick with the changes: what a fresh upload of the next tick holds


def _rank_within(keys: np.ndarray) -> np.ndarray:
    """Position of each element among the elements with the same (sorted-run) key before it."""
    n = keys.shape[0]
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    start = np.ones(n, dtype=bool)
    start[1:] = keys[1:] != keys[:-1]
    first = np.maximum.accumulate(np.where(start, np.arange(n), 0))
    return np.arange(n) - first


def next_tick(w: Workload, seed: int, *, dispatch: float = 0.05, arrive: float = 0.05, change: float = 0.05,
              order: Optional[np.ndarray] = None, remap: bool = True, dep_frac: float = 0.1,
              add_edge_frac: float = 0.01) -> EditTick:
    """The tick after `w`: a `dispatch` fraction of rows leaves (biased to the heads of the queues `order` ranked, the
    planner's last order, when given), an `arrive` fraction of each queue's size joins -- some rows join existing or new
    task groups and versions, a `dep_frac` of them depend on survivors or other arrivals -- an `add_edge_frac` of the
    survivors gain a dependency, and a `change` fraction of the composed rows take new scalars.  With `remap`, group and
    version ids are re-densified in first-appearance order over the composed queue (no dead slots); without it they are
    kept and new ones appended.  A stream of its own: make()'s ticks are unchanged."""
    rng = Rng(seed ^ EDIT_SALT)
    t, dt = w.tasks, w.distros
    D, T0 = dt.n_distros, t.n_tasks
    toff, goff = dt.task_off, dt.group_off
    sizes = np.diff(toff)
    distro_of = np.repeat(np.arange(D, dtype=np.int64), sizes)
    # dispatch
    p = np.full(T0, dispatch)
    if order is not None and T0:
        rank = np.empty(T0, dtype=np.int64)
        rank[toff[distro_of] + order.astype(np.int64)] = np.arange(T0) - toff[distro_of]
        p = 2.0 * dispatch * (1.0 - rank / np.maximum(sizes[distro_of], 1))
    keep = rng.uniform(T0) >= p
    remove = np.nonzero(~keep)[0].astype(np.int64)
    surv = np.nonzero(keep)[0]
    surv_d = distro_of[surv]
    n_surv = np.bincount(surv_d, minlength=D).astype(np.int64)
    # group / version ids of the survivors in the new id space
    nver_old = dt.cfg["n_versions"].astype(np.int64)
    vbase = np.concatenate([[0], np.cumsum(nver_old)])
    ng_old = np.diff(goff)
    if remap:
        grouped = t.group_id[surv] >= 0
        gremap = np.full(int(goff[-1]), -1, dtype=np.int64)
        vremap = np.full(int(vbase[-1]), -1, dtype=np.int64)
        for slot, dd, out in ((goff[surv_d[grouped]] + t.group_id[surv][grouped], surv_d[grouped], gremap),
                              (vbase[surv_d] + t.version_id[surv], surv_d, vremap)):
            u, first = np.unique(slot, return_index=True)
            by_first = np.argsort(first)  # survivors ascend by distro: first-appearance order is grouped by distro
            out[u[by_first]] = _rank_within(dd[first[by_first]])
        ng_cur = np.bincount(np.repeat(np.arange(D), ng_old)[gremap >= 0], minlength=D).astype(np.int64)
        nv_cur = np.bincount(np.repeat(np.arange(D), nver_old)[vremap >= 0], minlength=D).astype(np.int64)
        group_of_old = np.full(T0, -1, dtype=np.int64)
        mm = t.group_id >= 0
        group_of_old[mm] = gremap[goff[distro_of[mm]] + t.group_id[mm]]
        version_of_old = vremap[vbase[distro_of] + t.version_id]
    else:
        gremap = vremap = None
        ng_cur, nv_cur = ng_old.astype(np.int64), nver_old.copy()
        group_of_old, version_of_old = t.group_id.astype(np.int64), t.version_id.astype(np.int64)
    # each current group's version (a task group lives in one version)
    gbase_cur = np.concatenate([[0], np.cumsum(ng_cur)])
    grp_ver = np.zeros(int(gbase_cur[-1]), dtype=np.int64)
    m = group_of_old >= 0
    grp_ver[gbase_cur[distro_of[m]] + group_of_old[m]] = version_of_old[m]
    # arrivals
    n_ins = np.floor(arrive * sizes + rng.uniform(D)).astype(np.int64)
    I = int(n_ins.sum())
    ins_d = np.repeat(np.arange(D, dtype=np.int64), n_ins)
    ins_k = _rank_within(ins_d)
    new_n = n_surv + n_ins
    newv = (rng.uniform(I) < 0.2) | (nv_cur[ins_d] == 0)
    vid = np.minimum((rng.uniform(I) * nv_cur[ins_d]).astype(np.int64), np.maximum(nv_cur[ins_d] - 1, 0))
    o = np.lexsort((ins_k, ins_d, ~newv))
    nv_rank = np.empty(I, dtype=np.int64)
    nv_rank[o] = _rank_within((ins_d * 2 + newv)[o])
    vid = np.where(newv, nv_cur[ins_d] + nv_rank // 5, vid)
    nv_new = nv_cur.copy()
    np.maximum.at(nv_new, ins_d, vid + 1)
    is_tg = rng.uniform(I) < 0.15
    join = is_tg & (rng.uniform(I) < 0.5) & (ng_cur[ins_d] > 0)
    newg = is_tg & ~join
    gid = np.full(I, -1, dtype=np.int64)
    gj = np.minimum((rng.uniform(I) * ng_cur[ins_d]).astype(np.int64), np.maximum(ng_cur[ins_d] - 1, 0))
    gid[join] = gj[join]
    vid[join] = grp_ver[gbase_cur[ins_d[join]] + gj[join]]
    o = np.lexsort((ins_k, ins_d, ~newg))
    ng_rank = np.empty(I, dtype=np.int64)
    ng_rank[o] = _rank_within((ins_d * 2 + newg)[o])
    gid[newg] = ng_cur[ins_d[newg]] + ng_rank[newg] // 3
    ng_new = ng_cur.copy()
    np.maximum.at(ng_new, ins_d[newg], gid[newg] + 1)
    # a new group's members take the version of its first member
    key = ins_d * (1 << 32) + np.where(newg, gid, -1)
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    vid[newg] = vid[first[inv]][newg]
    tgo = np.where(is_tg, rng.integers(I, 1, 8), 0).astype(np.int32)
    # the arrivals' own edges, as new distro-local indices (never to themselves)
    has_dep = (rng.uniform(I) < dep_frac) & (new_n[ins_d] > 1)
    self_loc = n_surv[ins_d] + ins_k
    tgt = np.minimum((rng.uniform(I) * (new_n[ins_d] - 1)).astype(np.int64), np.maximum(new_n[ins_d] - 2, 0))
    tgt = np.where(tgt >= self_loc, tgt + 1, tgt)
    ins_dep_off = np.concatenate([[0], np.cumsum(has_dep)]).astype(np.int64)
    now = int(w.now)
    u = rng.uniform(I)
    flags = np.where(u < 0.4, L.EVG_TF_REQ_PATCH, np.where(u < 0.45, L.EVG_TF_REQ_MERGE_QUEUE, L.EVG_TF_REQ_OTHER)).astype(np.uint32)
    flags |= np.where(rng.uniform(I) < 0.95, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
    flags |= np.where(rng.uniform(I) < 0.01, L.EVG_TF_GENERATE, 0).astype(np.uint32)
    insert = TaskSoA(_zipf_priorities(rng, I), rng.integers(I, 10 * M.SECOND, 2 * M.HOUR), now - rng.integers(I, 0, 3 * M.HOUR),
                     now - rng.integers(I, 0, M.HOUR), rng.integers(I, 0, 3).astype(np.int32), tgo, gid.astype(np.int32),
                     vid.astype(np.int32), flags, ins_dep_off, tgt[has_dep].astype(np.int32)).normalize()
    # survivors that gain a dependency
    gain = rng.uniform(surv.shape[0]) < add_edge_frac
    surv_loc = _rank_within(surv_d)
    new_off = np.concatenate([[0], np.cumsum(new_n)])
    gain &= new_n[surv_d] > 1
    gt = np.minimum((rng.uniform(surv.shape[0]) * (new_n[surv_d] - 1)).astype(np.int64), np.maximum(new_n[surv_d] - 2, 0))
    gt = np.where(gt >= surv_loc, gt + 1, gt)
    # the new distro table
    G_new = int(ng_new.sum())
    goff_new = np.concatenate([[0], np.cumsum(ng_new)]).astype(np.int64)
    gmax = rng.integers(G_new, 1, 3).astype(np.int32)
    if remap:
        live = gremap >= 0
        old_d = np.repeat(np.arange(D, dtype=np.int64), ng_old)
        gmax[goff_new[old_d[live]] + gremap[live]] = dt.group_max_hosts[live]
    else:
        old_d = np.repeat(np.arange(D, dtype=np.int64), ng_old)
        gmax[goff_new[old_d] + (np.arange(int(goff[-1])) - goff[old_d])] = dt.group_max_hosts
    cfg = dt.cfg.copy()
    cfg["n_versions"] = nv_new.astype(np.int32)
    edit = TaskEdit(remove, insert, np.concatenate([[0], np.cumsum(n_ins)]).astype(np.int64),
                    (new_off[surv_d] + surv_loc)[gain].astype(np.int64), gt[gain].astype(np.int32),
                    None if gremap is None or gremap.shape[0] == 0 else gremap.astype(np.int32),
                    None if vremap is None else vremap.astype(np.int32), goff_new, gmax, cfg).normalize()
    tasks, distros = apply_edit(t, dt, edit)
    # value changes on the composed rows
    Tn = tasks.n_tasks
    rows = np.nonzero(rng.uniform(Tn) < change)[0].astype(np.int64)
    n = rows.shape[0]
    tasks.priority[rows] = _zipf_priorities(rng, n)
    tasks.expected_ns[rows] = rng.integers(n, 10 * M.SECOND, 2 * M.HOUR)
    tasks.wait_basis_ns[rows] = now - rng.integers(n, 0, 3 * M.HOUR)
    tasks.num_dependents[rows] = rng.integers(n, 0, 5).astype(np.int32)
    tasks.flags[rows] ^= np.where(rng.uniform(n) < 0.3, L.EVG_TF_DEPS_MET, 0).astype(np.uint32)
    values = TaskSoA(**{name: getattr(tasks, name)[rows] for name, _ in TaskSoA.COLUMNS}).normalize()
    hosts = w.hosts
    if hosts is not None and remap:
        hd = np.repeat(np.arange(D, dtype=np.int64), np.diff(hosts.host_off))
        hg = hosts.group_id.astype(np.int64)
        m = hg >= 0
        hg[m] = gremap[goff[hd[m]] + hg[m]]
        hg[m & (hg < 0)] = L.EVG_HG_UNQUEUED
        hosts = HostSoA(hosts.flags.copy(), hg.astype(np.int32), hosts.expected_ns.copy(), hosts.std_ns.copy(),
                        hosts.start_ns.copy(), hosts.host_off.copy(), hosts.cfg.copy()).normalize()
    return EditTick(edit, rows, values, Workload(w.name, w.now, tasks, distros, hosts))


ALIAS_SALT = 0xA11A5


def make_aliases(w: Workload, seed: int, *, name_frac: float = 0.2, big: int = 0):
    """The alias side of tick w, from its own random stream: w's rows are the tick's schedulable tasks (each once; a
    row's primary distro is the one w files it under) and w's distros the alias distros -> (AliasTable, cfg).
    A name_frac share of tasks carries 1-3 SecondaryDistros names: distro ids (the task's own among them), alias names
    that several distros share, and names no distro has.  Some rows fail a base-query bit, carry an unattainable
    dependency (with or without the override), or sit in a single-host task group (or carry TaskGroupMaxHosts == 1
    without one).  big > 0: the first `big` rows also name an alias of distro 0 and pass every filter, so its alias
    queue takes the general path once big > 12 288."""
    t, dt = w.tasks, w.distros
    T, D = t.n_tasks, dt.n_distros
    rng = Rng(seed ^ ALIAS_SALT)
    distro_of = np.repeat(np.arange(D, dtype=np.int64), np.diff(dt.task_off))
    vbase = np.concatenate([[0], np.cumsum(dt.cfg["n_versions"].astype(np.int64))])
    gid = np.where(t.group_id >= 0, dt.group_off[distro_of] + t.group_id, -1).astype(np.int32)
    vid = (vbase[distro_of] + t.version_id).astype(np.int32)
    flags = t.flags & np.uint32(~(L.EVG_TF_DEPS_MET | L.EVG_TF_OTHER_DISTRO) & 0xFFFFFFFF)
    dep_off, dep_idx = t.dep_off, t.dep_idx
    if t.n_edges:
        owner = np.repeat(np.arange(T, dtype=np.int64), np.diff(t.dep_off))
        dep_idx = (dt.task_off[distro_of[owner]] + t.dep_idx).astype(np.int32)
    tasks = TaskSoA(t.priority, t.expected_ns, t.queue_basis_ns, t.wait_basis_ns, t.num_dependents, t.task_group_order, gid, vid,
                    flags, dep_off, dep_idx).normalize()
    gmax = dt.group_max_hosts.astype(np.int32)  # 1 .. 3: the groups of 1 are single-host groups
    tgmax = np.where(gid >= 0, gmax[np.maximum(gid, 0)] if gmax.shape[0] else 0,
                     np.where(rng.uniform(T) < 0.02, 1, 0)).astype(np.int32)
    sched = np.full(T, SQ_BASE, dtype=np.uint8)
    for bit in (L.EVG_SQ_ACTIVATED, L.EVG_SQ_UNDISPATCHED, L.EVG_SQ_PRIORITY_OK, L.EVG_SQ_HOST_PLATFORM):
        sched &= np.where(rng.uniform(T) < 0.01, ~bit & 0xFF, 0xFF).astype(np.uint8)
    sched |= np.where(rng.uniform(T) < 0.04, L.EVG_SQ_UNATTAINABLE, 0).astype(np.uint8)
    sched |= np.where(rng.uniform(T) < 0.03, L.EVG_SQ_OVERRIDE_DEPS, 0).astype(np.uint8)
    primary = np.where(rng.uniform(T) < 0.02, -1, distro_of).astype(np.int32)
    # names: 0 .. D-1 the distros' own ids, then A alias names; each distro takes 0-2 of them (shared between distros)
    A = max(2, D // 3)
    n_alias = rng.integers(D, 0, 2)
    pick = rng.integers(2 * D, 0, A - 1).reshape(2, D) if D else np.zeros((2, 0), np.int64)
    dests = [[] for _ in range(D + A + (1 if big else 0))]
    for e in range(D):
        dests[e].append(e)
        for k in range(int(n_alias[e])):
            if e not in dests[D + int(pick[k, e])]:
                dests[D + int(pick[k, e])].append(e)
    if big:
        dests[D + A].append(0)
    carries = rng.uniform(T) < name_frac
    n_names = np.where(carries, rng.integers(T, 1, 3), 0)
    if big:
        n_names[:big] += 1
    sec_off = np.concatenate([[0], np.cumsum(n_names)]).astype(np.int64)
    NS = int(sec_off[-1])
    owner = np.repeat(np.arange(T, dtype=np.int64), n_names)
    u = rng.uniform(NS)
    own = distro_of[owner] if T else np.zeros(0, np.int64)
    sec = np.where(u < 0.2, own, np.where(u < 0.5, rng.integers(NS, 0, max(D - 1, 0)),
                                          np.where(u < 0.9, D + rng.integers(NS, 0, A - 1), -1))).astype(np.int32)
    if big:
        sec[sec_off[1:big + 1] - 1] = D + A
        sched[:big] = SQ_BASE
        tgmax[:big] = np.where(tgmax[:big] == 1, 0, tgmax[:big])
    dest_off = np.concatenate([[0], np.cumsum([len(x) for x in dests])]).astype(np.int64)
    dest_idx = np.array([e for x in dests for e in x], np.int32)
    # dependencies: a row's in-table edges (the rows' own states), then a few outside the table or missing
    E = tasks.n_edges
    n_ext = np.where(rng.uniform(T) < 0.05, 1, 0)
    per = (np.diff(tasks.dep_off) if E else np.zeros(T, np.int64)) + n_ext
    doff = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
    kind = np.full(int(doff[-1]), L.EVG_DEP_EXTERNAL, np.uint8)
    ref = np.zeros(int(doff[-1]), np.int32)
    X = 16
    if E:
        own_pos = doff[np.repeat(np.arange(T), np.diff(tasks.dep_off))] + (np.arange(E) - np.repeat(tasks.dep_off[:-1], np.diff(tasks.dep_off)))
        kind[own_pos] = L.EVG_DEP_IN_QUEUE
        ref[own_pos] = tasks.dep_idx
    ext_pos = doff[1:][n_ext > 0] - 1
    ref[ext_pos] = rng.integers(ext_pos.shape[0], 0, X - 1)
    kind[ext_pos] = np.where(rng.uniform(ext_pos.shape[0]) < 0.3, L.EVG_DEP_MISSING, L.EVG_DEP_EXTERNAL)
    us = rng.uniform(T)
    state = np.where(us < 0.85, 0, np.where(us < 0.93, 1, 2)).astype(np.uint8)
    state |= np.where(rng.uniform(T) < 0.03, L.EVG_TS_BLOCKED, 0).astype(np.uint8)
    want = np.where(rng.uniform(int(doff[-1])) < 0.9, L.EVG_WANT_SUCCESS, L.EVG_WANT_ANY).astype(np.uint8)
    pre = (np.where(rng.uniform(T) < 0.03, L.EVG_TP_OVERRIDE, 0) | np.where(rng.uniform(T) < 0.05, L.EVG_TP_MET_TIME, 0)).astype(np.uint8)
    deps = DepsTable(doff, kind, ref, want, state, pre, np.where(rng.uniform(X) < 0.8, 0, 1).astype(np.uint8))
    fin = np.where(rng.uniform(int(doff[-1])) < 0.7, w.now - rng.integers(int(doff[-1]), 0, 3 * M.HOUR), M.ZERO_TIME).astype(np.int64)
    at = AliasTable(tasks, gmax, int(vbase[-1]), sched, tgmax, primary, sec_off, sec, dest_off, dest_idx, deps, fin).normalize()
    return at, dt.cfg.copy()


def power_law_sizes(rng: Rng, D: int, alpha: float = 1.2, lo: int = 1, hi: int = 1_000_000) -> np.ndarray:
    u = np.maximum(rng.uniform(D), 1e-12)
    return np.floor(lo * u ** (-1.0 / alpha)).clip(lo, min(hi, L.MAX_TASKS_PER_DISTRO)).astype(np.int64)


def config(k: int, scale: float = 1.0, *, each: bool = False) -> Workload:
    """BASELINE.json configs[k-1].  `scale` shrinks the distro count (tests);
    `each` selects the per-distro reading of "N distros x M tasks" for C3/C4."""
    seed = SEED_BASE + k
    if k == 1:
        return make(np.array([1000]), seed, name="C1: 1 distro x 1000 tasks", n_hosts=20)
    if k == 2:
        D = max(1, int(round(1000 * scale)))
        return make(np.full(D, 10_000), seed, name=f"C2: {D} distros x 10k tasks each, uniform expected durations", n_hosts=5 * D)
    if k == 3:
        D = max(1, int(round(10_000 * scale)))
        per = 100_000 if each else 10
        return make(np.full(D, per), seed, name=f"C3: {D} distros x {per} tasks, Zipf priorities, 5% unmet deps",
                    zipf_priority=True, unmet_dep_frac=0.05, met_dep_frac=0.02, includes_dependencies=True, n_hosts=2 * D)
    if k == 4:
        D = max(1, int(round(10_000 * scale)))
        per = 1_000_000 if each else 100
        return make(np.full(D, per), seed, name=f"C4: {D} distros x {per} tasks, 50k-host pool",
                    zipf_priority=True, n_hosts=int(round(50_000 * scale)))
    if k == 5:
        D = max(1, int(round(100_000 * scale)))
        sizes = power_law_sizes(Rng(seed ^ 0x5A5A), D)
        return make(sizes, seed, name=f"C5: {D} distros, power-law queue sizes, mixed providers", zipf_priority=True,
                    unmet_dep_frac=0.03, met_dep_frac=0.01, group_versions_frac=0.2, includes_dependencies=True,
                    n_hosts=D // 2, providers=(0.6, 0.2, 0.2))
    raise ValueError(k)


@dataclass
class DurationWorkload:
    """The duration cache of tick w (make_duration_cache): the finished-task history, pair-major, and the cache
    fields of every task row and every host row."""
    history: "DurationHistory"
    tasks: "DurationCache"
    hosts: Optional["DurationCache"]


DURATION_SALT = 0x5DEECE66D


def make_duration_cache(w: Workload, seed: int, *, n_rows: int = 100_000, n_keys: int = 1000, zipf_s: float = 1.1,
                        pair_frac: float = 0.05, none_frac: float = 0.05) -> DurationWorkload:
    """History rows with Zipf-skewed keys over n_keys (project, build variant, display name) keys, numbered pair-major
    over about n_keys / 4 pairs of uneven size, and cache columns for every task and host of w that reach every EVG_DS_*
    outcome: fresh and stale predictions (zero, past and future CollectedAt, unset and explicit TTL), backfill rows, keys
    with and without matched rows, EVG_DK_NONE and EVG_DK_PAIR codes.  A key's TimeTaken values lie within 2^20 ns of
    the key's own base (1 min .. 1 h) so exact integer restatements of its statistics stay within int64."""
    from .soa import DurationCache, DurationHistory, DurationRows
    rng = Rng(seed ^ DURATION_SALT)
    now = w.now
    K, R = int(n_keys), int(n_rows)
    P = max(1, K // 4)
    cuts = np.sort(rng.integers(P - 1, 0, K)) if P > 1 else np.zeros(0, np.int64)
    pair_key_off = np.concatenate([[0], cuts, [K]]).astype(np.int64)
    ranks = np.arange(1, K + 1, dtype=np.float64) ** (-zipf_s)
    cdf = np.cumsum(ranks) / ranks.sum()
    perm = np.argsort(rng.u64(K))  # hot keys spread over the pairs
    key = perm[np.minimum(np.searchsorted(cdf, rng.uniform(R)), K - 1)].astype(np.int32)
    base = rng.integers(K, M.MINUTE, 60 * M.MINUTE)
    taken = base[key] + rng.integers(R, 0, (1 << 20) - 1)
    # a quarter of the keys have no row inside the window; other rows fall outside it now and then
    dead = rng.uniform(K) < 0.25
    finish = now - rng.integers(R, 0, 6 * 24 * 60 * M.MINUTE)
    out = (rng.uniform(R) < 0.05) | dead[key]
    finish = np.where(out, now - 8 * 24 * 60 * M.MINUTE, finish)
    flags = np.full(R, L.EVG_DR_COMPLETED, np.uint8)
    flags[rng.uniform(R) < 0.03] = 0
    flags[rng.uniform(R) < 0.03] |= L.EVG_DR_TIMED_OUT
    rows = DurationRows(key, taken.astype(np.int64), (finish - taken).astype(np.int64), finish.astype(np.int64), flags, K,
                        now - 7 * 24 * 60 * M.MINUTE, now)
    hist = DurationHistory(rows, pair_key_off, [], {}, {})

    def cache(n: int) -> DurationCache:
        u = rng.uniform(n)
        code = perm[np.minimum(np.searchsorted(cdf, rng.uniform(n)), K - 1)].astype(np.int32)
        code = np.where(u < none_frac, L.EVG_DK_NONE, code)
        code = np.where((u >= none_frac) & (u < none_frac + pair_frac), -2 - rng.integers(n, 0, P - 1), code).astype(np.int32)
        value = np.where(rng.uniform(n) < 0.3, 0, rng.integers(n, 1, 120 * M.MINUTE))
        std = np.where(rng.uniform(n) < 0.5, 0, rng.integers(n, 1, 10 * M.MINUTE))
        ttl = np.where(rng.uniform(n) < 0.5, 0, rng.integers(n, M.MINUTE, 600 * M.MINUTE))
        v = rng.uniform(n)
        coll = np.where(v < 0.2, M.ZERO_TIME, now - rng.integers(n, 0, 720 * M.MINUTE))
        coll = np.where(v > 0.9, now + rng.integers(n, 1, 60 * M.MINUTE), coll)
        exp = np.where(rng.uniform(n) < 0.2, rng.integers(n, 1, 120 * M.MINUTE), 0)
        exp_std = rng.integers(n, 0, 5 * M.MINUTE)
        return DurationCache(value, std, ttl, coll, exp, exp_std, code).normalize()

    return DurationWorkload(hist, cache(w.tasks.n_tasks), cache(w.hosts.n_hosts) if w.hosts is not None else None)


@dataclass
class IdleHostWorkload:
    """Inputs of the drawdown and idle-host jobs over one set of distros (make_idle_hosts)."""
    now: int
    groups: list            # [[Host]] per distro, in the query's order
    distros: list           # [Distro | None]: None = missing from the distro collection
    existing: np.ndarray    # CountHostsCanOrWillRunTasksInDistro
    drawdown: list          # [DrawdownInfo | None]
    queue_lengths: np.ndarray
    running_counts: np.ndarray
    sched_idle_seconds: int


def make_idle_hosts(sizes, seed: int, *, now: int = NOW_NS) -> IdleHostWorkload:
    """Idle hosts for the C4/C5 shapes: sizes[d] idle hosts in distro d.  The times sit at, and 1 ns around, every
    threshold the two jobs compare against (5 s, 4, 5, 8 and 10 min, the distro's idle time), and include Go's zero
    time, the Unix epoch and the int64 extremes; the flags and per-distro settings cover every branch, and the
    drawdown caps give targets <= 0, below and above the eligible count.  A generator of its own (seeded `seed` with
    its own salt): the streams of every other generator here are untouched."""
    sizes = np.asarray(sizes, dtype=np.int64)
    D, H = len(sizes), int(sizes.sum())
    rng = Rng(seed ^ 0x1D1E0057)
    pivots = np.array([0, 5 * M.SECOND, 90 * M.SECOND, 4 * M.MINUTE, 5 * M.MINUTE, 8 * M.MINUTE, 10 * M.MINUTE, 20 * M.MINUTE,
                       M.HOUR], dtype=np.int64)

    def times(n):
        k = rng.integers(n, 0, 99)
        near = now - pivots[rng.integers(n, 0, len(pivots) - 1)] + rng.integers(n, -1, 1)
        wide = now - rng.integers(n, -M.HOUR, 48 * M.HOUR)
        out = np.where(k < 55, near, wide)
        out = np.where(k >= 92, M.ZERO_TIME, out)
        out = np.where(k == 91, 0, out)
        out = np.where(k == 90, -(2 ** 63) + 1, out)
        return np.where(k == 89, 2 ** 63 - 1, out)

    cols = {f: times(H) for f in ("creation_time", "start_time", "provision_time", "agent_start_time", "last_communication_time",
                                  "last_task_completed_time")}
    cols["task_group_teardown_start_time"] = np.where(rng.uniform(H) < 0.7, M.ZERO_TIME, times(H))
    idle_choice = np.array([0, 5 * M.SECOND, 90 * M.SECOND, 4 * M.MINUTE, 10 * M.MINUTE, 2 ** 62], dtype=np.int64)
    cols["acceptable_host_idle_time"] = idle_choice[rng.integers(H, 0, len(idle_choice) - 1)]
    u = [rng.uniform(H) for _ in range(12)]
    methods = np.array(["", M.BOOTSTRAP_METHOD_LEGACY_SSH, M.BOOTSTRAP_METHOD_USER_DATA, "ssh"])[rng.integers(H, 0, 3)]
    single = np.where(u[9] < 0.1, 2, np.where(u[8] < 0.5, 1, 0))  # 2: the lookup fails
    hosts = []
    for i in range(H):
        hosts.append(M.Host(
            id=f"ih{i}", status=M.HOST_RUNNING if u[0][i] < 0.8 else "provisioning",
            running_task_group="g" if u[1][i] < 0.2 else "", last_task="t" if u[2][i] < 0.6 else "",
            last_group="g" if u[3][i] < 0.25 else "", needs_new_agent=bool(u[4][i] < 0.05),
            needs_new_agent_monitor=bool(u[5][i] < 0.05), ami="old" if u[6][i] < 0.1 else "",
            bootstrap_method=str(methods[i]), last_task_single_host_task_group=None if single[i] == 2 else bool(single[i]),
            time_til_next_payment=int(5 * M.MINUTE + (1 if u[10][i] < 0.05 else 0)), cloud_manager_error=bool(u[11][i] < 0.03),
            **{f: int(v[i]) for f, v in cols.items()}))
    off = np.concatenate([[0], np.cumsum(sizes)])
    groups = [hosts[off[d]:off[d + 1]] for d in range(D)]
    minimum = rng.integers(D, 0, 40)
    d_idle = idle_choice[rng.integers(D, 0, len(idle_choice) - 1)]
    distros = [None if x < 0.02 else M.Distro(id=f"d{d}", default_ami="old" if y < 0.05 else "",
                                              host_allocator_settings=M.HostAllocatorSettings(minimum_hosts=int(minimum[d]),
                                                                                              acceptable_host_idle_time=int(d_idle[d])))
               for d, (x, y) in enumerate(zip(rng.uniform(D), rng.uniform(D)))]
    running = sizes + rng.integers(D, 0, 50)
    existing = sizes + rng.integers(D, 0, 50)
    # the cap: no job, a target <= 0, or a target anywhere from 1 to past the distro's idle hosts
    kind, target = rng.uniform(D), rng.integers(D, 1, 1 << 20) % (sizes + 2) + 1
    cap = existing - np.where(kind < 0.3, -rng.integers(D, 0, 3), target)
    drawdown = [None if k < 0.1 else M.DrawdownInfo(f"d{d}", int(c)) for d, (k, c) in enumerate(zip(kind, cap))]
    qlen = np.where(rng.uniform(D) < 0.5, 0, rng.integers(D, 1, 100))
    return IdleHostWorkload(now, groups, distros, existing, drawdown, qlen, running, 120)
