"""The on-chip planners' radix sorts and the hand-back between them, at every digit width and pass count.

k_plan_cta<THREADS, CAP> (evg_plan_cta.cuh, phase 8) sorts u32 keys Vmax - V in npass = ceil(bits / D) stable LSD passes,
D = 7, 8, 9, 10 bits for THREADS = 64, 128, 256, 512, the bits split as evenly as they go (the first bits % npass passes
take one bit more).  A distro with a value outside u32 -- negative values and a task group's unit value past 2^32
included -- is handed back ("punted") to k_plan_smem, which sorts 8-bit digits in ceil(bits / 8) passes and reloads the
high key word at pass 4.  k_plan_warp ranks distros of at most 32 tasks by counting over all pairs in int64.

Routing (evg_sched.cu, upload_tasks / plan_route), restated in `route` and `punt_instance` and checked on every GPU tick
with the kernel names torch.profiler reports:
  <= 32 tasks                                   k_plan_warp
  <= 384 tasks, <= 60 task groups (resident)    k_plan_cta<64, 384>; the pipelined one-shot call takes <128, 1280>
  <= 1280 / 5120 / 10240 tasks, no GroupVersions, no in-queue edge, task groups within the instance's kGroupCap
                                                k_plan_cta<128, 1280> / <256, 5120> / <512, 10240>
  punts (resident)    k_plan_smem<128, 8> when the tick's largest k_plan_cta distro has <= 1024 tasks, <256, 16> up to
                      4096, else <1024, 12>; the pipelined call always takes <1024, 12>
  10241 .. 12288      k_plan_smem<1024, 12> (EVG_SPARSE_CLASS=0 keeps a sparse class off the general path)

Distros hold lone patch tasks (test_gpu_general_sort's crafting) unless a case says otherwise, so the expected queue is
lexsort((index, -v)) and TotalValue per rank v[order]; ticks with task groups are checked against the oracle.
"""
import copy
import re

import numpy as np
import pytest

import parity
from evergreen_b200 import soa, synth
from test_entry_guard import launched_kernels
from test_gpu_general_sort import (RANK_MIN, check_sorted, craft, craft_checked, lone_tick, lone_value, place,
                                   set_values, tick_values, width)

# ---------------------------------------------------------------- the instances, restated from evg_sched.cu / evg_plan_cta.cuh
CTA = ((64, 384), (128, 1280), (256, 5120), (512, 10240))       # k_plan_cta<THREADS, CAP>
CLASS_MIN = {(64, 384): 33, (128, 1280): 385, (256, 5120): 1281, (512, 10240): 5121}  # smallest distro of each
SMEM_A, SMEM_B, SMEM_C = (128, 8), (256, 16), (1024, 12)          # k_plan_smem<THREADS, ITEMS>: 1024, 4096, 12288 tasks
GENERAL = {"k_ginit", "k_gmark", "k_gtask", "k_glink", "k_galloc", "k_gfill", "k_gunit", "k_grank", "k_gbest", "k_gsched",
           "k_gsum", "k_gscan", "k_gplace", "k_gplace_unit", "k_ghist", "k_gdscan", "k_gscatter", "k_gemit",
           "k_finalize_info"}
U32 = 1 << 32
CTA_WIDTHS = tuple(range(33))


def digit_bits(threads):
    """CtaDigit<THREADS>::kBits: 2^bits == 2 * THREADS."""
    return (2 * threads).bit_length() - 1


def pass_widths(bits, threads):
    """The digit width of every k_plan_cta pass (wbase, plus one for the first wrem passes)."""
    k = digit_bits(threads)
    npass = -(-bits // k)
    return [bits // npass + (j < bits % npass) for j in range(npass)] if npass else []


def group_cap(threads, cap):
    """PlanCta::kGroupCap: task groups a distro may hold (84 bytes each in the idx + counter / TMA stage region)."""
    warps = threads // 32
    cnt = warps * (1 << (digit_bits(threads) - 1)) * 4
    return min(65535, max(2 * cap + cnt, 80 * threads) // 84)


def stretch(threads, cap):
    """Work-list entries of one warp (kListCap / warps); task i of a distro starting at residue off0 lands in warp
    ((i + off0) mod THREADS) // 32."""
    return cap // 4 // (threads // 32)


def route(n, groups, *, pipelined=False):
    """The kernel a lone / task-group distro (no GroupVersions, no in-queue edge) of n tasks is planned by."""
    if n <= 32:
        return "warp"
    for threads, cap in CTA:
        if n <= cap and groups <= group_cap(threads, cap):
            if (threads, cap) == (64, 384) and pipelined:
                return ("cta", (128, 1280))
            return ("cta", (threads, cap))
    return ("smem", SMEM_C) if n <= 12288 else "general"  # the 1025+ classes without task groups, EVG_SPARSE_CLASS=0


def punt_instance(max_cta_tasks, *, pipelined=False):
    if pipelined or max_cta_tasks > 4096:
        return SMEM_C
    return SMEM_A if max_cta_tasks <= 1024 else SMEM_B


def instances(names, kernel):
    """{template arguments} of every launch of `kernel` (torch.profiler's demangled 'k_plan_cta<128, 1280, 8>(...)')."""
    out = set()
    for n in names:
        m = re.match(kernel + r"<([^>]*)>", n)
        if m:
            out.add(tuple(int(x) for x in m.group(1).split(",")))
    return out


def expected_kernels(w, *, pipelined=False, breakdown=False):
    """(k_plan_cta instances, k_plan_smem instances, k_plan_warp launched) the routing sends tick w to."""
    n = np.diff(w.distros.task_off)
    g = np.diff(w.distros.group_off)
    routes = [route(int(a), int(b), pipelined=pipelined) for a, b in zip(n, g)]
    assert "general" not in routes
    cta = {r[1] for r in routes if r != "warp" and r[0] == "cta"}
    smem = {r[1] for r in routes if r != "warp" and r[0] == "smem"}
    warp = "warp" in routes
    if breakdown:  # every k_plan_cta distro through k_plan_smem's largest class, the tiny ones through its smallest
        smem |= {SMEM_C} if cta else set()
        smem |= {SMEM_A} if warp else set()
        return set(), smem, False
    if cta:
        smem.add(punt_instance(max(int(a) for a, r in zip(n, routes) if r != "warp" and r[0] == "cta"), pipelined=pipelined))
    return cta, smem, warp


def check_kernels(names, w, **kw):
    cta, smem, warp = expected_kernels(w, **kw)
    assert {k[:2] for k in instances(names, "k_plan_cta")} == cta, (cta, sorted(set(names)))
    assert {k[:2] for k in instances(names, "k_plan_smem")} == smem, (smem, sorted(set(names)))
    assert ("k_plan_warp" in {re.sub(r"[<(].*", "", n) for n in names}) == warp, sorted(set(names))
    assert not GENERAL & {re.sub(r"[<(].*", "", n) for n in names}, sorted(set(names))


def profiled(engine, fn, uncounted):
    """(fn's result, the kernels it launched).  torch.profiler can miss the first kernels of a window that opens straight
    onto them (evg_run_resident launches at once), so a torch kernel opens it; the context's launch count (every kernel
    of the call but the `uncounted` ones of its upload) tells whether the list is whole, and the call, which computes the
    same again, is repeated until it is."""
    import torch

    def call():
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        out.append(fn())

    for _ in range(3):
        out = []
        names = launched_kernels(call)
        if len(names) == engine.last_launch_count() + uncounted:
            return out[0], names
    raise AssertionError(f"the profiler saw {len(names)} kernels, the context counted {engine.last_launch_count()}: {names}")


def plan(engine, w, **kw):
    po, names = profiled(engine, lambda: engine.plan_batch(w.tasks, w.distros, w.now, **kw), 1)  # the upload's k_validate
    check_kernels(names, w, breakdown=kw.get("breakdown", False))
    return po


# ---------------------------------------------------------------- value crafting on top of test_gpu_general_sort's
def from_keys(keys):
    """(priority, rank) of lone tasks whose keys Vmax - V are `keys` (key 0 must be present: it is Vmax)."""
    keys = np.asarray(keys, np.int64)
    assert keys.min() == 0
    return np.zeros(keys.shape[0], np.int64), RANK_MIN + int(keys.max()) - keys


def keys_of(v):
    v = np.asarray(v, np.int64)
    return int(v.max()) - v


def pass_digits(v, threads, j):
    """Pass j's k_plan_cta digit of every key."""
    w = pass_widths(width(v), threads)
    return (keys_of(v) >> sum(w[:j])) & ((1 << w[j]) - 1)


def shape_values(n, b, threads, shape, rng):
    """(priority, rank) of n lone tasks of width b with a pass-0 digit shape for `threads`' digit split:
      all     every pass-0 digit present;
      zero    every key on pass-0 digit 0;
      odd     every key but Vmax's on one odd pass-0 digit (the high half of a packed counter pair);
      top     every key but Vmax's on the top pass-0 digit 2^w - 1;
      ties2 / ties3  two or three values dealt at random: every warp segment holds all of them."""
    w0 = pass_widths(b, threads)[0]
    # the largest key above the pass-0 digit: bit b - 1 set, and at width 32 low enough that Vmax = RANK_MIN + 1 + Kmax
    # still fits u32 (the distro must stay on k_plan_cta)
    top_hi = (1 << b) - (1 << w0) if b < 32 else U32 - (1 << 11)
    hi = rng.integers(0, (top_hi >> w0) + 1, n) << w0
    hi[1] = top_hi
    if shape == "all":
        keys = np.arange(n) % (1 << w0) + hi
    elif shape == "zero":
        keys = hi
    elif shape == "odd":
        keys = hi | ((1 << (w0 - 1)) + 1)
    elif shape == "top":
        keys = hi | ((1 << w0) - 1)
    else:
        levels = np.array([0, (1 << b) - 1 if b < 32 else top_hi, (1 << (b - 1)) + 5][:int(shape[4:])])
        keys = levels[rng.integers(0, levels.shape[0], n)]
        keys[:levels.shape[0]] = levels
    keys[0] = 0  # Vmax; keys[1] >= top_hi sets the width
    p, r = from_keys(keys)
    perm = rng.permutation(n)
    return p[perm], r[perm]


def join(a, b):
    """Tick a's distros, then tick b's (no in-queue edges)."""
    assert a.tasks.n_edges == 0 and b.tasks.n_edges == 0 and a.now == b.now
    ta, tb, da, db = a.tasks, b.tasks, a.distros, b.distros
    tasks = soa.TaskSoA(**{name: np.concatenate([getattr(ta, name), getattr(tb, name)]) for name, _ in ta.COLUMNS}).normalize()
    distros = soa.DistroTable(np.concatenate([da.task_off, db.task_off[1:] + da.task_off[-1]]),
                              np.concatenate([da.group_off, db.group_off[1:] + da.group_off[-1]]),
                              np.concatenate([da.cfg, db.cfg]),
                              np.concatenate([da.group_max_hosts, db.group_max_hosts])).normalize()
    return synth.Workload(f"{a.name} + {b.name}", a.now, tasks, distros, None)


def spans(w, d):
    return int(w.distros.task_off[d]), int(w.distros.task_off[d + 1])


# ---------------------------------------------------------------- the ticks
def width_specs(inst, seed, offset=0, widths=CTA_WIDTHS):
    """Case 1: every width at the class's smallest size, CAP - 1 and CAP, start residues cycling 0..3."""
    rng = np.random.default_rng(seed)
    sizes = (CLASS_MIN[inst], inst[1] - 1, inst[1])
    return [(n, k % 4, craft_checked(n, b, rng, offset=offset)) for k, (b, n) in enumerate((b, n) for b in widths for n in sizes)]


def width_tick(inst):
    return place(width_specs(inst, 400 + inst[0]), 400 + inst[0])


GROUP_BASE = 2520  # lcm(2 .. 9): a task group of L <= 8 members (synth.make's largest) can score any V with L + 1 | V + 1


def group_width_tick(inst):
    """Case 7: the case-1 widths again, with task groups only (no edges, no GroupVersions), at the same widths.  Under
    PLANNER a task group of L patch members of priority 0, all at rank r, scores (1 + L) * r + L (priority 1 + L, the
    unit's rank r: planner.go:209-300), so V + 1 = (1 + L) * (r + 1).  Every distro's lone values start at
    Vmin = GROUP_BASE - 1 (two lone tasks hold Vmin and Vmax), and each group takes the largest such value at or below
    Vmin + t, t drawn over the distro's range: inside the lone range, so the distro keeps its width (width 0: every
    group on Vmin).  One group per distro has its order reversed, so its smallest index carries the largest
    TaskGroupOrder and the pre-arrangement is no identity."""
    seed = 500 + inst[0]
    specs = width_specs(inst, seed, offset=GROUP_BASE - 2 - RANK_MIN)
    w, ids = place(specs, seed, units=True, edges=False)
    t = w.tasks
    rng = np.random.default_rng(seed)
    for (_, _, (_, r0)), d in zip(specs, ids):
        a, b = spans(w, d)
        top = int(r0.max() - r0.min())
        gid = t.group_id[a:b]
        lone = a + np.nonzero(gid < 0)[0][:2]
        set_values(t, lone, np.zeros(2, np.int64), np.array([GROUP_BASE - 2, GROUP_BASE - 2 + top]), keep_deps_met=True)
        reversed_one = False
        for g in np.unique(gid[gid >= 0]):
            m = a + np.nonzero(gid == g)[0]
            n = m.shape[0]
            r = (GROUP_BASE + int(rng.integers(0, top + 1))) // (1 + n) - 1
            set_values(t, m, np.zeros(n, np.int64), np.full(n, r, np.int64), keep_deps_met=True)
            if n >= 2 and not reversed_one:
                t.task_group_order[m] = t.task_group_order[m][::-1]
                reversed_one = True
    t.normalize()
    return w, ids


SHAPES = ("all", "zero", "odd", "top", "ties2", "ties3")


TOP_WIDTH = {7: 28, 8: 32, 9: 27, 10: 30}  # full k-bit passes: pass 0's top digit is 2^k - 1, the last scan word's high half


def shape_width(inst, shape):
    k = digit_bits(inst[0])
    return {"all": 2 * k, "zero": 2 * k + 1, "odd": k + 1, "top": TOP_WIDTH[k], "ties2": k, "ties3": 32}[shape]


def shape_tick():
    """Case 2: every digit shape on every instance, at CAP (every warp FULL); the ties also at CAP - 1."""
    rng = np.random.default_rng(600)
    specs, rows = [], []
    for inst in CTA:
        for s in SHAPES:
            for n in (inst[1], inst[1] - 1) if s.startswith("ties") else (inst[1],):
                rows.append((inst, s))
                specs.append((n, len(specs) % 4, shape_values(n, shape_width(inst, s), inst[0], s, rng)))
    w, ids = place(specs, 600)
    return w, ids, rows


BOUNDARY = ("u32max", "u32over", "wrapped")


def boundary_tick():
    """Case 3: on every instance, a distro whose largest value is 2^32 - 1 (stays on k_plan_cta), one whose largest is
    2^32 (handed back), one holding a wrapped negative value (handed back), then a task-group distro whose largest unit
    value alone passes 2^32 while every lone task's value fits u32 (the phase-3 punt)."""
    rng = np.random.default_rng(700)
    specs, rows = [], []
    for inst in CTA:
        n = (CLASS_MIN[inst] + inst[1]) // 2
        for kind in BOUNDARY:
            p = np.zeros(n, np.int64)
            r = rng.integers(RANK_MIN, U32 - 2, n)
            if kind == "u32max":
                r[0] = U32 - 2
            elif kind == "u32over":
                r[0] = U32 - 1
            else:  # (1 + 2^31 - 1) * 2^32 + 1 = 2^63 + 1: int64 wraps
                p[0], r[0] = 2 ** 31 - 1, U32
            perm = rng.permutation(n)
            specs.append((n, len(specs) % 4, (p[perm], r[perm])))
            rows.append((inst, kind))
    lone, ids = place(specs, 700)
    gspecs = [(inst[1] - 7, k % 4, craft(inst[1] - 7, 20, rng)) for k, inst in enumerate(CTA)]
    grp, gids = place(gspecs, 701, units=True, edges=False)
    t = grp.tasks
    rows_g = np.nonzero(t.group_id >= 0)[0]
    set_values(t, rows_g, np.zeros(rows_g.shape[0], np.int64), RANK_MIN + rng.integers(0, 1 << 16, rows_g.shape[0]), keep_deps_met=True)
    for d in gids:  # one group per distro: members of rank 2^31 -- each alone fits, their unit does not
        a, b = spans(grp, d)
        gid = t.group_id[a:b]
        g = np.bincount(gid[gid >= 0]).argmax()
        m = a + np.nonzero(gid == g)[0]
        set_values(t, m, np.zeros(m.shape[0], np.int64), np.full(m.shape[0], 2 ** 31, np.int64), keep_deps_met=True)
    w = join(lone, grp)
    return w, ids, [lone.distros.n_distros + d for d in gids], rows


def punt_tick(smem):
    """Case 4: widths 0..32 with every value past 2^32 (ranks offset by 2^33: one key word, a punt) and widths 33..64
    (two key words), on k_plan_cta distros whose largest picks k_plan_smem instance `smem`."""
    top = {SMEM_A: 1024, SMEM_B: 4096, SMEM_C: 10240}[smem]
    lo = {SMEM_A: 33, SMEM_B: 1025, SMEM_C: 4097}[smem]
    seed = 800 + smem[0]
    rng = np.random.default_rng(seed)
    specs = []
    for b in range(65):
        n = top if b == 0 else int(rng.integers(lo, top + 1))
        specs.append((n, b % 4, craft_checked(n, b, rng, offset=1 << 33 if b <= 32 else 0)))
    return place(specs, seed)


SMEM_SIZES = 65


def smem_tick():
    """Case 5: lone distros of 10241..12288 tasks (k_plan_smem<1024, 12> without a punt) at widths 0..64."""
    rng = np.random.default_rng(900)
    specs = []
    for b in range(SMEM_SIZES):
        n = 12288 if b % 8 == 0 else 10241 if b % 8 == 1 else int(rng.integers(10241, 12289))
        specs.append((n, b % 4, craft_checked(n, b, rng)))
    return place(specs, 900)


WARP_WIDTHS = (0, 1, 31, 32, 33, 63, 64)


def warp_tick():
    """Case 6: distros of 1..32 tasks at every WARP_WIDTHS width the size allows (dense, then three values with ties);
    widths 63 and 64 hold wrapped values."""
    rng = np.random.default_rng(1000)
    parts = []
    for n in range(1, 33):
        for b in WARP_WIDTHS:
            if (n == 1 and b) or (n < 3 and b > 34):
                continue
            parts.append(craft_checked(n, b, rng))
            if n >= 4 and b:
                parts.append(craft_checked(n, b, rng, "levels3"))
    return lone_tick(parts, 1000)


# ---------------------------------------------------------------- CPU: routing and crafting against the oracle
def oracle_values(w, distros=None):
    """TotalValue per rank from the oracle's planner, per distro."""
    from oracle import oracle as O
    ref = O.SoAJob(w.tasks, w.distros, None, distros).run(w.now, 8)
    sel = list(range(w.distros.n_distros)) if distros is None else list(distros)
    return {d: ref["total_value"][int(ref["task_off"][j]):int(ref["task_off"][j + 1])] for j, d in enumerate(sel)}


def segments(tn, threads):
    """k_plan_cta's warp segments [seg0, seg1) of a tn-task distro (empty ones included)."""
    nw = threads // 32
    seg = ((tn + nw - 1) // nw + 31) & ~31
    return [(w * seg, min(w * seg + seg, tn)) for w in range(nw)]


def test_routing_and_crafting_match_the_oracle():
    """The routing each tick is built for, and every crafted distro's width and digit shape for its instance's digit
    width and split, from the values the oracle's planner ranks."""
    assert [digit_bits(t) for t, _ in CTA] == [7, 8, 9, 10]
    assert [group_cap(*i) for i in CTA] == [60, 121, 243, 633]
    assert [stretch(*i) for i in CTA] == [48, 80, 160, 160]
    assert pass_widths(32, 64) == [7, 7, 6, 6, 6] and pass_widths(21, 512) == [7, 7, 7] and pass_widths(17, 128) == [6, 6, 5]
    for inst in CTA:  # every pass count and every uneven split of each digit width
        k = digit_bits(inst[0])
        assert {len(pass_widths(b, inst[0])) for b in CTA_WIDTHS} == set(range(-(-32 // k) + 1))
        assert route(CLASS_MIN[inst], 0) == ("cta", inst) and route(inst[1], 0) == ("cta", inst)
        assert route(CLASS_MIN[inst] - 1, 0) != ("cta", inst) and route(inst[1] + 1, 0) != ("cta", inst)
    assert route(384, 61) == ("cta", (128, 1280)) and route(300, 0, pipelined=True) == ("cta", (128, 1280))
    assert [punt_instance(n) for n in (384, 1024, 1025, 4096, 4097, 10240)] == [SMEM_A, SMEM_A, SMEM_B, SMEM_B, SMEM_C, SMEM_C]

    for inst in CTA:  # case 1: every width at its three sizes and four residues, on its own instance
        w, ids = width_tick(inst)
        assert expected_kernels(w) == ({inst}, {punt_instance(inst[1])}, True)
        v = tick_values(w)
        got = [(width(v[slice(*spans(w, d))]), spans(w, d)[1] - spans(w, d)[0], spans(w, d)[0] % 4) for d in ids]
        sizes = (CLASS_MIN[inst], inst[1] - 1, inst[1])
        assert got == [(b, n, k % 4) for k, (b, n) in enumerate((b, n) for b in CTA_WIDTHS for n in sizes)]
        assert max(v) < U32 and min(v) >= 0
        ov = oracle_values(w, ids)
        assert all(np.array_equal(ov[d], np.sort(v[slice(*spans(w, d))])[::-1]) for d in ids)
        # case 7: the same widths with task groups, inside every limit that keeps them on k_plan_cta
        wg, gids = group_width_tick(inst)
        assert expected_kernels(wg) == ({inst}, {punt_instance(inst[1])}, True)
        t = wg.tasks
        reversed_anchor, has_groups = 0, 0
        for d in gids:
            a, b = spans(wg, d)
            gid, tgo = t.group_id[a:b], t.task_group_order[a:b]
            ng = int(wg.distros.group_off[d + 1] - wg.distros.group_off[d])
            assert ng <= group_cap(*inst)
            has_groups += ng > 0
            warp = ((np.arange(b - a) + a % 4) % inst[0]) // 32
            assert np.bincount(warp[gid >= 0], minlength=inst[0] // 32).max() <= stretch(*inst)
            for g in range(ng):
                m = np.nonzero(gid == g)[0]
                assert len(set(tgo[m].tolist())) == m.shape[0] and tgo[m].max() < 64
                reversed_anchor += m.shape[0] > 1 and tgo[m[0]] == tgo[m].max()
        assert has_groups >= 0.9 * len(gids) and reversed_anchor >= 0.75 * len(gids), (has_groups, reversed_anchor)
        ov = oracle_values(wg, gids)
        assert all(ov[d].max() < U32 and ov[d].min() >= 0 for d in gids)
        # the case-1 widths with task groups present: every width (bits 0: phase 8 skipped, the pre-arrangement is the
        # queue; one and two passes over a pre-arrangement that is no identity) holds distros with groups
        assert [width(ov[d]) for d in gids] == [b for b in CTA_WIDTHS for _ in range(3)]
        grouped = {width(ov[d]) for d in gids if wg.distros.group_off[d + 1] > wg.distros.group_off[d]}
        assert grouped == set(CTA_WIDTHS), sorted(set(CTA_WIDTHS) - grouped)

    w, ids, rows = shape_tick()  # case 2
    assert expected_kernels(w) == (set(CTA), {SMEM_C}, True)
    v = tick_values(w)
    ov = oracle_values(w, ids)
    for d, (inst, s) in zip(ids, rows):
        x = v[slice(*spans(w, d))]
        assert np.array_equal(ov[d], np.sort(x)[::-1]) and width(x) == shape_width(inst, s), (inst, s)
        assert 0 <= x.min() and x.max() < U32  # no punt
        assert route(x.shape[0], 0) == ("cta", inst)
        dg = pass_digits(x, inst[0], 0)
        w0 = pass_widths(width(x), inst[0])[0]
        assert len(pass_widths(width(x), inst[0])) >= 2 or s.startswith("ties")
        if s == "all":
            assert np.unique(dg).shape[0] == 1 << w0
        elif s == "zero":
            assert np.all(dg == 0)
        elif s in ("odd", "top"):
            want = (1 << (w0 - 1)) + 1 if s == "odd" else (1 << w0) - 1
            assert want % 2 == 1 and np.count_nonzero(dg == want) == x.shape[0] - 1
            if s == "top":  # the instance's own top digit 2^k - 1, alone in its pass but for Vmax's 0
                assert w0 == digit_bits(inst[0]) and set(pass_widths(width(x), inst[0])) == {w0}
        else:
            levels = np.unique(x)
            assert levels.shape[0] == int(s[4:])
            for s0, s1 in segments(x.shape[0], inst[0]):
                assert s1 <= s0 or np.unique(x[s0:s1]).shape[0] == levels.shape[0], (inst, s, s0)

    w, ids, gids, rows = boundary_tick()  # case 3
    assert expected_kernels(w) == (set(CTA), {SMEM_C}, True)
    ov = oracle_values(w)
    v = tick_values(w)
    for d, (inst, kind) in zip(ids, rows):
        x = v[slice(*spans(w, d))]
        assert np.array_equal(ov[d], np.sort(x)[::-1]) and route(x.shape[0], 0) == ("cta", inst)
        assert {"u32max": x.max() == U32 - 1, "u32over": x.max() == U32, "wrapped": x.min() == lone_value(2 ** 31 - 1, U32)[0] == -(2 ** 63) + 1}[kind], kind
        assert np.count_nonzero((x >= U32) | (x < 0)) == (kind != "u32max")  # one value outside u32, or none
    for inst, d in zip(CTA, gids):
        a, b = spans(w, d)
        ng = int(w.distros.group_off[d + 1] - w.distros.group_off[d])
        assert route(b - a, ng) == ("cta", inst)
        lone = w.tasks.group_id[a:b] < 0
        assert v[a:b][lone].max() < U32
        assert ov[d].max() >= U32 and np.count_nonzero(ov[d] >= U32) < b - a  # the unit's members only

    for smem in (SMEM_A, SMEM_B, SMEM_C):  # case 4
        w, ids = punt_tick(smem)
        assert expected_kernels(w)[1] == {smem}
        v = tick_values(w)
        assert [width(v[slice(*spans(w, d))]) for d in ids] == list(range(65))
        assert all(v[slice(*spans(w, d))].max() >= U32 or v[slice(*spans(w, d))].min() < 0 for d in ids)

    w, ids = smem_tick()  # case 5
    assert expected_kernels(w) == (set(), {SMEM_C}, True)
    v = tick_values(w)
    assert [width(v[slice(*spans(w, d))]) for d in ids] == list(range(SMEM_SIZES))

    w = warp_tick()  # case 6
    assert expected_kernels(w) == (set(), set(), True)
    v = tick_values(w)
    ov = oracle_values(w)
    ws = set()
    for d in range(w.distros.n_distros):
        x = v[slice(*spans(w, d))]
        assert np.array_equal(ov[d], np.sort(x)[::-1])
        ws.add((x.shape[0], width(x)))
    assert {b for _, b in ws} == set(WARP_WIDTHS) and {n for n, _ in ws} == set(range(1, 33))
    assert np.any(v < 0)

    w = pipelined_tick()  # case 9
    assert w.n_tasks >= 1 << 21
    assert expected_kernels(w, pipelined=True) == ({(128, 1280)}, {SMEM_C}, False)
    assert expected_kernels(w) == ({(64, 384)}, {SMEM_A}, False)


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("inst", CTA, ids=lambda i: f"{i[0]}x{i[1]}")
def test_cta_every_width_on_every_instance(engine, inst):
    """Widths 0..32 (every pass count, every uneven split) at the class's smallest size, CAP - 1 and CAP, start residues
    0..3, all on one instance."""
    w, ids = width_tick(inst)
    po = plan(engine, w)
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_cta_digit_shapes(engine):
    """Every digit of a pass present, one digit for every key (digit 0, an odd digit in a counter's high half, the top
    digit), and two or three values in every warp segment where only stability keeps their order."""
    w, ids, rows = shape_tick()
    po = plan(engine, w)
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_cta_u32_boundary(engine):
    """Largest value 2^32 - 1 stays on k_plan_cta, 2^32 and a wrapped negative value are handed back, and so is a
    task-group distro whose unit value alone passes 2^32: the values outside u32 can only come from k_plan_smem."""
    w, ids, gids, rows = boundary_tick()
    po = plan(engine, w)
    v = tick_values(w)
    check_sorted(w, po, v, distros=ids)
    for d, (inst, kind) in zip(ids, rows):
        a, b = spans(w, d)
        assert int(po.total_value[a]) == {"u32max": U32 - 1, "u32over": U32, "wrapped": int(v[a:b].max())}[kind]
        if kind == "wrapped":
            assert int(po.total_value[b - 1]) == -(2 ** 63) + 1
    for d in gids:
        a, b = spans(w, d)
        assert int(po.total_value[a]) >= U32
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
@pytest.mark.parametrize("smem", (SMEM_A, SMEM_B, SMEM_C), ids=lambda s: f"{s[0]}x{s[1]}")
def test_punts_at_every_width(engine, smem):
    """Every k_plan_cta distro is handed back: widths 0..32 past 2^32 (one key word), 33..64 (the pass-4 high-word
    reload), on the k_plan_smem instance the tick's largest k_plan_cta distro picks."""
    w, ids = punt_tick(smem)
    po = plan(engine, w)
    v = tick_values(w)
    check_sorted(w, po, v)
    assert all(int(po.total_value[spans(w, d)[0]]) >= U32 or int(po.total_value[spans(w, d)[1] - 1]) < 0 for d in ids)
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_smem_every_width_without_punt(engine, monkeypatch):
    """Lone distros of 10241..12288 tasks on k_plan_smem<1024, 12> at widths 0..64: 0 to 8 passes, one and two key words."""
    monkeypatch.setenv("EVG_SPARSE_CLASS", "0")
    w, ids = smem_tick()
    po = plan(engine, w)
    check_sorted(w, po, tick_values(w))


@pytest.mark.gpu
def test_breakdown_sends_cta_distros_through_smem(engine):
    """A breakdown run of the <128, 1280> case-1 tick plans every k_plan_cta distro with k_plan_smem<1024, 12> (the 1-3
    task fillers with <128, 8>).  Against the oracle."""
    w, ids = width_tick((128, 1280))
    po = plan(engine, w, breakdown=True)
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
def test_warp_widths_and_ties(engine):
    """Distros of 1..32 tasks at widths 0, 1, 31, 32, 33, 63, 64 with wrapped values and ties: k_plan_warp's int64
    all-pairs count."""
    w = warp_tick()
    po = plan(engine, w)
    check_sorted(w, po, tick_values(w))
    parity.check_against_oracle(w, po, None)


@pytest.mark.gpu
@pytest.mark.parametrize("inst", CTA, ids=lambda i: f"{i[0]}x{i[1]}")
def test_cta_every_width_with_task_groups(engine, inst):
    """The case-1 widths with task groups only (they stay on k_plan_cta), one group per distro anchored at its largest
    TaskGroupOrder.  Against the oracle."""
    w, ids = group_width_tick(inst)
    po = plan(engine, w)
    assert int(po.total_value.max()) < U32 and int(po.total_value.min()) >= 0
    parity.check_against_oracle(w, po, None)
    parity.check_properties(w, po)


@pytest.mark.gpu
def test_resident_tick_across_the_u32_boundary(engine):
    """Upload once; evg_update_tasks moves the same k_plan_cta distros through widths 32 -> 33 -> 7 -> 64 -> 0, so each
    goes in and out of the punt list and the high key word k_plan_smem keeps changes between runs.  Each run equals a
    fresh plan_batch on a second context and the reference."""
    from evergreen_b200 import scheduler
    seq = (32, 33, 7, 64, 0)
    sizes = (300, 1000, 3001, 9000)
    rng = np.random.default_rng(1100)
    w = lone_tick([craft_checked(n, seq[0], rng) for n in sizes], 1100)
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
            _, names = profiled(engine, lambda: engine.run(w.now), 0)
            check_kernels(names, w)
            po, _ = copy.deepcopy(engine.download())
            v = tick_values(w)
            assert [width(v[slice(*spans(w, d))]) for d in range(len(sizes))] == [b] * len(sizes)
            assert (int(po.total_value.max()) >= U32 or int(po.total_value.min()) < 0) == (b > 32), step
            check_sorted(w, po, v)
            fo = fresh.plan_batch(t, w.distros, w.now)
            for f in ("order", "total_value", "info"):
                assert np.array_equal(getattr(po, f), getattr(fo, f)), (step, f)
    finally:
        fresh.close()


def pipelined_tick():
    """Case 9: 2^21+ tasks in distros of 33..384 tasks; every 16th distro's values pass 2^32 (a punt)."""
    rng = np.random.default_rng(1200)
    parts, total, k = [], 0, 0
    while total < (1 << 21) + 1000:
        n = int(rng.integers(33, 385))
        b = int(rng.integers(0, 33))
        parts.append(craft_checked(n, b, rng, offset=(1 << 33) if k % 16 == 5 else 0))
        total += n
        k += 1
    return lone_tick(parts, 1200, n_hosts=2000)


@pytest.mark.gpu
def test_pipelined_one_shot_call(engine):
    """plan_and_alloc_batch on a tick of 2^21+ tasks: the <= 384-task distros go to k_plan_cta<128, 1280>, the punts to
    k_plan_smem<1024, 12>, chunk by chunk."""
    w = pipelined_tick()
    (po, _), names = profiled(engine, lambda: engine.plan_and_alloc_batch(w.tasks, w.distros, w.hosts, w.now), 0)
    check_kernels(names, w, pipelined=True)
    v = tick_values(w)
    assert int(po.total_value.max()) >= U32
    check_sorted(w, po, v)
