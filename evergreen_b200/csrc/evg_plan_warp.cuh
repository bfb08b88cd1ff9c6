// evg_plan_warp.cuh -- k_plan_warp: one WARP plans one distro of at most 32 tasks.
//
// Power-law ticks (BASELINE configs[4]: 100k distros, most with a handful of tasks) are
// dominated by per-CTA overhead when every distro gets a block; here lane i holds task i,
// units are lane bitmasks, every loop is bounded by the distro's size (warp-uniform) and
// nothing touches shared memory or a block barrier.
//
//   unit of lane r      r is a unit's representative when it is the lowest lane filed under
//                       that unit's key (planner.go:434-446) -- which is also the unit's anchor
//   membership M_j      bit r set when task j belongs to r's unit: its own key, its version unit
//                       under GroupVersions (planner.go:439), the unit of every in-queue
//                       dependency (planner.go:449-456); bitmask OR == Unit.Add's set semantics
//   order               rank of j = number of tasks with a smaller (TotalValue desc, anchor,
//                       rank-in-unit) key -- a 32-step all-pairs count instead of a sort
//
// Reference: scheduler/planner.go:209-481, scheduler/scheduler.go:56-159.
#pragma once

__device__ __forceinline__ int64_t shfl64(int64_t v, int src) {
  const uint32_t lo = __shfl_sync(0xffffffffu, uint32_t(uint64_t(v)), src);
  const uint32_t hi = __shfl_sync(0xffffffffu, uint32_t(uint64_t(v) >> 32), src);
  return int64_t((uint64_t(hi) << 32) | lo);
}

// 4 blocks of 8 distros per SM: 64 registers (sm_90a: 16 B spill stores, 56 B spill loads) keep more distros in flight
// than 3 (no spill), which was slower on H100 for configs[2] total and configs[4]
constexpr int kWarpOcc = 4;
__global__ void __launch_bounds__(256, kWarpOcc) k_plan_warp(DTasks T, DDistros D, DWork W, const int32_t* __restrict__ list,
                                                   int n_list, int64_t now, int32_t* __restrict__ order,
                                                   int64_t* __restrict__ total_value) {
  if (*W.err) return;
  const int wid = int((int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  const unsigned full = 0xffffffffu;
  if (wid >= n_list) return;  // warp-uniform
  const int d = list[wid];
  const int64_t base = D.task_off[d];
  const int tn = int(D.task_off[d + 1] - base);  // <= 32
  const uint32_t ng = uint32_t(D.group_off[d + 1] - D.group_off[d]);
  const evg_distro_cfg cfg = D.cfg[d];
  const bool gv = cfg.group_versions != 0;
  const bool valid = lane < tn;
  const int64_t t = base + lane;

  int32_t prio = 0, nd = 0, gid = -1, vid = 0, tgo = 0;
  int64_t exp_ns = 0, qb = EVG_TIME_ZERO, wb = EVG_TIME_ZERO;
  uint32_t fl = 0;
  int64_t e0 = 0, e1 = 0;
  if (valid) {
    prio = T.priority[t]; nd = T.numdep[t]; gid = T.gid[t]; vid = T.vid[t]; tgo = T.tgo[t]; fl = T.flags[t];
    exp_ns = T.expected[t]; qb = T.qbasis[t]; wb = T.wbasis[t];
    if (T.n_edges > 0) { e0 = T.dep_off[t]; e1 = T.dep_off[t + 1]; }
  }
  const bool has_edges = __any_sync(full, e1 > e0);
  const bool any = ng > 0 || gv || has_edges;

  // ---- GetDistroQueueInfo (scheduler.go:56-159) ----
  const int64_t threshold = cfg.target_time_ns;
  const bool dm = valid && (fl & EVG_TF_DEPS_MET);
  const bool counted = valid && (!cfg.includes_dependencies || dm);
  const bool over = counted && exp_ns > threshold;
  const bool wait_over = counted && dm && since(now, wb) > threshold;
  const bool mq_dm = dm && (fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE;
  const bool in_tg = valid && gid >= 0;
  {
    const unsigned b_dm = __ballot_sync(full, dm), b_mq = __ballot_sync(full, mq_dm), b_over = __ballot_sync(full, over);
    const unsigned b_wait = __ballot_sync(full, wait_over), b_cnt = __ballot_sync(full, counted);
    const unsigned b_sec = __ballot_sync(full, valid && (fl & EVG_TF_OTHER_DISTRO)), b_tg = __ballot_sync(full, in_tg);
    const int64_t s_exp = warp_sum64(counted ? exp_ns : 0), s_over = warp_sum64(over ? exp_ns : 0);
    const int64_t s_uexp = warp_sum64(counted && !in_tg ? exp_ns : 0), s_uover = warp_sum64(over && !in_tg ? exp_ns : 0);
    if (lane == 0) {
      evg_queue_info q;
      q.length = tn;
      q.length_with_dependencies_met = __popc(b_dm);
      q.count_dep_filled_merge_queue_tasks = __popc(b_mq);
      q.expected_duration = s_exp;
      q.max_duration_threshold = threshold;
      q.count_duration_over_threshold = __popc(b_over);
      q.duration_over_threshold = s_over;
      q.count_wait_over_threshold = __popc(b_wait);
      q.secondary_queue = b_sec != 0;
      q.has_ungrouped = __popc(b_tg) < tn;
      q.ungrouped.count = __popc(b_cnt & ~b_tg);
      q.ungrouped.count_free = 0;
      q.ungrouped.count_required = 0;
      q.ungrouped.max_hosts = 0;
      q.ungrouped.expected_duration = s_uexp;
      q.ungrouped.count_duration_over_threshold = __popc(b_over & ~b_tg);
      q.ungrouped.count_wait_over_threshold = __popc(b_wait & ~b_tg);
      q.ungrouped.count_dep_filled_merge_queue_tasks = __popc(b_mq & ~b_tg);
      q.ungrouped.duration_over_threshold = s_uover;
      W.qinfo[d] = q;
    }
    for (uint32_t g = uint32_t(lane); g < ng; g += 32) {  // rows start from zero (no host-side memset)
      evg_group_info z;
      z.count = 0; z.count_free = 0; z.count_required = 0; z.max_hosts = D.gmax[D.group_off[d] + g];
      z.expected_duration = 0; z.count_duration_over_threshold = 0; z.count_wait_over_threshold = 0;
      z.count_dep_filled_merge_queue_tasks = 0; z.duration_over_threshold = 0;
      W.ginfo[D.group_off[d] + g] = z;
    }
    __syncwarp();
    if (in_tg) {
      evg_group_info* g = W.ginfo + D.group_off[d] + gid;
      atomic_add64(&g->count, counted);
      atomic_add64(&g->expected_duration, counted ? exp_ns : 0);
      atomic_add64(&g->count_duration_over_threshold, over);
      atomic_add64(&g->duration_over_threshold, over ? exp_ns : 0);
      atomic_add64(&g->count_wait_over_threshold, wait_over);
      atomic_add64(&g->count_dep_filled_merge_queue_tasks, mq_dm);
    }
  }

  // ---- units ----
  int64_t best_v = 0;
  uint32_t best_u = uint32_t(lane), rk = 0;
  if (!any) {
    const PlannerFactors pf = clamp_factors(cfg);
    if (now >= 0 && pf.nd_int != 0 && __all_sync(full, !valid || score_fast_domain(now, exp_ns, qb))) {
      const int64_t v = single_task_value_fast(pf, now, prio, exp_ns, qb, nd, fl);
      if (valid) best_v = v;
    } else if (valid) {
      best_v = single_task_value(pf, now, prio, exp_ns, qb, nd, fl);
    }
  } else {
    // key a task is filed under; invalid lanes get keys nobody shares
    const uint32_t s_own = valid ? own_slot_local(gid, vid, uint32_t(lane), ng, gv) : 0xF0000000u + uint32_t(lane);
    const uint32_t s_ver = (valid && gid >= 0 && gv) ? ng + uint32_t(vid) : 0xE0000000u;
    const unsigned own_peers = __match_any_sync(full, s_own);
    const uint32_t rep = uint32_t(__ffs(own_peers) - 1);  // lowest lane with the same key == the unit's anchor
    // rep of every lane, bit-sliced, so a lane can look up rep(dependency) without a divergent shuffle
    unsigned rep_bits[5];
#pragma unroll
    for (int b = 0; b < 5; b++) rep_bits[b] = __ballot_sync(full, (rep >> b) & 1u);
    uint32_t member_of = valid ? (1u << rep) : 0u;
    for (int i = 0; i < tn; i++) {  // version unit of task-group tasks under GroupVersions (planner.go:439)
      const uint32_t si = __shfl_sync(full, s_own, i), ri = __shfl_sync(full, rep, i);
      if (si == s_ver) member_of |= 1u << ri;
    }
    for (int64_t e = e0; e < e1; e++) {  // unit of each in-queue dependency (planner.go:449-456)
      const uint32_t dl = uint32_t(T.dep_idx[e]);
      uint32_t rd = 0;
#pragma unroll
      for (int b = 0; b < 5; b++) rd |= ((rep_bits[b] >> dl) & 1u) << b;
      member_of |= 1u << rd;
    }
    // member set of every representative
    uint32_t members = 0;
    for (int r = 0; r < tn; r++) {
      const unsigned m = __ballot_sync(full, valid && ((member_of >> r) & 1u));
      if (lane == r && rep == uint32_t(lane)) members = m;
    }
    // Unit.info + unitInfo.value per representative (planner.go:209-337)
    UnitAcc a;
    acc_init(a);
    for (int j = 0; j < tn; j++) {
      const int32_t pj = __shfl_sync(full, prio, j), ndj = __shfl_sync(full, nd, j), gj = __shfl_sync(full, gid, j);
      const uint32_t fj = __shfl_sync(full, fl, j);
      const int64_t ej = shfl64(exp_ns, j), qj = shfl64(qb, j);
      if ((members >> j) & 1u) acc_add(a, now, pj, ej, qj, ndj, gj, fj);
    }
    const int64_t unit_v = members ? unit_value(a, cfg, nullptr) : 0;
    // the unit each task is emitted from: best of its memberships (planner.go:467-477)
    bool have = false;
    for (int r = 0; r < tn; r++) {
      const int64_t vr = shfl64(unit_v, r);
      if (valid && ((member_of >> r) & 1u) && (!have || vr > best_v)) { have = true; best_v = vr; best_u = uint32_t(r); }
    }
    // rank inside that unit (TaskList.Less, planner.go:387-405; ties by input index)
    const uint32_t best_members = __shfl_sync(full, members, int(best_u));
    for (int m = 0; m < tn; m++) {
      const int32_t tm = __shfl_sync(full, tgo, m), ndm = __shfl_sync(full, nd, m), pm = __shfl_sync(full, prio, m);
      const int64_t em = shfl64(exp_ns, m);
      if (valid && ((best_members >> m) & 1u) && in_unit_less(tm, ndm, pm, em, uint32_t(m), tgo, nd, prio, exp_ns, uint32_t(lane))) rk++;
    }
  }

  // ---- TaskPlan.Export order: TotalValue desc, anchor asc, rank in unit asc (all-pairs count) ----
  uint32_t pos = 0;
  for (int m = 0; m < tn; m++) {
    const int64_t vm = shfl64(best_v, m);
    const uint32_t um = __shfl_sync(full, best_u, m), rm = __shfl_sync(full, rk, m);
    if (vm > best_v || (vm == best_v && (um < best_u || (um == best_u && rm < rk)))) pos++;
  }
  if (valid) {
    order[base + pos] = lane;
    total_value[base + pos] = best_v;
  }
}
