// evg_plan_smem.cuh -- k_plan_smem: one CTA plans one distro entirely on-chip.
//
// For distros of up to THREADS*ITEMS tasks (12288 with <1024,12>) the whole
// planner -- queue info, unit construction, scoring, first-occurrence choice,
// the canonical pre-arrangement and the stable LSD radix sort -- runs in one
// kernel with the distro's keys resident in shared memory, so HBM sees exactly
// the compulsory traffic: 48 B/task read once, 12 B/task written once.
//
// Shared memory (cap = THREADS*ITEMS):
//   key  [8*cap]  phases A-D: int64 V[cap] (TotalValue of the unit each task is emitted from)
//                 sort      : uint32 key[2][cap] ping-pong (Vmax - V, ascending == TotalValue descending)
//   idx  [4*cap]  uint16 idx[2][cap] ping-pong;  idx[1] doubles as the anchor histogram e[] before the sort
//   aux  [4*cap]  uint16 anchor[cap], rank_in_unit[cap]
//   wc   [W*256]  uint16 per-warp digit counters / running offsets
//
// Reference: scheduler/planner.go:209-481, scheduler/scheduler.go:56-159.
#pragma once

template <int THREADS, int ITEMS>
struct PlanSmem {
  static constexpr int kCap = THREADS * ITEMS;
  static constexpr int kWarps = THREADS / 32;
  static constexpr size_t kBytes = size_t(16) * kCap + size_t(kWarps) * 256 * 2 + 256 * 4 * 2 + (kCap / 8) * 2 + 512;
};

struct PlanShared {
  int64_t base, dep0;
  int32_t tn, ng, d, any_complex, gv, has_edges;
  uint32_t ub;
  unsigned long long vmax_enc, vmin_enc;   // encoded so that atomicMax / atomicMin work on unsigned
  int32_t n_displaced;
  int32_t tg_fallback;
  unsigned int n_list;
  // queue-info block accumulators
  unsigned int c[10];
  unsigned long long s[4];
  unsigned int tgc[5];           // task-group tasks: n, counted, over, wait, merge-queue
  unsigned long long tgs[2];     // task-group tasks: expected sum, over-threshold sum
};

// cp.async (LDGSTS): global -> shared without a register round trip
__device__ __forceinline__ void cp_async4_s(uint32_t smem_addr, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_addr), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async8_s(uint32_t smem_addr, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_addr), "l"(gmem_src) : "memory");
}
// 64-bit add into shared memory as two native 32-bit atomics (low word, then high word plus the carry the
// low word produced).  A 64-bit shared atomicAdd compiles to a compare-and-swap spin loop, which crawls when
// the lanes of a warp hit the same task group; sums commute, so the split form ends at the same 64-bit value.
__device__ __forceinline__ void smem_add64(unsigned long long* addr, unsigned long long v) {
  unsigned int* p = reinterpret_cast<unsigned int*>(addr);
  const unsigned int lo = (unsigned int)v;
  unsigned int hi = (unsigned int)(v >> 32);
  const unsigned int old = atomicAdd(p, lo);
  hi += (old + lo < old) ? 1u : 0u;
  if (hi) atomicAdd(p + 1, hi);
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

// (A vote-based replacement for MATCH.ANY -- 9 ballots per chunk -- issues more instructions per chunk.)
__device__ __forceinline__ unsigned long long ord_i64(int64_t v) { return uint64_t(v) ^ 0x8000000000000000ULL; }
__device__ __forceinline__ int64_t unord_i64(unsigned long long k) { return int64_t(k ^ 0x8000000000000000ULL); }

template <int THREADS, int ITEMS, int MIN_CTAS>
__global__ void __launch_bounds__(THREADS, MIN_CTAS)
k_plan_smem(DTasks T, DDistros D, DWork W, const int32_t* __restrict__ list, const int32_t* __restrict__ list_count,
            int64_t now, int lists_needed, int32_t* __restrict__ order, int64_t* __restrict__ total_value) {
  constexpr int CAP = THREADS * ITEMS;
  constexpr int NW = THREADS / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int64_t* sV = reinterpret_cast<int64_t*>(smem_raw);
  uint32_t* sKey = reinterpret_cast<uint32_t*>(smem_raw);                 // [2][CAP]
  uint16_t* sIdx = reinterpret_cast<uint16_t*>(smem_raw + size_t(8) * CAP);  // [2][CAP]
  uint16_t* sA = reinterpret_cast<uint16_t*>(smem_raw + size_t(12) * CAP);   // anchor
  uint16_t* sRk = sA + CAP;                                               // rank in unit
  uint16_t* sWc = reinterpret_cast<uint16_t*>(smem_raw + size_t(16) * CAP);  // [NW][256]
  uint32_t* sTot = reinterpret_cast<uint32_t*>(sWc + NW * 256);          // [256]
  uint32_t* sScan = sTot + 256;                                           // [256] scratch for block scans
  uint32_t* sHasDep = sScan + 256;                                        // [CAP/32]
  uint32_t* sDisp = sHasDep + CAP / 32;                                   // [CAP/32]
  PlanShared* S = reinterpret_cast<PlanShared*>(sDisp + CAP / 32);
  uint16_t* sE = sIdx + CAP;                                              // anchor histogram, aliases idx[1]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned full = 0xffffffffu;

  if (*W.err) return;  // k_validate found an out-of-range id in this upload: plan nothing (uniform exit)
  // list_count != nullptr: `list` was filled on the device (distros k_plan_cta handed back) and the grid is its capacity
  if (list_count && int(blockIdx.x) >= *list_count) return;
  // ---- phase 0: distro header ----
  if (tid == 0) {
    const int d = list[blockIdx.x];
    S->d = d;
    S->base = D.task_off[d];
    S->tn = int32_t(D.task_off[d + 1] - D.task_off[d]);
    S->ng = int32_t(D.group_off[d + 1] - D.group_off[d]);
    S->ub = uint32_t(D.unit_base[d]);
    S->gv = D.cfg[d].group_versions != 0;
    int64_t e0 = 0, e1 = 0;
    if (T.n_edges > 0) { e0 = T.dep_off[S->base]; e1 = T.dep_off[S->base + S->tn]; }
    S->dep0 = e0;
    S->has_edges = e1 > e0;
    S->any_complex = (S->ng > 0) || S->gv || (e1 > e0);
    S->vmax_enc = 0ull;
    S->vmin_enc = ~0ull;
    S->n_displaced = 0;
    S->n_list = 0;
    S->tg_fallback = 0;
    for (int k = 0; k < 10; k++) S->c[k] = 0;
    for (int k = 0; k < 4; k++) S->s[k] = 0;
    for (int k = 0; k < 5; k++) S->tgc[k] = 0;
    S->tgs[0] = 0; S->tgs[1] = 0;
  }
  for (int i = tid; i < CAP / 32; i += THREADS) { sHasDep[i] = 0; sDisp[i] = 0; }
  __syncthreads();
  const int d = S->d;
  const int64_t base = S->base;
  const int tn = S->tn;
  const uint32_t ng = uint32_t(S->ng), ub = S->ub;
  const bool gv = S->gv != 0, any = S->any_complex != 0, has_edges = S->has_edges != 0;
  const evg_distro_cfg cfg = D.cfg[d];

  // ---- phase 1: dependents (planner.go:449-456) and empty unit lists ----
  if (has_edges) {
    for (int i = tid; i < tn; i += THREADS) {
      const int64_t t = base + i;
      for (int64_t e = T.dep_off[t]; e < T.dep_off[t + 1]; e++) {
        const uint32_t dl = uint32_t(T.dep_idx[e]);
        atomicOr(&sHasDep[dl >> 5], 1u << (dl & 31));
      }
    }
    __syncthreads();
  }
  if (any) {
    const uint32_t nv = gv ? uint32_t(cfg.n_versions) : 0u;
    for (uint32_t s = tid; s < ng + nv; s += THREADS) W.head[ub + s] = kInactive;
    if (!gv && has_edges)
      for (int i = tid; i < tn; i += THREADS)
        if (sHasDep[i >> 5] & (1u << (i & 31))) W.head[ub + ng + i] = kInactive;
    // TaskGroupInfo rows start from zero (no host-side memset): the list-free path rewrites the sums in phase 3,
    // the other paths accumulate into them with global atomics after the barrier below
    for (uint32_t g = tid; g < ng; g += THREADS) {
      evg_group_info z;
      z.count = 0; z.count_free = 0; z.count_required = 0; z.max_hosts = D.gmax[D.group_off[d] + g];
      z.expected_duration = 0; z.count_duration_over_threshold = 0; z.count_wait_over_threshold = 0;
      z.count_dep_filled_merge_queue_tasks = 0; z.duration_over_threshold = 0;
      W.ginfo[D.group_off[d] + g] = z;
    }
    __syncthreads();
  }

  // ---- phase 2: per task -- queue info, score of single-task units; tasks that touch a
  // multi-member unit (task group, GroupVersions, in-queue dependency either way) are
  // compacted into a work list so the list phases below run with full warps ----
  uint16_t* sList = sWc;                      // free until the sort
  constexpr int kListCap = NW * 256;
  // distro totals only; the "" group is totals minus the task-group tasks, which phase 2b sums over the work list
  unsigned int c_dm = 0, c_mq = 0, c_over = 0, c_wait = 0, c_sec = 0, c_cnt = 0;
  int64_t s_exp = 0, s_over = 0;
  const int64_t threshold = cfg.target_time_ns;
  const PlannerFactors pf = clamp_factors(cfg);
  // since(now, wb) > threshold  <=>  wb < now - threshold whenever 0 <= threshold <= now (no overflow on either
  // side; the Go zero time is INT64_MIN and so always "waits"); other clocks take the literal saturating path.
  const bool sane_clock = threshold >= 0 && now >= threshold;
  const int64_t wait_cutoff = wsub(now, threshold);
  const bool fast_clock = now >= 0 && pf.nd_int != 0;  // single_task_value_fast's distro-wide preconditions
  // The seven columns of the next iteration are staged with cp.async while this one computes (4 x 4 B + 3 x 8 B per
  // thread; each thread reads back only what it copied itself).  One stage in flight: the loop is issue-bound, a
  // second stage does not shorten it.  The index region (b = 0) and the anchor/rank region (b = 1) are both idle until
  // phase 3; the stage lives in the index region.
  constexpr bool kStage = size_t(4) * CAP >= size_t(THREADS) * 40;
  // [4][THREADS] priority, num_dependents, group_id, flags, then [3][THREADS] expected, queue_basis, wait_basis
  auto stage32 = [&](int b) { return reinterpret_cast<uint32_t*>(b ? sA : sIdx); };
  auto stage64 = [&](int b) { return reinterpret_cast<int64_t*>(stage32(b) + 4 * THREADS); };
  const uint32_t a32 = uint32_t(__cvta_generic_to_shared(stage32(0) + tid)), a64 = uint32_t(__cvta_generic_to_shared(stage64(0) + tid));
  auto prefetch = [&](int i0) {  // always closes a copy group (possibly empty)
    const int i = i0 + tid;
    if (i < tn) {
      const int64_t t = base + i;
      cp_async4_s(a32 + 0 * THREADS * 4, T.priority + t);
      cp_async4_s(a32 + 1 * THREADS * 4, T.numdep + t);
      cp_async4_s(a32 + 2 * THREADS * 4, T.gid + t);
      cp_async4_s(a32 + 3 * THREADS * 4, T.flags + t);
      cp_async8_s(a64 + 0 * THREADS * 8, T.expected + t);
      cp_async8_s(a64 + 1 * THREADS * 8, T.qbasis + t);
      cp_async8_s(a64 + 2 * THREADS * 8, T.wbasis + t);
    }
    cp_async_commit();
  };
  if (kStage) prefetch(0);
  for (int i0 = 0; i0 < tn; i0 += THREADS) {
    const int i = i0 + tid;
    bool complex_task = false, scores = false;
    int32_t prio = 0, nd = 0, gid = -1;
    int64_t exp_ns = 0, qb = 0, wb = 0;
    uint32_t fl = 0;
    if (kStage) {
      cp_async_wait_all();
      if (i < tn) {
        const uint32_t* st32 = stage32(0);
        const int64_t* st64 = stage64(0);
        prio = int32_t(st32[0 * THREADS + tid]); nd = int32_t(st32[1 * THREADS + tid]);
        gid = int32_t(st32[2 * THREADS + tid]); fl = st32[3 * THREADS + tid];
        exp_ns = st64[0 * THREADS + tid]; qb = st64[1 * THREADS + tid]; wb = st64[2 * THREADS + tid];
      }
      prefetch(i0 + THREADS);  // refill the stage just consumed
    } else if (i < tn) {
      const int64_t t = base + i;
      prio = T.priority[t]; nd = T.numdep[t]; gid = T.gid[t]; fl = T.flags[t];
      exp_ns = T.expected[t]; qb = T.qbasis[t]; wb = T.wbasis[t];
    }
    if (i < tn) {
      const int64_t t = base + i;
      // GetDistroQueueInfo (scheduler.go:66-138)
      const bool dm = (fl & EVG_TF_DEPS_MET) != 0;
      const bool counted = !cfg.includes_dependencies || dm;
      const bool over = counted && exp_ns > threshold;
      const bool wait_over = counted && dm && (sane_clock ? wb < wait_cutoff : since(now, wb) > threshold);
      const bool mq_dm = dm && (fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE;
      c_dm += dm; c_mq += mq_dm; c_over += over; c_wait += wait_over; c_sec += (fl & EVG_TF_OTHER_DISTRO) != 0;
      c_cnt += counted;
      if (counted) s_exp += exp_ns;
      if (over) s_over += exp_ns;
      const bool own_complex = any && (gid >= 0 || gv || (sHasDep[i >> 5] & (1u << (i & 31))));
      complex_task = own_complex || (has_edges && T.dep_off[t + 1] > T.dep_off[t]);
      scores = !own_complex;  // unit == {this task}
    }
    // every scoring lane inside the exact-integer domain (the production case): one straight-line evaluation,
    // no data-dependent branch; otherwise each lane takes the literal path
    if (fast_clock && __all_sync(full, !scores || score_fast_domain(now, exp_ns, qb))) {
      const int64_t v = single_task_value_fast(pf, now, prio, exp_ns, qb, nd, fl);
      if (scores) sV[i] = v;
    } else if (scores) {
      sV[i] = single_task_value(pf, now, prio, exp_ns, qb, nd, fl);
    }
    if (any) {  // warp-aggregated append
      const unsigned m = __ballot_sync(full, complex_task);
      if (m) {
        unsigned int pos0 = 0;
        if (lane == 0) pos0 = atomicAdd(&S->n_list, (unsigned int)__popc(m));
        pos0 = __shfl_sync(full, pos0, 0);
        if (complex_task) {
          const unsigned int pos = pos0 + __popc(m & ((1u << lane) - 1u));
          if (pos < (unsigned)kListCap) sList[pos] = uint16_t(i);
        }
      }
    }
  }
  // fold the queue-info partials: warp shuffle, then shared atomics; the row is written after phase 2b
  {
    unsigned int cs[6] = {c_dm, c_mq, c_over, c_wait, c_sec, c_cnt};
#pragma unroll
    for (int k = 0; k < 6; k++) cs[k] = __reduce_add_sync(full, cs[k]);
    int64_t ss[2] = {s_exp, s_over};
#pragma unroll
    for (int k = 0; k < 2; k++) ss[k] = warp_sum64(ss[k]);
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 6; k++) if (cs[k]) atomicAdd(&S->c[k], cs[k]);
#pragma unroll
      for (int k = 0; k < 2; k++) if (ss[k]) atomicAdd(&S->s[k], (unsigned long long)ss[k]);
    }
  }
  __syncthreads();

  // The list phases iterate the compacted work list (or, if it overflowed, every task with a filter).
  const int n_list = int(S->n_list);
  const bool use_list = n_list <= kListCap;
  const int n_work = !any ? 0 : (use_list ? n_list : tn);
  auto work_item = [&](int k) -> int {
    if (use_list) return int(sList[k]);
    const int64_t t = base + k;
    const bool cx = T.gid[t] >= 0 || gv || (sHasDep[k >> 5] & (1u << (k & 31))) ||
                    (has_edges && T.dep_off[t + 1] > T.dep_off[t]);
    return cx ? k : -1;
  };

  // Task-group-only distros (no GroupVersions, no in-queue dependency edges) take a list-free path: every
  // multi-member unit is exactly one task group, so Unit.info is a handful of shared-memory atomics per member,
  // and -- when TaskGroupOrder is unique inside each group, which is what a task group's order means -- a
  // member's rank inside its unit is the number of smaller orders present (a 64-bit presence mask).
  // Anything else (orders >= 64, duplicate orders, too many groups, breakdown mode) falls back to the unit lists.
  constexpr int kGroupCap = (4 * CAP) / 84;
  unsigned long long* gTiq = reinterpret_cast<unsigned long long*>(sIdx);  // the staging area is idle again
  unsigned long long* gRt = gTiq + kGroupCap;
  unsigned long long* gMask = gRt + kGroupCap;
  long long* gV = reinterpret_cast<long long*>(gMask + kGroupCap);
  int* gMaxP = reinterpret_cast<int*>(gV + kGroupCap);
  int* gMaxD = gMaxP + kGroupCap;
  unsigned int* gFlags = reinterpret_cast<unsigned int*>(gMaxD + kGroupCap);
  unsigned int* gN = gFlags + kGroupCap;
  unsigned int* gAnchor = gN + kGroupCap;
  // TaskGroupInfo sums of the same groups (scheduler.go:79-137), written out once per group
  unsigned long long* qExp = reinterpret_cast<unsigned long long*>(gAnchor + kGroupCap + (kGroupCap & 1));
  unsigned long long* qDurOver = qExp + kGroupCap;
  unsigned int* qCnt = reinterpret_cast<unsigned int*>(qDurOver + kGroupCap);
  unsigned int* qOver = qCnt + kGroupCap;
  unsigned int* qWait = qOver + kGroupCap;
  unsigned int* qMq = qWait + kGroupCap;
  bool fast_tg = any && !gv && !has_edges && !lists_needed && int(ng) <= kGroupCap;
  const bool smem_ginfo = fast_tg;  // stays true even if the rank shortcut later falls back

  if (any) {
    // ---- phase 2b: task-group sums (scheduler.go:79-137) ----
    if (fast_tg)
      for (int g = tid; g < int(ng); g += THREADS) {
        gTiq[g] = 0ull; gRt[g] = 0ull; gMask[g] = 0ull; gMaxP[g] = 0; gMaxD[g] = 0; gFlags[g] = 0u; gN[g] = 0u;
        gAnchor[g] = kNoAnchor;
        qExp[g] = 0ull; qDurOver[g] = 0ull; qCnt[g] = 0u; qOver[g] = 0u; qWait[g] = 0u; qMq[g] = 0u;
      }
    __syncthreads();
    unsigned int t_n = 0, t_cnt = 0, t_over = 0, t_wait = 0, t_mq = 0;
    int64_t t_exp = 0, t_dover = 0;
    for (int k = tid; k < n_work; k += THREADS) {
      const int i = work_item(k);
      if (i < 0) continue;
      const int64_t t = base + i;
      // every column this phase needs, requested together: one L2 round trip instead of a chain of them
      const int32_t gid = T.gid[t];
      const int64_t exp_ns = T.expected[t], wb = T.wbasis[t];
      const uint32_t fl = T.flags[t];
      int32_t tgo = 0, prio = 0, nd = 0;
      int64_t qb = 0;
      if (fast_tg) { tgo = T.tgo[t]; qb = T.qbasis[t]; prio = T.priority[t]; nd = T.numdep[t]; }  // CTA-uniform
      if (gid < 0) continue;
      const bool dm = (fl & EVG_TF_DEPS_MET) != 0;
      const bool counted = !cfg.includes_dependencies || dm;
      const bool over = counted && exp_ns > threshold;
      const bool wait_over = counted && dm && since(now, wb) > threshold;
      const bool mq_dm = dm && (fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE;
      t_n += 1; t_cnt += counted; t_over += over; t_wait += wait_over; t_mq += mq_dm;
      if (counted) t_exp += exp_ns;
      if (over) t_dover += exp_ns;
      if (smem_ginfo) {
        if (counted) { atomicAdd(&qCnt[gid], 1u); smem_add64(&qExp[gid], (unsigned long long)exp_ns); }
        if (over) { atomicAdd(&qOver[gid], 1u); smem_add64(&qDurOver[gid], (unsigned long long)exp_ns); }
        if (wait_over) atomicAdd(&qWait[gid], 1u);
        if (mq_dm) atomicAdd(&qMq[gid], 1u);
      } else {
        evg_group_info* g = W.ginfo + D.group_off[d] + gid;
        atomic_add64(&g->count, counted);
        atomic_add64(&g->expected_duration, counted ? exp_ns : 0);
        atomic_add64(&g->count_duration_over_threshold, over);
        atomic_add64(&g->duration_over_threshold, over ? exp_ns : 0);
        atomic_add64(&g->count_wait_over_threshold, wait_over);
        atomic_add64(&g->count_dep_filled_merge_queue_tasks, mq_dm);
      }
      if (fast_tg) {  // Unit.info (planner.go:302-337) of the task-group unit, member by member
        if (tgo < 0 || tgo >= 64) { S->tg_fallback = 1; continue; }
        // phase 4 ranks this task from (group, order) alone: park them in the task's still unused value slot
        reinterpret_cast<uint32_t*>(&sV[i])[0] = uint32_t(gid) | (uint32_t(tgo) << 16);
        const uint32_t req = fl & EVG_TF_REQ_MASK;
        uint32_t uf = 0;
        if (req == EVG_TF_REQ_MERGE_QUEUE) uf |= UF_MERGE_QUEUE;
        else if (req == EVG_TF_REQ_PATCH) uf |= UF_PATCH;
        if (fl & EVG_TF_GENERATE) uf |= UF_GENERATE;
        if (fl & EVG_TF_STEPBACK) uf |= UF_STEPBACK;
        if (qb != EVG_TIME_ZERO) smem_add64(&gTiq[gid], (unsigned long long)since(now, qb));
        smem_add64(&gRt[gid], (unsigned long long)exp_ns);
        atomicMax(&gMaxP[gid], prio);
        atomicMax(&gMaxD[gid], nd);
        if (uf) atomicOr(&gFlags[gid], uf);
        atomicAdd(&gN[gid], 1u);
        atomicMin(&gAnchor[gid], uint32_t(i));
        atomicOr(reinterpret_cast<unsigned int*>(&gMask[gid]) + (tgo >> 5), 1u << (tgo & 31));  // 64-bit presence mask, word by word
      }
    }
    // one shared atomic per warp and field: a 64-bit shared atomicAdd is a CAS spin loop, and the work list
    // hands nearly every thread one task-group task, so per-thread adds would all fight over two addresses
    if (__any_sync(full, t_n != 0)) {
      t_n = __reduce_add_sync(full, t_n); t_cnt = __reduce_add_sync(full, t_cnt); t_over = __reduce_add_sync(full, t_over);
      t_wait = __reduce_add_sync(full, t_wait); t_mq = __reduce_add_sync(full, t_mq);
      t_exp = warp_sum64(t_exp); t_dover = warp_sum64(t_dover);
      if (lane == 0) {
        atomicAdd(&S->tgc[0], t_n); atomicAdd(&S->tgc[1], t_cnt); atomicAdd(&S->tgc[2], t_over);
        atomicAdd(&S->tgc[3], t_wait); atomicAdd(&S->tgc[4], t_mq);
        atomicAdd(&S->tgs[0], (unsigned long long)t_exp); atomicAdd(&S->tgs[1], (unsigned long long)t_dover);
      }
    }
    __syncthreads();
    if (fast_tg) {
      // ---- phase 3 (list-free): score each task group's unit (planner.go:209-300) ----
      for (int g = tid; g < int(ng); g += THREADS) {
        evg_group_info* gi = W.ginfo + D.group_off[d] + g;  // one writer per row (max_hosts was set in phase 1)
        gi->count = qCnt[g];
        gi->expected_duration = int64_t(qExp[g]);
        gi->count_duration_over_threshold = qOver[g];
        gi->duration_over_threshold = int64_t(qDurOver[g]);
        gi->count_wait_over_threshold = qWait[g];
        gi->count_dep_filled_merge_queue_tasks = qMq[g];
        if (gN[g] != uint32_t(__popcll(gMask[g]))) { S->tg_fallback = 1; continue; }  // duplicate TaskGroupOrder
        UnitAcc a;
        a.tiq = int64_t(gTiq[g]); a.rt = int64_t(gRt[g]); a.max_p = gMaxP[g]; a.max_d = gMaxD[g];
        a.n = gN[g]; a.flags = gFlags[g];
        gV[g] = a.n ? unit_value(a, cfg, nullptr) : 0;
      }
      __syncthreads();
      fast_tg = S->tg_fallback == 0;
    }
    if (fast_tg) {
      // ---- phase 4 (list-free): a task-group task is emitted from its group's unit, ranked by its order ----
      for (int k = tid; k < n_work; k += THREADS) {
        const int i = work_item(k);
        if (i < 0) continue;
        // work items are exactly the task-group tasks here (no GroupVersions, no edges); phase 2b parked (group, order)
        const uint32_t packed = reinterpret_cast<const uint32_t*>(&sV[i])[0];
        const uint32_t gid = packed & 0xFFFFu;
        const uint32_t brk = __popcll(gMask[gid] & ((1ull << (packed >> 16)) - 1ull));
        const uint32_t ba = gAnchor[gid];
        sV[i] = gV[gid];
        sA[i] = uint16_t(ba);
        sRk[i] = uint16_t(brk);
        if (!(ba == uint32_t(i) && brk == 0)) { atomicOr(&sDisp[i >> 5], 1u << (i & 31)); S->n_displaced = 1; }
      }
      __syncthreads();
    }
  }

  if (any && !fast_tg) {
    // ---- phase 2c: unit membership links (planner.go:431-456) ----
    for (int k = tid; k < n_work; k += THREADS) {
      const int i = work_item(k);
      if (i < 0) continue;
      const int64_t t = base + i;
      const int32_t gid = T.gid[t], vid = T.vid[t];
      const bool own_complex = gid >= 0 || gv || (sHasDep[i >> 5] & (1u << (i & 31)));
      const uint32_t s_own = own_slot_local(gid, vid, uint32_t(i), ng, gv);
      const uint32_t s_ver = (gid >= 0 && gv) ? ng + uint32_t(vid) : kInactive;
      if (own_complex) link_pair(W, uint32_t(t), ub + s_own);
      if (s_ver != kInactive) link_pair(W, uint32_t(T.n + t), ub + s_ver);  // planner.go:439
      if (has_edges) {
        const int64_t e0 = T.dep_off[t], e1 = T.dep_off[t + 1];
        for (int64_t e = e0; e < e1; e++) {
          const uint32_t dl = uint32_t(T.dep_idx[e]);
          const uint32_t s = own_slot_local(T.gid[base + dl], T.vid[base + dl], dl, ng, gv);
          bool dup = (s == s_own) || (s == s_ver);  // Unit.Add is keyed by task id (planner.go:131)
          for (int64_t f = e0; f < e && !dup; f++) {
            const uint32_t fl2 = uint32_t(T.dep_idx[f]);
            dup = own_slot_local(T.gid[base + fl2], T.vid[base + fl2], fl2, ng, gv) == s;
          }
          W.edge_task[e] = uint32_t(t);
          W.edge_live[e] = dup ? 0 : 1;
          if (!dup) link_pair(W, uint32_t(2 * T.n + e), ub + s);
        }
      }
    }
    __syncthreads();

    // ---- phase 3a: the pair at the head of a unit's list owns the unit: one walk for Unit.info / value / anchor ----
    auto unit_head = [&](uint32_t p) {
      const uint32_t slot = W.pair_slot[p];
      if (W.head[slot] != p) return;
      UnitAcc a;
      acc_init(a);
      uint32_t anchor = kNoAnchor;
      for (uint32_t q = p; q < kEnd; q = W.next[q]) {
        const uint32_t tq = pair_task(T, W, q);
        acc_add(a, now, T.priority[tq], T.expected[tq], T.qbasis[tq], T.numdep[tq], T.gid[tq], T.flags[tq]);
        if (q < uint32_t(T.n)) anchor = min(anchor, uint32_t(tq - base));  // own-key pairs are the SetDistro members (planner.go:446)
      }
      W.unit_v[slot] = unit_value(a, cfg, nullptr);
      W.unit_a[slot] = anchor;  // kNoAnchor: never got a distro -> not exported (planner.go:81-83)
      W.unit_n[slot] = uint32_t(a.n);
      W.unit_mask[slot] = 0ull;
    };
    for (int k = tid; k < n_work; k += THREADS) {
      const int i = work_item(k);
      if (i < 0) continue;
      const int64_t t = base + i;
      const int32_t gid = T.gid[t];
      const bool own_complex = gid >= 0 || gv || (sHasDep[i >> 5] & (1u << (i & 31)));
      if (own_complex) unit_head(uint32_t(t));
      if (gid >= 0 && gv) unit_head(uint32_t(T.n + t));
      if (has_edges)
        for (int64_t e = T.dep_off[t]; e < T.dep_off[t + 1]; e++)
          if (W.edge_live[e]) unit_head(uint32_t(2 * T.n + e));
    }
    __syncthreads();

    // ---- phase 3b/4: the unit each task is emitted from (first occurrence in TaskPlan.Export,
    // planner.go:467-477) and the task's rank inside it (TaskList.Less, planner.go:387-405) ----
    for (int k = tid; k < n_work; k += THREADS) {
      const int i = work_item(k);
      if (i < 0) continue;
      const int64_t t = base + i;
      const int32_t gid = T.gid[t];
      const bool own_complex = gid >= 0 || gv || (sHasDep[i >> 5] & (1u << (i & 31)));
      const bool has_ver = gid >= 0 && gv;
      const int64_t e0 = has_edges ? T.dep_off[t] : 0, e1 = has_edges ? T.dep_off[t + 1] : 0;
      bool have = false;
      int64_t bv = 0;
      uint32_t ba = 0, bslot = 0, bp = kInactive;
      auto consider = [&](uint32_t p) {
        const uint32_t slot = W.pair_slot[p];
        const uint32_t a = W.unit_a[slot];
        if (a == kNoAnchor) return;
        const int64_t v = W.unit_v[slot];
        if (!have || v > bv || (v == bv && a < ba)) { have = true; bv = v; ba = a; bslot = slot; bp = p; }
      };
      if (!own_complex) { have = true; bv = sV[i]; ba = uint32_t(i); }
      else consider(uint32_t(t));
      if (has_ver) consider(uint32_t(T.n + t));
      for (int64_t e = e0; e < e1; e++)
        if (W.edge_live[e]) consider(uint32_t(2 * T.n + e));
      uint32_t brk = 0;
      if (bp != kInactive) {  // rank among ALL members of the chosen unit
        const int32_t my_tgo = T.tgo[t], my_nd = T.numdep[t], my_pr = T.priority[t];
        const int64_t my_ex = T.expected[t];
        for (uint32_t q = W.head[bslot]; q < kEnd; q = W.next[q]) {
          const uint32_t tq = pair_task(T, W, q);
          if (in_unit_less(T.tgo[tq], T.numdep[tq], T.priority[tq], T.expected[tq], uint32_t(tq - base),
                           my_tgo, my_nd, my_pr, my_ex, uint32_t(i))) brk++;
        }
        // units of up to 64 members publish which ranks they emit, so phase 6 needs no second walk
        if (W.unit_n[bslot] <= 64) atomicOr(&W.unit_mask[bslot], 1ull << brk);
      }
      sV[i] = bv;
      sA[i] = uint16_t(ba);
      sRk[i] = uint16_t(brk);
      W.best_pair[t] = bp;
      if (!(ba == uint32_t(i) && brk == 0)) { atomicOr(&sDisp[i >> 5], 1u << (i & 31)); S->n_displaced = 1; }
    }
    __syncthreads();
  }

  if (tid == 0) {  // DistroQueueInfo row (scheduler.go:144-158); "" group = totals - task-group tasks
    evg_queue_info q;
    q.length = tn;
    q.length_with_dependencies_met = S->c[0];
    q.count_dep_filled_merge_queue_tasks = S->c[1];
    q.expected_duration = int64_t(S->s[0]);
    q.max_duration_threshold = threshold;
    q.count_duration_over_threshold = S->c[2];
    q.duration_over_threshold = int64_t(S->s[1]);
    q.count_wait_over_threshold = S->c[3];
    q.secondary_queue = S->c[4] != 0;
    q.has_ungrouped = (unsigned int)tn > S->tgc[0];
    q.ungrouped.count = S->c[5] - S->tgc[1];
    q.ungrouped.count_free = 0;
    q.ungrouped.count_required = 0;
    q.ungrouped.max_hosts = 0;
    q.ungrouped.expected_duration = int64_t(S->s[0] - S->tgs[0]);
    q.ungrouped.count_duration_over_threshold = S->c[2] - S->tgc[2];
    q.ungrouped.count_wait_over_threshold = S->c[3] - S->tgc[3];
    q.ungrouped.count_dep_filled_merge_queue_tasks = S->c[1] - S->tgc[4];
    q.ungrouped.duration_over_threshold = int64_t(S->s[1] - S->tgs[1]);
    W.qinfo[d] = q;
  }

  // ---- phase 5: value range ----
  {
    unsigned long long mx = 0ull, mn = ~0ull;
    for (int i = tid; i < tn; i += THREADS) {
      const unsigned long long k = ord_i64(sV[i]);
      mx = max(mx, k);
      mn = min(mn, k);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mx = max(mx, __shfl_xor_sync(full, mx, o));
      mn = min(mn, __shfl_xor_sync(full, mn, o));
    }
    if (lane == 0) { atomicMax(&S->vmax_enc, mx); atomicMin(&S->vmin_enc, mn); }
  }
  // ---- phase 6: canonical pre-arrangement (ties: unit anchor asc, rank in unit asc) ----
  const bool displaced = any && (S->n_displaced != 0);  // n_displaced was published by the barrier that closed phase 4
  if (displaced) {
    uint32_t* e32 = reinterpret_cast<uint32_t*>(sE);
    for (int i = tid; i < CAP / 2; i += THREADS) e32[i] = 0;
    __syncthreads();
    for (int i = tid; i < tn; i += THREADS) {
      const uint32_t a = (sDisp[i >> 5] & (1u << (i & 31))) ? uint32_t(sA[i]) : uint32_t(i);  // anchor of a task emitted alone / first is itself
      atomicAdd(&e32[a >> 1], 1u << (16 * (a & 1)));
    }
    __syncthreads();
    // exclusive scan of e[0..CAP): ITEMS consecutive entries per thread
    uint32_t loc[ITEMS];
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < ITEMS; k++) { loc[k] = sE[tid * ITEMS + k]; sum += loc[k]; }
    uint32_t run = block_scan_excl<NW>(sum, sScan);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) { sE[tid * ITEMS + k] = uint16_t(run); run += loc[k]; }
    __syncthreads();
    for (int i = tid; i < tn; i += THREADS)
      if (!(sDisp[i >> 5] & (1u << (i & 31)))) sIdx[sE[i]] = uint16_t(i);  // rank 0 of its own anchor
    for (int k = tid; k < n_work; k += THREADS) {
      const int i = work_item(k);
      if (i < 0 || !(sDisp[i >> 5] & (1u << (i & 31)))) continue;
      // offset among the tasks emitted from the same unit: members with the same best anchor and a smaller rank
      const uint32_t a = sA[i];
      uint32_t pos = sE[a];
      const uint32_t myrk = sRk[i];
      if (fast_tg) {  // every member of a task-group unit is emitted from it: the rank is the offset
        sIdx[pos + myrk] = uint16_t(i);
        continue;
      }
      const uint32_t slot = W.pair_slot[W.best_pair[base + i]];
      if (W.unit_n[slot] <= 64) {
        pos += __popcll(W.unit_mask[slot] & ((1ull << myrk) - 1ull));
      } else {
        for (uint32_t q = W.head[slot]; q < kEnd; q = W.next[q]) {
          const uint32_t lq = uint32_t(pair_task(T, W, q) - base);
          if (sA[lq] == a && sRk[lq] < myrk) pos++;
        }
      }
      sIdx[pos] = uint16_t(i);
    }
  } else {
    for (int i = tid; i < tn; i += THREADS) sIdx[i] = uint16_t(i);
  }
  __syncthreads();

  // ---- phase 7: compact keys: key = Vmax - V (ascending key == descending TotalValue) ----
  const int64_t vmax = unord_i64(S->vmax_enc);
  const uint64_t range = tn > 0 ? uint64_t(S->vmax_enc - S->vmin_enc) : 0;
  int bits = 64 - __clzll((long long)(range | 1ull));
  if (range == 0) bits = 0;
  const bool wide = bits > 32;
  {
    uint32_t kreg[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      const int p = tid + k * THREADS;
      kreg[k] = 0;
      if (p < tn) {
        const uint32_t i = sIdx[p];
        const uint64_t k64 = uint64_t(vmax) - uint64_t(sV[i]);
        kreg[k] = uint32_t(k64);
        if (wide) W.buf[0].key_v[base + i] = k64;  // high word is reloaded after the four low passes
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      const int p = tid + k * THREADS;
      if (p < tn) sKey[p] = kreg[k];
    }
  }
  __syncthreads();

  // ---- phase 8: stable LSD radix sort, 8-bit digits, warp-segmented ranking ----
  int cur = 0;
  const int seg = ((tn + NW - 1) / NW + 31) & ~31;  // elements per warp, multiple of 32
  const int seg0 = warp * seg;
  const int seg1 = min(seg0 + seg, tn);
  const unsigned lt = (1u << lane) - 1u;
  const int npass = (bits + 7) / 8;
  for (int pass = 0; pass < npass; pass++) {
    if (pass == 4) {  // wide keys: switch to the high word
      uint32_t* kc = sKey + cur * CAP;
      const uint16_t* ic = sIdx + cur * CAP;
      for (int p = tid; p < tn; p += THREADS) kc[p] = uint32_t(W.buf[0].key_v[base + ic[p]] >> 32);
      __syncthreads();
    }
    const int shift = 8 * (pass & 3);
    const uint32_t* kc = sKey + cur * CAP;
    const uint16_t* ic = sIdx + cur * CAP;
    uint32_t* kn = sKey + (cur ^ 1) * CAP;
    uint16_t* in_ = sIdx + (cur ^ 1) * CAP;
    uint32_t* wcAll = reinterpret_cast<uint32_t*>(sA);  // [NW][256]; anchor/rank arrays are dead after phase 7
    uint32_t* wc = wcAll + warp * 256;
    for (int k = lane; k < 256; k += 32) wc[k] = 0;
    __syncwarp();
    // histogram of this warp's segment: shared-memory atomics on the warp's private counters
    // (MATCH.ANY here was the sort's bottleneck: one shared unit per SM, ~50 cycles per warp instruction)
    for (int s0 = seg0; s0 < seg1; s0 += 128) {
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int p = s0 + u * 32 + lane;
        if (p < seg1) atomicAdd(&wc[(kc[p] >> shift) & 255u], 1u);
      }
    }
    __syncthreads();
    // per-digit totals of each slice of warps, digit bases, then running offsets (base folded in)
    constexpr int PARTS = THREADS >= 256 ? THREADS / 256 : 1;
    constexpr int WPP = NW / PARTS;
    uint32_t* sPart = reinterpret_cast<uint32_t*>(sWc);  // [PARTS][256]; the work list is dead by now
    for (int x = tid; x < 256 * PARTS; x += THREADS) {
      const int dgt = x & 255, part = x >> 8;
      uint32_t sum = 0;
#pragma unroll
      for (int w = 0; w < WPP; w++) sum += wcAll[(part * WPP + w) * 256 + dgt];
      sPart[part * 256 + dgt] = sum;
    }
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the 256 digit totals
      uint32_t v[8], sum = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        uint32_t tot = 0;
#pragma unroll
        for (int pp = 0; pp < PARTS; pp++) tot += sPart[pp * 256 + lane * 8 + k];
        v[k] = tot;
        sum += tot;
      }
      uint32_t run = warp_scan_incl(sum) - sum;
#pragma unroll
      for (int k = 0; k < 8; k++) { sTot[lane * 8 + k] = run; run += v[k]; }
    }
    __syncthreads();
    for (int x = tid; x < 256 * PARTS; x += THREADS) {
      const int dgt = x & 255, part = x >> 8;
      uint32_t run = sTot[dgt];
      for (int pp = 0; pp < part; pp++) run += sPart[pp * 256 + dgt];
#pragma unroll
      for (int w = 0; w < WPP; w++) {
        const uint32_t xx = wcAll[(part * WPP + w) * 256 + dgt];
        wcAll[(part * WPP + w) * 256 + dgt] = run;
        run += xx;
      }
    }
    __syncthreads();
    for (int s0 = seg0; s0 < seg1; s0 += 64) {
      uint32_t kk[2], dg[2], r[2];
      uint16_t ii[2];
      unsigned peers[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int p = s0 + u * 32 + lane;
        const bool ok = p < seg1;
        kk[u] = ok ? kc[p] : 0u;
        ii[u] = ok ? ic[p] : uint16_t(0);
        dg[u] = ok ? ((kk[u] >> shift) & 255u) : 0xFFFFu;
      }
#pragma unroll
      for (int u = 0; u < 2; u++) { peers[u] = __match_any_sync(full, dg[u]); r[u] = __popc(peers[u] & lt); }
#pragma unroll
      for (int u = 0; u < 2; u++) {  // chunks in order: stability
        const bool ok = dg[u] != 0xFFFFu;
        uint32_t off = 0;
        if (ok && r[u] == 0) off = atomicAdd(&wc[dg[u]], (uint32_t)__popc(peers[u]));
        off = __shfl_sync(full, off, __ffs(peers[u]) - 1);
        if (ok) {
          const uint32_t pos = off + r[u];
          kn[pos] = kk[u];
          in_[pos] = ii[u];
        }
      }
    }
    __syncthreads();
    cur ^= 1;
  }

  // ---- phase 9: ranked queue out (coalesced) ----
  {
    const uint32_t* kc = sKey + cur * CAP;
    const uint16_t* ic = sIdx + cur * CAP;
    if (!wide) {
      for (int p = tid; p < tn; p += THREADS) {
        order[base + p] = int32_t(ic[p]);
        total_value[base + p] = int64_t(uint64_t(vmax) - uint64_t(kc[p]));
      }
    } else {
      for (int p = tid; p < tn; p += THREADS) {
        const uint32_t i = ic[p];
        order[base + p] = int32_t(i);
        total_value[base + p] = int64_t(uint64_t(vmax) - W.buf[0].key_v[base + i]);
      }
    }
  }
}
