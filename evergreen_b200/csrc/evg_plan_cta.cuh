// evg_plan_cta.cuh -- k_plan_cta<THREADS, CAP>: the on-chip planner, second generation.
//
// One CTA plans one distro of up to CAP tasks entirely on-chip, like k_plan_smem (evg_plan_smem.cuh), but sized so
// that SEVERAL CTAs share an SM (2 x 512 threads for 10240-task distros, 4 x 256 for 5120, 8 x 128 for 1280, 16 x 64 for 384): while
// one distro sorts (shared-memory / MATCH bound) its neighbour scores tasks (ALU bound), and nobody idles at the
// other's barriers.  What makes it fit:
//   * TotalValue is kept as a u32 (4 B/task instead of 8).  Every production queue has values far below 2^32; a
//     distro where some value does not fit is handed back ("punted") to k_plan_smem untouched.
//   * the sort moves only a u16 permutation, in place: a pass reads its elements into registers, ranks them with
//     ONE MATCH.ANY per 32 elements (the leader's shared atomicAdd returns the warp-local offset), and scatters
//     after the block-wide counter scan -- 6 B/task of sort state instead of 12.
//   * digits are up to 10 bits wide (16 warps x 1024 u16 counters): a 20-bit value range sorts in 2 passes.
//   * task columns arrive by TMA: one thread issues cp.async.bulk (UBLKCP) copies of the seven columns of a
//     2*THREADS-task tile into one shared-memory stage guarded by a full and an empty mbarrier; the other threads
//     never compute a global address in the task pass.
//   * scoring runs in 32-bit arithmetic wherever the distro's factors and the task allow it (single_task_value32).
// Handles distros without GroupVersions and without in-queue dependency edges (task groups allowed); the host routes
// everything else to k_plan_smem.  Runtime punts: a value outside u32, work-list overflow, TaskGroupOrder >= 64 or
// repeated inside a group.
//
// Shared memory (bytes), CAP = tasks, T = THREADS, W = warps:
//   key   4*CAP            u32 TotalValue per task (phase 2b parks (group, order) of task-group tasks here)
//   idx   2*CAP            u16 permutation                 | task pass: the TMA stage (80*THREADS bytes, from here on)
//   cnt   W*2^bits*2       u16 per-warp digit counters     | task pass: rest of the TMA stage; group phases: per-group
//                                                          |   accumulators (with idx); pre-arrangement: e[] histogram
//   list  6*CAP/4          u16 work list: task, anchor, rank (one stretch per warp)
//
// Reference: scheduler/planner.go:209-481, scheduler/scheduler.go:56-159.
#pragma once

template <int THREADS>
struct CtaDigit {
  static constexpr int kBits = THREADS >= 512 ? 10 : (THREADS >= 256 ? 9 : (THREADS >= 128 ? 8 : 7));  // 2^bits == 2*THREADS: one u32 counter pair per thread in the scan
};

template <int THREADS, int CAP>
struct PlanCta {
  // Tasks per thread and tile of the task pass: one 2*THREADS-task stage, refilled as soon as every thread has its two
  // tasks in registers -- per-tile overhead (barrier wait, refill, list append) amortised over two tasks and two
  // independent scoring chains per thread.
  static constexpr int kTpt = 2;
  static constexpr int kTile = kTpt * THREADS;
  static constexpr int kWarps = THREADS / 32;
  static constexpr int kItems = CAP / THREADS;
  static constexpr int kDigitBits = CtaDigit<THREADS>::kBits;
  static constexpr int kDigitWords = (1 << kDigitBits) / 2;  // u32 words per warp row of u16 counters
  static constexpr int kListCap = CAP / 4;  // task-group tasks a distro may hold here (each warp owns 1/kWarps of it)
  static constexpr size_t kKeyBytes = size_t(4) * CAP;
  static constexpr size_t kIdxBytes = size_t(2) * CAP;
  static constexpr size_t kStageBytes = size_t(40) * kTile;
  static constexpr size_t kCntNeed = size_t(kWarps) * kDigitWords * 4;
  static constexpr size_t kMultiBytes = (kIdxBytes + kCntNeed) > kStageBytes ? (kIdxBytes + kCntNeed) : kStageBytes;  // idx + cnt, contiguous
  static constexpr size_t kListBytes = size_t(6) * kListCap;
  static constexpr size_t kOffKey = 0;
  static constexpr size_t kOffIdx = kKeyBytes;
  static constexpr size_t kOffCnt = kOffIdx + kIdxBytes;
  static constexpr size_t kOffList = kOffIdx + kMultiBytes;
  static constexpr size_t kOffDisp = kOffList + kListBytes;
  static constexpr size_t kOffScan = kOffDisp + size_t(CAP / 32) * 4;
  static constexpr size_t kOffBar = kOffScan + 32 * 4;
  static constexpr size_t kOffShared = kOffBar + 4 * 8;
  static constexpr size_t kOffNd = kOffShared + 160;   // u32[kNdTable]: int64(NumDependentsFactor * n)
  static constexpr size_t kBytes = kOffNd + 4 * 64;
  static constexpr int kGroupCap = int(kMultiBytes / 84) > 65535 ? 65535 : int(kMultiBytes / 84);
  static_assert(CAP % THREADS == 0 && kItems % 2 == 0 && kItems <= 20, "blocked entries per thread: even, at most 20");
  static_assert(CAP / kWarps == 32 * kItems, "a warp's sort segment is kItems chunks of 32");
  static_assert(size_t(2) * CAP <= kMultiBytes - kIdxBytes, "the anchor histogram lives in the counter region");
  static_assert(CAP <= 16384, "u16 permutation, 14-bit task index");
};

struct CtaShared {
  int64_t base;
  int32_t tn, ng, d, off0;
  uint32_t spare;
  int32_t punt, n_displaced;
  uint32_t vmin, vmax;
  unsigned int c[6];
  unsigned long long s[2];
  unsigned int tgc[5];
  unsigned long long tgs[2];
};
static_assert(sizeof(CtaShared) <= 160, "CtaShared outgrew its slot");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// arrive and wait on precomputed shared-window addresses: the task-pass loop issues them every tile
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@!p bra WAIT_%=;\n\t}" ::"r"(bar), "r"(parity)
      : "memory");
}
// TMA, non-tensor form: one contiguous run global -> shared, completion counted in bytes on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// The 64-bit scorers, out of line: the task pass keeps only the 32-bit form in its loop body.  Called by whole warps.
__device__ __noinline__ uint64_t score_slow(const PlannerFactors& pf, bool fast_clock, bool scores, int64_t now, int32_t prio,
                                            int64_t exp_ns, int64_t qb, int32_t nd, uint32_t fl) {
  if (fast_clock && __all_sync(0xffffffffu, !scores || score_fast_domain(now, exp_ns, qb)))
    return uint64_t(single_task_value_fast(pf, now, prio, exp_ns, qb, nd, fl));
  return scores ? uint64_t(single_task_value(pf, now, prio, exp_ns, qb, nd, fl)) : 0ull;
}

template <int THREADS, int CAP, int MIN_CTAS>
__global__ void __launch_bounds__(THREADS, MIN_CTAS)
k_plan_cta(DTasks T, DDistros D, DWork W, const int32_t* __restrict__ list, int64_t now, int64_t t_pad,
           int32_t* __restrict__ order, int64_t* __restrict__ total_value, int32_t* __restrict__ punt_list,
           int32_t* __restrict__ punt_count) {
  using L = PlanCta<THREADS, CAP>;
  constexpr int NW = L::kWarps, ITEMS = L::kItems, DW = L::kDigitWords, MAXBITS = L::kDigitBits;
  constexpr int kListCap = L::kListCap, kGroupCap = L::kGroupCap;
  extern __shared__ __align__(128) unsigned char smem_cta[];
  unsigned char* const smem_raw = smem_cta;
  uint32_t* sKey = reinterpret_cast<uint32_t*>(smem_raw + L::kOffKey);
  uint16_t* sIdx = reinterpret_cast<uint16_t*>(smem_raw + L::kOffIdx);
  uint32_t* sCnt = reinterpret_cast<uint32_t*>(smem_raw + L::kOffCnt);       // [NW][DW] packed u16 pairs
  uint16_t* sList = reinterpret_cast<uint16_t*>(smem_raw + L::kOffList);    // task of work item k
  uint16_t* sLA = sList + kListCap;                                          // its unit's anchor
  uint16_t* sLR = sLA + kListCap;                                            // its rank inside the unit
  uint32_t* sDisp = reinterpret_cast<uint32_t*>(smem_raw + L::kOffDisp);    // [CAP/32] task leaves its input position
  uint32_t* sScan = reinterpret_cast<uint32_t*>(smem_raw + L::kOffScan);    // [32] block-scan scratch
  uint64_t* sBar = reinterpret_cast<uint64_t*>(smem_raw + L::kOffBar);      // full[2], empty[2]; the one stage uses [0] of each
  CtaShared* S = reinterpret_cast<CtaShared*>(smem_raw + L::kOffShared);
  uint32_t* sNd = reinterpret_cast<uint32_t*>(smem_raw + L::kOffNd);
  unsigned char* sStage = smem_raw + L::kOffIdx;                             // the task pass's stage: 40*kTile bytes

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned full = 0xffffffffu;

  if (*W.err) return;  // k_validate found an out-of-range id in this upload: plan nothing (uniform exit)
  // ---- phase 0: distro header, barriers ----
  if (tid == 0) {
    const int d = list[blockIdx.x];
    S->d = d;
    S->base = D.task_off[d];
    S->tn = int32_t(D.task_off[d + 1] - D.task_off[d]);
    S->ng = int32_t(D.group_off[d + 1] - D.group_off[d]);
    S->off0 = int32_t(S->base & 3);
    S->punt = 0; S->n_displaced = 0;
    S->vmin = 0xFFFFFFFFu; S->vmax = 0u;
    for (int k = 0; k < 6; k++) S->c[k] = 0;
    for (int k = 0; k < 2; k++) S->s[k] = 0;
    for (int k = 0; k < 5; k++) S->tgc[k] = 0;
    S->tgs[0] = 0; S->tgs[1] = 0;
    mbar_init(&sBar[0], 1); mbar_init(&sBar[1], 1);
    mbar_init(&sBar[2], THREADS); mbar_init(&sBar[3], THREADS);
    mbar_fence_init();
  }
  for (int i = tid; i < CAP / 32; i += THREADS) sDisp[i] = 0;
  __syncthreads();
  const int d = S->d;
  const int64_t base = S->base;
  const int tn = S->tn, off0 = S->off0;
  const int ng = S->ng;
  const bool any = ng > 0;
  const evg_distro_cfg cfg = D.cfg[d];

  // ---- phase 2: one pass over the task columns ----
  // Tile k holds tasks [a0 + k*TILE, +TILE) of the concatenated table, a0 = base rounded down to a multiple of four
  // tasks so that every copy starts 16-byte aligned; slots `tid` and `tid + THREADS` of the stage are this thread's tasks.
  const int64_t a0 = base - off0;
  constexpr int TPT = L::kTpt, TILE = L::kTile;
  const int n_tiles = (off0 + tn + TILE - 1) / TILE;
  auto issue = [&](int k) {  // thread 0 only
    const int64_t start = a0 + int64_t(k) * TILE;
    const int64_t left = t_pad - start;
    const uint32_t cnt = uint32_t(left < int64_t(TILE) ? left : int64_t(TILE));  // multiple of 4, > 0
    uint64_t* bar = &sBar[0];
    mbar_arrive_expect_tx(bar, cnt * 40u);
    tma_load_1d(sStage + 0 * TILE * 4, T.priority + start, cnt * 4u, bar);
    tma_load_1d(sStage + 1 * TILE * 4, T.numdep + start, cnt * 4u, bar);
    tma_load_1d(sStage + 2 * TILE * 4, T.gid + start, cnt * 4u, bar);
    tma_load_1d(sStage + 3 * TILE * 4, T.flags + start, cnt * 4u, bar);
    tma_load_1d(sStage + 16 * TILE + 0 * TILE * 8, T.expected + start, cnt * 8u, bar);
    tma_load_1d(sStage + 16 * TILE + 1 * TILE * 8, T.qbasis + start, cnt * 8u, bar);
    tma_load_1d(sStage + 16 * TILE + 2 * TILE * 8, T.wbasis + start, cnt * 8u, bar);
  };
  if (tid == 0) issue(0);

  unsigned int c_dm = 0, c_mq = 0, c_over = 0, c_wait = 0, c_sec = 0, c_cnt = 0;
  int64_t s_exp = 0, s_over = 0;
  uint32_t vmn = 0xFFFFFFFFu, vmx = 0u;  // this thread's view of the value range (single tasks here, groups in phase 3)
  bool punt = false;
  const int64_t threshold = cfg.target_time_ns;
  const PlannerFactors pf = clamp_factors(cfg);
  const Factors32 f32 = factors32(pf, now);
  // since(now, wb) > threshold  <=>  wb < now - threshold whenever 0 <= threshold <= now (see k_plan_smem)
  const bool sane_clock = threshold >= 0 && now >= threshold;
  const int64_t wait_cutoff = wsub(now, threshold);
  const bool fast_clock = now >= 0 && pf.nd_int != 0;
  const bool incl = cfg.includes_dependencies != 0;
  // int64(NumDependentsFactor * n) for n < kNdTable: the 32-bit scorer then takes fractional factors too
  if (tid < kNdTable) {
    const int64_t e = nd_table_entry(pf, tid);
    sNd[tid] = (e >= 0 && e < int64_t(kNdTermLimit)) ? uint32_t(e) : 0xFFFFFFFFu;
  }
  __syncthreads();

  const uint32_t a_full = smem_u32(&sBar[0]), a_empty = smem_u32(&sBar[2]);
  const uint32_t opaque_zero = uint32_t(t_pad) & 3u;  // 0 at run time, unknown at compile time
  // Work list of task-group tasks: warp w owns entries [w*kSeg, (w+1)*kSeg) through every later phase.  Tile slots are dealt
  // to warps 32 tasks at a time, so the stretches fill evenly; one that overflows hands the distro to k_plan_smem.
  constexpr int kSeg = kListCap / NW;
  const int wl0 = warp * kSeg;
  const unsigned lt_mask = (1u << lane) - 1u;
  unsigned int wl_n = 0;
  const uint32_t* st32 = reinterpret_cast<const uint32_t*>(sStage) + tid;
  const int64_t* st64 = reinterpret_cast<const int64_t*>(sStage + 16 * TILE) + tid;
  for (int k = 0; k < n_tiles; k++) {
    const uint32_t ph = uint32_t(k) & 1u;
    mbar_wait_a(a_full, ph);  // the tile's bytes have landed
    int32_t prio[TPT], nd[TPT], gid[TPT];
    uint32_t fl[TPT];
    int64_t exp_ns[TPT], qb[TPT], wb[TPT];
#pragma unroll
    for (int u = 0; u < TPT; u++) {  // slot tid + u*THREADS of the tile is this thread's u-th task
      prio[u] = int32_t(st32[0 * TILE + u * THREADS]); nd[u] = int32_t(st32[1 * TILE + u * THREADS]);
      gid[u] = int32_t(st32[2 * TILE + u * THREADS]); fl[u] = st32[3 * TILE + u * THREADS];
      exp_ns[u] = st64[0 * TILE + u * THREADS]; qb[u] = st64[1 * TILE + u * THREADS]; wb[u] = st64[2 * TILE + u * THREADS];
    }
    // Release the slot as soon as every field IS in registers, so that it refills while this tile is scored.  "Is" needs
    // care: LDS completes asynchronously and neither program order nor the arrive's release semantics hold the arrive
    // back until the loads have actually read shared memory (without this, a rare warp scored the NEXT tile's bytes).
    // So the arrive's address is made data-dependent on every loaded register -- an AND with a zero the
    // compiler cannot prove (t_pad is a multiple of four) -- which waits on the loads' scoreboard and nothing else.
    {
      uint32_t acc = 0;
#pragma unroll
      for (int u = 0; u < TPT; u++)
        acc ^= uint32_t(prio[u]) ^ uint32_t(nd[u]) ^ uint32_t(gid[u]) ^ fl[u] ^ uint32_t(uint64_t(exp_ns[u])) ^ uint32_t(uint64_t(exp_ns[u]) >> 32) ^
               uint32_t(uint64_t(qb[u])) ^ uint32_t(uint64_t(qb[u]) >> 32) ^ uint32_t(uint64_t(wb[u])) ^ uint32_t(uint64_t(wb[u]) >> 32);
      mbar_arrive_a(a_empty + (acc & opaque_zero));
    }
    if (tid == 0 && k + 1 < n_tiles) { mbar_wait_a(a_empty, ph); issue(k + 1); }
    int idx[TPT];
    bool complex_task[TPT], scores[TPT];
    uint32_t nd_term[TPT];
    bool dom = true;
    // Straight-line on purpose: & and | on bools instead of && and ||, selects instead of guarded adds -- the
    // short-circuit forms compile to a branch (BSSY/BRA/BSYNC) per operator, which was a fifth of this loop.
#pragma unroll
    for (int u = 0; u < TPT; u++) {
      const int i = k * TILE + u * THREADS + tid - off0;
      idx[u] = i;
      const bool valid = (i >= 0) & (i < tn);
      // GetDistroQueueInfo (scheduler.go:66-138)
      const bool dm = valid & ((fl[u] & EVG_TF_DEPS_MET) != 0);
      const bool counted = valid & (!incl | dm);
      const bool over = counted & (exp_ns[u] > threshold);
      const bool waited = sane_clock ? (wb[u] < wait_cutoff) : (since(now, wb[u]) > threshold);  // sane_clock is CTA-uniform
      const bool wait_over = counted & dm & waited;
      const bool mq_dm = dm & ((fl[u] & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE);
      c_dm += dm; c_mq += mq_dm; c_over += over; c_wait += wait_over; c_sec += valid & ((fl[u] & EVG_TF_OTHER_DISTRO) != 0);
      c_cnt += counted;
      s_exp += counted ? exp_ns[u] : 0;
      s_over += over ? exp_ns[u] : 0;
      complex_task[u] = valid & (gid[u] >= 0);  // a task-group task: its unit has other members (no GroupVersions, no edges here)
      scores[u] = valid & (gid[u] < 0);         // unit == {this task}
      // the 32-bit scorer's domain (score32_domain_nd + the tabulated NumDependents term), branch-free
      const uint32_t ndc = uint32_t(nd[u] > 0 ? nd[u] : 0);
      const uint32_t tab = sNd[ndc < uint32_t(kNdTable) ? ndc : 0u];
      const uint32_t mul = (f32.ok & (ndc < kTask32Limit)) ? f32.nd * ndc : 0xFFFFFFFFu;
      nd_term[u] = ndc < uint32_t(kNdTable) ? tab : mul;
      const uint32_t bad = score32_bad(now, prio[u], exp_ns[u], qb[u], nd_term[u]);  // the 32-bit scorer's domain, branch-free
      dom = dom & (!scores[u] | (bad == 0u));
    }
    uint64_t v[TPT];
    if (f32.ok_base && __all_sync(full, dom)) {
#pragma unroll
      for (int u = 0; u < TPT; u++) v[u] = single_task_value32_nd(f32, now, prio[u], exp_ns[u], qb[u], nd_term[u], fl[u]);
    } else {
#pragma unroll
      for (int u = 0; u < TPT; u++) v[u] = score_slow(pf, fast_clock, scores[u], now, prio[u], exp_ns[u], qb[u], nd[u], fl[u]);
    }
#pragma unroll
    for (int u = 0; u < TPT; u++) {
      if (scores[u]) {
        if (v[u] >> 32) punt = true;  // does not fit the u32 key (negative values included): k_plan_smem plans this distro
        const uint32_t v32 = uint32_t(v[u]);
        sKey[idx[u]] = v32;
        vmn = min(vmn, v32); vmx = max(vmx, v32);
      }
      if (any) {  // the warp's own stretch of the work list: no atomic, the count stays in a (warp-uniform) register
        const unsigned m = __ballot_sync(full, complex_task[u]);
        const unsigned int pos = wl_n + __popc(m & lt_mask);
        if (complex_task[u] && pos < (unsigned)kSeg) sList[wl0 + pos] = uint16_t(idx[u]);
        wl_n += __popc(m);
      }
    }
  }
  // fold the queue-info partials: warp shuffle, then shared atomics
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
    if ((__any_sync(full, punt) || wl_n > (unsigned)kSeg) && lane == 0) S->punt = 1;  // a value outside u32, or more task-group tasks than the warp's stretch holds
  }
  __syncthreads();
  const int wl_cnt = int(wl_n);

  // ---- task groups: per-group accumulators in the (now idle) staging area ----
  unsigned long long* gTiq = reinterpret_cast<unsigned long long*>(smem_raw + L::kOffIdx);
  unsigned long long* gRt = gTiq + kGroupCap;
  unsigned long long* gMask = gRt + kGroupCap;
  unsigned long long* qExp = gMask + kGroupCap;
  unsigned long long* qDurOver = qExp + kGroupCap;
  int* gMaxP = reinterpret_cast<int*>(qDurOver + kGroupCap);
  int* gMaxD = gMaxP + kGroupCap;
  unsigned int* gFlags = reinterpret_cast<unsigned int*>(gMaxD + kGroupCap);
  unsigned int* gN = gFlags + kGroupCap;
  unsigned int* gAnchor = gN + kGroupCap;
  unsigned int* gV = gAnchor + kGroupCap;
  unsigned int* qCnt = gV + kGroupCap;
  unsigned int* qOver = qCnt + kGroupCap;
  unsigned int* qWait = qOver + kGroupCap;
  unsigned int* qMq = qWait + kGroupCap;  // 5*8 + 11*4 = 84 bytes per group

  if (any) {
    // ---- phase 2b: task-group sums (scheduler.go:79-137) and Unit.info (planner.go:302-337), member by member ----
    for (int g = tid; g < ng; g += THREADS) {
      gTiq[g] = 0ull; gRt[g] = 0ull; gMask[g] = 0ull; gMaxP[g] = 0; gMaxD[g] = 0; gFlags[g] = 0u; gN[g] = 0u;
      gAnchor[g] = kNoAnchor; gV[g] = 0u;
      qExp[g] = 0ull; qDurOver[g] = 0ull; qCnt[g] = 0u; qOver[g] = 0u; qWait[g] = 0u; qMq[g] = 0u;
    }
    __syncthreads();
    if (S->punt) {  // uniform: set before the barrier above
      if (tid == 0) punt_list[atomicAdd(punt_count, 1)] = d;
      return;
    }
    unsigned int t_n = 0, t_cnt = 0, t_over = 0, t_wait = 0, t_mq = 0;
    int64_t t_exp = 0, t_dover = 0;
    struct Member { int i; int32_t gid, tgo, prio, nd; uint32_t fl; int64_t exp_ns, wb, qb; };
    auto fetch = [&](int k) {  // every column this phase needs, requested together: one L2 round trip, not a chain
      Member m;
      m.i = int(sList[k]);
      const int64_t t = base + m.i;
      m.gid = T.gid[t]; m.exp_ns = T.expected[t]; m.wb = T.wbasis[t]; m.qb = T.qbasis[t];
      m.fl = T.flags[t]; m.tgo = T.tgo[t]; m.prio = T.priority[t]; m.nd = T.numdep[t];
      return m;
    };
    auto member = [&](const Member& m) {
      const int i = m.i;
      const int32_t gid = m.gid, tgo = m.tgo, prio = m.prio, nd = m.nd;
      const uint32_t fl = m.fl;
      const int64_t exp_ns = m.exp_ns, wb = m.wb, qb = m.qb;
      const bool dm = (fl & EVG_TF_DEPS_MET) != 0;
      const bool counted = !incl || dm;
      const bool over = counted && exp_ns > threshold;
      const bool wait_over = counted && dm && since(now, wb) > threshold;
      const bool mq_dm = dm && (fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE;
      t_n += 1; t_cnt += counted; t_over += over; t_wait += wait_over; t_mq += mq_dm;
      if (counted) t_exp += exp_ns;
      if (over) t_dover += exp_ns;
      if (counted) { atomicAdd(&qCnt[gid], 1u); smem_add64(&qExp[gid], (unsigned long long)exp_ns); }
      if (over) { atomicAdd(&qOver[gid], 1u); smem_add64(&qDurOver[gid], (unsigned long long)exp_ns); }
      if (wait_over) atomicAdd(&qWait[gid], 1u);
      if (mq_dm) atomicAdd(&qMq[gid], 1u);
      if (tgo < 0 || tgo >= 64) { S->punt = 1; return; }  // the presence-mask rank needs orders 0..63
      sKey[i] = uint32_t(gid) | (uint32_t(tgo) << 16);  // parked for phase 4
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
      atomicOr(reinterpret_cast<unsigned int*>(&gMask[gid]) + (tgo >> 5), 1u << (tgo & 31));
    };
    for (int k = lane; k < wl_cnt; k += 64) {  // two members per trip: sixteen loads in flight
      const bool two = k + 32 < wl_cnt;
      const Member m0 = fetch(wl0 + k);
      const Member m1 = fetch(wl0 + (two ? k + 32 : k));
      member(m0);
      if (two) member(m1);
    }
    if (__any_sync(full, t_n != 0)) {  // one shared atomic per warp and field
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
    // ---- phase 3: TaskGroupInfo rows out, one unit_value per group (planner.go:209-300) ----
    for (int g = tid; g < ng; g += THREADS) {
      evg_group_info gi;
      gi.count = qCnt[g]; gi.count_free = 0; gi.count_required = 0; gi.max_hosts = D.gmax[D.group_off[d] + g];
      gi.expected_duration = int64_t(qExp[g]);
      gi.count_duration_over_threshold = qOver[g];
      gi.count_wait_over_threshold = qWait[g];
      gi.count_dep_filled_merge_queue_tasks = qMq[g];
      gi.duration_over_threshold = int64_t(qDurOver[g]);
      W.ginfo[D.group_off[d] + g] = gi;
      if (gN[g] != uint32_t(__popcll(gMask[g]))) { S->punt = 1; continue; }  // duplicate TaskGroupOrder inside the group
      if (gN[g] == 0) continue;
      UnitAcc a;
      a.tiq = int64_t(gTiq[g]); a.rt = int64_t(gRt[g]); a.max_p = gMaxP[g]; a.max_d = gMaxD[g];
      a.n = gN[g]; a.flags = gFlags[g];
      const uint64_t v = uint64_t(unit_value(a, cfg, nullptr));
      if (v >> 32) { S->punt = 1; continue; }
      gV[g] = uint32_t(v);
      vmn = min(vmn, uint32_t(v)); vmx = max(vmx, uint32_t(v));
    }
    __syncthreads();
    if (S->punt) {
      if (tid == 0) punt_list[atomicAdd(punt_count, 1)] = d;
      return;
    }
    // ---- phase 4: a task-group task is emitted from its group's unit, ranked by its order ----
    for (int kk = lane; kk < wl_cnt; kk += 32) {
      const int k = wl0 + kk;
      const int i = int(sList[k]);
      const uint32_t packed = sKey[i];
      const uint32_t gid = packed & 0xFFFFu;
      const uint32_t brk = __popcll(gMask[gid] & ((1ull << (packed >> 16)) - 1ull));
      const uint32_t ba = gAnchor[gid];
      sKey[i] = gV[gid];
      sLA[k] = uint16_t(ba);
      sLR[k] = uint16_t(brk);
      if (!(ba == uint32_t(i) && brk == 0)) { atomicOr(&sDisp[i >> 5], 1u << (i & 31)); S->n_displaced = 1; }
    }
  } else if (S->punt) {  // uniform: published by the barrier after the fold
    if (tid == 0) punt_list[atomicAdd(punt_count, 1)] = d;
    return;
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
  vmn = __reduce_min_sync(full, vmn);
  vmx = __reduce_max_sync(full, vmx);
  if (lane == 0) { atomicMin(&S->vmin, vmn); atomicMax(&S->vmax, vmx); }
  __syncthreads();  // closes phase 4 as well: sDisp, n_displaced, the keys of task-group tasks
  const uint32_t vmax = S->vmax;
  const uint32_t range = tn > 0 ? vmax - S->vmin : 0u;
  const int bits = range == 0 ? 0 : 32 - __clz(int(range));

  // ---- phase 6: canonical pre-arrangement (ties: unit anchor asc, rank in unit asc) ----
  // e[a] = tasks emitted under anchor a; the exclusive scan of e is where anchor a's run starts.  A task that keeps
  // its own anchor with rank 0 (every single task, the first member of a group) counts itself; displaced ones are
  // added by the work list.  ITEMS consecutive entries per thread.
  const int j0 = tid * ITEMS;
  if (any && S->n_displaced != 0) {
    uint16_t* sE = reinterpret_cast<uint16_t*>(sCnt);
    uint32_t* e32 = sCnt;
#pragma unroll
    for (int k = 0; k < ITEMS; k += 2) {
      const int j = j0 + k;
      const uint32_t w = sDisp[j >> 5];  // j even: j and j+1 share the word
      const uint32_t lo = (j < tn && !((w >> (j & 31)) & 1u)) ? 1u : 0u;
      const uint32_t hi = (j + 1 < tn && !((w >> ((j + 1) & 31)) & 1u)) ? 1u : 0u;
      e32[j >> 1] = lo | (hi << 16);
    }
    __syncthreads();
    for (int kk = lane; kk < wl_cnt; kk += 32) {
      const int k = wl0 + kk;
      const int i = int(sList[k]);
      if (!((sDisp[i >> 5] >> (i & 31)) & 1u)) continue;
      const uint32_t a = sLA[k];
      atomicAdd(&e32[a >> 1], 1u << (16 * (a & 1)));
    }
    __syncthreads();
    uint32_t loc[ITEMS];
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < ITEMS; k += 2) {
      const uint32_t w = e32[(j0 + k) >> 1];
      loc[k] = w & 0xFFFFu; loc[k + 1] = w >> 16;
      sum += loc[k] + loc[k + 1];
    }
    uint32_t run = block_scan_excl<NW>(sum, sScan);
#pragma unroll
    for (int k = 0; k < ITEMS; k += 2) {
      const int j = j0 + k;
      const uint32_t w = sDisp[j >> 5];
      const uint32_t p0 = run, p1 = run + loc[k];
      e32[j >> 1] = p0 | (p1 << 16);  // positions stay below CAP <= 16384
      if (j < tn && !((w >> (j & 31)) & 1u)) sIdx[p0] = uint16_t(j);          // rank 0 under its own anchor
      if (j + 1 < tn && !((w >> ((j + 1) & 31)) & 1u)) sIdx[p1] = uint16_t(j + 1);
      run = p1 + loc[k + 1];
    }
    __syncthreads();
    for (int kk = lane; kk < wl_cnt; kk += 32) {
      const int k = wl0 + kk;
      const int i = int(sList[k]);
      if (!((sDisp[i >> 5] >> (i & 31)) & 1u)) continue;
      // every member of a task-group unit is emitted from it, so the rank inside the unit is the offset in the run
      sIdx[uint32_t(sE[sLA[k]]) + uint32_t(sLR[k])] = uint16_t(i);
    }
  } else {
#pragma unroll
    for (int k = 0; k < ITEMS; k += 2) {
      const int j = j0 + k;
      reinterpret_cast<uint32_t*>(sIdx)[j >> 1] = uint32_t(j) | (uint32_t(j + 1) << 16);
    }
  }
  __syncthreads();

  // ---- phase 8: stable LSD radix sort of the permutation by key = vmax - V, digits of up to MAXBITS bits ----
  // Warp w owns positions [seg0, seg1); it ranks them chunk by chunk (32 at a time, in order: stability).  One
  // MATCH.ANY per chunk gives each element its rank among the chunk's equal digits; the group's first lane adds the
  // group size to the warp's counter and the value the atomic returns is the number of equal digits in the warp's
  // earlier chunks.  After the block-wide scan of the counters an element's position is base[warp][digit] + that
  // warp-local rank.  Elements wait in registers between the two steps, so the permutation is scattered in place.
  {
    const int seg = ((tn + NW - 1) / NW + 31) & ~31;
    const int seg0 = warp * seg;
    const int seg1 = min(seg0 + seg, tn);
    const bool full_seg = seg1 - seg0 == ITEMS * 32;  // warp-uniform: every lane of every chunk holds an element
    const unsigned lt = (1u << lane) - 1u;
    const int npass = (bits + MAXBITS - 1) / MAXBITS;
    const int wbase = npass ? bits / npass : 0, wrem = npass ? bits % npass : 0;
    uint32_t* wc = sCnt + warp * DW;
    int shift = 0;
    for (int pass = 0; pass < npass; pass++) {
      const int wbits = wbase + (pass < wrem ? 1 : 0);
      const uint32_t nd = 1u << wbits, mask = nd - 1u;
      for (uint32_t x = lane; x < (nd + 1) / 2; x += 32) wc[x] = 0u;
      __syncwarp();
      uint32_t ci[ITEMS];  // task index of the element at chunk j
      uint32_t cr[ITEMS];  // its digit | warp-local rank << 10
      // FULL: no per-element bounds (15 of 16 warps of a 10k-task distro); otherwise padding lanes carry digit 0x7FFF
      // and match only each other.  All permutation loads first, then all key gathers (independent shared-memory
      // loads in flight together), only then the MATCH / atomic / shuffle chain, which must run chunk by chunk.
      auto rank = [&](auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          const int p = seg0 + j * 32 + lane;
          ci[j] = (FULL || p < seg1) ? uint32_t(sIdx[p]) : 0u;
        }
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          const uint32_t dg = ((vmax - sKey[ci[j]]) >> shift) & mask;
          cr[j] = (FULL || seg0 + j * 32 + lane < seg1) ? dg : 0x7FFFu;
        }
        // RB chunks per trip: their MATCHes, then their leader atomics (issued back to back -- one warp's shared-memory
        // atomics execute in order, so chunk j+1's returned count includes chunk j's add), then their shuffles.  The
        // returns are first needed by the shuffles, so RB atomic round trips overlap instead of queueing behind each other
        // (the single-chunk form waits on that one dependent chain per chunk).
        constexpr int RB = 1;  // one chunk per trip: with more, the extra live registers spill
#pragma unroll
        for (int j0 = 0; j0 < ITEMS; j0 += RB) {
          unsigned peers[RB];
          uint32_t old[RB];
#pragma unroll
          for (int b = 0; b < RB; b++) peers[b] = (FULL || seg0 + (j0 + b) * 32 < seg1) ? __match_any_sync(full, cr[j0 + b]) : 0u;
#pragma unroll
          for (int b = 0; b < RB; b++) {
            const uint32_t dg = cr[j0 + b];
            old[b] = 0;
            if ((FULL || seg0 + (j0 + b) * 32 < seg1) && (peers[b] & lt) == 0u && (FULL || dg != 0x7FFFu))
              old[b] = atomicAdd(&wc[dg >> 1], uint32_t(__popc(peers[b])) << ((dg & 1u) << 4));
          }
#pragma unroll
          for (int b = 0; b < RB; b++) {
            if (FULL || seg0 + (j0 + b) * 32 < seg1) {  // warp-uniform
              const uint32_t dg = cr[j0 + b];
              const uint32_t o = __shfl_sync(full, old[b], __ffs(peers[b]) - 1);
              cr[j0 + b] = (dg & 0x3FFu) | ((((o >> ((dg & 1u) << 4)) & 0xFFFFu) + uint32_t(__popc(peers[b] & lt))) << 10);
            }
          }
        }
      };
      if (full_seg) rank(std::true_type{}); else rank(std::false_type{});
      __syncthreads();
      {  // block-wide scan: thread t owns digits 2t and 2t+1 (one u32 of every warp's row)
        uint32_t tot = 0;
        const bool act = uint32_t(2 * tid) < nd;
        if (act) {
#pragma unroll
          for (int w = 0; w < NW; w++) tot += sCnt[w * DW + tid];  // packed halves never carry: totals <= CAP
        }
        const uint32_t t0 = tot & 0xFFFFu, t1 = tot >> 16;
        const uint32_t ex = block_scan_excl<NW>(t0 + t1, sScan);
        uint32_t run = ex | ((ex + t0) << 16);
        if (act) {
#pragma unroll
          for (int w = 0; w < NW; w++) { const uint32_t x = sCnt[w * DW + tid]; sCnt[w * DW + tid] = run; run += x; }
        }
      }
      __syncthreads();
      auto scatter = [&](auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
          if (FULL || seg0 + j * 32 + lane < seg1) {
            const uint32_t dg = cr[j] & 0x3FFu, wr = cr[j] >> 10;
            const uint32_t bs = (wc[dg >> 1] >> ((dg & 1u) << 4)) & 0xFFFFu;
            sIdx[bs + wr] = uint16_t(ci[j]);
          }
        }
      };
      if (full_seg) scatter(std::true_type{}); else scatter(std::false_type{});
      __syncthreads();
      shift += wbits;
    }
  }

  // ---- phase 9: ranked queue out (coalesced) ----
  for (int p = tid; p < tn; p += THREADS) {
    const uint32_t i = sIdx[p];
    order[base + p] = int32_t(i);
    total_value[base + p] = int64_t(uint64_t(sKey[i]));
  }
}
