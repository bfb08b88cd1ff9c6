// evg_plan_general.cuh -- the general path: distros too large for one CTA (any size up to 2^21-1 tasks).
//
// Second generation.  The first one sorted a 64-bit value word plus a 42-bit tie word per task with a 16-pass
// segmented LSD radix sort (20 B/task each way per pass).  This one:
//   k_gtask        per 2048-task tile: 128-bit column loads, 32-bit scoring (single_task_value32) where the
//                  distro allows it, queue-info sums folded per tile, TotalValue of single-task units, per-distro
//                  value range; tasks of multi-member units are compacted into a work list of packed entries (unit
//                  slots + member payload, written from registers)
//   k_glink/k_galloc/k_gfill  the unit table: every membership draws its place in its unit's run of entry ids
//   k_gunit/k_grank  per unit: Unit.info / value / anchor, and every member's rank in the unit, once
//   k_gbest        per work-list task: its first-occurrence choice (planner.go:467-477) and that unit's rank of it;
//                  anchor histogram e[]
//   k_gsum/k_gscan/k_gplace
//                  canonical pre-arrangement by COUNTING instead of sorting tie bytes: an exclusive scan of e[] per tile
//                  (k_gsum) and of the tile totals per distro (k_gscan) gives every anchor's run start; tasks are
//                  written to (key, index) buffers in (anchor, rank-in-unit) order by one kernel, k_gplace, a block per
//                  tile: the tile's tasks emitted from their own single-task unit and the tasks of the small units
//                  anchored in it, then a share of the large units, a warp each.  The writers touch disjoint slots and
//                  write only those.  Distros without multi-member units skip the scans (identity).
//   k_ghist/k_gdscan/k_gscatter
//                  stable LSD radix sort on key = Vmax - V only: 32-bit keys, ceil(bits(Vmax-Vmin)/8) passes (3 for
//                  a 20-bit range), 8 B/task each way per pass; a distro whose range exceeds 32 bits carries a
//                  second key word and up to 8 passes (per-distro branch, same kernels); a distro's last pass writes
//                  the ranked queue and TotalValue instead of keys
// TotalValue per task is parked in the total_value OUTPUT buffer between k_gtask and k_gplace (no 8 B/task scratch); the
// last radix pass overwrites it with TotalValue by rank.
//
// Reference: scheduler/planner.go:209-481, scheduler/scheduler.go:56-159.
#pragma once

constexpr int kGTile = 2048;  // tasks per tile; tiles start at multiples of 4 tasks (16-byte aligned vector loads)

struct DGen {
  // tiles of the general-path distros, in distro order
  int64_t n_tiles;
  int64_t tile0;               // first tile this launch covers (a chunk of the pipelined one-shot call); grids are relative to it
  const int32_t* tile_distro;  // [NT]
  const int64_t* tile_start;   // [NT] first task slot of the tile: (base & ~3) + k*kGTile, may precede the distro by <= 3
  const int64_t* dtile_off;    // [D+1]
  unsigned long long* vmm;     // [D*2] ord(Vmax), ord(Vmin)
  uint32_t* key_lo[2];         // [T] low word of Vmax - V, in sort position
  uint32_t* key_hi[2];         // [T] high word (distros with a range above 32 bits only)
  uint32_t* idx[2];            // [T] distro-local task index, in sort position
  uint32_t* e;                 // [T] anchor histogram, then (k_gsum) the offset of the anchor's run inside its tile's
                               //     stretch; the run starts at tile_sum[tile] + e in the distro (gen_run_start)
  uint32_t* tile_sum;          // [NT] sum of e over the tile, then the tile's exclusive offset inside its distro
  uint32_t* tile_hist;         // [NT*256]
  uint4* wl;                   // work list, one entry per task that touches a multi-member unit: x = global task index,
                               //     y = distro, z = global slot of its own-key unit (kInactive: not a member of it),
                               //     w = global slot of its version unit (kInactive: none); k_gfill replaces both slots
                               //     with the units' ids
  struct URec* pay;            // [work list] the entry's member payload (what k_gunit and k_gbest ask of a member)
  unsigned int* ccount;        // [1] work-list entries
  int32_t* maxpass;            // [1]
  uint32_t* run;               // unit table: the members of every multi-member unit as work-list entry ids (bit 31: an
                               //     own-key membership), one contiguous run per unit
  uint32_t* pown;              // [work list] place of the entry's own-key membership in its unit's run
  uint32_t* pver;              // [work list] place of its version membership
  uint32_t* pedge;             // [E] place of the edge's dependency membership
  uint32_t* sedge;             // [E] unit slot of that membership (kInactive: the task already joined that unit); k_gfill
                               //     replaces it with the unit's id
  uint32_t* rank;              // [run positions] the member's rank inside its unit (TaskList.Less)
  uint32_t* emit;              // [run positions] by rank: emit[start + r] = distro-local index of the unit's rank-r member
                               //     if the unit emits it (k_gbest), else kInactive (k_gunit / k_grank reset it per tick)
  unsigned int* rcount;        // [1] run positions reserved
  uint2* blist;                // units above kRankOne members, in 32-member chunks: x = id, y = chunk (k_grank ranks them)
  unsigned int* bcount;        // [1]
  struct GUnit* unit;          // [units] the multi-member units of the tick by dense id (k_galloc numbers them)
  unsigned int* hcount;        // [1] units numbered
  int64_t* tv;                 // [T] TotalValue by task (the output buffer, reused)
};

__device__ __forceinline__ int gen_bits(const DGen& G, int d) {  // significant bits of Vmax - Vmin
  const unsigned long long r = G.vmm[2 * d] - G.vmm[2 * d + 1];
  return r == 0 ? 0 : 64 - __clzll((long long)r);
}
// at least one: the last pass writes the ranked queue, so a distro of width 0 takes one pass too
__device__ __forceinline__ int gen_npass(int bits) { return bits ? (bits + 7) >> 3 : 1; }

// A work-list entry's member payload: the fields Unit.info, the in-unit order and TaskGroupInfo need.
struct __align__(16) URec {
  int32_t prio, nd;
  int64_t exp_ns, qb;
  int32_t tgo;
  uint32_t lif;  // bits 0..20 distro-local task index, 22 group_id >= 0, 23 wait over threshold (k_gtask's verdict),
                 // 24..29 task flags
};
static_assert(sizeof(URec) == 32, "one L2 sector per member");
constexpr uint32_t kRecGrouped = 1u << 22, kRecWaitOver = 1u << 23;
constexpr uint32_t kRunOwn = 1u << 31, kRunEntry = kRunOwn - 1u;  // a run position: entry id | own-key membership
__device__ __forceinline__ uint32_t rec_li(const URec& r) { return r.lif & 0x1FFFFFu; }
__device__ __forceinline__ URec rec_load(const URec* p) {  // two 128-bit loads
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  URec r;
  r.prio = int32_t(a.x); r.nd = int32_t(a.y); r.exp_ns = int64_t((unsigned long long)a.z | ((unsigned long long)a.w << 32));
  r.qb = int64_t((unsigned long long)b.x | ((unsigned long long)b.y << 32)); r.tgo = int32_t(b.z); r.lif = b.w;
  return r;
}
__device__ __forceinline__ void rec_store(URec* p, const URec& r) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(uint32_t(r.prio), uint32_t(r.nd), uint32_t(uint64_t(r.exp_ns)), uint32_t(uint64_t(r.exp_ns) >> 32));
  reinterpret_cast<uint4*>(p)[1] = make_uint4(uint32_t(uint64_t(r.qb)), uint32_t(uint64_t(r.qb) >> 32), uint32_t(r.tgo), r.lif);
}

// A multi-member unit: everything the kernels after k_gfill ask of it, in one sector.  Units are numbered densely: the
// ~10 000 units of a 100 000-task distro take ~0.3 MB of L2, where fields indexed by its ~100 000 unit slots spread over
// megabytes and fell out of L2 between the blocks of one grid-wide kernel.
struct __align__(16) GUnit {
  int64_t value;    // TotalValue (k_gunit)
  uint32_t anchor;  // kNoAnchor: the unit never got a distro, it is not exported (planner.go:81-83) (k_gunit)
  uint32_t n;       // members (k_galloc)
  uint32_t start;   // its run: run[start .. start + n), and its ranks: emit[start .. start + n) (k_galloc)
  int32_t d;        // distro (k_galloc)
  uint32_t spare[2];  // unused: keeps the record one sector (written as zero)
};
static_assert(sizeof(GUnit) == 32, "one L2 sector per unit");
__device__ __forceinline__ GUnit unit_load(const GUnit* p) {  // two 128-bit loads of one sector
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  GUnit u;
  u.value = int64_t((unsigned long long)a.x | ((unsigned long long)a.y << 32)); u.anchor = a.z; u.n = a.w;
  u.start = b.x; u.d = int32_t(b.y); u.spare[0] = u.spare[1] = 0u;
  return u;
}
__device__ __forceinline__ void unit_store(GUnit* p, const GUnit& u) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(uint32_t(uint64_t(u.value)), uint32_t(uint64_t(u.value) >> 32), u.anchor, u.n);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(u.start, uint32_t(u.d), 0u, 0u);
}
// The slot map of the general path: k_galloc files a unit's id and run start under its slot, in the on-chip planners'
// unit_v (no general-path slot is an on-chip one), so that k_gfill finds both with one load (and k_gplace the id of the
// unit a task anchors, under its own-key slot).
__device__ __forceinline__ int64_t slot_unit(uint32_t id, uint32_t start) { return int64_t(uint64_t(id) | (uint64_t(start) << 32)); }

__global__ void k_ginit(DGen G, const int32_t* __restrict__ general_list, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0) { *G.ccount = 0u; *G.maxpass = 0; *G.rcount = 0u; *G.hcount = 0u; *G.bcount = 0u; }
  if (k >= n) return;
  const int d = general_list[k];
  G.vmm[2 * d] = 0ull;
  G.vmm[2 * d + 1] = ~0ull;
}

// planner.go:449-456 (pass 2): mark every task some in-queue task depends on (general-path distros only).
__global__ void __launch_bounds__(256) k_gmark(DTasks T, DDistros D, DWork W, DGen G) {
  if (*W.err) return;
  const int tile = int(blockIdx.x + G.tile0);
  const int d = G.tile_distro[tile];
  const int64_t base = D.task_off[d], end = D.task_off[d + 1];
  const int64_t lo = max(G.tile_start[tile], base), hi = min(G.tile_start[tile] + kGTile, end);
  for (int64_t t = lo + threadIdx.x; t < hi; t += 256)
    for (int64_t e = T.dep_off[t]; e < T.dep_off[t + 1]; e++) W.has_dep[base + T.dep_idx[e]] = 1;
}

struct TileFold {  // queue-info partials of one tile (scheduler.go:66-138)
  unsigned int c[10];
  unsigned long long s[4];
  unsigned long long vmax, vmin;
};

// Per tile: queue info, single-task scores, unit links.  256 threads x 8 tasks: thread q of group u owns the four
// consecutive task slots tile_start + 4*(u*256 + q) .. +3, so every column is read with 128-bit loads.
// 2 blocks of 256 per SM: k_gtask fits its registers without spilling on sm_90a (at 3 it spills ~200 B a thread);
// on H100 that took the kernel from 0.17 to 0.135 ms on 48 distros x 100 000 tasks of configs[2]'s mix
constexpr int kGTaskOcc = 2;
__global__ void __launch_bounds__(256, kGTaskOcc) k_gtask(DTasks T, DDistros D, DWork W, DGen G, int64_t now, int any_complex) {
  if (*W.err) return;
  __shared__ TileFold F;
  __shared__ evg_distro_cfg s_cfg;
  __shared__ uint32_t s_nd[kNdTable];  // int64(NumDependentsFactor * n), n < kNdTable: fractional factors stay on the 32-bit scorer
  const int tile = int(blockIdx.x + G.tile0);
  const int d = G.tile_distro[tile];
  const int tid = threadIdx.x, lane = tid & 31;
  const unsigned full = 0xffffffffu;
  if (tid == 0) {
    for (int k = 0; k < 10; k++) F.c[k] = 0;
    for (int k = 0; k < 4; k++) F.s[k] = 0;
    F.vmax = 0ull; F.vmin = ~0ull;
    s_cfg = D.cfg[d];
  }
  __syncthreads();
  const evg_distro_cfg& cfg = s_cfg;
  const int64_t base = D.task_off[d], end = D.task_off[d + 1];
  const int64_t ts = G.tile_start[tile];
  const uint32_t ng = uint32_t(D.group_off[d + 1] - D.group_off[d]);
  const uint32_t ub = uint32_t(D.unit_base[d]);
  const bool gv = cfg.group_versions != 0;
  const int64_t threshold = cfg.target_time_ns;
  const PlannerFactors pf = clamp_factors(cfg);
  const Factors32 f32 = factors32(pf, now);
  const bool sane_clock = threshold >= 0 && now >= threshold;
  const int64_t wait_cutoff = wsub(now, threshold);
  const bool fast_clock = now >= 0 && pf.nd_int != 0;
  const bool incl = cfg.includes_dependencies != 0;
  if (tid < kNdTable) {
    const int64_t e = nd_table_entry(pf, tid);
    s_nd[tid] = (e >= 0 && e < int64_t(kNdTermLimit)) ? uint32_t(e) : 0xFFFFFFFFu;
  }
  __syncthreads();
  const bool dcomplex = any_complex && (ng > 0 || gv || (T.n_edges > 0 && T.dep_off[end] > T.dep_off[base]));

  unsigned int c_dm = 0, c_mq = 0, c_over = 0, c_wait = 0, c_sec = 0, c_ung = 0, c_ucnt = 0, c_uover = 0, c_uwait = 0, c_umq = 0;
  int64_t s_exp = 0, s_over = 0, s_uexp = 0, s_uover = 0;
  unsigned long long kmax = 0ull, kmin = ~0ull;

#pragma unroll 1
  for (int u = 0; u < 2; u++) {
    const int64_t t4 = ts + 4 * int64_t(u * 256 + tid);  // multiple of 4: 16-byte aligned in every column
    const bool live = t4 < end;  // the columns are readable 8 slots past the last task (upload pads them)
    int4 prio4 = make_int4(0, 0, 0, 0), nd4 = prio4, gid4 = make_int4(-1, -1, -1, -1), tgo4 = prio4, vid4 = prio4;
    uint4 fl4 = make_uint4(0, 0, 0, 0);
    uint32_t cmask = 0, womask = 0;  // bit m: task t4 + m goes on the work list / its wait is over the threshold
    if (live && dcomplex) {  // what only the work list's payload needs
      tgo4 = *reinterpret_cast<const int4*>(T.tgo + t4);
      if (gv) vid4 = *reinterpret_cast<const int4*>(T.vid + t4);
    }
    longlong2 ex01 = make_longlong2(0, 0), ex23 = ex01, qb01 = ex01, qb23 = ex01, wb01 = ex01, wb23 = ex01;
    if (live) {
      prio4 = *reinterpret_cast<const int4*>(T.priority + t4);
      nd4 = *reinterpret_cast<const int4*>(T.numdep + t4);
      gid4 = *reinterpret_cast<const int4*>(T.gid + t4);
      fl4 = *reinterpret_cast<const uint4*>(T.flags + t4);
      ex01 = *reinterpret_cast<const longlong2*>(T.expected + t4); ex23 = *reinterpret_cast<const longlong2*>(T.expected + t4 + 2);
      qb01 = *reinterpret_cast<const longlong2*>(T.qbasis + t4); qb23 = *reinterpret_cast<const longlong2*>(T.qbasis + t4 + 2);
      wb01 = *reinterpret_cast<const longlong2*>(T.wbasis + t4); wb23 = *reinterpret_cast<const longlong2*>(T.wbasis + t4 + 2);
    }
    // dependency offsets of the four tasks (five consecutive entries) and their "has dependents" bytes, as vectors too
    int64_t doff[5] = {0, 0, 0, 0, 0};
    uint32_t hd4 = 0;
    if (live && dcomplex) {
      if (T.n_edges > 0) {
        const longlong2 d01 = *reinterpret_cast<const longlong2*>(T.dep_off + t4), d23 = *reinterpret_cast<const longlong2*>(T.dep_off + t4 + 2);
        doff[0] = d01.x; doff[1] = d01.y; doff[2] = d23.x; doff[3] = d23.y; doff[4] = T.dep_off[t4 + 4];
      }
      hd4 = *reinterpret_cast<const uint32_t*>(W.has_dep + t4);
    }
    const int32_t prio_[4] = {prio4.x, prio4.y, prio4.z, prio4.w}, nd_[4] = {nd4.x, nd4.y, nd4.z, nd4.w};
    const int32_t gid_[4] = {gid4.x, gid4.y, gid4.z, gid4.w};
    const uint32_t fl_[4] = {fl4.x, fl4.y, fl4.z, fl4.w};
    const int64_t ex_[4] = {ex01.x, ex01.y, ex23.x, ex23.y}, qb_[4] = {qb01.x, qb01.y, qb23.x, qb23.y};
    const int64_t wb_[4] = {wb01.x, wb01.y, wb23.x, wb23.y};
    int64_t vout[4];
    uint32_t eout[4], nd_term[4];
    bool wr_v[4], solo[4];
    bool dom = true;
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const int64_t t = t4 + m;
      const bool valid = live & (t >= base) & (t < end);
      const int32_t prio = prio_[m], nd = nd_[m], gid = gid_[m];
      const uint32_t fl = fl_[m];
      const int64_t exp_ns = ex_[m], qb = qb_[m], wb = wb_[m];
      // straight-line (bitwise bool operators, selects): the short-circuit forms cost a branch per operator
      const bool dm = valid & ((fl & EVG_TF_DEPS_MET) != 0);
      const bool counted = valid & (!incl | dm);
      const bool over = counted & (exp_ns > threshold);
      const bool waited = sane_clock ? (wb < wait_cutoff) : (since(now, wb) > threshold);  // sane_clock is block-uniform
      const bool wait_over = counted & dm & waited;
      const bool mq_dm = dm & ((fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE);
      const bool ung = valid & (gid < 0);
      c_dm += dm; c_mq += mq_dm; c_over += over; c_wait += wait_over; c_sec += valid & ((fl & EVG_TF_OTHER_DISTRO) != 0);
      s_exp += counted ? exp_ns : 0;
      s_over += over ? exp_ns : 0;
      c_ung += ung; c_ucnt += ung & counted; c_uover += ung & over; c_uwait += ung & wait_over; c_umq += ung & mq_dm;
      s_uexp += (ung & counted) ? exp_ns : 0;
      s_uover += (ung & over) ? exp_ns : 0;
      // membership links, dependency edges and the TaskGroupInfo sums of multi-member-unit tasks are k_glink's job:
      // pointer chasing with a few active lanes per warp would stall this streaming pass
      const bool own_complex = valid & dcomplex & ((gid >= 0) | gv | (((hd4 >> (8 * m)) & 0xFFu) != 0));
      const bool complex_task = own_complex | (valid & dcomplex & (doff[m + 1] > doff[m]));
      const bool scores = valid & !own_complex;  // the unit filed under this task's own key is {this task}
      const uint32_t ndc = uint32_t(nd > 0 ? nd : 0);
      const uint32_t tab = s_nd[ndc < uint32_t(kNdTable) ? ndc : 0u];
      const uint32_t mul = (f32.ok & (ndc < kTask32Limit)) ? f32.nd * ndc : 0xFFFFFFFFu;
      nd_term[m] = ndc < uint32_t(kNdTable) ? tab : mul;
      dom = dom & (!scores | (score32_bad(now, prio, exp_ns, qb, nd_term[m]) == 0u));
      wr_v[m] = scores;
      solo[m] = scores & !complex_task;  // final: the task is emitted from its own unit
      eout[m] = (valid & !complex_task) ? 1u : 0u;
      cmask |= (complex_task ? 1u : 0u) << m;
      womask |= (wait_over ? 1u : 0u) << m;
    }
    if (f32.ok_base && __all_sync(full, dom)) {  // one warp vote per four tasks; the 64-bit scorers stay out of line
#pragma unroll
      for (int m = 0; m < 4; m++) vout[m] = int64_t(single_task_value32_nd(f32, now, prio_[m], ex_[m], qb_[m], nd_term[m], fl_[m]));
    } else {
#pragma unroll
      for (int m = 0; m < 4; m++) vout[m] = int64_t(score_slow(pf, fast_clock, wr_v[m], now, prio_[m], ex_[m], qb_[m], nd_[m], fl_[m]));
    }
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const unsigned long long k = ord_i64(vout[m]);
      kmax = solo[m] ? max(kmax, k) : kmax;
      kmin = solo[m] ? min(kmin, k) : kmin;
    }
    // TotalValue of single-task units (also the own-unit candidate of a task that only joins other units by edges)
    if (!live) {
    } else if (t4 >= base && t4 + 3 < end) {  // whole sectors even when some of the four are multi-member-unit tasks: k_gbest rewrites theirs
      *reinterpret_cast<longlong2*>(G.tv + t4) = make_longlong2(vout[0], vout[1]);
      *reinterpret_cast<longlong2*>(G.tv + t4 + 2) = make_longlong2(vout[2], vout[3]);
    } else {
#pragma unroll
      for (int m = 0; m < 4; m++)
        if (wr_v[m]) G.tv[t4 + m] = vout[m];
    }
    if (dcomplex && live) {
      if (t4 >= base && t4 + 3 < end) *reinterpret_cast<uint4*>(G.e + t4) = make_uint4(eout[0], eout[1], eout[2], eout[3]);
      else {
#pragma unroll
        for (int m = 0; m < 4; m++)
          if (t4 + m >= base && t4 + m < end) G.e[t4 + m] = eout[m];
      }
    }
    // Work list: ONE global atomic per half tile (a block scan of the per-thread counts gives every entry its
    // place) -- an atomic per warp and task slot serialised every tile of the tick on one L2 address.  The entry carries
    // what every later kernel asks of the task (its unit slots and member payload), written here from registers, so
    // that those kernels read it coalesced instead of gathering the columns again.
    if (dcomplex) {  // block-uniform
      __shared__ uint32_t s_wsum[8];
      __shared__ uint32_t s_lbase;
      uint32_t total;
      const uint32_t before = block_scan_excl<8>(uint32_t(__popc(cmask)), s_wsum, &total);
      if (total) {  // block-uniform
        if (tid == 0) s_lbase = atomicAdd(G.ccount, total);
        __syncthreads();
        uint32_t pos = s_lbase + before;
        const int32_t vid_[4] = {vid4.x, vid4.y, vid4.z, vid4.w}, tgo_[4] = {tgo4.x, tgo4.y, tgo4.z, tgo4.w};
#pragma unroll
        for (int m = 0; m < 4; m++) {
          if (!((cmask >> m) & 1u)) continue;
          const uint32_t t = uint32_t(t4 + m), li = uint32_t(t4 + m - base);
          const int32_t gid = gid_[m], vid = vid_[m];
          const bool own_complex = (gid >= 0) | gv | (((hd4 >> (8 * m)) & 0xFFu) != 0);
          const uint32_t s_own = own_complex ? ub + own_slot_local(gid, vid, li, ng, gv) : kInactive;
          const uint32_t s_ver = (gid >= 0 && gv) ? ub + ng + uint32_t(vid) : kInactive;
          G.wl[pos] = make_uint4(t, uint32_t(d), s_own, s_ver);
          URec r;
          r.prio = prio_[m]; r.nd = nd_[m]; r.exp_ns = ex_[m]; r.qb = qb_[m]; r.tgo = tgo_[m];
          r.lif = li | (gid >= 0 ? kRecGrouped : 0u) | (((womask >> m) & 1u) ? kRecWaitOver : 0u) | ((fl_[m] & 0x3Fu) << 24);
          rec_store(G.pay + pos, r);
          pos++;
        }
      }
      __syncthreads();  // s_wsum / s_lbase are rewritten by the next half
    }
  }
  // fold: warp, then block (shared atomics), then one set of global atomics per tile
  {
    unsigned int cs[10] = {c_dm, c_mq, c_over, c_wait, c_sec, c_ung, c_ucnt, c_uover, c_uwait, c_umq};
#pragma unroll
    for (int k = 0; k < 10; k++) cs[k] = __reduce_add_sync(full, cs[k]);
    int64_t ss[4] = {s_exp, s_over, s_uexp, s_uover};
#pragma unroll
    for (int k = 0; k < 4; k++) ss[k] = warp_sum64(ss[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      kmax = max(kmax, __shfl_xor_sync(full, kmax, o));
      kmin = min(kmin, __shfl_xor_sync(full, kmin, o));
    }
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 10; k++) if (cs[k]) atomicAdd(&F.c[k], cs[k]);
#pragma unroll
      for (int k = 0; k < 4; k++) if (ss[k]) atomicAdd(&F.s[k], (unsigned long long)ss[k]);
      atomicMax(&F.vmax, kmax); atomicMin(&F.vmin, kmin);
    }
  }
  __syncthreads();
  if (tid < 16) {
    evg_queue_info* q = W.qinfo + d;
    switch (tid) {
      case 0: atomic_add64(&q->length_with_dependencies_met, F.c[0]); break;
      case 1: atomic_add64(&q->count_dep_filled_merge_queue_tasks, F.c[1]); break;
      case 2: atomic_add64(&q->count_duration_over_threshold, F.c[2]); break;
      case 3: atomic_add64(&q->count_wait_over_threshold, F.c[3]); break;
      case 4: atomic_add64(&q->secondary_queue, F.c[4]); break;
      case 5: atomic_add64(&q->has_ungrouped, F.c[5]); break;
      case 6: atomic_add64(&q->ungrouped.count, F.c[6]); break;
      case 7: atomic_add64(&q->ungrouped.count_duration_over_threshold, F.c[7]); break;
      case 8: atomic_add64(&q->ungrouped.count_wait_over_threshold, F.c[8]); break;
      case 9: atomic_add64(&q->ungrouped.count_dep_filled_merge_queue_tasks, F.c[9]); break;
      case 10: atomic_add64(&q->expected_duration, int64_t(F.s[0])); break;
      case 11: atomic_add64(&q->duration_over_threshold, int64_t(F.s[1])); break;
      case 12: atomic_add64(&q->ungrouped.expected_duration, int64_t(F.s[2])); break;
      case 13: atomic_add64(&q->ungrouped.duration_over_threshold, int64_t(F.s[3])); break;
      case 14: if (F.vmax > __ldcg(G.vmm + 2 * d)) atomicMax(G.vmm + 2 * d, F.vmax); break;
      case 15: if (F.vmin < __ldcg(G.vmm + 2 * d + 1)) atomicMin(G.vmm + 2 * d + 1, F.vmin); break;
    }
  }
}

// ---- multi-member units: the unit table ----
// A membership ("pair": a task filed under a unit slot by its own key, by its version, or by one of its in-queue
// dependencies' keys; planner.go:431-456) used to be a node of a linked list per slot, and every walk a chain of
// dependent scattered loads through six task columns.  Now the members of a unit are one contiguous run of work-list
// entry ids, each naming the 32-byte payload k_gtask wrote for the task:
//   k_glink   per pair: k = atomicAdd(unit_n[slot], 1) -- its place in the run (any order: everything computed from a
//             run is order-free); TaskGroupInfo sums of task-group tasks, from the payload
//   k_galloc  the pair that drew k == 0 reserves unit_n[slot] run positions and numbers the unit: unit_v[slot] = its id
//             and run start, unit[id] = {members, run start, distro}
//   k_gfill   every pair writes its entry id at run start + k, and replaces its slot with the unit's id
//   k_gunit   per unit, in id order: the run folded into Unit.info (planner.go:302-337), value (planner.go:209-300),
//             anchor; the members' ranks (TaskList.Less, planner.go:387-405) for units of up to kRankOne members
//   k_grank   the ranks of the larger units, a warp per 32 members
//   k_gbest   per task: the first unit it is emitted from among its memberships (TaskPlan.Export, planner.go:467-477)
//             and its rank there, one record load per membership; the task is filed under that rank in the unit's
//             emitted-by-rank slots, emit[start + rank], from which k_gplace writes the unit's tasks in order
// A membership's place in its run is kept next to the membership, so every access is coalesced: by work-list entry for
// the own-key (pown) and version (pver) memberships, by edge for dependency memberships (pedge, with the edge's unit slot
// in sedge).  After k_gfill the slot space (one slot per task and group, ~10x the units) is read once more, by k_gplace,
// for the unit each anchor task anchors; what the other later kernels ask of a unit is its 32-byte record, by id.  The
// on-chip planner's next[] / pair_slot[], indexed by pair id over 2T+E entries of which the general path would touch
// about a quarter (a sector per access), are not used here.

// what a work-list task is filed under: one 16-byte entry k_gtask wrote (the same answers in every kernel below)
struct WlTask {
  uint32_t t; int d; int64_t base; uint32_t li; bool own_complex; uint32_t s_own, s_ver;  // global slots
};
__device__ __forceinline__ WlTask wl_task(const DDistros& D, const DGen& G, unsigned int k) {
  const uint4 e = G.wl[k];
  WlTask x;
  x.t = e.x; x.d = int(e.y); x.s_own = e.z; x.s_ver = e.w;
  x.base = D.task_off[x.d];
  x.li = uint32_t(int64_t(x.t) - x.base);
  x.own_complex = x.s_own != kInactive;
  return x;
}
// f(place, unit, own) for every membership of work-list entry k: `place` points at its place in the unit's run, `unit`
// is the unit's slot (up to k_gfill) or id (after it), `own` marks the own-key membership (after k_glink: the places
// are final)
template <typename F>
__device__ __forceinline__ void wl_pairs(const DTasks& T, const DGen& G, const WlTask& x, unsigned int k, F&& f) {
  if (x.own_complex) f(G.pown + k, x.s_own, true);
  if (x.s_ver != kInactive) f(G.pver + k, x.s_ver, false);
  if (T.n_edges > 0)
    for (int64_t e = T.dep_off[x.t]; e < T.dep_off[x.t + 1]; e++) {
      const uint32_t sl = G.sedge[e];
      if (sl != kInactive) f(G.pedge + e, sl, false);
    }
}

// minimum resident blocks of the unit-table kernels k_glink .. k_gbest (latency-bound: one thread per task or unit,
// scattered sectors)
constexpr int kUnitTableOcc = 4;

__global__ void __launch_bounds__(256, kUnitTableOcc) k_glink(DTasks T, DDistros D, DWork W, DGen G, int64_t now) {
  if (*W.err) return;
  const unsigned int n = *G.ccount;
  for (unsigned int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const WlTask x = wl_task(D, G, k);
    const uint32_t t = x.t;
    const int d = x.d;
    const uint32_t ub = uint32_t(D.unit_base[d]), ng = uint32_t(D.group_off[d + 1] - D.group_off[d]);
    // own_slot_local files a task with group_id >= 0 under its group's slot (local slot = group_id < ng) and every other
    // task at ng or above, so the own-key slot tells task-group tasks apart without loading the payload
    if (x.own_complex && x.s_own - ub < ng) {
      const URec me = rec_load(G.pay + k);
      const evg_distro_cfg* cf = D.cfg + d;
      const uint32_t fl = (me.lif >> 24) & 0x3Fu;
      const int64_t exp_ns = me.exp_ns, threshold = cf->target_time_ns;
      const bool dm = (fl & EVG_TF_DEPS_MET) != 0;
      const bool counted = !cf->includes_dependencies || dm;
      const bool over = counted && exp_ns > threshold;
      const bool wait_over = (me.lif & kRecWaitOver) != 0;
      const bool mq_dm = dm && (fl & EVG_TF_REQ_MASK) == EVG_TF_REQ_MERGE_QUEUE;
      evg_group_info* g = W.ginfo + D.group_off[d] + (x.s_own - ub);
      atomic_add64(&g->count, counted);
      atomic_add64(&g->expected_duration, counted ? exp_ns : 0);
      atomic_add64(&g->count_duration_over_threshold, over);
      atomic_add64(&g->duration_over_threshold, over ? exp_ns : 0);
      atomic_add64(&g->count_wait_over_threshold, wait_over);
      atomic_add64(&g->count_dep_filled_merge_queue_tasks, mq_dm);
    }
    // a membership's place in its unit's run: any order, everything computed from a run is order-free
    if (x.own_complex) G.pown[k] = atomicAdd(W.unit_n + x.s_own, 1u);
    if (x.s_ver != kInactive) G.pver[k] = atomicAdd(W.unit_n + x.s_ver, 1u);  // planner.go:439
    if (T.n_edges > 0) {
      const bool gv = D.cfg[d].group_versions != 0;
      const int64_t e0 = T.dep_off[t], e1 = T.dep_off[t + 1];
      for (int64_t e = e0; e < e1; e++) {
        const uint32_t dl = uint32_t(T.dep_idx[e]);
        const uint32_t sl = ub + own_slot_local(T.gid[x.base + dl], T.vid[x.base + dl], dl, ng, gv);
        // Unit.Add is keyed by task id (planner.go:131): join each unit once.  A task without an own-key membership
        // has no dependents, so no edge of its own leads back to its own-key slot.
        bool dup = (sl == x.s_own) || (sl == x.s_ver);
        for (int64_t f = e0; f < e && !dup; f++) {
          const uint32_t fl2 = uint32_t(T.dep_idx[f]);
          dup = ub + own_slot_local(T.gid[x.base + fl2], T.vid[x.base + fl2], fl2, ng, gv) == sl;
        }
        G.sedge[e] = dup ? kInactive : sl;
        if (!dup) G.pedge[e] = atomicAdd(W.unit_n + sl, 1u);
      }
    }
  }
}

// Runs are reserved block by block: a block scan of the records its threads need, ONE atomic on the bump counter per
// block and trip (an atomic per unit serialises ~10^5 units of a tick on one L2 address).
__global__ void __launch_bounds__(256, kUnitTableOcc) k_galloc(DTasks T, DDistros D, DWork W, DGen G) {
  if (*W.err) return;
  __shared__ uint64_t s_wsum[8];
  __shared__ uint32_t s_base, s_hbase;
  const unsigned int n = *G.ccount;
  for (unsigned int k0 = blockIdx.x * blockDim.x; k0 < n; k0 += gridDim.x * blockDim.x) {  // block-uniform trip count
    const unsigned int k = k0 + threadIdx.x;
    WlTask x;
    uint32_t need = 0, heads = 0;  // records / units this thread's k == 0 pairs stand for
    if (k < n) {
      x = wl_task(D, G, k);
      wl_pairs(T, G, x, k, [&](const uint32_t* place, uint32_t slot, bool) { if (*place == 0u) { need += W.unit_n[slot]; heads++; } });
    }
    // both counts in one scan, records in the low half: they never carry into the units, as the tick's record total
    // is below 2^32 (upload_tasks)
    uint64_t both;
    const uint64_t ex = block_scan_excl<8>(uint64_t(need) | (uint64_t(heads) << 32), s_wsum, &both);
    const uint32_t total = uint32_t(both), htotal = uint32_t(both >> 32);
    if (threadIdx.x == 0 && htotal) { s_base = atomicAdd(G.rcount, total); s_hbase = atomicAdd(G.hcount, htotal); }
    __syncthreads();
    if (heads) {
      uint32_t pos = s_base + uint32_t(ex), hp = s_hbase + uint32_t(ex >> 32);
      wl_pairs(T, G, x, k, [&](const uint32_t* place, uint32_t slot, bool) {
        if (*place != 0u) return;
        GUnit u;
        u.value = 0; u.anchor = kNoAnchor; u.n = W.unit_n[slot]; u.start = pos; u.d = x.d;
        unit_store(G.unit + hp, u);
        W.unit_v[slot] = slot_unit(hp++, pos);
        pos += u.n;
      });
    }
    __syncthreads();  // the shared scratch is rewritten by the next trip
  }
}

// Two entries per trip, all their loads before any store: a store to the run could alias the next entry's loads, so one
// entry at a time would wait on every load in turn.
constexpr int kFillEntries = 2;
__global__ void __launch_bounds__(256, kUnitTableOcc) k_gfill(DTasks T, DDistros D, DWork W, DGen G) {
  if (*W.err) return;
  const unsigned int n = *G.ccount, stride = gridDim.x * blockDim.x;
  for (unsigned int k0 = blockIdx.x * blockDim.x + threadIdx.x; k0 < n; k0 += kFillEntries * stride) {
    WlTask x[kFillEntries];
    uint32_t place[kFillEntries][2], id[kFillEntries][2], start[kFillEntries][2];
#pragma unroll
    for (int j = 0; j < kFillEntries; j++) {
      const unsigned int k = k0 + j * stride;
      x[j].s_own = x[j].s_ver = kInactive;
      if (k < n) x[j] = wl_task(D, G, k);
      const uint32_t sl[2] = {x[j].s_own, x[j].s_ver};
#pragma unroll
      for (int m = 0; m < 2; m++) {
        place[j][m] = sl[m] != kInactive ? (m ? G.pver : G.pown)[k] : 0u;
        const uint64_t su = sl[m] != kInactive ? uint64_t(W.unit_v[sl[m]]) : ~0ull;
        id[j][m] = uint32_t(su);
        start[j][m] = uint32_t(su >> 32);
      }
    }
#pragma unroll
    for (int j = 0; j < kFillEntries; j++) {
      const unsigned int k = k0 + j * stride;
      if (k >= n) continue;
      // own-key members are the SetDistro members (planner.go:446)
      if (id[j][0] != kInactive) G.run[start[j][0] + place[j][0]] = k | kRunOwn;
      if (id[j][1] != kInactive) G.run[start[j][1] + place[j][1]] = k;
      G.wl[k] = make_uint4(x[j].t, uint32_t(x[j].d), id[j][0], id[j][1]);  // the units' ids replace their slots
      if (T.n_edges > 0)
        for (int64_t e = T.dep_off[x[j].t]; e < T.dep_off[x[j].t + 1]; e++) {
          const uint32_t sl = G.sedge[e];
          if (sl == kInactive) continue;
          const uint64_t su = uint64_t(W.unit_v[sl]);
          G.run[uint32_t(su >> 32) + G.pedge[e]] = k;
          G.sedge[e] = uint32_t(su);
        }
    }
  }
}

__device__ __forceinline__ void rec_acc(UnitAcc& a, int64_t now, const URec& r) {
  acc_add(a, now, r.prio, r.exp_ns, r.qb, r.nd, (r.lif & kRecGrouped) ? 0 : -1, (r.lif >> 24) & 0x3Fu);
}
__device__ __forceinline__ bool rec_less(const URec& x, const URec& y) {  // TaskList.Less, then input index
  return in_unit_less(x.tgo, x.nd, x.prio, x.exp_ns, rec_li(x), y.tgo, y.nd, y.prio, y.exp_ns, rec_li(y));
}
// Units up to this many members are ranked by the thread that folds them (at most kRankOne^2 comparisons on the keys it
// stashed in shared memory while folding); larger ones by k_grank, a warp per 32 members.
constexpr uint32_t kRankOne = 8;
constexpr int kRankKey = 6;  // tgo, nd, prio, expected (two words), index

// One thread per multi-member unit, in id order (dense warps: the unit records, not the work list).
__global__ void __launch_bounds__(256, kUnitTableOcc) k_gunit(DDistros D, DWork W, DGen G, int64_t now) {
  if (*W.err) return;
  const unsigned int n = *G.hcount;
  __shared__ uint32_t s_key[kRankOne * kRankKey][256];  // this thread's column: the rank keys of a small unit's members
  for (unsigned int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {  // the host cannot know n: fixed grid
    GUnit u = unit_load(G.unit + k);
    const uint32_t cnt = u.n, h = u.start;
    const uint32_t* run = G.run + h;
    UnitAcc a;
    acc_init(a);
    uint32_t anchor = kNoAnchor;
    const bool small = cnt <= kRankOne;
    for (uint32_t i = 0; i < cnt; i++) {
      const uint32_t q = run[i];
      const URec r = rec_load(G.pay + (q & kRunEntry));
      rec_acc(a, now, r);
      if (q & kRunOwn) anchor = min(anchor, rec_li(r));
      if (small) {
        uint32_t* kx = &s_key[i * kRankKey][threadIdx.x];
        kx[0] = uint32_t(r.tgo); kx[256] = uint32_t(r.nd); kx[512] = uint32_t(r.prio);
        kx[768] = uint32_t(uint64_t(r.exp_ns)); kx[1024] = uint32_t(uint64_t(r.exp_ns) >> 32); kx[1280] = rec_li(r);
      }
    }
    u.value = unit_value(a, D.cfg[u.d], nullptr);
    u.anchor = anchor;
    unit_store(G.unit + k, u);
    // every member's rank in the unit: a count over the member set, so the order of the run does not matter.  The
    // emitted-by-rank slots are cleared with the ranks, unit by unit (no memset; nothing of an earlier tick survives).
    if (small) {
      auto key = [&](uint32_t i, URec& r) {
        const uint32_t* kx = &s_key[i * kRankKey][threadIdx.x];
        r.tgo = int32_t(kx[0]); r.nd = int32_t(kx[256]); r.prio = int32_t(kx[512]);
        r.exp_ns = int64_t((unsigned long long)kx[768] | ((unsigned long long)kx[1024] << 32)); r.lif = kx[1280];
      };
      for (uint32_t i = 0; i < cnt; i++) {
        URec me, o;
        key(i, me);
        uint32_t rk = 0;
        for (uint32_t j = 0; j < cnt; j++) { key(j, o); rk += rec_less(o, me) ? 1u : 0u; }
        G.rank[h + i] = rk;
        G.emit[h + i] = kInactive;
      }
    } else {
      const uint32_t nch = (cnt + 31) >> 5;
      const uint32_t b = atomicAdd(G.bcount, nch);
      for (uint32_t c = 0; c < nch; c++) G.blist[b + c] = make_uint2(k, c);
    }
  }
}

// Ranks of the units above kRankOne members: a warp per 32 members (lane = member), the whole run streamed past them 32
// records at a time (coalesced) and broadcast with shuffles.  n members cost n comparisons per lane, in parallel over
// the ceil(n / 32) warps of the unit.
__global__ void __launch_bounds__(256, kUnitTableOcc) k_grank(DWork W, DGen G) {
  if (*W.err) return;
  const unsigned int n = *G.bcount;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned int nw = gridDim.x * (blockDim.x >> 5);
  for (unsigned int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < n; c += nw) {  // warp-uniform
    const uint2 ch = G.blist[c];
    const GUnit u = unit_load(G.unit + ch.x);
    const uint32_t cnt = u.n, h = u.start;
    const uint32_t* run = G.run + h;
    const uint32_t i = ch.y * 32u + uint32_t(lane);
    URec me;
    me.tgo = 0; me.nd = 0; me.prio = 0; me.exp_ns = 0; me.lif = 0;
    if (i < cnt) me = rec_load(G.pay + (run[i] & kRunEntry));
    uint32_t rk = 0;
    for (uint32_t j0 = 0; j0 < cnt; j0 += 32) {
      URec o;
      o.tgo = 0; o.nd = 0; o.prio = 0; o.exp_ns = 0; o.lif = 0;
      if (j0 + lane < cnt) o = rec_load(G.pay + (run[j0 + lane] & kRunEntry));
      const uint32_t m = min(32u, cnt - j0);
      for (uint32_t q = 0; q < m; q++) {
        URec y;
        y.tgo = __shfl_sync(full, o.tgo, q); y.nd = __shfl_sync(full, o.nd, q); y.prio = __shfl_sync(full, o.prio, q);
        y.exp_ns = __shfl_sync(full, o.exp_ns, q); y.lif = __shfl_sync(full, o.lif, q);
        rk += (i < cnt && rec_less(y, me)) ? 1u : 0u;
      }
    }
    if (i < cnt) { G.rank[h + i] = rk; G.emit[h + i] = kInactive; }
  }
}

__global__ void __launch_bounds__(256, kUnitTableOcc) k_gbest(DTasks T, DDistros D, DWork W, DGen G, int want_best_pair) {
  if (*W.err) return;
  const unsigned int n = *G.ccount;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  // Warp-uniform trips (every lane of a warp runs the same ones, lanes past n idle), so that the value-range fold at the
  // end of a trip is a full-warp reduction that needs no assumption about which lanes reconverged.
  for (unsigned int kw = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); kw < n; kw += gridDim.x * blockDim.x) {
    const unsigned int k = kw + lane;
    int d = -1;
    unsigned long long kk = 0ull;
    if (k < n) {
      const WlTask x = wl_task(D, G, k);
      const uint32_t t = x.t, li = x.li;
      d = x.d;
      bool have = false;
      int64_t bv = 0;
      uint32_t ba = 0, bid = kInactive, bstart = 0, bpos = 0;
      if (!x.own_complex) { have = true; bv = G.tv[t]; ba = li; }  // its own single-task unit, scored by k_gtask
      wl_pairs(T, G, x, k, [&](const uint32_t* place, uint32_t id, bool) {
        const GUnit u = unit_load(G.unit + id);
        const uint32_t kx = *place;  // this task's place in that unit's run (requested together with the record)
        if (u.anchor == kNoAnchor) return;
        if (!have || u.value > bv || (u.value == bv && u.anchor < ba)) {
          have = true; bv = u.value; ba = u.anchor; bid = id; bstart = u.start; bpos = u.start + kx;
        }
      });
      // Emitted from a multi-member unit: filed under its rank among ALL members of the unit, as k_gunit / k_grank
      // counted it (ranks are unique inside a unit: a plain store), and k_gplace writes it with the unit's value.
      // Emitted from its own single-task unit: k_gplace writes it with the value k_gtask left in tv.
      if (bid != kInactive) {
        G.emit[bstart + G.rank[bpos]] = li;
        W.has_dep[t] |= 2;  // only this thread touches the byte now (k_gmark and k_gtask are done)
      }
      if (want_best_pair) W.best_pair[t] = bid;  // k_breakdown's way back to the unit (general path: its id)
      atomicAdd(G.e + x.base + ba, 1u);
      kk = ord_i64(bv);
    }
    // The distro's value range.  The work list is in task order, so a warp nearly always sits inside one distro: its 32
    // values are folded with full-warp shuffles (idle lanes hold the identities 0 / ~0) and ONE lane looks at the
    // distro's pair (instead of every thread polling the same two L2 lines).  Lane 0 is never idle (kw < n).
    const int d0 = __shfl_sync(full, d, 0);
    if (__all_sync(full, d < 0 || d == d0)) {
      unsigned long long hi = d < 0 ? 0ull : kk, lo = d < 0 ? ~0ull : kk;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        hi = max(hi, __shfl_xor_sync(full, hi, o));
        lo = min(lo, __shfl_xor_sync(full, lo, o));
      }
      if (lane == 0) {
        if (hi > __ldcg(G.vmm + 2 * d0)) atomicMax(G.vmm + 2 * d0, hi);
        if (lo < __ldcg(G.vmm + 2 * d0 + 1)) atomicMin(G.vmm + 2 * d0 + 1, lo);
      }
    } else if (d >= 0) {
      if (kk > __ldcg(G.vmm + 2 * d)) atomicMax(G.vmm + 2 * d, kk);
      if (kk < __ldcg(G.vmm + 2 * d + 1)) atomicMin(G.vmm + 2 * d + 1, kk);
    }
  }
}

// radix pass count of the tick (the host launches that many pass triples... it cannot know: it launches 8, the
// kernels of passes beyond *maxpass exit at once)
__global__ void k_gsched(DGen G, const int32_t* __restrict__ general_list, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  atomicMax(G.maxpass, gen_npass(gen_bits(G, general_list[k])));
}

// e[] of the eight task slots t8 .. t8+7 of a tile (t8 a multiple of 4): 128-bit accesses inside the distro, slot by
// slot at its edges (slots outside it read as 0 and are not written)
__device__ __forceinline__ void gen_e_load8(const DGen& G, int64_t t8, int64_t base, int64_t end, uint32_t (&ev)[8]) {
  if (t8 >= base && t8 + 7 < end) {
    const uint4 a = *reinterpret_cast<const uint4*>(G.e + t8), b = *reinterpret_cast<const uint4*>(G.e + t8 + 4);
    ev[0] = a.x; ev[1] = a.y; ev[2] = a.z; ev[3] = a.w; ev[4] = b.x; ev[5] = b.y; ev[6] = b.z; ev[7] = b.w;
  } else {
#pragma unroll
    for (int m = 0; m < 8; m++) { const int64_t t = t8 + m; ev[m] = (t >= base && t < end) ? G.e[t] : 0u; }
  }
}

// Per tile: exclusive scan of e[] (thread q owns 8 consecutive slots).  Every task's e becomes the offset of its anchor's
// run inside the tile's stretch, and tile_sum the tile's total (k_gscan turns the totals into the tiles' offsets in the
// distro).  The offsets are final before k_gplace starts, so a unit placed by any block finds its anchor's run start
// without waiting for the block that places the anchor's tile.
__global__ void __launch_bounds__(256) k_gsum(DDistros D, DGen G) {
  const int tile = int(blockIdx.x + G.tile0);
  const int d = G.tile_distro[tile];
  const int64_t base = D.task_off[d], end = D.task_off[d + 1];
  const int64_t t8 = G.tile_start[tile] + 8 * int64_t(threadIdx.x);  // multiple of 4
  uint32_t ev[8];
  gen_e_load8(G, t8, base, end, ev);
  uint32_t sum = 0;
#pragma unroll
  for (int m = 0; m < 8; m++) sum += ev[m];
  __shared__ uint32_t sw[8];
  uint32_t total;
  uint32_t run = block_scan_excl<8>(sum, sw, &total);
#pragma unroll
  for (int m = 0; m < 8; m++) { const uint32_t x = ev[m]; ev[m] = run; run += x; }
  if (t8 >= base && t8 + 7 < end) {
    *reinterpret_cast<uint4*>(G.e + t8) = make_uint4(ev[0], ev[1], ev[2], ev[3]);
    *reinterpret_cast<uint4*>(G.e + t8 + 4) = make_uint4(ev[4], ev[5], ev[6], ev[7]);
  } else {
#pragma unroll
    for (int m = 0; m < 8; m++) { const int64_t t = t8 + m; if (t >= base && t < end) G.e[t] = ev[m]; }
  }
  if (threadIdx.x == 0) G.tile_sum[tile] = total;
}

// Where the run of the distro-local task `anchor` starts in its distro's pre-arrangement (after k_gsum and k_gscan): its
// tile's offset plus its offset inside the tile.  Tiles of a distro start at (base & ~3) + k * kGTile.
__device__ __forceinline__ uint32_t gen_run_start(const DDistros& D, const DGen& G, int d, uint32_t anchor) {
  const int64_t base = D.task_off[d];
  const int64_t tile = G.dtile_off[d] + ((int64_t(anchor) + (base & 3)) / kGTile);
  return G.tile_sum[tile] + G.e[base + anchor];
}

// exclusive scan of the tile sums of one distro (<= 1025 tiles), one block per general-path distro
__global__ void __launch_bounds__(1024) k_gscan(DGen G, const int32_t* __restrict__ general_list) {
  const int d = general_list[blockIdx.x];
  const int64_t t0 = G.dtile_off[d];
  block_scan_segment(G.tile_sum + t0, G.dtile_off[d + 1] - t0);
}

__device__ __forceinline__ void gen_put_key(const DGen& G, int64_t base, uint32_t pos, unsigned long long key, bool wide, uint32_t li) {
  G.key_lo[0][base + pos] = uint32_t(key);
  if (wide) G.key_hi[0][base + pos] = uint32_t(key >> 32);
  G.idx[0][base + pos] = li;
}
__device__ __forceinline__ void gen_put(const DGen& G, int64_t base, uint32_t pos, unsigned long long vmax_ord, bool wide,
                                        int64_t v, uint32_t li) {
  gen_put_key(G, base, pos, vmax_ord - ord_i64(v), wide, li);
}

// Placement: the (Vmax - V, index) pairs go to key_lo[0] / key_hi[0] / idx[0] in (anchor, rank-in-unit) order, by one
// kernel, a block per tile.  The block writes its tile's stretch: the tasks emitted from their own single-task unit, and
// the tasks of every unit of up to kRankOne members anchored in the tile.  Then it takes its share of blist: the larger
// units, a warp each, wherever they are anchored.
//
// Every writer writes only the slots it fills, and the writers touch disjoint slots: a task emitted from its own unit
// has a run of one slot (it anchors no multi-member unit, whose anchor is an own-key member), and a unit writes only
// inside its anchor's run.  So no slot is written twice, none is left with an earlier tick's data, and the order of the
// writers does not reach the result.  Placing a small unit from the block that holds its anchor puts the unit's bytes
// into the same sectors as the tile's, while they are in L2 (in the stage, when the stretch fits it).  Walked in id
// order, the units reach a stretch long after its tile has left L2 (k_galloc hands out ids in waves of resident
// blocks, not in work-list order), and every sector a unit shares with a tile costs a DRAM read and a write.
__device__ __forceinline__ void gplace_tile(const DTasks& T, const DDistros& D, const DWork& W, const DGen& G, int tile, int use_e) {
  const int d = G.tile_distro[tile];
  const int64_t base = D.task_off[d], end = D.task_off[d + 1];
  const int64_t ts = G.tile_start[tile];
  const unsigned long long vmax_ord = G.vmm[2 * d];
  const bool wide = gen_bits(G, d) > 32;
  const int tid = threadIdx.x;
  const int64_t t8 = ts + 8 * int64_t(tid);  // multiple of 4
  const bool interior = t8 >= base && t8 + 7 < end;  // the common case: 128-bit loads
  // use_e: the tile's tasks land in ONE contiguous stretch of the distro's segment, [tile_sum[tile], + the tile's total),
  // at the offsets k_gsum left in e.  The block's tasks are staged in shared memory and copied out slot by slot,
  // skipping the slots of the warp-walked units (kInactive in st_ix): 4-byte stores straight from registers cost a
  // sector each, several times the sectors of the payload.  A stretch above kStage slots is written from registers.
  constexpr int kStage = 3072;
  __shared__ uint32_t st_lo[kStage], st_ix[kStage], st_hi[kStage];
  uint32_t p_tile = 0, total = 0;
  if (use_e) {
    p_tile = G.tile_sum[tile];
    // every task of the distro is emitted once, so the distro's stretches add up to its task count
    const uint32_t p_next = tile + 1 < G.dtile_off[d + 1] ? G.tile_sum[tile + 1] : uint32_t(end - base);
    total = p_next - p_tile;
    if (total <= uint32_t(kStage))  // the barrier before the stage is filled publishes this
      for (uint32_t q = tid; q < total; q += 256) st_ix[q] = kInactive;
  }
  const bool staged = total <= uint32_t(kStage);  // block-uniform
  int64_t vv[8];
  uint32_t dsp = 0;  // bit m: task t8+m is emitted from a multi-member unit (placed with that unit)
  if (interior) {
#pragma unroll
    for (int m = 0; m < 8; m += 2) {
      const longlong2 x = *reinterpret_cast<const longlong2*>(G.tv + t8 + m);
      vv[m] = x.x; vv[m + 1] = x.y;
    }
    if (use_e) {
      const uint32_t h0 = *reinterpret_cast<const uint32_t*>(W.has_dep + t8), h1 = *reinterpret_cast<const uint32_t*>(W.has_dep + t8 + 4);
#pragma unroll
      for (int m = 0; m < 4; m++) dsp |= (((h0 >> (8 * m + 1)) & 1u) << m) | (((h1 >> (8 * m + 1)) & 1u) << (m + 4));
    }
  } else {
#pragma unroll
    for (int m = 0; m < 8; m++) {
      const int64_t t = t8 + m;
      const bool in = t >= base && t < end;
      vv[m] = in ? G.tv[t] : 0;
      if (use_e && in && (W.has_dep[t] & 2)) dsp |= 1u << m;
    }
  }
  if (use_e) {
    uint32_t ps[8];
    gen_e_load8(G, t8, base, end, ps);
    // the run length of every slot: the next slot's offset (the next thread's first, across warps through s_first)
    __shared__ uint32_t s_first[8];
    const int lane = tid & 31, warp = tid >> 5;
    if (lane == 0) s_first[warp] = ps[0];
    __syncthreads();
    uint32_t nx = __shfl_down_sync(0xffffffffu, ps[0], 1);
    if (lane == 31) nx = warp < 7 ? s_first[warp + 1] : total;
#pragma unroll
    for (int m = 0; m < 8; m++) {
      const int64_t t = t8 + m;
      if (t >= base && t < end && !((dsp >> m) & 1u)) {
        if (staged) {
          const unsigned long long key = vmax_ord - ord_i64(vv[m]);
          st_lo[ps[m]] = uint32_t(key); st_ix[ps[m]] = uint32_t(t - base);
          if (wide) st_hi[ps[m]] = uint32_t(key >> 32);
        } else {
          gen_put(G, base, p_tile + ps[m], vmax_ord, wide, vv[m], uint32_t(t - base));
        }
      }
    }
    // the small units anchored in this tile: a task emitted from a multi-member unit that has a run anchors the unit
    // filed under its own key (an anchor is an own-key member), whose id k_galloc left in that slot.  The unit's
    // emitted tasks fill the run in rank order.
    uint32_t amask = 0;
#pragma unroll
    for (int m = 0; m < 8; m++) {
      const int64_t t = t8 + m;
      // the distro's last task runs to the end of the stretch: the slots past the distro read as 0
      const uint32_t run_end = t + 1 < end ? (m < 7 ? ps[m + 1] : nx) : total;
      amask |= ((t >= base && t < end && ((dsp >> m) & 1u) && run_end != ps[m]) ? 1u : 0u) << m;
    }
    if (amask) {
      const uint32_t ub = uint32_t(D.unit_base[d]), ng = uint32_t(D.group_off[d + 1] - D.group_off[d]);
      const bool gv = D.cfg[d].group_versions != 0;
      do {
        const int m = __ffs(amask) - 1;
        amask &= amask - 1u;
        uint32_t q = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) q = j == m ? ps[j] : q;
        const int64_t t = t8 + m;
        const uint32_t id = uint32_t(W.unit_v[ub + own_slot_local(T.gid[t], T.vid[t], uint32_t(t - base), ng, gv)]);
        const GUnit u = unit_load(G.unit + id);
        if (u.n > kRankOne) continue;  // a warp's job (gplace_big_units)
        uint32_t li[kRankOne];
#pragma unroll
        for (uint32_t i = 0; i < kRankOne; i++) li[i] = i < u.n ? G.emit[u.start + i] : kInactive;
        const unsigned long long key = vmax_ord - ord_i64(u.value);
#pragma unroll
        for (uint32_t i = 0; i < kRankOne; i++) {
          if (li[i] == kInactive) continue;
          if (staged) {
            st_lo[q] = uint32_t(key); st_ix[q] = li[i];
            if (wide) st_hi[q] = uint32_t(key >> 32);
          } else {
            gen_put_key(G, base, p_tile + q, key, wide, li[i]);
          }
          q++;
        }
      } while (amask);
    }
    if (staged) {
      __syncthreads();
      uint32_t* dlo = G.key_lo[0] + base + p_tile;
      uint32_t* dix = G.idx[0] + base + p_tile;
      uint32_t* dhi = G.key_hi[0] + base + p_tile;
      for (uint32_t q = tid; q < total; q += 256) {
        const uint32_t ix = st_ix[q];
        if (ix == kInactive) continue;
        dlo[q] = st_lo[q]; dix[q] = ix;
        if (wide) dhi[q] = st_hi[q];
      }
    }
  } else if (interior) {  // identity placement: position base + (t - base) = t, and t8 is a multiple of four -> 128-bit stores
    uint32_t kl[8], kh[8];
#pragma unroll
    for (int m = 0; m < 8; m++) {
      const unsigned long long key = vmax_ord - ord_i64(vv[m]);
      kl[m] = uint32_t(key); kh[m] = uint32_t(key >> 32);
    }
    const uint32_t p0 = uint32_t(t8 - base);
    *reinterpret_cast<uint4*>(G.key_lo[0] + t8) = make_uint4(kl[0], kl[1], kl[2], kl[3]);
    *reinterpret_cast<uint4*>(G.key_lo[0] + t8 + 4) = make_uint4(kl[4], kl[5], kl[6], kl[7]);
    *reinterpret_cast<uint4*>(G.idx[0] + t8) = make_uint4(p0, p0 + 1, p0 + 2, p0 + 3);
    *reinterpret_cast<uint4*>(G.idx[0] + t8 + 4) = make_uint4(p0 + 4, p0 + 5, p0 + 6, p0 + 7);
    if (wide) {
      *reinterpret_cast<uint4*>(G.key_hi[0] + t8) = make_uint4(kh[0], kh[1], kh[2], kh[3]);
      *reinterpret_cast<uint4*>(G.key_hi[0] + t8 + 4) = make_uint4(kh[4], kh[5], kh[6], kh[7]);
    }
  } else {
#pragma unroll
    for (int m = 0; m < 8; m++) {
      const int64_t t = t8 + m;
      if (t >= base && t < end) gen_put(G, base, uint32_t(t - base), vmax_ord, wide, vv[m], uint32_t(t - base));
    }
  }
}

// The tasks a unit emits share one key, Vmax - unit value, and one stretch of the pre-arrangement, from its anchor's run
// start in rank order: the unit walks its emitted-by-rank slots, so no member is placed by a loop over the others.  Units
// above kRankOne members: a warp per unit (its chunk-0 entry in blist), 32 ranks per step, a ballot giving every lane its
// place after the running count.  Block `item` of n_items takes that share of blist.
__device__ __forceinline__ void gplace_big_units(const DDistros& D, const DGen& G, unsigned int item, unsigned int n_items) {
  const unsigned long long nb = *G.bcount;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const unsigned int c1 = unsigned(nb * (item + 1) / n_items);
  for (unsigned int c = unsigned(nb * item / n_items) + (threadIdx.x >> 5); c < c1; c += blockDim.x >> 5) {  // warp-uniform
    const uint2 ch = G.blist[c];
    if (ch.y != 0u) continue;  // one warp per unit
    const GUnit u = unit_load(G.unit + ch.x);
    if (u.anchor == kNoAnchor) continue;
    const int64_t base = D.task_off[u.d];
    const unsigned long long key = G.vmm[2 * u.d] - ord_i64(u.value);
    const bool wide = gen_bits(G, u.d) > 32;
    uint32_t pos = gen_run_start(D, G, u.d, u.anchor);
    for (uint32_t r0 = 0; r0 < u.n; r0 += 32) {
      const uint32_t li = r0 + lane < u.n ? G.emit[u.start + r0 + lane] : kInactive;
      const unsigned b = __ballot_sync(full, li != kInactive);
      if (li != kInactive) gen_put_key(G, base, pos + uint32_t(__popc(b & lt)), key, wide, li);
      pos += uint32_t(__popc(b));
    }
  }
}

// use_e == 0 (no multi-member unit in any general-path distro): positions are the input order, and there are no units.
// 48 registers (5 blocks of 256 per SM); at the 40 of 6 blocks, the bound the stage allows, the kernel was no faster
__global__ void __launch_bounds__(256) k_gplace(DTasks T, DDistros D, DWork W, DGen G, int use_e) {
  gplace_tile(T, D, W, G, int(G.tile0 + blockIdx.x), use_e);
  if (use_e && !*W.err) gplace_big_units(D, G, blockIdx.x, gridDim.x);
}

__device__ __forceinline__ bool gen_tile(const DDistros& D, const DGen& G, int tile, int j, int* d_out, int64_t* seg, int64_t* lo,
                                         int* cnt, bool* wide, bool* last) {
  const int d = G.tile_distro[tile];
  const int bits = gen_bits(G, d), np = gen_npass(bits);
  if (j >= np) return false;
  *last = j == np - 1;
  const int64_t base = D.task_off[d], end = D.task_off[d + 1];
  const int64_t a = max(G.tile_start[tile], base), b = min(G.tile_start[tile] + kGTile, end);
  *d_out = d; *seg = base; *lo = a; *cnt = int(b - a); *wide = bits > 32;
  return true;
}

__global__ void __launch_bounds__(256) k_ghist(int j, DDistros D, DGen G) {
  if (j >= *G.maxpass) return;
  int d, cnt; int64_t seg, lo; bool wide, last;
  const int tile = int(blockIdx.x + G.tile0);
  if (!gen_tile(D, G, tile, j, &d, &seg, &lo, &cnt, &wide, &last)) return;
  const uint32_t* src = (j < 4 ? G.key_lo[j & 1] : G.key_hi[j & 1]) + lo;
  const int shift = 8 * (j & 3);
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < cnt; i += 256) atomicAdd(&h[(src[i] >> shift) & 255u], 1u);
  __syncthreads();
  G.tile_hist[int64_t(tile) * 256 + threadIdx.x] = h[threadIdx.x];
}

// Offsets of every (tile, digit) counter of one distro: exclusive over the tiles of a digit, then over the digits
// (four thread groups split the tiles, eight independent loads in flight per thread).
__global__ void __launch_bounds__(1024) k_gdscan(int j, const int32_t* __restrict__ general_list, DGen G) {
  if (j >= *G.maxpass) return;
  const int d = general_list[blockIdx.x];
  if (j >= gen_npass(gen_bits(G, d))) return;
  const int dg = threadIdx.x & 255, grp = threadIdx.x >> 8;
  const int64_t t0 = G.dtile_off[d], nt = G.dtile_off[d + 1] - t0;
  const int64_t per = (nt + 3) / 4;
  const int64_t a = t0 + (grp * per < nt ? grp * per : nt), b = t0 + ((grp + 1) * per < nt ? (grp + 1) * per : nt);
  uint32_t* h = G.tile_hist + dg;
  uint32_t sum = 0;
  int64_t tile = a;
  for (; tile + 8 <= b; tile += 8) {
    uint32_t x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = h[(tile + k) * 256];
#pragma unroll
    for (int k = 0; k < 8; k++) sum += x[k];
  }
  for (; tile < b; tile++) sum += h[tile * 256];
  __shared__ uint32_t part[4][256];
  __shared__ uint32_t s[256];
  part[grp][dg] = sum;
  __syncthreads();
  const uint32_t total = part[0][dg] + part[1][dg] + part[2][dg] + part[3][dg];
  // group 0 (threads 0 .. 255, one per digit) holds the digit totals, so their block scan is the scan over the digits;
  // s passes it to the other groups
  const uint32_t before = block_scan_excl<32>(grp == 0 ? total : 0u, s);
  __syncthreads();
  if (grp == 0) s[dg] = before;
  __syncthreads();
  uint32_t run = s[dg];
  for (int g = 0; g < grp; g++) run += part[g][dg];
  tile = a;
  for (; tile + 8 <= b; tile += 8) {
    uint32_t x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = h[(tile + k) * 256];
#pragma unroll
    for (int k = 0; k < 8; k++) { h[(tile + k) * 256] = run; run += x[k]; }
  }
  for (; tile < b; tile++) { const uint32_t x = h[tile * 256]; h[tile * 256] = run; run += x; }
}

// Warp w ranks chunks 8w .. 8w+7 of the tile in order (stability): one MATCH.ANY per chunk, the group's first lane adds
// the group size to the warp's digit counter and gets back the count of equal digits in the warp's earlier chunks (as in
// k_plan_cta).  The tile is then sorted by digit IN SHARED MEMORY and written out in that order: consecutive threads
// write consecutive addresses inside a digit's run, so a run costs its sectors once -- scattering straight from
// registers puts nearly every 4-byte store in a sector of its own (L2-write bound).  A distro's last pass writes order[]
// and TotalValue per rank (planner.go:467-477) instead of the key / index pair.
template <bool WIDE>
__device__ __forceinline__ void gscatter_tile(int j, const DGen& G, int tile, int d, int64_t seg, int64_t lo, int cnt, bool last,
                                              int32_t* __restrict__ order, int64_t* __restrict__ total_value, uint32_t (*wcnt)[256],
                                              uint32_t* s_lo, uint32_t* s_ix, uint32_t* s_hi, int32_t* s_delta, uint32_t* s_wsum) {
  constexpr bool wide = WIDE;
  const int sb = j & 1, db = sb ^ 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
#pragma unroll
  for (int w = 0; w < 8; w++) wcnt[w][tid] = 0u;
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  const int shift = 8 * (j & 3);
  const bool use_hi = j >= 4;
  const uint32_t* src_lo = G.key_lo[sb] + lo;
  const uint32_t* src_hi = G.key_hi[sb] + lo;
  const uint32_t* src_ix = G.idx[sb] + lo;
  uint32_t kl[8], kh[8], ix[8], dg[8], rk[8];
#pragma unroll
  for (int k = 0; k < 8; k++) {  // all loads first
    const int i = (warp * 8 + k) * 32 + lane;
    const bool ok = i < cnt;
    kl[k] = ok ? src_lo[i] : 0u;
    kh[k] = (ok && wide) ? src_hi[i] : 0u;
    ix[k] = ok ? src_ix[i] : 0u;
  }
  // all eight MATCHes, then the eight leader atomics back to back (one warp's shared-memory atomics execute in issue
  // order: chunk k+1's returned count includes chunk k's add), then the shuffles: the atomic round trips overlap
  unsigned peers[8];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int i = (warp * 8 + k) * 32 + lane;
    dg[k] = i < cnt ? (((use_hi ? kh[k] : kl[k]) >> shift) & 255u) : 256u;
    peers[k] = __match_any_sync(0xffffffffu, dg[k]);
  }
#pragma unroll
  for (int k = 0; k < 8; k++) {
    rk[k] = 0;
    if (dg[k] < 256u && (peers[k] & lt) == 0u) rk[k] = atomicAdd(&wcnt[warp][dg[k]], uint32_t(__popc(peers[k])));
  }
#pragma unroll
  for (int k = 0; k < 8; k++) rk[k] = __shfl_sync(0xffffffffu, rk[k], __ffs(peers[k]) - 1) + uint32_t(__popc(peers[k] & lt));
  __syncthreads();
  {  // thread = digit: the eight warp counters become offsets inside the digit; the digit totals are scanned over the block
    uint32_t x[8], tot = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) { x[w] = wcnt[w][tid]; tot += x[w]; }
    const uint32_t lbase = block_scan_excl<8>(tot, s_wsum);  // where digit `tid` starts in the sorted tile
    s_delta[tid] = int32_t(G.tile_hist[int64_t(tile) * 256 + tid]) - int32_t(lbase);
    uint32_t run = lbase;
#pragma unroll
    for (int w = 0; w < 8; w++) { wcnt[w][tid] = run; run += x[w]; }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    if (dg[k] < 256u) {
      const uint32_t lp = wcnt[warp][dg[k]] + rk[k];
      s_lo[lp] = kl[k];
      s_ix[lp] = ix[k];
      if (wide) s_hi[lp] = kh[k];
    }
  }
  __syncthreads();
  if (last) {
    const unsigned long long vmax_ord = G.vmm[2 * d];
    int32_t* dst_o = order + seg;
    int64_t* dst_v = total_value + seg;
    for (int i = tid; i < cnt; i += 256) {
      const uint32_t a = s_lo[i], h = wide ? s_hi[i] : 0u;
      const int64_t pos = int64_t(s_delta[((use_hi ? h : a) >> shift) & 255u]) + i;
      dst_o[pos] = int32_t(s_ix[i]);
      dst_v[pos] = unord_i64(vmax_ord - (((unsigned long long)h << 32) | a));
    }
    return;
  }
  uint32_t* dst_lo = G.key_lo[db] + seg;
  uint32_t* dst_hi = G.key_hi[db] + seg;
  uint32_t* dst_ix = G.idx[db] + seg;
  for (int i = tid; i < cnt; i += 256) {
    const uint32_t a = s_lo[i], h = wide ? s_hi[i] : 0u;
    const uint32_t dgt = ((use_hi ? h : a) >> shift) & 255u;
    const int64_t pos = int64_t(s_delta[dgt]) + i;
    dst_lo[pos] = a;
    dst_ix[pos] = s_ix[i];
    if (wide) dst_hi[pos] = h;
  }
}

// The key's high word travels only for distros whose value range exceeds 32 bits (a handful of registers and 8 KB of
// shared memory the common case does not pay for).
__global__ void __launch_bounds__(256, 4) k_gscatter(int j, DDistros D, DGen G, int32_t* __restrict__ order,
                                                     int64_t* __restrict__ total_value) {
  if (j >= *G.maxpass) return;
  int d, cnt; int64_t seg, lo; bool wide, last;
  const int tile = int(blockIdx.x + G.tile0);
  if (!gen_tile(D, G, tile, j, &d, &seg, &lo, &cnt, &wide, &last)) return;
  __shared__ uint32_t wcnt[8][256];   // per-warp digit counters, then local positions
  __shared__ uint32_t s_lo[kGTile], s_ix[kGTile], s_hi[kGTile];
  __shared__ int32_t s_delta[256];    // digit -> (offset of the digit's run in the distro) - (its offset in the sorted tile)
  __shared__ uint32_t s_wsum[8];
  if (wide) gscatter_tile<true>(j, G, tile, d, seg, lo, cnt, last, order, total_value, wcnt, s_lo, s_ix, s_hi, s_delta, s_wsum);
  else gscatter_tile<false>(j, G, tile, d, seg, lo, cnt, last, order, total_value, wcnt, s_lo, s_ix, s_hi, s_delta, s_wsum);
}
