// evg_sched.cu -- libevgsched.so: CUDA kernels (sm_90a) + the C-ABI of
// include/evg_sched.h.  See DESIGN.md for the data layout and the kernel list.
//
// Distros are routed by size and shape on the host:
//   <= 32 tasks      k_plan_warp (evg_plan_warp.cuh): one warp plans the distro
//   <= 10240 tasks, no GroupVersions, no in-queue dependency edges
//                    k_plan_cta<THREADS,CAP> (evg_plan_cta.cuh): one CTA plans the distro on-chip, several CTAs per
//                    SM, TMA-staged columns, u32 keys; distros it cannot hold (values beyond 32 bits, ...) are
//                    handed back ("punted") to k_plan_smem on the device
//   <= 12288 tasks   k_plan_smem<THREADS,ITEMS> (evg_plan_smem.cuh): one CTA per distro, any unit structure
//   larger           the general path (evg_plan_general.cuh), any size up to 2^21-1 tasks:
//     k_gmark/k_gtask/k_gunit/k_gbest  dependents, per-task pass, multi-member units
//     k_gsum/k_gscan/k_gplace*     canonical pre-arrangement by counting
//     k_ghist/k_gdscan/k_gscatter  segmented stable LSD radix sort of 32-bit keys; the last pass writes the ranked
//                                  queue + TotalValue
//     k_finalize_info              DistroQueueInfo / TaskGroupInfo scalars (scheduler.go:144-158)
// Both:
//   k_breakdown           the 13-field SortingValueBreakdown per ranked task (EVG_OPT_BREAKDOWN)
//   k_alloc<TPD>          utilization host allocator, a warp or a block per distro (utilization_based_host_allocator.go:26-409)
//   k_validate            range check of the distro-local ids the planners index with
// The rows either side of the path (SURVEY.md §8f):
//   k_deps_met            Task.DependenciesMet / AllDependenciesSatisfied (model/task/task.go:632-671,795-821)
//   k_runnable            the task finders' filter + stable compaction (scheduler/task_finder.go:40-317)
//   k_runnable_pipe       the same with the pipeline finder's codes (model/task/db.go:887-1066)
//   k_pl_deps             the pipeline's $graphLookup dependency filter (db.go:923-996)
//   k_pl_plan, k_pl_edge_*  what the planner receives from a pipeline distro (evg_plan_from_finder_ex)
//   k_dur_sum/dev/final   expected-duration statistics (model/task/expected_duration.go:36-96)
//   k_dur_pair            the single matched key of a (project, build variant) pair (expected_duration.go:54-56)
//   k_dur_resolve         Task.FetchExpectedDuration per listed row (model/task/task.go:3519-3590) into staging
//   k_dur_commit          the resolved durations into the resident columns, unless the call found an error
//   k_host_job            hostAllocatorJob.Run past the allocator: single-task bypass, report, drawdown (units/host_allocator.go:180-425)
//   k_next_verdict/serve  the DAG dispatcher's FindNextTask, a warp per distro (model/task_queue_service_dependency.go:258-692)
// No CPU fallback exists in this file: without a device every entry point fails.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <type_traits>
#include <cstdlib>
#include <future>
#include <mutex>
#include <string>
#include <vector>

#include "evg_score.cuh"
#include "evg_intern.h"

using namespace evg;

// --------------------------------------------------------------------------
// host-side helpers
// --------------------------------------------------------------------------
namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

// The CSR offset tables of the C boundary are indexed directly, so each is checked before its first use: off[0 .. n] starts
// at 0, never decreases, ends at `total` (< 0: its last entry is the count); the error names `who`, `name` and the bad row.
int check_offsets(const int64_t* off, int64_t n, int64_t total, const char* who, const char* name) {
  int64_t row = off[0] != 0 ? 0 : -1;
  for (int64_t i = 0; row < 0 && i < n; i++)
    if (off[i + 1] < off[i]) row = i + 1;
  if (row < 0 && total >= 0 && off[n] != total) row = n;
  if (row < 0) return EVG_OK;
  return fail(EVG_ERR_INVALID, "%s: %s[%lld] = %lld breaks the offsets (they start at 0, never decrease and end at %s)", who, name,
              (long long)row, (long long)off[row], total >= 0 ? std::to_string(total).c_str() : "the count");
}

#define CK(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return fail(e_ == cudaErrorMemoryAllocation ? EVG_ERR_NOMEM : EVG_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                  cudaGetErrorString(e_), __FILE__, __LINE__);                                \
  } while (0)

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  bool owned = true;  // false: p is caller-owned device memory (evg_upload_device)
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p && owned) cudaFree(p);
  }
  void adopt(void* q) {
    if (owned && p) cudaFree(p);
    p = q; cap = 0; owned = false;
  }
  void swap(DevBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
    std::swap(owned, o.owned);
  }
  cudaError_t ensure(size_t bytes) {
    if (!owned) { p = nullptr; cap = 0; owned = true; }
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) return e;
    cap = want;
    return cudaSuccess;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// Grow `buf` to `count` elements of `type` (at least one) and copy them from host memory at `ptr` on stream `st`.
#define UP(st, buf, ptr, count, type)                                                                             \
  do {                                                                                                            \
    CK((buf).ensure(sizeof(type) * size_t((count) > 0 ? (count) : 1)));                                           \
    if ((count) > 0) CK(cudaMemcpyAsync((buf).p, (ptr), sizeof(type) * size_t(count), cudaMemcpyHostToDevice, st)); \
  } while (0)

// The planner's size classes.  upload_tasks routes every distro to one (route_of); each class has its own list.
enum Route : int {
  kWarp,                    // <= 32 tasks: k_plan_warp
  kGeneral,                 // the general path
  kSmemA, kSmemB, kSmemC,   // k_plan_smem's classes
  kCtaA, kCtaB, kCtaC,      // k_plan_cta's classes (kCtaA: the <128,1280> and <64,384> instances)
  kRoutes,
  kPunted = kRoutes,        // not a list: the distros the k_plan_cta classes hand back, replanned by k_plan_smem
};
constexpr bool is_cta(int r) { return r == kCtaA || r == kCtaB || r == kCtaC; }
// the resident tick launches the on-chip classes largest distro first (upload_tasks keeps a second copy of their lists)
constexpr bool largest_first(int r) { return r != kWarp && r != kGeneral; }
// the resident tick's stream of each class (kPunted runs behind the k_plan_cta classes)
constexpr int kRouteStream[kRoutes + 1] = {4, 5, 3, 2, 1, 0, 0, 0, 0};

// on-chip planner classes <THREADS, ITEMS>: capacity = THREADS*ITEMS tasks per distro
constexpr int kThreadsC = 1024, kItemsC = 12;  // the largest class: 12288 tasks in 218 KB
constexpr int kCapA = 128 * 8, kCapB = 256 * 16, kCapC = kThreadsC * kItemsC;
constexpr int64_t kWideAllocGroups = 1024;  // k_alloc<128> (a block per distro) once some distro has more task groups
constexpr int kCapW = 32;  // k_plan_warp: one warp per distro
constexpr int64_t kGrouplessHosts = 64;  // k_alloc_groupless walks a distro's hosts with one thread: only short walks
constexpr int64_t kBigUnitTasks = 128;  // GroupVersions distros above this size in k_plan_smem's smallest class count as a class of their own
constexpr int64_t kSparseClass = 64;  // a k_plan_smem class of 1025+ task distros with fewer members than this goes to the general path
// second-generation on-chip planner classes <THREADS, CAP, CTAs per SM> (evg_plan_cta.cuh)
constexpr int kNT_A = 128, kNCapA = 1280, kNOccA = 8;
// the smallest k_plan_cta class: a launch list's distros of at most 384 tasks (and few task groups) take 64-thread CTAs,
// sixteen per SM -- twice the distros in flight (configs[3] "total": 10 000 distros of 100 tasks)
constexpr int kNT_S = 64, kNCapS = 384, kNOccS = 16;
constexpr int kNT_B = 256, kNCapB = 5120, kNOccB = 4;
constexpr int kNT_C = 512, kNCapC = 10240, kNOccC = 2;
constexpr uint32_t kInactive = 0xFFFFFFFFu;  // next[]: pair not linked / head[]: empty list
constexpr uint32_t kEnd = 0xFFFFFFFEu;       // next[]: end of list
constexpr uint32_t kNoAnchor = 0xFFFFFFFFu;
// k_gs_wave: a wave whose largest symMerge call spans more tasks than this rotates with a CTA per call, otherwise a warp
constexpr int64_t kGsWarpRotation = 1024;
// Columns are padded so that 128-bit loads and TMA copies that start inside the table may run past its last row.
constexpr int64_t kColPad = 8;

}  // namespace

// --------------------------------------------------------------------------
// device-side views
// --------------------------------------------------------------------------
struct DTasks {
  int64_t n, n_edges;
  const int32_t* priority;
  const int64_t* expected;
  const int64_t* qbasis;
  const int64_t* wbasis;
  const int32_t* numdep;
  const int32_t* tgo;
  const int32_t* gid;
  const int32_t* vid;
  const uint32_t* flags;
  const int64_t* dep_off;
  const int32_t* dep_idx;
};

struct EdDst {  // the shadow column set the composed table is written to
  int32_t *priority, *numdep, *tgo, *gid, *vid;
  uint32_t* flags;
  int64_t *expected, *qbasis, *wbasis;
};

struct DDistros {
  int32_t n;
  const int64_t* task_off;
  const int64_t* group_off;
  const evg_distro_cfg* cfg;
  const int32_t* gmax;
  const int64_t* unit_base;  // n+1: first unit slot of each distro
};

struct SortBuf {
  uint64_t* key_v;  // [T] k_plan_smem: Vmax - V of a distro whose value range exceeds 32 bits
};

struct DWork {
  uint8_t* has_dep;      // [T]
  uint32_t* head;        // [unit slots]
  uint32_t* next;        // [2T+E]
  uint32_t* pair_slot;   // [2T+E]
  uint32_t* edge_task;   // [E]
  uint8_t* edge_live;    // [E] on-chip path: 1 = edge pair linked (not a duplicate membership)
  const uint8_t* route;  // [D] 1 = distro planned by k_plan_smem (general kernels skip it)
  int* err;              // [1] set by k_validate when a distro-local id is out of range; planners then do nothing
  int64_t* unit_v;       // [unit slots] on-chip path: TotalValue of the unit; general path: id | run start << 32 (slot_unit)
  uint32_t* unit_a;      // [unit slots] anchor
  uint32_t* unit_n;      // [unit slots] member count
  unsigned long long* unit_mask;  // [unit slots] ranks emitted from the unit (units of <= 64 members)
  uint32_t* best_pair;   // [T]
  SortBuf buf[1];
  evg_queue_info* qinfo; // [D]
  evg_group_info* ginfo; // [G]
};

struct DHosts {
  int64_t n;
  const uint32_t* flags;
  const int32_t* gid;
  const int64_t* expected;
  const int64_t* stddev;
  const int64_t* start;
  const int64_t* host_off;
  const evg_alloc_cfg* cfg;
};

// --------------------------------------------------------------------------
// device helpers
// --------------------------------------------------------------------------
__device__ __forceinline__ int find_distro(const int64_t* __restrict__ off, int lo, int hi, int64_t t) {
  // largest d in [lo, hi] with off[d] <= t  (off[lo] <= t guaranteed)
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Block-cooperative distro lookup: thread 0 / last thread bracket the block's
// range, then each thread searches only inside the bracket.
__device__ __forceinline__ int block_find_distro(const int64_t* __restrict__ off, int n_distros, int64_t t,
                                                 int64_t n_items) {
  __shared__ int s_lo, s_hi;
  int64_t first = int64_t(blockIdx.x) * blockDim.x;
  if (threadIdx.x == 0) s_lo = find_distro(off, 0, n_distros - 1, first);
  if (threadIdx.x == blockDim.x - 1) {
    int64_t last = first + blockDim.x - 1;
    if (last >= n_items) last = n_items - 1;
    s_hi = find_distro(off, 0, n_distros - 1, last);
  }
  __syncthreads();
  if (t >= n_items) return -1;
  return find_distro(off, s_lo, s_hi, t);
}

// One pass of a segmented stable merge sort, one thread per element: inside each segment [off[d], off[d+1]) of src,
// runs of length L are merged pairwise into dst.  An element of a left run goes after the sibling run's elements that
// sort strictly before it, one of a right run after those that do not sort after it: equal elements keep their order.
// The total off[n_segs] is read here, so the grid may be sized by any bound above it.  Order::pivot(d, base, me) reads
// what it needs of `me` once and answers before(x) ("x sorts strictly before me") and after(x) ("strictly after").
template <class Order>
__global__ void __launch_bounds__(256) k_seg_merge_pass(Order order, const int64_t* __restrict__ off, int32_t n_segs,
                                                        const typename Order::Elem* __restrict__ src,
                                                        typename Order::Elem* __restrict__ dst, int64_t L) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, n_segs, p, off[n_segs]);
  if (d < 0) return;
  const int64_t base = off[d], n = off[d + 1] - base, q = p - base;
  const typename Order::Elem me = src[p];
  if (L >= n) { dst[p] = me; return; }
  const int64_t r = q / L, own0 = r * L;
  const bool left = (r & 1) == 0;
  const int64_t s0 = left ? own0 + L : own0 - L, s1 = left ? min(s0 + L, n) : own0;  // the sibling run
  if (s0 >= n) { dst[p] = me; return; }  // a last left run without a sibling is copied
  const auto pv = order.pivot(d, base, me);
  int64_t lo = s0, hi = s1;
  if (left) {  // the merged pair starts at own0: q - own0 of the own run and lo - s0 of the sibling's go first
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (pv.before(src[base + m])) lo = m + 1; else hi = m; }
    dst[base + q + (lo - s0)] = me;
  } else {     // the merged pair starts at s0: lo - s0 of the sibling's and q - own0 of the own run go first
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (!pv.after(src[base + m])) lo = m + 1; else hi = m; }
    dst[base + lo + (q - own0)] = me;
  }
}

__device__ __forceinline__ int64_t warp_sum64(int64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Inclusive prefix sum of v over the lanes of a full warp (T: uint32_t, int64_t or uint64_t).
template <class T>
__device__ __forceinline__ T warp_scan_incl(T v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  return v;
}

__device__ __forceinline__ uint32_t warp_add(uint32_t v) { return __reduce_add_sync(0xffffffffu, v); }
__device__ __forceinline__ uint64_t warp_add(uint64_t v) { return uint64_t(warp_sum64(int64_t(v))); }

// Exclusive prefix sum of v over a block of NW full warps, and the block's total in *total when asked.  Every thread of
// the block calls it.  s_warp is NW entries of shared memory the caller owns: the helper writes it before its first
// barrier and reads it after its last, so a __syncthreads() must separate this call from any earlier read of s_warp
// and from any later write to it (another scan included).  Up to 8 warps one barrier suffices: lane w reads warp w's
// total and each warp adds up those of the warps before it (one load a thread, where reading all NW in turn costs the
// on-chip planners spills); above that warp 0 scans the totals and a second barrier publishes them.
template <int NW, class T>
__device__ __forceinline__ T block_scan_excl(T v, T* s_warp, T* total = nullptr) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T inc = warp_scan_incl(v);
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  T before = 0;
  if constexpr (NW <= 8) {
    const T x = lane < NW ? s_warp[lane] : T(0);
    before = warp_add(lane < warp ? x : T(0));
    if (total) *total = warp_add(x);
  } else {
    if (warp == 0) {  // s_warp[w] becomes the total of warps 0 .. w
      const T x = warp_scan_incl(lane < NW ? s_warp[lane] : T(0));
      if (lane < NW) s_warp[lane] = x;
    }
    __syncthreads();
    if (warp > 0) before = s_warp[warp - 1];
    if (total) *total = s_warp[NW - 1];
  }
  return before + inc - v;
}

// One block of 1024 threads scans a[0 .. n) in place (exclusive), 1024 entries at a time with a carry, and returns the
// total.
template <class T>
__device__ T block_scan_segment(T* a, int64_t n) {
  __shared__ T s_warp[32];
  T carry = 0;
  for (int64_t c0 = 0; c0 < n; c0 += 1024) {
    const int64_t i = c0 + threadIdx.x;
    const T v = i < n ? a[i] : T(0);
    T chunk;
    const T ex = block_scan_excl<32>(v, s_warp, &chunk);
    if (i < n) a[i] = carry + ex;
    carry += chunk;
    __syncthreads();  // s_warp is rewritten by the next chunk
  }
  return carry;
}

__device__ __forceinline__ void atomic_add64(int64_t* p, int64_t v) {
  if (v != 0) atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}

// unit slot (distro-local) a task is filed under by its id key (planner.go:434-445)
__device__ __forceinline__ uint32_t own_slot_local(int32_t gid, int32_t vid, uint32_t local_idx, uint32_t n_groups,
                                                   bool group_versions) {
  if (gid >= 0) return uint32_t(gid);
  return n_groups + (group_versions ? uint32_t(vid) : local_idx);
}

__device__ __forceinline__ void link_pair(DWork& W, uint32_t pair, uint32_t slot) {
  W.pair_slot[pair] = slot;
  uint32_t prev = atomicExch(W.head + slot, pair);
  W.next[pair] = (prev == kInactive) ? kEnd : prev;
}

__device__ __forceinline__ uint32_t pair_task(const DTasks& T, const DWork& W, uint32_t p) {
  if (p < uint32_t(T.n)) return p;
  if (p < uint32_t(2 * T.n)) return p - uint32_t(T.n);
  return W.edge_task[p - uint32_t(2 * T.n)];
}

#include "evg_plan_smem.cuh"
#include "evg_plan_warp.cuh"
#include "evg_plan_cta.cuh"
#include "evg_plan_general.cuh"
#include "evg_legacy.cuh"
#include "evg_dag.cuh"
#include "evg_next.cuh"
#include "evg_estimate.cuh"

// --------------------------------------------------------------------------
// kernels (general path: any distro size)
// --------------------------------------------------------------------------

// Distro-local ids index device tables directly, so they are range-checked once per upload:
// group_id in [-1, n_groups), version_id in [0, n_versions), dep_idx in [0, tasks of the distro).
__global__ void __launch_bounds__(256) k_validate(DTasks T, DDistros D, DWork W, int64_t t_begin, int64_t t_end) {
  const int64_t t = t_begin + int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= t_end) return;
  const int d = find_distro(D.task_off, 0, D.n - 1, t);
  const int64_t tn = D.task_off[d + 1] - D.task_off[d];
  const int64_t ng = D.group_off[d + 1] - D.group_off[d];
  const int32_t gid = T.gid[t], vid = T.vid[t];
  bool bad = gid < -1 || gid >= ng || vid < 0 || vid >= D.cfg[d].n_versions;
  if (T.n_edges > 0) {
    const int64_t e0 = T.dep_off[t], e1 = T.dep_off[t + 1];
    bad = bad || e1 < e0 || e0 < 0 || e1 > T.n_edges;
    if (!bad)
      for (int64_t e = e0; e < e1; e++) bad = bad || T.dep_idx[e] < 0 || T.dep_idx[e] >= tn;
  }
  if (bad) atomicOr(W.err, 1);
}

// Task.DependenciesMet over direct dependencies (model/task/task.go:529-543,632-671).
struct DDeps {
  int64_t n_tasks, n_deps;
  const int64_t* dep_off;
  const uint8_t* dep_kind;
  const int32_t* dep_ref;
  const uint8_t* dep_want;
  const uint8_t* task_state;
  const uint8_t* task_pre;
  const uint8_t* ext_state;
  int64_t n_ext;
};
// deps->dep_off is checked by the first kernel that reads a row (k_deps_met, k_pl_deps): a row outside [0, n_deps] or
// decreasing sets this bit of the error word and is not walked.  Bit 1 there: a dep_ref (or a finder's project row), 2: a status id.
constexpr int kErrDepOff = 4;
__device__ __forceinline__ bool deps_row_bad(const DDeps& X, int64_t e0, int64_t e1) { return e0 < 0 || e1 < e0 || e1 > X.n_deps; }
// met[t] bit 0: Task.DependenciesMet (with the HasDependenciesMet short-circuit); with `both`, bit 1:
// Task.AllDependenciesSatisfied (task.go:795-821: the same walk without the short-circuit).
__global__ void __launch_bounds__(256) k_deps_met(DDeps X, uint8_t* met, int* err, int both, const int64_t* __restrict__ dep_fin,
                                                  int64_t now, int64_t* __restrict__ met_time) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= X.n_tasks) return;
  const int64_t e0 = X.dep_off[t], e1 = X.dep_off[t + 1];
  bool ok = !deps_row_bad(X, e0, e1);  // a bad row is walked nowhere below
  if (!ok) atomicOr(err, kErrDepOff);
  const bool shortcut = (X.task_pre[t] & (EVG_TP_OVERRIDE | EVG_TP_MET_TIME)) != 0;  // HasDependenciesMet task.go:3393
  if (ok && e1 > e0 && (both || !shortcut)) {
    for (int64_t e = e0; e < e1 && ok; e++) {
      const uint8_t kind = X.dep_kind[e];
      const int32_t ref = X.dep_ref[e];
      uint8_t st;
      if (kind == EVG_DEP_IN_QUEUE) {
        if (ref < 0 || ref >= X.n_tasks) { atomicOr(err, 1); ok = false; break; }
        st = X.task_state[ref];
      } else if (kind == EVG_DEP_EXTERNAL) {
        if (ref < 0 || ref >= X.n_ext) { atomicOr(err, 1); ok = false; break; }
        st = X.ext_state[ref];
      } else {
        ok = false;  // lookup error -> false (scheduler.go:161-168)
        break;
      }
      const uint32_t status = st & EVG_TS_STATUS_MASK;
      switch (X.dep_want[e]) {  // SatisfiesDependency task.go:529-543
        case EVG_WANT_SUCCESS: ok = status == 0; break;
        case EVG_WANT_FAILED: ok = status == 1; break;
        case EVG_WANT_ANY: ok = status < 2 || (st & EVG_TS_BLOCKED); break;
        default: ok = false;
      }
    }
  }
  met[t] = uint8_t(((ok || shortcut) ? 1 : 0) | ((both && ok) ? 2 : 0));
  if (met_time) {
    // a fresh evaluation that comes out met stamps DependenciesMetTime (setDependenciesMetTime, task.go:653,673-684):
    // the latest non-zero FinishedAt of the dependencies (utility.IsZeroTime: Go's zero time or the Unix epoch), else now
    int64_t stamp = EVG_TIME_ZERO;
    if (ok && !shortcut && e1 > e0) {
      if (dep_fin)
        for (int64_t e = e0; e < e1; e++) {
          const int64_t f = dep_fin[e];
          if (f != EVG_TIME_ZERO && f != 0 && f > stamp) stamp = f;
        }
      if (stamp == EVG_TIME_ZERO || stamp == 0) stamp = now;
    }
    met_time[t] = stamp;
  }
}

// The resident planner inputs take the device's own verdict: the EVG_TF_DEPS_MET bit of every task, and for freshly
// stamped tasks the later of the wait basis the caller gave (ScheduledTime) and the stamp (scheduler.go:119-122).
__global__ void __launch_bounds__(256) k_apply_deps(int64_t n, const uint8_t* __restrict__ met, const int64_t* __restrict__ met_time,
                                                    uint32_t* __restrict__ flags, int64_t* __restrict__ wbasis) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  flags[t] = (flags[t] & ~EVG_TF_DEPS_MET) | ((met[t] & 1) ? EVG_TF_DEPS_MET : 0u);
  const int64_t s = met_time[t];
  if (s != EVG_TIME_ZERO && s > wbasis[t]) wbasis[t] = s;
}

// The task finders' filter (task_finder.go:40-197) with a stable per-distro compaction: one block per distro,
// 256 tasks per step, ballot + warp totals for the positions.
struct DRunnable {
  int64_t n_tasks;
  int32_t n_distros, n_projects;
  const int64_t* task_off;
  const uint8_t* sched;
  const int32_t* project;
  const uint8_t* project_flags;
  const int64_t* valid_off;
  const int32_t* valid_idx;
  const uint8_t* finder;
  const uint8_t* met;  // k_deps_met(both) output, or nullptr
};
__global__ void __launch_bounds__(256) k_runnable(DRunnable R, int32_t* __restrict__ out, int64_t* __restrict__ count, int* err) {
  constexpr int ITEMS = 4;  // candidates per thread and step: their loads are in flight together, one barrier pair per 1024
  const int d = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned full = 0xffffffffu;
  const int64_t base = R.task_off[d], end = R.task_off[d + 1];
  const int64_t v0 = R.valid_off[d], v1 = R.valid_off[d + 1];
  const uint32_t finder = R.finder[d];
  const uint32_t met_bit = finder == EVG_FINDER_LEGACY ? 1u : 2u;
  __shared__ uint32_t s_cnt[ITEMS * 8];  // survivors of (item j, warp w), in output order j-major
  int64_t running = 0;  // kept identically by every thread
  for (int64_t c0 = base; c0 < end; c0 += 256 * ITEMS) {
    uint32_t sq[ITEMS], mt[ITEMS];
    int32_t pj[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const int64_t t = c0 + j * 256 + threadIdx.x;
      const bool in = t < end;
      sq[j] = in ? R.sched[t] : 0u;
      pj[j] = in ? R.project[t] : -1;
      mt[j] = (in && finder != EVG_FINDER_NO_DEPS) ? R.met[t] : 3u;
    }
    bool keep[ITEMS];
    unsigned m[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const uint32_t q = sq[j];
      // schedulableHostTasksQuery (model/task/db.go:671-689)
      bool k = (q & EVG_SQ_ACTIVATED) && (q & EVG_SQ_UNDISPATCHED) && (q & EVG_SQ_PRIORITY_OK) && (q & EVG_SQ_HOST_PLATFORM) &&
               (!(q & EVG_SQ_UNATTAINABLE) || (q & EVG_SQ_OVERRIDE_DEPS));
      const int32_t p = pj[j];
      if (p >= R.n_projects) { atomicOr(err, 1); k = false; }
      else if (p < 0) k = false;  // "could not find project for task" (task_finder.go:57-67)
      else if (k) {
        const uint32_t pf = R.project_flags[p];
        // ProjectCanDispatchTask (model/project_ref.go:3441-3462)
        if (!(pf & EVG_PF_ENABLED) && !((q & EVG_SQ_GITHUB_PR) && (pf & EVG_PF_HIDDEN))) k = false;
        if (pf & EVG_PF_DISPATCHING_DISABLED) k = false;
        if ((q & EVG_SQ_PATCH_REQUEST) && (pf & EVG_PF_PATCHING_DISABLED)) k = false;
        if (k && v1 > v0) {  // len(d.ValidProjects) > 0 && !contains(ref.Id) (task_finder.go:74-84)
          bool found = false;
          for (int64_t x = v0; x < v1 && !found; x++) found = R.valid_idx[x] == p;
          k = found;
        }
        if (k) k = (mt[j] & met_bit) != 0;  // the finder's dependency predicate (NO_DEPS reads 3: always met)
      }
      keep[j] = k;
      m[j] = __ballot_sync(full, k);
      if (lane == 0) s_cnt[j * 8 + warp] = __popc(m[j]);
    }
    __syncthreads();
    uint32_t total = 0, before[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
#pragma unroll
      for (int w = 0; w < 8; w++) {
        if (w == warp) before[j] = total;
        total += s_cnt[j * 8 + w];
      }
    }
#pragma unroll
    for (int j = 0; j < ITEMS; j++)
      if (keep[j]) out[base + running + before[j] + __popc(m[j] & ((1u << lane) - 1u))] = int32_t(c0 + j * 256 + threadIdx.x - base);
    running += total;
    __syncthreads();
  }
  for (int64_t i = base + running + threadIdx.x; i < end; i += 256) out[i] = -1;  // unused tail of the distro's slots
  if (threadIdx.x == 0) count[d] = running;
}
// k_runnable's filter (EVG_FINDER_NO_DEPS / LEGACY / ALTERNATE) for one candidate, as k_runnable_pipe applies it.
__device__ __forceinline__ bool finder_keep(const DRunnable& R, uint32_t q, int32_t p, uint32_t mt, uint32_t met_bit, int64_t v0,
                                            int64_t v1, int* err) {
  // schedulableHostTasksQuery (model/task/db.go:671-689)
  bool k = (q & EVG_SQ_ACTIVATED) && (q & EVG_SQ_UNDISPATCHED) && (q & EVG_SQ_PRIORITY_OK) && (q & EVG_SQ_HOST_PLATFORM) &&
           (!(q & EVG_SQ_UNATTAINABLE) || (q & EVG_SQ_OVERRIDE_DEPS));
  if (p >= R.n_projects) { atomicOr(err, 1); k = false; }
  else if (p < 0) k = false;  // "could not find project for task" (task_finder.go:57-67)
  else if (k) {
    const uint32_t pf = R.project_flags[p];
    // ProjectCanDispatchTask (model/project_ref.go:3441-3462)
    if (!(pf & EVG_PF_ENABLED) && !((q & EVG_SQ_GITHUB_PR) && (pf & EVG_PF_HIDDEN))) k = false;
    if (pf & EVG_PF_DISPATCHING_DISABLED) k = false;
    if ((q & EVG_SQ_PATCH_REQUEST) && (pf & EVG_PF_PATCHING_DISABLED)) k = false;
    if (k && v1 > v0) {  // len(d.ValidProjects) > 0 && !contains(ref.Id) (task_finder.go:74-84)
      bool found = false;
      for (int64_t x = v0; x < v1 && !found; x++) found = R.valid_idx[x] == p;
      k = found;
    }
    if (k) k = (mt & met_bit) != 0;  // the finder's dependency predicate (NO_DEPS reads 3: always met)
  }
  return k;
}
// The pipeline finder's filter (task.FindHostRunnable, model/task/db.go:887-1066) for one candidate: the same base query
// and ValidProjects match, the RAW project_ref document (filterDisabledProjects / filterPatchingDisabledProjects,
// :1030-1048: no hidden-project exemption; patching_disabled must be stored false), and for EVG_FINDER_PIPELINE the
// $graphLookup verdict, bit 2 of k_deps_met's byte (k_pl_deps).
__device__ __forceinline__ bool pipeline_keep(const DRunnable& R, const uint8_t* __restrict__ praw, uint32_t q, int32_t p, uint32_t mt,
                                              uint32_t finder, int64_t v0, int64_t v1, int* err) {
  bool k = (q & EVG_SQ_ACTIVATED) && (q & EVG_SQ_UNDISPATCHED) && (q & EVG_SQ_PRIORITY_OK) && (q & EVG_SQ_HOST_PLATFORM) &&
           (!(q & EVG_SQ_UNATTAINABLE) || (q & EVG_SQ_OVERRIDE_DEPS));
  if (p >= R.n_projects) { atomicOr(err, 1); k = false; }
  else if (p < 0) k = false;  // the $lookup finds no project_ref: project_ref.0.enabled is missing
  else if (k) {
    const uint32_t pr = praw[p];
    if (!(pr & EVG_PR_ENABLED) || (pr & EVG_PR_DISPATCHING_DISABLED)) k = false;
    if ((q & EVG_SQ_PATCH_REQUEST) && !(pr & EVG_PR_PATCHING_FALSE)) k = false;  // Requester $in PatchRequesters
    if (k && v1 > v0) {  // filterInvalidDistros: project $in ValidProjects (db.go:1031-1033)
      bool found = false;
      for (int64_t x = v0; x < v1 && !found; x++) found = R.valid_idx[x] == p;
      k = found;
    }
    if (k && finder == EVG_FINDER_PIPELINE) k = (mt & 4u) != 0;
  }
  return k;
}
// k_runnable with the pipeline finder's codes (evg_find_runnable_ex / evg_plan_from_finder_ex with an evg_pipeline_in;
// praw: evg_pipeline_in.project_raw).  The same compaction; k_runnable itself is left as it was, so that its code does
// not change for the callers that never use the pipeline.
__global__ void __launch_bounds__(256) k_runnable_pipe(DRunnable R, const uint8_t* __restrict__ praw, int32_t* __restrict__ out,
                                                       int64_t* __restrict__ count, int* err) {
  constexpr int ITEMS = 4;  // candidates per thread and step: their loads are in flight together, one barrier pair per 1024
  const int d = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned full = 0xffffffffu;
  const int64_t base = R.task_off[d], end = R.task_off[d + 1];
  const int64_t v0 = R.valid_off[d], v1 = R.valid_off[d + 1];
  const uint32_t finder = R.finder[d];
  const uint32_t met_bit = finder == EVG_FINDER_LEGACY ? 1u : 2u;
  const bool reads_met = finder != EVG_FINDER_NO_DEPS && finder != EVG_FINDER_PIPELINE_NO_DEPS;
  __shared__ uint32_t s_cnt[ITEMS * 8];  // survivors of (item j, warp w), in output order j-major
  int64_t running = 0;  // kept identically by every thread
  for (int64_t c0 = base; c0 < end; c0 += 256 * ITEMS) {
    uint32_t sq[ITEMS], mt[ITEMS];
    int32_t pj[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const int64_t t = c0 + j * 256 + threadIdx.x;
      const bool in = t < end;
      sq[j] = in ? R.sched[t] : 0u;
      pj[j] = in ? R.project[t] : -1;
      mt[j] = (in && reads_met) ? R.met[t] : 3u;
    }
    bool keep[ITEMS];
    unsigned m[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      bool k;
      if (finder > EVG_FINDER_ALTERNATE) k = pipeline_keep(R, praw, sq[j], pj[j], mt[j], finder, v0, v1, err);
      else k = finder_keep(R, sq[j], pj[j], mt[j], met_bit, v0, v1, err);
      keep[j] = k;
      m[j] = __ballot_sync(full, k);
      if (lane == 0) s_cnt[j * 8 + warp] = __popc(m[j]);
    }
    __syncthreads();
    uint32_t total = 0, before[ITEMS];
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
#pragma unroll
      for (int w = 0; w < 8; w++) {
        if (w == warp) before[j] = total;
        total += s_cnt[j * 8 + w];
      }
    }
#pragma unroll
    for (int j = 0; j < ITEMS; j++)
      if (keep[j]) out[base + running + before[j] + __popc(m[j] & ((1u << lane) - 1u))] = int32_t(c0 + j * 256 + threadIdx.x - base);
    running += total;
    __syncthreads();
  }
  for (int64_t i = base + running + threadIdx.x; i < end; i += 256) out[i] = -1;  // unused tail of the distro's slots
  if (threadIdx.x == 0) count[d] = running;
}
// The pipeline's dependency filter (model/task/db.go:923-996, with removeDeps): met[t] |= 4 when t survives it.  The
// $graphLookup finds the existing documents among the DependsOn ids, the two $unwinds and matchIds pair each entry with
// its own document, and $group / $redact keep t iff every such pair is satisfied -- the entry's status string equals
// the document's, or it is "*" and the document is success / failed or has an unattainable depends_on entry.  An entry
// without a document pairs with nothing; a t whose entries ALL lack one leaves no row and is dropped; a t without
// DependsOn is kept (both sides of matchIds are missing, which compares equal).  err bit 2: a status id out of range.
struct DPipe {
  int32_t n_status;
  const int32_t* dep_status;
  const int32_t* task_status;
  const int32_t* ext_status;
  const uint8_t* task_unatt;
  const uint8_t* ext_unatt;
};
__global__ void __launch_bounds__(256) k_pl_deps(DDeps X, DPipe P, uint8_t* __restrict__ met, int* err) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= X.n_tasks) return;
  const int64_t e0 = X.dep_off[t], e1 = X.dep_off[t + 1];
  if (deps_row_bad(X, e0, e1)) { atomicOr(err, kErrDepOff); return; }
  const int32_t own = P.task_status[t];
  bool ok = true, paired = false;
  if (own < 0 || own >= P.n_status) { atomicOr(err, 2); ok = false; }
  for (int64_t e = e0; e < e1 && ok; e++) {
    const uint8_t kind = X.dep_kind[e];
    const int32_t ref = X.dep_ref[e];
    int32_t st;
    bool un;
    if (kind == EVG_DEP_IN_QUEUE) {
      if (ref < 0 || ref >= X.n_tasks) { atomicOr(err, 1); ok = false; break; }
      st = P.task_status[ref]; un = P.task_unatt[ref] != 0;
    } else if (kind == EVG_DEP_EXTERNAL) {
      if (ref < 0 || ref >= X.n_ext) { atomicOr(err, 1); ok = false; break; }
      st = P.ext_status[ref]; un = P.ext_unatt[ref] != 0;
    } else {
      continue;  // no document with that id: the entry pairs with nothing
    }
    const int32_t w = P.dep_status[e];
    if (w < 0 || w >= P.n_status || st < 0 || st >= P.n_status) { atomicOr(err, 2); ok = false; break; }
    paired = true;
    ok = w == st || (w == EVG_STATUS_ANY && (st == EVG_STATUS_SUCCESS || st == EVG_STATUS_FAILED || un));
  }
  if (ok && (paired || e1 == e0)) met[t] |= 4u;
}

// What the planner receives from a pipeline distro, once the keep mask exists (evg_plan_from_finder_ex):
//   EVG_FINDER_PIPELINE: the decoded task has no DependsOn, so HasDependenciesMet holds (task.go:3393-3395): met, no stamp;
//   EVG_FINDER_PIPELINE_NO_DEPS: Task.DependenciesMet (task.go:632-671) as k_deps_met's bit 0 and stamp, except that a
//     dependency that is a kept candidate of the same distro comes from the finder's output, whose depends_on.unattainable
//     was projected away (db.go:916-921): it is never Blocked().
// Other finders' rows are left as k_deps_met wrote them.
__global__ void __launch_bounds__(256) k_pl_plan(DDeps X, int32_t D, const int64_t* __restrict__ off, const uint8_t* __restrict__ finder,
                                                 const int32_t* __restrict__ keep, uint8_t* __restrict__ met,
                                                 const int64_t* __restrict__ dep_fin, int64_t now, int64_t* __restrict__ met_time) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, t, X.n_tasks);
  if (d < 0) return;
  const uint32_t f = finder[d];
  if (f == EVG_FINDER_PIPELINE) {
    met[t] |= 1u;
    met_time[t] = EVG_TIME_ZERO;
    return;
  }
  if (f != EVG_FINDER_PIPELINE_NO_DEPS) return;
  const int64_t e0 = X.dep_off[t], e1 = X.dep_off[t + 1], lo = off[d], hi = off[d + 1];
  const bool shortcut = (X.task_pre[t] & (EVG_TP_OVERRIDE | EVG_TP_MET_TIME)) != 0;
  bool ok = true;
  if (e1 > e0 && !shortcut) {
    for (int64_t e = e0; e < e1 && ok; e++) {
      const int32_t ref = X.dep_ref[e];
      uint8_t st;
      if (X.dep_kind[e] == EVG_DEP_IN_QUEUE) {  // dep_ref was range-checked by k_deps_met
        st = X.task_state[ref];
        if (ref >= lo && ref < hi && keep[ref]) st &= ~EVG_TS_BLOCKED;
      } else if (X.dep_kind[e] == EVG_DEP_EXTERNAL) {
        st = X.ext_state[ref];
      } else {
        ok = false;
        break;
      }
      const uint32_t status = st & EVG_TS_STATUS_MASK;
      switch (X.dep_want[e]) {
        case EVG_WANT_SUCCESS: ok = status == 0; break;
        case EVG_WANT_FAILED: ok = status == 1; break;
        case EVG_WANT_ANY: ok = status < 2 || (st & EVG_TS_BLOCKED); break;
        default: ok = false;
      }
    }
  }
  met[t] = uint8_t((met[t] & ~1u) | ((ok || shortcut) ? 1u : 0u));
  int64_t stamp = EVG_TIME_ZERO;
  if (ok && !shortcut && e1 > e0) {
    if (dep_fin)
      for (int64_t e = e0; e < e1; e++) {
        const int64_t fin = dep_fin[e];
        if (fin != EVG_TIME_ZERO && fin != 0 && fin > stamp) stamp = fin;
      }
    if (stamp == EVG_TIME_ZERO || stamp == 0) stamp = now;
  }
  met_time[t] = stamp;
}

// The candidates' edges without those of EVG_FINDER_PIPELINE rows (whose DependsOn decodes empty): count, then (after a
// scan into new_off) copy.  The kept rows of the other finders keep their edges for compose_tick to re-index.
__global__ void __launch_bounds__(256) k_pl_edge_count(int64_t n, int32_t D, const int64_t* __restrict__ off, const uint8_t* __restrict__ finder,
                                                       const int64_t* __restrict__ dep_off, int32_t* __restrict__ cnt) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, t, n);
  if (d < 0) return;
  cnt[t] = finder[d] == EVG_FINDER_PIPELINE ? 0 : int32_t(dep_off[t + 1] - dep_off[t]);
}
__global__ void __launch_bounds__(256) k_pl_edge_write(int64_t n, const int64_t* __restrict__ dep_off, const int32_t* __restrict__ dep_idx,
                                                       const int64_t* __restrict__ new_off, int32_t* __restrict__ new_idx) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int64_t w = new_off[t], k = new_off[t + 1] - w, e0 = dep_off[t];
  for (int64_t j = 0; j < k; j++) new_idx[w + j] = dep_idx[e0 + j];
}

// Expected-duration statistics (model/task/expected_duration.go:36-96): the $match, then per key count / sum, then
// the squared deviations from floor(mean) as an exact 128-bit integer, then one rounding per output.
struct DDur {
  int64_t n_rows;
  int32_t n_keys;
  const int32_t* key;
  const int64_t* taken;
  const int64_t* start;
  const int64_t* finish;
  const uint8_t* flags;
  int64_t w0, w1;
  unsigned long long* cnt;  // [n_keys]
  unsigned long long* sum;  // [n_keys] two's complement
  unsigned long long* sq_lo;
  unsigned long long* sq_hi;
};
__device__ __forceinline__ bool dur_row_matches(const DDur& X, int64_t r) {
  const uint32_t f = X.flags[r];
  return (f & EVG_DR_COMPLETED) && !(f & EVG_DR_TIMED_OUT) && X.start[r] > X.w0 && X.finish[r] <= X.w1;
}
__global__ void __launch_bounds__(256) k_dur_sum(DDur X, int* err) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= X.n_rows) return;
  const int32_t k = X.key[r];
  if (k < 0 || k >= X.n_keys) { atomicOr(err, 1); return; }
  if (!dur_row_matches(X, r)) return;
  atomicAdd(X.cnt + k, 1ull);
  atomicAdd(X.sum + k, (unsigned long long)X.taken[r]);
}
__global__ void __launch_bounds__(256) k_dur_dev(DDur X) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= X.n_rows) return;
  const int32_t k = X.key[r];
  if (k < 0 || k >= X.n_keys || !dur_row_matches(X, r)) return;
  const int64_t n = int64_t(X.cnt[k]), s = int64_t(X.sum[k]);
  int64_t m0 = s / n;
  if ((s % n) < 0) m0 -= 1;  // floor
  const int64_t dv = X.taken[r] - m0;
  const unsigned long long a = dv < 0 ? (unsigned long long)(-dv) : (unsigned long long)dv;
  const unsigned long long lo = a * a, hi = __umul64hi(a, a);
  const unsigned long long old = atomicAdd(X.sq_lo + k, lo);
  const unsigned long long carry = (old + lo < old) ? 1ull : 0ull;
  if (hi + carry) atomicAdd(X.sq_hi + k, hi + carry);
}
__global__ void __launch_bounds__(256) k_dur_final(DDur X, evg_duration_stat* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= X.n_keys) return;
  evg_duration_stat st;
  st.count = int64_t(X.cnt[k]);
  st.mean_ns = 0.0;
  st.stddev_ns = 0.0;
  if (st.count > 0) {
    const int64_t n = st.count, s = int64_t(X.sum[k]);
    int64_t m0 = s / n, rem = s % n;
    if (rem < 0) { m0 -= 1; rem += n; }
    const double dn = __ll2double_rn(n);
    st.mean_ns = __ddiv_rn(__ll2double_rn(s), dn);
    // variance = S2/n - (rem/n)^2 with S2 = sum (x - floor(mean))^2 held exactly in 128 bits
    const double s2 = __dadd_rn(__dmul_rn(__ull2double_rn(X.sq_hi[k]), 18446744073709551616.0), __ull2double_rn(X.sq_lo[k]));
    const double fr = __ddiv_rn(__ll2double_rn(rem), dn);
    double var = __dadd_rn(__ddiv_rn(s2, dn), -__dmul_rn(fr, fr));
    if (var < 0.0) var = 0.0;
    st.stddev_ns = __dsqrt_rn(var);
  }
  out[k] = st;
}

// The duration cache of a resident tick (evg_resolve_durations).  Pair p's keys are pair_key_off[p] .. [p+1]: a task
// with DisplayName "" queries the pair without a name filter and gets one document only when ONE of them matched.
__global__ void __launch_bounds__(256) k_dur_pair(int32_t n_pairs, const int64_t* __restrict__ pair_key_off,
                                                  const unsigned long long* __restrict__ cnt, int32_t* __restrict__ single) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  int32_t k1 = -1;
  int n = 0;
  for (int64_t k = pair_key_off[p]; k < pair_key_off[p + 1] && n < 2; k++)
    if (cnt[k] > 0) { k1 = int32_t(k); n++; }
  single[p] = n == 1 ? k1 : -1;
}

// The listed rows of one call: tasks first (n_t), then hosts (n_h).  A NULL row list means rows 0 .. n-1.
struct DDurRows {
  int64_t n_t, n_h;
  const int64_t* trows;
  const int64_t* hrows;
  const int64_t* value;
  const int64_t* pstd;
  const int64_t* ttl;
  const int64_t* coll;
  const int64_t* exp;
  const int64_t* exp_std;
  const int32_t* key;
  int64_t *o_avg, *o_std, *o_value, *o_pstd, *o_coll;
  uint8_t* o_src;
};

// One listed row: FetchExpectedDuration with CachedDurationValue.Get and the refresher (task.go:3519-3590,
// cached_value.go:125-145) against the statistics of its key.  Out-of-range keys set bit 2 of *err.
__global__ void __launch_bounds__(256) k_dur_resolve(DDurRows R, int32_t n_keys, int32_t n_pairs, const evg_duration_stat* __restrict__ stat,
                                                     const int32_t* __restrict__ single, int64_t now, int* err) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= R.n_t + R.n_h) return;
  const int64_t value = R.value[i], pstd = R.pstd[i], coll = R.coll[i], e = R.exp[i];
  const int64_t ttl = R.ttl[i] == 0 ? 8 * kHour : R.ttl[i];  // predictionTTL (task.go:67), unjittered
  const int32_t key = R.key[i];
  int32_t doc = -1;  // the key whose statistics the window query returns as its one document
  if (key >= 0) {
    if (key >= n_keys) { atomicOr(err, 2); return; }
    if (stat[key].count > 0) doc = key;
  } else if (key != EVG_DK_NONE) {
    const int64_t p = -2 - int64_t(key);
    if (p >= n_pairs) { atomicOr(err, 2); return; }
    doc = single[p];
  }
  int64_t avg, sd, nv = value, ns = pstd, nc = coll;
  uint8_t src;
  if (value == 0 && e != 0) {  // backfill: Value and CollectedAt set, StdDev kept (task.go:3524-3538)
    avg = e; sd = R.exp_std[i]; nv = e; nc = now - kMinute;
    src = EVG_DS_BACKFILL;
  } else if (since(now, coll) < ttl) {
    avg = value; sd = pstd;
    src = EVG_DS_FRESH;
  } else {
    if (doc < 0) {
      src = value == 0 ? EVG_DS_DEFAULT : EVG_DS_PREVIOUS;
      avg = value == 0 ? 10 * kMinute : value; sd = value == 0 ? 0 : pstd;
    } else {
      const int64_t a = __double2ll_rz(stat[doc].mean_ns);  // time.Duration(float64) truncates toward zero
      src = a == 0 ? EVG_DS_DEFAULT : EVG_DS_HISTORY;
      avg = a == 0 ? 10 * kMinute : a; sd = a == 0 ? 0 : __double2ll_rz(stat[doc].stddev_ns);
    }
    nv = avg; ns = sd; nc = now;
  }
  R.o_avg[i] = avg; R.o_std[i] = sd; R.o_value[i] = nv; R.o_pstd[i] = ns; R.o_coll[i] = nc; R.o_src[i] = src;
}

// The resolved rows into the resident columns -- only when the call found no error, so a rejected call leaves the
// tick as it was without a host round trip in between.
__global__ void __launch_bounds__(256) k_dur_commit(DDurRows R, const int* __restrict__ err, int64_t* __restrict__ texp,
                                                    int64_t* __restrict__ hexp, int64_t* __restrict__ hstd) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= R.n_t + R.n_h || *err) return;
  if (i < R.n_t) {
    texp[R.trows ? R.trows[i] : i] = R.o_avg[i];
  } else {
    const int64_t j = i - R.n_t, r = R.hrows ? R.hrows[j] : j;
    hexp[r] = R.o_avg[i];
    hstd[r] = R.o_std[i];
  }
}

// The 13-field SortingValueBreakdown of the unit each ranked task was emitted
// from (planner.go:472-476, model/task/task.go:3990-4038); both paths.
__global__ void __launch_bounds__(256) k_breakdown(DTasks T, DDistros D, DWork W, const uint32_t* run_all, const URec* pay, const GUnit* units,
                                                   int64_t now, int any_complex, const int32_t* order, int64_t* breakdown) {
  if (*W.err) return;
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(D.task_off, D.n, t, T.n);
  if (d < 0) return;
  const int64_t base = D.task_off[d];
  const int64_t g = base + order[t];
  UnitAcc a;
  acc_init(a);
  const uint32_t bp = any_complex ? W.best_pair[g] : kInactive;
  if (bp == kInactive) {
    acc_add(a, now, T.priority[g], T.expected[g], T.qbasis[g], T.numdep[g], T.gid[g], T.flags[g]);
  } else if (W.route[d]) {  // on-chip planners leave member lists (breakdown mode only)
    for (uint32_t q = W.head[W.pair_slot[bp]]; q < kEnd; q = W.next[q]) {
      const uint32_t tq = pair_task(T, W, q);
      acc_add(a, now, T.priority[tq], T.expected[tq], T.qbasis[tq], T.numdep[tq], T.gid[tq], T.flags[tq]);
    }
  } else {  // general path: the unit table (k_gbest stored the chosen unit's id)
    const GUnit u = unit_load(units + bp);
    const uint32_t* run = run_all + u.start;
    for (uint32_t i = 0; i < u.n; i++) rec_acc(a, now, rec_load(pay + (run[i] & kRunEntry)));
  }
  int64_t bd[EVG_BD_N];
  unit_value(a, D.cfg[d], bd);
  for (int k = 0; k < EVG_BD_N; k++) breakdown[t * EVG_BD_N + k] = bd[k];
}

// scheduler.go:144-158: scalars of DistroQueueInfo / TaskGroupInfo that are not sums.
__global__ void k_finalize_info(DDistros D, DWork W, int32_t d_begin, int32_t d_end, int64_t g_begin, int64_t g_end) {
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t di = d_begin + i;
  if (di < d_end && !W.route[di]) {  // on-chip planners write their rows whole (and may be doing so right now on another stream)
    evg_queue_info* q = W.qinfo + di;
    q->length = D.task_off[di + 1] - D.task_off[di];
    q->max_duration_threshold = D.cfg[di].target_time_ns;
    q->secondary_queue = q->secondary_queue != 0;
    q->has_ungrouped = q->has_ungrouped != 0;
  }
  // group rows between the first and the last general-path distro; an on-chip distro in between stores the same value
  if (g_begin + i < g_end) W.ginfo[g_begin + i].max_hosts = D.gmax[g_begin + i];
}

// UtilizationBasedHostAllocator (utilization_based_host_allocator.go:26-130 and
// the helpers it calls).  FP64 sums run in host-index order (the canonical
// order; the reference's channel order is nondeterministic, allocator.go:381-391).
struct GroupScratch {
  int32_t n_hosts;
  int32_t n_free;
  double soon;
};

__device__ int eval_group(const evg_alloc_cfg& c, const evg_group_info& info, int64_t threshold, int64_t max_hosts,
                          int64_t n_hosts, int64_t n_free, double soon, int64_t* out_new, int64_t* out_free) {
  // evalHostUtilization allocator.go:135-220
  *out_new = 0;
  *out_free = 0;
  if (c.provider == EVG_PROVIDER_STATIC) return EVG_ALLOC_OK;
  if (c.has_pool) {
    if (!c.parent_found) return EVG_ALLOC_ERR_PARENT_MISSING;
    max_hosts = int64_t(c.parent_maximum_hosts) * int64_t(c.pool_max_containers);
  }
  // allocator.go:302-304 rejects a fraction above 1; a NaN or negative one is rejected too, so that every soon-to-be-free
  // term lies in [0, 1] or is NaN (threshold 0, whose floor is 0 by DESIGN.md §3 (iv)) and free_hosts fits its int32
  // field (evg_sched.h)
  if (!(c.future_host_fraction >= 0.0 && c.future_host_fraction <= 1.0)) return EVG_ALLOC_ERR_FUTURE_FRACTION;
  const int64_t exp_free = n_free + d2i_floor(soon);  // allocator.go:317
  const int64_t overdue = c.waits_over_thresh_feedback ? info.count_wait_over_threshold : 0;
  const int64_t short_ns = wsub(info.expected_duration, info.duration_over_threshold);
  int64_t n = calc_new_hosts_needed(short_ns, threshold, exp_free, info.count_duration_over_threshold, overdue,
                                    info.count_dep_filled_merge_queue_tasks, !c.round_up);
  if (n > info.count) n = info.count;
  if (is_max_hosts_capacity(max_hosts, c.has_pool != 0, c.pool_max_containers, n, n_hosts)) n = max_hosts - n_hosts;
  if (n < 0) n = 0;
  if (max_hosts < 1) return EVG_ALLOC_ERR_POOL_SIZE;
  *out_new = n;
  *out_free = exp_free;
  return EVG_ALLOC_OK;
}

// TPD threads per distro: a warp (four distros per block) when task groups are few, the whole 128-thread block
// when some distro has thousands of them (a distro of a million tasks has tens of thousands).  The first warp
// of the team walks the hosts in index order; the lane that owns a bucket (lane 0 for "", lane g%32 for group
// g) does that bucket's updates, so every bucket's FP64 sum is accumulated in host order while buckets proceed
// in parallel.  The team then evaluates the task groups; per-group results are integers, so the reduction is exact.
template <int TPD>
__global__ void __launch_bounds__(128, TPD == 32 ? 6 : 4) k_alloc(DHosts H, int32_t d_begin, int32_t n_distros, const int64_t* group_off,
                                               const evg_queue_info* qinfo, evg_group_info* ginfo, GroupScratch* gs,
                                               int64_t now, evg_alloc_result* result, int32_t* status, int skip_groupless,
                                               const int32_t* list, int32_t n_list) {
  constexpr int TEAMS = 128 / TPD, TW = TPD / 32;  // teams per block, warps per team
  const int team = threadIdx.x / TPD, tt = threadIdx.x % TPD;
  const int ti = int(blockIdx.x) * TEAMS + team;
  if (list && ti >= n_list) return;  // team-uniform; a team never shares a barrier with another
  const int d = list ? list[ti] : d_begin + ti;  // `list`: the distros k_alloc_groupless does not take (built at upload)
  const int lane = threadIdx.x & 31, warp = tt >> 5;
  const unsigned full = 0xffffffffu;
  if (d >= n_distros) return;  // team-uniform (n_distros = end of the range)
  auto team_sync = [&]() { if (TPD == 128) __syncthreads(); else __syncwarp(); };
  __shared__ long long sh_nfree[TEAMS], sh_uhosts[TEAMS], sh_ufree[TEAMS], sh_req[TEAMS][TW], sh_fre[TEAMS][TW];
  __shared__ double sh_usoon[TEAMS];
  __shared__ int sh_st[TEAMS][TW];
  long long& s_nfree = sh_nfree[team]; long long& s_uhosts = sh_uhosts[team]; long long& s_ufree = sh_ufree[team];
  double& s_usoon = sh_usoon[team];
  long long* s_req = sh_req[team]; long long* s_fre = sh_fre[team];
  int* s_st = sh_st[team];
  const int64_t g0 = group_off[d], g1 = group_off[d + 1];
  const int64_t h0 = H.host_off[d], h1 = H.host_off[d + 1];
  if (skip_groupless && g1 == g0 && h1 - h0 <= kGrouplessHosts) return;  // team-uniform: k_alloc_groupless plans it, one thread instead of a warp
  const evg_alloc_cfg c = H.cfg[d];
  const evg_queue_info qi = qinfo[d];
  const int64_t threshold = qi.max_duration_threshold;
  const int64_t n_existing = h1 - h0;
  // IsFree count (allocator.go:33-37), bucket sizes (groupByTaskGroup :223-260), soon-to-be-free sums (:324-394).
  // The buckets of kCache task groups at a time live in SHARED memory while the hosts are walked (a distro with more
  // groups walks its hosts once per stretch of kCache): a bucket update used to be a load-add-store on global scratch,
  // an L2 round trip per host in a serial loop.
  constexpr int kCache = TPD == 32 ? 128 : 512;
  __shared__ GroupScratch sh_gs[TEAMS][kCache];
  GroupScratch* sg = sh_gs[team];
  if (warp == 0) {
    int64_t n_free_all = 0, u_hosts = 0, u_free = 0;
    double u_soon = 0.0;
    const int64_t ng = g1 - g0;
    for (int64_t gb = 0; gb == 0 || gb < ng; gb += kCache) {
      const bool first = gb == 0;  // the "" bucket and the free count are taken on the first walk only
      const int64_t ge = ng - gb < kCache ? ng - gb : kCache;  // groups of this stretch: [gb, gb + ge)
      for (int64_t i = lane; i < ge; i += 32) { sg[i].n_hosts = 0; sg[i].n_free = 0; sg[i].soon = 0.0; }
      __syncwarp();
      // 32 hosts per trip: lane L loads host hc + L (coalesced) and evaluates ITS host's soon-to-be-free term
      // (allocator.go:357-378: an FP64 division and a dozen overflow-checked integer steps, independent of the bucket).
      // Everything that is a COUNT is order-free and taken in parallel (lane-local counters, shared-memory atomics on the
      // bucket); only the FP64 sums need host order, so only the RUNNING hosts of this stretch are replayed in index
      // order through shuffles, the bucket's owner lane adding the term.
      for (int64_t hc = h0; hc < h1; hc += 32) {
        const int64_t hm = hc + lane;
        const bool in = hm < h1;
        const uint32_t my_f = in ? H.flags[hm] : 0u;
        const int32_t my_g = in ? H.gid[hm] : -2;
        const bool my_free = in && !(my_f & EVG_HF_RUNNING) && !(my_f & EVG_HF_TEARDOWN);
        const bool my_run = in && (my_f & EVG_HF_RUNNING) && (my_f & EVG_HF_RT_FOUND);
        const bool my_none = in && my_g == EVG_HG_NONE;
        const bool my_here = in && my_g >= gb && my_g < gb + ge;  // a bucket of this stretch
        const double my_term = my_run ? soon_free_term(now, H.expected[hm], H.stddev[hm], H.start[hm], threshold, c.future_host_fraction) : 0.0;
        if (first) {
          n_free_all += my_free;
          u_hosts += my_none;
          u_free += my_none && my_free;
        }
        if (my_here) {
          atomicAdd(&sg[my_g - gb].n_hosts, 1);
          if (my_free) atomicAdd(&sg[my_g - gb].n_free, 1);
        }
        unsigned todo = __ballot_sync(full, my_run && (my_here || (first && my_none)));
        while (todo) {  // warp-uniform
          const int j = __ffs(todo) - 1;
          todo &= todo - 1u;
          const int32_t g = __shfl_sync(full, my_g, j);
          const double term = __shfl_sync(full, my_term, j);
          if (g == EVG_HG_NONE) { if (lane == 0) u_soon = fadd64(u_soon, term); }
          else if (((g - int32_t(gb)) & 31) == lane) sg[g - gb].soon = fadd64(sg[g - gb].soon, term);
        }
      }
      __syncwarp();
      for (int64_t i = lane; i < ge; i += 32) gs[g0 + gb + i] = sg[i];
    }
    n_free_all = warp_sum64(n_free_all); u_hosts = warp_sum64(u_hosts); u_free = warp_sum64(u_free);  // lane-local counts
    if (lane == 0) { s_nfree = n_free_all; s_uhosts = u_hosts; s_ufree = u_free; s_usoon = u_soon; }
  }
  team_sync();
  const int64_t n_free_all = s_nfree;
  int32_t st = EVG_ALLOC_OK;
  int64_t n_new = 0, n_free_out = n_free_all;
  if (c.provider != EVG_PROVIDER_DOCKER && n_existing >= c.maximum_hosts) {
    n_new = 0;  // allocator.go:39-48
  } else if (c.disabled) {
    n_new = int64_t(c.minimum_hosts) - n_existing;  // allocator.go:51-66
    if (n_new < 0) n_new = 0;
  } else {  // team-uniform branch: c and the host count are per distro
    int64_t required = 0, free_approx = 0;
    // "" bucket exists when standalone tasks are queued or hosts are bucketed under ""
    if (tt == 0 && (qi.has_ungrouped || s_uhosts > 0)) {
      int64_t n, f;
      st = eval_group(c, qi.ungrouped, threshold, c.maximum_hosts, s_uhosts, s_ufree, s_usoon, &n, &f);
      required += n;
      free_approx += f;
    }
    for (int64_t g = g0 + tt; g < g1; g += TPD) {
      evg_group_info* gi = ginfo + g;
      if (gi->count == 0) continue;  // allocator.go:84-86
      int64_t n, f;
      const int e = eval_group(c, *gi, threshold, gi->max_hosts, gs[g].n_hosts, gs[g].n_free, gs[g].soon, &n, &f);
      if (e != EVG_ALLOC_OK) { st = max(st, e); continue; }
      required += n;
      free_approx += f;
      gi->count_free = f;  // allocator.go:107-110
      gi->count_required = n;
    }
    // a data error is distro-wide (fraction, parent) or the pool-size check of some group: any thread's error wins
    st = __reduce_max_sync(full, st);
    required = warp_sum64(required);
    free_approx = warp_sum64(free_approx);
    if (TW > 1) {
      if (lane == 0) { s_st[warp] = st; s_req[warp] = required; s_fre[warp] = free_approx; }
      team_sync();
      st = s_st[0]; required = s_req[0]; free_approx = s_fre[0];
#pragma unroll
      for (int w = 1; w < TW; w++) { st = max(st, s_st[w]); required += s_req[w]; free_approx += s_fre[w]; }
    }
    if (st == EVG_ALLOC_OK) {
      if (required + n_free_all > qi.length_with_dependencies_met) required = qi.length_with_dependencies_met - n_free_all;
      if (required < 0) required = 0;
      int64_t topup = 0;
      if (n_existing + required < c.minimum_hosts) topup = c.minimum_hosts - (n_existing + required);
      n_new = required + topup;
      n_free_out = free_approx;
    } else {
      n_new = 0;  // (0, len(freeHosts), err) allocator.go:99-101
      n_free_out = n_free_all;
      // the reference stops at the first failing group of a randomised map walk: which groups it had written is not
      // defined, so an error leaves every group of the distro at 0 (evg_sched.h)
      for (int64_t g = g0 + tt; g < g1; g += TPD) { ginfo[g].count_free = 0; ginfo[g].count_required = 0; }
    }
  }
  if (tt == 0) {
    int64_t deficit = wsub(qi.expected_duration, wmul(n_free_out, threshold));
    if (deficit < 0) deficit = 0;
    result[d].new_hosts = int32_t(n_new);
    result[d].free_hosts = int32_t(n_free_out);
    result[d].deficit_ns = deficit;
    status[d] = st;
  }
}

// Distros without task groups -- nearly all of a tick with 10^5 small queues -- have one bucket (""): the whole
// decision is a scalar chain over a handful of hosts, so ONE THREAD plans a distro (k_alloc<32> spent a warp, and its
// latency chain, on each).  Same arithmetic in the same order as k_alloc: hosts in index order, FP64 sum of the
// soon-to-be-free terms, eval_group on the "" bucket, the same tail.
__global__ void __launch_bounds__(128) k_alloc_groupless(DHosts H, int32_t d_begin, int32_t n_distros, const int64_t* group_off,
                                                         const evg_queue_info* qinfo, int64_t now, evg_alloc_result* result, int32_t* status) {
  const int d = d_begin + int(blockIdx.x * blockDim.x + threadIdx.x);
  if (d >= n_distros) return;
  const int64_t h0 = H.host_off[d], h1 = H.host_off[d + 1];
  if (group_off[d + 1] != group_off[d] || h1 - h0 > kGrouplessHosts) return;  // k_alloc's
  const evg_alloc_cfg c = H.cfg[d];
  const evg_queue_info qi = qinfo[d];
  const int64_t threshold = qi.max_duration_threshold;
  const int64_t n_existing = h1 - h0;
  int64_t n_free_all = 0, u_hosts = 0, u_free = 0;
  double u_soon = 0.0;
  for (int64_t h = h0; h < h1; h++) {
    const uint32_t f = H.flags[h];
    const bool is_free = !(f & EVG_HF_RUNNING) && !(f & EVG_HF_TEARDOWN);
    n_free_all += is_free;
    if (H.gid[h] == EVG_HG_NONE) {  // a host bucketed under a group name the queue does not have joins no bucket (allocator.go:223-260)
      const bool running = (f & EVG_HF_RUNNING) && (f & EVG_HF_RT_FOUND);
      u_hosts++;
      u_free += is_free;
      if (running) u_soon = fadd64(u_soon, soon_free_term(now, H.expected[h], H.stddev[h], H.start[h], threshold, c.future_host_fraction));
    }
  }
  int32_t st = EVG_ALLOC_OK;
  int64_t n_new = 0, n_free_out = n_free_all;
  if (c.provider != EVG_PROVIDER_DOCKER && n_existing >= c.maximum_hosts) {
    n_new = 0;  // allocator.go:39-48
  } else if (c.disabled) {
    n_new = int64_t(c.minimum_hosts) - n_existing;  // allocator.go:51-66
    if (n_new < 0) n_new = 0;
  } else {
    int64_t required = 0, free_approx = 0;
    if (qi.has_ungrouped || u_hosts > 0) {
      int64_t n, f;
      st = eval_group(c, qi.ungrouped, threshold, c.maximum_hosts, u_hosts, u_free, u_soon, &n, &f);
      required += n;
      free_approx += f;
    }
    if (st == EVG_ALLOC_OK) {
      if (required + n_free_all > qi.length_with_dependencies_met) required = qi.length_with_dependencies_met - n_free_all;
      if (required < 0) required = 0;
      int64_t topup = 0;
      if (n_existing + required < c.minimum_hosts) topup = c.minimum_hosts - (n_existing + required);
      n_new = required + topup;
      n_free_out = free_approx;
    } else {
      n_new = 0;  // (0, len(freeHosts), err) allocator.go:99-101
      n_free_out = n_free_all;
    }
  }
  int64_t deficit = wsub(qi.expected_duration, wmul(n_free_out, threshold));
  if (deficit < 0) deficit = 0;
  result[d].new_hosts = int32_t(n_new);
  result[d].free_hosts = int32_t(n_free_out);
  result[d].deficit_ns = deficit;
  status[d] = st;
}

// --------------------------------------------------------------------------
// context
// --------------------------------------------------------------------------
// The nine planner columns of a task table.  each() is the one list of them: every check, copy and view of the columns
// goes through it, so a column is added or changed there alone.
struct TaskCols {
  DevBuf prio, nd, tgo, gid, vid, flags, exp, qb, wb;

  // f(buffer, evg_task_soa field, field name) -> int for every column, the 8-byte ones first (evg_update_tasks packs
  // them in this order); stops at the first f that does not return EVG_OK and returns its code.
  template <class F>
  static int each(F&& f) {
    int rc = EVG_OK;
    auto col = [&](DevBuf TaskCols::*b, auto field, const char* name) { if (rc == EVG_OK) rc = f(b, field, name); };
    col(&TaskCols::exp, &evg_task_soa::expected_ns, "expected_ns");
    col(&TaskCols::qb, &evg_task_soa::queue_basis_ns, "queue_basis_ns");
    col(&TaskCols::wb, &evg_task_soa::wait_basis_ns, "wait_basis_ns");
    col(&TaskCols::prio, &evg_task_soa::priority, "priority");
    col(&TaskCols::nd, &evg_task_soa::num_dependents, "num_dependents");
    col(&TaskCols::tgo, &evg_task_soa::task_group_order, "task_group_order");
    col(&TaskCols::gid, &evg_task_soa::group_id, "group_id");
    col(&TaskCols::vid, &evg_task_soa::version_id, "version_id");
    col(&TaskCols::flags, &evg_task_soa::flags, "flags");
    return rc;
  }
  template <class T>
  static constexpr size_t elem(const T* evg_task_soa::*) { return sizeof(T); }
  template <class T>
  static void point(const T*& field, const void* p) { field = static_cast<const T*>(p); }
  static bool is_id(DevBuf TaskCols::*b) { return b == &TaskCols::gid || b == &TaskCols::vid; }

  // Some column of t is null; without `ids`, group_id and version_id are not looked at.
  static bool missing(const evg_task_soa* t, bool ids = true) {
    return each([&](auto b, auto f, const char*) { return t->*f || (!ids && is_id(b)) ? EVG_OK : EVG_ERR_INVALID; }) != EVG_OK;
  }
  // Every column grown to n rows and kColPad rows of padding; with `zero_pad`, the padding zeroed on s as an upload
  // leaves it.
  int size(int64_t n, cudaStream_t s = nullptr, bool zero_pad = false) {
    return each([&](auto b, auto f, const char*) -> int {
      CK((this->*b).ensure(elem(f) * size_t(n + kColPad)));
      if (zero_pad) CK(cudaMemsetAsync(static_cast<char*>((this->*b).p) + elem(f) * n, 0, elem(f) * kColPad, s));
      return EVG_OK;
    });
  }
  // Rows [t0, t0 + n) of t's columns from host memory into the same rows here, on s.
  int copy_rows(const evg_task_soa* t, int64_t t0, int64_t n, cudaStream_t s) {
    return each([&](auto b, auto f, const char*) -> int {
      if (n > 0) CK(cudaMemcpyAsync(static_cast<char*>((this->*b).p) + elem(f) * t0, t->*f + t0, elem(f) * n, cudaMemcpyHostToDevice, s));
      return EVG_OK;
    });
  }
  // The first n rows of t's columns, each grown to at least one row.
  int stage(const evg_task_soa* t, int64_t n, cudaStream_t s) {
    const int rc = each([&](auto b, auto f, const char*) -> int {
      CK((this->*b).ensure(elem(f) * size_t(n > 0 ? n : 1)));
      return EVG_OK;
    });
    return rc != EVG_OK ? rc : copy_rows(t, 0, n, s);
  }
  // t's columns are caller-owned device memory, borrowed as they are (evg_upload_device).
  int adopt(const evg_task_soa* t) {
    return each([&](auto b, auto f, const char* name) -> int {
      if ((reinterpret_cast<uintptr_t>(t->*f) & 15u) != 0) return fail(EVG_ERR_INVALID, "device column t->%s is not 16-byte aligned", name);
      (this->*b).adopt(const_cast<void*>(static_cast<const void*>(t->*f)));
      return EVG_OK;
    });
  }
  // The columns as an evg_task_soa of n rows without edges.
  evg_task_soa soa(int64_t n) const {
    evg_task_soa s;
    memset(&s, 0, sizeof(s));
    s.n_tasks = n;
    each([&](auto b, auto f, const char*) -> int { point(s.*f, (this->*b).p); return EVG_OK; });
    return s;
  }
  // The device views: DTasks of n rows without edges, and the EdDst a composed table is written to.
  template <class V>
  V fill(V v) const {
    v.priority = prio.as<int32_t>(); v.expected = exp.as<int64_t>(); v.qbasis = qb.as<int64_t>(); v.wbasis = wb.as<int64_t>();
    v.numdep = nd.as<int32_t>(); v.tgo = tgo.as<int32_t>(); v.gid = gid.as<int32_t>(); v.vid = vid.as<int32_t>();
    v.flags = flags.as<uint32_t>();
    return v;
  }
  DTasks view(int64_t n) const {
    DTasks v;
    memset(&v, 0, sizeof(v));
    v.n = n;
    return fill(v);
  }
  EdDst dst() const { return fill(EdDst{}); }
  void swap(TaskCols& o) {
    each([&](auto b, auto, const char*) -> int { (this->*b).swap(o.*b); return EVG_OK; });
  }
};

// Whose columns the resident tick is: none; the context's own but no base for edits (what a one-shot call leaves, or a
// call that failed after upload_tasks); caller-owned device memory (evg_upload_device); the context's own, editable.
enum class Tick : uint8_t { kNone, kFixed, kBorrowed, kOwn };

struct evg_ctx {
  int device = 0;
  int num_sms = 0;  // the device's multiprocessor count: grid cap of the grid-stride work-list kernels
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // Entry points may be called from any OS thread (cgo runs a call on whatever M the goroutine sits on): every
  // extern "C" function that takes a context holds this lock for its duration, so one context serialises its
  // callers and several contexts (one per worker) run side by side on their own streams.
  std::recursive_mutex mu;
  cudaEvent_t ev_begin = nullptr, ev_sort0 = nullptr, ev_sort1 = nullptr, ev_end = nullptr, ev_gt0 = nullptr, ev_gt1 = nullptr;
  bool general_timed = false;
  // ring of event pairs around the dominant kernel of a tick: per-run kernel time without syncing inside a timed loop
  static constexpr int kRing = 128;
  cudaEvent_t ring0[kRing] = {}, ring1[kRing] = {};
  int64_t runs = 0;
  int64_t max_groups = 0;  // most task groups in any distro: picks the allocator's team width
  int sort_slot = -1;      // ring slot of the last run's dominant-kernel pair
  // route streams: the size classes of one tick are independent until the allocator, so they run side by side
  static constexpr int kAux = 6;
  cudaStream_t s_aux[kAux] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[kAux] = {};
  // The resident tick (need_tick checks it; upload_tasks and drop_tick replace it), and whether the allocator's tables,
  // evg_upload_with_deps' verdicts (`deps`), evg_plan_aliases' map (`al`) and evg_resolve_durations' results (`dur`)
  // belong to it.  `allocated`: run state -- the allocator's results (queue and group infos, result rows, status) are
  // from a run on this tick, into the result buffer bound now; evg_host_job reads them.  `host_job`: run state --
  // evg_host_job's reports in hj.out are from the current run; a chained evg_host_drawdown reads them.  `dispatchers`:
  // run state -- evg_rebuild_dispatchers built dp and nx from the current run; evg_find_next_tasks serves from them.
  struct {
    Tick kind = Tick::kNone;
    bool hosts = false, deps = false, aliases = false, durations = false, allocated = false, host_job = false, dispatchers = false;
  } tick;
  int64_t T = 0, E = 0, G = 0, H = 0, U = 0, NT = 0, t_pad = 0;
  int32_t Dn = 0;
  int any_complex = 0;
  int64_t launches = 0;
  bool timed = false;
  TaskCols tasks;  // the resident planner columns
  DevBuf b_depoff, b_depidx;
  DevBuf b_taskoff, b_groupoff, b_cfg, b_gmax, b_unitbase;
  DevBuf b_hasdep, b_head, b_next, b_pslot, b_etask, b_elive, b_bestpair;
  DevBuf b_rn0, b_rn1, b_rn2, b_rn3, b_rn4, b_rn5, b_rn6, b_rn7;
  struct {
    DevBuf off, kind, ref, want, state, pre, ext;  // an evg_deps_in table, staged
    DevBuf met, fin, stamp;                        // k_deps_met's verdicts, its dep_finished_ns input, its stamps
  } deps;
  struct {
    DevBuf task_off, sched, project, project_flags, valid_off, valid_idx, finder;  // the finder tables
    DevBuf kept, count;  // k_runnable's kept lists and per-distro counts
    TaskCols cand;       // evg_plan_from_finder: the candidates' columns
    DevBuf dep_off, dep_idx;  // and their edges
  } pf;
  struct {  // the pipeline finder's tables (the first evg_find_runnable_ex / evg_plan_from_finder_ex with a pipeline allocates them)
    DevBuf dep_status, task_status, ext_status, task_unatt, ext_unatt, project_raw;  // an evg_pipeline_in, staged
    DevBuf edge_cnt, dep_off, dep_idx;  // the candidates' edges without those of EVG_FINDER_PIPELINE rows
  } pl;
  struct {  // compose_tick's buffers (the first evg_edit_tasks or evg_plan_from_finder allocates them) and the staged edit
    TaskCols out;            // the shadow set: the composed table is written here, then swapped with the resident columns
    DevBuf dep_off, dep_idx; // the composed edges (swapped too)
    TaskCols ins;            // the inserted rows, staged
    DevBuf ins_dep_off, ins_dep_idx, rm, add_task, add_dep, gremap, vremap;
    DevBuf new_off, old_off, old_goff, ins_off, old_vbase, edge_at;  // D+1 tables
    DevBuf keep, pos, src, edge_cnt, err;
  } ed;
  // evg_plan_aliases (the first call allocates these): the staged source table, the (queue, task) pairs and the alias
  // map evg_download_alias_map returns while tick.aliases holds
  struct {
    TaskCols src;
    DevBuf dep_off, dep_idx, gmax, sched, tgmax, primary, soff, sidx, doff, didx;  // the source table
    DevBuf cnt, poff, keys[2], hist, hoff;     // pairs per row, their offsets, the pair keys, the radix pass counters
    DevBuf hk, hv, gslot, vslot, fg, fv, pg, pv;  // first-appearance ids of groups and versions per queue
    DevBuf qoff, samp, gout, srow, gsrc, err;  // queue offsets, per-distro samples, group slots, the alias map
  } al;
  // evg_resolve_durations (the first call allocates these): the staged history, the per-key accumulators and statistics,
  // the pairs' single keys, the listed rows (tasks, then hosts) and their results, which evg_download_durations returns
  // while tick.durations holds
  struct {
    DevBuf key, taken, start, finish, flags, acc, stat, pair_off, single;
    DevBuf rows, in, out, src, err;
    int64_t n_t = 0, n_h = 0;
  } dur;
  // evg_rebuild_dispatchers (the first call allocates these): the persisted queues' DAG input gathered from the tick,
  // and the scratch and results of the k_dag_* kernels, so that the resident tick is only read
  struct {
    DevBuf item_off, rank_of, row, first, gslot_of, gindex, cnt, dep_off, dep_item, pos, group_off, group_slot, group_id;
    DevBuf succ_off, succ, index, low, stack, cs_node, cs_pos, emit, on_stack, sorted, stats, buf[2], unit_off;
  } dp;
  // evg_host_job (the first call allocates these): the staged job settings and spawned counts, and the outputs
  struct { DevBuf cfg, spawned, out; } hj;
  // FindNextTask: the per-item fields and per-group tables of the dispatchers being served (evg_rebuild_dispatchers
  // gathers them, evg_find_next_batch stages them with the dispatchers themselves), their state, the staged snapshot
  // and requests of a call, and the host copies of the offsets the requests are checked against
  struct {
    DevBuf gmh, deps_met, gfirst, unit_max, verdict, bits, deleted, running, inert;
    DevBuf flags, est, ingest, running_db, req_off, req_group, req_ami, list, out_item, out_outcome;
    DevBuf item_off, group_off, sorted, n_sorted, unit_items, unit_off, group_id;  // evg_find_next_batch's dispatchers
    DNext x{};  // the chained dispatchers
    std::vector<int64_t> h_item_off, h_group_off;
  } nx;
  // evg_host_drawdown / evg_idle_hosts (the first call allocates these): the staged idle-host table, its offsets and the
  // per-distro inputs, the verdicts, the decided flags and their scan, and the per-distro outputs
  struct { DevBuf cols, off, din, verdict, flag, pos, dout; } ih;
  // evg_estimate_start_times / evg_estimate_start_batch (the first call allocates these): the staged host table, each
  // row's timeToCompletion and whether it counts, their scan, the packed pools (two copies: the merge sort's), the
  // queues' offsets and durations, the launch list and the outputs
  struct { DevBuf kind, expected, dispatch, host_off, ttc, used, pos, pool[2], pool_off, item_off, dur, list, start, hosts_used; } es;
  DevBuf b_err;
  DevBuf b_scansum;  // scan_counts' per-block sums
  DevBuf b_route, b_unitv, b_unita, b_unitn, b_unitmask;
  DevBuf b_punt, b_puntcnt;
  // The distros of each size class: ascending ids on the host and the device (the pipelined call cuts them by distro
  // range), and for the on-chip classes the same list largest distro first (the resident tick's launch order).
  struct RouteList {
    std::vector<int32_t> h;
    DevBuf b, lpt;
    int32_t n() const { return int32_t(h.size()); }
  };
  RouteList routes[kRoutes];
  int64_t max_cta_tasks = 0;  // largest distro routed to k_plan_cta: picks the fallback instance for what it hands back
  int32_t nNA_big = 0;  // leading entries of the largest-first kCtaA list that need the 128-thread instance
  DevBuf b_alist;            // distros k_alloc plans itself (task groups, or more than kGrouplessHosts hosts), listed by upload_hosts
  int64_t n_alist = 0;
  bool alist_valid = false;
  std::vector<int64_t> h_taskoff, h_groupoff, h_unitbase, h_edgeoff, h_dtileoff;
  std::vector<int32_t> h_nver;  // n_versions of each distro (evg_edit_tasks sizes version_remap by it)
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  static constexpr int kMaxChunks = 16;
  cudaEvent_t ev_h[kMaxChunks] = {}, ev_c[kMaxChunks] = {};
  int general_complex = 0;
  int64_t Tgc = 0;  // tasks in general-path distros that can hold multi-member units (work-list capacity)
  DevBuf b_kv, b_vmm, b_klo[2], b_khi[2], b_ix[2], b_e, b_tilesum, b_gmisc;
  DevBuf b_tiledistro, b_tilestart, b_dtileoff, b_tilehist, b_wl, b_pay, b_place, b_eplace, b_run, b_rank, b_emit, b_blist, b_unit, b_upd;
  DevBuf b_qinfo, b_ginfo, b_order, b_tv, b_bd;
  DevBuf b_hflags, b_hgid, b_hexp, b_hstd, b_hstart, b_hostoff, b_acfg, b_gs, b_result, b_status;
  bool bd_valid = false;
  evg_alloc_result* ext_result = nullptr;  // caller-owned send buffer (evg_bind_result_buffer)
  int64_t ext_capacity = 0;
  evg_alloc_result* result_ptr() const { return ext_result ? ext_result : b_result.as<evg_alloc_result>(); }
};

namespace {

DTasks dtasks(const evg_ctx* c);
DDistros ddistros(const evg_ctx* c);
DWork dwork(const evg_ctx* c);
DGen dgen(const evg_ctx* c);
inline unsigned grid_for(int64_t n, int block) { return unsigned((n + block - 1) / block); }

// Every kernel of this file is launched here: an empty grid launches nothing, any other launch adds one to the count
// evg_last_launch_count reports.  Launch errors are left to the caller's CK(cudaGetLastError()).
template <class... P, class... A>
void launch(evg_ctx* c, cudaStream_t st, void (*kernel)(P...), unsigned grid, unsigned block, size_t smem, A&&... args) {
  if (grid == 0) return;
  kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
  c->launches++;
}

// Sorts every segment of buf[0] that off (on the device, n_segs + 1 entries) delimits: ceil(log2 max_len) passes of
// k_seg_merge_pass over n_threads threads, max_len and n_threads bounding the longest segment and the element total.
// Returns the buffer that holds the result: buf[0] when max_len <= 1 and no pass runs.
template <class Order>
typename Order::Elem* seg_merge_sort(evg_ctx* c, cudaStream_t s, const Order& order, const int64_t* off, int32_t n_segs,
                                     int64_t n_threads, int64_t max_len, typename Order::Elem* const buf[2]) {
  int cur = 0;
  for (int64_t L = 1; L < max_len; L <<= 1, cur ^= 1)
    launch(c, s, k_seg_merge_pass<Order>, grid_for(n_threads, 256), 256, 0, order, off, n_segs, buf[cur], buf[cur ^ 1], L);
  return buf[cur];
}

// The start of every entry point that takes a context: it names the call once (`who`, for its later messages too), fails
// a null context with that name, holds the context's lock for the rest of the call and selects the context's device.
#define ENTER(c, name)                                                    \
  const char* const who = (name);                                         \
  if (!(c)) return fail(EVG_ERR_INVALID, "%s: null context", who);       \
  std::lock_guard<std::recursive_mutex> lock_((c)->mu);                   \
  CK(cudaSetDevice((c)->device))

// A call that writes the resident columns or the tables beside them (a new table, or scratch it shares with the
// planner's inputs) drops the tick before its first such write: a call that fails partway must not leave the next
// evg_run_resident a tick whose buffers it has half replaced.
void drop_tick(evg_ctx* c) { c->tick = {}; }

// What a call needs of the resident tick.  EVG_ERR_STATE names the call and the first unmet condition: a tick, then
// its kind, then the state the call reads.
enum class Need { kTick, kOwnColumns, kEditable, kHosts, kVerdicts, kAliasMap, kDurations, kAllocated, kHostJob, kDispatchers };
int need_tick(const evg_ctx* c, const char* who, Need what) {
  const auto& t = c->tick;
  const bool own = what == Need::kOwnColumns || what == Need::kEditable;
  const char* unmet = t.kind == Tick::kNone                               ? "no resident tick"
                      : own && t.kind == Tick::kBorrowed                  ? "the resident columns are borrowed (evg_upload_device)"
                      : what == Need::kEditable && t.kind == Tick::kFixed ? "the resident tick is what a one-shot call left"
                      : (what == Need::kHosts || what == Need::kAllocated) && !t.hosts ? "the resident tick has no hosts"
                      : what == Need::kAllocated && !t.allocated          ? "no allocator run on the resident tick since it was set or a result buffer was bound"
                      : what == Need::kVerdicts && !t.deps                ? "the resident tick was not uploaded with evg_upload_with_deps"
                      : what == Need::kAliasMap && !t.aliases             ? "the resident tick was not built by evg_plan_aliases"
                      : what == Need::kDurations && !t.durations          ? "no evg_resolve_durations on the resident tick's rows"
                      : what == Need::kHostJob && !t.host_job             ? "no evg_host_job on the resident tick's current run"
                      : what == Need::kDispatchers && !t.dispatchers      ? "no evg_rebuild_dispatchers on the resident tick's current run" : nullptr;
  return unmet ? fail(EVG_ERR_STATE, "%s: %s", who, unmet) : EVG_OK;
}

// Where upload_tasks finds the task columns.
enum class Cols {
  kCopy,      // host memory: copied into the context's buffers
  kChunked,   // host memory: the pipelined call copies them chunk by chunk
  kAdopt,     // device memory the context borrows (evg_upload_device)
  kResident,  // already in the context's own buffers (compose_tick swapped them in): `t` points at them
};

// Route every distro of the tick, stage the small tables, size the work buffers.  Every mode but kChunked range-checks
// the ids here (the pipelined call checks chunk by chunk).
// `edge_off` (D+1, host) is dep_off sampled at the distro boundaries; NULL when the host can read t->dep_off itself.
int upload_tasks(evg_ctx* c, const char* who, const evg_task_soa* t, const evg_distro_table* dt, Cols cols = Cols::kCopy,
                 const int64_t* edge_off = nullptr) {
  const bool copy_columns = cols == Cols::kCopy, adopt = cols == Cols::kAdopt;
  if (!t || !dt) return fail(EVG_ERR_INVALID, "null task table / distro table");
  const int64_t T = t->n_tasks, E = t->n_edges;
  const int32_t D = dt->n_distros;
  if (T < 0 || E < 0 || D < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (T >= (int64_t(1) << 31) - 2) return fail(EVG_ERR_INVALID, "n_tasks %lld exceeds 2^31-2 per call", (long long)T);
  if (2 * T + E >= int64_t(0xFFFFFFF0u)) return fail(EVG_ERR_INVALID, "2*n_tasks+n_edges exceeds the 32-bit pair id space");
  if (D > 0 && (!dt->task_off || !dt->group_off || !dt->cfg)) return fail(EVG_ERR_INVALID, "null distro arrays");
  if (T > 0 && TaskCols::missing(t)) return fail(EVG_ERR_INVALID, "null task column");
  if (E > 0 && (!t->dep_off || !t->dep_idx)) return fail(EVG_ERR_INVALID, "n_edges > 0 but dep_off/dep_idx null");
  if (D == 0 && T != 0) return fail(EVG_ERR_INVALID, "tasks without distros");
  int rc = D > 0 ? check_offsets(dt->task_off, D, T, who, "task_off") : EVG_OK;
  if (rc == EVG_OK && D > 0) rc = check_offsets(dt->group_off, D, -1, who, "group_off");
  if (rc != EVG_OK) return rc;
  std::vector<int64_t> unit_base(size_t(D) + 1, 0), dtile_off(size_t(D) + 1, 0);
  std::vector<int32_t> tile_distro, list[kRoutes];
  std::vector<int64_t> tile_start;
  std::vector<uint8_t> route(size_t(D) + 1, 0);
  int general_complex = 0;
  int any_complex = E > 0 ? 1 : 0;
  int64_t Tgc = 0, Prec = 0, Urec = 0;
  constexpr int kGA = PlanCta<kNT_A, kNCapA>::kGroupCap, kGB = PlanCta<kNT_B, kNCapB>::kGroupCap, kGC = PlanCta<kNT_C, kNCapC>::kGroupCap;
  // Size class of distro d by its own shape (no side effects).  kBigUnits: a GroupVersions distro of k_plan_smem's
  // smallest class above kBigUnitTasks tasks, whose version units of dozens of tasks are walked member by member.
  constexpr int kBigUnits = kRoutes;
  auto size_class = [&](int32_t d) -> int {
    const int64_t a = dt->task_off[d], b = dt->task_off[d + 1];
    const int64_t n = b - a, g = dt->group_off[d + 1] - dt->group_off[d];
    const evg_distro_cfg& cf = dt->cfg[d];
    const int64_t de = (E > 0) ? (edge_off ? edge_off[d + 1] - edge_off[d] : t->dep_off[b] - t->dep_off[a]) : 0;
    const bool narrow = !cf.group_versions && de == 0;  // k_plan_cta: task groups are the only multi-member units it knows
    if (n <= kCapW) return kWarp;
    if (narrow && n <= kNCapA && g <= kGA) return kCtaA;
    if (narrow && n <= kNCapB && g <= kGB) return kCtaB;
    if (narrow && n <= kNCapC && g <= kGC) return kCtaC;
    if (n <= kCapA) return (cf.group_versions && n > kBigUnitTasks) ? kBigUnits : kSmemA;
    if (n <= kCapB) return kSmemB;
    if (n <= kCapC) return kSmemC;
    return kGeneral;
  };
  // k_plan_smem walks the unit lists of GroupVersions / dependency distros with ONE CTA per distro: fine when a class
  // has enough distros to fill the GPU, a millisecond-long tail when it has a handful (configs[4]: ~20 distros of 1-6k
  // tasks held the whole tick, then ~50 GroupVersions distros of 129-1024 tasks whose version units are walked member by
  // member).  The general path spreads every distro over all SMs, so sparse classes go there.
  int64_t n_class[kBigUnits + 1] = {};
  for (int32_t d = 0; d < D; d++) n_class[size_class(d)]++;
  const char* sparse_env = getenv("EVG_SPARSE_CLASS");  // tests set 0 to keep every class on its own kernel
  const int64_t sparse = sparse_env ? atoll(sparse_env) : kSparseClass;
  // The route of distro d: its size class, after the sparse-class rule (needs every class's size: the count above).
  auto route_of = [&](int32_t d) -> int {
    const int k = size_class(d);
    if ((k == kSmemB || k == kSmemC || k == kBigUnits) && n_class[k] < sparse) return kGeneral;
    return k == kBigUnits ? kSmemA : k;
  };
  for (int32_t d = 0; d < D; d++) {
    const int64_t a = dt->task_off[d], b = dt->task_off[d + 1];
    const int64_t ga = dt->group_off[d], gb = dt->group_off[d + 1];
    if (b - a > kMaxTasksPerDistro) return fail(EVG_ERR_INVALID, "distro %d holds %lld tasks (max %lld)", d, (long long)(b - a), (long long)kMaxTasksPerDistro);
    const evg_distro_cfg& cf = dt->cfg[d];
    if (cf.n_versions < 0) return fail(EVG_ERR_INVALID, "distro %d: negative n_versions", d);
    if (gb > ga || cf.group_versions) any_complex = 1;
    unit_base[d + 1] = unit_base[d] + (gb - ga) + (cf.group_versions ? int64_t(cf.n_versions) : (b - a));
    const int64_t n = b - a;
    const int64_t de = (E > 0) ? (edge_off ? edge_off[d + 1] - edge_off[d] : t->dep_off[b] - t->dep_off[a]) : 0;
    const int r = route_of(d);
    list[r].push_back(d);
    route[d] = r != kGeneral;
    if (r == kGeneral) {
      if (gb > ga || cf.group_versions || de > 0) {
        general_complex = 1;
        Tgc += n;
        Prec += n + ((cf.group_versions && gb > ga) ? n : 0) + de;  // own-key, version and dependency memberships at most
        // units: every unit has an own-key member (a dependency joins its target's own-key unit) or is a version unit
        Urec += n + ((cf.group_versions && gb > ga) ? std::min<int64_t>(cf.n_versions, n) : 0);
      }
      const int64_t a0 = a & ~int64_t(3);  // tiles start 16-byte aligned in every column
      for (int64_t s = a0; s < b; s += kGTile) { tile_distro.push_back(d); tile_start.push_back(s); }
    }
    dtile_off[d + 1] = int64_t(tile_distro.size());
  }
  const int64_t G = D > 0 ? dt->group_off[D] : 0;
  if (G > 0 && !dt->group_max_hosts) return fail(EVG_ERR_INVALID, "null group_max_hosts");
  const int64_t U = unit_base[D];
  if (U >= int64_t(0xFFFFFFF0u)) return fail(EVG_ERR_INVALID, "unit slot space exceeds 32 bits");
  if (Prec >= int64_t(0xFFFFFFF0u)) return fail(EVG_ERR_INVALID, "unit table exceeds 32 bits");
  if (Tgc >= int64_t(kRunOwn)) return fail(EVG_ERR_INVALID, "work list exceeds 31 bits (a run position is entry id | own bit)");
  const int64_t NT = int64_t(tile_distro.size());
  const int64_t P = 2 * T + E;
  cudaStream_t s = c->stream;
  drop_tick(c);
  if (adopt) rc = c->tasks.adopt(t);
  else if (cols != Cols::kResident) rc = c->tasks.size(T);
  if (rc == EVG_OK && copy_columns) rc = c->tasks.copy_rows(t, 0, T, s);
  if (rc != EVG_OK) return rc;
#define UPC(buf, ptr, count, type)                                                                    \
  do {                                                                                                \
    if (cols == Cols::kResident) break;                                                               \
    if (adopt) {                                                                                      \
      if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0) return fail(EVG_ERR_INVALID, "device column %s is not 16-byte aligned", #ptr); \
      (buf).adopt(const_cast<void*>(static_cast<const void*>(ptr)));                                  \
    } else {                                                                                          \
      CK((buf).ensure(sizeof(type) * size_t((count) + kColPad)));                                     \
      if (copy_columns && (count) > 0) CK(cudaMemcpyAsync((buf).p, (ptr), sizeof(type) * size_t(count), cudaMemcpyHostToDevice, s)); \
    }                                                                                                 \
  } while (0)
  if (E > 0) {
    UPC(c->b_depoff, t->dep_off, T + 1, int64_t);
    UPC(c->b_depidx, t->dep_idx, E, int32_t);
  }
#undef UPC
  UP(s, c->b_taskoff, dt->task_off, D + 1, int64_t);
  UP(s, c->b_groupoff, dt->group_off, D + 1, int64_t);
  UP(s, c->b_cfg, dt->cfg, D, evg_distro_cfg);
  UP(s, c->b_gmax, dt->group_max_hosts, G, int32_t);
  UP(s, c->b_unitbase, unit_base.data(), D + 1, int64_t);
  UP(s, c->b_tiledistro, tile_distro.data(), NT, int32_t);
  UP(s, c->b_tilestart, tile_start.data(), NT, int64_t);
  UP(s, c->b_dtileoff, dtile_off.data(), D + 1, int64_t);
  UP(s, c->b_route, route.data(), D + 1, uint8_t);
  for (int r = 0; r < kRoutes; r++) UP(s, c->routes[r].b, list[r].data(), int64_t(list[r].size()), int32_t);
  // One CTA per distro: with the largest first, the last (partial) wave of a launch holds the smallest distros and the
  // tail is short (configs[4]: 1371 distros of 33..1024 tasks on 132 x 8 = 1056 CTA slots).  The ascending lists stay: the
  // pipelined one-shot call cuts them by distro range.
  std::vector<int32_t> lpt[kRoutes];
  for (int r = 0; r < kRoutes; r++) {
    if (!largest_first(r)) continue;
    lpt[r] = list[r];
    std::stable_sort(lpt[r].begin(), lpt[r].end(), [&](int32_t x, int32_t y) {
      return dt->task_off[x + 1] - dt->task_off[x] > dt->task_off[y + 1] - dt->task_off[y];
    });
  }
  // the tail of the smallest class that fits the 64-thread instance (size AND task groups) goes last, largest first
  constexpr int kGS = PlanCta<kNT_S, kNCapS>::kGroupCap;
  auto fits_s = [&](int32_t x) { return dt->task_off[x + 1] - dt->task_off[x] <= kNCapS && dt->group_off[x + 1] - dt->group_off[x] <= kGS; };
  std::vector<int32_t>& lpt_a = lpt[kCtaA];
  std::stable_partition(lpt_a.begin(), lpt_a.end(), [&](int32_t x) { return !fits_s(x); });
  c->nNA_big = int32_t(std::count_if(lpt_a.begin(), lpt_a.end(), [&](int32_t x) { return !fits_s(x); }));
  c->max_cta_tasks = 0;
  for (int r = 0; r < kRoutes; r++)
    if (is_cta(r))
      for (int32_t x : list[r]) c->max_cta_tasks = std::max<int64_t>(c->max_cta_tasks, dt->task_off[x + 1] - dt->task_off[x]);
  for (int r = 0; r < kRoutes; r++)
    if (largest_first(r)) UP(s, c->routes[r].lpt, lpt[r].data(), int64_t(lpt[r].size()), int32_t);
  // the staging vectors above must outlive the async copies
  CK(cudaStreamSynchronize(s));
  // work buffers
  const bool on_chip = list[kGeneral].size() < size_t(D);  // some distro is planned by k_plan_cta, k_plan_smem or k_plan_warp
  if (any_complex) {
    CK(c->b_hasdep.ensure(size_t(T) + 16));
    CK(c->b_head.ensure(sizeof(uint32_t) * size_t(U + 1)));
    if (on_chip) {  // k_plan_smem's member lists, by pair id (a breakdown run plans tiny distros with it)
      CK(c->b_next.ensure(sizeof(uint32_t) * size_t(P + 1)));
      CK(c->b_pslot.ensure(sizeof(uint32_t) * size_t(P + 1)));
    }
    CK(c->b_etask.ensure(sizeof(uint32_t) * size_t(E + 1)));
    CK(c->b_elive.ensure(size_t(E) + 1));
    CK(c->b_unitv.ensure(sizeof(int64_t) * size_t(U + 1)));
    CK(c->b_unita.ensure(sizeof(uint32_t) * size_t(U + 1)));
    CK(c->b_unitn.ensure(sizeof(uint32_t) * size_t(U + 1)));
    CK(c->b_unitmask.ensure(sizeof(uint64_t) * size_t(U + 1)));
    CK(c->b_bestpair.ensure(sizeof(uint32_t) * size_t(T + 1)));
  }
  // k_plan_smem's scratch for value ranges above 32 bits; a breakdown run plans the tiny distros with it too
  if (on_chip) CK(c->b_kv.ensure(sizeof(uint64_t) * size_t(T + 1)));
  if (!list[kGeneral].empty()) {  // the general path's buffers exist only when a distro takes it
    for (int k = 0; k < 2; k++) {
      CK(c->b_klo[k].ensure(sizeof(uint32_t) * size_t(T + 1)));
      CK(c->b_khi[k].ensure(sizeof(uint32_t) * size_t(T + 1)));
      CK(c->b_ix[k].ensure(sizeof(uint32_t) * size_t(T + 1)));
    }
    CK(c->b_vmm.ensure(sizeof(uint64_t) * 2 * size_t(D + 1)));
    CK(c->b_gmisc.ensure(64));
    CK(c->b_tilesum.ensure(sizeof(uint32_t) * size_t(NT + 1)));
    CK(c->b_tilehist.ensure(sizeof(uint32_t) * 256 * size_t(NT + 1)));
    if (general_complex) {
      CK(c->b_e.ensure(sizeof(uint32_t) * size_t(T + kColPad)));
      CK(c->b_wl.ensure(sizeof(uint4) * size_t(Tgc + 1)));
      CK(c->b_pay.ensure(sizeof(URec) * size_t(Tgc + 1)));
      CK(c->b_place.ensure(sizeof(uint32_t) * 2 * size_t(Tgc + 1)));
      CK(c->b_eplace.ensure(sizeof(uint32_t) * 2 * size_t(E + 1)));
      CK(c->b_run.ensure(sizeof(uint32_t) * size_t(Prec + 1)));
      CK(c->b_rank.ensure(sizeof(uint32_t) * size_t(Prec + 1)));
      CK(c->b_emit.ensure(sizeof(uint32_t) * size_t(Prec + 1)));
      CK(c->b_blist.ensure(sizeof(uint2) * size_t(Prec / kRankOne + 1)));  // a unit of n > kRankOne members: ceil(n/32) <= n/kRankOne chunks
      CK(c->b_unit.ensure(sizeof(GUnit) * size_t(Urec + 1)));
    }
  }
  CK(c->b_punt.ensure(sizeof(int32_t) * size_t(D + 1)));
  CK(c->b_puntcnt.ensure(sizeof(int32_t) * (evg_ctx::kMaxChunks + 2)));
  CK(c->b_qinfo.ensure(sizeof(evg_queue_info) * size_t(D + 1)));
  CK(c->b_ginfo.ensure(sizeof(evg_group_info) * size_t(G + 1)));
  CK(c->b_order.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(c->b_tv.ensure(sizeof(int64_t) * size_t(T + kColPad)));
  c->T = T; c->E = E; c->G = G; c->U = U; c->NT = NT; c->Dn = D;
  c->t_pad = (T + 3) & ~int64_t(3);
  c->Tgc = Tgc;
  c->max_groups = 0;
  for (int32_t d = 0; d < D; d++) c->max_groups = std::max(c->max_groups, dt->group_off[d + 1] - dt->group_off[d]);
  c->any_complex = any_complex;
  c->general_complex = general_complex;
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  for (int r = 0; r < kRoutes; r++) c->routes[r].h.swap(list[r]);
  c->h_taskoff.assign(dt->task_off, dt->task_off + D + 1);
  c->h_groupoff.assign(dt->group_off, dt->group_off + D + 1);
  c->h_edgeoff.assign(size_t(D) + 1, 0);
  if (E > 0)
    for (int32_t d = 0; d <= D; d++) c->h_edgeoff[size_t(d)] = edge_off ? edge_off[d] : t->dep_off[dt->task_off[d]];
  c->h_nver.resize(size_t(D));
  for (int32_t d = 0; d < D; d++) c->h_nver[size_t(d)] = dt->cfg[d].n_versions;
  c->h_unitbase.swap(unit_base);
  c->h_dtileoff.swap(dtile_off);
  c->tick.kind = adopt ? Tick::kBorrowed : Tick::kFixed;  // the entry point that uploaded says whether evg_edit_tasks may follow
  c->alist_valid = false;  // upload_hosts lists the allocator's distros against THIS table
  if (cols != Cols::kChunked && T > 0) {  // range-check the ids the kernels index with
    launch(c, s, k_validate, grid_for(T, 256), 256, 0, dtasks(c), ddistros(c), dwork(c), int64_t(0), T);
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (bad) { drop_tick(c); return fail(EVG_ERR_INVALID, "a group_id / version_id / dep_idx is out of range for its distro"); }
  }
  return EVG_OK;
}

int upload_hosts(evg_ctx* c, const char* who, const evg_host_soa* h, const int64_t* host_off, const evg_alloc_cfg* acfg, int32_t D) {
  if (!h || (D > 0 && !acfg)) return fail(EVG_ERR_INVALID, "null host table / allocator config");
  const int64_t H = h->n_hosts;
  if (H < 0) return fail(EVG_ERR_INVALID, "negative n_hosts");
  if (D > 0 && !host_off) return fail(EVG_ERR_INVALID, "null host_off");
  if (D == 0 && H != 0) return fail(EVG_ERR_INVALID, "hosts without distros");
  const int rc = D > 0 ? check_offsets(host_off, D, H, who, "host_off") : EVG_OK;
  if (rc != EVG_OK) return rc;
  if (H > 0 && (!h->flags || !h->group_id || !h->expected_ns || !h->std_ns || !h->start_ns)) return fail(EVG_ERR_INVALID, "null host column");
  cudaStream_t s = c->stream;
  UP(s, c->b_hflags, h->flags, H, uint32_t);
  UP(s, c->b_hgid, h->group_id, H, int32_t);
  UP(s, c->b_hexp, h->expected_ns, H, int64_t);
  UP(s, c->b_hstd, h->std_ns, H, int64_t);
  UP(s, c->b_hstart, h->start_ns, H, int64_t);
  if (D > 0) UP(s, c->b_hostoff, host_off, D + 1, int64_t);
  UP(s, c->b_acfg, acfg, D, evg_alloc_cfg);
  c->alist_valid = false;
  std::vector<int32_t> alist;
  if (c->tick.kind != Tick::kNone && c->Dn == D && int64_t(c->h_groupoff.size()) == int64_t(D) + 1) {
    for (int32_t d = 0; d < D; d++)
      if (c->h_groupoff[d + 1] != c->h_groupoff[d] || host_off[d + 1] - host_off[d] > kGrouplessHosts) alist.push_back(d);
    UP(s, c->b_alist, alist.data(), int64_t(alist.size()), int32_t);
    CK(cudaStreamSynchronize(s));  // `alist` is a local
    c->n_alist = int64_t(alist.size());
    c->alist_valid = true;
  }
  CK(c->b_result.ensure(sizeof(evg_alloc_result) * size_t(D + 1)));
  CK(c->b_status.ensure(sizeof(int32_t) * size_t(D + 1)));
  c->H = H;
  c->tick.hosts = true;
  return EVG_OK;
}

DTasks dtasks(const evg_ctx* c) {
  DTasks t = c->tasks.view(c->T);
  t.n_edges = c->E;
  t.dep_off = c->b_depoff.as<int64_t>(); t.dep_idx = c->b_depidx.as<int32_t>();
  return t;
}
DDistros ddistros(const evg_ctx* c) {
  DDistros d;
  d.n = c->Dn; d.task_off = c->b_taskoff.as<int64_t>(); d.group_off = c->b_groupoff.as<int64_t>();
  d.cfg = c->b_cfg.as<evg_distro_cfg>(); d.gmax = c->b_gmax.as<int32_t>(); d.unit_base = c->b_unitbase.as<int64_t>();
  return d;
}
DWork dwork(const evg_ctx* c) {
  DWork w;
  w.has_dep = c->b_hasdep.as<uint8_t>(); w.head = c->b_head.as<uint32_t>(); w.next = c->b_next.as<uint32_t>();
  w.pair_slot = c->b_pslot.as<uint32_t>(); w.edge_task = c->b_etask.as<uint32_t>();
  w.edge_live = c->b_elive.as<uint8_t>(); w.route = c->b_route.as<uint8_t>();
  w.err = c->b_err.as<int>();
  w.unit_v = c->b_unitv.as<int64_t>(); w.unit_a = c->b_unita.as<uint32_t>(); w.unit_n = c->b_unitn.as<uint32_t>();
  w.unit_mask = c->b_unitmask.as<unsigned long long>();
  w.best_pair = c->b_bestpair.as<uint32_t>();
  w.buf[0].key_v = c->b_kv.as<uint64_t>();
  w.qinfo = c->b_qinfo.as<evg_queue_info>(); w.ginfo = c->b_ginfo.as<evg_group_info>();
  return w;
}
DGen dgen(const evg_ctx* c) {
  DGen g;
  g.n_tiles = c->NT;
  g.tile0 = 0;
  g.tile_distro = c->b_tiledistro.as<int32_t>(); g.tile_start = c->b_tilestart.as<int64_t>();
  g.dtile_off = c->b_dtileoff.as<int64_t>();
  g.vmm = c->b_vmm.as<unsigned long long>();
  for (int k = 0; k < 2; k++) {
    g.key_lo[k] = c->b_klo[k].as<uint32_t>(); g.key_hi[k] = c->b_khi[k].as<uint32_t>(); g.idx[k] = c->b_ix[k].as<uint32_t>();
  }
  g.e = c->b_e.as<uint32_t>(); g.tile_sum = c->b_tilesum.as<uint32_t>(); g.tile_hist = c->b_tilehist.as<uint32_t>();
  g.wl = c->b_wl.as<uint4>();
  g.pay = c->b_pay.as<URec>();
  g.pown = c->b_place.as<uint32_t>();
  g.pver = c->b_place.as<uint32_t>() + (c->Tgc + 1);
  g.pedge = c->b_eplace.as<uint32_t>();
  g.sedge = c->b_eplace.as<uint32_t>() + (c->E + 1);
  g.ccount = c->b_gmisc.as<unsigned int>();
  g.maxpass = c->b_gmisc.as<int32_t>() + 1;
  g.rcount = c->b_gmisc.as<unsigned int>() + 2;
  g.hcount = c->b_gmisc.as<unsigned int>() + 3;
  g.bcount = c->b_gmisc.as<unsigned int>() + 4;
  g.blist = c->b_blist.as<uint2>();
  g.rank = c->b_rank.as<uint32_t>();
  g.emit = c->b_emit.as<uint32_t>();
  g.unit = c->b_unit.as<GUnit>();
  g.run = c->b_run.as<uint32_t>();
  g.tv = c->b_tv.as<int64_t>();
  return g;
}


int run_alloc_range(evg_ctx* c, int64_t now, int32_t d0, int32_t d1) {
  DHosts h;
  h.n = c->H; h.flags = c->b_hflags.as<uint32_t>(); h.gid = c->b_hgid.as<int32_t>();
  h.expected = c->b_hexp.as<int64_t>(); h.stddev = c->b_hstd.as<int64_t>(); h.start = c->b_hstart.as<int64_t>();
  h.host_off = c->b_hostoff.as<int64_t>(); h.cfg = c->b_acfg.as<evg_alloc_cfg>();
  if (c->ext_result && c->ext_capacity < c->Dn) return fail(EVG_ERR_INVALID, "bound result buffer holds %lld rows, need %d", (long long)c->ext_capacity, c->Dn);
  CK(c->b_gs.ensure(sizeof(GroupScratch) * size_t(c->G + 1)));
  // a warp per distro (four per block) unless some distro has thousands of task groups, then a block per distro
  // ... and a thread per distro for the distros that have no task groups, when there are enough distros for that to matter
  const int split = (d1 - d0) >= 4096 ? 1 : 0;
  // ... and only for the distros it has to take when the upload listed them (whole-table ranges)
  const bool listed = split && c->alist_valid && d0 == 0 && d1 == c->Dn;
  const int32_t* al = listed ? c->b_alist.as<int32_t>() : nullptr;
  const int64_t teams = listed ? c->n_alist : int64_t(d1 - d0);
  if (c->max_groups > kWideAllocGroups)
    launch(c, c->stream, k_alloc<128>, unsigned(teams), 128, 0, h, d0, d1, c->b_groupoff.as<int64_t>(), c->b_qinfo.as<evg_queue_info>(),
           c->b_ginfo.as<evg_group_info>(), c->b_gs.as<GroupScratch>(), now, c->result_ptr(), c->b_status.as<int32_t>(), split, al, int32_t(c->n_alist));
  else
    launch(c, c->stream, k_alloc<32>, grid_for(teams, 4), 128, 0, h, d0, d1, c->b_groupoff.as<int64_t>(), c->b_qinfo.as<evg_queue_info>(),
           c->b_ginfo.as<evg_group_info>(), c->b_gs.as<GroupScratch>(), now, c->result_ptr(), c->b_status.as<int32_t>(), split, al, int32_t(c->n_alist));
  if (split)
    launch(c, c->stream, k_alloc_groupless, grid_for(d1 - d0, 128), 128, 0, h, d0, d1, c->b_groupoff.as<int64_t>(), c->b_qinfo.as<evg_queue_info>(),
           now, c->result_ptr(), c->b_status.as<int32_t>());
  CK(cudaGetLastError());
  return EVG_OK;
}
int run_alloc(evg_ctx* c, int64_t now) { return run_alloc_range(c, now, 0, c->Dn); }

template <int THREADS, int ITEMS, int MIN_CTAS>
int launch_smem(evg_ctx* c, cudaStream_t st, const DTasks& dt, const DDistros& dd, const DWork& w, const int32_t* list, int32_t n,
                int64_t now, int lists_needed = 0, const int32_t* list_count = nullptr) {
  if (n <= 0) return EVG_OK;
  const size_t bytes = PlanSmem<THREADS, ITEMS>::kBytes;
  CK(cudaFuncSetAttribute(k_plan_smem<THREADS, ITEMS, MIN_CTAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes)));
  launch(c, st, k_plan_smem<THREADS, ITEMS, MIN_CTAS>, unsigned(n), THREADS, bytes, dt, dd, w, list, list_count, now, lists_needed,
         c->b_order.as<int32_t>(), c->b_tv.as<int64_t>());
  return EVG_OK;
}

// Second-generation on-chip planner for one class; distros it hands back land in punt_list[0 .. *punt_count).
template <int THREADS, int CAP, int OCC>
int launch_cta(evg_ctx* c, cudaStream_t st, const DTasks& dt, const DDistros& dd, const DWork& w, const int32_t* list, int32_t n,
               int64_t now, int32_t* punt_list, int32_t* punt_count) {
  if (n <= 0) return EVG_OK;
  const size_t bytes = PlanCta<THREADS, CAP>::kBytes;
  CK(cudaFuncSetAttribute(k_plan_cta<THREADS, CAP, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes)));
  launch(c, st, k_plan_cta<THREADS, CAP, OCC>, unsigned(n), THREADS, bytes, dt, dd, w, list, now, c->t_pad, c->b_order.as<int32_t>(),
         c->b_tv.as<int64_t>(), punt_list, punt_count);
  return EVG_OK;
}

// Distros of at most 32 tasks: one warp each (k_plan_warp).  Breakdown mode needs the unit lists, so it
// sends them through the smallest on-chip class instead.
int launch_tiny(evg_ctx* c, cudaStream_t st, const DTasks& dt, const DDistros& dd, const DWork& w, const int32_t* list, int32_t n,
                int64_t now, int lists_needed) {
  if (lists_needed) return launch_smem<128, 8, 8>(c, st, dt, dd, w, list, n, now, 1);
  launch(c, st, k_plan_warp, grid_for(int64_t(n) * 32, 256), 256, 0, dt, dd, w, list, n, now, c->b_order.as<int32_t>(), c->b_tv.as<int64_t>());
  return EVG_OK;
}

// Everything the general path accumulates into or links through starts from zero / "empty", for the distros
// [d0, d1) (first to last general-path distro of the tick, or of one chunk of the pipelined call).  On the resident
// path this runs on the context stream BEFORE the routes fork: an on-chip distro inside the span rewrites its own rows
// afterwards.
int prepare_general(evg_ctx* c, cudaStream_t s, int32_t d0, int32_t d1) {
  const int64_t t0 = c->h_taskoff[d0], t1 = c->h_taskoff[d1], u0 = c->h_unitbase[d0], u1 = c->h_unitbase[d1];
  const int64_t g0 = c->h_groupoff[d0], g1 = c->h_groupoff[d1], e0 = c->h_edgeoff[d0], e1 = c->h_edgeoff[d1];
  CK(cudaMemsetAsync(c->b_qinfo.as<evg_queue_info>() + d0, 0, sizeof(evg_queue_info) * size_t(d1 - d0), s));
  if (g1 > g0) CK(cudaMemsetAsync(c->b_ginfo.as<evg_group_info>() + g0, 0, sizeof(evg_group_info) * size_t(g1 - g0), s));
  if (c->general_complex) {
    const size_t nt = size_t(t1 - t0);
    CK(cudaMemsetAsync(c->b_hasdep.as<uint8_t>() + t0, 0, nt, s));
    CK(cudaMemsetAsync(c->b_unitn.as<uint32_t>() + u0, 0, sizeof(uint32_t) * size_t(u1 - u0), s));   // members drawn so far
  }
  return EVG_OK;
}

// The general path on stream `st` for the general-path distros routes[kGeneral][gfirst .. gfirst + gcount) (evg_plan_general.cuh).
int run_general(evg_ctx* c, cudaStream_t st, const DTasks& dt, const DDistros& dd, const DWork& w, int64_t now, int32_t gfirst,
                int32_t gcount) {
  if (gcount <= 0) return EVG_OK;
  DGen g = dgen(c);
  const int gc = c->general_complex;
  const std::vector<int32_t>& gh = c->routes[kGeneral].h;
  const int32_t d_first = gh[size_t(gfirst)], d_last = gh[size_t(gfirst + gcount - 1)];
  g.tile0 = c->h_dtileoff[size_t(d_first)];
  const unsigned nt = unsigned(c->h_dtileoff[size_t(d_last) + 1] - g.tile0);
  const int32_t* gl = c->routes[kGeneral].b.as<int32_t>() + gfirst;
  launch(c, st, k_ginit, grid_for(gcount, 256), 256, 0, g, gl, gcount);
  if (gc && c->E > 0) launch(c, st, k_gmark, nt, 256, 0, dt, dd, w, g);
  if (c->timed) CK(cudaEventRecord(c->ev_gt0, st));
  launch(c, st, k_gtask, nt, 256, 0, dt, dd, w, g, now, gc);
  if (c->timed) { CK(cudaEventRecord(c->ev_gt1, st)); c->general_timed = true; }
  const unsigned wl_grid = unsigned(std::min<int64_t>(std::max<int64_t>(1, (c->Tgc + 255) / 256), int64_t(c->num_sms) * 16));
  if (gc) {
    launch(c, st, k_glink, wl_grid, 256, 0, dt, dd, w, g, now);
    launch(c, st, k_galloc, wl_grid, 256, 0, dt, dd, w, g);
    launch(c, st, k_gfill, wl_grid, 256, 0, dt, dd, w, g);
    launch(c, st, k_gunit, wl_grid, 256, 0, dd, w, g, now);
    launch(c, st, k_grank, wl_grid, 256, 0, w, g);
    launch(c, st, k_gbest, wl_grid, 256, 0, dt, dd, w, g, c->bd_valid ? 1 : 0);
  }
  launch(c, st, k_gsched, grid_for(gcount, 128), 128, 0, g, gl, gcount);
  if (gc) {
    launch(c, st, k_gsum, nt, 256, 0, dd, g);
    launch(c, st, k_gscan, unsigned(gcount), 1024, 0, g, gl);
  }
  launch(c, st, k_gplace, nt, 256, 0, dd, w, g, gc);
  if (gc) launch(c, st, k_gplace_unit, wl_grid, 256, 0, dd, w, g);
  if (c->timed) CK(cudaEventRecord(c->ev_sort0, st));  // the general path's segmented sort
  for (int j = 0; j < 8; j++) {  // passes beyond the tick's longest key exit at once (*maxpass is device-side)
    launch(c, st, k_ghist, nt, 256, 0, j, dd, g);
    launch(c, st, k_gdscan, unsigned(gcount), 1024, 0, j, gl, g);
    launch(c, st, k_gscatter, nt, 256, 0, j, dd, g, c->b_order.as<int32_t>(), c->b_tv.as<int64_t>());
  }
  if (c->timed) CK(cudaEventRecord(c->ev_sort1, st));
  const int64_t g0 = c->h_groupoff[size_t(d_first)], g1 = c->h_groupoff[size_t(d_last) + 1];
  launch(c, st, k_finalize_info, grid_for(std::max<int64_t>(d_last + 1 - d_first, g1 - g0), 256), 256, 0, dd, w, d_first, d_last + 1, g0, g1);
  return EVG_OK;
}

int ensure_aux_streams(evg_ctx* c) {
  if (c->ev_fork) return EVG_OK;
  for (int k = 0; k < evg_ctx::kAux; k++) {
    CK(cudaStreamCreateWithFlags(&c->s_aux[k], cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&c->ev_join[k], cudaEventDisableTiming));
  }
  CK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  return EVG_OK;
}

// The resident tick, the resident tick with the unit lists EVG_OPT_BREAKDOWN reads, or one chunk of the pipelined
// one-shot call.
enum class Mode { kResident, kBreakdown, kPipelined };

// The planner launch of size class r in `mode`: entries [first, first + n) of its list -- the largest-first copy on the
// resident tick, the ascending list (cut by chunk) on the pipelined call -- on stream st.  The k_plan_cta classes hand
// distros back into punt[0 .. *punt_count); r = kPunted replans them, n being how many could come back.
int plan_route(evg_ctx* c, int r, Mode mode, cudaStream_t st, const DTasks& dt, const DDistros& dd, const DWork& w, int64_t now,
               int32_t first, int32_t n, int32_t* punt, int32_t* punt_count) {
  if (n <= 0) return EVG_OK;
  const int bd = mode == Mode::kBreakdown ? 1 : 0;
  const int32_t* list = punt;
  if (r != kPunted) list = (mode != Mode::kPipelined && largest_first(r) ? c->routes[r].lpt : c->routes[r].b).as<int32_t>() + first;
  // breakdown needs the unit lists: every k_plan_cta distro goes through k_plan_smem (its largest class holds them all)
  if (bd && is_cta(r)) return launch_smem<kThreadsC, kItemsC, 1>(c, st, dt, dd, w, list, n, now, 1);
  int rc;
  switch (r) {
    case kCtaC: return launch_cta<kNT_C, kNCapC, kNOccC>(c, st, dt, dd, w, list, n, now, punt, punt_count);
    case kCtaB: return launch_cta<kNT_B, kNCapB, kNOccB>(c, st, dt, dd, w, list, n, now, punt, punt_count);
    case kCtaA:
      if (mode == Mode::kResident) {  // the distros that fit the 64-thread instance are the tail of the largest-first list
        if ((rc = launch_cta<kNT_A, kNCapA, kNOccA>(c, st, dt, dd, w, list, c->nNA_big, now, punt, punt_count)) != EVG_OK) return rc;
        return launch_cta<kNT_S, kNCapS, kNOccS>(c, st, dt, dd, w, list + c->nNA_big, n - c->nNA_big, now, punt, punt_count);
      }
      return launch_cta<kNT_A, kNCapA, kNOccA>(c, st, dt, dd, w, list, n, now, punt, punt_count);
    case kPunted:
      // the resident tick takes the smallest k_plan_smem instance that holds the largest distro given to k_plan_cta (the
      // launch has one CTA per distro that COULD come back; CTAs beyond *punt_count exit at once, and 10^4 empty
      // 1024-thread CTAs are not free); the pipelined call always takes the largest
      if (mode == Mode::kResident && c->max_cta_tasks <= kCapA) return launch_smem<128, 8, 8>(c, st, dt, dd, w, list, n, now, 0, punt_count);
      if (mode == Mode::kResident && c->max_cta_tasks <= kCapB) return launch_smem<256, 16, 3>(c, st, dt, dd, w, list, n, now, 0, punt_count);
      return launch_smem<kThreadsC, kItemsC, 1>(c, st, dt, dd, w, list, n, now, 0, punt_count);
    case kSmemC: return launch_smem<kThreadsC, kItemsC, 1>(c, st, dt, dd, w, list, n, now, bd);
    case kSmemB: return launch_smem<256, 16, 3>(c, st, dt, dd, w, list, n, now, bd);
    case kSmemA: return launch_smem<128, 8, 8>(c, st, dt, dd, w, list, n, now, bd);
    case kWarp: return launch_tiny(c, st, dt, dd, w, list, n, now, bd);
    default: {  // kGeneral; the resident tick prepares all its general-path distros before the routes fork
      const std::vector<int32_t>& gh = c->routes[kGeneral].h;
      if (mode == Mode::kPipelined && (rc = prepare_general(c, st, gh[size_t(first)], gh[size_t(first + n - 1)] + 1)) != EVG_OK) return rc;
      return run_general(c, st, dt, dd, w, now, first, n);
    }
  }
}

int run_plan(evg_ctx* c, int64_t now, uint32_t opts) {
  const int64_t T = c->T;
  const int32_t D = c->Dn;
  cudaStream_t s = c->stream;
  DTasks dt = dtasks(c);
  DDistros dd = ddistros(c);
  DWork w = dwork(c);
  int64_t* bd = nullptr;
  c->bd_valid = false;
  if (opts & EVG_OPT_BREAKDOWN) {
    CK(c->b_bd.ensure(sizeof(int64_t) * EVG_BD_N * size_t(T + 1)));
    bd = c->b_bd.as<int64_t>();
    c->bd_valid = true;
  }
  c->sort_slot = -1;
  if (D == 0) {
    if (c->timed) { CK(cudaEventRecord(c->ev_sort0, s)); CK(cudaEventRecord(c->ev_sort1, s)); }
    return EVG_OK;
  }
  const std::vector<int32_t>& gh = c->routes[kGeneral].h;
  const bool general = !gh.empty();
  // breakdown mode reads best_pair for every task: tasks emitted from their own single-task unit keep kInactive
  if (bd && c->any_complex) CK(cudaMemsetAsync(c->b_bestpair.p, 0xFF, sizeof(uint32_t) * size_t(T + 1), s));
  const int32_t n_new = bd ? 0 : c->routes[kCtaA].n() + c->routes[kCtaB].n() + c->routes[kCtaC].n();  // could be handed back
  if (n_new > 0) CK(cudaMemsetAsync(c->b_puntcnt.p, 0, sizeof(int32_t), s));
  if (general) { int rcg = prepare_general(c, s, gh.front(), gh.back() + 1); if (rcg != EVG_OK) return rcg; }
  // Routes run side by side when the tick has more than one: fork the aux streams off the context stream here, join
  // them before returning (the allocator and the caller's later work are ordered behind every planner kernel).
  bool busy[evg_ctx::kAux] = {};
  for (int r = 0; r < kRoutes; r++) busy[kRouteStream[r]] |= c->routes[r].n() > 0;
  const bool fork = std::count(busy, busy + evg_ctx::kAux, true) > 1;
  if (fork) {
    int rc0 = ensure_aux_streams(c);
    if (rc0 != EVG_OK) return rc0;
    CK(cudaEventRecord(c->ev_fork, s));
    for (int k = 0; k < evg_ctx::kAux; k++) CK(cudaStreamWaitEvent(c->s_aux[k], c->ev_fork, 0));
  }
  int rc;
  const int slot = int(c->runs % evg_ctx::kRing);
  const Mode mode = bd ? Mode::kBreakdown : Mode::kResident;
  // stream 0: k_plan_cta (the dominant kernel of configs[1]-like ticks), then the distros it handed back; streams 1..3:
  // k_plan_smem (GroupVersions, in-queue dependency edges, very many task groups); 4: tiny distros; 5: the general path
  for (int r : {kCtaC, kCtaB, kCtaA, kPunted, kSmemC, kSmemB, kSmemA, kWarp, kGeneral}) {
    const int32_t n = r == kPunted ? n_new : c->routes[r].n();
    cudaStream_t sr = fork ? c->s_aux[kRouteStream[r]] : s;
    // the timing ring brackets k_plan_cta's largest class (not in breakdown mode), else k_plan_smem's largest class; a
    // tick with general-path distros has its own sort events instead
    const bool time_it = c->timed && !general && c->sort_slot < 0 && n > 0 && (r == kSmemC || (r == kCtaC && !bd));
    if (time_it) CK(cudaEventRecord(c->ring0[slot], sr));
    if ((rc = plan_route(c, r, mode, sr, dt, dd, w, now, 0, n, c->b_punt.as<int32_t>(), c->b_puntcnt.as<int32_t>())) != EVG_OK) return rc;
    if (time_it) { CK(cudaEventRecord(c->ring1[slot], sr)); c->runs++; c->sort_slot = slot; }
  }
  if (fork) {
    for (int k = 0; k < evg_ctx::kAux; k++) {
      CK(cudaEventRecord(c->ev_join[k], c->s_aux[k]));
      CK(cudaStreamWaitEvent(s, c->ev_join[k], 0));
    }
  }
  if (bd) launch(c, c->stream, k_breakdown, grid_for(T, 256), 256, 0, dt, dd, w, c->b_run.as<uint32_t>(), c->b_pay.as<URec>(), c->b_unit.as<GUnit>(), now, c->any_complex, c->b_order.as<int32_t>(), bd);
  CK(cudaGetLastError());
  return EVG_OK;
}

}  // namespace

// --------------------------------------------------------------------------
// C-ABI
// --------------------------------------------------------------------------
extern "C" {

const char* evg_last_error(void) { return g_err.c_str(); }
int evg_abi_version(void) { return EVG_ABI_VERSION; }

int evg_init(int device, void* stream, evg_ctx** out) {
  if (!out) return fail(EVG_ERR_INVALID, "evg_init: out is null");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) return fail(EVG_ERR_CUDA, "no CUDA device: %s (libevgsched has no CPU fallback)", cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(EVG_ERR_INVALID, "device %d out of range (%d devices)", device, n);
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(EVG_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  evg_ctx* c = new evg_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  if (stream) { c->stream = reinterpret_cast<cudaStream_t>(stream); c->own_stream = false; }
  else { CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
  CK(cudaEventCreate(&c->ev_begin)); CK(cudaEventCreate(&c->ev_sort0));
  CK(cudaEventCreate(&c->ev_sort1)); CK(cudaEventCreate(&c->ev_end));
  CK(cudaEventCreate(&c->ev_gt0)); CK(cudaEventCreate(&c->ev_gt1));
  for (int k = 0; k < evg_ctx::kRing; k++) { CK(cudaEventCreate(&c->ring0[k])); CK(cudaEventCreate(&c->ring1[k])); }
  *out = c;
  return EVG_OK;
}

void evg_shutdown(evg_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (int k = 0; k < evg_ctx::kRing; k++) { if (c->ring0[k]) cudaEventDestroy(c->ring0[k]); if (c->ring1[k]) cudaEventDestroy(c->ring1[k]); }
  cudaEventDestroy(c->ev_begin); cudaEventDestroy(c->ev_sort0); cudaEventDestroy(c->ev_sort1); cudaEventDestroy(c->ev_end);
  cudaEventDestroy(c->ev_gt0); cudaEventDestroy(c->ev_gt1);
  for (int k = 0; k < evg_ctx::kMaxChunks; k++) { if (c->ev_h[k]) cudaEventDestroy(c->ev_h[k]); if (c->ev_c[k]) cudaEventDestroy(c->ev_c[k]); }
  if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
  if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
  for (int k = 0; k < evg_ctx::kAux; k++) { if (c->s_aux[k]) cudaStreamDestroy(c->s_aux[k]); if (c->ev_join[k]) cudaEventDestroy(c->ev_join[k]); }
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->own_stream) cudaStreamDestroy(c->stream);
  delete c;  // its buffers free themselves, on the device selected above
}

// evg_upload for the entry point `who` (the caller holds the context's lock), leaving a tick of the given kind; `cols`
// and `edge_off` as for upload_tasks
static int upload(evg_ctx* c, const char* who, const evg_task_soa* tasks, const evg_distro_table* distros, const evg_host_soa* hosts,
                  const int64_t* host_off, const evg_alloc_cfg* acfg, Tick kind, Cols cols = Cols::kCopy,
                  const int64_t* edge_off = nullptr) {
  int rc = upload_tasks(c, who, tasks, distros, cols, edge_off);
  if (rc != EVG_OK) return rc;
  if (hosts) {
    rc = upload_hosts(c, who, hosts, host_off, acfg, distros->n_distros);
    if (rc != EVG_OK) return rc;
    CK(cudaStreamSynchronize(c->stream));
  }
  c->tick.kind = kind;
  return EVG_OK;
}
int evg_upload(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_table* distros, const evg_host_soa* hosts,
               const int64_t* host_off, const evg_alloc_cfg* acfg) {
  ENTER(c, "evg_upload");
  return upload(c, who, tasks, distros, hosts, host_off, acfg, Tick::kOwn);
}

__global__ void k_gather_i64(const int64_t* __restrict__ src, const int64_t* __restrict__ at, int64_t* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[at[i]];
}

// evg_update_tasks: scatter changed rows into the resident columns.
__global__ void __launch_bounds__(256) k_update_rows(int64_t n, const int64_t* __restrict__ rows, int64_t T, int32_t* priority, int32_t* numdep,
                                                     int32_t* tgo, uint32_t* flags, int64_t* expected, int64_t* qbasis, int64_t* wbasis,
                                                     const int32_t* v_priority, const int32_t* v_numdep, const int32_t* v_tgo,
                                                     const uint32_t* v_flags, const int64_t* v_expected, const int64_t* v_qbasis,
                                                     const int64_t* v_wbasis, int* bad) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = rows[i];
  if (r < 0 || r >= T) { *bad = 1; return; }
  priority[r] = v_priority[i]; numdep[r] = v_numdep[i]; tgo[r] = v_tgo[i]; flags[r] = v_flags[i];
  expected[r] = v_expected[i]; qbasis[r] = v_qbasis[i]; wbasis[r] = v_wbasis[i];
}

int evg_update_tasks(evg_ctx* c, int64_t n_rows, const int64_t* rows, const evg_task_soa* v) {
  ENTER(c, "evg_update_tasks");
  if (const int rc = need_tick(c, who, Need::kOwnColumns); rc != EVG_OK) return rc;
  if (n_rows < 0) return fail(EVG_ERR_INVALID, "negative row count");
  if (n_rows == 0) return EVG_OK;
  if (!rows || !v || v->n_tasks != n_rows || TaskCols::missing(v, /*ids=*/false))
    return fail(EVG_ERR_INVALID, "evg_update_tasks: rows and a %lld-row value table (priority, num_dependents, task_group_order, flags, "
                                 "expected_ns, queue_basis_ns, wait_basis_ns) are required", (long long)n_rows);
  cudaStream_t s = c->stream;
  const size_t n = size_t(n_rows);
  // staging: rows (8) + the nine columns but group_id and version_id, the 8-byte ones first = 48 B per changed row
  CK(c->b_upd.ensure(n * 48 + 64));
  unsigned char* at = c->b_upd.as<unsigned char>();
  const int64_t* d_rows = reinterpret_cast<int64_t*>(at);
  CK(cudaMemcpyAsync(at, rows, n * 8, cudaMemcpyHostToDevice, s));
  at += n * 8;
  evg_task_soa d{};  // the staged values
  const int rc = TaskCols::each([&](auto b, auto f, const char*) -> int {
    if (TaskCols::is_id(b)) return EVG_OK;
    TaskCols::point(d.*f, at);
    CK(cudaMemcpyAsync(at, v->*f, TaskCols::elem(f) * n, cudaMemcpyHostToDevice, s));
    at += TaskCols::elem(f) * n;
    return EVG_OK;
  });
  if (rc != EVG_OK) return rc;
  int* bad = reinterpret_cast<int*>(at);
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  const EdDst o = c->tasks.dst();
  launch(c, s, k_update_rows, grid_for(n_rows, 256), 256, 0, n_rows, d_rows, c->T, o.priority, o.numdep, o.tgo, o.flags, o.expected,
         o.qbasis, o.wbasis, d.priority, d.num_dependents, d.task_group_order, d.flags, d.expected_ns, d.queue_basis_ns, d.wait_basis_ns, bad);
  CK(cudaGetLastError());
  int h_bad = 0;
  CK(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));  // the caller's staging arrays are free again
  if (h_bad) return fail(EVG_ERR_INVALID, "evg_update_tasks: a row index is outside [0, n_tasks)");
  c->tick.deps = false;  // flags / wait bases written by a device-side dependency evaluation may have been replaced
  return EVG_OK;
}

int evg_upload_device(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_table* distros, const evg_host_soa* hosts,
                      const int64_t* host_off, const evg_alloc_cfg* acfg) {
  ENTER(c, "evg_upload_device");
  if (!tasks || !distros) return fail(EVG_ERR_INVALID, "null task table / distro table");
  std::vector<int64_t> edge_off;
  const int32_t D = distros->n_distros;
  if (tasks->n_edges > 0 && D > 0) {  // dep_off is device memory: sample it at the distro boundaries for the routing
    if (!tasks->dep_off || !distros->task_off) return fail(EVG_ERR_INVALID, "null dep_off / task_off");
    edge_off.resize(size_t(D) + 1);
    CK(c->b_rn0.ensure(sizeof(int64_t) * size_t(D + 1)));
    CK(c->b_rn1.ensure(sizeof(int64_t) * size_t(D + 1)));
    CK(cudaMemcpyAsync(c->b_rn0.p, distros->task_off, sizeof(int64_t) * size_t(D + 1), cudaMemcpyHostToDevice, c->stream));
    launch(c, c->stream, k_gather_i64, grid_for(D + 1, 256), 256, 0, tasks->dep_off, c->b_rn0.as<int64_t>(), c->b_rn1.as<int64_t>(), D + 1);
    CK(cudaMemcpyAsync(edge_off.data(), c->b_rn1.p, sizeof(int64_t) * size_t(D + 1), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  return upload(c, who, tasks, distros, hosts, host_off, acfg, Tick::kBorrowed, Cols::kAdopt,
                edge_off.empty() ? nullptr : edge_off.data());
}

int evg_run_resident(evg_ctx* c, int64_t now_ns, uint32_t opts) {
  ENTER(c, "evg_run_resident");
  if (const int rc = need_tick(c, who, Need::kTick); rc != EVG_OK) return rc;
  c->launches = 0;
  c->timed = true;
  c->general_timed = false;
  c->tick.allocated = c->tick.host_job = c->tick.dispatchers = false;
  CK(cudaEventRecord(c->ev_begin, c->stream));
  int rc = run_plan(c, now_ns, opts);
  if (rc != EVG_OK) return rc;
  if (c->tick.hosts) {
    rc = run_alloc(c, now_ns);
    if (rc != EVG_OK) return rc;
    c->tick.allocated = true;
  }
  CK(cudaEventRecord(c->ev_end, c->stream));
  return EVG_OK;
}

int evg_download(evg_ctx* c, evg_plan_out* po, evg_alloc_out* ao) {
  ENTER(c, "evg_download");
  if (const int rc = need_tick(c, who, Need::kTick); rc != EVG_OK) return rc;
  cudaStream_t s = c->stream;
  if (po) {
    if (po->order && c->T) CK(cudaMemcpyAsync(po->order, c->b_order.p, sizeof(int32_t) * size_t(c->T), cudaMemcpyDeviceToHost, s));
    if (po->total_value && c->T) CK(cudaMemcpyAsync(po->total_value, c->b_tv.p, sizeof(int64_t) * size_t(c->T), cudaMemcpyDeviceToHost, s));
    if (po->breakdown && c->T) {
      if (!c->bd_valid) return fail(EVG_ERR_STATE, "breakdown requested but the run did not set EVG_OPT_BREAKDOWN");
      CK(cudaMemcpyAsync(po->breakdown, c->b_bd.p, sizeof(int64_t) * EVG_BD_N * size_t(c->T), cudaMemcpyDeviceToHost, s));
    }
    if (po->info && c->Dn) CK(cudaMemcpyAsync(po->info, c->b_qinfo.p, sizeof(evg_queue_info) * size_t(c->Dn), cudaMemcpyDeviceToHost, s));
    if (po->group_info && c->G) CK(cudaMemcpyAsync(po->group_info, c->b_ginfo.p, sizeof(evg_group_info) * size_t(c->G), cudaMemcpyDeviceToHost, s));
  }
  if (ao) {
    if (const int rc = need_tick(c, who, Need::kHosts); rc != EVG_OK) return rc;
    if (ao->result && c->Dn) CK(cudaMemcpyAsync(ao->result, c->result_ptr(), sizeof(evg_alloc_result) * size_t(c->Dn), cudaMemcpyDeviceToHost, s));
    if (ao->status && c->Dn) CK(cudaMemcpyAsync(ao->status, c->b_status.p, sizeof(int32_t) * size_t(c->Dn), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

// TaskQueueItem rows of the persisted head of every queue (task_queue_persister.go:14-42): one thread per output row.
__global__ void __launch_bounds__(256) k_project_queue(DTasks T, DDistros D, const int64_t* __restrict__ item_off, int64_t n_items,
                                                       const int32_t* __restrict__ order, const int64_t* __restrict__ total_value,
                                                       evg_queue_item* __restrict__ items) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= n_items) return;
  const int d = find_distro(item_off, 0, D.n - 1, j);
  const int64_t base = D.task_off[d];
  const int64_t r = j - item_off[d];
  const int32_t i = order[base + r];
  const int64_t t = base + i;
  const int32_t gid = T.gid[t];
  evg_queue_item q;
  q.task = i;
  q.group_index = T.tgo[t];
  q.group_max_hosts = gid >= 0 ? D.gmax[D.group_off[d] + gid] : 0;
  q.flags = (T.flags[t] & EVG_TF_DEPS_MET) ? EVG_QI_DEPS_MET : 0u;
  q.priority = T.priority[t];
  q.expected_ns = T.expected[t];
  q.total_value = total_value[base + r];
  items[j] = q;
}

// The persisted head of every queue of the resident tick: item_off[d + 1] - item_off[d] = min(length, cap) (cap > 0).
// Returns the rows in all.
static int64_t persisted_item_off(const evg_ctx* c, int32_t cap, int64_t* item_off) {
  item_off[0] = 0;
  for (int32_t d = 0; d < c->Dn; d++) item_off[d + 1] = item_off[d] + std::min<int64_t>(c->h_taskoff[d + 1] - c->h_taskoff[d], cap);
  return item_off[c->Dn];
}

int evg_download_queue(evg_ctx* c, int32_t cap, int64_t* item_off, evg_queue_item* items, int64_t items_capacity) {
  ENTER(c, "evg_download_queue");
  if (const int rc = need_tick(c, who, Need::kTick); rc != EVG_OK) return rc;
  if (cap < 0 || !item_off) return fail(EVG_ERR_INVALID, "evg_download_queue: bad argument");
  if (cap == 0) cap = EVG_PERSISTED_QUEUE_CAP;
  const int32_t D = c->Dn;
  const int64_t n = persisted_item_off(c, cap, item_off);
  if (n > items_capacity || (n > 0 && !items)) return fail(EVG_ERR_INVALID, "evg_download_queue: %lld rows needed, %lld available", (long long)n, (long long)items_capacity);
  if (n == 0) return EVG_OK;
  cudaStream_t s = c->stream;
  CK(c->b_rn0.ensure(sizeof(int64_t) * size_t(D + 1)));
  CK(c->b_rn1.ensure(sizeof(evg_queue_item) * size_t(n)));
  CK(cudaMemcpyAsync(c->b_rn0.p, item_off, sizeof(int64_t) * size_t(D + 1), cudaMemcpyHostToDevice, s));
  launch(c, s, k_project_queue, grid_for(n, 256), 256, 0, dtasks(c), ddistros(c), c->b_rn0.as<int64_t>(), n, c->b_order.as<int32_t>(),
         c->b_tv.as<int64_t>(), c->b_rn1.as<evg_queue_item>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(items, c->b_rn1.p, sizeof(evg_queue_item) * size_t(n), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

// The two queries that return no status take the lock and leave the device alone.
void* evg_device_result_ptr(evg_ctx* c) {
  if (!c) return nullptr;
  std::lock_guard<std::recursive_mutex> lock_(c->mu);
  return c->result_ptr();
}
int64_t evg_last_launch_count(evg_ctx* c) {
  if (!c) return 0;
  std::lock_guard<std::recursive_mutex> lock_(c->mu);
  return c->launches;
}
int evg_bind_result_buffer(evg_ctx* c, void* device_ptr, int64_t capacity) {
  ENTER(c, "evg_bind_result_buffer");
  if (device_ptr && capacity < 0) return fail(EVG_ERR_INVALID, "negative capacity");
  c->ext_result = reinterpret_cast<evg_alloc_result*>(device_ptr);
  c->ext_capacity = device_ptr ? capacity : 0;
  c->tick.allocated = c->tick.host_job = false;  // the last run's result rows are not in the buffer bound now
  return EVG_OK;
}
int evg_last_timing_ms(evg_ctx* c, float* total_ms, float* sort_ms) {
  ENTER(c, "evg_last_timing_ms");
  if (!c->timed) return fail(EVG_ERR_STATE, "no timed run");
  CK(cudaEventSynchronize(c->ev_end));
  if (total_ms) CK(cudaEventElapsedTime(total_ms, c->ev_begin, c->ev_end));
  if (sort_ms) {
    if (c->sort_slot >= 0) CK(cudaEventElapsedTime(sort_ms, c->ring0[c->sort_slot], c->ring1[c->sort_slot]));
    else if (c->general_timed) CK(cudaEventElapsedTime(sort_ms, c->ev_sort0, c->ev_sort1));
    else *sort_ms = 0.0f;  // a tick of small distros only: no kernel of its own was bracketed
  }
  return EVG_OK;
}

int evg_general_timing_ms(evg_ctx* c, float* task_pass_ms, float* sort_ms) {
  ENTER(c, "evg_general_timing_ms");
  if (!c->timed || !c->general_timed) return fail(EVG_ERR_STATE, "the last timed run had no general-path distro");
  CK(cudaEventSynchronize(c->ev_end));
  if (task_pass_ms) CK(cudaEventElapsedTime(task_pass_ms, c->ev_gt0, c->ev_gt1));
  if (sort_ms) CK(cudaEventElapsedTime(sort_ms, c->ev_sort0, c->ev_sort1));
  return EVG_OK;
}

int evg_kernel_timing_ms(evg_ctx* c, float* out_ms, int32_t n) {
  ENTER(c, "evg_kernel_timing_ms");
  if (!out_ms || n < 0) return fail(EVG_ERR_INVALID, "%s: bad argument", who);
  if (n > evg_ctx::kRing || n > c->runs) return fail(EVG_ERR_STATE, "only %lld timed runs recorded (ring of %d)", (long long)c->runs, evg_ctx::kRing);
  for (int32_t k = 0; k < n; k++) {
    const int slot = int((c->runs - n + k) % evg_ctx::kRing);
    CK(cudaEventSynchronize(c->ring1[slot]));
    CK(cudaEventElapsedTime(out_ms + k, c->ring0[slot], c->ring1[slot]));
  }
  return EVG_OK;
}

int evg_plan_batch(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_table* distros, int64_t now_ns, uint32_t opts,
                   evg_plan_out* out) {
  ENTER(c, "evg_plan_batch");
  int rc = upload(c, who, tasks, distros, nullptr, nullptr, nullptr, Tick::kFixed);
  if (rc != EVG_OK) return rc;
  rc = evg_run_resident(c, now_ns, opts);
  if (rc != EVG_OK) return rc;
  return evg_download(c, out, nullptr);
}

// The one-shot call as a three-stage pipeline over chunks of whole distros: H2D of chunk k+1, kernels of chunk k
// and D2H of chunk k-1 overlap on three streams, so the tick costs about max(H2D, D2H) instead of their sum.
// Used for ticks of at least 2^21 tasks when no breakdown is requested; a chunk's general-path distros run through the
// general path restricted to their tiles.
static int plan_and_alloc_pipelined(evg_ctx* c, const evg_task_soa* t, const evg_distro_table* dt, const evg_host_soa* hosts,
                                    const int64_t* host_off, const evg_alloc_cfg* acfg, int64_t now, evg_plan_out* po,
                                    evg_alloc_out* ao) {
  const int64_t T = c->T, E = c->E;
  const int32_t D = c->Dn;
  if (!c->s_h2d) {
    CK(cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
    for (int k = 0; k < evg_ctx::kMaxChunks; k++) {
      CK(cudaEventCreateWithFlags(&c->ev_h[k], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&c->ev_c[k], cudaEventDisableTiming));
    }
  }
  cudaStream_t s = c->stream;
  DTasks dtk = dtasks(c);
  DDistros dd = ddistros(c);
  DWork w = dwork(c);
  if (c->ext_result && c->ext_capacity < D) return fail(EVG_ERR_INVALID, "bound result buffer too small");
  CK(c->b_gs.ensure(sizeof(GroupScratch) * size_t(c->G + 1)));
  c->launches = 0;
  c->timed = false;
  c->bd_valid = false;
  CK(cudaMemsetAsync(c->b_puntcnt.p, 0, sizeof(int32_t) * (evg_ctx::kMaxChunks + 2), s));
  // chunk boundaries: whole distros, about equal task counts
  const int n_chunks = int(std::min<int64_t>(evg_ctx::kMaxChunks, std::max<int64_t>(1, T / (1 << 20))));
  std::vector<int32_t> cut(size_t(n_chunks) + 1, D);
  cut[0] = 0;
  {
    int32_t d = 0;
    for (int k = 1; k < n_chunks; k++) {
      const int64_t want = T * k / n_chunks;
      while (d < D && c->h_taskoff[d] < want) d++;
      cut[k] = d;
    }
  }
  auto sub = [](const std::vector<int32_t>& v, int32_t d0, int32_t d1, int32_t* first) {
    auto a = std::lower_bound(v.begin(), v.end(), d0), b = std::lower_bound(v.begin(), v.end(), d1);
    *first = int32_t(a - v.begin());
    return int32_t(b - a);
  };
#define H2D(buf, ptr, off, count, type)                                                                  \
  if ((count) > 0) CK(cudaMemcpyAsync((buf).as<type>() + (off), (ptr) + (off), sizeof(type) * size_t(count), cudaMemcpyHostToDevice, c->s_h2d))
#define D2H(dst, src, off, count, type)                                                                  \
  if ((dst) && (count) > 0) CK(cudaMemcpyAsync((dst) + (off), (src) + (off), sizeof(type) * size_t(count), cudaMemcpyDeviceToHost, c->s_d2h))
  int rc;
  for (int k = 0; k < n_chunks; k++) {
    const int32_t d0 = cut[k], d1 = cut[k + 1];
    if (d1 <= d0) continue;
    const int64_t t0 = c->h_taskoff[d0], n = c->h_taskoff[d1] - t0;
    const int64_t g0 = c->h_groupoff[d0], ng = c->h_groupoff[d1] - g0;
    if ((rc = c->tasks.copy_rows(t, t0, n, c->s_h2d)) != EVG_OK) return rc;
    if (E > 0) {
      const int64_t e0 = t->dep_off[t0], ne = t->dep_off[t0 + n] - e0;
      H2D(c->b_depoff, t->dep_off, t0, n + 1, int64_t);
      H2D(c->b_depidx, t->dep_idx, e0, ne, int32_t);
    }
    CK(cudaEventRecord(c->ev_h[k], c->s_h2d));
    CK(cudaStreamWaitEvent(s, c->ev_h[k], 0));
    launch(c, s, k_validate, grid_for(n, 256), 256, 0, dtk, dd, w, t0, t0 + n);
    // the chunk's distros of each class; what k_plan_cta hands back is replanned by k_plan_smem right behind it, and the
    // general path runs restricted to the chunk's tiles
    int32_t* pl = c->b_punt.as<int32_t>() + d0;  // a chunk hands back at most its own d1 - d0 distros
    int32_t* pc = c->b_puntcnt.as<int32_t>() + 1 + k;
    int32_t n_cta = 0;
    for (int r : {kCtaC, kCtaB, kCtaA, kPunted, kGeneral, kSmemC, kSmemB, kSmemA, kWarp}) {
      int32_t first = 0, cnt = n_cta;
      if (r != kPunted) cnt = sub(c->routes[r].h, d0, d1, &first);
      if (is_cta(r)) n_cta += cnt;
      if ((rc = plan_route(c, r, Mode::kPipelined, s, dtk, dd, w, now, first, cnt, pl, pc)) != EVG_OK) return rc;
    }
    if ((rc = run_alloc_range(c, now, d0, d1)) != EVG_OK) return rc;
    CK(cudaEventRecord(c->ev_c[k], s));
    CK(cudaStreamWaitEvent(c->s_d2h, c->ev_c[k], 0));
    if (po) {
      D2H(po->order, c->b_order.as<int32_t>(), t0, n, int32_t);
      D2H(po->total_value, c->b_tv.as<int64_t>(), t0, n, int64_t);
      D2H(po->info, c->b_qinfo.as<evg_queue_info>(), d0, d1 - d0, evg_queue_info);
      D2H(po->group_info, c->b_ginfo.as<evg_group_info>(), g0, ng, evg_group_info);
    }
    if (ao) {
      D2H(ao->result, c->result_ptr(), d0, d1 - d0, evg_alloc_result);
      D2H(ao->status, c->b_status.as<int32_t>(), d0, d1 - d0, int32_t);
    }
  }
#undef H2D
#undef D2H
  CK(cudaGetLastError());
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(c->s_d2h));
  CK(cudaStreamSynchronize(s));
  if (bad) { drop_tick(c); return fail(EVG_ERR_INVALID, "a group_id / version_id / dep_idx is out of range for its distro"); }
  return EVG_OK;
}

int evg_plan_and_alloc_batch(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_table* distros,
                             const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg, int64_t now_ns,
                             uint32_t opts, evg_plan_out* plan_out, evg_alloc_out* alloc_out) {
  ENTER(c, "evg_plan_and_alloc_batch");
  if (!hosts || (!acfg && distros && distros->n_distros > 0)) return fail(EVG_ERR_INVALID, "evg_plan_and_alloc_batch needs hosts and allocator config");
  if (!(opts & EVG_OPT_BREAKDOWN) && tasks && distros && tasks->n_tasks >= (int64_t(1) << 21)) {
    // large tick: stage the small tables, then pipeline the columns chunk by chunk
    const int rc0 = upload(c, who, tasks, distros, hosts, host_off, acfg, Tick::kFixed, Cols::kChunked);
    if (rc0 != EVG_OK) return rc0;
    const int rc1 = plan_and_alloc_pipelined(c, tasks, distros, hosts, host_off, acfg, now_ns, plan_out, alloc_out);
    c->tick.allocated = rc1 == EVG_OK;
    return rc1;
  }
  int rc = upload(c, who, tasks, distros, hosts, host_off, acfg, Tick::kFixed);
  if (rc != EVG_OK) return rc;
  rc = evg_run_resident(c, now_ns, opts);
  if (rc != EVG_OK) return rc;
  return evg_download(c, plan_out, alloc_out);
}

int evg_alloc_batch(evg_ctx* c, const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* cfg,
                    const evg_queue_info* info, evg_group_info* groups, const int64_t* group_off, int32_t n_distros,
                    int64_t now_ns, evg_alloc_out* out) {
  ENTER(c, "evg_alloc_batch");
  if (n_distros < 0 || (n_distros > 0 && (!info || !group_off || !out))) return fail(EVG_ERR_INVALID, "evg_alloc_batch: null argument");
  int rc = n_distros > 0 ? check_offsets(group_off, n_distros, -1, who, "group_off") : EVG_OK;
  if (rc != EVG_OK) return rc;
  const int64_t G = n_distros > 0 ? group_off[n_distros] : 0;
  if (G > 0 && !groups) return fail(EVG_ERR_INVALID, "evg_alloc_batch: groups is null");
  drop_tick(c);  // before upload_hosts, which must not list distros from the tick's tables
  rc = upload_hosts(c, who, hosts, host_off, cfg, n_distros);
  if (rc != EVG_OK) return rc;
  cudaStream_t s = c->stream;
  CK(c->b_groupoff.ensure(sizeof(int64_t) * size_t(n_distros + 1)));
  CK(c->b_qinfo.ensure(sizeof(evg_queue_info) * size_t(n_distros + 1)));
  CK(c->b_ginfo.ensure(sizeof(evg_group_info) * size_t(G + 1)));
  if (n_distros > 0) {
    CK(cudaMemcpyAsync(c->b_groupoff.p, group_off, sizeof(int64_t) * size_t(n_distros + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(c->b_qinfo.p, info, sizeof(evg_queue_info) * size_t(n_distros), cudaMemcpyHostToDevice, s));
  }
  if (G > 0) CK(cudaMemcpyAsync(c->b_ginfo.p, groups, sizeof(evg_group_info) * size_t(G), cudaMemcpyHostToDevice, s));
  c->Dn = n_distros;
  c->G = G;
  c->max_groups = 0;
  for (int32_t d = 0; d < n_distros; d++) c->max_groups = std::max(c->max_groups, group_off[d + 1] - group_off[d]);
  c->launches = 0;
  rc = run_alloc(c, now_ns);
  if (rc != EVG_OK) return rc;
  if (out->result && n_distros) CK(cudaMemcpyAsync(out->result, c->result_ptr(), sizeof(evg_alloc_result) * size_t(n_distros), cudaMemcpyDeviceToHost, s));
  if (out->status && n_distros) CK(cudaMemcpyAsync(out->status, c->b_status.p, sizeof(int32_t) * size_t(n_distros), cudaMemcpyDeviceToHost, s));
  if (G > 0) CK(cudaMemcpyAsync(groups, c->b_ginfo.p, sizeof(evg_group_info) * size_t(G), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

// The device view of the dependency table deps_to_device staged from `in`.
static DDeps ddeps(const evg_ctx* c, const evg_deps_in* in) {
  const auto& x = c->deps;
  DDeps d;
  d.n_tasks = in->n_tasks; d.n_deps = in->n_deps; d.n_ext = in->n_ext;
  d.dep_off = x.off.as<int64_t>(); d.dep_kind = x.kind.as<uint8_t>(); d.dep_ref = x.ref.as<int32_t>(); d.dep_want = x.want.as<uint8_t>();
  d.task_state = x.state.as<uint8_t>(); d.task_pre = x.pre.as<uint8_t>(); d.ext_state = x.ext.as<uint8_t>();
  return d;
}

// Stage an evg_deps_in table and run k_deps_met into deps.met (left on the device); `both` adds the no-short-circuit bit.
// The host checks the ends of dep_off; its rows, n_tasks of them, are checked by k_deps_met (kErrDepOff).
static int deps_to_device(evg_ctx* c, const char* who, const evg_deps_in* in, int both, const int64_t* dep_finished = nullptr,
                          int64_t now = 0, bool want_stamp = false) {
  const int64_t T = in->n_tasks, E = in->n_deps, X = in->n_ext;
  if (T < 0 || E < 0 || X < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (T == 0) return EVG_OK;
  if (!in->dep_off || !in->task_state || !in->task_pre) return fail(EVG_ERR_INVALID, "null task arrays");
  if (E > 0 && (!in->dep_kind || !in->dep_ref || !in->dep_want)) return fail(EVG_ERR_INVALID, "null dependency arrays");
  if (X > 0 && !in->ext_state) return fail(EVG_ERR_INVALID, "null ext_state");
  if (in->dep_off[0] != 0 || in->dep_off[T] != E)
    return fail(EVG_ERR_INVALID, "%s: deps->dep_off runs from %lld to %lld, not from 0 to n_deps", who, (long long)in->dep_off[0], (long long)in->dep_off[T]);
  cudaStream_t s = c->stream;
  auto& x = c->deps;
  UP(s, x.off, in->dep_off, T + 1, int64_t);
  UP(s, x.kind, in->dep_kind, E, uint8_t);
  UP(s, x.ref, in->dep_ref, E, int32_t);
  UP(s, x.want, in->dep_want, E, uint8_t);
  UP(s, x.state, in->task_state, T, uint8_t);
  UP(s, x.pre, in->task_pre, T, uint8_t);
  UP(s, x.ext, in->ext_state, X, uint8_t);
  CK(x.met.ensure(size_t(T)));
  int64_t* stamp = nullptr;
  const int64_t* fin = nullptr;
  if (want_stamp) {
    CK(x.stamp.ensure(sizeof(int64_t) * size_t(T)));
    stamp = x.stamp.as<int64_t>();
    if (dep_finished && E > 0) {
      UP(s, x.fin, dep_finished, E, int64_t);
      fin = x.fin.as<int64_t>();
    }
  }
  launch(c, s, k_deps_met, grid_for(T, 256), 256, 0, ddeps(c, in), x.met.as<uint8_t>(), c->b_err.as<int>(), both, fin, now, stamp);
  CK(cudaGetLastError());
  return EVG_OK;
}

// The device-side checks of the dependency and finder passes (c->b_err, bits as at kErrDepOff) as one message.
static int deps_bad(const char* who, int bad) {
  if (bad & kErrDepOff) return fail(EVG_ERR_INVALID, "%s: deps->dep_off decreases or leaves [0, n_deps] at some row", who);
  if (bad & 2) return fail(EVG_ERR_INVALID, "%s: a status id of the evg_pipeline_in is outside [0, n_status)", who);
  return fail(EVG_ERR_INVALID, "%s: a dep_ref or project row is out of range", who);
}

int evg_deps_met_batch(evg_ctx* c, const evg_deps_in* in, uint8_t* met) {
  ENTER(c, "evg_deps_met_batch");
  if (!in || (in->n_tasks > 0 && !met)) return fail(EVG_ERR_INVALID, "evg_deps_met_batch: null argument");
  if (in->n_tasks == 0) return EVG_OK;
  cudaStream_t s = c->stream;
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  c->launches = 0;
  c->tick.deps = false;  // deps_to_device overwrites the resident tick's verdicts and stamps
  int rc = deps_to_device(c, who, in, 0);
  if (rc != EVG_OK) return rc;
  int bad = 0;
  CK(cudaMemcpyAsync(met, c->deps.met.p, size_t(in->n_tasks), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) return deps_bad(who, bad);
  return EVG_OK;
}

int evg_upload_with_deps(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_table* distros, const evg_host_soa* hosts,
                         const int64_t* host_off, const evg_alloc_cfg* acfg, const evg_deps_in* deps, const int64_t* dep_finished_ns,
                         int64_t now_ns) {
  ENTER(c, "evg_upload_with_deps");
  if (!tasks || !deps) return fail(EVG_ERR_INVALID, "evg_upload_with_deps: null argument");
  if (deps->n_tasks != tasks->n_tasks) return fail(EVG_ERR_INVALID, "deps covers %lld tasks, the task table %lld", (long long)deps->n_tasks, (long long)tasks->n_tasks);
  int rc = upload(c, who, tasks, distros, hosts, host_off, acfg, Tick::kOwn);
  if (rc != EVG_OK) return rc;
  const int64_t T = tasks->n_tasks;
  if (T == 0) return EVG_OK;
  cudaStream_t s = c->stream;
  rc = deps_to_device(c, who, deps, 0, dep_finished_ns, now_ns, /*want_stamp=*/true);
  if (rc != EVG_OK) { drop_tick(c); return rc; }
  launch(c, s, k_apply_deps, grid_for(T, 256), 256, 0, T, c->deps.met.as<uint8_t>(), c->deps.stamp.as<int64_t>(), c->tasks.flags.as<uint32_t>(),
         c->tasks.wb.as<int64_t>());
  int bad = 0;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) { drop_tick(c); return deps_bad(who, bad); }
  c->tick.deps = true;
  return EVG_OK;
}

int evg_download_deps(evg_ctx* c, uint8_t* met, int64_t* met_time_ns) {
  ENTER(c, "evg_download_deps");
  if (const int rc = need_tick(c, who, Need::kTick); rc != EVG_OK) return rc;
  if (c->T == 0) return EVG_OK;
  if (const int rc = need_tick(c, who, Need::kVerdicts); rc != EVG_OK) return rc;
  if (met) CK(cudaMemcpyAsync(met, c->deps.met.p, size_t(c->T), cudaMemcpyDeviceToHost, c->stream));
  if (met_time_ns) CK(cudaMemcpyAsync(met_time_ns, c->deps.stamp.p, sizeof(int64_t) * size_t(c->T), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return EVG_OK;
}

int evg_expected_durations_batch(evg_ctx* c, const evg_duration_rows* in, evg_duration_stat* out) {
  ENTER(c, "evg_expected_durations_batch");
  if (!in) return fail(EVG_ERR_INVALID, "evg_expected_durations_batch: null argument");
  const int64_t R = in->n_rows;
  const int32_t K = in->n_keys;
  if (R < 0 || K < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (K == 0) return R == 0 ? EVG_OK : fail(EVG_ERR_INVALID, "rows without keys");
  if (!out) return fail(EVG_ERR_INVALID, "null output");
  if (R > 0 && (!in->key || !in->time_taken_ns || !in->start_ns || !in->finish_ns || !in->flags)) return fail(EVG_ERR_INVALID, "null row column");
  cudaStream_t s = c->stream;
  c->launches = 0;
  drop_tick(c);
  UP(s, c->b_rn0, in->key, R, int32_t);
  UP(s, c->b_rn1, in->time_taken_ns, R, int64_t);
  UP(s, c->b_rn2, in->start_ns, R, int64_t);
  UP(s, c->b_rn3, in->finish_ns, R, int64_t);
  UP(s, c->b_rn4, in->flags, R, uint8_t);
  CK(c->b_rn5.ensure(sizeof(unsigned long long) * 4 * size_t(K)));
  CK(c->b_rn6.ensure(sizeof(evg_duration_stat) * size_t(K)));
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  CK(cudaMemsetAsync(c->b_rn5.p, 0, sizeof(unsigned long long) * 4 * size_t(K), s));
  DDur x;
  x.n_rows = R; x.n_keys = K; x.key = c->b_rn0.as<int32_t>(); x.taken = c->b_rn1.as<int64_t>(); x.start = c->b_rn2.as<int64_t>();
  x.finish = c->b_rn3.as<int64_t>(); x.flags = c->b_rn4.as<uint8_t>(); x.w0 = in->window_start_ns; x.w1 = in->window_end_ns;
  x.cnt = c->b_rn5.as<unsigned long long>(); x.sum = x.cnt + K; x.sq_lo = x.sum + K; x.sq_hi = x.sq_lo + K;
  launch(c, s, k_dur_sum, grid_for(R, 256), 256, 0, x, c->b_err.as<int>());
  launch(c, s, k_dur_dev, grid_for(R, 256), 256, 0, x);
  launch(c, s, k_dur_final, grid_for(K, 256), 256, 0, x, c->b_rn6.as<evg_duration_stat>());
  CK(cudaGetLastError());
  int bad = 0;
  CK(cudaMemcpyAsync(out, c->b_rn6.p, sizeof(evg_duration_stat) * size_t(K), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) return fail(EVG_ERR_INVALID, "a key is out of range");
  return EVG_OK;
}

// The host's checks of one evg_duration_cache against a resident table of n rows.
static int check_duration_cache(const evg_duration_cache* dc, int64_t n, const char* what) {
  if (dc->n_rows < 0) return fail(EVG_ERR_INVALID, "evg_resolve_durations: negative %s n_rows", what);
  if (!dc->rows && dc->n_rows != n)
    return fail(EVG_ERR_INVALID, "evg_resolve_durations: %s rows == NULL but n_rows %lld != %lld resident rows", what,
                (long long)dc->n_rows, (long long)n);
  if (dc->n_rows > 0 && (!dc->value_ns || !dc->std_ns || !dc->ttl_ns || !dc->collected_ns || !dc->expected_ns ||
                         !dc->expected_std_ns || !dc->key))
    return fail(EVG_ERR_INVALID, "evg_resolve_durations: null %s column", what);
  if (dc->rows)
    for (int64_t i = 0; i < dc->n_rows; i++) {
      const int64_t r = dc->rows[i];
      if (r < 0 || r >= n || (i > 0 && r <= dc->rows[i - 1]))
        return fail(EVG_ERR_INVALID, "evg_resolve_durations: %s rows[%lld] = %lld is out of range or not strictly ascending", what,
                    (long long)i, (long long)r);
    }
  return EVG_OK;
}

int evg_resolve_durations(evg_ctx* c, const evg_duration_in* in, int64_t now_ns) {
  ENTER(c, "evg_resolve_durations");
  if (!in) return fail(EVG_ERR_INVALID, "evg_resolve_durations: null argument");
  int rc;
  if ((rc = need_tick(c, who, Need::kEditable)) != EVG_OK) return rc;
  if (in->hosts && (rc = need_tick(c, who, Need::kHosts)) != EVG_OK) return rc;
  const evg_duration_rows* h = in->history;
  const int64_t R = h ? h->n_rows : 0;
  const int32_t K = h ? h->n_keys : 0, P = in->n_pairs;
  if (R < 0 || K < 0 || P < 0) return fail(EVG_ERR_INVALID, "evg_resolve_durations: negative sizes");
  if (R > 0 && (!h->key || !h->time_taken_ns || !h->start_ns || !h->finish_ns || !h->flags))
    return fail(EVG_ERR_INVALID, "evg_resolve_durations: null history column");
  if (P > 0 && !in->pair_key_off) return fail(EVG_ERR_INVALID, "evg_resolve_durations: null pair_key_off");
  if (in->pair_key_off && (rc = check_offsets(in->pair_key_off, P, K, who, "pair_key_off")) != EVG_OK) return rc;
  if (in->tasks && (rc = check_duration_cache(in->tasks, c->T, "tasks")) != EVG_OK) return rc;
  if (in->hosts && (rc = check_duration_cache(in->hosts, c->H, "hosts")) != EVG_OK) return rc;
  cudaStream_t s = c->stream;
  auto& d = c->dur;
  c->tick.durations = false;  // the staging below is overwritten whatever the outcome
  const int64_t Nt = in->tasks ? in->tasks->n_rows : 0, Nh = in->hosts ? in->hosts->n_rows : 0, N = Nt + Nh;
  // history -> per-key statistics, on the call's own buffers (evg_expected_durations_batch's scratch is not touched)
  UP(s, d.key, h ? h->key : nullptr, R, int32_t);
  UP(s, d.taken, h ? h->time_taken_ns : nullptr, R, int64_t);
  UP(s, d.start, h ? h->start_ns : nullptr, R, int64_t);
  UP(s, d.finish, h ? h->finish_ns : nullptr, R, int64_t);
  UP(s, d.flags, h ? h->flags : nullptr, R, uint8_t);
  CK(d.acc.ensure(sizeof(unsigned long long) * 4 * size_t(K)));
  CK(d.stat.ensure(sizeof(evg_duration_stat) * size_t(K)));
  UP(s, d.pair_off, in->pair_key_off, P > 0 ? P + 1 : 0, int64_t);
  CK(d.single.ensure(sizeof(int32_t) * size_t(P)));
  CK(d.err.ensure(sizeof(int)));
  CK(cudaMemsetAsync(d.err.p, 0, sizeof(int), s));
  if (K > 0) CK(cudaMemsetAsync(d.acc.p, 0, sizeof(unsigned long long) * 4 * size_t(K), s));
  // the listed rows: six int64 columns and the key, tasks then hosts; the results: five int64 columns and the source
  CK(d.rows.ensure(sizeof(int64_t) * size_t(N)));
  CK(d.in.ensure((sizeof(int64_t) * 6 + sizeof(int32_t)) * size_t(N)));
  CK(d.out.ensure(sizeof(int64_t) * 5 * size_t(N)));
  CK(d.src.ensure(size_t(N)));
  DDurRows X;
  int64_t* col = d.in.as<int64_t>();
  X.n_t = Nt; X.n_h = Nh;
  X.value = col; X.pstd = col + N; X.ttl = col + 2 * N; X.coll = col + 3 * N; X.exp = col + 4 * N; X.exp_std = col + 5 * N;
  X.key = reinterpret_cast<const int32_t*>(col + 6 * N);
  int64_t* o = d.out.as<int64_t>();
  X.o_avg = o; X.o_std = o + N; X.o_value = o + 2 * N; X.o_pstd = o + 3 * N; X.o_coll = o + 4 * N;
  X.o_src = d.src.as<uint8_t>();
  X.trows = (in->tasks && in->tasks->rows) ? d.rows.as<int64_t>() : nullptr;
  X.hrows = (in->hosts && in->hosts->rows) ? d.rows.as<int64_t>() + Nt : nullptr;
  const evg_duration_cache* seg[2] = {in->tasks, in->hosts};
  const int64_t base[2] = {0, Nt};
  for (int k = 0; k < 2; k++) {
    const evg_duration_cache* dc = seg[k];
    if (!dc || dc->n_rows == 0) continue;
    const size_t n = size_t(dc->n_rows), b = size_t(base[k]);
    if (dc->rows) CK(cudaMemcpyAsync(d.rows.as<int64_t>() + b, dc->rows, 8 * n, cudaMemcpyHostToDevice, s));
    const int64_t* src[6] = {dc->value_ns, dc->std_ns, dc->ttl_ns, dc->collected_ns, dc->expected_ns, dc->expected_std_ns};
    for (int j = 0; j < 6; j++) CK(cudaMemcpyAsync(col + size_t(j) * size_t(N) + b, src[j], 8 * n, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(const_cast<int32_t*>(X.key) + b, dc->key, 4 * n, cudaMemcpyHostToDevice, s));
  }
  DDur x;
  x.n_rows = R; x.n_keys = K; x.key = d.key.as<int32_t>(); x.taken = d.taken.as<int64_t>(); x.start = d.start.as<int64_t>();
  x.finish = d.finish.as<int64_t>(); x.flags = d.flags.as<uint8_t>();
  x.w0 = h ? h->window_start_ns : 0; x.w1 = h ? h->window_end_ns : 0;
  x.cnt = d.acc.as<unsigned long long>(); x.sum = x.cnt + K; x.sq_lo = x.sum + K; x.sq_hi = x.sq_lo + K;
  launch(c, s, k_dur_sum, grid_for(R, 256), 256, 0, x, d.err.as<int>());
  launch(c, s, k_dur_dev, grid_for(R, 256), 256, 0, x);
  launch(c, s, k_dur_final, grid_for(K, 256), 256, 0, x, d.stat.as<evg_duration_stat>());
  launch(c, s, k_dur_pair, grid_for(P, 256), 256, 0, P, d.pair_off.as<int64_t>(), x.cnt, d.single.as<int32_t>());
  launch(c, s, k_dur_resolve, grid_for(N, 256), 256, 0, X, K, P, d.stat.as<evg_duration_stat>(), d.single.as<int32_t>(), now_ns, d.err.as<int>());
  launch(c, s, k_dur_commit, grid_for(N, 256), 256, 0, X, d.err.as<int>(), c->tasks.exp.as<int64_t>(), c->b_hexp.as<int64_t>(),
         c->b_hstd.as<int64_t>());
  CK(cudaGetLastError());
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d.err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));  // the caller's arrays are free again
  if (bad & 1) return fail(EVG_ERR_INVALID, "evg_resolve_durations: a history key is outside [0, n_keys)");
  if (bad) return fail(EVG_ERR_INVALID, "evg_resolve_durations: a row's key or pair is out of range");
  d.n_t = Nt; d.n_h = Nh;
  c->tick.durations = true;
  return EVG_OK;
}

int evg_download_durations(evg_ctx* c, evg_duration_out* tasks, evg_duration_out* hosts) {
  ENTER(c, "evg_download_durations");
  if (const int rc = need_tick(c, who, Need::kDurations); rc != EVG_OK) return rc;
  cudaStream_t s = c->stream;
  auto& d = c->dur;
  const int64_t N = d.n_t + d.n_h;
  const int64_t* o = d.out.as<int64_t>();
  evg_duration_out* seg[2] = {tasks, hosts};
  const int64_t base[2] = {0, d.n_t}, cnt[2] = {d.n_t, d.n_h};
  for (int k = 0; k < 2; k++) {
    evg_duration_out* q = seg[k];
    if (!q || cnt[k] == 0) continue;
    const size_t n = size_t(cnt[k]), b = size_t(base[k]);
    int64_t* dst[5] = {q->avg_ns, q->std_ns, q->value_ns, q->pred_std_ns, q->collected_ns};
    for (int j = 0; j < 5; j++)
      if (dst[j]) CK(cudaMemcpyAsync(dst[j], o + size_t(j) * size_t(N) + b, 8 * n, cudaMemcpyDeviceToHost, s));
    if (q->source) CK(cudaMemcpyAsync(q->source, d.src.as<uint8_t>() + b, n, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

// The finder tables of evg_find_runnable_batch and evg_plan_from_finder: checked, staged into pf.*, and k_runnable's view
// of them (the caller sets r->met).  `any_deps`: some distro's finder reads the dependency verdicts.  `pipe`: the pipeline
// codes are allowed, `any_pipe` / `pipe_deps` report whether some distro uses one / EVG_FINDER_PIPELINE.  n_distros > 0.
static int stage_finder(evg_ctx* c, const char* who, const evg_runnable_in* in, DRunnable* r, bool* any_deps,
                        const evg_pipeline_in* pipe = nullptr, bool* any_pipe = nullptr, bool* pipe_deps = nullptr) {
  const int64_t T = in->n_tasks;
  const int32_t D = in->n_distros, P = in->n_projects;
  if (!in->task_off || !in->valid_off || !in->finder) return fail(EVG_ERR_INVALID, "null distro arrays");
  if (T > 0 && (!in->sched || !in->project)) return fail(EVG_ERR_INVALID, "null task column");
  if (P > 0 && !in->project_flags) return fail(EVG_ERR_INVALID, "null project_flags");
  int rc = check_offsets(in->task_off, D, T, who, "task_off");
  if (rc == EVG_OK) rc = check_offsets(in->valid_off, D, -1, who, "valid_off");
  if (rc != EVG_OK) return rc;
  *any_deps = false;
  const uint8_t max_code = pipe ? EVG_FINDER_PIPELINE_NO_DEPS : EVG_FINDER_ALTERNATE;
  for (int32_t d = 0; d < D; d++) {
    if (in->finder[d] > max_code)
      return fail(EVG_ERR_INVALID, in->finder[d] <= EVG_FINDER_PIPELINE_NO_DEPS ? "distro %d: the pipeline finder (%d) needs an evg_pipeline_in"
                                                                                 : "distro %d: unknown finder %d", d, int(in->finder[d]));
    *any_deps = *any_deps || (in->finder[d] != EVG_FINDER_NO_DEPS && in->finder[d] != EVG_FINDER_PIPELINE_NO_DEPS);
    if (any_pipe) *any_pipe = *any_pipe || in->finder[d] >= EVG_FINDER_PIPELINE;
    if (pipe_deps) *pipe_deps = *pipe_deps || in->finder[d] == EVG_FINDER_PIPELINE;
  }
  const int64_t V = in->valid_off[D];
  if (V > 0 && !in->valid_idx) return fail(EVG_ERR_INVALID, "null valid_idx");
  if (pipe_deps && *pipe_deps && in->n_tasks > 0) {  // what the host can check of the pipeline's dependency tables
    const evg_deps_in* x = in->deps;
    if (!x || x->n_tasks != in->n_tasks) return fail(EVG_ERR_INVALID, "the pipeline finder needs the candidates' dependency table");
    if (pipe->n_status < 3) return fail(EVG_ERR_INVALID, "evg_pipeline_in: n_status %d < 3 (the reserved ids)", int(pipe->n_status));
    if (!pipe->task_status || !pipe->task_unattainable || (x->n_deps > 0 && !pipe->dep_status) ||
        (x->n_ext > 0 && (!pipe->ext_status || !pipe->ext_unattainable)))
      return fail(EVG_ERR_INVALID, "evg_pipeline_in: null status column");
  }
  cudaStream_t s = c->stream;
  auto& pf = c->pf;
  UP(s, pf.task_off, in->task_off, D + 1, int64_t);
  UP(s, pf.sched, in->sched, T, uint8_t);
  UP(s, pf.project, in->project, T, int32_t);
  UP(s, pf.project_flags, in->project_flags, P, uint8_t);
  UP(s, pf.valid_off, in->valid_off, D + 1, int64_t);
  UP(s, pf.valid_idx, in->valid_idx, V, int32_t);
  UP(s, pf.finder, in->finder, D, uint8_t);
  CK(pf.kept.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(pf.count.ensure(sizeof(int64_t) * size_t(D + 1)));
  r->n_tasks = T; r->n_distros = D; r->n_projects = P;
  r->task_off = pf.task_off.as<int64_t>(); r->sched = pf.sched.as<uint8_t>(); r->project = pf.project.as<int32_t>();
  r->project_flags = pf.project_flags.as<uint8_t>(); r->valid_off = pf.valid_off.as<int64_t>(); r->valid_idx = pf.valid_idx.as<int32_t>();
  r->finder = pf.finder.as<uint8_t>(); r->met = nullptr;
  if (pipe && P > 0) {
    if (!pipe->project_raw) return fail(EVG_ERR_INVALID, "null project_raw");
    UP(s, c->pl.project_raw, pipe->project_raw, P, uint8_t);
  }
  return EVG_OK;
}

// The status columns of an evg_pipeline_in over the staged dependency table `x` (deps_to_device ran) and k_pl_deps,
// which adds bit 2 to deps.met.  stage_finder checked the sizes; the ids are checked on the device.
static int pipeline_deps(evg_ctx* c, const evg_deps_in* x, const evg_pipeline_in* pipe) {
  const int64_t T = x->n_tasks, E = x->n_deps, X = x->n_ext;
  cudaStream_t s = c->stream;
  auto& p = c->pl;
  UP(s, p.dep_status, pipe->dep_status, E, int32_t);
  UP(s, p.task_status, pipe->task_status, T, int32_t);
  UP(s, p.ext_status, pipe->ext_status, X, int32_t);
  UP(s, p.task_unatt, pipe->task_unattainable, T, uint8_t);
  UP(s, p.ext_unatt, pipe->ext_unattainable, X, uint8_t);
  DPipe dp;
  dp.n_status = pipe->n_status; dp.dep_status = p.dep_status.as<int32_t>(); dp.task_status = p.task_status.as<int32_t>();
  dp.ext_status = p.ext_status.as<int32_t>(); dp.task_unatt = p.task_unatt.as<uint8_t>(); dp.ext_unatt = p.ext_unatt.as<uint8_t>();
  launch(c, s, k_pl_deps, grid_for(T, 256), 256, 0, ddeps(c, x), dp, c->deps.met.as<uint8_t>(), c->b_err.as<int>());
  CK(cudaGetLastError());
  return EVG_OK;
}

// evg_find_runnable_batch and evg_find_runnable_ex (`name`; the former passes no pipe)
static int find_runnable(const char* name, evg_ctx* c, const evg_runnable_in* in, const evg_pipeline_in* pipe, int32_t* runnable, int64_t* count) {
  ENTER(c, name);
  if (!in) return fail(EVG_ERR_INVALID, "%s: null argument", who);
  const int64_t T = in->n_tasks;
  const int32_t D = in->n_distros, P = in->n_projects;
  if (T < 0 || D < 0 || P < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (D == 0) return T == 0 ? EVG_OK : fail(EVG_ERR_INVALID, "tasks without distros");
  if (!count || (T > 0 && !runnable)) return fail(EVG_ERR_INVALID, "null output");
  DRunnable r;
  bool any_deps, any_pipe = false, pipe_deps = false;
  int rc = stage_finder(c, who, in, &r, &any_deps, pipe, &any_pipe, &pipe_deps);
  if (rc != EVG_OK) return rc;
  if (any_deps && T > 0 && (!in->deps || in->deps->n_tasks != T)) return fail(EVG_ERR_INVALID, "a finder checks dependencies but deps is null or of another size");
  cudaStream_t s = c->stream;
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  c->launches = 0;
  drop_tick(c);
  if (any_deps && T > 0) {
    rc = deps_to_device(c, who, in->deps, 1);
    if (rc != EVG_OK) return rc;
    if (pipe_deps) {
      rc = pipeline_deps(c, in->deps, pipe);
      if (rc != EVG_OK) return rc;
    }
    r.met = c->deps.met.as<uint8_t>();
  }
  if (any_pipe)
    launch(c, s, k_runnable_pipe, unsigned(D), 256, 0, r, c->pl.project_raw.as<uint8_t>(), c->pf.kept.as<int32_t>(), c->pf.count.as<int64_t>(),
           c->b_err.as<int>());
  else
    launch(c, s, k_runnable, unsigned(D), 256, 0, r, c->pf.kept.as<int32_t>(), c->pf.count.as<int64_t>(), c->b_err.as<int>());
  CK(cudaGetLastError());
  int bad = 0;
  if (T > 0) CK(cudaMemcpyAsync(runnable, c->pf.kept.p, sizeof(int32_t) * size_t(T), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(count, c->pf.count.p, sizeof(int64_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) return deps_bad(who, bad);
  return EVG_OK;
}
int evg_find_runnable_batch(evg_ctx* c, const evg_runnable_in* in, int32_t* runnable, int64_t* count) {
  return find_runnable("evg_find_runnable_batch", c, in, nullptr, runnable, count);
}
int evg_find_runnable_ex(evg_ctx* c, const evg_runnable_in* in, const evg_pipeline_in* pipe, int32_t* runnable, int64_t* count) {
  return find_runnable("evg_find_runnable_ex", c, in, pipe, runnable, count);
}

// --------------------------------------------------------------------------
// compose_tick: a new resident table built on the device from the kept rows of a source table, in their order, and
// each distro's inserted rows after them -- evg_edit_tasks (source: the resident tick) and evg_plan_from_finder
// (source: the candidates; nothing inserted)
// --------------------------------------------------------------------------
// exclusive scan of int32 counts into int64 offsets (n + 1 entries), three launches
__global__ void __launch_bounds__(1024) k_scan_blocks(const int32_t* __restrict__ in, int64_t n, int64_t* __restrict__ out, int64_t* __restrict__ block_sum) {
  __shared__ int64_t sw[32];
  const int64_t i = int64_t(blockIdx.x) * 1024 + threadIdx.x;
  int64_t total;
  const int64_t ex = block_scan_excl<32>(i < n ? int64_t(in[i]) : int64_t(0), sw, &total);
  if (i < n) out[i] = ex;
  if (threadIdx.x == 0) block_sum[blockIdx.x] = total;
}
__global__ void __launch_bounds__(1024) k_scan_sums(int64_t* __restrict__ block_sum, int64_t nb) {  // one block
  const int64_t total = block_scan_segment(block_sum, nb);
  if (threadIdx.x == 0) block_sum[nb] = total;  // the grand total
}
__global__ void __launch_bounds__(1024) k_scan_add(int64_t* __restrict__ out, int64_t n, const int64_t* __restrict__ block_sum, int64_t nb) {
  const int64_t i = int64_t(blockIdx.x) * 1024 + threadIdx.x;
  if (i < n) out[i] += block_sum[blockIdx.x];
  if (i == 0) out[n] = block_sum[nb];
}
// Where row i of the composed table comes from.  Distro d's composed rows are its survivors in their source order
// (S_d of them), then its inserted rows ins_off[d] .. ins_off[d+1].  The source is the resident table (an edit) or the
// candidates (the finder).
struct EdMap {
  int32_t D;
  const int64_t* new_off;    // D+1: composed task_off
  const int64_t* old_off;    // D+1: source task_off
  const int64_t* ins_off;    // D+1: CSR of the inserted rows over distros
  const int32_t* keep;       // [source T]: 1 = survives
  const int64_t* pos;        // [source T + 1]: exclusive scan of keep (survivors before a source row, all distros)
  const int32_t* src;        // [composed T]: source row of a survivor (unset for inserted rows)
  const int64_t* old_goff;   // D+1: resident group_off
  const int64_t* old_vbase;  // D+1: prefix sum of the resident n_versions
  const int32_t* gremap;     // per resident group slot: new distro-local id, -1 = none; NULL = ids kept
  const int32_t* vremap;     // per resident (distro, version): new id; NULL = ids kept
  int64_t n_add;
  const int64_t* add_task;   // ascending composed row of a survivor that gains an edge
  const int32_t* add_dep;    // its new distro-local dependency
};
__device__ __forceinline__ int64_t ed_survivors(const EdMap& m, int d) {
  return (m.new_off[d + 1] - m.new_off[d]) - (m.ins_off[d + 1] - m.ins_off[d]);
}
// first index in add_task[0, n) that is >= row
__device__ __forceinline__ int64_t ed_lower(const int64_t* __restrict__ a, int64_t n, int64_t row) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < row) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// keep[t] = 0 for the removed rows (ascending rm), 1 otherwise
__global__ void __launch_bounds__(256) k_ed_keep(int64_t n_old, const int64_t* __restrict__ rm, int64_t n_rm, int32_t* __restrict__ keep) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n_old) return;
  const int64_t k = ed_lower(rm, n_rm, t);
  keep[t] = (k < n_rm && rm[k] == t) ? 0 : 1;
}
// src[composed row of survivor t] = t: a distro's survivors keep their order, behind the inserted rows of the distros before it
__global__ void __launch_bounds__(256) k_ed_src(int64_t n_old, EdMap m, int32_t* __restrict__ src) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(m.old_off, m.D, t, n_old);
  if (d < 0 || !m.keep[t]) return;
  src[m.pos[t] + m.ins_off[d]] = int32_t(t);
}
// One thread per composed row: a survivor's row of the source columns (group and version ids remapped), or a staged
// inserted row.  err[0] = 1 when a survivor's task group maps to -1.
__global__ void __launch_bounds__(256) k_ed_gather(int64_t n_new, EdMap m, DTasks O, DTasks I, EdDst o, int* __restrict__ err) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(m.new_off, m.D, i, n_new);
  if (d < 0) return;
  const int64_t k = i - m.new_off[d], S = ed_survivors(m, d);
  if (k < S) {
    const int64_t t = m.src[i];
    int32_t gid = O.gid[t], vid = O.vid[t];
    if (m.gremap && gid >= 0) {
      gid = m.gremap[m.old_goff[d] + gid];
      if (gid < 0) *err = 1;
    }
    if (m.vremap) vid = m.vremap[m.old_vbase[d] + vid];
    o.priority[i] = O.priority[t]; o.numdep[i] = O.numdep[t]; o.tgo[i] = O.tgo[t]; o.gid[i] = gid; o.vid[i] = vid;
    o.flags[i] = O.flags[t]; o.expected[i] = O.expected[t]; o.qbasis[i] = O.qbasis[t]; o.wbasis[i] = O.wbasis[t];
  } else {
    const int64_t j = m.ins_off[d] + (k - S);
    o.priority[i] = I.priority[j]; o.numdep[i] = I.numdep[j]; o.tgo[i] = I.tgo[j]; o.gid[i] = I.gid[j]; o.vid[i] = I.vid[j];
    o.flags[i] = I.flags[j]; o.expected[i] = I.expected[j]; o.qbasis[i] = I.qbasis[j]; o.wbasis[i] = I.wbasis[j];
  }
}
// Edges of composed row i: a survivor's source edges whose dependency survived, re-indexed and in their order, then
// its added edges; an inserted row's own edges.  o_dep_idx == NULL: count them, raising bit 2 of *err for a source
// dep_idx outside its distro (the count pass runs before the source's ids are range-checked); otherwise write them at
// o_dep_off[i].
__device__ __forceinline__ int64_t ed_edges(const EdMap& m, const DTasks& O, const DTasks& I, int64_t i, int d,
                                            const int64_t* __restrict__ o_dep_off, int32_t* __restrict__ o_dep_idx, int* err) {
  const int64_t k = i - m.new_off[d], S = ed_survivors(m, d);
  int64_t w = o_dep_off ? o_dep_off[i] : 0, n = 0;
  if (k < S) {
    const int64_t t = m.src[i], base = m.old_off[d];
    if (O.n_edges > 0) {
      const int64_t first = m.pos[base];
      for (int64_t e = O.dep_off[t]; e < O.dep_off[t + 1]; e++) {
        const int32_t x = O.dep_idx[e];
        if (err && (x < 0 || x >= m.old_off[d + 1] - base)) { atomicOr(err, 2); continue; }
        const int64_t u = base + x;
        if (!m.keep[u]) continue;
        if (o_dep_idx) o_dep_idx[w + n] = int32_t(m.pos[u] - first);
        n++;
      }
    }
    if (m.n_add > 0)
      for (int64_t a = ed_lower(m.add_task, m.n_add, i); a < m.n_add && m.add_task[a] == i; a++) {
        if (o_dep_idx) o_dep_idx[w + n] = m.add_dep[a];
        n++;
      }
  } else if (I.n_edges > 0) {
    const int64_t j = m.ins_off[d] + (k - S);
    for (int64_t e = I.dep_off[j]; e < I.dep_off[j + 1]; e++) {
      if (o_dep_idx) o_dep_idx[w + n] = I.dep_idx[e];
      n++;
    }
  }
  return n;
}
__global__ void __launch_bounds__(256) k_ed_edge_count(int64_t n_new, EdMap m, DTasks O, DTasks I, int32_t* __restrict__ cnt, int* err) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(m.new_off, m.D, i, n_new);
  if (d < 0) return;
  cnt[i] = int32_t(ed_edges(m, O, I, i, d, nullptr, nullptr, err));
}
__global__ void __launch_bounds__(256) k_ed_edge_write(int64_t n_new, EdMap m, DTasks O, DTasks I, const int64_t* __restrict__ o_dep_off,
                                                       int32_t* __restrict__ o_dep_idx) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(m.new_off, m.D, i, n_new);
  if (d < 0) return;
  ed_edges(m, O, I, i, d, o_dep_off, o_dep_idx, nullptr);
}

// keep[candidate] = 1 for every candidate k_runnable kept (keep zeroed before): kept[] holds each distro's kept
// candidates as distro-local indices, its unused slots -1
__global__ void __launch_bounds__(256) k_kept_mask(int64_t n, int32_t D, const int64_t* __restrict__ off, const int32_t* __restrict__ kept,
                                                   int32_t* __restrict__ keep) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, i, n);
  if (d < 0) return;
  const int32_t k = kept[i];
  if (k >= 0) keep[off[d] + k] = 1;
}

// Exclusive scan of n int32 counts into out[0 .. n] (int64; out[n] = the total) on c->stream, the per-block sums in
// c->b_scansum.
static cudaError_t scan_counts(evg_ctx* c, const int32_t* in, int64_t n, int64_t* out) {
  const int64_t nb = (n + 1023) / 1024;
  const cudaError_t e = c->b_scansum.ensure(sizeof(int64_t) * size_t(nb + 1));
  if (e != cudaSuccess) return e;
  int64_t* sum = c->b_scansum.as<int64_t>();
  launch(c, c->stream, k_scan_blocks, unsigned(nb), 1024, 0, in, n, out, sum);
  launch(c, c->stream, k_scan_sums, 1, 1024, 0, sum, nb);
  launch(c, c->stream, k_scan_add, unsigned(nb), 1024, 0, out, n, sum, nb);
  return cudaSuccess;
}

// The composed table in the shadow set (Tn rows) and in ed.dep_off / ed.dep_idx (En edges; edge_off: dep_off at the
// distro boundaries) becomes the resident one, routed, sized and range-checked like an upload.  An error leaves no tick.
static int install_composed(evg_ctx* c, const char* who, int64_t Tn, int64_t En, const int64_t* edge_off, const evg_distro_table* distros) {
  auto& e = c->ed;
  drop_tick(c);
  c->tasks.swap(e.out);
  if (En > 0) { c->b_depoff.swap(e.dep_off); c->b_depidx.swap(e.dep_idx); }
  evg_task_soa ts = c->tasks.soa(Tn);
  ts.n_edges = En;
  if (En > 0) { ts.dep_off = c->b_depoff.as<int64_t>(); ts.dep_idx = c->b_depidx.as<int32_t>(); }
  return upload_tasks(c, who, &ts, distros, Cols::kResident, En > 0 ? edge_off : nullptr);
}

// The rows of O that ed.keep marks (O.n entries, staged by the caller) survive in their order, distro d's inserted rows
// m.ins_off[d] .. m.ins_off[d+1] of In follow them, and the composed table over `distros` becomes the resident tick.  The
// caller fills m but for new_off, keep, pos and src.  A device-side error leaves no resident tick.
static int compose_tick(evg_ctx* c, const char* who, EdMap m, const DTasks& O, const DTasks& In, const evg_distro_table* distros) {
  cudaStream_t s = c->stream;
  auto& e = c->ed;
  const int32_t D = m.D;
  const int64_t T0 = O.n, Tn = D > 0 ? distros->task_off[D] : 0;
  UP(s, e.new_off, distros->task_off, D + 1, int64_t);
  CK(e.pos.ensure(sizeof(int64_t) * size_t(T0 + 1)));
  CK(e.src.ensure(sizeof(int32_t) * size_t(Tn + 1)));
  CK(e.err.ensure(sizeof(int)));
  CK(cudaMemsetAsync(e.err.p, 0, sizeof(int), s));
  m.new_off = e.new_off.as<int64_t>(); m.keep = e.keep.as<int32_t>(); m.pos = e.pos.as<int64_t>(); m.src = e.src.as<int32_t>();
  // ---- 1. survivors: the keep mask's scan (each survivor's place), composed row -> source row
  if (T0 > 0) {
    CK(scan_counts(c, e.keep.as<int32_t>(), T0, e.pos.as<int64_t>()));
    launch(c, s, k_ed_src, grid_for(T0, 256), 256, 0, T0, m, e.src.as<int32_t>());
  }
  // ---- 2. the nine columns of the composed table into the shadow set, its padding zeroed as an upload leaves it
  int rc = e.out.size(Tn, s, /*zero_pad=*/true);
  if (rc != EVG_OK) return rc;
  launch(c, s, k_ed_gather, grid_for(Tn, 256), 256, 0, Tn, m, O, In, e.out.dst(), e.err.as<int>());
  // ---- 3. edges: count (range-checking the source's), scan, dep_off at the distro boundaries for the routing (one D2H,
  // one sync), write
  int64_t En = 0;
  std::vector<int64_t> edge_off;
  int bad = 0;
  const bool edges = Tn > 0 && (O.n_edges > 0 || In.n_edges > 0 || m.n_add > 0);
  if (edges) {
    CK(e.edge_cnt.ensure(sizeof(int32_t) * size_t(Tn + 1)));
    CK(e.dep_off.ensure(sizeof(int64_t) * size_t(Tn + 1 + kColPad)));
    launch(c, s, k_ed_edge_count, grid_for(Tn, 256), 256, 0, Tn, m, O, In, e.edge_cnt.as<int32_t>(), e.err.as<int>());
    CK(scan_counts(c, e.edge_cnt.as<int32_t>(), Tn, e.dep_off.as<int64_t>()));
    CK(e.edge_at.ensure(sizeof(int64_t) * size_t(D + 1)));
    launch(c, s, k_gather_i64, grid_for(D + 1, 256), 256, 0, e.dep_off.as<int64_t>(), e.new_off.as<int64_t>(), e.edge_at.as<int64_t>(), D + 1);
    edge_off.resize(size_t(D) + 1);
    CK(cudaMemcpyAsync(edge_off.data(), e.edge_at.p, sizeof(int64_t) * size_t(D + 1), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(&bad, e.err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (bad) drop_tick(c);
  if (bad & 1) return fail(EVG_ERR_INVALID, "group_remap maps the task group of a surviving task to -1");
  if (bad & 2) return fail(EVG_ERR_INVALID, "an in-queue dep_idx is outside its distro");
  if (edges) {
    En = edge_off[size_t(D)];
    CK(e.dep_idx.ensure(sizeof(int32_t) * size_t(En + kColPad)));
    if (En > 0) {
      launch(c, s, k_ed_edge_write, grid_for(Tn, 256), 256, 0, Tn, m, O, In, e.dep_off.as<int64_t>(), e.dep_idx.as<int32_t>());
      CK(cudaGetLastError());
    }
  }
  // ---- 4. the shadow set becomes the resident one
  return install_composed(c, who, Tn, En, edge_off.data(), distros);
}

// --------------------------------------------------------------------------
// evg_plan_from_finder: finder -> dependency predicate -> compaction -> resident planner inputs, all on the device
// --------------------------------------------------------------------------
// evg_plan_from_finder and evg_plan_from_finder_ex (`name`; the former passes no pipe)
static int plan_from_finder(const char* name, evg_ctx* c, const evg_runnable_in* in, const evg_pipeline_in* pipe, const evg_task_soa* cand,
                            const evg_distro_table* distros, const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg,
                            const int64_t* dep_finished_ns, int64_t now_ns, int32_t* runnable, int64_t* count) {
  ENTER(c, name);
  if (!in || !cand || !distros) return fail(EVG_ERR_INVALID, "%s: null argument", who);
  const int64_t T = in->n_tasks, E = cand->n_edges;
  const int32_t D = in->n_distros, P = in->n_projects;
  if (T < 0 || D < 0 || P < 0 || E < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (cand->n_tasks != T || distros->n_distros != D) return fail(EVG_ERR_INVALID, "the candidate table, the finder table and the distro table disagree on their sizes");
  if (D == 0) return T == 0 ? upload(c, who, cand, distros, hosts, host_off, acfg, Tick::kOwn) : fail(EVG_ERR_INVALID, "tasks without distros");
  if (!count) return fail(EVG_ERR_INVALID, "null count");
  // a composed row's source row is 32-bit (compose_tick's src)
  if (T > (int64_t(1) << 31) - 2) return fail(EVG_ERR_INVALID, "evg_plan_from_finder: %lld candidates exceed 2^31-2", (long long)T);
  if (!distros->task_off) return fail(EVG_ERR_INVALID, "null distro arrays");
  if (T > 0 && (!in->deps || in->deps->n_tasks != T)) return fail(EVG_ERR_INVALID, "evg_plan_from_finder needs the candidates' dependency table (the planner's EVG_TF_DEPS_MET comes from it)");
  if (T > 0 && TaskCols::missing(cand)) return fail(EVG_ERR_INVALID, "null candidate column");
  if (E > 0 && (!cand->dep_off || !cand->dep_idx)) return fail(EVG_ERR_INVALID, "null candidate dependency edges");
  // The candidates' dep_off (8 B per candidate, ~10 ms of host memory reads at 8e6 candidates) is checked on a second
  // host thread while this one stages the tables and the device runs the finders; it indexes nothing before step 4.
  // (Where no thread can be started, the check runs at get().)  The thread hands back its message, empty when it passed.
  std::future<std::string> dep_off_err;
  if (E > 0 && T > 0)
    dep_off_err = std::async(std::launch::async | std::launch::deferred,
                             [=] { return check_offsets(cand->dep_off, T, E, who, "candidates->dep_off") == EVG_OK ? std::string() : g_err; });
  DRunnable r;
  bool any_deps, any_pipe = false, pipe_deps = false;
  int rc = stage_finder(c, who, in, &r, &any_deps, pipe, &any_pipe, &pipe_deps);
  if (rc != EVG_OK) return rc;
  for (int32_t d = 0; d <= D; d++)
    if (in->task_off[d] != distros->task_off[d]) return fail(EVG_ERR_INVALID, "the finder table and the distro table cut the candidates differently at distro %d", d);
  cudaStream_t s = c->stream;
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  c->launches = 0;
  drop_tick(c);
  if (T == 0) {
    for (int32_t d = 0; d < D; d++) count[d] = 0;
    return upload(c, who, cand, distros, hosts, host_off, acfg, Tick::kOwn);
  }
  // 1. Task.DependenciesMet / AllDependenciesSatisfied of every candidate, with the DependenciesMetTime stamps
  rc = deps_to_device(c, who, in->deps, 1, dep_finished_ns, now_ns, /*want_stamp=*/true);
  if (rc != EVG_OK) return rc;
  if (pipe_deps) {
    rc = pipeline_deps(c, in->deps, pipe);
    if (rc != EVG_OK) return rc;
  }
  // 2. the finders
  auto& pf = c->pf;
  r.met = c->deps.met.as<uint8_t>();
  if (any_pipe)
    launch(c, s, k_runnable_pipe, unsigned(D), 256, 0, r, c->pl.project_raw.as<uint8_t>(), pf.kept.as<int32_t>(), pf.count.as<int64_t>(),
           c->b_err.as<int>());
  else
    launch(c, s, k_runnable, unsigned(D), 256, 0, r, pf.kept.as<int32_t>(), pf.count.as<int64_t>(), c->b_err.as<int>());
  CK(cudaGetLastError());
  // 3. the only thing the host needs before the planner can be routed: how many tasks each distro kept
  int bad = 0;
  CK(cudaMemcpyAsync(count, pf.count.p, sizeof(int64_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (runnable) CK(cudaMemcpyAsync(runnable, pf.kept.p, sizeof(int32_t) * size_t(T), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) return deps_bad(who, bad);
  const std::string dep_off_msg = dep_off_err.valid() ? dep_off_err.get() : std::string();
  if (!dep_off_msg.empty()) return fail(EVG_ERR_INVALID, "%s", dep_off_msg.c_str());
  std::vector<int64_t> new_off(size_t(D) + 1, 0);
  for (int32_t d = 0; d < D; d++) {
    if (count[d] < 0 || count[d] > in->task_off[d + 1] - in->task_off[d]) return fail(EVG_ERR_CUDA, "finder count out of range");
    new_off[size_t(d) + 1] = new_off[size_t(d)] + count[d];
  }
  // 4. the candidates' columns, with the device's own verdict applied as evg_upload_with_deps applies it; the kept list
  // as a keep mask
  rc = pf.cand.stage(cand, T, s);
  if (rc != EVG_OK) return rc;
  DTasks O = pf.cand.view(T);
  if (E > 0) {
    UP(s, pf.dep_off, cand->dep_off, T + 1, int64_t);
    UP(s, pf.dep_idx, cand->dep_idx, E, int32_t);
    O.n_edges = E; O.dep_off = pf.dep_off.as<int64_t>(); O.dep_idx = pf.dep_idx.as<int32_t>();
  }
  auto& e = c->ed;
  CK(e.keep.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(cudaMemsetAsync(e.keep.p, 0, sizeof(int32_t) * size_t(T), s));
  launch(c, s, k_kept_mask, grid_for(T, 256), 256, 0, T, D, pf.task_off.as<int64_t>(), pf.kept.as<int32_t>(), e.keep.as<int32_t>());
  if (any_pipe) {
    // what the pipeline distros' planner receives: their verdicts (k_pl_plan needs the keep mask), and no candidate
    // edges for EVG_FINDER_PIPELINE rows (compose_tick then re-indexes the rest as for any finder)
    const int64_t* fin = dep_finished_ns && in->deps->n_deps > 0 ? c->deps.fin.as<int64_t>() : nullptr;
    launch(c, s, k_pl_plan, grid_for(T, 256), 256, 0, ddeps(c, in->deps), D, pf.task_off.as<int64_t>(), pf.finder.as<uint8_t>(),
           e.keep.as<int32_t>(), c->deps.met.as<uint8_t>(), fin, now_ns, c->deps.stamp.as<int64_t>());
    if (pipe_deps && E > 0) {
      auto& p = c->pl;
      CK(p.edge_cnt.ensure(sizeof(int32_t) * size_t(T + 1)));
      CK(p.dep_off.ensure(sizeof(int64_t) * size_t(T + 1)));
      launch(c, s, k_pl_edge_count, grid_for(T, 256), 256, 0, T, D, pf.task_off.as<int64_t>(), pf.finder.as<uint8_t>(), pf.dep_off.as<int64_t>(),
             p.edge_cnt.as<int32_t>());
      CK(scan_counts(c, p.edge_cnt.as<int32_t>(), T, p.dep_off.as<int64_t>()));
      // the kept edges fit in the candidates' E: no count has to reach the host
      CK(p.dep_idx.ensure(sizeof(int32_t) * size_t(E)));
      launch(c, s, k_pl_edge_write, grid_for(T, 256), 256, 0, T, pf.dep_off.as<int64_t>(), pf.dep_idx.as<int32_t>(), p.dep_off.as<int64_t>(),
             p.dep_idx.as<int32_t>());
      O.dep_off = p.dep_off.as<int64_t>(); O.dep_idx = p.dep_idx.as<int32_t>();
    }
  }
  launch(c, s, k_apply_deps, grid_for(T, 256), 256, 0, T, c->deps.met.as<uint8_t>(), c->deps.stamp.as<int64_t>(), pf.cand.flags.as<uint32_t>(),
         pf.cand.wb.as<int64_t>());
  CK(e.ins_off.ensure(sizeof(int64_t) * size_t(D + 1)));
  CK(cudaMemsetAsync(e.ins_off.p, 0, sizeof(int64_t) * size_t(D + 1), s));
  // 5. the kept candidates become the resident tick, in the context's own columns
  EdMap m;
  memset(&m, 0, sizeof(m));
  m.D = D; m.old_off = pf.task_off.as<int64_t>(); m.ins_off = e.ins_off.as<int64_t>();
  DTasks none;
  memset(&none, 0, sizeof(none));
  evg_distro_table dn = *distros;
  dn.task_off = new_off.data();
  rc = compose_tick(c, who, m, O, none, &dn);
  if (rc != EVG_OK) return rc;
  if (hosts) {
    rc = upload_hosts(c, who, hosts, host_off, acfg, D);
    if (rc != EVG_OK) return rc;
  }
  CK(cudaStreamSynchronize(s));
  c->tick.kind = Tick::kOwn;
  return EVG_OK;
}
int evg_plan_from_finder(evg_ctx* c, const evg_runnable_in* in, const evg_task_soa* cand, const evg_distro_table* distros,
                         const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg, const int64_t* dep_finished_ns,
                         int64_t now_ns, int32_t* runnable, int64_t* count) {
  return plan_from_finder("evg_plan_from_finder", c, in, nullptr, cand, distros, hosts, host_off, acfg, dep_finished_ns, now_ns, runnable, count);
}
int evg_plan_from_finder_ex(evg_ctx* c, const evg_runnable_in* in, const evg_pipeline_in* pipe, const evg_task_soa* cand,
                            const evg_distro_table* distros, const evg_host_soa* hosts, const int64_t* host_off, const evg_alloc_cfg* acfg,
                            const int64_t* dep_finished_ns, int64_t now_ns, int32_t* runnable, int64_t* count) {
  return plan_from_finder("evg_plan_from_finder_ex", c, in, pipe, cand, distros, hosts, host_off, acfg, dep_finished_ns, now_ns, runnable, count);
}

// --------------------------------------------------------------------------
// evg_edit_tasks: the composed table (survivors, then inserted rows, per distro) built on the device
// --------------------------------------------------------------------------
int evg_edit_tasks(evg_ctx* c, const evg_task_edit* ed, const evg_distro_table* distros, const evg_host_soa* hosts,
                   const int64_t* host_off, const evg_alloc_cfg* acfg) {
  ENTER(c, "evg_edit_tasks");
  if (const int rc = need_tick(c, who, Need::kEditable); rc != EVG_OK) return rc;
  if (!ed || !distros) return fail(EVG_ERR_INVALID, "evg_edit_tasks: null edit / distro table");
  // ---- every check the host can make, before anything resident changes
  const int32_t D = c->Dn;
  const int64_t T0 = c->T, R = ed->n_remove, NA = ed->n_add_edges;
  const evg_task_soa* ins = ed->insert;
  const int64_t I = ins ? ins->n_tasks : 0, EI = ins ? ins->n_edges : 0;
  if (distros->n_distros != D) return fail(EVG_ERR_INVALID, "evg_edit_tasks: n_distros %d, the resident tick has %d", distros->n_distros, D);
  if (R < 0 || I < 0 || EI < 0 || NA < 0) return fail(EVG_ERR_INVALID, "evg_edit_tasks: negative sizes");
  if (R > 0 && !ed->remove_rows) return fail(EVG_ERR_INVALID, "evg_edit_tasks: null remove_rows");
  if (I > 0 && (!ed->insert_off || TaskCols::missing(ins))) return fail(EVG_ERR_INVALID, "evg_edit_tasks: null insert_off / inserted column");
  if (EI > 0 && (I == 0 || !ins->dep_off || !ins->dep_idx)) return fail(EVG_ERR_INVALID, "evg_edit_tasks: inserted edges without dep_off / dep_idx");
  if (NA > 0 && (!ed->add_edge_task || !ed->add_edge_dep)) return fail(EVG_ERR_INVALID, "evg_edit_tasks: null added edges");
  if (D > 0 && (!distros->task_off || !distros->group_off || !distros->cfg)) return fail(EVG_ERR_INVALID, "evg_edit_tasks: null distro arrays");
  if (D == 0 && (R > 0 || I > 0)) return fail(EVG_ERR_INVALID, "evg_edit_tasks: rows without distros");
  std::vector<int64_t> removed(size_t(D) + 1, 0), ins_off(size_t(D) + 1, 0), old_vbase(size_t(D) + 1, 0);
  for (int64_t k = 0; k < R; k++) {
    const int64_t r = ed->remove_rows[k];
    if (r < 0 || r >= T0 || (k > 0 && r <= ed->remove_rows[k - 1]))
      return fail(EVG_ERR_INVALID, "evg_edit_tasks: remove_rows[%lld] = %lld is not ascending inside [0, %lld)", (long long)k, (long long)r, (long long)T0);
    removed[size_t(std::upper_bound(c->h_taskoff.begin(), c->h_taskoff.end(), r) - c->h_taskoff.begin() - 1)]++;
  }
  int rc = I > 0 ? check_offsets(ed->insert_off, D, I, who, "insert_off") : EVG_OK;
  if (rc == EVG_OK && EI > 0) rc = check_offsets(ins->dep_off, I, EI, who, "insert->dep_off");
  if (rc == EVG_OK && D > 0) rc = check_offsets(distros->task_off, D, -1, who, "task_off");
  if (rc == EVG_OK && D > 0) rc = check_offsets(distros->group_off, D, -1, who, "group_off");
  if (rc != EVG_OK) return rc;
  if (I > 0) ins_off.assign(ed->insert_off, ed->insert_off + D + 1);
  for (int32_t d = 0; d < D; d++) {
    const int64_t want = (c->h_taskoff[d + 1] - c->h_taskoff[d]) - removed[d] + (ins_off[d + 1] - ins_off[d]);
    if (distros->task_off[d + 1] - distros->task_off[d] != want)
      return fail(EVG_ERR_INVALID, "evg_edit_tasks: distro %d holds %lld tasks after the edit, task_off says %lld", d, (long long)want,
                  (long long)(distros->task_off[d + 1] - distros->task_off[d]));
    old_vbase[d + 1] = old_vbase[d] + c->h_nver[d];
  }
  const int64_t Tn = D > 0 ? distros->task_off[D] : 0;
  for (int64_t k = 0, d = 0; k < NA; k++) {
    const int64_t row = ed->add_edge_task[k];
    if (k > 0 && row < ed->add_edge_task[k - 1]) return fail(EVG_ERR_INVALID, "evg_edit_tasks: add_edge_task is not ascending at %lld", (long long)k);
    if (row < 0 || row >= Tn) return fail(EVG_ERR_INVALID, "evg_edit_tasks: add_edge_task[%lld] = %lld is outside the composed table", (long long)k, (long long)row);
    while (distros->task_off[d + 1] <= row) d++;
    const int64_t survivors = (c->h_taskoff[d + 1] - c->h_taskoff[d]) - removed[d];
    if (row - distros->task_off[d] >= survivors)
      return fail(EVG_ERR_INVALID, "evg_edit_tasks: add_edge_task[%lld] = %lld is not a surviving task", (long long)k, (long long)row);
  }
  cudaStream_t s = c->stream;
  auto& e = c->ed;
  c->launches = 0;
  // ---- stage the edit
  UP(s, e.rm, ed->remove_rows, R, int64_t);
  if (I > 0 && (rc = e.ins.stage(ins, I, s)) != EVG_OK) return rc;
  UP(s, e.ins_dep_off, EI > 0 ? ins->dep_off : nullptr, EI > 0 ? I + 1 : 0, int64_t);
  UP(s, e.ins_dep_idx, EI > 0 ? ins->dep_idx : nullptr, EI, int32_t);
  UP(s, e.add_task, ed->add_edge_task, NA, int64_t);
  UP(s, e.add_dep, ed->add_edge_dep, NA, int32_t);
  const int64_t G0 = c->h_groupoff[size_t(D)];
  UP(s, e.gremap, ed->group_remap, ed->group_remap ? G0 : 0, int32_t);
  UP(s, e.vremap, ed->version_remap, ed->version_remap ? old_vbase[D] : 0, int32_t);
  UP(s, e.old_off, c->h_taskoff.data(), D + 1, int64_t);
  UP(s, e.old_goff, c->h_groupoff.data(), D + 1, int64_t);
  UP(s, e.ins_off, ins_off.data(), D + 1, int64_t);
  UP(s, e.old_vbase, old_vbase.data(), D + 1, int64_t);
  CK(e.keep.ensure(sizeof(int32_t) * size_t(T0 + 1)));
  launch(c, s, k_ed_keep, grid_for(T0, 256), 256, 0, T0, e.rm.as<int64_t>(), R, e.keep.as<int32_t>());
  EdMap m;
  memset(&m, 0, sizeof(m));
  m.D = D; m.old_off = e.old_off.as<int64_t>(); m.ins_off = e.ins_off.as<int64_t>();
  m.old_goff = e.old_goff.as<int64_t>(); m.old_vbase = e.old_vbase.as<int64_t>();
  m.gremap = ed->group_remap ? e.gremap.as<int32_t>() : nullptr;
  m.vremap = ed->version_remap ? e.vremap.as<int32_t>() : nullptr;
  m.n_add = NA; m.add_task = e.add_task.as<int64_t>(); m.add_dep = e.add_dep.as<int32_t>();
  DTasks In = e.ins.view(I);
  In.n_edges = EI; In.dep_off = e.ins_dep_off.as<int64_t>(); In.dep_idx = e.ins_dep_idx.as<int32_t>();
  rc = compose_tick(c, who, m, dtasks(c), In, distros);
  if (rc != EVG_OK) return rc;
  if (hosts) {
    rc = upload_hosts(c, who, hosts, host_off, acfg, D);
    if (rc != EVG_OK) return rc;
    CK(cudaStreamSynchronize(s));
  }
  c->tick.kind = Tick::kOwn;
  return EVG_OK;
}

// --------------------------------------------------------------------------
// evg_plan_aliases: every distro's alias queue built on the device from the tick's schedulable tasks, each staged once
// --------------------------------------------------------------------------
// A (queue, task) pair is the 64-bit key distro << 32 | source row: sorted, the keys list every alias queue in
// ascending source row, and a queue's rows are found by binary search.
struct AlView {
  int64_t n;
  int32_t D, n_names, n_groups, n_versions;
  const uint8_t* sched;
  const int32_t* tgmax;
  const int32_t* primary;
  const int64_t* soff;
  const int32_t* sidx;
  const int64_t* doff;
  const int32_t* didx;
};
// The distinct alias queues row t joins (FindHostSchedulableForAlias, model/task/task.go:3371-3386): their keys go to
// out[0 ..] unless out is NULL; returns how many.  A destination counts once: the (name, destination) entries before it
// are searched again rather than kept in a local array, which a long SecondaryDistros could overflow.  *err bit 0: a
// name index out of range.
__device__ int64_t al_dests(const AlView& v, int64_t t, uint64_t* __restrict__ out, int* err) {
  constexpr uint32_t kBase = EVG_SQ_ACTIVATED | EVG_SQ_UNDISPATCHED | EVG_SQ_PRIORITY_OK | EVG_SQ_HOST_PLATFORM;  // db.go:671-689
  const uint32_t sq = v.sched[t];
  if ((sq & kBase) != kBase || ((sq & EVG_SQ_UNATTAINABLE) && !(sq & EVG_SQ_OVERRIDE_DEPS))) return 0;
  if (v.tgmax[t] == 1) return 0;  // TaskGroupMaxHosts != 1, the raw field (task.go:3382)
  const int64_t j0 = v.soff[t], j1 = v.soff[t + 1];
  int64_t n = 0;
  for (int64_t j = j0; j < j1; j++) {
    const int32_t name = v.sidx[j];
    if (name == -1) continue;  // a name no distro has
    if (name < 0 || name >= v.n_names) { if (err) atomicOr(err, 1); continue; }
    for (int64_t k = v.doff[name]; k < v.doff[name + 1]; k++) {
      const int32_t e = v.didx[k];
      bool seen = false;
      for (int64_t j2 = j0; j2 <= j && !seen; j2++) {
        const int32_t nm = v.sidx[j2];
        if (nm < 0 || nm >= v.n_names) continue;
        const int64_t k_end = j2 < j ? v.doff[nm + 1] : k;
        for (int64_t k2 = v.doff[nm]; k2 < k_end && !seen; k2++) seen = v.didx[k2] == e;
      }
      if (seen) continue;
      if (out) out[n] = (uint64_t(uint32_t(e)) << 32) | uint64_t(t);
      n++;
    }
  }
  return n;
}
// Per source row: its pair count, and the range check of the ids it carries (err bit 0).
__global__ void __launch_bounds__(256) k_al_count(AlView v, DTasks S, int32_t* __restrict__ cnt, int* err) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= v.n) return;
  const int32_t g = S.gid[t], ver = S.vid[t], p = v.primary[t];
  if (g < -1 || g >= v.n_groups || ver < 0 || ver >= v.n_versions || p < -1 || p >= v.D) atomicOr(err, 1);
  cnt[t] = int32_t(al_dests(v, t, nullptr, err));
}
// Per source row: its pairs at poff[t], so that the key array is in source-row order.
__global__ void __launch_bounds__(256) k_al_pairs(AlView v, const int64_t* __restrict__ poff, uint64_t* __restrict__ keys) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= v.n) return;
  al_dests(v, t, keys + poff[t], nullptr);
}
// Stable LSD radix sort of the keys by the distro bits, 8 bits a pass, 2048 keys a block: the keys start in source-row
// order, so sorting by distro alone leaves every queue in source-row order.
constexpr int kAlTile = 2048;
// counters of digit b of tile k at hist[b * n_tiles + k] (digit-major: their exclusive scan is every tile's run start)
__global__ void __launch_bounds__(256) k_al_hist(const uint64_t* __restrict__ keys, int64_t n, int shift, int32_t* __restrict__ hist,
                                                 int64_t n_tiles) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t t0 = int64_t(blockIdx.x) * kAlTile;
  for (int k = threadIdx.x; k < kAlTile; k += 256)
    if (t0 + k < n) atomicAdd(&h[uint32_t(keys[t0 + k] >> shift) & 255u], 1u);
  __syncthreads();
  hist[int64_t(threadIdx.x) * n_tiles + blockIdx.x] = int32_t(h[threadIdx.x]);
}
// The tile in chunks of 256 keys, in order: a key's place is its digit's run start + the keys of that digit in the
// earlier chunks (base) + those of the earlier warps in this chunk (wcnt) + those of the earlier lanes (MATCH.ANY).
__global__ void __launch_bounds__(256) k_al_scatter(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, int64_t n, int shift,
                                                    const int64_t* __restrict__ off, int64_t n_tiles) {
  __shared__ uint32_t base[256];
  __shared__ uint32_t wcnt[8][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  base[tid] = 0;
  for (int w = 0; w < 8; w++) wcnt[w][tid] = 0;
  __syncthreads();
  const int64_t t0 = int64_t(blockIdx.x) * kAlTile;
  for (int c0 = 0; c0 < kAlTile; c0 += 256) {
    const int64_t i = t0 + c0 + tid;
    const bool ok = i < n;
    const uint64_t key = ok ? in[i] : 0;
    const uint32_t dg = ok ? (uint32_t(key >> shift) & 255u) : 256u;
    const uint32_t peers = __match_any_sync(0xffffffffu, dg);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (ok && rank == 0) wcnt[warp][dg] = __popc(peers);
    __syncthreads();
    if (ok) {
      uint32_t r = base[dg] + rank;
      for (int w = 0; w < warp; w++) r += wcnt[w][dg];
      out[off[int64_t(dg) * n_tiles + blockIdx.x] + r] = key;
    }
    __syncthreads();
    uint32_t sum = 0;
    for (int w = 0; w < 8; w++) { sum += wcnt[w][tid]; wcnt[w][tid] = 0; }
    base[tid] += sum;
    __syncthreads();
  }
}
// qoff[e] = first pair of distro e (e = 0 .. D; qoff[D] = n): the alias queues' task_off
__global__ void __launch_bounds__(256) k_al_qoff(const uint64_t* __restrict__ keys, int64_t n, int32_t D, int64_t* __restrict__ qoff) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e > D) return;
  const uint64_t want = uint64_t(e) << 32;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < want) lo = mid + 1; else hi = mid;
  }
  qoff[e] = lo;
}
constexpr uint64_t kAlEmpty = ~uint64_t(0);
// Open-addressing slot of `key` in (hk, hv), inserted if new; hv[slot] becomes the smallest pair index that carries it.
__device__ __forceinline__ int64_t al_insert(uint64_t* hk, uint32_t* hv, uint64_t mask, uint64_t key, uint32_t i) {
  uint64_t h = key * 0x9E3779B97F4A7C15ull;
  h ^= h >> 29;
  for (uint64_t slot = h & mask;; slot = (slot + 1) & mask) {
    const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(hk + slot), (unsigned long long)kAlEmpty,
                                              (unsigned long long)key);
    if (prev == kAlEmpty || prev == key) {
      atomicMin(hv + slot, i);
      return int64_t(slot);
    }
  }
}
// Per pair: the (queue, task group) and (queue, version) it belongs to, keyed queue << 32 | global id (bit 63 marks a
// version), and the first pair of each.
__global__ void __launch_bounds__(256) k_al_first(int64_t n, const uint64_t* __restrict__ keys, DTasks S, uint64_t* hk, uint32_t* hv,
                                                  uint64_t mask, int64_t* __restrict__ gslot, int64_t* __restrict__ vslot) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys[i], q = k >> 32 << 32;
  const uint32_t t = uint32_t(k);
  const int32_t g = S.gid[t];
  gslot[i] = g >= 0 ? al_insert(hk, hv, mask, q | uint32_t(g), uint32_t(i)) : -1;
  vslot[i] = al_insert(hk, hv, mask, (uint64_t(1) << 63) | q | uint32_t(S.vid[t]), uint32_t(i));
}
// first-appearance flags: their exclusive scans number each queue's groups and versions in first-appearance order
__global__ void __launch_bounds__(256) k_al_flag(int64_t n, const int64_t* __restrict__ gslot, const int64_t* __restrict__ vslot,
                                                 const uint32_t* __restrict__ hv, int32_t* __restrict__ fg, int32_t* __restrict__ fv) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  fg[i] = gslot[i] >= 0 && hv[gslot[i]] == uint32_t(i);
  fv[i] = hv[vslot[i]] == uint32_t(i);
}
struct AlIds {
  const int64_t *qoff, *gslot, *vslot, *pg, *pv;
  const uint32_t* hv;
};
// Pair i = (queue e, source row t) becomes row i of the composed table: the source row's columns with the queue's
// group and version ids and EVG_TF_OTHER_DISTRO for e; its alias map entry, and the group slot of a group's first pair.
__global__ void __launch_bounds__(256) k_al_gather(int64_t n, const uint64_t* __restrict__ keys, AlIds a, DTasks S,
                                                   const int32_t* __restrict__ primary, const int32_t* __restrict__ gmax, EdDst o,
                                                   int32_t* __restrict__ srow, int32_t* __restrict__ gout, int32_t* __restrict__ gsrc) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys[i];
  const int64_t t = uint32_t(k);
  const int e = int(k >> 32);
  const int64_t q0 = a.qoff[e];
  int32_t g = S.gid[t];
  if (g >= 0) {
    const int64_t slot = a.pg[i];
    if (a.hv[a.gslot[i]] == uint32_t(i)) { gout[slot] = gmax[g]; gsrc[slot] = g; }
    g = int32_t(a.pg[a.hv[a.gslot[i]]] - a.pg[q0]);
  }
  o.priority[i] = S.priority[t]; o.numdep[i] = S.numdep[t]; o.tgo[i] = S.tgo[t]; o.gid[i] = g;
  o.vid[i] = int32_t(a.pv[a.hv[a.vslot[i]]] - a.pv[q0]);
  o.flags[i] = (S.flags[t] & ~EVG_TF_OTHER_DISTRO) | (primary[t] != e ? EVG_TF_OTHER_DISTRO : 0u);  // scheduler.go:75
  o.expected[i] = S.expected[t]; o.qbasis[i] = S.qbasis[t]; o.wbasis[i] = S.wbasis[t];
  srow[i] = int32_t(t);
}
// Edges of pair i = (e, t): t's source edges t -> u with (e, u) a pair, re-indexed to u's place in e, in DependsOn order
// (duplicates kept).  o_dep_idx == NULL: count them, raising *err bit 1 for a dep_idx outside the table.
__device__ int64_t al_edges(int64_t i, const uint64_t* __restrict__ keys, const int64_t* __restrict__ qoff, const DTasks& S,
                            const int64_t* __restrict__ o_dep_off, int32_t* __restrict__ o_dep_idx, int* err) {
  const uint64_t k = keys[i];
  const int64_t t = uint32_t(k);
  const uint64_t q = k >> 32 << 32;
  const int64_t a = qoff[k >> 32], b = qoff[(k >> 32) + 1];
  int64_t w = o_dep_off ? o_dep_off[i] : 0, n = 0;
  for (int64_t j = S.dep_off[t]; j < S.dep_off[t + 1]; j++) {
    const int32_t x = S.dep_idx[j];
    if (x < 0 || x >= S.n) { if (err) atomicOr(err, 2); continue; }
    const uint64_t want = q | uint32_t(x);
    int64_t lo = a, hi = b;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] < want) lo = mid + 1; else hi = mid;
    }
    if (lo == b || keys[lo] != want) continue;
    if (o_dep_idx) o_dep_idx[w + n] = int32_t(lo - a);
    n++;
  }
  return n;
}
__global__ void __launch_bounds__(256) k_al_edge_count(int64_t n, const uint64_t* __restrict__ keys, const int64_t* __restrict__ qoff,
                                                       DTasks S, int32_t* __restrict__ cnt, int* err) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  cnt[i] = int32_t(al_edges(i, keys, qoff, S, nullptr, nullptr, err));
}
__global__ void __launch_bounds__(256) k_al_edge_write(int64_t n, const uint64_t* __restrict__ keys, const int64_t* __restrict__ qoff,
                                                       DTasks S, const int64_t* __restrict__ o_dep_off, int32_t* __restrict__ o_dep_idx) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  al_edges(i, keys, qoff, S, o_dep_off, o_dep_idx, nullptr);
}

int evg_plan_aliases(evg_ctx* c, const evg_alias_in* in, const evg_distro_cfg* cfg, int32_t D, int64_t now_ns, evg_alias_out* out) {
  ENTER(c, "evg_plan_aliases");
  if (!in || !out || !in->deps) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null argument");
  // ---- every check the host can make, before anything resident changes
  const evg_task_soa* t = &in->tasks;
  const evg_deps_in* dp = in->deps;
  const int64_t T = t->n_tasks, E = t->n_edges;
  const int32_t NG = in->n_groups, NV = in->n_versions, NN = in->n_names;
  if (T < 0 || E < 0 || D < 0 || NG < 0 || NV < 0 || NN < 0 || dp->n_deps < 0 || dp->n_ext < 0)
    return fail(EVG_ERR_INVALID, "evg_plan_aliases: negative sizes");
  if (dp->n_tasks != T) return fail(EVG_ERR_INVALID, "evg_plan_aliases: deps covers %lld rows, the table %lld", (long long)dp->n_tasks, (long long)T);
  if (T > (int64_t(1) << 31) - 2) return fail(EVG_ERR_INVALID, "evg_plan_aliases: %lld rows exceed 2^31-2", (long long)T);
  if (!out->task_off || !out->group_off || (D > 0 && (!out->n_versions || !cfg))) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null cfg / output");
  if (!in->secondary_off || !in->dest_off || (NG > 0 && !in->group_max_hosts)) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null offsets / group_max_hosts");
  if (T > 0 && (TaskCols::missing(t) || !in->sched || !in->task_group_max_hosts || !in->primary || !dp->dep_off || !dp->task_state ||
                !dp->task_pre))
    return fail(EVG_ERR_INVALID, "evg_plan_aliases: null task column");
  if (E > 0 && (!t->dep_off || !t->dep_idx)) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null dep_off / dep_idx");
  if (dp->n_deps > 0 && (!dp->dep_kind || !dp->dep_ref || !dp->dep_want)) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null dependency arrays");
  if (dp->n_ext > 0 && !dp->ext_state) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null ext_state");
  // deps->dep_off is checked by deps_to_device and k_deps_met, like every evg_deps_in
  int rc = check_offsets(in->secondary_off, T, -1, who, "secondary_off");
  if (rc == EVG_OK) rc = check_offsets(in->dest_off, NN, -1, who, "dest_off");
  if (rc == EVG_OK && E > 0) rc = check_offsets(t->dep_off, T, E, who, "tasks.dep_off");
  if (rc != EVG_OK) return rc;
  const int64_t NS = in->secondary_off[T], ND = in->dest_off[NN];
  if (NS > 0 && !in->secondary_idx) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null secondary_idx");
  if (ND > 0 && !in->dest_idx) return fail(EVG_ERR_INVALID, "evg_plan_aliases: null dest_idx");
  for (int64_t k = 0; k < ND; k++)
    if (in->dest_idx[k] < 0 || in->dest_idx[k] >= D)
      return fail(EVG_ERR_INVALID, "evg_plan_aliases: dest_idx[%lld] = %d is outside [0, %d)", (long long)k, in->dest_idx[k], D);
  // ---- from here the previous tick is gone: the dependency state and the resident columns are replaced
  cudaStream_t s = c->stream;
  auto& a = c->al;
  drop_tick(c);
  c->launches = 0;
  CK(c->b_err.ensure(sizeof(int) * 4));
  CK(cudaMemsetAsync(c->b_err.p, 0, sizeof(int) * 4, s));
  CK(a.err.ensure(sizeof(int)));
  CK(cudaMemsetAsync(a.err.p, 0, sizeof(int), s));
  int* err = a.err.as<int>();
  // 1. the source table, Task.DependenciesMet with its stamps over the source rows, once
  rc = a.src.stage(t, T, s);
  if (rc != EVG_OK) return rc;
  DTasks S = a.src.view(T);
  UP(s, a.dep_off, E > 0 ? t->dep_off : nullptr, E > 0 ? T + 1 : 0, int64_t);
  UP(s, a.dep_idx, t->dep_idx, E, int32_t);
  S.n_edges = E; S.dep_off = a.dep_off.as<int64_t>(); S.dep_idx = a.dep_idx.as<int32_t>();
  UP(s, a.gmax, in->group_max_hosts, NG, int32_t);
  UP(s, a.sched, in->sched, T, uint8_t);
  UP(s, a.tgmax, in->task_group_max_hosts, T, int32_t);
  UP(s, a.primary, in->primary, T, int32_t);
  UP(s, a.soff, in->secondary_off, T + 1, int64_t);
  UP(s, a.sidx, in->secondary_idx, NS, int32_t);
  UP(s, a.doff, in->dest_off, NN + 1, int64_t);
  UP(s, a.didx, in->dest_idx, ND, int32_t);
  if (T > 0) {
    rc = deps_to_device(c, who, dp, 0, in->dep_finished_ns, now_ns, /*want_stamp=*/true);
    if (rc != EVG_OK) return rc;
    launch(c, s, k_apply_deps, grid_for(T, 256), 256, 0, T, c->deps.met.as<uint8_t>(), c->deps.stamp.as<int64_t>(), a.src.flags.as<uint32_t>(),
           a.src.wb.as<int64_t>());
  }
  // 2. per row: eligibility and its distinct alias queues; the pair offsets (one value crosses to the host)
  AlView v;
  v.n = T; v.D = D; v.n_names = NN; v.n_groups = NG; v.n_versions = NV;
  v.sched = a.sched.as<uint8_t>(); v.tgmax = a.tgmax.as<int32_t>(); v.primary = a.primary.as<int32_t>();
  v.soff = a.soff.as<int64_t>(); v.sidx = a.sidx.as<int32_t>(); v.doff = a.doff.as<int64_t>(); v.didx = a.didx.as<int32_t>();
  CK(a.cnt.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(a.poff.ensure(sizeof(int64_t) * size_t(T + 1)));
  int64_t P = 0;
  int bad = 0;
  if (T > 0) {
    launch(c, s, k_al_count, grid_for(T, 256), 256, 0, v, S, a.cnt.as<int32_t>(), err);
    CK(scan_counts(c, a.cnt.as<int32_t>(), T, a.poff.as<int64_t>()));
    CK(cudaMemcpyAsync(&P, a.poff.as<int64_t>() + T, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(&bad, err, sizeof(int), cudaMemcpyDeviceToHost, s));
  int bad_ref = 0;
  CK(cudaMemcpyAsync(&bad_ref, c->b_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (bad_ref) return deps_bad(who, bad_ref);
  if (bad) return fail(EVG_ERR_INVALID, "evg_plan_aliases: a secondary_idx, primary, group_id or version_id is out of range");
  if (P > (int64_t(1) << 31) - 2) return fail(EVG_ERR_INVALID, "evg_plan_aliases: %lld (queue, task) pairs exceed 2^31-2", (long long)P);
  // 3. the pairs, in source-row order, sorted by queue
  for (int k = 0; k < 2; k++) CK(a.keys[k].ensure(sizeof(uint64_t) * size_t(P + 1)));
  int cur = 0;
  if (P > 0) {
    launch(c, s, k_al_pairs, grid_for(T, 256), 256, 0, v, a.poff.as<int64_t>(), a.keys[0].as<uint64_t>());
    int bits = 0;
    while (bits < 31 && (int64_t(1) << bits) < D) bits++;
    const int64_t n_tiles = (P + kAlTile - 1) / kAlTile, nh = 256 * n_tiles;
    if (bits > 0) {
      CK(a.hist.ensure(sizeof(int32_t) * size_t(nh)));
      CK(a.hoff.ensure(sizeof(int64_t) * size_t(nh + 1)));
    }
    for (int shift = 32; shift < 32 + bits; shift += 8, cur ^= 1) {
      launch(c, s, k_al_hist, unsigned(n_tiles), 256, 0, a.keys[cur].as<uint64_t>(), P, shift, a.hist.as<int32_t>(), n_tiles);
      CK(scan_counts(c, a.hist.as<int32_t>(), nh, a.hoff.as<int64_t>()));
      launch(c, s, k_al_scatter, unsigned(n_tiles), 256, 0, a.keys[cur].as<uint64_t>(), a.keys[cur ^ 1].as<uint64_t>(), P, shift,
             a.hoff.as<int64_t>(), n_tiles);
    }
  }
  const uint64_t* keys = a.keys[cur].as<uint64_t>();
  CK(a.qoff.ensure(sizeof(int64_t) * size_t(D + 1)));
  launch(c, s, k_al_qoff, grid_for(D + 1, 256), 256, 0, keys, P, D, a.qoff.as<int64_t>());
  // 4. per queue, dense group and version ids in first-appearance order
  uint64_t cap = 64;
  while (cap < 4 * uint64_t(P)) cap <<= 1;  // at most 2P keys: load factor <= 1/2
  for (DevBuf* b : {&a.pg, &a.pv}) CK(b->ensure(sizeof(int64_t) * size_t(P + 1)));
  for (DevBuf* b : {&a.gslot, &a.vslot}) CK(b->ensure(sizeof(int64_t) * size_t(P + 1)));
  for (DevBuf* b : {&a.fg, &a.fv, &a.srow, &a.gout, &a.gsrc}) CK(b->ensure(sizeof(int32_t) * size_t(P + 1)));
  CK(cudaMemsetAsync(a.pg.p, 0, sizeof(int64_t), s));  // P == 0: the scans do not run
  CK(cudaMemsetAsync(a.pv.p, 0, sizeof(int64_t), s));
  if (P > 0) {
    CK(a.hk.ensure(sizeof(uint64_t) * cap));
    CK(a.hv.ensure(sizeof(uint32_t) * cap));
    CK(cudaMemsetAsync(a.hk.p, 0xFF, sizeof(uint64_t) * cap, s));
    CK(cudaMemsetAsync(a.hv.p, 0xFF, sizeof(uint32_t) * cap, s));
    launch(c, s, k_al_first, grid_for(P, 256), 256, 0, P, keys, S, a.hk.as<uint64_t>(), a.hv.as<uint32_t>(), cap - 1, a.gslot.as<int64_t>(),
           a.vslot.as<int64_t>());
    launch(c, s, k_al_flag, grid_for(P, 256), 256, 0, P, a.gslot.as<int64_t>(), a.vslot.as<int64_t>(), a.hv.as<uint32_t>(), a.fg.as<int32_t>(),
           a.fv.as<int32_t>());
    CK(scan_counts(c, a.fg.as<int32_t>(), P, a.pg.as<int64_t>()));
    CK(scan_counts(c, a.fv.as<int32_t>(), P, a.pv.as<int64_t>()));
  }
  // 5. the nine columns into the shadow set, its padding zeroed as an upload leaves it
  auto& e = c->ed;
  rc = e.out.size(P, s, /*zero_pad=*/true);
  if (rc != EVG_OK) return rc;
  AlIds ids;
  ids.qoff = a.qoff.as<int64_t>(); ids.gslot = a.gslot.as<int64_t>(); ids.vslot = a.vslot.as<int64_t>();
  ids.pg = a.pg.as<int64_t>(); ids.pv = a.pv.as<int64_t>(); ids.hv = a.hv.as<uint32_t>();
  launch(c, s, k_al_gather, grid_for(P, 256), 256, 0, P, keys, ids, S, a.primary.as<int32_t>(), a.gmax.as<int32_t>(), e.out.dst(),
         a.srow.as<int32_t>(), a.gout.as<int32_t>(), a.gsrc.as<int32_t>());
  // 6. edges: count, scan; the queue, group, version and edge offsets of every distro cross to the host (one sync)
  const bool edges = P > 0 && E > 0;
  CK(a.samp.ensure(sizeof(int64_t) * 3 * size_t(D + 1)));
  int64_t* samp = a.samp.as<int64_t>();
  launch(c, s, k_gather_i64, grid_for(D + 1, 256), 256, 0, a.pg.as<int64_t>(), a.qoff.as<int64_t>(), samp, D + 1);
  launch(c, s, k_gather_i64, grid_for(D + 1, 256), 256, 0, a.pv.as<int64_t>(), a.qoff.as<int64_t>(), samp + (D + 1), D + 1);
  if (edges) {
    CK(e.edge_cnt.ensure(sizeof(int32_t) * size_t(P + 1)));
    CK(e.dep_off.ensure(sizeof(int64_t) * size_t(P + 1 + kColPad)));
    launch(c, s, k_al_edge_count, grid_for(P, 256), 256, 0, P, keys, a.qoff.as<int64_t>(), S, e.edge_cnt.as<int32_t>(), err);
    CK(scan_counts(c, e.edge_cnt.as<int32_t>(), P, e.dep_off.as<int64_t>()));
    launch(c, s, k_gather_i64, grid_for(D + 1, 256), 256, 0, e.dep_off.as<int64_t>(), a.qoff.as<int64_t>(), samp + 2 * (D + 1), D + 1);
  }
  std::vector<int64_t> h(3 * size_t(D + 1), 0);
  CK(cudaMemcpyAsync(out->task_off, a.qoff.p, sizeof(int64_t) * size_t(D + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h.data(), samp, sizeof(int64_t) * size_t(edges ? 3 : 2) * size_t(D + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, err, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (bad) return fail(EVG_ERR_INVALID, "evg_plan_aliases: a dep_idx is outside the table");
  const int64_t* vs = h.data() + (D + 1);
  const int64_t* edge_off = h.data() + 2 * (D + 1);
  for (int32_t d = 0; d < D; d++) {
    const int64_t len = out->task_off[d + 1] - out->task_off[d];
    if (len > kMaxTasksPerDistro) return fail(EVG_ERR_INVALID, "evg_plan_aliases: the alias queue of distro %d holds %lld tasks (max %lld)", d, (long long)len, (long long)kMaxTasksPerDistro);
    out->group_off[d] = h[size_t(d)];
    out->n_versions[d] = int32_t(vs[d + 1] - vs[d]);
  }
  out->group_off[D] = h[size_t(D)];
  const int64_t G = h[size_t(D)], En = edges ? edge_off[D] : 0;
  // 7. the group slots' max hosts (O(alias groups) values) and the edges; then the composed table becomes the tick
  std::vector<int32_t> gmax(size_t(G) + 1);
  if (G > 0) CK(cudaMemcpyAsync(gmax.data(), a.gout.p, sizeof(int32_t) * size_t(G), cudaMemcpyDeviceToHost, s));
  if (edges) {
    CK(e.dep_idx.ensure(sizeof(int32_t) * size_t(En + kColPad)));
    if (En > 0)
      launch(c, s, k_al_edge_write, grid_for(P, 256), 256, 0, P, keys, a.qoff.as<int64_t>(), S, e.dep_off.as<int64_t>(), e.dep_idx.as<int32_t>());
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  std::vector<evg_distro_cfg> cf(cfg, cfg + D);
  for (int32_t d = 0; d < D; d++) cf[size_t(d)].n_versions = out->n_versions[d];
  evg_distro_table dt;
  memset(&dt, 0, sizeof(dt));
  dt.n_distros = D; dt.task_off = out->task_off; dt.group_off = out->group_off; dt.cfg = cf.data(); dt.group_max_hosts = gmax.data();
  rc = install_composed(c, who, P, En, edge_off, &dt);
  if (rc != EVG_OK) return rc;
  c->tick.kind = Tick::kOwn;
  c->tick.aliases = true;
  return EVG_OK;
}

int evg_download_alias_map(evg_ctx* c, int32_t* source_row, int32_t* group_source) {
  ENTER(c, "evg_download_alias_map");
  if (const int rc = need_tick(c, who, Need::kAliasMap); rc != EVG_OK) return rc;
  if (source_row && c->T) CK(cudaMemcpyAsync(source_row, c->al.srow.p, sizeof(int32_t) * size_t(c->T), cudaMemcpyDeviceToHost, c->stream));
  if (group_source && c->G) CK(cudaMemcpyAsync(group_source, c->al.gsrc.p, sizeof(int32_t) * size_t(c->G), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return EVG_OK;
}

// --------------------------------------------------------------------------
// evg_intern_columns: host-side string interning (evg_intern.h)
// --------------------------------------------------------------------------
int evg_intern_columns(const evg_string_cols* in, evg_intern_out* out, int32_t threads) {
  using namespace evg_intern;
  if (!in || !out) return fail(EVG_ERR_INVALID, "evg_intern_columns: null argument");
  const int64_t T = in->n_tasks;
  const int32_t D = in->n_distros;
  if (T < 0 || D < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (!out->group_off || (D > 0 && (!in->task_off || !out->n_versions))) return fail(EVG_ERR_INVALID, "null distro arrays");
  if (D == 0) { out->group_off[0] = 0; return T == 0 ? EVG_OK : fail(EVG_ERR_INVALID, "tasks without distros"); }
  int rc = check_offsets(in->task_off, D, T, "evg_intern_columns", "task_off");
  if (rc != EVG_OK) return rc;
  if (T > 0 && (!in->id.off || !in->version.off || !in->group_key.off || !in->group_max_hosts || !in->dep_off || !out->group_id ||
                !out->version_id || !out->group_max_hosts || !out->group_first || !out->dep_off))
    return fail(EVG_ERR_INVALID, "null column");
  const int64_t E = T > 0 ? in->dep_off[T] : 0;
  if (E > 0 && (!in->dep_id.off || !out->dep_idx)) return fail(EVG_ERR_INVALID, "null dependency columns");
  // per distro: groups found, surviving edges (phase 1 counts into per-distro scratch, phase 2 writes at the scanned offsets)
  std::vector<int64_t> n_groups(size_t(D), 0), n_edges(size_t(D), 0);
  std::vector<std::vector<int32_t>> grp_max_by_distro(static_cast<size_t>(D));
  std::vector<std::vector<int64_t>> grp_first_by_distro(static_cast<size_t>(D));
  std::vector<std::vector<int32_t>> edge_by_distro(static_cast<size_t>(D));
  std::atomic<int32_t> next{0};
  std::atomic<int64_t> bad_row{-1};
  // dep_off, a row per task, is checked by the workers as they walk it (a serial scan before them would cost a visible
  // share of the call): a row outside [0, E] or decreasing is not walked, and sends the table through check_offsets
  std::atomic<bool> bad_dep{false};
  int nt = threads > 0 ? threads : int(std::thread::hardware_concurrency());
  nt = std::max(1, std::min(nt, int(D)));
  auto work = [&]() {
    Table groups, versions, ids;
    for (;;) {
      const int32_t d = next.fetch_add(1);
      if (d >= D) return;
      const int64_t a = in->task_off[d], b = in->task_off[d + 1];
      const int64_t n = b - a;
      groups.reset(n); versions.reset(n); ids.reset(n);
      int32_t ng = 0, nv = 0;
      bool ins;
      for (int64_t t = a; t < b; t++) {
        ids.get_or_put(str_at(in->id.bytes, in->id.off, t), in->id.bytes, in->id.off, t, int32_t(t - a), &ins);  // a repeated id keeps its first index
        const Str gk = str_at(in->group_key.bytes, in->group_key.off, t);
        int32_t gid = -1;
        if (gk.n > 0) {
          gid = groups.get_or_put(gk, in->group_key.bytes, in->group_key.off, t, ng, &ins);
          if (ins) { ng++; grp_max_by_distro[size_t(d)].push_back(in->group_max_hosts[t]); grp_first_by_distro[size_t(d)].push_back(t); }
          else if (grp_max_by_distro[size_t(d)][size_t(gid)] != in->group_max_hosts[t]) { int64_t none = -1; bad_row.compare_exchange_strong(none, t); }
        }
        out->group_id[t] = gid;
        const int32_t vid = versions.get_or_put(str_at(in->version.bytes, in->version.off, t), in->version.bytes, in->version.off, t, nv, &ins);
        if (ins) nv++;
        out->version_id[t] = vid;
      }
      out->n_versions[d] = nv;
      n_groups[size_t(d)] = ng;
      std::vector<int32_t>& ed = edge_by_distro[size_t(d)];
      for (int64_t t = a; t < b; t++) {
        int64_t kept = 0;
        const int64_t e0 = in->dep_off[t], e1 = in->dep_off[t + 1];
        if (e0 < 0 || e1 < e0 || e1 > E) { bad_dep.store(true); return; }
        for (int64_t e = e0; e < e1; e++) {
          const int32_t j = ids.find(str_at(in->dep_id.bytes, in->dep_id.off, e), in->id.bytes, in->id.off);
          if (j >= 0) { ed.push_back(j); kept++; }
        }
        out->dep_off[t + 1] = kept;  // counts for now; scanned below
      }
      n_edges[size_t(d)] = int64_t(ed.size());
    }
  };
  std::vector<std::thread> pool;
  for (int k = 1; k < nt; k++) pool.emplace_back(work);
  work();
  for (std::thread& th : pool) th.join();
  if (bad_dep.load() || (T > 0 && in->dep_off[0] != 0)) return check_offsets(in->dep_off, T, -1, "evg_intern_columns", "dep_off");
  if (bad_row.load() >= 0) return fail(EVG_ERR_INVALID, "task group of row %lld: TaskGroupMaxHosts differs between members", (long long)bad_row.load());
  // offsets, then the per-distro pieces move to their places
  out->group_off[0] = 0;
  for (int32_t d = 0; d < D; d++) out->group_off[d + 1] = out->group_off[d] + n_groups[size_t(d)];
  if (T > 0) {
    out->dep_off[0] = 0;
    for (int64_t t = 0; t < T; t++) out->dep_off[t + 1] += out->dep_off[t];
  }
  for (int32_t d = 0; d < D; d++) {
    const int64_t g0 = out->group_off[d];
    for (size_t k = 0; k < grp_max_by_distro[size_t(d)].size(); k++) { out->group_max_hosts[g0 + int64_t(k)] = grp_max_by_distro[size_t(d)][k]; out->group_first[g0 + int64_t(k)] = grp_first_by_distro[size_t(d)][k]; }
    if (!edge_by_distro[size_t(d)].empty()) memcpy(out->dep_idx + out->dep_off[in->task_off[d]], edge_by_distro[size_t(d)].data(), sizeof(int32_t) * edge_by_distro[size_t(d)].size());
  }
  return EVG_OK;
}

int evg_prioritize_legacy_batch(evg_ctx* c, const evg_legacy_soa* in, const int64_t* task_off, const uint8_t* list_mode,
                                int32_t n_distros, int32_t* order, int64_t* count, int32_t* status) {
  ENTER(c, "evg_prioritize_legacy_batch");
  if (!in) return fail(EVG_ERR_INVALID, "evg_prioritize_legacy_batch: null argument");
  const int64_t T = in->n_tasks;
  const int32_t D = n_distros;
  if (T < 0 || D < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (D == 0) return T == 0 ? EVG_OK : fail(EVG_ERR_INVALID, "tasks without distros");
  if (!task_off || !list_mode || !count || !status || (T > 0 && !order)) return fail(EVG_ERR_INVALID, "null argument");
  if (T > 0 && (!in->priority || !in->ingest_ns || !in->expected_ns || !in->num_dependents || !in->revision_order || !in->project_id ||
                !in->tg_rank || !in->tg_pair_id || !in->task_group_order || !in->presort_rank || !in->flags))
    return fail(EVG_ERR_INVALID, "null task column");
  const int rc = check_offsets(task_off, D, T, who, "task_off");
  if (rc != EVG_OK) return rc;
  int64_t max_n = 0;
  for (int32_t d = 0; d < D; d++) max_n = std::max(max_n, task_off[d + 1] - task_off[d]);
  int64_t max_gs = 0;  // the longest distro with a GO_STABLE list: a bound on that list's length
  for (int64_t k = 0; k < 3 * int64_t(D); k++) {
    if (list_mode[k] > EVG_LEGACY_MODE_GO_STABLE) return fail(EVG_ERR_INVALID, "unknown list mode %d", int(list_mode[k]));
    if (list_mode[k] == EVG_LEGACY_MODE_GO_STABLE) max_gs = std::max(max_gs, task_off[k / 3 + 1] - task_off[k / 3]);
  }
  cudaStream_t s = c->stream;
  c->launches = 0;
  drop_tick(c);
  UP(s, c->tasks.exp, in->priority, T, int64_t);
  UP(s, c->tasks.qb, in->ingest_ns, T, int64_t);
  UP(s, c->tasks.wb, in->expected_ns, T, int64_t);
  UP(s, c->tasks.nd, in->num_dependents, T, int32_t);
  UP(s, c->tasks.prio, in->revision_order, T, int32_t);
  UP(s, c->tasks.vid, in->project_id, T, int32_t);
  UP(s, c->tasks.gid, in->tg_rank, T, int32_t);
  UP(s, c->b_rn0, in->tg_pair_id, T, int32_t);
  UP(s, c->tasks.tgo, in->task_group_order, T, int32_t);
  UP(s, c->b_rn1, in->presort_rank, T, int32_t);
  UP(s, c->tasks.flags, in->flags, T, uint32_t);
  UP(s, c->b_rn2, list_mode, 3 * int64_t(D), uint8_t);
  UP(s, c->b_taskoff, task_off, D + 1, int64_t);
  CK(c->b_order.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(c->b_rn3.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(c->b_rn4.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(c->b_rn5.ensure(sizeof(unsigned int) * 4 * size_t(D)));
  CK(c->b_rn6.ensure(sizeof(int64_t) * size_t(D)));
  CK(c->b_status.ensure(sizeof(int32_t) * size_t(D + 1)));
  CK(cudaMemsetAsync(c->b_rn5.p, 0, sizeof(unsigned int) * 4 * size_t(D), s));
  DLegacy x;
  x.n = T; x.priority = c->tasks.exp.as<int64_t>(); x.ingest = c->tasks.qb.as<int64_t>(); x.expected = c->tasks.wb.as<int64_t>();
  x.numdep = c->tasks.nd.as<int32_t>(); x.revision = c->tasks.prio.as<int32_t>(); x.project = c->tasks.vid.as<int32_t>();
  x.tg_rank = c->tasks.gid.as<int32_t>(); x.tg_pair = c->b_rn0.as<int32_t>(); x.tgo = c->tasks.tgo.as<int32_t>();
  x.presort = c->b_rn1.as<int32_t>(); x.flags = c->tasks.flags.as<uint32_t>(); x.list_mode = c->b_rn2.as<uint8_t>();
  x.task_off = c->b_taskoff.as<int64_t>(); x.n_distros = D;
  int32_t* buf[2] = {c->b_rn3.as<int32_t>(), c->b_rn4.as<int32_t>()};
  int gs_err = 0;
  int* d_gs_err = nullptr;
  if (T > 0) {
    const unsigned int* counts = c->b_rn5.as<unsigned int>();
    launch(c, c->stream, k_legacy_init, grid_for(T, 256), 256, 0, x, buf[0], c->b_rn5.as<unsigned int>());
    int32_t* sorted = seg_merge_sort(c, c->stream, LegacyOrder{x}, x.task_off, D, T, max_n, buf);
    if (max_gs > 1) {  // sort.Stable on the GO_STABLE lists, now in presort order; the other buffer is the rotations' scratch
      int32_t* scratch = sorted == buf[0] ? buf[1] : buf[0];
      const auto waves_of = [](int64_t size) { return 64 - __builtin_clzll(uint64_t(size - 1)); };  // ceil(log2 size), size >= 2
      int64_t n_waves = 0;
      for (int64_t block = 20; block < max_gs; block *= 2) n_waves += waves_of(std::min(2 * block, max_gs));
      // [n_waves + 1] task counts, the error flag, then two task queues: a wave's calls own disjoint ranges of >= 2 tasks
      const int64_t cap = T / 2 + 1, head = (sizeof(unsigned int) * (n_waves + 2) + 15) / 16 * 16;
      CK(c->b_rn7.ensure(size_t(head) + 2 * sizeof(GsTask) * size_t(cap)));
      CK(cudaMemsetAsync(c->b_rn7.p, 0, size_t(head), s));
      unsigned int* n_tasks = c->b_rn7.as<unsigned int>();
      d_gs_err = reinterpret_cast<int*>(n_tasks + n_waves + 1);
      GsTask* queue[2] = {reinterpret_cast<GsTask*>(c->b_rn7.as<char>() + head), reinterpret_cast<GsTask*>(c->b_rn7.as<char>() + head) + cap};
      const unsigned int grid_cta = unsigned(std::min<int64_t>(cap, int64_t(c->num_sms) * 8)), grid_warp = unsigned(std::min<int64_t>((cap + 7) / 8, int64_t(c->num_sms) * 8));
      launch(c, s, k_gs_insertion, grid_for(T, 256), 256, 0, x, counts, sorted);
      int64_t w = 0;
      for (int64_t block = 20; block < max_gs; block *= 2) {
        const int64_t size = std::min(2 * block, max_gs), level_waves = waves_of(size);
        launch(c, s, k_gs_seed, grid_for(T, 256), 256, 0, x, counts, block, queue[w & 1], n_tasks + w);
        for (int64_t k = 0; k < level_waves; k++, w++) {
          const bool last = k == level_waves - 1;
          GsTask* out = last ? nullptr : queue[(w + 1) & 1];
          unsigned int* out_n = last ? nullptr : n_tasks + w + 1;
          if (((size - 1) >> k) + 1 > kGsWarpRotation)  // the wave's largest call: a CTA rotates it
            launch(c, s, k_gs_wave<256>, grid_cta, 256, 0, x, sorted, scratch, queue[w & 1], n_tasks + w, out, out_n, d_gs_err);
          else
            launch(c, s, k_gs_wave<32>, grid_warp, 256, 0, x, sorted, scratch, queue[w & 1], n_tasks + w, out, out_n, d_gs_err);
        }
      }
      CK(cudaMemcpyAsync(&gs_err, d_gs_err, sizeof(int), cudaMemcpyDeviceToHost, s));
    }
    launch(c, c->stream, k_legacy_interleave, grid_for(T, 256), 256, 0, x, sorted, c->b_rn5.as<unsigned int>(), c->b_order.as<int32_t>(),
           c->b_rn6.as<int64_t>(), c->b_status.as<int32_t>());
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(order, c->b_order.p, sizeof(int32_t) * size_t(T), cudaMemcpyDeviceToHost, s));
  }
  // distros without tasks never reach k_legacy_interleave's q == 0 thread
  std::vector<int64_t> cnt(size_t(D), 0);
  std::vector<int32_t> st(size_t(D), EVG_LEGACY_OK);
  if (T > 0) {
    CK(cudaMemcpyAsync(cnt.data(), c->b_rn6.p, sizeof(int64_t) * size_t(D), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(st.data(), c->b_status.p, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  if (gs_err) return fail(EVG_ERR_CUDA, "%s: a symMerge call outlived its level's wave bound", who);
  for (int32_t d = 0; d < D; d++) {
    const bool empty = task_off[d + 1] == task_off[d];
    count[d] = empty ? 0 : cnt[d];
    status[d] = empty ? EVG_LEGACY_OK : st[d];
  }
  return EVG_OK;
}

// Where dag_run's kernels write: d.sorted, (n_sorted, n_cycles, grouped) at 0, D+1, 2(D+1), the two merge-sort buffers,
// the groups' offsets (D+1, on the device) and the unit offsets.
struct DagBufs {
  int32_t* sorted;
  int32_t* stats;
  int32_t* buf[2];
  const int64_t* group_off;
  int32_t* unit_off;
};
// k_dag_topo, then the task-group buckets (k_dag_group_init / seg_merge_sort / k_dag_units) over x, and the results
// copied to the host.  item_off / group_off (D+1) are the host copies of x's offsets; max_n is the longest queue.
static int dag_run(evg_ctx* c, const DDag& x, const DagBufs& b, int64_t max_n, const int64_t* item_off, const int64_t* group_off,
                   int32_t* sorted, int32_t* n_sorted, int32_t* n_cycles, int32_t* unit_items, int32_t* unit_off,
                   const int32_t** d_unit_items = nullptr) {
  const int64_t N = x.n;
  const int32_t D = x.n_distros;
  const int64_t G = group_off[D];
  cudaStream_t s = c->stream;
  int32_t* d_nsorted = b.stats;
  int32_t* d_ncycles = d_nsorted + (D + 1);
  int32_t* d_grouped = d_ncycles + (D + 1);
  launch(c, c->stream, k_dag_topo, grid_for(int64_t(D) * 32, 64), 64, 0, x, b.sorted, d_nsorted, d_ncycles);
  std::vector<int32_t> grouped(size_t(D), 0);
  int32_t* items = b.buf[0];
  if (N > 0) {
    CK(cudaMemcpyAsync(sorted, b.sorted, sizeof(int32_t) * size_t(N), cudaMemcpyDeviceToHost, s));
    // every item has a group or not: "no ungrouped item" leaves grouped[d] at the distro's length
    for (int32_t d = 0; d < D; d++) grouped[size_t(d)] = int32_t(item_off[d + 1] - item_off[d]);
    CK(cudaMemcpyAsync(d_grouped, grouped.data(), sizeof(int32_t) * size_t(D), cudaMemcpyHostToDevice, s));
    launch(c, c->stream, k_dag_group_init, grid_for(N, 256), 256, 0, x, b.buf[0]);
    items = seg_merge_sort(c, c->stream, DagGroupOrder{x}, x.item_off, D, N, max_n, b.buf);
    launch(c, c->stream, k_dag_units, grid_for(N, 256), 256, 0, x, items, b.group_off, b.unit_off, d_grouped);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(unit_items, items, sizeof(int32_t) * size_t(N), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(unit_off, b.unit_off, sizeof(int32_t) * size_t(G + D), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(grouped.data(), d_grouped, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(n_sorted, d_nsorted, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(n_cycles, d_ncycles, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  for (int32_t d = 0; d < D; d++) unit_off[group_off[d + 1] + d] = grouped[size_t(d)];  // the closing entry of each distro
  if (d_unit_items) *d_unit_items = items;
  return EVG_OK;
}

int evg_dag_rebuild_batch(evg_ctx* c, const evg_dag_in* in, const int64_t* item_off, const int64_t* group_off, int32_t n_distros,
                          int32_t* sorted, int32_t* n_sorted, int32_t* n_cycles, int32_t* unit_items, int32_t* unit_off) {
  ENTER(c, "evg_dag_rebuild_batch");
  if (!in) return fail(EVG_ERR_INVALID, "evg_dag_rebuild_batch: null argument");
  const int64_t N = in->n_items, E = in->n_deps;
  const int32_t D = n_distros;
  if (N < 0 || E < 0 || D < 0) return fail(EVG_ERR_INVALID, "negative sizes");
  if (D == 0) return N == 0 ? EVG_OK : fail(EVG_ERR_INVALID, "items without distros");
  if (!item_off || !group_off || !n_sorted || !n_cycles || !unit_off || (N > 0 && (!sorted || !unit_items))) return fail(EVG_ERR_INVALID, "null argument");
  if (N > 0 && (!in->dep_off || !in->group_id || !in->group_index)) return fail(EVG_ERR_INVALID, "null item column");
  if (E > 0 && !in->dep_item) return fail(EVG_ERR_INVALID, "null dep_item");
  int rc = check_offsets(item_off, D, N, who, "item_off");
  if (rc == EVG_OK) rc = check_offsets(group_off, D, -1, who, "group_off");
  if (rc == EVG_OK && N > 0) rc = check_offsets(in->dep_off, N, E, who, "dep_off");
  if (rc != EVG_OK) return rc;
  int64_t max_n = 0;
  for (int32_t d = 0; d < D; d++) max_n = std::max(max_n, item_off[d + 1] - item_off[d]);
  if (max_n >= (int64_t(1) << 31) - 1) return fail(EVG_ERR_INVALID, "a queue exceeds 2^31 items");
  const int64_t G = group_off[D];
  cudaStream_t s = c->stream;
  c->launches = 0;
  drop_tick(c);
  UP(s, c->b_taskoff, item_off, D + 1, int64_t);
  UP(s, c->b_groupoff, group_off, D + 1, int64_t);
  UP(s, c->b_depoff, in->dep_off, N + 1, int64_t);
  UP(s, c->b_depidx, in->dep_item, E, int32_t);
  UP(s, c->tasks.gid, in->group_id, N, int32_t);
  UP(s, c->tasks.tgo, in->group_index, N, int32_t);
  DevBuf* scratch[] = {&c->tasks.prio, &c->tasks.nd, &c->tasks.vid, &c->tasks.flags, &c->b_rn0, &c->b_rn1, &c->b_rn2, &c->b_rn3, &c->b_rn4};
  for (DevBuf* b : scratch) CK(b->ensure(sizeof(int32_t) * size_t(N + D + 1)));
  CK(c->b_rn5.ensure(sizeof(int32_t) * size_t(E + 1)));
  CK(c->b_hasdep.ensure(size_t(N) + 16));
  CK(c->b_order.ensure(sizeof(int32_t) * size_t(N + 1)));
  CK(c->b_rn6.ensure(sizeof(int32_t) * 3 * size_t(D + 1)));
  CK(c->b_rn7.ensure(sizeof(int32_t) * size_t(G + D + 1)));
  DDag x;
  x.n = N; x.n_deps = E; x.n_distros = D;
  x.item_off = c->b_taskoff.as<int64_t>(); x.dep_off = c->b_depoff.as<int64_t>(); x.dep_item = c->b_depidx.as<int32_t>();
  x.group_id = c->tasks.gid.as<int32_t>(); x.group_index = c->tasks.tgo.as<int32_t>();
  x.succ_off = c->tasks.prio.as<int32_t>(); x.succ = c->b_rn5.as<int32_t>(); x.index = c->tasks.nd.as<int32_t>(); x.low = c->tasks.vid.as<int32_t>();
  x.stack = c->tasks.flags.as<int32_t>(); x.cs_node = c->b_rn0.as<int32_t>(); x.cs_pos = c->b_rn1.as<int32_t>(); x.emit = c->b_rn2.as<int32_t>();
  x.on_stack = c->b_hasdep.as<uint8_t>();
  DagBufs b{c->b_order.as<int32_t>(), c->b_rn6.as<int32_t>(), {c->b_rn3.as<int32_t>(), c->b_rn4.as<int32_t>()}, c->b_groupoff.as<int64_t>(),
            c->b_rn7.as<int32_t>()};
  return dag_run(c, x, b, max_n, item_off, group_off, sorted, n_sorted, n_cycles, unit_items, unit_off);
}

// ---- FindNextTask over dispatchers on the device (evg_next.cuh) ----

// The tables derived from the dispatchers x describes (each unit's maxHosts) and their state: `st` (host) or, NULL, the
// state a rebuild leaves.  Fills x's derived and state pointers.
static int next_reset(evg_ctx* c, DNext& x, int32_t D, int64_t G, const evg_next_state* st) {
  auto& q = c->nx;
  cudaStream_t s = c->stream;
  const int64_t N = x.n;
  CK(q.verdict.ensure(sizeof(uint16_t) * size_t(N + 1)));
  CK(q.bits.ensure(size_t(N + 1)));
  for (DevBuf* b : {&q.gfirst, &q.unit_max, &q.running}) CK(b->ensure(sizeof(int32_t) * size_t(G + 1)));
  for (DevBuf* b : {&q.deleted, &q.inert}) CK(b->ensure(size_t(G + 1)));
  x.gfirst = q.gfirst.as<int32_t>(); x.unit_max = q.unit_max.as<int32_t>(); x.verdict = q.verdict.as<uint16_t>();
  x.bits = q.bits.as<uint8_t>(); x.deleted = q.deleted.as<uint8_t>(); x.running = q.running.as<int32_t>(); x.inert = q.inert.as<uint8_t>();
  if (st && st->item_bits && N > 0) CK(cudaMemcpyAsync(x.bits, st->item_bits, size_t(N), cudaMemcpyHostToDevice, s));
  else CK(cudaMemsetAsync(x.bits, 0, size_t(N + 1), s));
  if (st && st->group_deleted && G > 0) CK(cudaMemcpyAsync(x.deleted, st->group_deleted, size_t(G), cudaMemcpyHostToDevice, s));
  else CK(cudaMemsetAsync(x.deleted, 0, size_t(G + 1), s));
  if (st && st->group_running && G > 0) CK(cudaMemcpyAsync(x.running, st->group_running, sizeof(int32_t) * size_t(G), cudaMemcpyHostToDevice, s));
  else CK(cudaMemsetAsync(x.running, 0, sizeof(int32_t) * size_t(G + 1), s));
  if (G > 0) {
    CK(cudaMemsetAsync(x.gfirst, 0x7F, sizeof(int32_t) * size_t(G), s));
    CK(cudaMemsetAsync(x.unit_max, 0, sizeof(int32_t) * size_t(G), s));
    launch(c, s, k_next_first, grid_for(N, 256), 256, 0, x, D);
    launch(c, s, k_next_unit_max, grid_for(N, 256), 256, 0, x, D);
    CK(cudaGetLastError());
  }
  return EVG_OK;
}

// evg_rebuild_dispatchers' last step: the dispatchers in c->dp become the ones evg_find_next_tasks serves.  GroupMaxHosts
// and DependenciesMet of every item are gathered from the tick now, so that later changes to the tick do not reach them.
static int next_adopt(evg_ctx* c, const int32_t* d_unit_items, const evg_dispatch_out* out) {
  auto& q = c->nx;
  auto& p = c->dp;
  const int32_t D = c->Dn;
  q.h_item_off.assign(out->item_off, out->item_off + D + 1);
  q.h_group_off.assign(out->group_off, out->group_off + D + 1);
  const int64_t N = out->item_off[D], G = out->group_off[D];
  DNext x{};
  x.n = N;
  if (N > 0) {
    cudaStream_t s = c->stream;
    CK(q.gmh.ensure(sizeof(int32_t) * size_t(N)));
    CK(q.deps_met.ensure(size_t(N)));
    int32_t* stats = p.stats.as<int32_t>();
    launch(c, s, k_next_gather, grid_for(N, 256), 256, 0, D, N, p.item_off.as<int64_t>(), c->b_taskoff.as<int64_t>(), c->b_groupoff.as<int64_t>(),
           p.row.as<int32_t>(), c->tasks.gid.as<int32_t>(), c->b_gmax.as<int32_t>(), c->tasks.flags.as<uint32_t>(), q.gmh.as<int32_t>(),
           q.deps_met.as<uint8_t>());
    launch(c, s, k_next_close, grid_for(D, 256), 256, 0, D, p.group_off.as<int64_t>(), stats + 2 * (D + 1), p.unit_off.as<int32_t>());
    x.item_off = p.item_off.as<int64_t>(); x.group_off = p.group_off.as<int64_t>(); x.sorted = p.sorted.as<int32_t>();
    x.n_sorted = stats; x.unit_items = d_unit_items; x.unit_off = p.unit_off.as<int32_t>(); x.group_id = p.group_id.as<int32_t>();
    x.gmh = q.gmh.as<int32_t>(); x.deps_met = q.deps_met.as<uint8_t>();
    if (const int rc = next_reset(c, x, D, G, nullptr); rc != EVG_OK) return rc;
    CK(cudaStreamSynchronize(s));
  }
  q.x = x;
  c->tick.dispatchers = true;
  return EVG_OK;
}

// What a serving call checks of its snapshot, requests and outputs against the dispatchers' offsets (host copies).
static int next_check(const char* who, const int64_t* item_off, const int64_t* group_off, int32_t D, const evg_next_db* db,
                      const evg_next_req* req, const evg_next_out* out) {
  if (!db || !req || !out) return fail(EVG_ERR_INVALID, "%s: null argument", who);
  const int64_t N = item_off[D], G = group_off[D], R = req->n_requests;
  if (db->n_items != N || db->n_groups != G)
    return fail(EVG_ERR_INVALID, "%s: the snapshot has %lld items and %lld groups, the dispatchers %lld and %lld", who, (long long)db->n_items,
                (long long)db->n_groups, (long long)N, (long long)G);
  if (R < 0) return fail(EVG_ERR_INVALID, "%s: negative n_requests", who);
  if (!req->req_off) return fail(EVG_ERR_INVALID, "%s: null req_off", who);
  if (const int rc = check_offsets(req->req_off, D, R, who, "req_off"); rc != EVG_OK) return rc;
  if (R > 0 && (!req->group || !req->ami_updated_ns || !out->item || !out->outcome)) return fail(EVG_ERR_INVALID, "%s: null request column or output", who);
  if ((N > 0 && (!db->flags || !db->est_generated || !db->ingest_ns)) || (G > 0 && !db->running_hosts))
    return fail(EVG_ERR_INVALID, "%s: null snapshot column", who);
  if (db->pending_generate < -1 || db->num_large_parser < -1)
    return fail(EVG_ERR_INVALID, "%s: pending_generate / num_large_parser below -1", who);
  for (int64_t j = 0; j < N; j++)
    if (db->est_generated[j] < 0) return fail(EVG_ERR_INVALID, "%s: est_generated[%lld] is negative", who, (long long)j);
  for (int64_t g = 0; g < G; g++)
    if (db->running_hosts[g] < -1) return fail(EVG_ERR_INVALID, "%s: running_hosts[%lld] is below -1", who, (long long)g);
  for (int32_t d = 0; d < D; d++) {
    const int64_t ng = group_off[d + 1] - group_off[d];
    for (int64_t r = req->req_off[d]; r < req->req_off[d + 1]; r++)
      if (req->group[r] < -1 || req->group[r] >= ng)
        return fail(EVG_ERR_INVALID, "%s: request %lld asks for group %d of distro %d, which has %lld", who, (long long)r, req->group[r], d, (long long)ng);
  }
  return EVG_OK;
}

// One call's snapshot and requests (checked) staged, k_next_verdict over the items, k_next_serve over the distros that
// have requests, and the rows copied out.
static int next_serve(evg_ctx* c, const DNext& x, const int64_t* item_off, const int64_t* group_off, int32_t D, const evg_next_db* db,
                      const evg_next_req* req, evg_next_out* out) {
  auto& q = c->nx;
  cudaStream_t s = c->stream;
  const int64_t N = item_off[D], G = group_off[D], R = req->n_requests;
  if (R == 0) return EVG_OK;
  if (N == 0) {  // every queue is empty (no dispatcher buffers exist): each walk ends at once (:468)
    for (int64_t r = 0; r < R; r++) { out->item[r] = -1; out->outcome[r] = EVG_NEXT_NONE; }
    return EVG_OK;
  }
  std::vector<int32_t> list;
  for (int32_t d = 0; d < D; d++)
    if (req->req_off[d + 1] > req->req_off[d]) list.push_back(d);
  UP(s, q.flags, db->flags, N, uint8_t);
  UP(s, q.est, db->est_generated, N, int32_t);
  UP(s, q.ingest, db->ingest_ns, N, int64_t);
  UP(s, q.running_db, db->running_hosts, G, int32_t);
  UP(s, q.req_off, req->req_off, D + 1, int64_t);
  UP(s, q.req_group, req->group, R, int32_t);
  UP(s, q.req_ami, req->ami_updated_ns, R, int64_t);
  UP(s, q.list, list.data(), int64_t(list.size()), int32_t);
  CK(q.out_item.ensure(sizeof(int32_t) * size_t(R)));
  CK(q.out_outcome.ensure(sizeof(int32_t) * size_t(R)));
  CK(cudaMemsetAsync(x.inert, 0, size_t(G + 1), s));
  DNextDb B{q.flags.as<uint8_t>(), q.est.as<int32_t>(), db->generate_limit, db->pending_generate, db->max_large_parser, db->num_large_parser};
  launch(c, s, k_next_verdict, grid_for(N, 256), 256, 0, x, B);
  DNextReq Q{q.list.as<int32_t>(), int32_t(list.size()), q.req_off.as<int64_t>(), q.req_group.as<int32_t>(), q.req_ami.as<int64_t>(),
             q.ingest.as<int64_t>(), q.running_db.as<int32_t>(), q.out_item.as<int32_t>(), q.out_outcome.as<int32_t>()};
  launch(c, s, k_next_serve, grid_for(int64_t(list.size()) * 32, 128), 128, 0, x, Q);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out->item, q.out_item.p, sizeof(int32_t) * size_t(R), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->outcome, q.out_outcome.p, sizeof(int32_t) * size_t(R), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

static int next_download_state(evg_ctx* c, const DNext& x, int64_t G, const evg_next_state* st) {
  cudaStream_t s = c->stream;
  if (st->item_bits && x.n > 0) CK(cudaMemcpyAsync(st->item_bits, x.bits, size_t(x.n), cudaMemcpyDeviceToHost, s));
  if (st->group_deleted && G > 0) CK(cudaMemcpyAsync(st->group_deleted, x.deleted, size_t(G), cudaMemcpyDeviceToHost, s));
  if (st->group_running && G > 0) CK(cudaMemcpyAsync(st->group_running, x.running, sizeof(int32_t) * size_t(G), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

int evg_find_next_tasks(evg_ctx* c, const evg_next_db* db, const evg_next_req* req, evg_next_out* out) {
  ENTER(c, "evg_find_next_tasks");
  int rc;
  if ((rc = need_tick(c, who, Need::kTick)) != EVG_OK || (rc = need_tick(c, who, Need::kDispatchers)) != EVG_OK) return rc;
  auto& q = c->nx;
  const int32_t D = c->Dn;
  if ((rc = next_check(who, q.h_item_off.data(), q.h_group_off.data(), D, db, req, out)) != EVG_OK) return rc;
  c->launches = 0;
  return next_serve(c, q.x, q.h_item_off.data(), q.h_group_off.data(), D, db, req, out);
}

int evg_download_dispatch_state(evg_ctx* c, evg_next_state* state) {
  ENTER(c, "evg_download_dispatch_state");
  if (!state) return fail(EVG_ERR_INVALID, "evg_download_dispatch_state: null argument");
  int rc;
  if ((rc = need_tick(c, who, Need::kTick)) != EVG_OK || (rc = need_tick(c, who, Need::kDispatchers)) != EVG_OK) return rc;
  return next_download_state(c, c->nx.x, c->nx.h_group_off[size_t(c->Dn)], state);
}

int evg_find_next_batch(evg_ctx* c, const evg_next_dispatchers* disp, const evg_next_db* db, const evg_next_req* req,
                        const evg_next_state* state_in, evg_next_state* state_out, evg_next_out* out) {
  ENTER(c, "evg_find_next_batch");
  if (!disp) return fail(EVG_ERR_INVALID, "evg_find_next_batch: null argument");
  const int32_t D = disp->n_distros;
  if (D < 0) return fail(EVG_ERR_INVALID, "evg_find_next_batch: negative n_distros");
  if (!disp->item_off || !disp->group_off) return fail(EVG_ERR_INVALID, "evg_find_next_batch: null offsets");
  int rc = check_offsets(disp->item_off, D, -1, who, "item_off");
  if (rc == EVG_OK) rc = check_offsets(disp->group_off, D, -1, who, "group_off");
  if (rc != EVG_OK) return rc;
  const int64_t N = disp->item_off[D], G = disp->group_off[D];
  if ((D > 0 && (!disp->n_sorted || !disp->unit_off)) ||
      (N > 0 && (!disp->sorted || !disp->unit_items || !disp->group_id || !disp->group_max_hosts || !disp->dependencies_met)))
    return fail(EVG_ERR_INVALID, "evg_find_next_batch: null dispatcher column");
  // the kernels index with these: every entry inside its distro
  for (int32_t d = 0; d < D; d++) {
    const int64_t b = disp->item_off[d], n = disp->item_off[d + 1] - b, g0 = disp->group_off[d], ng = disp->group_off[d + 1] - g0;
    bool ok = n < (int64_t(1) << 31) - 1 && ng <= n && disp->n_sorted[d] >= 0 && disp->n_sorted[d] <= n;
    for (int64_t k = 0; ok && k < n; k++)
      ok = disp->sorted[b + k] >= -2 && disp->sorted[b + k] < n && disp->group_id[b + k] >= -1 && disp->group_id[b + k] < ng &&
           disp->unit_items[b + k] >= 0 && disp->unit_items[b + k] < n;
    const int32_t* uo = disp->unit_off + g0 + d;
    for (int64_t g = 0; ok && g < ng; g++) ok = uo[g] >= 0 && uo[g] <= uo[g + 1] && uo[g + 1] <= n;
    if (!ok) return fail(EVG_ERR_INVALID, "evg_find_next_batch: distro %d's dispatcher holds an entry outside the distro", d);
  }
  if ((rc = next_check(who, disp->item_off, disp->group_off, D, db, req, out)) != EVG_OK) return rc;
  c->launches = 0;
  drop_tick(c);  // the dispatcher buffers below are the ones a chained evg_find_next_tasks serves from
  auto& q = c->nx;
  cudaStream_t s = c->stream;
  UP(s, q.item_off, disp->item_off, D + 1, int64_t);
  UP(s, q.group_off, disp->group_off, D + 1, int64_t);
  UP(s, q.sorted, disp->sorted, N, int32_t);
  UP(s, q.n_sorted, disp->n_sorted, D, int32_t);
  UP(s, q.unit_items, disp->unit_items, N, int32_t);
  UP(s, q.unit_off, disp->unit_off, G + D, int32_t);
  UP(s, q.group_id, disp->group_id, N, int32_t);
  UP(s, q.gmh, disp->group_max_hosts, N, int32_t);
  UP(s, q.deps_met, disp->dependencies_met, N, uint8_t);
  DNext x{};
  x.n = N;
  x.item_off = q.item_off.as<int64_t>(); x.group_off = q.group_off.as<int64_t>(); x.sorted = q.sorted.as<int32_t>();
  x.n_sorted = q.n_sorted.as<int32_t>(); x.unit_items = q.unit_items.as<int32_t>(); x.unit_off = q.unit_off.as<int32_t>();
  x.group_id = q.group_id.as<int32_t>(); x.gmh = q.gmh.as<int32_t>(); x.deps_met = q.deps_met.as<uint8_t>();
  if ((rc = next_reset(c, x, D, G, state_in)) != EVG_OK) return rc;
  if ((rc = next_serve(c, x, disp->item_off, disp->group_off, D, db, req, out)) != EVG_OK) return rc;
  return state_out ? next_download_state(c, x, G, state_out) : EVG_OK;
}

// The persisted queue of every distro of the resident tick as a DAG input (evg_rebuild_dispatchers).  Item j of distro d
// is rank r = j - item_off[d], the task order[task_off[d] + r].
struct DDisp {
  int32_t D;
  int64_t n;                   // items
  const int64_t* task_off;     // [D+1] resident
  const int64_t* group_off;    // [D+1] resident group slots
  const int64_t* item_off;     // [D+1]
  const int32_t* order;        // the resident rank order (distro-local tasks)
  const int32_t* gid;          // resident group slot ids
  const int32_t* tgo;          // resident TaskGroupOrder
  const int64_t* dep_off;      // resident edges; NULL when the tick has none
  const int32_t* dep_idx;
  int32_t* rank_of;            // [T]: rank of a task below the cap, -1 otherwise (set to -1 before k_dp_gather)
  int32_t* row;                // [n]: distro-local task of an item, -1 for an order entry outside the distro
  int32_t* first;              // [G]: first rank of each group slot (INT32_MAX-like before k_dp_gather: never seen)
};
// per item: its task, rank_of, GroupIndex, group slot, edge count, and the slot's first rank
__global__ void __launch_bounds__(256) k_dp_gather(DDisp X, int32_t* __restrict__ gslot_of, int32_t* __restrict__ gindex, int32_t* __restrict__ cnt) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(X.item_off, X.D, j, X.n);
  if (d < 0) return;
  const int64_t base = X.task_off[d];
  const int32_t r = int32_t(j - X.item_off[d]);
  const int32_t i = X.order[base + r];
  if (i < 0 || i >= X.task_off[d + 1] - base) { X.row[j] = -1; gslot_of[j] = -1; gindex[j] = 0; cnt[j] = 0; return; }
  const int64_t t = base + i;
  X.row[j] = i;
  X.rank_of[t] = r;
  gindex[j] = X.tgo[t];
  const int32_t g = X.gid[t];
  gslot_of[j] = g;
  if (g >= 0) atomicMin(X.first + X.group_off[d] + g, r);
  cnt[j] = X.dep_off ? int32_t(X.dep_off[t + 1] - X.dep_off[t]) : 0;
}
// per item: its edges as ranks (-1 past the cap), in the resident order; and the flag of the item that first holds its slot
__global__ void __launch_bounds__(256) k_dp_edges(DDisp X, const int64_t* __restrict__ e_off, int32_t* __restrict__ dep_item,
                                                  const int32_t* __restrict__ gslot_of, int32_t* __restrict__ flag) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(X.item_off, X.D, j, X.n);
  if (d < 0) return;
  const int32_t g = gslot_of[j];
  flag[j] = (g >= 0 && X.first[X.group_off[d] + g] == int32_t(j - X.item_off[d])) ? 1 : 0;
  const int32_t i = X.row[j];
  if (i < 0 || !X.dep_off) return;
  const int64_t base = X.task_off[d], t = base + i;
  int64_t w = e_off[j];
  for (int64_t e = X.dep_off[t]; e < X.dep_off[t + 1]; e++) dep_item[w++] = X.rank_of[base + X.dep_idx[e]];
}
// pos = exclusive scan of the flags: the dense id of an item's group is the position of its slot's first item within
// the distro; group_off[d] = pos[item_off[d]] (threads 0 .. D); group_slot[pos[j]] = the slot of a first item j
__global__ void __launch_bounds__(256) k_dp_groups(DDisp X, const int64_t* __restrict__ pos, const int32_t* __restrict__ gslot_of,
                                                   int32_t* __restrict__ group_id, int32_t* __restrict__ group_slot,
                                                   int64_t* __restrict__ group_off) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j <= X.D) group_off[j] = pos[X.item_off[j]];
  if (j >= X.n) return;
  const int d = find_distro(X.item_off, 0, X.D - 1, j);
  const int32_t g = gslot_of[j];
  if (g < 0) { group_id[j] = -1; return; }
  const int64_t head = X.item_off[d] + X.first[X.group_off[d] + g];
  group_id[j] = int32_t(pos[head] - pos[X.item_off[d]]);
  if (head == j) group_slot[pos[j]] = g;
}

int evg_rebuild_dispatchers(evg_ctx* c, int32_t cap, int64_t items_capacity, int64_t groups_capacity, evg_dispatch_out* out) {
  ENTER(c, "evg_rebuild_dispatchers");
  if (!out) return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: null argument");
  if (const int rc = need_tick(c, who, Need::kTick); rc != EVG_OK) return rc;
  if (cap < 0) return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: negative cap");
  if (cap == 0) cap = EVG_PERSISTED_QUEUE_CAP;
  if (!out->item_off || !out->n_sorted || !out->n_cycles || !out->group_off || !out->unit_off)
    return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: null output");
  const int32_t D = c->Dn;
  int64_t* item_off = out->item_off;
  item_off[0] = 0;
  int64_t max_n = 0, g_need = 0;
  for (int32_t d = 0; d < D; d++) {
    const int64_t n = std::min<int64_t>(c->h_taskoff[d + 1] - c->h_taskoff[d], cap);
    item_off[d + 1] = item_off[d] + n;
    max_n = std::max(max_n, n);
    g_need += std::min(c->h_groupoff[d + 1] - c->h_groupoff[d], n);
  }
  const int64_t N = item_off[D];
  if (N > items_capacity || g_need > groups_capacity)
    return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: %lld items and %lld groups needed, capacities %lld and %lld", (long long)N,
                (long long)g_need, (long long)items_capacity, (long long)groups_capacity);
  if (N > 0 && (!out->sorted || !out->unit_items)) return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: null item output");
  if (g_need > 0 && !out->group_slot) return fail(EVG_ERR_INVALID, "evg_rebuild_dispatchers: null group_slot");
  c->launches = 0;
  c->tick.dispatchers = false;  // until the dispatchers below are built and their state reset
  if (N == 0) {  // every queue is empty: no items, no groups
    for (int32_t d = 0; d < D; d++) out->n_sorted[d] = out->n_cycles[d] = out->unit_off[d] = 0;
    for (int32_t d = 0; d <= D; d++) out->group_off[d] = 0;
    return next_adopt(c, nullptr, out);
  }
  cudaStream_t s = c->stream;
  auto& p = c->dp;
  const int64_t T = c->T, E = c->E, G = c->G;
  UP(s, p.item_off, item_off, D + 1, int64_t);
  CK(p.rank_of.ensure(sizeof(int32_t) * size_t(T + 1)));
  CK(p.first.ensure(sizeof(int32_t) * size_t(G + 1)));
  for (DevBuf* b : {&p.row, &p.gslot_of, &p.gindex, &p.cnt, &p.group_id, &p.index, &p.low, &p.stack, &p.cs_node, &p.cs_pos, &p.emit,
                    &p.sorted, &p.buf[0], &p.buf[1]})
    CK(b->ensure(sizeof(int32_t) * size_t(N + 1)));
  CK(p.on_stack.ensure(size_t(N) + 16));
  CK(p.dep_off.ensure(sizeof(int64_t) * size_t(N + 1)));
  CK(p.pos.ensure(sizeof(int64_t) * size_t(N + 1)));
  CK(p.dep_item.ensure(sizeof(int32_t) * size_t(E + 1)));  // the persisted items hold at most every resident edge
  CK(p.succ.ensure(sizeof(int32_t) * size_t(E + 1)));
  CK(p.succ_off.ensure(sizeof(int32_t) * size_t(N + D + 1)));
  CK(p.group_off.ensure(sizeof(int64_t) * size_t(D + 1)));
  CK(p.group_slot.ensure(sizeof(int32_t) * size_t(g_need + 1)));
  CK(p.unit_off.ensure(sizeof(int32_t) * size_t(g_need + D + 1)));
  CK(p.stats.ensure(sizeof(int32_t) * 3 * size_t(D + 1)));
  CK(cudaMemsetAsync(p.rank_of.p, 0xFF, sizeof(int32_t) * size_t(T), s));
  if (G > 0) CK(cudaMemsetAsync(p.first.p, 0x7F, sizeof(int32_t) * size_t(G), s));
  DDisp X;
  X.D = D; X.n = N;
  X.task_off = c->b_taskoff.as<int64_t>(); X.group_off = c->b_groupoff.as<int64_t>(); X.item_off = p.item_off.as<int64_t>();
  X.order = c->b_order.as<int32_t>(); X.gid = c->tasks.gid.as<int32_t>(); X.tgo = c->tasks.tgo.as<int32_t>();
  X.dep_off = E > 0 ? c->b_depoff.as<int64_t>() : nullptr; X.dep_idx = E > 0 ? c->b_depidx.as<int32_t>() : nullptr;
  X.rank_of = p.rank_of.as<int32_t>(); X.row = p.row.as<int32_t>(); X.first = p.first.as<int32_t>();
  int32_t* cnt = p.cnt.as<int32_t>();
  launch(c, c->stream, k_dp_gather, grid_for(N, 256), 256, 0, X, p.gslot_of.as<int32_t>(), p.gindex.as<int32_t>(), cnt);
  CK(scan_counts(c, cnt, N, p.dep_off.as<int64_t>()));
  launch(c, c->stream, k_dp_edges, grid_for(N, 256), 256, 0, X, p.dep_off.as<int64_t>(), p.dep_item.as<int32_t>(), p.gslot_of.as<int32_t>(), cnt);
  CK(scan_counts(c, cnt, N, p.pos.as<int64_t>()));
  launch(c, c->stream, k_dp_groups, grid_for(std::max<int64_t>(N, D + 1), 256), 256, 0, X, p.pos.as<int64_t>(), p.gslot_of.as<int32_t>(),
         p.group_id.as<int32_t>(), p.group_slot.as<int32_t>(), p.group_off.as<int64_t>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out->group_off, p.group_off.p, sizeof(int64_t) * size_t(D + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));  // group_off sizes the unit table and closes each distro's unit_off
  const int64_t G2 = out->group_off[D];
  if (G2 > 0) CK(cudaMemcpyAsync(out->group_slot, p.group_slot.p, sizeof(int32_t) * size_t(G2), cudaMemcpyDeviceToHost, s));
  DDag x;
  x.n = N; x.n_deps = E; x.n_distros = D;
  x.item_off = p.item_off.as<int64_t>(); x.dep_off = p.dep_off.as<int64_t>(); x.dep_item = p.dep_item.as<int32_t>();
  x.group_id = p.group_id.as<int32_t>(); x.group_index = p.gindex.as<int32_t>();
  x.succ_off = p.succ_off.as<int32_t>(); x.succ = p.succ.as<int32_t>(); x.index = p.index.as<int32_t>(); x.low = p.low.as<int32_t>();
  x.stack = p.stack.as<int32_t>(); x.cs_node = p.cs_node.as<int32_t>(); x.cs_pos = p.cs_pos.as<int32_t>(); x.emit = p.emit.as<int32_t>();
  x.on_stack = p.on_stack.as<uint8_t>();
  DagBufs b{p.sorted.as<int32_t>(), p.stats.as<int32_t>(), {p.buf[0].as<int32_t>(), p.buf[1].as<int32_t>()}, p.group_off.as<int64_t>(),
            p.unit_off.as<int32_t>()};
  const int32_t* d_unit_items = nullptr;
  if (const int rc = dag_run(c, x, b, max_n, item_off, out->group_off, out->sorted, out->n_sorted, out->n_cycles, out->unit_items,
                             out->unit_off, &d_unit_items); rc != EVG_OK) return rc;
  return next_adopt(c, d_unit_items, out);
}

// The group sums of the job's report (units/host_allocator.go:271-280) over slots [g, g1) with stride `step`, in wrapping
// int64.  A single-task distro's CountFree / CountRequired stay 0: the reference never runs the allocator for it.
struct JobSums { uint64_t overdue, n_over, d_over, expected, free, required; };
__device__ __forceinline__ JobSums job_group_sums(const evg_group_info* __restrict__ gi, int64_t g, int64_t g1, int step, bool single) {
  JobSums s{0, 0, 0, 0, 0, 0};
  for (; g < g1; g += step) {
    const evg_group_info& x = gi[g];
    s.overdue += uint64_t(x.count_wait_over_threshold);
    s.n_over += uint64_t(x.count_duration_over_threshold);
    s.d_over += uint64_t(x.duration_over_threshold);
    s.expected += uint64_t(x.expected_duration);
    if (!single) { s.free += uint64_t(x.count_free); s.required += uint64_t(x.count_required); }
  }
  return s;
}

constexpr int64_t kHostJobWarpGroups = 16;  // k_host_job: a distro with more group slots has them summed by its warp
constexpr int64_t kMaxPossibleTime = int64_t(2532000) * 3600 * 1000000000;  // maxPossibleHours * time.Hour (:309)

// hostAllocatorJob.Run past the allocator (units/host_allocator.go:180-196, 253-337, 394-425), one thread per distro.
// A distro with few group slots sums them itself; the warp sums those of each distro with many, one distro at a time,
// all lanes striding over its slots (the k_alloc_groupless / k_alloc split).  Only reads the tick.
__global__ void __launch_bounds__(128) k_host_job(int32_t n_distros, const int64_t* __restrict__ group_off, const int64_t* __restrict__ host_off,
                                                  const evg_queue_info* __restrict__ qinfo, const evg_group_info* __restrict__ ginfo,
                                                  const evg_alloc_result* __restrict__ result, const int32_t* __restrict__ status,
                                                  const evg_alloc_cfg* __restrict__ acfg, const evg_host_job_cfg* __restrict__ cfg,
                                                  const int32_t* __restrict__ spawned, int64_t* __restrict__ n_hosts_out,
                                                  int64_t* __restrict__ n_free_out, int32_t* __restrict__ status_out,
                                                  evg_host_report* __restrict__ report) {
  const unsigned full = 0xffffffffu;
  const int d = int(blockIdx.x * blockDim.x + threadIdx.x), lane = int(threadIdx.x & 31);
  const bool in = d < n_distros;  // lanes past the end still take part in the warp's sums
  const int64_t g0 = in ? group_off[d] : 0, g1 = in ? group_off[d + 1] : 0;
  const evg_host_job_cfg jc = in ? cfg[d] : evg_host_job_cfg{0, 0, 0, 0, 0};
  const bool wide = g1 - g0 > kHostJobWarpGroups;
  JobSums s = job_group_sums(ginfo, g0, wide ? g0 : g1, 1, jc.single_task_distro != 0);
  for (unsigned todo = __ballot_sync(full, wide); todo; todo &= todo - 1u) {
    const int j = __ffs(todo) - 1;
    const int64_t a = __shfl_sync(full, g0, j), b = __shfl_sync(full, g1, j);
    const JobSums w = job_group_sums(ginfo, a + lane, b, 32, __shfl_sync(full, jc.single_task_distro, j) != 0);
    const JobSums r{uint64_t(warp_sum64(int64_t(w.overdue))), uint64_t(warp_sum64(int64_t(w.n_over))),
                    uint64_t(warp_sum64(int64_t(w.d_over))), uint64_t(warp_sum64(int64_t(w.expected))),
                    uint64_t(warp_sum64(int64_t(w.free))), uint64_t(warp_sum64(int64_t(w.required)))};
    if (lane == j) s = r;
  }
  if (!in) return;
  const evg_queue_info& q = qinfo[d];
  int64_t n_hosts, n_free;
  int32_t st = EVG_ALLOC_OK;
  if (jc.single_task_distro) {  // :182-184
    n_hosts = wsub(q.length_with_dependencies_met, jc.n_provisioning);
    n_free = 0;
  } else {  // :186-195
    const evg_alloc_result r = result[d];
    n_hosts = r.new_hosts;
    n_free = r.free_hosts;
    st = status[d];
  }
  evg_host_report o{};
  if (st == EVG_ALLOC_OK) {
    const int64_t n_spawned = spawned ? int64_t(spawned[d]) : (n_hosts > 0 ? n_hosts : 0);
    const int64_t sched = wsub(wsub(q.expected_duration, int64_t(s.expected)), wsub(q.duration_over_threshold, int64_t(s.d_over)));  // :283-287
    const int64_t over_no_groups = wsub(q.count_duration_over_threshold, int64_t(s.n_over));                                         // :289
    const int64_t spawned_standalone = wsub(n_spawned, int64_t(s.required));                                                        // :292
    const int64_t avail = wsub(wadd(wsub(n_free, int64_t(s.free)), spawned_standalone), over_no_groups);                            // :294
    int64_t tte = 0, tte_ns = 0;
    if (sched > 0) {  // :304-321
      const int64_t avail_ns = wsub(avail, spawned_standalone);
      tte = avail <= 0 ? kMaxPossibleTime : sched / avail;
      tte_ns = avail <= 0 || avail_ns <= 0 ? kMaxPossibleTime : sched / avail_ns;
    }
    const float thr = __ll2float_rn(q.max_duration_threshold);
    const float ratio = __fdiv_rn(__ll2float_rn(tte), thr), ratio_ns = __fdiv_rn(__ll2float_rn(tte_ns), thr);  // :324-326
    const evg_alloc_cfg ac = acfg[d];
    const int64_t n_up = host_off[d + 1] - host_off[d];
    if (jc.terminate_when_overallocated && ac.provider != EVG_PROVIDER_STATIC && ratio < 0.25f && n_up > 0 && !jc.hourly_billing) {
      // setTargetAndTerminate (:394-425); the float -> int conversion saturates
      const int64_t killable = ratio == 0.0f ? n_up : __float2ll_rz(__fmul_rn(__ll2float_rn(n_up), __fsub_rn(1.0f, ratio)));
      int64_t cap = ratio == 0.0f ? 0 : n_up - killable;
      if (cap < ac.minimum_hosts) cap = ac.minimum_hosts;
      o.killable_hosts = killable;
      o.new_cap_target = cap;
      o.drawdown = killable > 0;
    }
    o.time_to_empty_ns = tte;
    o.time_to_empty_no_spawns_ns = tte_ns;
    o.scheduled_duration_ns = sched;
    o.hosts_avail = avail;
    o.hosts_spawned = n_spawned;
    o.overdue_in_groups = int64_t(s.overdue);
    o.free_in_groups = int64_t(s.free);
    o.required_in_groups = int64_t(s.required);
    o.host_queue_ratio = ratio;
    o.no_spawns_ratio = ratio_ns;
  }
  n_hosts_out[d] = n_hosts;
  n_free_out[d] = n_free;
  status_out[d] = st;
  report[d] = o;
}

int evg_host_job(evg_ctx* c, const evg_host_job_cfg* cfg, const int32_t* spawned, evg_host_job_out* out) {
  ENTER(c, "evg_host_job");
  if (!cfg || !out || !out->n_hosts || !out->n_hosts_free || !out->status || !out->report)
    return fail(EVG_ERR_INVALID, "evg_host_job: null cfg or output");
  if (const int rc = need_tick(c, who, Need::kAllocated); rc != EVG_OK) return rc;
  const int32_t D = c->Dn;
  for (int32_t d = 0; d < D; d++)
    if (cfg[d].n_provisioning < 0) return fail(EVG_ERR_INVALID, "evg_host_job: cfg[%d].n_provisioning is negative", d);
  c->launches = 0;
  c->tick.host_job = false;  // until the reports below are written
  if (D == 0) return c->tick.host_job = true, EVG_OK;
  cudaStream_t s = c->stream;
  auto& h = c->hj;
  UP(s, h.cfg, cfg, D, evg_host_job_cfg);
  if (spawned) UP(s, h.spawned, spawned, D, int32_t);
  // outputs: the reports, then n_hosts, n_hosts_free and status
  CK(h.out.ensure((sizeof(evg_host_report) + 2 * sizeof(int64_t) + sizeof(int32_t)) * size_t(D)));
  evg_host_report* rep = h.out.as<evg_host_report>();
  int64_t* nh = reinterpret_cast<int64_t*>(rep + D);
  int64_t* nf = nh + D;
  int32_t* st = reinterpret_cast<int32_t*>(nf + D);
  launch(c, c->stream, k_host_job, grid_for(D, 128), 128, 0, D, c->b_groupoff.as<int64_t>(), c->b_hostoff.as<int64_t>(), c->b_qinfo.as<evg_queue_info>(),
         c->b_ginfo.as<evg_group_info>(), c->result_ptr(), c->b_status.as<int32_t>(), c->b_acfg.as<evg_alloc_cfg>(),
         h.cfg.as<evg_host_job_cfg>(), spawned ? h.spawned.as<int32_t>() : nullptr, nh, nf, st, rep);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out->report, rep, sizeof(evg_host_report) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->n_hosts, nh, sizeof(int64_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->n_hosts_free, nf, sizeof(int64_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->status, st, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));  // the caller's cfg / spawned arrays are free again and the outputs are written
  c->tick.host_job = true;
  return EVG_OK;
}

// ---- host termination: the drawdown job and the idle-host job over one idle-host table ----

constexpr int64_t kMaxTeardownGroup = 4 * kMinute;   // evergreen.MaxTeardownGroupThreshold (globals.go:348)
constexpr int64_t kAgentUnresponsive = 5 * kMinute;  // MaxAgentUnresponsiveInterval = MaxAgentMonitorUnresponsiveInterval (host.go:624, 634)
constexpr int64_t kWaitingForAgentCutoff = 10 * kMinute;  // idleWaitingForAgentCutoff (host_monitoring_idle_termination.go:24)

struct DIdleHosts {  // evg_idle_host_soa staged on the device
  const int64_t *creation, *start, *provision, *agent_start, *last_comm, *last_done, *teardown, *acceptable;
  const uint32_t* flags;
};

// The host predicates both jobs share, for a row without a running task, at the frozen `now`.
struct IdleHostRow {
  int64_t idle, comm, since_td;
  uint32_t f;
  bool tearing, td_exceeded;
  int32_t exempt;  // checkTerminationExemptions' outcome: an EVG_HT_* code, EVG_HT_NOT_CHECKED when none applies
};
__device__ __forceinline__ IdleHostRow idle_host_row(const DIdleHosts& h, int64_t i, int64_t now) {
  IdleHostRow r;
  r.f = h.flags[i];
  const int64_t td = h.teardown[i], lc = h.last_comm[i], ct = h.creation[i], st = h.start[i];
  r.tearing = td != EVG_TIME_ZERO;  // IsTearingDown (model/host/host.go:219-221)
  r.since_td = since(now, td);
  r.td_exceeded = r.since_td > kMaxTeardownGroup;  // TeardownTimeExceededMax (:2241-2243)
  if (r.tearing) r.idle = r.td_exceeded ? r.since_td : 0;  // IdleTime (:671-706)
  else if (r.f & EVG_IH_LAST_TASK) r.idle = since(now, h.last_done[i]);
  else if (r.f & EVG_IH_USER_DATA) r.idle = h.agent_start[i] > 0 ? since(now, h.agent_start[i]) : 0;  // After(Unix 0)
  else r.idle = (r.f & EVG_IH_STATUS_RUNNING) ? since(now, h.provision[i]) : 0;
  if (r.tearing) r.comm = 0;  // GetElapsedCommunicationTime (:2220-2238)
  else if (lc > ct) r.comm = since(now, lc);
  else if (st > ct) r.comm = since(now, st);
  else if (lc != EVG_TIME_ZERO) r.comm = since(now, lc);
  else r.comm = since(now, ct);
  const bool legacy = r.f & EVG_IH_LEGACY_BOOTSTRAP;  // IsWaitingForAgent (:2006-2026)
  const int64_t cutoff = now < kI64Min + kAgentUnresponsive ? kI64Min : now - kAgentUnresponsive;
  const bool waiting = (legacy && (r.f & EVG_IH_NEEDS_NEW_AGENT)) || (!legacy && (r.f & EVG_IH_NEEDS_NEW_AGENT_MONITOR)) ||
                       lc == EVG_TIME_ZERO || lc == 0 || lc < cutoff;
  // checkTerminationExemptions (units/host_monitoring_idle_termination.go:287-338) past its !IsEphemeral branch
  r.exempt = waiting && (r.comm < kWaitingForAgentCutoff || r.idle < kWaitingForAgentCutoff) ? EVG_HT_EXEMPT_AGENT
             : (r.f & EVG_IH_CLOUD_MANAGER_FAILED)                                          ? EVG_HT_ERR_CLOUD_MANAGER
             : (r.f & EVG_IH_PAYMENT_NOT_DUE)                                                ? EVG_HT_EXEMPT_PAYMENT
                                                                                             : EVG_HT_NOT_CHECKED;
  return r;
}

// The drawdown job's inputs for distro d: its NewCapTarget (EVG_NO_DRAWDOWN: no job) and LengthWithDependenciesMet,
// from the last evg_host_job's report and the tick's queue infos (chained, `rep` given) or from the caller's arrays.
struct DrawdownSrc {
  const evg_host_report* rep;
  const evg_queue_info* qinfo;
  const int64_t *cap, *qlen, *existing;
};
__device__ __forceinline__ int64_t dd_cap(const DrawdownSrc& s, int d) {
  return s.rep ? (s.rep[d].drawdown ? s.rep[d].new_cap_target : EVG_NO_DRAWDOWN) : s.cap[d];
}

__device__ __forceinline__ void put_verdict(evg_host_verdict* __restrict__ v, int64_t i, const IdleHostRow& r, int64_t thr, int32_t code) {
  evg_host_verdict o;
  o.idle_ns = r.idle; o.communication_ns = r.comm; o.threshold_ns = thr; o.since_teardown_ns = r.since_td;
  o.decision = code; o._reserved = 0;
  v[i] = o;
}

// checkAndDecommission (units/host_drawdown.go:127-159) for every row of a distro with a drawdown job, as if the target
// were not yet reached; decom[i] = 1 when the row would be decommissioned.  k_hd_cap applies the target.
__global__ void __launch_bounds__(256) k_hd_host(int64_t n, int32_t D, const int64_t* __restrict__ off, DIdleHosts h, DrawdownSrc s,
                                                 int64_t now, evg_host_verdict* __restrict__ verdict, int32_t* __restrict__ decom) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, i, n);
  if (d < 0) return;
  decom[i] = 0;
  if (dd_cap(s, d) == EVG_NO_DRAWDOWN) { verdict[i] = evg_host_verdict{}; return; }
  const IdleHostRow r = idle_host_row(h, i, now);
  int64_t thr = 0;
  int32_t code;
  if (r.exempt != EVG_HT_NOT_CHECKED) code = r.exempt;                       // :128-131
  else if (r.tearing && !r.td_exceeded) code = EVG_HT_KEPT;                  // :134-136
  else if (r.f & EVG_IH_TASK_LOOKUP_FAILED) code = EVG_HT_ERR_TASK_LOOKUP;   // :139-142
  else if (r.f & EVG_IH_SINGLE_HOST_TASK_GROUP) code = EVG_HT_KEPT;          // :143-145
  else {                                                                     // :147-158
    const int64_t qlen = s.rep ? s.qinfo[d].length_with_dependencies_met : s.qlen[d];
    thr = (r.f & EVG_IH_RUNNING_TASK_GROUP) ? 10 * kMinute : 5 * kSecond;
    if (h.last_done[i] != EVG_TIME_ZERO && qlen > 0) thr = h.acceptable[i];
    code = r.idle > thr ? EVG_HT_DECOMMISSION : EVG_HT_KEPT;
  }
  put_verdict(verdict, i, r, thr, code);
  decom[i] = code == EVG_HT_DECOMMISSION;
}

// The loop stops before any row once the target is <= 0 and the target drops only on a decommission (:93-97, :149-151):
// a row is checked iff fewer than `target` rows before it in its distro would be decommissioned (pos: their exclusive
// scan over the whole table).  Rows past that point get no decision.
__global__ void __launch_bounds__(256) k_hd_cap(int64_t n, int32_t D, const int64_t* __restrict__ off, DrawdownSrc s,
                                                const int64_t* __restrict__ pos, evg_host_verdict* __restrict__ verdict) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, i, n);
  if (d < 0) return;
  const int64_t cap = dd_cap(s, d);
  if (cap != EVG_NO_DRAWDOWN && pos[i] - pos[off[d]] >= wsub(s.existing[d], cap)) verdict[i] = evg_host_verdict{};
}

__global__ void __launch_bounds__(256) k_hd_distro(int32_t D, const int64_t* __restrict__ off, DrawdownSrc s, const int64_t* __restrict__ pos,
                                                   evg_drawdown_distro* __restrict__ out) {
  const int d = int(blockIdx.x * blockDim.x + threadIdx.x);
  if (d >= D) return;
  const int64_t cap = dd_cap(s, d);
  evg_drawdown_distro o{};
  if (cap != EVG_NO_DRAWDOWN) {
    o.ran = 1;
    o.target = wsub(s.existing[d], cap);  // :91
    const int64_t would = pos ? pos[off[d + 1]] - pos[off[d]] : 0;
    o.decommissioned = o.target <= 0 ? 0 : (would < o.target ? would : o.target);
  }
  out[d] = o;
}

// idleHostJob.Run's loop (units/host_monitoring_idle_termination.go:128-140), checkAndTerminateHost (:158-180),
// getIdleInfo (:194-226) and getTerminationReason (:258-283) per row; term[i] = 1 when the row is terminated.
__global__ void __launch_bounds__(256) k_idle_host(int64_t n, int32_t D, const int64_t* __restrict__ off, DIdleHosts h,
                                                   const evg_idle_cfg* __restrict__ cfg, int64_t now,
                                                   evg_host_verdict* __restrict__ verdict, int32_t* __restrict__ term) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(off, D, i, n);
  if (d < 0) return;
  term[i] = 0;
  const evg_idle_cfg c = cfg[d];
  const int64_t n_idle = off[d + 1] - off[d], room = c.running_hosts_count - c.minimum_hosts;
  const int64_t min_eval = room <= 0 ? 0 : (room < n_idle ? room : n_idle);  // getMinNumHostsToEvaluate (:143-156)
  const uint32_t f = h.flags[i];
  if (i - off[d] >= min_eval && !(f & EVG_IH_OUTDATED_AMI)) { verdict[i] = evg_host_verdict{}; return; }
  const IdleHostRow r = idle_host_row(h, i, now);
  int64_t thr = 0;
  int32_t code;
  if (r.exempt != EVG_HT_NOT_CHECKED) code = r.exempt;                      // :160-163
  else if (f & EVG_IH_TASK_LOOKUP_FAILED) code = EVG_HT_ERR_TASK_LOOKUP;    // :209-212
  else {
    const bool single = f & EVG_IH_SINGLE_HOST_TASK_GROUP;
    thr = single ? 5 * kMinute : (f & EVG_IH_RUNNING_TASK_GROUP) ? wadd(c.acceptable_idle_ns, c.acceptable_idle_ns) : c.acceptable_idle_ns;
    code = (f & EVG_IH_OUTDATED_AMI) && r.idle > 0 && !single ? EVG_HT_TERM_OUTDATED_AMI
           : r.comm >= thr && !r.tearing                       ? EVG_HT_TERM_COMMUNICATION
           : r.idle > 0 && r.idle >= thr                       ? EVG_HT_TERM_IDLE
           : r.since_td > kMaxTeardownGroup && r.tearing       ? EVG_HT_TERM_TEARDOWN
                                                               : EVG_HT_KEPT;
  }
  put_verdict(verdict, i, r, thr, code);
  term[i] = code >= EVG_HT_TERM_OUTDATED_AMI;
}

__global__ void __launch_bounds__(256) k_idle_distro(int32_t D, const int64_t* __restrict__ off, const evg_idle_cfg* __restrict__ cfg,
                                                     const int64_t* __restrict__ pos, evg_idle_distro* __restrict__ out) {
  const int d = int(blockIdx.x * blockDim.x + threadIdx.x);
  if (d >= D) return;
  const int64_t n_idle = off[d + 1] - off[d], room = cfg[d].running_hosts_count - cfg[d].minimum_hosts;
  evg_idle_distro o;
  o.min_evaluate = room <= 0 ? 0 : (room < n_idle ? room : n_idle);
  o.terminated = pos ? pos[off[d + 1]] - pos[off[d]] : 0;
  out[d] = o;
}

// The idle-host table and its offsets, checked before anything is staged or launched.
static int check_idle_hosts(const char* who, const evg_idle_host_soa* t, const int64_t* off) {
  if (!t || !off) return fail(EVG_ERR_INVALID, "%s: null host table or idle_off", who);
  if (t->n_hosts < 0 || t->n_distros < 0) return fail(EVG_ERR_INVALID, "%s: negative n_hosts or n_distros", who);
  if (t->n_hosts > 0 && (!t->creation_ns || !t->start_ns || !t->provision_ns || !t->agent_start_ns || !t->last_communication_ns ||
                         !t->last_task_completed_ns || !t->teardown_start_ns || !t->acceptable_idle_ns || !t->flags))
    return fail(EVG_ERR_INVALID, "%s: null host column", who);
  return check_offsets(off, t->n_distros, t->n_hosts, who, "idle_off");
}

// Stage the table's columns, its offsets and `per_distro_bytes` of per-distro input into ih, and size the outputs and
// the scan.  Returns the device view in `v`.
static int stage_idle_hosts(evg_ctx* c, const evg_idle_host_soa* t, const int64_t* off, const void* per_distro, size_t per_distro_bytes,
                            DIdleHosts* v) {
  auto& x = c->ih;
  const int64_t H = t->n_hosts;
  const int32_t D = t->n_distros;
  cudaStream_t s = c->stream;
  CK(x.cols.ensure((8 * sizeof(int64_t) + sizeof(uint32_t)) * size_t(H > 0 ? H : 1)));
  const int64_t* src[8] = {t->creation_ns, t->start_ns, t->provision_ns, t->agent_start_ns, t->last_communication_ns,
                           t->last_task_completed_ns, t->teardown_start_ns, t->acceptable_idle_ns};
  int64_t* col = x.cols.as<int64_t>();
  const int64_t* dcol[8];
  for (int k = 0; k < 8; k++) {
    dcol[k] = col + k * H;
    if (H > 0) CK(cudaMemcpyAsync(col + k * H, src[k], sizeof(int64_t) * size_t(H), cudaMemcpyHostToDevice, s));
  }
  uint32_t* flags = reinterpret_cast<uint32_t*>(col + 8 * H);
  if (H > 0) CK(cudaMemcpyAsync(flags, t->flags, sizeof(uint32_t) * size_t(H), cudaMemcpyHostToDevice, s));
  UP(s, x.off, off, D + 1, int64_t);
  CK(x.din.ensure(per_distro_bytes > 0 ? per_distro_bytes : 1));
  if (per_distro_bytes > 0) CK(cudaMemcpyAsync(x.din.p, per_distro, per_distro_bytes, cudaMemcpyHostToDevice, s));
  CK(x.verdict.ensure(sizeof(evg_host_verdict) * size_t(H > 0 ? H : 1)));
  CK(x.flag.ensure(sizeof(int32_t) * size_t(H > 0 ? H : 1)));
  CK(x.pos.ensure(sizeof(int64_t) * size_t(H + 1)));
  *v = DIdleHosts{dcol[0], dcol[1], dcol[2], dcol[3], dcol[4], dcol[5], dcol[6], dcol[7], flags};
  return EVG_OK;
}

// Scan the decided flags (none: pos stays NULL), copy the verdicts and `dout_bytes` of per-distro output back, wait.
static int finish_idle_hosts(evg_ctx* c, int64_t H, evg_host_verdict* verdicts, void* dout, size_t dout_bytes) {
  auto& x = c->ih;
  cudaStream_t s = c->stream;
  CK(cudaGetLastError());
  if (H > 0) CK(cudaMemcpyAsync(verdicts, x.verdict.p, sizeof(evg_host_verdict) * size_t(H), cudaMemcpyDeviceToHost, s));
  if (dout_bytes > 0) CK(cudaMemcpyAsync(dout, x.dout.p, dout_bytes, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));  // the caller's arrays are free again and the outputs are written
  return EVG_OK;
}

int evg_host_drawdown(evg_ctx* c, const evg_idle_host_soa* hosts, const int64_t* idle_off, const evg_drawdown_in* in, int64_t now_ns,
                      evg_host_drawdown_out* out) {
  ENTER(c, "evg_host_drawdown");
  int rc = check_idle_hosts(who, hosts, idle_off);
  if (rc != EVG_OK) return rc;
  const int64_t H = hosts->n_hosts;
  const int32_t D = hosts->n_distros;
  if (!in || !in->existing_hosts || !out || (H > 0 && !out->hosts) || (D > 0 && !out->distros))
    return fail(EVG_ERR_INVALID, "%s: null input or output", who);
  if (!in->new_cap_target != !in->queue_length_dm)
    return fail(EVG_ERR_INVALID, "%s: new_cap_target and queue_length_dm must be both NULL (chained) or both given", who);
  const bool chained = !in->new_cap_target;
  for (int32_t d = 0; d < D; d++)
    if (in->existing_hosts[d] < 0 || (!chained && in->queue_length_dm[d] < 0))
      return fail(EVG_ERR_INVALID, "%s: distro %d has a negative existing_hosts or queue_length_dm", who, d);
  if (chained) {
    if ((rc = need_tick(c, who, Need::kTick)) != EVG_OK || (rc = need_tick(c, who, Need::kHostJob)) != EVG_OK) return rc;
    if (D != c->Dn) return fail(EVG_ERR_INVALID, "%s: chained on a tick of %d distros, the host table has %d", who, c->Dn, D);
  }
  c->launches = 0;
  // per-distro input: existing_hosts, then (standalone) new_cap_target and queue_length_dm
  std::vector<int64_t> din(size_t(D) * (chained ? 1 : 3));
  std::copy(in->existing_hosts, in->existing_hosts + D, din.begin());
  if (!chained) {
    std::copy(in->new_cap_target, in->new_cap_target + D, din.begin() + D);
    std::copy(in->queue_length_dm, in->queue_length_dm + D, din.begin() + 2 * D);
  }
  DIdleHosts v;
  if ((rc = stage_idle_hosts(c, hosts, idle_off, din.data(), din.size() * sizeof(int64_t), &v)) != EVG_OK) return rc;
  auto& x = c->ih;
  CK(x.dout.ensure(sizeof(evg_drawdown_distro) * size_t(D > 0 ? D : 1)));
  const int64_t* dd = x.din.as<int64_t>();
  const DrawdownSrc src{chained ? c->hj.out.as<evg_host_report>() : nullptr, chained ? c->b_qinfo.as<evg_queue_info>() : nullptr,
                        chained ? nullptr : dd + D, chained ? nullptr : dd + 2 * D, dd};
  const int64_t* off = x.off.as<int64_t>();
  int64_t* pos = H > 0 ? x.pos.as<int64_t>() : nullptr;
  launch(c, c->stream, k_hd_host, grid_for(H, 256), 256, 0, H, D, off, v, src, now_ns, x.verdict.as<evg_host_verdict>(), x.flag.as<int32_t>());
  if (H > 0) {
    CK(scan_counts(c, x.flag.as<int32_t>(), H, pos));
    launch(c, c->stream, k_hd_cap, grid_for(H, 256), 256, 0, H, D, off, src, static_cast<const int64_t*>(pos), x.verdict.as<evg_host_verdict>());
  }
  launch(c, c->stream, k_hd_distro, grid_for(D, 256), 256, 0, D, off, src, static_cast<const int64_t*>(pos), x.dout.as<evg_drawdown_distro>());
  return finish_idle_hosts(c, H, out->hosts, out->distros, sizeof(evg_drawdown_distro) * size_t(D));
}

int evg_idle_hosts(evg_ctx* c, const evg_idle_host_soa* hosts, const int64_t* idle_off, const evg_idle_cfg* cfg, int64_t now_ns,
                   evg_idle_hosts_out* out) {
  ENTER(c, "evg_idle_hosts");
  int rc = check_idle_hosts(who, hosts, idle_off);
  if (rc != EVG_OK) return rc;
  const int64_t H = hosts->n_hosts;
  const int32_t D = hosts->n_distros;
  if ((D > 0 && !cfg) || !out || (H > 0 && !out->hosts) || (D > 0 && !out->distros))
    return fail(EVG_ERR_INVALID, "%s: null cfg or output", who);
  for (int32_t d = 0; d < D; d++)
    if (cfg[d].minimum_hosts < 0 || cfg[d].running_hosts_count < 0)
      return fail(EVG_ERR_INVALID, "%s: cfg[%d] has a negative minimum_hosts or running_hosts_count", who, d);
  c->launches = 0;
  DIdleHosts v;
  if ((rc = stage_idle_hosts(c, hosts, idle_off, cfg, sizeof(evg_idle_cfg) * size_t(D), &v)) != EVG_OK) return rc;
  auto& x = c->ih;
  CK(x.dout.ensure(sizeof(evg_idle_distro) * size_t(D > 0 ? D : 1)));
  const int64_t* off = x.off.as<int64_t>();
  const evg_idle_cfg* dcfg = x.din.as<evg_idle_cfg>();
  int64_t* pos = H > 0 ? x.pos.as<int64_t>() : nullptr;
  launch(c, c->stream, k_idle_host, grid_for(H, 256), 256, 0, H, D, off, v, dcfg, now_ns, x.verdict.as<evg_host_verdict>(), x.flag.as<int32_t>());
  if (H > 0) CK(scan_counts(c, x.flag.as<int32_t>(), H, pos));
  launch(c, c->stream, k_idle_distro, grid_for(D, 256), 256, 0, D, off, dcfg, static_cast<const int64_t*>(pos), x.dout.as<evg_idle_distro>());
  return finish_idle_hosts(c, H, out->hosts, out->distros, sizeof(evg_idle_distro) * size_t(D));
}

// The host table and its offsets, checked before anything is staged or launched.
static int check_est_hosts(const char* who, const evg_est_host_soa* h, const int64_t* off, int32_t D) {
  if (!h || !off) return fail(EVG_ERR_INVALID, "%s: null host table or est_host_off", who);
  if (h->n_hosts < 0) return fail(EVG_ERR_INVALID, "%s: negative n_hosts", who);
  if (h->n_hosts > 0 && (!h->kind || !h->expected_ns || !h->dispatch_ns)) return fail(EVG_ERR_INVALID, "%s: null host column", who);
  if (const int rc = check_offsets(off, D, h->n_hosts, who, "est_host_off"); rc != EVG_OK) return rc;
  for (int64_t i = 0; i < h->n_hosts; i++)
    if (h->kind[i] > EVG_EH_IGNORED) return fail(EVG_ERR_INVALID, "%s: host row %lld has kind %d", who, (long long)i, int(h->kind[i]));
  return EVG_OK;
}

// What the two estimate entry points share: the queues' offsets and durations are in es.item_off / es.dur (item_off is
// the host copy); the pools are built, sorted and simulated, and the estimates and pool sizes copied out.
static int estimate_run(evg_ctx* c, int32_t D, const evg_est_host_soa* h, const int64_t* host_off, int64_t now, const int64_t* item_off,
                        int64_t* start_ns, int32_t* hosts_used) {
  const int64_t H = h->n_hosts, N = item_off[D];
  if (H == 0) {  // len(s.hosts) == 0 everywhere (:54-56): answered here, as evg_find_next_tasks answers empty queues
    std::fill(start_ns, start_ns + N, int64_t(-1));
    std::fill(hosts_used, hosts_used + D, 0);
    return EVG_OK;
  }
  auto& x = c->es;
  cudaStream_t s = c->stream;
  UP(s, x.kind, h->kind, H, uint8_t);
  UP(s, x.expected, h->expected_ns, H, int64_t);
  UP(s, x.dispatch, h->dispatch_ns, H, int64_t);
  UP(s, x.host_off, host_off, D + 1, int64_t);
  for (DevBuf* b : {&x.ttc, &x.pool[0], &x.pool[1]}) CK(b->ensure(sizeof(int64_t) * size_t(H)));
  CK(x.used.ensure(sizeof(int32_t) * size_t(H)));
  CK(x.pos.ensure(sizeof(int64_t) * size_t(H + 1)));
  CK(x.pool_off.ensure(sizeof(int64_t) * size_t(D + 1)));
  CK(x.hosts_used.ensure(sizeof(int32_t) * size_t(D)));
  launch(c, s, k_es_host, grid_for(H, 256), 256, 0, H, x.kind.as<uint8_t>(), x.expected.as<int64_t>(), x.dispatch.as<int64_t>(), now,
         x.ttc.as<int64_t>(), x.used.as<int32_t>());
  CK(scan_counts(c, x.used.as<int32_t>(), H, x.pos.as<int64_t>()));
  launch(c, s, k_es_compact, grid_for(H, 256), 256, 0, H, x.ttc.as<int64_t>(), x.used.as<int32_t>(), x.pos.as<int64_t>(), x.pool[0].as<int64_t>());
  launch(c, s, k_es_pool_off, grid_for(D + 1, 256), 256, 0, D, x.host_off.as<int64_t>(), x.pos.as<int64_t>(), x.pool_off.as<int64_t>(),
         x.hosts_used.as<int32_t>());
  // one warp per distro that has host rows and items, the largest items x hosts first
  std::vector<int32_t> list;
  int64_t max_hosts = 0;
  for (int32_t d = 0; d < D; d++)
    if (host_off[d + 1] > host_off[d] && item_off[d + 1] > item_off[d]) {
      list.push_back(d);
      max_hosts = std::max(max_hosts, host_off[d + 1] - host_off[d]);
    }
  if (!list.empty()) {
    const auto work = [&](int32_t d) { return double(host_off[d + 1] - host_off[d]) * double(item_off[d + 1] - item_off[d]); };
    std::stable_sort(list.begin(), list.end(), [&](int32_t a, int32_t b) { return work(a) > work(b); });
    UP(s, x.list, list.data(), int64_t(list.size()), int32_t);
    CK(x.start.ensure(sizeof(int64_t) * size_t(N)));
    int64_t* const pools[2] = {x.pool[0].as<int64_t>(), x.pool[1].as<int64_t>()};
    int64_t* pool = seg_merge_sort(c, s, EsValueOrder{}, x.pool_off.as<int64_t>(), D, H, max_hosts, pools);
    CK(cudaMemsetAsync(x.start.p, 0xFF, sizeof(int64_t) * size_t(N), s));  // -1: no estimate
    const DEst X{x.list.as<int32_t>(), int32_t(list.size()), x.pool_off.as<int64_t>(), x.item_off.as<int64_t>(), x.dur.as<int64_t>(),
                 pool, x.start.as<int64_t>()};
    launch(c, s, k_es_sim, grid_for(int64_t(list.size()), kEsWarps), 32 * kEsWarps, 0, X);
  }
  CK(cudaGetLastError());
  if (list.empty()) std::fill(start_ns, start_ns + N, int64_t(-1));  // the distros with items have no host rows
  else CK(cudaMemcpyAsync(start_ns, x.start.p, sizeof(int64_t) * size_t(N), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(hosts_used, x.hosts_used.p, sizeof(int32_t) * size_t(D), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return EVG_OK;
}

int evg_estimate_start_times(evg_ctx* c, int32_t cap, const evg_est_host_soa* hosts, const int64_t* est_host_off, int64_t now_ns,
                             int64_t* item_off, int64_t* start_ns, int64_t items_capacity, int32_t* hosts_used) {
  ENTER(c, "evg_estimate_start_times");
  int rc = need_tick(c, who, Need::kTick);
  if (rc != EVG_OK) return rc;
  const int32_t D = c->Dn;
  if (cap < 0 || !item_off || (D > 0 && !hosts_used)) return fail(EVG_ERR_INVALID, "%s: negative cap, or null item_off or hosts_used", who);
  if ((rc = check_est_hosts(who, hosts, est_host_off, D)) != EVG_OK) return rc;
  const int64_t N = persisted_item_off(c, cap == 0 ? EVG_PERSISTED_QUEUE_CAP : cap, item_off);
  if (N > items_capacity || (N > 0 && !start_ns))
    return fail(EVG_ERR_INVALID, "%s: %lld rows needed, %lld available", who, (long long)N, (long long)items_capacity);
  c->launches = 0;
  if (N > 0 && hosts->n_hosts > 0) {
    auto& x = c->es;
    UP(c->stream, x.item_off, item_off, D + 1, int64_t);
    CK(x.dur.ensure(sizeof(int64_t) * size_t(N)));
    launch(c, c->stream, k_es_gather, grid_for(N, 256), 256, 0, D, N, x.item_off.as<int64_t>(), c->b_taskoff.as<int64_t>(),
           c->b_order.as<int32_t>(), dtasks(c).expected, x.dur.as<int64_t>());
  }
  return estimate_run(c, D, hosts, est_host_off, now_ns, item_off, start_ns, hosts_used);
}

int evg_estimate_start_batch(evg_ctx* c, const int64_t* durations, const int64_t* item_off, int32_t D, const evg_est_host_soa* hosts,
                             const int64_t* est_host_off, int64_t now_ns, int64_t* start_ns, int32_t* hosts_used) {
  ENTER(c, "evg_estimate_start_batch");
  if (D < 0 || !item_off || (D > 0 && !hosts_used)) return fail(EVG_ERR_INVALID, "%s: negative n_distros, or null item_off or hosts_used", who);
  int rc = check_offsets(item_off, D, -1, who, "item_off");
  if (rc != EVG_OK) return rc;
  const int64_t N = item_off[D];
  if (N > 0 && (!durations || !start_ns)) return fail(EVG_ERR_INVALID, "%s: null durations or start_ns", who);
  if ((rc = check_est_hosts(who, hosts, est_host_off, D)) != EVG_OK) return rc;
  c->launches = 0;
  if (N > 0 && hosts->n_hosts > 0) {
    UP(c->stream, c->es.item_off, item_off, D + 1, int64_t);
    UP(c->stream, c->es.dur, durations, N, int64_t);
  }
  return estimate_run(c, D, hosts, est_host_off, now_ns, item_off, start_ns, hosts_used);
}

int evg_plan_distro(evg_ctx* c, const evg_task_soa* tasks, const evg_distro_cfg* cfg, int32_t n_groups,
                    const int32_t* group_max_hosts, int64_t now_ns, uint32_t opts, evg_plan_out* out) {
  ENTER(c, "evg_plan_distro");
  if (!tasks || !cfg) return fail(EVG_ERR_INVALID, "evg_plan_distro: null argument");
  int64_t task_off[2] = {0, tasks->n_tasks};
  int64_t group_off[2] = {0, n_groups};
  evg_distro_table dt;
  dt.n_distros = 1; dt._reserved = 0; dt.task_off = task_off; dt.group_off = group_off; dt.cfg = cfg;
  dt.group_max_hosts = group_max_hosts;
  return evg_plan_batch(c, tasks, &dt, now_ns, opts, out);
}

int evg_alloc_distro(evg_ctx* c, const evg_host_soa* hosts, const evg_alloc_cfg* cfg, const evg_queue_info* info,
                     evg_group_info* groups, int32_t n_groups, int64_t now_ns, evg_alloc_result* result, int32_t* status) {
  ENTER(c, "evg_alloc_distro");
  if (!hosts || !cfg || !info) return fail(EVG_ERR_INVALID, "evg_alloc_distro: null argument");
  int64_t host_off[2] = {0, hosts->n_hosts};
  int64_t group_off[2] = {0, n_groups};
  evg_alloc_out ao;
  ao.result = result; ao.status = status;
  return evg_alloc_batch(c, hosts, host_off, cfg, info, groups, group_off, 1, now_ns, &ao);
}

void* evg_host_alloc(uint64_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    g_err = "cudaHostAlloc failed";
    return nullptr;
  }
  return p;
}
void evg_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
