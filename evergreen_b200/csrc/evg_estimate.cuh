// evg_estimate.cuh -- task start-time estimates (SURVEY.md §8): the third reader of the persisted queue.
//
// Reference: model.GetEstimatedStartTime (model/task_start_estimation.go:99-122) with createSimulatorModel :124-163,
// simulate :53-67 and dispatchNextTask :69-96; restated on the CPU in oracle/oracle_estimate.py.
//
// The reference replays pos + 1 dispatches per task asked about.  The replay for position p is a prefix of the replay
// for any later position, so ONE run over a distro's queue yields the estimate of every position.  The run is
// sequential within a distro and independent across distros: one WARP per distro (k_es_sim), and the warp
// parallelises the step -- the first-match scan over adjacent pairs goes 32 pairs at a time, and the insertion shifts
// whichever side of the insertion point is shorter.
//
// "Subtract the fast-forward time from every remaining host" (:75-77) is one running offset: the pool stores
// value + elapsed-at-insert and a host's current value is stored - elapsed.  Go's int64 arithmetic wraps, so this is
// exact for every input.  The fast-forward itself then reads elapsed' = elapsed + (stored[0] - elapsed) = stored[0].
#pragma once

constexpr int kEsOnChip = EVG_EST_ONCHIP_HOSTS;  // a pool of at most this many hosts is simulated in shared memory
constexpr int kEsWarps = 4;                      // distros per CTA: 4 x 8 KB of pool

// One thread per host row: timeToCompletion by status (:130-158).  used = 0: the row contributes no host.
__global__ void __launch_bounds__(256) k_es_host(int64_t n, const uint8_t* __restrict__ kind, const int64_t* __restrict__ expected,
                                                 const int64_t* __restrict__ dispatch, int64_t now, int64_t* __restrict__ ttc,
                                                 int32_t* __restrict__ used) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t v = 0;
  int32_t u = 1;
  switch (kind[i]) {
    case EVG_EH_UNINITIALIZED: v = 4 * kMinute; break;  // hostInitializingDelay
    case EVG_EH_STARTING: v = 3 * kMinute; break;       // hostStartingDelay
    case EVG_EH_PROVISIONING: v = kMinute; break;       // hostProvisiongingDelay
    case EVG_EH_FREE: break;
    case EVG_EH_RUNNING: v = wsub(expected[i], since(now, dispatch[i])); break;  // may be negative: an overrun task
    default: u = 0;
  }
  ttc[i] = v;
  used[i] = u;
}
// The rows that contribute, packed: pos is the exclusive scan of `used`.
__global__ void __launch_bounds__(256) k_es_compact(int64_t n, const int64_t* __restrict__ ttc, const int32_t* __restrict__ used,
                                                    const int64_t* __restrict__ pos, int64_t* __restrict__ pool) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n && used[i]) pool[pos[i]] = ttc[i];
}
// Each distro's slice of the packed pools, and its size: the hosts the simulation used.
__global__ void __launch_bounds__(256) k_es_pool_off(int32_t n_distros, const int64_t* __restrict__ host_off, const int64_t* __restrict__ pos,
                                                     int64_t* __restrict__ pool_off, int32_t* __restrict__ hosts_used) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d > n_distros) return;
  const int64_t p = pos[host_off[d]];
  pool_off[d] = p;
  if (d < n_distros) hosts_used[d] = int32_t(pos[host_off[d + 1]] - p);
}

// sort.Sort(s.hosts) (:60) for every distro: k_seg_merge_pass's order of the pool values, signed int64 ascending.
// Pools of any size; equal values are interchangeable.
struct EsValueOrder {
  using Elem = int64_t;
  struct Pivot {
    int64_t me;
    __device__ bool before(int64_t x) const { return x < me; }
    __device__ bool after(int64_t x) const { return x > me; }
  };
  __device__ Pivot pivot(int, int64_t, int64_t me) const { return {me}; }
};

// The chained call's queue: TaskQueueItem.ExpectedDuration of every persisted rank, the column and rank order
// k_project_queue reads.
__global__ void __launch_bounds__(256) k_es_gather(int32_t n_distros, int64_t n, const int64_t* __restrict__ item_off,
                                                   const int64_t* __restrict__ task_off, const int32_t* __restrict__ order,
                                                   const int64_t* __restrict__ expected, int64_t* __restrict__ dur) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(item_off, n_distros, j, n);
  if (d < 0) return;
  const int64_t base = task_off[d];
  dur[j] = expected[base + order[base + (j - item_off[d])]];
}

struct DEst {
  const int32_t* list;      // the distros with at least one host row and one item, largest items x hosts first
  int32_t n_list;
  const int64_t* pool_off;  // [D+1]
  const int64_t* item_off;  // [D+1]
  const int64_t* dur;       // [items]
  int64_t* pool;            // the sorted pools; a pool above kEsOnChip is simulated where it lies
  int64_t* start;           // [items] preset to -1
};

// slot of logical index i of a ring of m slots that starts at `head` (head < m, i <= m)
__device__ __forceinline__ int es_slot(int head, int i, int m) {
  const int r = head + i;
  return r >= m ? r - m : r;
}

// simulate (:53-67) of a fresh simulator, for every position of the queue at once.  The pool is a ring of m slots:
// dispatchNextTask pops the first host (:72-74), which frees the slot the insertion (:84-95) needs, so the ring never
// grows.  The pool is sorted once, before the run; the insertion leaves it unsorted (it puts the value in FRONT of a
// smaller-or-equal element and appends a value below every element), so the first-match scan is the specification.
__global__ void __launch_bounds__(32 * kEsWarps) k_es_sim(DEst X) {
  __shared__ int64_t s_pool[kEsWarps][kEsOnChip];
  constexpr unsigned kAll = 0xffffffffu;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= X.n_list) return;
  const int d = X.list[w];
  const int64_t p0 = X.pool_off[d], i0 = X.item_off[d];
  const int m = int(X.pool_off[d + 1] - p0);
  const int n = int(X.item_off[d + 1] - i0);
  if (m == 0) return;  // every row of the distro was EVG_EH_IGNORED: len(s.hosts) == 0 (:54)
  int64_t* pool = X.pool + p0;
  if (m <= kEsOnChip) {
    int64_t* s = s_pool[threadIdx.x >> 5];
    for (int i = lane; i < m; i += 32) s[i] = pool[i];
    pool = s;
    __syncwarp();
  }
  uint64_t elapsed = 0;  // s.timeElapsed, the same in every lane
  int head = 0;
  for (int c0 = 0; c0 < n; c0 += 32) {  // 32 positions: one coalesced read of durations, one coalesced write of estimates
    const int64_t my_dur = c0 + lane < n ? X.dur[i0 + c0 + lane] : 0;
    int64_t my_est = 0;
    const int steps = min(32, n - c0);
    for (int s = 0; s < steps; s++) {
      const int64_t dur = __shfl_sync(kAll, my_dur, s);
      elapsed = uint64_t(pool[head]);  // timeElapsed += hosts[0] (:72-73), as stored
      if (lane == s) my_est = int64_t(elapsed);
      head = es_slot(head, 1, m);      // s.hosts = s.hosts[1:]
      // the first i < count - 2 with hosts[i] <= duration <= hosts[i+1] (:85-87); none: append (:92)
      int k = m - 1;
      for (int b = 0; b < m - 2; b += 32) {
        const int i = b + lane;
        bool hit = false;
        if (i < m - 2) {
          const int64_t lo = int64_t(uint64_t(pool[es_slot(head, i, m)]) - elapsed);
          const int64_t hi = int64_t(uint64_t(pool[es_slot(head, i + 1, m)]) - elapsed);
          hit = lo <= dur && hi >= dur;
        }
        const unsigned hits = __ballot_sync(kAll, hit);
        if (hits) { k = b + __ffs(hits) - 1; break; }
      }
      // insert at k among the m - 1 hosts left: move the shorter side by one slot
      if (k < m - 1 - k) {  // the k hosts in front move into the slot the pop freed, lowest first
        const int nh = head == 0 ? m - 1 : head - 1;
        for (int b = 0; b < k; b += 32) {
          const int i = b + lane;
          int64_t v = 0;
          if (i < k) v = pool[es_slot(head, i, m)];
          __syncwarp();
          if (i < k) pool[es_slot(nh, i, m)] = v;
        }
        head = nh;
      } else {              // the hosts from k on move back, highest first
        for (int e = m - 1; e > k; e -= 32) {
          const int i = e - 1 - lane;
          int64_t v = 0;
          if (i >= k) v = pool[es_slot(head, i, m)];
          __syncwarp();
          if (i >= k) pool[es_slot(head, i + 1, m)] = v;
        }
      }
      if (lane == 0) pool[es_slot(head, k, m)] = int64_t(uint64_t(dur) + elapsed);
      __syncwarp();
    }
    if (c0 + lane < n) X.start[i0 + c0 + lane] = my_est;
  }
}
