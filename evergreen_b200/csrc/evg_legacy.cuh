// evg_legacy.cuh -- the LEGACY comparator prioritiser (SURVEY.md §8 row L) behind the TaskPrioritizer interface.
//
// Reference: CmpBasedTaskPrioritizer.PrioritizeTasks (scheduler/task_prioritizer.go:80-142): split the distro's tasks
// into high-priority / repotracker / patch lists (:214-247), presort each list reverse-lexically by
// "BuildId-TaskGroup-Id" (groupTaskGroups, setup_funcs.go:72-87), sort.Stable it with the first-definitive
// comparator chain [byTaskGroupOrder, byCommitQueue, byPriority, byNumDeps, byGenerateTasks, byAge, byRuntime]
// (task_priority_cmp.go:25-208), then merge: high-priority first, then patch and repotracker tasks alternately
// starting with a patch task (:251-278).
//
// Here: ONE segmented merge sort of every distro's tasks by the total order
//     (list, comparator chain, presort rank)
// -- on inputs where the chain is a strict weak order ("key-decomposable": the host marks each list's byAge mode)
// a stable sort from the presorted order IS the sort by (chain, presort rank), whatever algorithm runs it -- followed
// by a closed-form interleave.  Strings never reach the device: the shim interns "BuildId-TaskGroup" to its rank
// among the distro's distinct such strings, the (TaskGroup, BuildId) pair to a dense id, the presort to a rank.
// A list the host marks EVG_LEGACY_MODE_LITERAL (the chain is not transitive there: commit builds of several
// projects, zero and non-zero expected durations mixed) has no order that every stable sort agrees on -- Go's result
// depends on the exact steps of its insertion-sort / symMerge.  Such a list is sorted by the nearest transitive key
// (byAge by IngestTime only, byRuntime on the raw durations) so that the output is still a permutation with task
// groups, merge-queue tasks, priorities, dependents and generators where the reference puts them, and the distro is
// reported EVG_LEGACY_NOT_DECOMPOSABLE.
// A list marked EVG_LEGACY_MODE_GO_STABLE is sorted by presort rank alone in the merge sort, which leaves it in
// groupTaskGroups order at offset sum(counts of the lists before it) of its distro; sort.Stable is then replayed on it
// step for step with the literal comparator chain (legacy_more_important):
//   k_gs_insertion   insertionSort of every 20-block, one thread per block
//   per level (block = 20, 40, ... below the longest list):
//     k_gs_seed      the level's symMerge(a, a + block, min(a + 2 block, n)) calls, one task each
//     k_gs_wave      one recursion depth of every pending symMerge: its binary search (one thread, Go's probe sequence),
//                    its rotation (the task's warp or CTA, through the spare merge-sort buffer) and its two recursive
//                    calls, queued for the next wave
// Every task of a wave owns a range no other task of the wave touches, so the waves run them in any order.  A call of
// size s has calls of at most ceil(s / 2) below it and none at size 2, so a level of merges of at most s elements ends
// after ceil(log2 s) waves: the host launches exactly those, without reading anything back.
// The reference also returns an O(compares) map of reason strings (orderingLogic); it is not produced.
#pragma once

struct DLegacy {
  int64_t n;
  const int64_t* priority;
  const int64_t* ingest;
  const int64_t* expected;
  const int32_t* numdep;
  const int32_t* revision;
  const int32_t* project;
  const int32_t* tg_rank;
  const int32_t* tg_pair;
  const int32_t* tgo;
  const int32_t* presort;
  const uint32_t* flags;
  const uint8_t* list_mode;  // [D*3] per (distro, list): EVG_LEGACY_MODE_*; lists in the order high, patch, repotracker
  const int64_t* task_off;
  int32_t n_distros;
};

// list a task is filed under (splitTasksByRequester): 0 high priority, 1 patch, 2 repotracker, 3 dropped
__device__ __forceinline__ int legacy_list(const DLegacy& X, int64_t t) {
  if (X.priority[t] > 100) return 0;  // evergreen.MaxTaskPriority (globals.go:185)
  const uint32_t rq = X.flags[t] & EVG_LF_REQ_MASK;
  if (rq == EVG_LF_REQ_SYSTEM) return 2;
  if (rq == EVG_LF_REQ_PATCH) return 1;
  return 3;
}

// true when task a sorts strictly before task b (both global indices inside distro d)
__device__ bool legacy_less(const DLegacy& X, int d, int64_t a, int64_t b) {
  const int la = legacy_list(X, a), lb = legacy_list(X, b);
  if (la != lb) return la < lb;
  const uint32_t fa = X.flags[a], fb = X.flags[b];
  const int mode = la < 3 ? X.list_mode[d * 3 + la] : 0;
  if (mode == EVG_LEGACY_MODE_GO_STABLE) return X.presort[a] < X.presort[b];  // groupTaskGroups; k_gs_* sort it
  const int32_t ra = X.tg_rank[a], rb = X.tg_rank[b];
  if (ra >= 0 || rb >= 0) {  // byTaskGroupOrder (task_priority_cmp.go:132-169): always definitive between two group tasks
    if (rb < 0) return true;
    if (ra < 0) return false;
    if (X.tg_pair[a] == X.tg_pair[b] && X.tgo[a] != X.tgo[b]) return X.tgo[a] < X.tgo[b];
    if (ra != rb) return ra < rb;
    return X.presort[a] < X.presort[b];  // "-1" both ways: the stable sort keeps the presorted order
  }
  const bool ca = fa & EVG_LF_MERGE_QUEUE_VERSION, cb = fb & EVG_LF_MERGE_QUEUE_VERSION;  // byCommitQueue :191-204
  if (ca != cb) return ca;
  const int64_t pa = X.priority[a], pb = X.priority[b];  // byPriority :25-36
  if (pa != pb) return pa > pb;
  const int32_t na = X.numdep[a], nb = X.numdep[b];  // byNumDeps :43-54
  if (na != nb) return na > nb;
  const bool ga = fa & EVG_LF_GENERATE, gb = fb & EVG_LF_GENERATE;  // byGenerateTasks :175-185
  if (ga != gb) return ga;
  // byAge :73-95
  if (mode == EVG_LEGACY_MODE_REVISION) {
    if (X.revision[a] != X.revision[b]) return X.revision[a] > X.revision[b];
  } else {
    if (X.ingest[a] != X.ingest[b]) return X.ingest[a] < X.ingest[b];
  }
  const int64_t ea = X.expected[a], eb = X.expected[b];  // byRuntime :104-123 (a zero duration ties with everything: LITERAL lists)
  if ((mode == EVG_LEGACY_MODE_LITERAL || (ea != 0 && eb != 0)) && ea != eb) return ea > eb;
  return X.presort[a] < X.presort[b];
}

__global__ void __launch_bounds__(256) k_legacy_init(DLegacy X, int32_t* idx, unsigned int* counts) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= X.n) return;
  const int d = find_distro(X.task_off, 0, X.n_distros - 1, t);
  idx[t] = int32_t(t - X.task_off[d]);
  atomicAdd(&counts[d * 4 + legacy_list(X, t)], 1u);
}

// k_seg_merge_pass's order of a distro's task indices (distro-local) by legacy_less
struct LegacyOrder {
  using Elem = int32_t;
  DLegacy X;
  struct Pivot {
    DLegacy X; int d; int64_t base, gm;
    __device__ bool before(int32_t x) const { return legacy_less(X, d, base + x, gm); }
    __device__ bool after(int32_t x) const { return legacy_less(X, d, gm, base + x); }
  };
  __device__ Pivot pivot(int d, int64_t base, int32_t me) const { return {X, d, base, base + me}; }
};

// mergeTasks (task_prioritizer.go:251-278): high-priority tasks, then patch / repotracker alternately (patch first)
// until one list runs out, then the rest of the other; dropped tasks leave -1 slots at the end.
__global__ void __launch_bounds__(256) k_legacy_interleave(DLegacy X, const int32_t* __restrict__ sorted, const unsigned int* __restrict__ counts,
                                                           int32_t* __restrict__ out, int64_t* __restrict__ count_out, int32_t* __restrict__ status) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= X.n) return;
  const int d = find_distro(X.task_off, 0, X.n_distros - 1, p);
  const int64_t base = X.task_off[d];
  const int64_t q = p - base;
  const int64_t nH = counts[d * 4 + 0], nP = counts[d * 4 + 1], nR = counts[d * 4 + 2];
  const int32_t me = sorted[p];
  int64_t pos;
  if (q < nH) pos = q;
  else if (q < nH + nP) {
    const int64_t j = q - nH;
    pos = nH + (j < nR ? 2 * j : nR + j);
  } else if (q < nH + nP + nR) {
    const int64_t j = q - nH - nP;
    pos = nH + (j < nP ? 2 * j + 1 : nP + j);
  } else pos = q;
  out[base + pos] = q < nH + nP + nR ? me : -1;
  if (q == 0) {
    count_out[d] = nH + nP + nR;
    status[d] = (X.list_mode[d * 3] == EVG_LEGACY_MODE_LITERAL || X.list_mode[d * 3 + 1] == EVG_LEGACY_MODE_LITERAL ||
                 X.list_mode[d * 3 + 2] == EVG_LEGACY_MODE_LITERAL) ? EVG_LEGACY_NOT_DECOMPOSABLE : EVG_LEGACY_OK;
  }
}

// ---- EVG_LEGACY_MODE_GO_STABLE: sort.Stable (src/sort/zsortinterface.go) replayed on the presorted list -------------

// taskMoreImportantThan (task_prioritizer.go:159-184) of global tasks a, b of one distro: the first comparator of the
// chain that is not 0 decides; all 0 is false.  Not a key: byAge picks its field per pair, byRuntime ties a zero
// with everything and byTaskGroupOrder answers -1 both ways on equal strings.
__device__ bool legacy_more_important(const DLegacy& X, int64_t a, int64_t b) {
  const int32_t ra = X.tg_rank[a], rb = X.tg_rank[b];
  if (ra >= 0 || rb >= 0) {  // byTaskGroupOrder :132-169 (tg_rank < 0: TaskGroup == "")
    if (rb < 0) return true;
    if (ra < 0) return false;
    if (X.tg_pair[a] == X.tg_pair[b] && X.tgo[a] != X.tgo[b]) return X.tgo[a] < X.tgo[b];
    return ra < rb;  // "BuildId-TaskGroup" strings: equal ones are -1 both ways
  }
  const uint32_t fa = X.flags[a], fb = X.flags[b];
  const bool ca = fa & EVG_LF_MERGE_QUEUE_VERSION, cb = fb & EVG_LF_MERGE_QUEUE_VERSION;  // byCommitQueue :191-204
  if (ca != cb) return ca;
  const int64_t pa = X.priority[a], pb = X.priority[b];  // byPriority :25-36
  if (pa != pb) return pa > pb;
  const int32_t na = X.numdep[a], nb = X.numdep[b];  // byNumDeps :43-54
  if (na != nb) return na > nb;
  const bool ga = fa & EVG_LF_GENERATE, gb = fb & EVG_LF_GENERATE;  // byGenerateTasks :175-185
  if (ga != gb) return ga;
  // byAge :73-95: RevisionOrderNumber between two commit builds of one project, IngestTime otherwise
  if ((fa & EVG_LF_REQ_MASK) == EVG_LF_REQ_SYSTEM && (fb & EVG_LF_REQ_MASK) == EVG_LF_REQ_SYSTEM && X.project[a] == X.project[b]) {
    if (X.revision[a] != X.revision[b]) return X.revision[a] > X.revision[b];
  } else if (X.ingest[a] != X.ingest[b]) {
    return X.ingest[a] < X.ingest[b];
  }
  const int64_t ea = X.expected[a], eb = X.expected[b];  // byRuntime :104-123: a zero on either side ties
  return ea != 0 && eb != 0 && ea > eb;
}

// Distro d's list that distro-local position q of the presorted buffer falls in: true when it is a GO_STABLE list,
// with its first position `off` and length `n`.
__device__ __forceinline__ bool gs_list_at(const DLegacy& X, const unsigned int* counts, int d, int64_t q, int64_t& off, int64_t& n) {
  off = 0;
  for (int l = 0; l < 3; l++) {
    n = counts[d * 4 + l];
    if (q < off + n) return X.list_mode[d * 3 + l] == EVG_LEGACY_MODE_GO_STABLE;
    off += n;
  }
  return false;
}

// One pending symMerge(a, m, b) of distro d; positions are distro-local in the presorted buffer.  Go's midpoints are
// taken on list-relative indices, and (i + o + j + o) >> 1 = o + ((i + j) >> 1): shifting by the list's offset o
// changes no probe.
struct GsTask { int32_t d, a, m, b; };

// A slot of a task queue for each calling thread, one atomic per warp.
__device__ __forceinline__ unsigned int gs_slot(unsigned int* count) {
  const unsigned int act = __activemask();
  const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
  unsigned int first = 0;
  if (lane == leader) first = atomicAdd(count, unsigned(__popc(act)));
  first = __shfl_sync(act, first, leader);
  return first + unsigned(__popc(act & ((1u << lane) - 1u)));
}

// insertionSort (zsortinterface.go) of every 20-block of every GO_STABLE list, one thread per block.
__global__ void __launch_bounds__(256) k_gs_insertion(DLegacy X, const unsigned int* __restrict__ counts, int32_t* __restrict__ v) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= X.n) return;
  const int d = find_distro(X.task_off, 0, X.n_distros - 1, p);
  const int64_t base = X.task_off[d], q = p - base;
  int64_t off, n;
  if (!gs_list_at(X, counts, d, q, off, n) || (q - off) % 20 != 0) return;
  const int e = int(min(n - (q - off), int64_t(20)));
  int32_t r[20];
  for (int i = 0; i < e; i++) r[i] = v[p + i];
  for (int i = 1; i < e; i++)
    for (int j = i; j > 0 && legacy_more_important(X, base + r[j], base + r[j - 1]); j--) {
      const int32_t t = r[j]; r[j] = r[j - 1]; r[j - 1] = t;
    }
  for (int i = 0; i < e; i++) v[p + i] = r[i];
}

// The level of sort.Stable with blocks of `block`: symMerge(a, a + block, min(a + 2 block, n)) for every a = 0, 2 block,
// ... with a + block < n, queued as tasks.
__global__ void __launch_bounds__(256) k_gs_seed(DLegacy X, const unsigned int* __restrict__ counts, int64_t block,
                                                 GsTask* __restrict__ out, unsigned int* __restrict__ out_count) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= X.n) return;
  const int d = find_distro(X.task_off, 0, X.n_distros - 1, p);
  const int64_t q = p - X.task_off[d];
  int64_t off, n;
  if (!gs_list_at(X, counts, d, q, off, n)) return;
  const int64_t j = q - off;
  if (j % (2 * block) != 0 || j + block >= n) return;
  out[gs_slot(out_count)] = {d, int32_t(q), int32_t(q + block), int32_t(off + min(j + 2 * block, n))};
}

// One wave: every queued symMerge call runs on a group of G threads (a warp, or the whole 256-thread CTA).  Its lane 0
// takes Go's steps up to the rotation -- the one-element binary searches or the symmetric search -- and queues the two
// recursive calls; then the group rotates [rs, re) at rm through the same positions of `scratch`.  The last wave of a
// level gets no output queue: a call it would queue there means the wave bound is wrong, and sets *err.
template <int G>
__global__ void __launch_bounds__(256) k_gs_wave(DLegacy X, int32_t* __restrict__ v, int32_t* __restrict__ scratch,
                                                 const GsTask* __restrict__ in, const unsigned int* __restrict__ in_count,
                                                 GsTask* __restrict__ out, unsigned int* __restrict__ out_count, int* __restrict__ err) {
  constexpr int NG = 256 / G;
  __shared__ int32_t s_rot[NG][3];
  const int g = threadIdx.x / G, lane = threadIdx.x % G;
  const int64_t n_in = *in_count;
  for (int64_t t = int64_t(blockIdx.x) * NG + g; t < n_in; t += int64_t(gridDim.x) * NG) {
    const GsTask k = in[t];
    const int64_t base = X.task_off[k.d];
    int32_t* w = v + base;
    if (lane == 0) {
      auto less = [&](int64_t i, int64_t j) { return legacy_more_important(X, base + w[i], base + w[j]); };
      const int64_t a = k.a, m = k.m, b = k.b;
      int64_t rs = 0, rm = 0, re = 0;
      if (m - a == 1) {  // Go swaps data[a] up to i - 1, data[m] down to i: both are rotations by one
        int64_t i = m, j = b;
        while (i < j) { const int64_t h = (i + j) >> 1; if (less(h, a)) i = h + 1; else j = h; }
        rs = a; rm = a + 1; re = i;
      } else if (b - m == 1) {
        int64_t i = a, j = m;
        while (i < j) { const int64_t h = (i + j) >> 1; if (!less(m, h)) i = h + 1; else j = h; }
        rs = i; rm = m; re = m + 1;
      } else {
        const int64_t mid = (a + b) >> 1, n = mid + m;
        int64_t start, r;
        if (m > mid) { start = n - b; r = mid; } else { start = a; r = m; }
        const int64_t p = n - 1;
        while (start < r) { const int64_t c = (start + r) >> 1; if (!less(p - c, c)) start = c + 1; else r = c; }
        const int64_t end = n - start;
        if (start < m && m < end) { rs = start; rm = m; re = end; }
        const bool left = a < start && start < mid, right = mid < end && end < b;
        if ((left || right) && !out) atomicExch(err, 1);
        else {
          if (left) out[gs_slot(out_count)] = {k.d, int32_t(a), int32_t(start), int32_t(mid)};
          if (right) out[gs_slot(out_count)] = {k.d, int32_t(mid), int32_t(end), int32_t(b)};
        }
      }
      s_rot[g][0] = int32_t(rs); s_rot[g][1] = int32_t(rm); s_rot[g][2] = int32_t(re);
    }
    if (G == 32) __syncwarp(); else __syncthreads();
    const int64_t rs = s_rot[g][0], rm = s_rot[g][1], re = s_rot[g][2];
    if (rs < rm && rm < re) {  // rotate: [rm, re) then [rs, rm)
      const int64_t len = re - rs, sh = rm - rs;
      for (int64_t i = lane; i < len; i += G) scratch[base + rs + i] = w[rs + i];
      if (G == 32) __syncwarp(); else __syncthreads();
      for (int64_t i = lane; i < len; i += G) {
        const int64_t s = i + sh;
        w[rs + i] = scratch[base + rs + (s < len ? s : s - len)];
      }
    }
    if (G == 32) __syncwarp(); else __syncthreads();
  }
}
