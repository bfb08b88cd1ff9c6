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
