// evg_next.cuh -- the DAG dispatcher's FindNextTask (SURVEY.md §8 f.3): what reads d.sorted and d.taskGroups.
//
// Reference: basicCachedDAGDispatcherImpl.FindNextTask (model/task_queue_service_dependency.go:258-469) with
// tryMarkItemDispatched :486-498, tryMarkNextTaskGroupTaskDispatched :500-519, getTaskGroup :524-538,
// checkMaxConcurrentLargeParserProjectTasks :549-603, nextTaskGroupTask :614-692, isBlockedSingleHostTaskGroup :696-698;
// restated on the CPU in oracle/oracle_dispatch.py.
//
// Every database answer of one call is a frozen snapshot (evg_next_db).  k_next_verdict folds it and the item's own
// fields into one word per item, independent of dispatcher state; k_next_serve, one WARP per distro, serves the
// distro's requests in order against the state in HBM: the walk over d.sorted and the scans over a unit's tasks go
// 32 entries at a time, __ballot_sync picks the first entry that needs action and lane 0 applies the state change.
#pragma once

// verdict word of an item (k_next_verdict)
constexpr uint32_t kNvStandMask = 0x3;    // the standalone path after the mark (:312-401): ...
constexpr uint32_t kNvStandTake = 1;      //   handed out unless the request's AMI rule skips it (:392)
constexpr uint32_t kNvStandSkip = 2;      //   skipped: started, generate limit, parser limit, dependencies
constexpr uint32_t kNvStandGiveUp = 3;    //   the request returns nil: no task document, no version
constexpr uint32_t kNvGroupPath = 0x4;    // GroupMaxHosts != 0 (:305)
constexpr uint32_t kNvUnitShift = 3;      // nextTaskGroupTask's verdict on the task as a unit member (:630-677): ...
constexpr uint32_t kNvUnitSkip = 0, kNvUnitTake = 1, kNvUnitNotFound = 2;
constexpr uint32_t kNvBlocked = 0x20;     // found, finished and not succeeded: blocks a single-host unit (:696-698)
constexpr uint32_t kNvWalkShift = 6;      // the walk's parser check on a unit's task after the mark (:456-462): ...
constexpr uint32_t kNvWalkReturn = 0, kNvWalkSkip = 1, kNvWalkGiveUp = 2;
constexpr uint32_t kNvDepsMet = 0x100;    // TaskQueueItem.DependenciesMet, as persisted
// state bits of an item
constexpr uint8_t kNsNode = EVG_NS_NODE, kNsUnit = EVG_NS_UNIT;

struct DNext {
  int64_t n;                    // items
  const int64_t* item_off;      // [D+1]
  const int64_t* group_off;     // [D+1]
  const int32_t* sorted;        // [n] d.sorted: item, -1 for a cycle
  const int32_t* n_sorted;      // [D]
  const int32_t* unit_items;    // [n]
  const int32_t* unit_off;      // [G+D], each distro's closing entry included
  const int32_t* group_id;      // [n] dense group id, -1 = Group == ""
  const int32_t* gmh;           // [n] GroupMaxHosts
  const uint8_t* deps_met;      // [n] DependenciesMet
  int32_t* gfirst;              // [G] first item (queue order) of each group: its GroupMaxHosts is the unit's maxHosts (:172-180)
  int32_t* unit_max;            // [G]
  uint16_t* verdict;            // [n]
  uint8_t* bits;                // [n] state: kNsNode | kNsUnit
  uint8_t* deleted;             // [G] state: the unit left d.taskGroups
  int32_t* running;             // [G] state: the unit's cached runningHosts
  uint8_t* inert;               // [G] per call: the walk found the unit unable to yield under this snapshot
};

// The unit's maxHosts is the GroupMaxHosts of the group's first item in queue order (:166-186).
__global__ void __launch_bounds__(256) k_next_first(DNext X, int32_t n_distros) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(X.item_off, n_distros, j, X.n);
  if (d < 0) return;
  const int32_t g = X.group_id[j];
  if (g >= 0) atomicMin(X.gfirst + X.group_off[d] + g, int32_t(j - X.item_off[d]));
}
__global__ void __launch_bounds__(256) k_next_unit_max(DNext X, int32_t n_distros) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(X.item_off, n_distros, j, X.n);
  if (d < 0) return;
  const int32_t g = X.group_id[j];
  if (g >= 0 && X.gfirst[X.group_off[d] + g] == int32_t(j - X.item_off[d])) X.unit_max[X.group_off[d] + g] = X.gmh[j];
}

struct DNextDb {
  const uint8_t* flags;          // [n] EVG_ND_*
  const int32_t* est_generated;  // [n]
  int32_t generate_limit, pending_generate, max_large_parser, num_large_parser;
};

// One thread per item: everything FindNextTask would learn about the item from the database, decided once per call.
__global__ void __launch_bounds__(256) k_next_verdict(DNext X, DNextDb B) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= X.n) return;
  const uint32_t f = B.flags[j];
  const bool found = f & EVG_ND_FOUND;
  const bool deps_now = !(f & EVG_ND_DEPS_ERR) && (f & EVG_ND_DEPS_MET_NOW);
  // checkMaxConcurrentLargeParserProjectTasks as its call sites use the two results (:365-371, :456-462)
  uint32_t parser = kNvWalkReturn;
  if (B.max_large_parser > 0) {
    if (!(f & EVG_ND_VERSION_FOUND)) parser = kNvWalkGiveUp;
    else if ((f & EVG_ND_VERSION_S3) && (B.num_large_parser < 0 || B.num_large_parser >= B.max_large_parser)) parser = kNvWalkSkip;
  }
  uint32_t v = X.deps_met[j] ? kNvDepsMet : 0;
  if (X.gmh[j] != 0) {
    v |= kNvGroupPath;
  } else if (X.deps_met[j]) {
    uint32_t s = kNvStandTake;
    const int32_t est = B.est_generated[j];
    if (!found) s = kNvStandGiveUp;
    else if (f & EVG_ND_STARTED) s = kNvStandSkip;
    else if (B.generate_limit > 0 && est > 0 &&
             (B.pending_generate < 0 || int64_t(B.pending_generate) + est >= B.generate_limit)) s = kNvStandSkip;  // :341-363
    else if (parser == kNvWalkGiveUp) s = kNvStandGiveUp;
    else if (parser == kNvWalkSkip || !deps_now) s = kNvStandSkip;
    v |= s;
  }
  // as a member of a unit (whatever its own GroupMaxHosts): :630-677 in the reference's order
  uint32_t u = kNvUnitTake;
  if (!found) u = kNvUnitNotFound;
  else if ((f & EVG_ND_STARTED_GROUP) || !deps_now) u = kNvUnitSkip;
  v |= u << kNvUnitShift;
  if (found && (f & EVG_ND_FINISHED_NOT_SUCCEEDED)) v |= kNvBlocked;
  v |= parser << kNvWalkShift;
  X.verdict[j] = uint16_t(v);
}

struct DNextReq {
  const int32_t* list;        // the distros that have requests
  int32_t n_list;
  const int64_t* req_off;     // [D+1]
  const int32_t* group;       // per request
  const int64_t* ami;         // per request, 0 = zero time
  const int64_t* ingest_ns;   // [n] snapshot
  const int32_t* running_db;  // [G] snapshot
  int32_t* item;              // per request
  int32_t* outcome;
};

// getTaskGroup's hasDispatchableTask (:531-536) for unit [u0, u1) of the distro at `base`; warp-wide.
__device__ __forceinline__ bool next_has_dispatchable(const DNext& X, int64_t base, int u0, int u1, int lane) {
  for (int p = u0; p < u1; p += 32) {
    const int q = p + lane;
    bool yes = false;
    if (q < u1) {
      const int32_t it = X.unit_items[base + q];
      yes = (X.verdict[base + it] & kNvDepsMet) && !(X.bits[base + it] & kNsUnit);
    }
    if (__any_sync(0xffffffffu, yes)) return true;
  }
  return false;
}

// tryMarkNextTaskGroupTaskDispatched (:500-519) over nextTaskGroupTask (:614-692) for group g (global index) of the
// distro at `base`; warp-wide, every lane returns the item or -1.  The first task of the unit that is not yet marked in
// the unit's copy and is not skipped decides: no document -> nil; a blocked single-host unit -> deleted, nil; else it
// is marked in both copies, and the unit is deleted when it sits at the unit's last position.
__device__ __forceinline__ int32_t next_group_task(const DNext& X, int64_t base, int64_t g, int u0, int u1, int lane) {
  const bool single = X.unit_max[g] == 1;
  for (int p = u0; p < u1; p += 32) {
    const int q = p + lane;
    int32_t it = -1;
    uint32_t v = 0;
    bool stop = false;
    if (q < u1) {
      it = X.unit_items[base + q];
      if (!(X.bits[base + it] & kNsUnit)) {
        v = X.verdict[base + it];
        stop = ((v >> kNvUnitShift) & 3) != kNvUnitSkip || (single && (v & kNvBlocked));
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, stop);
    if (!m) continue;
    const int l = __ffs(m) - 1;
    it = __shfl_sync(0xffffffffu, it, l);
    v = __shfl_sync(0xffffffffu, v, l);
    const uint32_t cls = (v >> kNvUnitShift) & 3;
    int32_t res = -1;
    if (cls != kNvUnitNotFound) {
      const bool blocked = single && (v & kNvBlocked);
      if (!blocked) res = it;
      if (lane == 0) {
        if (blocked) X.deleted[g] = 1;
        else {
          X.bits[base + it] |= kNsNode | kNsUnit;
          if (p + l == u1 - 1) X.deleted[g] = 1;
        }
      }
    }
    __syncwarp();
    return res;
  }
  return -1;
}

__global__ void __launch_bounds__(128) k_next_serve(DNext X, DNextReq R) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= R.n_list) return;
  const int d = R.list[w];
  const int64_t base = X.item_off[d], G0 = X.group_off[d];
  const int64_t U = G0 + d;  // the distro's unit offsets
  const int ns = X.n_sorted[d];
  for (int64_t r = R.req_off[d]; r < R.req_off[d + 1]; r++) {
    const int64_t ami = R.ami[r];
    int32_t item = -1, outcome = -1;
    // "If the host just ran a task group, give it one back" (:268-282): neither runningHosts nor the AMI is looked at
    const int32_t sg = R.group[r];
    if (sg >= 0 && !X.deleted[G0 + sg]) {
      item = next_group_task(X, base, G0 + sg, X.unit_off[U + sg], X.unit_off[U + sg + 1], lane);
      if (item >= 0) outcome = EVG_NEXT_FOUND;
    }
    int pos = 0;
    while (outcome < 0 && pos < ns) {
      int32_t e = pos + lane < ns ? X.sorted[base + pos + lane] : -1;  // -1: a cycle's placeholder (:290-292)
      uint32_t v = 0;
      bool act = false;
      if (e >= 0) {
        v = X.verdict[base + e];
        if (v & kNvGroupPath) {
          const int32_t g = X.group_id[base + e];
          act = g >= 0 && !X.deleted[G0 + g] && !X.inert[G0 + g];
        } else {
          act = (v & kNvStandMask) != 0 && !(X.bits[base + e] & kNsNode);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, act);
      if (!m) { pos += 32; continue; }
      const int l = __ffs(m) - 1;
      e = __shfl_sync(0xffffffffu, e, l);
      v = __shfl_sync(0xffffffffu, v, l);
      pos += l + 1;  // the walk resumes behind this entry
      if (!(v & kNvGroupPath)) {
        if (lane == 0) X.bits[base + e] |= kNsNode;  // marked before any database check (:309)
        __syncwarp();
        const uint32_t s = v & kNvStandMask;
        if (s == kNvStandGiveUp) outcome = EVG_NEXT_GAVE_UP;
        else if (s == kNvStandTake && !(ami != 0 && R.ingest_ns[base + e] > ami)) { item = e; outcome = EVG_NEXT_FOUND; }
        continue;
      }
      const int64_t g = G0 + X.group_id[base + e];
      const int u0 = X.unit_off[U + (g - G0)], u1 = X.unit_off[U + (g - G0) + 1];
      // Under one snapshot a unit that cannot yield now cannot yield later in the call (its bits only get set, its
      // cached runningHosts only moves while it is below maxHosts): remember that instead of scanning it per entry.
      bool dead = !next_has_dispatchable(X, base, u0, u1, lane);
      if (!dead && X.running[g] < X.unit_max[g]) {  // :411
        const int32_t hosts = R.running_db[g];
        if (hosts < 0) { outcome = EVG_NEXT_GAVE_UP; continue; }  // :413-425
        if (lane == 0) X.running[g] = hosts;
        __syncwarp();
        if (hosts < X.unit_max[g]) {
          const int32_t t = next_group_task(X, base, g, u0, u1, lane);
          if (t >= 0) {
            const uint32_t wv = (X.verdict[base + t] >> kNvWalkShift) & 3;
            if (wv == kNvWalkGiveUp) outcome = EVG_NEXT_GAVE_UP;
            else if (wv == kNvWalkReturn) { item = t; outcome = EVG_NEXT_FOUND; }
            continue;  // kNvWalkSkip: the parser limit's `continue` comes after the mark (:460)
          }
          dead = true;  // nil: no document, everything skipped, or the unit was just deleted
        } else dead = true;
      } else dead = true;
      if (lane == 0) X.inert[g] = 1;
      __syncwarp();
    }
    if (lane == 0) {
      R.item[r] = item;
      R.outcome[r] = outcome < 0 ? EVG_NEXT_NONE : outcome;
    }
  }
}

// The chained call's per-item fields, gathered from the tick when the dispatchers are built: GroupMaxHosts and
// DependenciesMet as evg_download_queue reports them for rank j - item_off[d].
__global__ void __launch_bounds__(256) k_next_gather(int32_t n_distros, int64_t n, const int64_t* __restrict__ item_off,
                                                     const int64_t* __restrict__ task_off, const int64_t* __restrict__ tick_group_off,
                                                     const int32_t* __restrict__ row, const int32_t* __restrict__ gid,
                                                     const int32_t* __restrict__ gmax, const uint32_t* __restrict__ flags,
                                                     int32_t* __restrict__ gmh, uint8_t* __restrict__ deps_met) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(item_off, n_distros, j, n);
  if (d < 0) return;
  const int32_t i = row[j];
  if (i < 0) { gmh[j] = 0; deps_met[j] = 0; return; }
  const int64_t t = task_off[d] + i;
  const int32_t g = gid[t];
  gmh[j] = g >= 0 ? gmax[tick_group_off[d] + g] : 0;
  deps_met[j] = (flags[t] & EVG_TF_DEPS_MET) ? 1 : 0;
}
// each distro's closing unit offset on the device (the rebuild writes it on the host only)
__global__ void __launch_bounds__(256) k_next_close(int32_t n_distros, const int64_t* __restrict__ group_off,
                                                    const int32_t* __restrict__ grouped, int32_t* __restrict__ unit_off) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d < n_distros) unit_off[group_off[d + 1] + d] = grouped[d];
}
