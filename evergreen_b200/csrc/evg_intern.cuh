// evg_intern.cuh -- evg_intern_columns on the device (evg_intern_batch, evg_upload_strings): task-group keys, versions
// and task ids to dense first-appearance ids per distro, dependency ids to queue indices.
//
// One warp per string.  The lanes read 32 consecutive bytes of the column a step (one or two sectors) and fold each
// (position, byte) through a 64-bit mix; the terms are summed, so a string's hash is one warp reduction.  Each key
// column has an open-addressing table in global memory whose slot is one 64-bit word, hash << 32 | the row that
// claimed it, published by one CAS.  A prober whose hash matches compares its bytes with that row's (the warp again),
// so equal hashes never decide equality and no lane waits on a half-written slot.  The distro is mixed into the hash
// and a claimant must lie in the prober's distro, so one table serves every distro.  atomicMin gives each distinct key
// the first row that carries it: which row claimed a slot depends on atomic order, the first row does not.
#pragma once

struct DStr {  // an evg_str_col staged on the device; n_bytes = off[n], the bytes staged
  const uint8_t* bytes;
  const int64_t* off;
  int64_t n_bytes;
};

struct InView {
  int64_t T, E;
  int32_t D;
  const int64_t* task_off;
  DStr grp, ver, id, dep;  // group keys, versions, task ids (rows), dependency ids (edges)
  const int64_t* dep_off;
  const int32_t* gmh;      // Task.TaskGroupMaxHosts per row
  uint32_t hmask;          // EVG_INTERN_HASH_BITS: the hash is masked to this many bits
  uint64_t cap;            // slots per key column (a power of two, at least twice the rows)
  unsigned long long* key; // three regions of cap slots: group keys, versions, task ids
  uint32_t* first;         // per slot: the first row whose key is there
};
enum : int { kInGroup = 0, kInVersion = 1, kInId = 2 };
// k_in_keys / k_in_deps error bits: a dep_off row, then a bad string row of each column
constexpr int kInErrDepOff = 1, kInErrGroupOff = 2, kInErrVersionOff = 4, kInErrIdOff = 8, kInErrDepIdOff = 16;
constexpr unsigned long long kInEmpty = ~0ull;

__device__ __forceinline__ uint64_t in_mix(uint64_t x) {  // MurmurHash3's 64-bit finaliser
  x ^= x >> 33;
  x *= 0xFF51AFD7ED558CCDull;
  x ^= x >> 33;
  x *= 0xC4CEB9FE1A85EC53ull;
  return x ^ (x >> 33);
}
__device__ __forceinline__ bool in_row_bad(const DStr& s, int64_t o0, int64_t o1) { return o0 < 0 || o1 < o0 || o1 > s.n_bytes; }

// Hash of bytes [o0, o0 + n) of s in distro d, the same on every lane.
__device__ __forceinline__ uint32_t in_hash(const DStr& s, int64_t o0, int64_t n, int d, uint32_t hmask, int lane) {
  uint64_t acc = 0;
  for (int64_t i = lane; i < n; i += 32) acc += in_mix(((uint64_t(i) << 8) | s.bytes[o0 + i]) + 0x9E3779B97F4A7C15ull);
  for (int k = 16; k > 0; k >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, k);
  return uint32_t(in_mix(acc ^ (uint64_t(n) * 0xD6E8FEB86659FD93ull) ^ (uint64_t(uint32_t(d)) << 40)) >> 32) & hmask;
}

// Bytes [a0, a0 + n) of s equal bytes [b0, b0 + n) of k, the same on every lane.
__device__ __forceinline__ bool in_same(const DStr& s, int64_t a0, const DStr& k, int64_t b0, int64_t n, int lane) {
  for (int64_t i = lane; i - lane < n; i += 32)
    if (__any_sync(0xffffffffu, i < n && s.bytes[a0 + i] != k.bytes[b0 + i])) return false;
  return true;
}

// Slot (an index of v.key / v.first) of the key bytes [o0, o0 + n) of s, hash h, in column r among the rows [a, b) of
// its distro.  With `row` >= 0 an absent key is inserted, claimed by `row`; otherwise absent is -1.  Warp-uniform.
__device__ int64_t in_probe(const InView& v, int r, const DStr& s, int64_t o0, int64_t n, uint32_t h, int64_t row, int64_t a,
                            int64_t b, int lane) {
  const DStr& k = r == kInGroup ? v.grp : r == kInVersion ? v.ver : v.id;
  unsigned long long* key = v.key + uint64_t(r) * v.cap;
  const unsigned long long mine = (uint64_t(h) << 32) | uint64_t(row);
  for (uint64_t slot = h & (v.cap - 1);; slot = (slot + 1) & (v.cap - 1)) {
    unsigned long long w = 0;
    if (lane == 0) {
      w = key[slot];
      if (w == kInEmpty && row >= 0) w = atomicCAS(key + slot, kInEmpty, mine);  // kInEmpty back: this row claimed it
    }
    w = __shfl_sync(0xffffffffu, w, 0);
    if (w == kInEmpty) return row >= 0 ? int64_t(uint64_t(r) * v.cap + slot) : -1;
    if (uint32_t(w >> 32) != h) continue;
    const int64_t q = int64_t(uint32_t(w));  // the claimant: its row passed in_row_bad before it claimed
    if (q < a || q >= b) continue;
    const int64_t q0 = k.off[q];
    if (k.off[q + 1] - q0 == n && in_same(s, o0, k, q0, n, lane)) return int64_t(uint64_t(r) * v.cap + slot);
  }
}

// A warp per row: its group key (none when empty), version and task id into their tables; the row's group and version
// slots.  A string row outside its byte column raises its column's error bit and gets no slot.
__global__ void __launch_bounds__(256) k_in_keys(InView v, int64_t* __restrict__ gslot, int64_t* __restrict__ vslot, int* err) {
  const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= v.T) return;
  const int d = find_distro(v.task_off, 0, v.D - 1, t);
  const int64_t a = v.task_off[d], b = v.task_off[d + 1];
  for (int r = kInGroup; r <= kInId; r++) {
    const DStr& s = r == kInGroup ? v.grp : r == kInVersion ? v.ver : v.id;
    const int64_t o0 = s.off[t], o1 = s.off[t + 1];
    int64_t slot = -1;
    if (in_row_bad(s, o0, o1)) {
      if (lane == 0) atomicOr(err, kInErrGroupOff << r);
    } else if (r != kInGroup || o1 > o0) {
      slot = in_probe(v, r, s, o0, o1 - o0, in_hash(s, o0, o1 - o0, d, v.hmask, lane), t, a, b, lane);
      if (lane == 0) atomicMin(v.first + slot, uint32_t(t));
    }
    if (lane == 0 && r == kInGroup) gslot[t] = slot;
    if (lane == 0 && r == kInVersion) vslot[t] = slot;
  }
}

// A warp per row: each DependsOn id looked up among the task ids of the row's distro; res[e] = the distro-local index of
// the first task with that id, -1 when none; cnt[t] = the row's resolved edges.  The row of dep_off is checked here.
__global__ void __launch_bounds__(256) k_in_deps(InView v, int32_t* __restrict__ res, int32_t* __restrict__ cnt, int* err) {
  const int64_t t = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= v.T) return;
  const int64_t e0 = v.dep_off[t], e1 = v.dep_off[t + 1];
  int32_t kept = 0;
  if (e0 < 0 || e1 < e0 || e1 > v.E) {
    if (lane == 0) atomicOr(err, kInErrDepOff);
  } else if (e1 > e0) {
    const int d = find_distro(v.task_off, 0, v.D - 1, t);
    const int64_t a = v.task_off[d], b = v.task_off[d + 1];
    for (int64_t e = e0; e < e1; e++) {
      const int64_t o0 = v.dep.off[e], o1 = v.dep.off[e + 1];
      int32_t j = -1;
      if (in_row_bad(v.dep, o0, o1)) {
        if (lane == 0) atomicOr(err, kInErrDepIdOff);
      } else {
        const int64_t slot = in_probe(v, kInId, v.dep, o0, o1 - o0, in_hash(v.dep, o0, o1 - o0, d, v.hmask, lane), -1, a, b, lane);
        if (slot >= 0) j = int32_t(int64_t(v.first[slot]) - a);
      }
      if (lane == 0) res[e] = j;
      kept += j >= 0;
    }
  }
  if (lane == 0) cnt[t] = kept;
}

// Per row, after k_al_flag and the scans of its flags (pg, pv): the dense group and version ids, the group tables from
// each group's first member, and the lowest row whose TaskGroupMaxHosts differs from its group's first member's.
__global__ void __launch_bounds__(256) k_in_ids(InView v, const int64_t* __restrict__ gslot, const int64_t* __restrict__ vslot,
                                                const int64_t* __restrict__ pg, const int64_t* __restrict__ pv, int32_t* __restrict__ gid,
                                                int32_t* __restrict__ vid, int32_t* __restrict__ gmax, int64_t* __restrict__ gfirst,
                                                unsigned long long* bad_row) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(v.task_off, v.D, t, v.T);
  if (d < 0) return;
  const int64_t a = v.task_off[d];
  int32_t g = -1;
  if (gslot[t] >= 0) {
    const int64_t f = v.first[gslot[t]];
    g = int32_t(pg[f] - pg[a]);
    if (f == t) {
      gmax[pg[t]] = v.gmh[t];
      gfirst[pg[t]] = t;
    } else if (v.gmh[t] != v.gmh[f]) {
      atomicMin(bad_row, (unsigned long long)t);
    }
  }
  gid[t] = g;
  vid[t] = int32_t(pv[v.first[vslot[t]]] - pv[a]);
}

// Per row: its resolved dependencies, in DependsOn order, at dep_off_out[t].
__global__ void __launch_bounds__(256) k_in_edges(InView v, const int32_t* __restrict__ res, const int64_t* __restrict__ dep_off_out,
                                                  int32_t* __restrict__ dep_idx) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= v.T) return;
  int64_t w = dep_off_out[t];
  for (int64_t e = v.dep_off[t]; e < v.dep_off[t + 1]; e++)
    if (res[e] >= 0) dep_idx[w++] = res[e];
}

// ---- evg_queue_index_batch: every persisted queue's items joined by task id --------------------------------------
// FindMinimumQueuePositionForTask and FindDuplicateEnqueuedTasks (model/task_queue.go:407-435, 505-547) for every id at
// once.  The whole item list is one range: one task-id table spans every queue, so the distro mixed into the hash is 0
// and every claimant counts.  The ids sit in InView's first column (grp) and the table in its first region of cap slots.
struct QxView {
  InView v;                 // v.grp: the ids, one row per item; v.key / v.first: cap slots
  int64_t N;                // items
  int32_t Q;                // queues
  const int64_t* item_off;  // Q + 1: the items of queue q are [item_off[q], item_off[q + 1])
};
constexpr int kQxErrIdOff = 1;  // an id row outside its byte column

// A warp per item: its id into the table (slot[i]) and its queue (queue[i]); atomicMin gives each slot its first item.
__global__ void __launch_bounds__(256) k_qx_keys(QxView x, int64_t* __restrict__ slot, int32_t* __restrict__ queue, int* err) {
  const int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= x.N) return;
  const DStr& s = x.v.grp;
  const int64_t o0 = s.off[i], o1 = s.off[i + 1];
  int64_t k = -1;
  if (in_row_bad(s, o0, o1)) {
    if (lane == 0) atomicOr(err, kQxErrIdOff);
  } else {
    k = in_probe(x.v, kInGroup, s, o0, o1 - o0, in_hash(s, o0, o1 - o0, 0, x.v.hmask, lane), i, 0, x.N, lane);
    if (lane == 0) atomicMin(x.v.first + k, uint32_t(i));
  }
  if (lane == 0) {
    slot[i] = k;
    queue[i] = find_distro(x.item_off, 0, x.Q - 1, i);
  }
}

// first-appearance flags: their exclusive scan numbers the distinct ids in first-appearance order
__global__ void __launch_bounds__(256) k_qx_flag(int64_t n, const int64_t* __restrict__ slot, const uint32_t* __restrict__ first,
                                                 int32_t* __restrict__ f) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  f[i] = first[slot[i]] == uint32_t(i);
}

// Per item, after the scan pk of the flags: its id's dense number (key[i]); per id the smallest index in any queue and
// the lowest and highest queue that hold it (two distinct queues: lo != hi).  Mins and maxes: no order of atomics shows.
__global__ void __launch_bounds__(256) k_qx_reduce(QxView x, const int64_t* __restrict__ slot, const int32_t* __restrict__ queue,
                                                   const int64_t* __restrict__ pk, int32_t* __restrict__ key, int32_t* pos, int32_t* qlo,
                                                   int32_t* qhi) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= x.N) return;
  const int64_t k = pk[x.v.first[slot[i]]];
  const int32_t q = queue[i];
  key[i] = int32_t(k);
  atomicMin(pos + k, int32_t(i - x.item_off[q]));
  atomicMin(qlo + k, q);
  atomicMax(qhi + k, q);
}

// Per item: min_position = 1 + its id's smallest index; fm[i] = the id is duplicated; f[i] (the first-appearance flag)
// is kept only for a duplicated id, so its scan numbers the duplicated ids in first-appearance order.
__global__ void __launch_bounds__(256) k_qx_dup(int64_t n, const int32_t* __restrict__ key, const int32_t* __restrict__ pos,
                                                const int32_t* __restrict__ qlo, const int32_t* __restrict__ qhi,
                                                int32_t* __restrict__ min_position, int32_t* __restrict__ f, int32_t* __restrict__ fm) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t k = key[i];
  const bool dup = qlo[k] != qhi[k];
  min_position[i] = pos[k] + 1;
  fm[i] = dup;
  f[i] = f[i] && dup;
}

// Per item of a duplicated id, at pm[i]: the pair (duplicate number << 32 | queue), in item order and so in queue order
// within each id; per duplicated id, its first item (dup_item).
__global__ void __launch_bounds__(256) k_qx_pairs(QxView x, const int64_t* __restrict__ slot, const int32_t* __restrict__ queue,
                                                  const int32_t* __restrict__ fm, const int64_t* __restrict__ pd,
                                                  const int64_t* __restrict__ pm, uint64_t* __restrict__ pairs, int64_t* __restrict__ dup_item) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= x.N || !fm[i]) return;
  const int64_t f = x.v.first[slot[i]];
  pairs[pm[i]] = (uint64_t(pd[f]) << 32) | uint32_t(queue[i]);
  if (f == i) dup_item[pd[i]] = i;
}

// After the pairs are sorted by duplicate number (stably, so each id's queues stay ascending): u[j] = pair j is the
// first of its (id, queue).
__global__ void __launch_bounds__(256) k_qx_uniq(int64_t m, const uint64_t* __restrict__ pairs, int32_t* __restrict__ u) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= m) return;
  u[j] = j == 0 || pairs[j] != pairs[j - 1];
}

// Per pair, after the scan pu of u: the distinct queues at pu[j], and each id's row of dup_off at its first pair.
__global__ void __launch_bounds__(256) k_qx_write(int64_t m, int64_t n_dups, const uint64_t* __restrict__ pairs,
                                                  const int64_t* __restrict__ pu, int64_t* __restrict__ dup_off,
                                                  int32_t* __restrict__ dup_queue) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint64_t p = pairs[j];
  if (j == 0 || p != pairs[j - 1]) dup_queue[pu[j]] = int32_t(uint32_t(p));
  if (j == 0 || (p >> 32) != (pairs[j - 1] >> 32)) dup_off[p >> 32] = pu[j];
  if (j == m - 1) dup_off[n_dups] = pu[m];
}

// ---- evg_edit_strings: the string table of an edited tick, composed on the device ---------------------------------
// Composed row i of distro d is its survivors in their previous order (resident row src[i]), then its inserted rows
// ins_off[d] .. ins_off[d+1] of the staged edit -- compose_tick's map.  Each composed string has a source code: >= 0 a
// row of the resident column, < 0 row ~code of the staged one.  A staged row outside its column raises the lowest
// composed row that holds it (bad_row); it gets length 0, so nothing reads through it.
struct SxMap {
  int32_t D;
  const int64_t* new_off;  // D + 1: composed task_off
  const int64_t* ins_off;  // D + 1: the staged rows' CSR over distros
  const int32_t* src;      // composed row -> resident row, for survivors
};
struct SxCol {  // one string column: the resident one, the staged one, the composed one written here
  DStr res, ins;
  int64_t* out_off;
  uint8_t* out_bytes;
};

// Per composed row: its source code, its TaskGroupMaxHosts and its DependsOn count (a staged dep_off row checked here).
__global__ void __launch_bounds__(256) k_sx_rows(int64_t n, SxMap m, const int32_t* __restrict__ res_gmh, const int32_t* __restrict__ ins_gmh,
                                                 const int64_t* __restrict__ res_dep_off, const int64_t* __restrict__ ins_dep_off,
                                                 int64_t ins_E, int64_t* __restrict__ code, int32_t* __restrict__ gmh,
                                                 int32_t* __restrict__ dep_cnt, unsigned long long* bad_row) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int d = block_find_distro(m.new_off, m.D, i, n);
  if (d < 0) return;
  const int64_t k = i - m.new_off[d], S = (m.new_off[d + 1] - m.new_off[d]) - (m.ins_off[d + 1] - m.ins_off[d]);
  if (k < S) {
    const int64_t t = m.src[i];
    code[i] = t;
    gmh[i] = res_gmh[t];
    dep_cnt[i] = int32_t(res_dep_off[t + 1] - res_dep_off[t]);
  } else {
    const int64_t j = m.ins_off[d] + (k - S), e0 = ins_dep_off[j], e1 = ins_dep_off[j + 1];
    const bool bad = e0 < 0 || e1 < e0 || e1 > ins_E || e1 - e0 > INT32_MAX;
    if (bad) atomicMin(bad_row, (unsigned long long)i);
    code[i] = ~j;
    gmh[i] = ins_gmh[j];
    dep_cnt[i] = bad ? 0 : int32_t(e1 - e0);
  }
}

// Per composed row, after the scan dep_off of the counts: the source code of each of its DependsOn ids.
__global__ void __launch_bounds__(256) k_sx_edges(int64_t n, const int64_t* __restrict__ code, const int64_t* __restrict__ res_dep_off,
                                                  const int64_t* __restrict__ ins_dep_off, const int64_t* __restrict__ dep_off,
                                                  int64_t* __restrict__ ecode) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t c = code[i], w0 = dep_off[i], w1 = dep_off[i + 1];
  const int64_t e0 = c >= 0 ? res_dep_off[c] : ins_dep_off[~c];
  for (int64_t w = w0; w < w1; w++) ecode[w] = c >= 0 ? e0 + (w - w0) : ~(e0 + (w - w0));
}

// Per composed string: its length (scanned into out_off next).  owner_off: the composed dep_off when the strings are
// DependsOn ids (a bad one names its row), NULL when string r is row r.
__global__ void __launch_bounds__(256) k_sx_len(int64_t n, const int64_t* __restrict__ code, SxCol col, const int64_t* __restrict__ owner_off,
                                                int32_t n_owner, int32_t* __restrict__ len, unsigned long long* bad_row) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int64_t c = code[r], q = c >= 0 ? c : ~c;
  const int64_t* __restrict__ off = c >= 0 ? col.res.off : col.ins.off;
  const int64_t o0 = off[q], o1 = off[q + 1];
  if (c < 0 && (in_row_bad(col.ins, o0, o1) || o1 - o0 > INT32_MAX)) {
    atomicMin(bad_row, (unsigned long long)(owner_off ? find_distro(owner_off, 0, n_owner - 1, r) : r));
    len[r] = 0;
  } else {
    len[r] = int32_t(o1 - o0);
  }
}

// Bytes [0, n) of src to dst by one warp, V-wide where both are V-aligned (their distance is a multiple of V).
template <class V>
__device__ __forceinline__ void sx_copy_as(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int64_t n, int lane) {
  constexpr int W = sizeof(V);
  const int64_t head = min(n, int64_t((W - (reinterpret_cast<uintptr_t>(dst) & (W - 1))) & (W - 1)));
  for (int64_t i = lane; i < head; i += 32) dst[i] = src[i];
  const int64_t nv = (n - head) / W;
  V* __restrict__ d = reinterpret_cast<V*>(dst + head);
  const V* __restrict__ s = reinterpret_cast<const V*>(src + head);
  for (int64_t v = lane; v < nv; v += 32) d[v] = s[v];
  for (int64_t i = head + nv * W + lane; i < n; i += 32) dst[i] = src[i];
}

// A warp per composed string: its bytes from its source column to out_off[r].
__global__ void __launch_bounds__(256) k_sx_copy(int64_t n, const int64_t* __restrict__ code, SxCol col) {
  const int64_t r = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int64_t o = col.out_off[r], len = col.out_off[r + 1] - o;
  if (len == 0) return;
  const int64_t c = code[r];
  const uint8_t* src = c >= 0 ? col.res.bytes + col.res.off[c] : col.ins.bytes + col.ins.off[~c];
  uint8_t* dst = col.out_bytes + o;
  const uintptr_t mis = reinterpret_cast<uintptr_t>(src) ^ reinterpret_cast<uintptr_t>(dst);
  if ((mis & 15) == 0) sx_copy_as<uint4>(dst, src, len, lane);
  else if ((mis & 7) == 0) sx_copy_as<uint2>(dst, src, len, lane);
  else if ((mis & 3) == 0) sx_copy_as<uint32_t>(dst, src, len, lane);
  else sx_copy_as<uint8_t>(dst, src, len, lane);
}
