// Trace grouping on the GPU: the body of the reference's preprocess.py main() after get_df() (:269-381).
//
// The reference walks a pandas frame: groupby("traceid").apply(" ".join) over a string column gives every trace its
// runtime key (factorized into runtime ids), then for every entry a groupby("traceid") visits the traces one Python
// iteration each, counting runtimes per entry and building a graph from the first trace of every runtime it meets.
// Here the whole table is processed at once, with integer keys only:
//   1. group by traceid: count rows per traceid, scan, atomic fill, then every trace's slots are rank-sorted by row id
//      (file order); memory O(R + max traceid);
//   2. one warp per trace: bucket = floor(min timestamp / 30000) * 30000, y = max |rt|, the entry and its consistency,
//      and two order-sensitive 64-bit hashes = sums over rows of a mix of (position, um, dm, interface);
//   3. one warp per trace inserts it into an open-addressing table: a slot matches when the hashes and the length agree
//      AND a row-by-row comparison with the slot's owner agrees.  atomicMin of the trace index per group gives the
//      smallest traceid; runtime ids are a scan of "first member" flags in traceid order (= Series.factorize);
//   4. stable counting sort of the traces by entry (per-tile histograms, rank inside a tile of 1024 traces): the
//      iteration order of tr2data;
//   5. representative of a runtime = its member with the smallest iteration position (atomicMin); a second table keyed
//      (entry, runtime) holds count and first position; scans of the two "first" flags over positions give the
//      runtime-insertion order and each entry's key order; probability = count / entry total in fp64 (IEEE division,
//      the same correctly rounded quotient as Python's int / int below 2^53).
// Every atomic is a min, an add or a slot claim whose winner does not change any output, so the results do not depend
// on scheduling.
#include "common.cuh"
#include "scan.cuh"

#include <algorithm>

namespace {

constexpr int TG_WARPS = 8;             // warps per CTA of the warp-per-trace kernels
constexpr int TG_SHORT = 1024;          // longer traces are rank-sorted by a whole CTA
constexpr int TG_TILE = 1024;           // traces per tile of the entry counting sort
constexpr int TG_EMPTY = -1;
constexpr unsigned long long TG_NOKEY = ~0ull;

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {   // splitmix64 finaliser
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ unsigned long long row_mix(unsigned long long seed, int pos, int64_t um, int64_t dm,
                                                      int64_t itf) {
  unsigned long long h = mix64(seed ^ (unsigned long long)pos);
  h = mix64(h ^ (unsigned long long)um);
  h = mix64(h ^ (unsigned long long)dm);
  return mix64(h ^ (unsigned long long)itf);
}

__device__ __forceinline__ bool valid_id(int64_t v) { return v >= 0 && v <= 0x7fffffffLL; }

__global__ void k_range(PertSpanTable tab, int* maxes, int* status) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= tab.R) return;
  const int64_t tid = tab.traceid[r], ent = tab.entryid[r];
  if (!valid_id(tid) || !valid_id(ent)) {
    atomicExch(status, PERT_ERR_RANGE);
    if (!valid_id(tid)) return;
  } else {
    atomicMax(&maxes[1], (int)ent);
  }
  atomicMax(&maxes[0], (int)tid);
}

__global__ void k_key_count(PertSpanTable tab, long long n_keys, int* key_ptr, int* key_trace) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= tab.R) return;
  const int64_t tid = tab.traceid[r];
  if (!valid_id(tid) || tid >= n_keys) return;
  atomicAdd(&key_ptr[tid + 1], 1);
  key_trace[tid + 1] = 1;
}

// traceid k present (key_trace steps) -> trace t = key_trace[k]: its first row slot and id
__global__ void k_compact_keys(long long n_keys, const int* key_ptr, const int* key_trace, int* row_ptr,
                               int64_t* trace_id) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_keys) return;
  if (k == n_keys) {
    row_ptr[key_trace[k]] = key_ptr[k];
    return;
  }
  const int t = key_trace[k];
  if (key_trace[k + 1] != t) {
    row_ptr[t] = key_ptr[k];
    trace_id[t] = k;
  }
}

__global__ void k_fill(PertSpanTable tab, long long n_keys, const int* key_ptr, const int* key_trace, int* fill,
                       int* slot) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= tab.R) return;
  const int64_t tid = tab.traceid[r];
  if (!valid_id(tid) || tid >= n_keys) return;
  slot[key_ptr[tid] + atomicAdd(&fill[key_trace[tid]], 1)] = (int)r;
}

// warp per trace: row ids are unique, so a slot's rank among its trace's slots is its file-order position
__global__ void __launch_bounds__(TG_WARPS * 32) k_sort_short(long long T, const int* row_ptr, const int* slot,
                                                              int* perm, int* long_list, int* long_count) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int b = row_ptr[t], len = row_ptr[t + 1] - b;
  if (len > TG_SHORT) {
    if (lane == 0) long_list[atomicAdd(long_count, 1)] = (int)t;
    return;
  }
  for (int i = lane; i < len; i += 32) {
    const int x = __ldg(slot + b + i);
    int rank = 0;
    for (int j = 0; j < len; ++j) rank += (__ldg(slot + b + j) < x);
    perm[b + rank] = x;
  }
}

__global__ void __launch_bounds__(256) k_sort_long(const int* row_ptr, const int* slot, int* perm,
                                                   const int* long_list, const int* long_count) {
  __shared__ int tile[1024];
  const int cnt = *long_count;
  for (int k = blockIdx.x; k < cnt; k += gridDim.x) {
    const int t = long_list[k];
    const int b = row_ptr[t], len = row_ptr[t + 1] - b;
    for (int i0 = 0; i0 < len; i0 += blockDim.x) {
      const int i = i0 + threadIdx.x;
      const int x = (i < len) ? slot[b + i] : 0;
      int rank = 0;
      for (int j0 = 0; j0 < len; j0 += 1024) {
        const int m = min(1024, len - j0);
        __syncthreads();
        for (int j = threadIdx.x; j < m; j += blockDim.x) tile[j] = slot[b + j0 + j];
        __syncthreads();
        if (i < len)
          for (int j = 0; j < m; ++j) rank += (tile[j] < x);
      }
      if (i < len) perm[b + rank] = x;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ int64_t warp_min64(int64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, (int64_t)__shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int64_t warp_max64(int64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, (int64_t)__shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// warp per trace: bucket, y, entry (+ consistency) and the two hashes, in one pass over the grouped rows
__global__ void __launch_bounds__(TG_WARPS * 32) k_trace_reduce(PertSpanTable tab, long long T, long long n_ent,
                                                                int hash_bits, const int* row_ptr, const int* perm,
                                                                int64_t* bucket, int64_t* y, int* entry,
                                                                unsigned long long* h1, unsigned long long* h2,
                                                                int* status) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int b = row_ptr[t], len = row_ptr[t + 1] - b;
  const int64_t e0 = tab.entryid[perm[b]];
  int64_t tmin = INT64_MAX, amax = 0;
  unsigned long long s1 = 0, s2 = 0;
  bool mixed = false;
  for (int i = lane; i < len; i += 32) {
    const int r = perm[b + i];
    const int64_t ts = tab.timestamp[r], rt = tab.rt[r];
    tmin = min(tmin, ts);
    amax = max(amax, rt < 0 ? -rt : rt);
    mixed |= tab.entryid[r] != e0;
    const int64_t um = tab.um[r], dm = tab.dm[r], itf = tab.interface[r];
    s1 += row_mix(0x243f6a8885a308d3ull, i, um, dm, itf);
    s2 += row_mix(0x13198a2e03707344ull, i, um, dm, itf);
  }
  tmin = warp_min64(tmin);
  amax = warp_max64(amax);
  s1 = warp_sum64(s1);
  s2 = warp_sum64(s2);
  mixed = __any_sync(0xffffffffu, mixed);
  if (lane == 0) {
    bucket[t] = pert_time_bucket(tmin);                  // floor division (pandas //)
    y[t] = amax;
    const bool ok = !mixed && e0 >= 0 && e0 < n_ent;
    if (!ok) atomicExch(status, PERT_ERR_RANGE);        // a trace filed under two entries (or an entry out of range)
    entry[t] = ok ? (int)e0 : 0;
    const unsigned long long mask = hash_bits >= 64 ? ~0ull : ((1ull << hash_bits) - 1);
    h1[t] = s1 & mask;
    h2[t] = s2 & mask;
  }
}

__device__ __forceinline__ bool same_rows(PertSpanTable tab, const int* perm, int a, int b, int len, int lane) {
  bool eq = true;
  for (int i = lane; i < len && eq; i += 32) {
    const int ra = perm[a + i], rb = perm[b + i];
    eq = tab.um[ra] == tab.um[rb] && tab.dm[ra] == tab.dm[rb] && tab.interface[ra] == tab.interface[rb];
  }
  return __all_sync(0xffffffffu, eq);
}

// warp per trace: find (or claim) the slot of its runtime; slots only ever go from empty to an owner
__global__ void __launch_bounds__(TG_WARPS * 32) k_runtime_insert(PertSpanTable tab, long long T, long long S,
                                                                  const int* row_ptr, const int* perm,
                                                                  const unsigned long long* h1,
                                                                  const unsigned long long* h2, int* owner,
                                                                  int* gmin, int* gcnt, int* slot_of) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int b = row_ptr[t], len = row_ptr[t + 1] - b;
  const unsigned long long a1 = h1[t], a2 = h2[t];
  long long s = (long long)(mix64(a1 ^ mix64(a2 ^ (unsigned long long)len)) & (unsigned long long)(S - 1));
  for (;;) {
    int o = 0;
    if (lane == 0) o = atomicCAS(&owner[s], TG_EMPTY, (int)t);
    o = __shfl_sync(0xffffffffu, o, 0);
    if (o == TG_EMPTY) break;                                            // claimed: a new runtime
    const int ob = row_ptr[o];
    if (h1[o] == a1 && h2[o] == a2 && row_ptr[o + 1] - ob == len && same_rows(tab, perm, b, ob, len, lane)) break;
    s = (s + 1) & (S - 1);
  }
  if (lane == 0) {
    atomicMin(&gmin[s], (int)t);
    atomicAdd(&gcnt[s], 1);
    slot_of[t] = (int)s;
  }
}

__global__ void k_first_flags(long long T, const int* slot_of, const int* gmin, int* flags) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) flags[t + 1] = gmin[slot_of[t]] == t;
}

// flags (scanned) -> runtime id = rank of the group's smallest trace among the groups' smallest traces
__global__ void k_runtime_assign(long long T, const int* slot_of, const int* gmin, const int* gcnt, const int* flags,
                                 int* runtime, int* occurrences) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int s = slot_of[t], f = gmin[s], rid = flags[f];
  runtime[t] = rid;
  if (f == t) occurrences[rid] = gcnt[s];
}

// stable counting sort by entry, part 1: rank of every trace among the earlier traces of its entry inside its tile;
// the last trace of an entry in the tile stores the tile's count
__global__ void __launch_bounds__(TG_TILE) k_entry_rank(long long T, int n_tiles, const int* entry, int* rank,
                                                        int* hist) {
  __shared__ int es[TG_TILE];
  const long long t = (long long)blockIdx.x * TG_TILE + threadIdx.x;
  const int e = t < T ? entry[t] : -1;
  es[threadIdx.x] = e;
  __syncthreads();
  if (t >= T) return;
  int before = 0, after = 0;
  for (int j = 0; j < TG_TILE; ++j) {
    const bool m = es[j] == e;
    before += m && j < (int)threadIdx.x;
    after += m && j > (int)threadIdx.x;
  }
  rank[t] = before;
  if (after == 0) hist[(long long)e * n_tiles + blockIdx.x + 1] = before + 1;
}

__global__ void k_entry_place(long long T, int n_tiles, const int* entry, const int* rank, const int* hist,
                              int* order, int* pos_of) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int p = hist[(long long)entry[t] * n_tiles + t / TG_TILE] + rank[t];
  order[p] = (int)t;
  pos_of[t] = p;
}

__global__ void k_entry_ptr(long long n_ent, int n_tiles, const int* hist, int* ent_trace_ptr) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e <= n_ent) ent_trace_ptr[e] = hist[e * n_tiles];
}

__global__ void k_rep_min(long long T, const int* runtime, const int* pos_of, int* rep_pos) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) atomicMin(&rep_pos[runtime[t]], pos_of[t]);
}

// position p: (entry, runtime) pair into the second table; flag the first position of every runtime
__global__ void k_pair_insert(long long T, long long S, const int* order, const int* entry, const int* runtime,
                              const int* rep_pos, unsigned long long* pkey, int* pfirst, int* pcnt, int* pslot,
                              int* ins_flags) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= T) return;
  const int t = order[p], rid = runtime[t];
  const unsigned long long key = ((unsigned long long)(unsigned)entry[t] << 32) | (unsigned)rid;
  long long s = (long long)(mix64(key) & (unsigned long long)(S - 1));
  for (;;) {
    const unsigned long long o = atomicCAS(&pkey[s], TG_NOKEY, key);
    if (o == TG_NOKEY || o == key) break;
    s = (s + 1) & (S - 1);
  }
  atomicMin(&pfirst[s], (int)p);
  atomicAdd(&pcnt[s], 1);
  pslot[p] = (int)s;
  ins_flags[p + 1] = rep_pos[rid] == p;
}

__global__ void k_pair_flags(long long T, const int* pslot, const int* pfirst, int* pair_flags) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < T) pair_flags[p + 1] = pfirst[pslot[p]] == p;
}

// scanned flags -> the runtime-insertion arrays and the entry mixes
__global__ void k_emit(long long T, const int* order, const int* entry, const int* runtime, const int* row_ptr,
                       const int* ins_flags, const int* pair_flags, const int* pslot, const int* pcnt,
                       const int* ent_trace_ptr, PertTraceGroups out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= T) return;
  const int t = order[p], rid = runtime[t];
  const int k = ins_flags[p];
  if (ins_flags[p + 1] != k) {
    out.ins_runtime[k] = rid;
    out.rep_trace[k] = t;
    out.runtime_ins[rid] = k;
    out.rep_ptr[k + 1] = row_ptr[t + 1] - row_ptr[t];
  }
  const int q = pair_flags[p];
  if (pair_flags[p + 1] != q) {
    const int e = entry[t];
    out.pair_runtime[q] = rid;
    out.pair_prob[q] = (double)pcnt[pslot[p]] / (double)(ent_trace_ptr[e + 1] - ent_trace_ptr[e]);
  }
}

__global__ void k_ent_pair_ptr(long long n_ent, const int* ent_trace_ptr, const int* pair_flags, int* ent_pair_ptr) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e <= n_ent) ent_pair_ptr[e] = pair_flags[ent_trace_ptr[e]];
}

__global__ void k_sizes(long long T, const int* ins_flags, const int* pair_flags, const int* rep_ptr,
                        int64_t* sizes) {
  sizes[0] = ins_flags[T];
  sizes[1] = pair_flags[T];
  sizes[2] = rep_ptr[T];
}

// warp per representative: its rows, file order, in the 8 gathered columns
__global__ void __launch_bounds__(TG_WARPS * 32) k_gather(PertSpanTable tab, const int* perm, const int* row_ptr,
                                                          const int* rep_trace, const int* rep_ptr, long long n_rt,
                                                          long long R2, int64_t* rows) {
  const long long k = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= n_rt) return;
  const int t = rep_trace[k], b = row_ptr[t], len = row_ptr[t + 1] - b, o = rep_ptr[k];
  for (int i = lane; i < len; i += 32) {
    const int r = perm[b + i];
    const long long j = (long long)o + i;
    const int64_t ts = tab.timestamp[r], rt = tab.rt[r];
    rows[j] = tab.um[r];
    rows[R2 + j] = tab.dm[r];
    rows[2 * R2 + j] = tab.interface[r];
    rows[3 * R2 + j] = tab.rpctype[r];
    rows[4 * R2 + j] = ts;
    rows[5 * R2 + j] = ts + (rt < 0 ? -rt : rt);           // endTimestamp, preprocess.py:263
    rows[6 * R2 + j] = tab.rpcid[r];
    rows[7 * R2 + j] = rt;
  }
}

bool table_ok(const PertSpanTable* t) {
  return t && t->R >= 0 && t->R <= 0x7ffffff0LL &&
         (t->R == 0 || (t->traceid && t->timestamp && t->rpcid && t->um && t->dm && t->interface && t->rpctype &&
                        t->rt && t->entryid));
}

long long table_size(long long T) {            // power of two >= 2T: every probe sequence ends at an empty slot
  long long S = 64;
  while (S < 2 * T) S <<= 1;
  return S;
}

long long n_tiles_of(long long T) { return (T + TG_TILE - 1) / TG_TILE; }

int scan(int* a0, int* a1, long long L, int* bsum, cudaStream_t st) {   // inclusive, in place; a1 may be NULL
  const int nb = pert_cdiv(L, SCAN_TILE), ny = a1 ? 2 : 1;
  k_scan_tile_sums<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
  k_scan_block_sums<<<dim3(1, ny), SCAN_THREADS, 0, st>>>(bsum, nb);
  k_scan_apply<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long scan_bytes(long long L) { return 2LL * pert_cdiv(L, SCAN_TILE) * 4 + 16; }

}  // namespace

extern "C" {

int pert_trace_group_range(const PertSpanTable* table, int* maxes, int* status, void* stream_) {
  if (!table_ok(table) || !maxes || !status) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  cudaError_t e;
  if ((e = cudaMemsetAsync(maxes, 0xff, 2 * sizeof(int), st)) != cudaSuccess) return (int)e;
  if (table->R == 0) return PERT_OK;
  k_range<<<pert_cdiv(table->R, 256), 256, 0, st>>>(*table, maxes, status);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_trace_group_workspace_bytes(long long R, long long n_keys, long long T, long long n_ent) {
  if (R < 0 || n_keys < 0 || n_keys > 0x80000000LL || R > 0x7ffffff0LL) return PERT_ERR_BADARG;
  if (T < 0) return scan_bytes(n_keys + 1);
  if (T > R || n_ent < 0) return PERT_ERR_BADARG;
  const long long S = table_size(T), H = n_ent * n_tiles_of(T) + 1;
  if (H > 0x7ffffff0LL) return PERT_ERR_BADARG;
  const long long u64 = 2 * T + S;
  const long long i32 = R + 7 * T + 5 * S + 2 * (T + 1) + 2 + H;
  return u64 * 8 + i32 * 4 + scan_bytes(std::max(T + 1, H)) + 64;
}

int pert_trace_group_keys(const PertSpanTable* table, long long n_keys, int* key_ptr, int* key_trace, void* workspace,
                          long long workspace_bytes, void* stream_) {
  if (!table_ok(table) || n_keys < 0 || n_keys > 0x80000000LL || !key_ptr || !key_trace || !workspace)
    return PERT_ERR_BADARG;
  if (workspace_bytes < pert_trace_group_workspace_bytes(table->R, n_keys, -1, 0)) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  const long long L = n_keys + 1;
  cudaError_t e;
  if ((e = cudaMemsetAsync(key_ptr, 0, sizeof(int) * L, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(key_trace, 0, sizeof(int) * L, st)) != cudaSuccess) return (int)e;
  if (table->R == 0) return PERT_OK;
  k_key_count<<<pert_cdiv(table->R, 256), 256, 0, st>>>(*table, n_keys, key_ptr, key_trace);
  PERT_LAUNCH_CHECK();
  return scan(key_ptr, key_trace, L, (int*)workspace, st);
}

int pert_trace_group_build(const PertSpanTable* table, long long n_keys, long long T, long long n_ent, int hash_bits,
                           const int* key_ptr, const int* key_trace, const PertTraceGroups* out, void* workspace,
                           long long workspace_bytes, int* status, void* stream_) {
  if (!table_ok(table) || n_keys < 0 || T < 0 || n_ent < 0 || n_ent > 0x7fffffffLL || hash_bits < 1 ||
      hash_bits > 64 || !key_ptr || !key_trace || !out || !workspace || !status)
    return PERT_ERR_BADARG;
  const PertTraceGroups& o = *out;
  if (!o.row_ptr || !o.perm || !o.trace_id || !o.bucket || !o.y || !o.entry || !o.runtime || !o.order ||
      !o.ent_trace_ptr || !o.ent_pair_ptr || !o.pair_runtime || !o.pair_prob || !o.occurrences || !o.ins_runtime ||
      !o.rep_trace || !o.runtime_ins || !o.rep_ptr || !o.sizes)
    return PERT_ERR_BADARG;
  const long long need = pert_trace_group_workspace_bytes(table->R, n_keys, T, n_ent);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  cudaError_t e;
  if ((e = cudaMemsetAsync(o.sizes, 0, 3 * sizeof(int64_t), st)) != cudaSuccess) return (int)e;
  if (T == 0) return PERT_OK;
  const long long R = table->R, S = table_size(T), nt = n_tiles_of(T), H = n_ent * nt + 1;
  unsigned long long* u = (unsigned long long*)workspace;
  unsigned long long *h1 = u, *h2 = u + T, *pkey = u + 2 * T;
  int* w = (int*)(u + 2 * T + S);
  int* slot = w;        w += R;
  int* fill = w;        w += T;
  int* slot_of = w;     w += T;
  int* rank = w;        w += T;
  int* pos_of = w;      w += T;
  int* rep_pos = w;     w += T;
  int* pslot = w;       w += T;
  int* long_list = w;   w += T;
  int* owner = w;       w += S;
  int* gmin = w;        w += S;
  int* gcnt = w;        w += S;
  int* pfirst = w;      w += S;
  int* pcnt = w;        w += S;
  int* fl_ins = w;      w += T + 1;
  int* fl_pair = w;     w += T + 1;
  int* long_count = w;  w += 2;
  int* hist = w;        w += H;
  int* bsum = w;

  // 0x7f bytes = 0x7f7f7f7f: the "no position yet" start of every atomicMin
  auto zero = [&](void* p, long long bytes, int v) { return cudaMemsetAsync(p, v, (size_t)bytes, st); };
  if ((e = zero(fill, 4 * T, 0)) || (e = zero(owner, 4 * S, 0xff)) || (e = zero(gmin, 4 * S, 0x7f)) ||
      (e = zero(gcnt, 4 * S, 0)) || (e = zero(pkey, 8 * S, 0xff)) || (e = zero(pfirst, 4 * S, 0x7f)) ||
      (e = zero(pcnt, 4 * S, 0)) || (e = zero(rep_pos, 4 * T, 0x7f)) || (e = zero(fl_ins, 4 * (T + 1), 0)) ||
      (e = zero(fl_pair, 4 * (T + 1), 0)) || (e = zero(long_count, 8, 0)) || (e = zero(hist, 4 * H, 0)) ||
      (e = zero(o.rep_ptr, 4 * (T + 1), 0)))
    return (int)e;

  const int B = 256, WB = TG_WARPS * 32;
  const int gR = pert_cdiv(R, B), gT = pert_cdiv(T, B), gW = pert_cdiv(T * 32, WB);
  // 1. group rows by traceid
  k_compact_keys<<<pert_cdiv(n_keys + 1, B), B, 0, st>>>(n_keys, key_ptr, key_trace, o.row_ptr, o.trace_id);
  k_fill<<<gR, B, 0, st>>>(*table, n_keys, key_ptr, key_trace, fill, slot);
  k_sort_short<<<gW, WB, 0, st>>>(T, o.row_ptr, slot, o.perm, long_list, long_count);
  k_sort_long<<<PERT_NUM_SMS, 256, 0, st>>>(o.row_ptr, slot, o.perm, long_list, long_count);
  // 2. per-trace reductions + hashes
  k_trace_reduce<<<gW, WB, 0, st>>>(*table, T, n_ent, hash_bits, o.row_ptr, o.perm, o.bucket, o.y, o.entry, h1, h2,
                                    status);
  // 3. runtimes
  k_runtime_insert<<<gW, WB, 0, st>>>(*table, T, S, o.row_ptr, o.perm, h1, h2, owner, gmin, gcnt, slot_of);
  k_first_flags<<<gT, B, 0, st>>>(T, slot_of, gmin, fl_ins);
  PERT_LAUNCH_CHECK();
  int rc;
  if ((rc = scan(fl_ins, nullptr, T + 1, bsum, st)) != PERT_OK) return rc;
  k_runtime_assign<<<gT, B, 0, st>>>(T, slot_of, gmin, gcnt, fl_ins, o.runtime, o.occurrences);
  // 4. iteration order: stable counting sort by entry
  k_entry_rank<<<(int)nt, TG_TILE, 0, st>>>(T, (int)nt, o.entry, rank, hist);
  PERT_LAUNCH_CHECK();
  if ((rc = scan(hist, nullptr, H, bsum, st)) != PERT_OK) return rc;
  k_entry_place<<<gT, B, 0, st>>>(T, (int)nt, o.entry, rank, hist, o.order, pos_of);
  k_entry_ptr<<<pert_cdiv(n_ent + 1, B), B, 0, st>>>(n_ent, (int)nt, hist, o.ent_trace_ptr);
  // 5. representatives, insertion order, entry mixes
  if ((e = zero(fl_ins, 4 * (T + 1), 0))) return (int)e;
  k_rep_min<<<gT, B, 0, st>>>(T, o.runtime, pos_of, rep_pos);
  k_pair_insert<<<gT, B, 0, st>>>(T, S, o.order, o.entry, o.runtime, rep_pos, pkey, pfirst, pcnt, pslot, fl_ins);
  k_pair_flags<<<gT, B, 0, st>>>(T, pslot, pfirst, fl_pair);
  PERT_LAUNCH_CHECK();
  if ((rc = scan(fl_ins, fl_pair, T + 1, bsum, st)) != PERT_OK) return rc;
  k_emit<<<gT, B, 0, st>>>(T, o.order, o.entry, o.runtime, o.row_ptr, fl_ins, fl_pair, pslot, pcnt, o.ent_trace_ptr,
                           o);
  k_ent_pair_ptr<<<pert_cdiv(n_ent + 1, B), B, 0, st>>>(n_ent, o.ent_trace_ptr, fl_pair, o.ent_pair_ptr);
  PERT_LAUNCH_CHECK();
  if ((rc = scan(o.rep_ptr, nullptr, T + 1, bsum, st)) != PERT_OK) return rc;
  k_sizes<<<1, 1, 0, st>>>(T, fl_ins, fl_pair, o.rep_ptr, o.sizes);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_trace_group_gather(const PertSpanTable* table, const int* perm, const int* row_ptr, const int* rep_trace,
                            const int* rep_ptr, long long n_rt, long long R2, int64_t* rows, void* stream_) {
  if (!table_ok(table) || n_rt < 0 || R2 < 0 || !perm || !row_ptr || !rep_trace || !rep_ptr || !rows)
    return PERT_ERR_BADARG;
  if (n_rt == 0) return PERT_OK;
  const int WB = TG_WARPS * 32;
  k_gather<<<pert_cdiv(n_rt * 32, WB), WB, 0, (cudaStream_t)stream_>>>(*table, perm, row_ptr, rep_trace, rep_ptr,
                                                                         n_rt, R2, rows);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
