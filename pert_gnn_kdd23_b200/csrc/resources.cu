// Appending and evicting resource rows of a live pattern store (PatternStore.append_resources).
//
// The store keeps its resource rows sorted by key = timestamp * n_ms + ms (res_keys / res_vals, equal keys in arrival
// order: the constructor's stable argsort) and an as-of index that regroups them by microservice (PertResourceAsOf,
// store.py asof_index).  An update appends k rows and drops every row older than a cut.  Its result must be the state
// a store built from scratch from the surviving rows in arrival order would have, bit for bit, so:
//   * the old rows were all there before the new ones: on equal keys they come first, and among themselves they keep
//     their order; the new rows keep the order of a stable sort of their keys (the caller sorts the k new keys);
//   * a cut c (drop timestamp < c) removes exactly the keys < c * n_ms, because 0 <= ms < n_ms: a prefix of the sorted
//     table, of the sorted batch, and of every microservice's segment of either index.
// The old rows are never re-sorted.  The work is one pass over the n old rows and one over the k new ones, each thread
// doing a binary search in the other array and moving its own row: every output slot is written exactly once, without
// atomics, so the result does not depend on scheduling.  The merge writes fresh arrays: a parallel in-place merge
// would overwrite rows that other threads have not read yet.
//
// A replace or delete (pert_store_resources_update_*) also takes a drop set D: sorted unique keys whose old rows all
// leave the table.  c[d] = the old rows of key d that the cut does not already evict, C its exclusive scan over D in
// key order and G over D in (ms, ts) order.  An old row of key x not in D moves C[#(D < x)] slots further down than
// without D, an old index entry G[...] slots within its microservice, and a new row as many as D drops below it; an
// old row of a key in D is not written.  The same kernels serve both pairs: DROP = false is the plain append.
#include "scan.cuh"

namespace {

constexpr int NF = 8;          // resource statistics per row (store.cu)
constexpr int RU_THREADS = 256;

__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) {
  int64_t q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}

// first i in [lo, hi) with key[i] >= v (strict = false) or key[i] > v (strict = true); hi if none
__device__ __forceinline__ long long bound(const int64_t* __restrict__ key, long long lo, long long hi, int64_t v,
                                           bool strict) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const int64_t x = key[mid];
    if (x < v || (strict && x == v)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The same over the batch's rows of one microservice in grouped order (key nk[grp[i]]).
__device__ __forceinline__ int group_bound(const int64_t* __restrict__ nk, const int* __restrict__ grp, int lo, int hi,
                                           int64_t v, bool strict) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int64_t x = nk[grp[mid]];
    if (x < v || (strict && x == v)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The drop set of a replace or delete (see the top of the file): n sorted unique keys, grp their positions ordered by
// (ms, ts), and cnt [2 (n + 1)] the exclusive scans C (key order) then G (grouped order) of the old rows each drops.
struct DropSet {
  const int64_t* key;
  const int* grp;
  const int* cnt;
  int n;
};

// The batch's rows in grouped order are sorted by (ms, timestamp): first grouped index of microservice m.
__device__ __forceinline__ int group_start(const int64_t* __restrict__ nk, const int* __restrict__ grp, int k, int n_ms,
                                           int m) {
  int lo = 0, hi = k;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int64_t x = nk[grp[mid]];
    const int64_t ms = x - floor_div(x, n_ms) * n_ms;
    if (ms < m) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Threads g <= n: the drop key at grouped index g (g = n: none) gets c = the old rows of its key at or above the cut
// (keys below the cut are in the evicted prefix already), written at its key-order slot of C and its grouped slot of
// G; thread n zeroes both totals' slots, which the exclusive scan turns into the totals.  Threads m <= n_ms: seg_d[m] =
// the first grouped index of microservice m's drop keys (n for m = n_ms).
__global__ void __launch_bounds__(RU_THREADS) k_res_drop_count(PertStore s, DropSet d, int64_t cut, int* __restrict__ cnt,
                                                               int* __restrict__ seg_d) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= s.n_ms) seg_d[g] = group_start(d.key, d.grp, d.n, s.n_ms, g);
  if (g > d.n) return;
  if (g == d.n) {
    cnt[d.n] = 0;
    cnt[2 * d.n + 1] = 0;
    return;
  }
  const int i = d.grp[g];
  const int64_t x = d.key[i];
  const int c = floor_div(x, s.n_ms) < cut ? 0
                                           : (int)(bound(s.res_keys, 0, s.n_res, x, true) -
                                                   bound(s.res_keys, 0, s.n_res, x, false));
  cnt[i] = c;
  cnt[d.n + 1 + g] = c;
}

// One thread per microservice m (thread n_ms: the table-wide sizes).  seg[m] = first surviving entry of m's old as-of
// segment (asof.ms_ptr[m] + its evicted rows), seg[n_ms + m] = first surviving grouped index of m's batch rows; the
// surviving row count of m goes to ms_ptr_out[m] (scanned into offsets afterwards).  sizes = {p, q, n_out}: evicted
// prefix of the table, evicted prefix of the sorted batch, rows after the update.  With a drop set (whose boundaries
// k_res_drop_count wrote to seg[2 n_ms ..]) m's count loses the old rows its drop keys remove, and sizes[3] = them all.
template <bool DROP>
__global__ void __launch_bounds__(RU_THREADS) k_res_count(PertStore s, PertResourceAsOf a, const int64_t* __restrict__ nk,
                                                          const int* __restrict__ grp, int k, int64_t cut, DropSet d,
                                                          int* __restrict__ ms_ptr_out, int* __restrict__ seg,
                                                          long long* __restrict__ sizes) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m > s.n_ms) return;
  if (m == s.n_ms) {
    long long lo = 0, hi = s.n_res;                 // p: rows whose timestamp is < cut
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (floor_div(s.res_keys[mid], s.n_ms) < cut) lo = mid + 1;
      else hi = mid;
    }
    const long long p = lo;
    lo = 0, hi = k;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (floor_div(nk[mid], s.n_ms) < cut) lo = mid + 1;
      else hi = mid;
    }
    sizes[0] = p;
    sizes[1] = lo;
    sizes[2] = ((long long)s.n_res - p) + ((long long)k - lo);
    if (DROP) {
      sizes[2] -= d.cnt[d.n];
      sizes[3] = d.cnt[d.n];
    }
    ms_ptr_out[m] = 0;                              // the scan turns it into the total
    return;
  }
  int lo = a.ms_ptr[m], hi = a.ms_ptr[m + 1];
  const int old_end = hi;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a.ts[mid] < cut) lo = mid + 1;
    else hi = mid;
  }
  const int old_lo = lo;
  const int g0 = group_start(nk, grp, k, s.n_ms, m), g1 = group_start(nk, grp, k, s.n_ms, m + 1);
  lo = g0, hi = g1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (floor_div(nk[grp[mid]], s.n_ms) < cut) lo = mid + 1;
    else hi = mid;
  }
  seg[m] = old_lo;
  seg[s.n_ms + m] = lo;
  int kept = (old_end - old_lo) + (g1 - lo);
  if (DROP) kept -= d.cnt[d.n + 1 + seg[2 * s.n_ms + m + 1]] - d.cnt[d.n + 1 + seg[2 * s.n_ms + m]];
  ms_ptr_out[m] = kept;
}

// Surviving old row j (p <= j < n_res) of the table: it moves to j - p + #(surviving new keys < key[j]), less the old
// rows the drop set removes below it; a row of a dropped key is not written.
template <bool DROP>
__global__ void __launch_bounds__(RU_THREADS) k_res_merge_old(PertStore s, const int64_t* __restrict__ nk, int k, int p,
                                                              int q, DropSet d, int64_t* __restrict__ keys_out,
                                                              float* __restrict__ vals_out) {
  const long long j = p + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= s.n_res) return;
  const int64_t key = s.res_keys[j];
  long long pos = (j - p) + (bound(nk, q, k, key, false) - q);
  if (DROP) {
    const int l = (int)bound(d.key, 0, d.n, key, false);
    if (l < d.n && d.key[l] == key) return;                // dropped
    pos -= d.cnt[l];
  }
  keys_out[pos] = key;
  const float4* src = reinterpret_cast<const float4*>(s.res_vals + (size_t)j * NF);
  float4* dst = reinterpret_cast<float4*>(vals_out + (size_t)pos * NF);
  dst[0] = __ldg(src);
  dst[1] = __ldg(src + 1);
}

// Surviving old entry i of the as-of index (microservice m, timestamp t, table row r): merged with m's surviving batch
// rows by timestamp, old entries first on equal timestamps, and its row renumbered to r's new table position.
// Why the result equals asof_index(keys_out): that index lists m's rows by timestamp and, within one timestamp, by
// ascending table position.  Within (m, t) all rows share one key, so in the merged table the old ones precede the new
// ones (ties go to old rows), the old ones keep their old relative order (which the old index lists ascending) and the
// new ones keep their sorted-batch order (which the grouped order lists ascending: it is a stable regrouping).  The
// merge below produces exactly that order.  A drop set removes whole (m, t) runs, so it changes no order: the entries
// of a dropped key are not written, and the others move down by the drops before them in m's segment and in the table.
template <bool DROP>
__global__ void __launch_bounds__(RU_THREADS) k_res_merge_asof(PertStore s, PertResourceAsOf a,
                                                               const int64_t* __restrict__ nk,
                                                               const int* __restrict__ grp, int k, int p, int q,
                                                               DropSet d, const int* __restrict__ ms_ptr_out,
                                                               const int* __restrict__ seg, int64_t* __restrict__ ts_out,
                                                               int* __restrict__ row_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= s.n_res) return;
  const int m = upper_seg(a.ms_ptr, s.n_ms, i);
  const int old_lo = seg[m];
  if (i < old_lo) return;                                  // evicted
  const int64_t t = a.ts[i];
  const int64_t key = t * s.n_ms + m;
  int dropped_m = 0, dropped_before = 0, dropped_rows = 0;
  if (DROP) {
    const int* G = d.cnt + d.n + 1;
    const int h0 = seg[2 * s.n_ms + m], h1 = seg[2 * s.n_ms + m + 1];
    const int l = group_bound(d.key, d.grp, h0, h1, key, false);
    if (l < h1 && d.key[d.grp[l]] == key) return;         // dropped
    dropped_m = G[h1] - G[h0];
    dropped_before = G[l] - G[h0];
    dropped_rows = d.cnt[bound(d.key, 0, d.n, key, false)];
  }
  const int new_lo = seg[s.n_ms + m];
  const int old_cnt = a.ms_ptr[m + 1] - old_lo;
  const int new_hi = new_lo + (ms_ptr_out[m + 1] - ms_ptr_out[m]) - old_cnt + dropped_m;
  const long long pos = ms_ptr_out[m] + (i - old_lo) - dropped_before +
                        (group_bound(nk, grp, new_lo, new_hi, key, false) - new_lo);
  ts_out[pos] = t;
  row_out[pos] = (int)((a.row[i] - p) - dropped_rows + (bound(nk, q, k, key, false) - q));
}

// Surviving new row at grouped index g (sorted-batch position sp = grp[g] >= q): its table position is
// sp - q + #(surviving old keys <= its key), its index position ms_ptr_out[m] + its rank among m's surviving batch rows
// + #(m's surviving old entries with timestamp <= its timestamp), both counts less what the drop set removes.  Threads
// g < n_ms also write ms_has_res.
template <bool DROP>
__global__ void __launch_bounds__(RU_THREADS) k_res_merge_new(PertStore s, PertResourceAsOf a,
                                                              const int64_t* __restrict__ nk,
                                                              const int64_t* __restrict__ perm,
                                                              const float* __restrict__ vals, const int* __restrict__ grp,
                                                              int k, int p, int q, DropSet d,
                                                              const int* __restrict__ ms_ptr_out,
                                                              const int* __restrict__ seg,
                                                              int64_t* __restrict__ keys_out,
                                                              float* __restrict__ vals_out,
                                                              uint8_t* __restrict__ has_out,
                                                              int64_t* __restrict__ ts_out, int* __restrict__ row_out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < s.n_ms) has_out[g] = ms_ptr_out[g + 1] > ms_ptr_out[g];
  if (g >= k) return;
  const int sp = grp[g];
  if (sp < q) return;                                      // evicted
  const int64_t key = nk[sp];
  const int64_t t = floor_div(key, s.n_ms);
  const int m = (int)(key - t * s.n_ms);
  int dropped_rows = 0, dropped_entries = 0;
  if (DROP) {
    const int* G = d.cnt + d.n + 1;
    const int h0 = seg[2 * s.n_ms + m], h1 = seg[2 * s.n_ms + m + 1];
    dropped_rows = d.cnt[bound(d.key, 0, d.n, key, true)];
    dropped_entries = G[group_bound(d.key, d.grp, h0, h1, key, true)] - G[h0];
  }
  const long long pos = (sp - q) + (bound(s.res_keys, p, s.n_res, key, true) - p) - dropped_rows;
  keys_out[pos] = key;
  const float4* src = reinterpret_cast<const float4*>(vals + (size_t)perm[sp] * NF);
  float4* dst = reinterpret_cast<float4*>(vals_out + (size_t)pos * NF);
  dst[0] = __ldg(src);
  dst[1] = __ldg(src + 1);
  const int old_lo = seg[m], old_hi = a.ms_ptr[m + 1];
  const long long apos = ms_ptr_out[m] + (g - seg[s.n_ms + m]) + (bound(a.ts, old_lo, old_hi, t, true) - old_lo) -
                         dropped_entries;
  ts_out[apos] = t;
  row_out[apos] = (int)pos;
}

bool store_ok(const PertStore* s, const PertResourceAsOf* a) {
  return s && a && a->ms_ptr && s->n_ms > 0 && s->n_res >= 0 &&
         (s->n_res == 0 || (s->res_keys && s->res_vals && a->ts && a->row));
}

// The launches the two pairs of entry points share; DROP = false ignores d.
template <bool DROP>
void launch_count(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                  const int32_t* new_group, long long k, long long evict_before, DropSet d, int32_t* ms_ptr_out,
                  int32_t* seg, long long* sizes, cudaStream_t st) {
  const int n_ms = store->n_ms;
  k_res_count<DROP><<<pert_cdiv(n_ms + 1, RU_THREADS), RU_THREADS, 0, st>>>(*store, *asof, new_keys, new_group, (int)k,
                                                                           evict_before, d, ms_ptr_out, seg, sizes);
  // counts -> exclusive offsets (scan.cuh's one-CTA carry scan); the total is the last count plus its offset
  k_scan_block_sums<<<dim3(1, 1), SCAN_THREADS, 0, st>>>(ms_ptr_out, n_ms + 1);
}

template <bool DROP>
void launch_merge(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                  const int64_t* new_perm, const float* new_vals, const int32_t* new_group, long long k, DropSet d,
                  const int32_t* ms_ptr_out, const int32_t* seg, long long p, long long q, int64_t* keys_out,
                  float* vals_out, uint8_t* has_out, int64_t* ts_out, int32_t* row_out, cudaStream_t st) {
  const long long n_old = store->n_res - p;
  if (n_old > 0) {
    k_res_merge_old<DROP><<<pert_cdiv(n_old, RU_THREADS), RU_THREADS, 0, st>>>(*store, new_keys, (int)k, (int)p,
                                                                               (int)q, d, keys_out, vals_out);
    k_res_merge_asof<DROP><<<pert_cdiv(store->n_res, RU_THREADS), RU_THREADS, 0, st>>>(
        *store, *asof, new_keys, new_group, (int)k, (int)p, (int)q, d, ms_ptr_out, seg, ts_out, row_out);
  }
  const long long g = k > store->n_ms ? k : store->n_ms;
  k_res_merge_new<DROP><<<pert_cdiv(g, RU_THREADS), RU_THREADS, 0, st>>>(*store, *asof, new_keys, new_perm, new_vals,
                                                                         new_group, (int)k, (int)p, (int)q, d,
                                                                         ms_ptr_out, seg, keys_out, vals_out, has_out,
                                                                         ts_out, row_out);
}

}  // namespace

extern "C" {

int pert_store_resources_count(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                               const int32_t* new_group, long long k, long long evict_before, int32_t* ms_ptr_out,
                               int32_t* seg, long long* sizes, void* stream) {
  if (!store_ok(store, asof) || k < 0 || k > 0x7fffffffLL || (k > 0 && (!new_keys || !new_group)) || !ms_ptr_out ||
      !seg || !sizes)
    return PERT_ERR_BADARG;
  launch_count<false>(store, asof, new_keys, new_group, k, evict_before, DropSet{}, ms_ptr_out, seg, sizes,
                      (cudaStream_t)stream);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_store_resources_merge(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                               const int64_t* new_perm, const float* new_vals, const int32_t* new_group, long long k,
                               const int32_t* ms_ptr_out, const int32_t* seg, long long p, long long q,
                               long long n_out, int64_t* keys_out, float* vals_out, uint8_t* has_out, int64_t* ts_out,
                               int32_t* row_out, void* stream) {
  if (!store_ok(store, asof) || k < 0 || k > 0x7fffffffLL || p < 0 || q < 0 || n_out < 0 || p > store->n_res ||
      q > k || n_out != (store->n_res - p) + (k - q) || n_out > 0x7fffffffLL)
    return PERT_ERR_BADARG;
  if ((k > 0 && (!new_keys || !new_perm || !new_vals || !new_group)) || !ms_ptr_out || !seg || !has_out ||
      (n_out > 0 && (!keys_out || !vals_out || !ts_out || !row_out)))
    return PERT_ERR_BADARG;
  // the value rows move with 16-byte vector loads and stores
  if (((uintptr_t)new_vals | (uintptr_t)vals_out | (uintptr_t)store->res_vals) % 16 != 0) return PERT_ERR_BADARG;
  launch_merge<false>(store, asof, new_keys, new_perm, new_vals, new_group, k, DropSet{}, ms_ptr_out, seg, p, q,
                      keys_out, vals_out, has_out, ts_out, row_out, (cudaStream_t)stream);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_store_resources_update_count(const PertStore* store, const PertResourceAsOf* asof, const int64_t* drop_keys,
                                      const int32_t* drop_group, long long n_drop, const int64_t* new_keys,
                                      const int32_t* new_group, long long k, long long evict_before,
                                      int32_t* drop_cnt, int32_t* ms_ptr_out, int32_t* seg, long long* sizes,
                                      void* stream) {
  if (!store_ok(store, asof) || k < 0 || k > 0x7fffffffLL || n_drop < 0 || n_drop >= 0x7fffffffLL ||
      (k > 0 && (!new_keys || !new_group)) || (n_drop > 0 && (!drop_keys || !drop_group)) || !drop_cnt ||
      !ms_ptr_out || !seg || !sizes)
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const DropSet d{drop_keys, drop_group, drop_cnt, (int)n_drop};
  const long long g = n_drop > store->n_ms ? n_drop : store->n_ms;
  k_res_drop_count<<<pert_cdiv(g + 1, RU_THREADS), RU_THREADS, 0, st>>>(*store, d, evict_before, drop_cnt,
                                                                        seg + 2 * store->n_ms);
  // both count arrays -> exclusive offsets, one CTA each (blockIdx.y); each ends with its total
  k_scan_block_sums<<<dim3(1, 2), SCAN_THREADS, 0, st>>>(drop_cnt, (int)n_drop + 1);
  launch_count<true>(store, asof, new_keys, new_group, k, evict_before, d, ms_ptr_out, seg, sizes, st);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_store_resources_update_merge(const PertStore* store, const PertResourceAsOf* asof, const int64_t* drop_keys,
                                      const int32_t* drop_group, const int32_t* drop_cnt, long long n_drop,
                                      const int64_t* new_keys, const int64_t* new_perm, const float* new_vals,
                                      const int32_t* new_group, long long k, const int32_t* ms_ptr_out,
                                      const int32_t* seg, long long p, long long q, long long n_dropped,
                                      long long n_out, int64_t* keys_out, float* vals_out, uint8_t* has_out,
                                      int64_t* ts_out, int32_t* row_out, void* stream) {
  if (!store_ok(store, asof) || k < 0 || k > 0x7fffffffLL || n_drop < 0 || n_drop >= 0x7fffffffLL || p < 0 || q < 0 ||
      n_dropped < 0 || n_out < 0 || p > store->n_res || q > k || n_dropped > store->n_res - p ||
      (n_drop == 0 && n_dropped > 0) || n_out != (store->n_res - p - n_dropped) + (k - q) || n_out > 0x7fffffffLL)
    return PERT_ERR_BADARG;
  if ((k > 0 && (!new_keys || !new_perm || !new_vals || !new_group)) ||
      (n_drop > 0 && (!drop_keys || !drop_group)) || !drop_cnt || !ms_ptr_out || !seg || !has_out ||
      (n_out > 0 && (!keys_out || !vals_out || !ts_out || !row_out)))
    return PERT_ERR_BADARG;
  if (((uintptr_t)new_vals | (uintptr_t)vals_out | (uintptr_t)store->res_vals) % 16 != 0) return PERT_ERR_BADARG;
  launch_merge<true>(store, asof, new_keys, new_perm, new_vals, new_group, k,
                     DropSet{drop_keys, drop_group, drop_cnt, (int)n_drop}, ms_ptr_out, seg, p, q, keys_out, vals_out,
                     has_out, ts_out, row_out, (cudaStream_t)stream);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
