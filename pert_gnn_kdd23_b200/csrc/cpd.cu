// Split-conformal predictive distribution (pert_cpd_fit, pert_cpd_tail, pert_cpd_quantile).
//
// Fit: the scores s = (float)y - yhat[:, col] of n labelled graphs are counting-sorted by group (entry id, the code
// of calib.cuh), the group-ordered keys are copied once more behind themselves as the global row, and every row is
// sorted by its order-preserving uint32 key.  Only keys are kept, so the sorted row is unique and any correct sort is
// bit-identical to np.sort.  Two tiers, as in calib.cu: a row of at most CB_SMALL keys is sorted by one CTA in shared
// memory (k_cpd_small, bitonic); a larger one -- the global row of any real set, and a hot entry -- is partitioned
// MSD-first over its 8-bit digits: its CB_TILE-key tiles add their digit counts into one 256-bin histogram per
// segment (k_cpd_hist), one CTA per segment scans it into bucket bases and queues the buckets (k_cpd_split), and the
// tile CTAs scatter their keys into the ping-pong buffer (k_cpd_scatter).  A bucket of at most CB_SMALL keys goes to
// the small tier; a larger one is the next pass's segment, and after the fourth digit its keys are all equal, so the
// last scatter writes the values straight into the table.  No segment above CB_SMALL is handled by one CTA, and the
// host never reads the device: every grid is sized from n and the work lists live on the device.
//
// Queries: one thread per (request, threshold) or (request, level), a binary search in the request's row.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "calib.cuh"

#define CPD_THREADS 256
#define CPD_PASSES 4
#define CPD_SMALL_GRID 4096              // CTAs of the small-tier sort, which loops over its work list

namespace {

// meta words: segments and tiles of every pass, then the small-tier work items
#define CPD_SEGS 0
#define CPD_TILES CPD_PASSES
#define CPD_ITEMS (2 * CPD_PASSES)

// One thread per row s: its start in the table (row G after rows 0 .. G-1), ptr64, and its first work item: a row of
// more than CB_SMALL keys becomes a pass-0 segment with its tiles, a smaller non-empty one a small-tier item.
__global__ void k_cpd_plan(const int* __restrict__ ptr, int G, int n, int* __restrict__ meta, int2* __restrict__ segs,
                           int2* __restrict__ tiles, int2* __restrict__ items, long long* __restrict__ ptr64) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > G) return;
  int start, len;
  calib_seg(ptr, G, n, s, &start, &len);
  if (s == G) {
    start = ptr[G];
    ptr64[G + 1] = (long long)start + n;
  }
  ptr64[s] = start;
  if (len > CB_SMALL) {
    const int slot = atomicAdd(meta + CPD_SEGS, 1);
    segs[slot] = make_int2(start, len);
    const int nt = (len + CB_TILE - 1) / CB_TILE;
    const int base = atomicAdd(meta + CPD_TILES, nt);
    for (int j = 0; j < nt; ++j) tiles[base + j] = make_int2(slot, j * CB_TILE);
  } else if (len > 0) {
    items[atomicAdd(meta + CPD_ITEMS, 1)] = make_int2(start, len);        // in buffer 0
  }
}

// One pass: every tile CTA adds the digit counts of its keys into its segment's histogram.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_hist(const uint32_t* __restrict__ src, const int2* __restrict__ segs,
                                                          const int2* __restrict__ tiles, const int* __restrict__ meta,
                                                          int pass, int* __restrict__ hist) {
  __shared__ int h[256];
  if ((int)blockIdx.x >= meta[CPD_TILES + pass]) return;
  const int2 tl = tiles[blockIdx.x];
  const int2 sg = segs[tl.x];
  const int shift = 24 - 8 * pass, end = min(tl.y + CB_TILE, sg.y);
  h[threadIdx.x] = 0;
  __syncthreads();
  for (int i = tl.y + threadIdx.x; i < end; i += CPD_THREADS)
    atomicAdd(h + ((__ldg(src + sg.x + i) >> shift) & 255u), 1);
  __syncthreads();
  const int c = h[threadIdx.x];
  if (c) atomicAdd(hist + tl.x * 256 + threadIdx.x, c);
}

// One pass, one CTA per segment: the bucket bases (the scatter's cursors), the histogram cleared for the next pass,
// and the buckets queued: at most CB_SMALL keys -> a small-tier item in the destination buffer, more -> a segment of
// the next pass.  After the last digit nothing is queued: the scatter writes the final values.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_split(const int2* __restrict__ segs, int* __restrict__ meta,
                                                           int pass, int* __restrict__ hist, int* __restrict__ cursor,
                                                           int2* __restrict__ next_segs, int2* __restrict__ next_tiles,
                                                           int2* __restrict__ items) {
  __shared__ int sw[32];
  const int slot = blockIdx.x;
  if (slot >= meta[CPD_SEGS + pass]) return;
  const int2 sg = segs[slot];
  const int at = slot * 256 + threadIdx.x;
  const int c = hist[at];
  hist[at] = 0;
  const int base = sg.x + block_scan_inclusive(c, sw) - c;
  cursor[at] = base;
  if (c == 0 || pass == CPD_PASSES - 1) return;
  if (c <= CB_SMALL) {
    items[atomicAdd(meta + CPD_ITEMS, 1)] = make_int2(base, c | (((pass + 1) & 1) << 16));
  } else {
    const int ns = atomicAdd(meta + CPD_SEGS + pass + 1, 1);
    next_segs[ns] = make_int2(base, c);
    const int nt = (c + CB_TILE - 1) / CB_TILE;
    const int tb = atomicAdd(meta + CPD_TILES + pass + 1, nt);
    for (int j = 0; j < nt; ++j) next_tiles[tb + j] = make_int2(ns, j * CB_TILE);
  }
}

// One pass: every tile CTA reserves a range of each bucket for its keys and scatters them there (the order inside a
// bucket is free).  The last pass writes the keys' fp32 values into the table.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_scatter(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                                             const int2* __restrict__ segs,
                                                             const int2* __restrict__ tiles,
                                                             const int* __restrict__ meta, int pass,
                                                             int* __restrict__ cursor) {
  __shared__ uint32_t sk[CB_TILE];
  __shared__ int cnt[256], gbase[256];
  if ((int)blockIdx.x >= meta[CPD_TILES + pass]) return;
  const int2 tl = tiles[blockIdx.x];
  const int2 sg = segs[tl.x];
  const int shift = 24 - 8 * pass, len = min(CB_TILE, sg.y - tl.y);
  cnt[threadIdx.x] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < len; i += CPD_THREADS) {
    const uint32_t k = __ldg(src + sg.x + tl.y + i);
    sk[i] = k;
    atomicAdd(cnt + ((k >> shift) & 255u), 1);
  }
  __syncthreads();
  const int c = cnt[threadIdx.x];
  if (c) gbase[threadIdx.x] = atomicAdd(cursor + tl.x * 256 + threadIdx.x, c);
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const bool last = pass == CPD_PASSES - 1;
  for (int i = threadIdx.x; i < len; i += CPD_THREADS) {
    const uint32_t k = sk[i];
    const int d = (k >> shift) & 255u;
    dst[gbase[d] + warp_counter_add(cnt, d)] = last ? __float_as_uint(calib_value(k)) : k;
  }
}

// Small tier: every work item {start, len | buffer << 16} (at most CB_SMALL keys) is sorted by one CTA in shared
// memory (bitonic over the next power of two, padded with the largest key) and written to the table as values.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_small(const uint32_t* __restrict__ buf0,
                                                           const uint32_t* __restrict__ buf1,
                                                           const int2* __restrict__ items, const int* __restrict__ meta,
                                                           float* __restrict__ scores) {
  __shared__ uint32_t sk[CB_SMALL];
  const int n_items = meta[CPD_ITEMS];
  for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
    const int2 w = items[it];
    const int start = w.x, len = w.y & 0xffff;
    const uint32_t* src = (w.y >> 16) ? buf1 : buf0;
    int P = 1;
    while (P < len) P <<= 1;
    for (int i = threadIdx.x; i < P; i += CPD_THREADS) sk[i] = i < len ? src[start + i] : 0xffffffffu;
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int t = threadIdx.x; t < P / 2; t += CPD_THREADS) {
          const int i = 2 * j * (t / j) + (t % j), ixj = i + j;
          const uint32_t a = sk[i], b = sk[ixj];
          if (((i & k) == 0) == (a > b)) {
            sk[i] = b;
            sk[ixj] = a;
          }
        }
        __syncthreads();
      }
    }
    for (int i = threadIdx.x; i < len; i += CPD_THREADS) scores[start + i] = calib_value(sk[i]);
    __syncthreads();                          // sk is rewritten by the next item
  }
}

// The row a tail query of group id g reads: g's own row iff 0 <= g < G and n_g >= min_count (>= 1), else row G.
__device__ __forceinline__ int cpd_row(const long long* __restrict__ ptr, int G, long long min_count, long long g) {
  return (g >= 0 && g < G && ptr[g + 1] - ptr[g] >= min_count) ? (int)g : G;
}

// fl(v - yhat) with -0 -> +0; a NaN (a NaN input, or inf - inf) sets the status
__device__ __forceinline__ float cpd_score(float v, float yh, int* status) {
  float c = __fsub_rn(v, yh);
  if (isnan(c)) *status = PERT_ERR_RANGE;
  return c == 0.f ? 0.f : c;
}

__global__ void k_cpd_tail(const float* __restrict__ scores, const long long* __restrict__ ptr, int G,
                           long long min_count, const float* __restrict__ yhat, long long ld,
                           const int64_t* __restrict__ group, int Q, const float* __restrict__ x, int S,
                           const int64_t* __restrict__ y, int* __restrict__ ge, int* __restrict__ gt,
                           int* __restrict__ row, int* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q * S) return;
  const int q = i / S;
  const int r = cpd_row(ptr, G, min_count, group ? group[q] : -1);
  const float c = cpd_score(x ? x[i] : (float)y[q], yhat[(long long)q * ld], status);
  const float* a = scores + ptr[r];
  const int m = (int)(ptr[r + 1] - ptr[r]);
  int lo = 0, hi = m;                         // lower bound: the first score >= c
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < c) lo = mid + 1;
    else hi = mid;
  }
  int lo2 = lo, hi2 = m;                      // upper bound: the first score > c
  while (lo2 < hi2) {
    const int mid = (lo2 + hi2) >> 1;
    if (a[mid] <= c) lo2 = mid + 1;
    else hi2 = mid;
  }
  ge[i] = m - lo;
  gt[i] = m - lo2;
  if (i % S == 0) row[q] = r;
}

__global__ void k_cpd_quantile(const float* __restrict__ scores, const long long* __restrict__ ptr, int G,
                               long long min_count, const float* __restrict__ yhat, long long ld,
                               const int64_t* __restrict__ group, int Q, int L, CalibTaus taus,
                               float* __restrict__ out, int* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q * L) return;
  const int q = i / L;
  const int l = i % L;
  double tau = taus.v[0];
#pragma unroll
  for (int j = 1; j < PERT_MAX_QUANTILES; ++j)      // a select, not a dynamic index: the levels stay in registers
    if (j == l) tau = taus.v[j];
  const float yh = yhat[(long long)q * ld];
  if (isnan(yh)) *status = PERT_ERR_RANGE;
  const long long g = group ? group[q] : -1;
  int r = G;
  if (g >= 0 && g < G && calib_own(ptr[g + 1] - ptr[g], tau, min_count, false)) r = (int)g;
  const long long m = ptr[r + 1] - ptr[r], k = calib_k(m, tau);
  out[i] = k > m ? INFINITY : __fadd_rn(yh, scores[ptr[r] + k - 1]);
}

// ---- pert_cpd_merge: old table (G_old) plus or minus a delta table (G_new >= G_old) -> new table (G_new).
// Output row r reads old row r (r < G_old), no old row (G_old <= r < G_new) or old row G_old (r = G_new), and delta
// row r.  Work is cut into tiles of CM_TILE elements of the output row (insert) or of the old row (remove); the tile
// counts are scanned beside the row sizes, and tile t finds its row by a binary search in that prefix, so every grid
// is sized from the host's sizes and no row is handled by a single CTA.
#define CM_TILE 4096
#define CM_ITEMS (CM_TILE / CPD_THREADS)

__device__ __forceinline__ int cm_old_row(int r, int G_old, int G_new) {
  return r < G_old ? r : (r == G_new ? G_old : -1);
}

// One thread per output row: its size (old +- delta) and its tile count, int32, scanned next.  A removal longer than
// its old row sets the status and gives the row no elements.
__global__ void k_cpd_merge_count(const long long* __restrict__ ptr, int G_old, const long long* __restrict__ dptr,
                                  int G_new, int sign, int* __restrict__ cnt, int* __restrict__ ntile,
                                  int* __restrict__ status) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > G_new) return;
  const int ro = cm_old_row(r, G_old, G_new);
  const long long a = ro < 0 ? 0 : ptr[ro + 1] - ptr[ro], b = dptr[r + 1] - dptr[r];
  long long c = a + b, work = c;
  if (sign < 0) {
    c = a - b;
    work = a;
    if (c < 0) {
      *status = PERT_ERR_RANGE;
      c = 0;
      work = 0;
    }
  }
  cnt[r] = (int)c;
  ntile[r] = (int)((work + CM_TILE - 1) / CM_TILE);
}

// ptr_out from the scanned row sizes
__global__ void k_cpd_merge_ptr(const int* __restrict__ cnt, int G_new, long long* __restrict__ out_ptr) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > G_new) return;
  out_ptr[r + 1] = cnt[r];
  if (r == 0) out_ptr[0] = 0;
}

// tile t -> (row, first tile of the row) from the inclusive tile prefix; false past the last tile
__device__ __forceinline__ bool cm_tile_row(const int* __restrict__ ntile, int G_new, int t, int* row, int* first) {
  if (t >= ntile[G_new]) return false;
  int lo = 0, hi = G_new;                     // the first row whose inclusive prefix exceeds t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ntile[mid] <= t) lo = mid + 1;
    else hi = mid;
  }
  *row = lo;
  *first = lo ? ntile[lo - 1] : 0;
  return true;
}

// first index in a[lo, hi) whose key is >= k (upper: > k)
__device__ __forceinline__ int cm_search_g(const float* __restrict__ a, int lo, int hi, uint32_t k, bool upper) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const uint32_t v = calib_key(a[mid]);
    if (upper ? v <= k : v < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ int cm_search_s(const uint32_t* a, int lo, int hi, uint32_t k, bool upper) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const uint32_t v = a[mid];
    if (upper ? v <= k : v < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Merge path with old elements first on ties: of the first d outputs of A (len a) merged with B (len b), how many
// come from A.  ka / kb read the keys.
template <class KA, class KB>
__device__ __forceinline__ int cm_split(int d, int a, int b, KA ka, KB kb) {
  int lo = max(0, d - b), hi = min(d, a);
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ka(mid) <= kb(d - 1 - mid)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Insert: one CTA per output tile.  Its two diagonal searches bound the old and delta ranges, both are staged in
// shared memory, every thread merges CM_ITEMS outputs from its own diagonal, and the tile is written out coalesced.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_merge_insert(
    const float* __restrict__ scores, const long long* __restrict__ ptr, int G_old, const float* __restrict__ dsc,
    const long long* __restrict__ dptr, int G_new, const int* __restrict__ ntile, float* __restrict__ out,
    const long long* __restrict__ out_ptr, long long n_out) {
  __shared__ uint32_t sk[CM_TILE];
  __shared__ float so[CM_TILE];
  __shared__ int split[2];
  int r, first;
  if (!cm_tile_row(ntile, G_new, blockIdx.x, &r, &first)) return;
  const int ro = cm_old_row(r, G_old, G_new);
  const float* A = ro < 0 ? scores : scores + ptr[ro];
  const float* B = dsc + dptr[r];
  const int a = ro < 0 ? 0 : (int)(ptr[ro + 1] - ptr[ro]), b = (int)(dptr[r + 1] - dptr[r]);
  const int o0 = (blockIdx.x - first) * CM_TILE, o1 = min(o0 + CM_TILE, a + b), len = o1 - o0;
  if (threadIdx.x < 2) {
    const int d = threadIdx.x ? o1 : o0;
    split[threadIdx.x] = cm_split(d, a, b, [&](int i) { return calib_key(A[i]); },
                                  [&](int j) { return calib_key(B[j]); });
  }
  __syncthreads();
  const int i0 = split[0], na = split[1] - i0, j0 = o0 - i0, nb = len - na;
  for (int i = threadIdx.x; i < na; i += CPD_THREADS) sk[i] = calib_key(A[i0 + i]);
  for (int j = threadIdx.x; j < nb; j += CPD_THREADS) sk[na + j] = calib_key(B[j0 + j]);
  __syncthreads();
  const uint32_t* sa = sk;
  const uint32_t* sb = sk + na;
  const int d0 = threadIdx.x * CM_ITEMS;
  if (d0 < len) {
    int i = cm_split(d0, na, nb, [&](int x) { return sa[x]; }, [&](int x) { return sb[x]; }), j = d0 - i;
    const int d1 = min(d0 + CM_ITEMS, len);
    for (int d = d0; d < d1; ++d) {
      const bool take_a = j >= nb || (i < na && sa[i] <= sb[j]);
      so[d] = calib_value(take_a ? sa[i++] : sb[j++]);
    }
  }
  __syncthreads();
  const long long base = out_ptr[r] + o0;
  for (int d = threadIdx.x; d < len; d += CPD_THREADS)
    if (base + d < n_out) out[base + d] = so[d];
}

// Remove: one CTA per tile [s0, s1) of the old row.  The delta range the tile can touch, [lb(first), ub(last)), is
// staged in shared memory when it fits (else searched in place).  A value v drops its first c(v) copies, c(v) its
// count in the delta row, so a kept element i goes to i - ub_delta(v).  One search finds where the run of the tile's
// first value starts in the old row.
__global__ void __launch_bounds__(CPD_THREADS) k_cpd_merge_remove(
    const float* __restrict__ scores, const long long* __restrict__ ptr, int G_old, const float* __restrict__ dsc,
    const long long* __restrict__ dptr, int G_new, const int* __restrict__ ntile, float* __restrict__ out,
    const long long* __restrict__ out_ptr, long long n_out, int* __restrict__ status) {
  __shared__ uint32_t sa[CM_TILE];
  __shared__ uint32_t sd[CM_TILE];
  __shared__ int info[3];
  int r, first;
  if (!cm_tile_row(ntile, G_new, blockIdx.x, &r, &first)) return;
  const int ro = cm_old_row(r, G_old, G_new);  // a row with tiles has an old row
  const float* A = scores + ptr[ro];
  const float* D = dsc + dptr[r];
  const int a = (int)(ptr[ro + 1] - ptr[ro]), b = (int)(dptr[r + 1] - dptr[r]);
  const int s0 = (blockIdx.x - first) * CM_TILE, len = min(CM_TILE, a - s0);
  const long long out_len = out_ptr[r + 1] - out_ptr[r];
  for (int i = threadIdx.x; i < len; i += CPD_THREADS) sa[i] = calib_key(A[s0 + i]);
  __syncthreads();
  if (threadIdx.x == 0) info[0] = cm_search_g(A, 0, s0, sa[0], false);            // the first value's run start
  else if (threadIdx.x == 1) info[1] = cm_search_g(D, 0, b, sa[0], false);
  else if (threadIdx.x == 2) info[2] = cm_search_g(D, 0, b, sa[len - 1], true);
  __syncthreads();
  const int run0 = info[0], dlo = info[1], dn = info[2] - info[1];
  const bool staged = dn <= CM_TILE;
  if (staged)
    for (int j = threadIdx.x; j < dn; j += CPD_THREADS) sd[j] = calib_key(D[dlo + j]);
  __syncthreads();
  for (int i = threadIdx.x; i < len; i += CPD_THREADS) {
    const uint32_t v = sa[i];
    const int l = cm_search_s(sa, 0, i, v, false);
    const int lb_a = l ? s0 + l : run0;
    int lb_d, ub_d;
    if (staged) {
      lb_d = dlo + cm_search_s(sd, 0, dn, v, false);
      ub_d = dlo + cm_search_s(sd, lb_d - dlo, dn, v, true);
    } else {
      lb_d = cm_search_g(D, dlo, dlo + dn, v, false);
      ub_d = cm_search_g(D, lb_d, dlo + dn, v, true);
    }
    if (s0 + i - lb_a < ub_d - lb_d) continue;                                      // one of the first c(v) copies
    const long long pos = (long long)s0 + i - ub_d;
    if (pos < 0 || pos >= out_len || out_ptr[r] + pos >= n_out) {
      *status = PERT_ERR_RANGE;                                                     // a corrupted delta
      continue;
    }
    out[out_ptr[r] + pos] = calib_value(v);
  }
}

// Remove: one thread per delta element; the j-th copy of v in its delta row (j from 0) needs at least j + 1 copies of
// v in the old row.  A delta holding a value more often than the table does sets PERT_ERR_RANGE.
__global__ void k_cpd_merge_check(const float* __restrict__ scores, const long long* __restrict__ ptr, int G_old,
                                  const float* __restrict__ dsc, const long long* __restrict__ dptr, int G_new,
                                  int n_delta, int* __restrict__ status) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_delta) return;
  int lo = 0, hi = G_new;                     // the delta row holding element t: the last r with dptr[r] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (dptr[mid] <= t) lo = mid;
    else hi = mid - 1;
  }
  const int r = lo, ro = cm_old_row(r, G_old, G_new);
  if (ro < 0) {
    *status = PERT_ERR_RANGE;
    return;
  }
  const float* D = dsc + dptr[r];
  const float* A = scores + ptr[ro];
  const int j = t - (int)dptr[r], a = (int)(ptr[ro + 1] - ptr[ro]);
  const uint32_t v = calib_key(D[j]);
  const int rank = j - cm_search_g(D, 0, j, v, false);
  const int lb = cm_search_g(A, 0, a, v, false);
  if (cm_search_g(A, lb, a, v, true) - lb <= rank) *status = PERT_ERR_RANGE;
}

struct CmLayout {
  long long cnt, ntile, bsum, total, tiles_max;
};

bool cm_layout(long long G_old, long long G_new, long long n_old, long long n_delta, int sign, CmLayout* l) {
  if (G_old < 0 || G_new < G_old || G_new > INT_MAX - 2 || n_old < 1 || n_delta < 1) return false;
  if (sign != 1 && sign != -1) return false;
  const long long n_out = n_old + sign * n_delta;
  if (n_out < 1 || n_out >= (1LL << 31) || n_old >= (1LL << 31)) return false;
  l->tiles_max = std::max(n_old, n_out) / CM_TILE + G_new + 1;
  const long long rows = G_new + 1;
  long long o = 0;
  l->cnt = o;
  o += al256(4 * rows);
  l->ntile = o;
  o += al256(4 * rows);
  l->bsum = o;
  o += al256(2LL * pert_cdiv(rows, SCAN_TILE) * 4 + 16);
  l->total = o;
  return true;
}

struct CpdLayout {
  long long ptr, fill, bsum, buf0, buf1, meta, segs, tiles, hist, cursor, items, total;
  long long segs_max, tiles_max, items_max;
};

bool cpd_layout(long long n, long long G, CpdLayout* l) {
  if (n < 1 || n >= (1LL << 30) || G < 0 || G > INT_MAX - 2) return false;
  const long long total = 2 * n;              // the table's size bound: rows 0 .. G-1 and row G
  // disjoint segments of more than CB_SMALL keys; the tiles of one pass; the small items: the rows, then at most 256
  // buckets of every segment of the first three passes
  l->segs_max = total / (CB_SMALL + 1) + 1;
  l->tiles_max = total / CB_TILE + l->segs_max;
  l->items_max = std::min(G, n) + 1 + 3 * 256 * l->segs_max;
  long long o = 0;
  auto take = [&](long long bytes) {
    const long long at = o;
    o += al256(bytes);
    return at;
  };
  l->ptr = take(4 * (G + 1));
  l->fill = take(4 * std::max(G, 1LL));
  l->bsum = take(2LL * pert_cdiv(std::max(G, 1LL), SCAN_TILE) * 4 + 16);
  l->meta = take(4 * (3 * CPD_PASSES));
  l->hist = take(4 * 256 * l->segs_max);
  l->buf0 = take(4 * total);
  l->buf1 = take(4 * total);
  l->segs = take(2 * 8 * l->segs_max);
  l->tiles = take(2 * 8 * l->tiles_max);
  l->cursor = take(4 * 256 * l->segs_max);
  l->items = take(8 * l->items_max);
  l->total = o;
  return true;
}

bool cpd_query_args(const float* scores, const long long* ptr, long long G, long long min_count, const float* yhat,
                    long long ld, int col, long long Q, long long per, const int* status) {
  if (Q < 0 || per < 1 || Q * per >= (1LL << 31) || G < 0 || G > INT_MAX - 2 || min_count < 1) return false;
  if (ld < 1 || col < 0 || col >= ld) return false;
  return Q == 0 || (scores && ptr && yhat && status);
}

}  // namespace

extern "C" {

long long pert_cpd_workspace_bytes(long long n, long long n_groups) {
  CpdLayout l;
  if (!cpd_layout(n, n_groups, &l)) return PERT_ERR_BADARG;
  return l.total;
}

int pert_cpd_fit(const int64_t* y, const float* yhat, long long ld, int col, const int64_t* group, long long n,
                 long long n_groups, float* scores, long long* ptr, void* workspace, long long workspace_bytes,
                 int* status, void* stream) {
  CpdLayout l;
  if (!y || !yhat || !scores || !ptr || !workspace || !status) return PERT_ERR_BADARG;
  if (ld < 1 || col < 0 || col >= ld || !cpd_layout(n, n_groups, &l) || workspace_bytes < l.total)
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  char* w = (char*)workspace;
  int* p32 = (int*)(w + l.ptr);
  int* meta = (int*)(w + l.meta);
  int* hist = (int*)(w + l.hist);
  uint32_t* buf[2] = {(uint32_t*)(w + l.buf0), (uint32_t*)(w + l.buf1)};
  int2* segs[2] = {(int2*)(w + l.segs), (int2*)(w + l.segs) + l.segs_max};
  int2* tiles[2] = {(int2*)(w + l.tiles), (int2*)(w + l.tiles) + l.tiles_max};
  int* cursor = (int*)(w + l.cursor);
  int2* items = (int2*)(w + l.items);
  const int N = (int)n, G = (int)n_groups;
  cudaError_t e;
  // ptr, fill, bsum, meta and hist are adjacent
  if ((e = cudaMemsetAsync(w + l.ptr, 0, l.buf0 - l.ptr, st)) != cudaSuccess) return (int)e;
  calib_group_scatter(y, yhat + col, ld, group, N, 1, G, p32, (int*)(w + l.fill), (int*)(w + l.bsum), buf[0], status,
                      st);
  if (group && (e = cudaMemcpyAsync(buf[0] + n, buf[0], 4 * n, cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
    return (int)e;                            // the global row, in group order
  k_cpd_plan<<<pert_cdiv(G + 1, 256), 256, 0, st>>>(p32, G, N, meta, segs[0], tiles[0], items, ptr);
  for (int p = 0; p < CPD_PASSES; ++p) {
    const int c = p & 1, nx = c ^ 1;
    uint32_t* dst = p == CPD_PASSES - 1 ? (uint32_t*)scores : buf[nx];
    k_cpd_hist<<<(unsigned)l.tiles_max, CPD_THREADS, 0, st>>>(buf[c], segs[c], tiles[c], meta, p, hist);
    k_cpd_split<<<(unsigned)l.segs_max, CPD_THREADS, 0, st>>>(segs[c], meta, p, hist, cursor, segs[nx], tiles[nx],
                                                               items);
    k_cpd_scatter<<<(unsigned)l.tiles_max, CPD_THREADS, 0, st>>>(buf[c], dst, segs[c], tiles[c], meta, p, cursor);
  }
  k_cpd_small<<<(unsigned)std::min<long long>(l.items_max, CPD_SMALL_GRID), CPD_THREADS, 0, st>>>(buf[0], buf[1], items,
                                                                                                 meta, scores);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_cpd_merge_workspace_bytes(long long G_old, long long G_new, long long n_old, long long n_delta) {
  CmLayout l;
  if (!cm_layout(G_old, G_new, n_old, n_delta, 1, &l) && !cm_layout(G_old, G_new, n_old, n_delta, -1, &l))
    return PERT_ERR_BADARG;
  return l.total;
}

int pert_cpd_merge(const float* scores, const long long* ptr, long long G_old, long long n_old, const float* d_scores,
                   const long long* d_ptr, long long G_new, long long n_delta, int sign, float* out_scores,
                   long long* out_ptr, void* workspace, long long workspace_bytes, int* status, void* stream) {
  CmLayout l;
  if (!scores || !ptr || !d_scores || !d_ptr || !out_scores || !out_ptr || !workspace || !status)
    return PERT_ERR_BADARG;
  if (!cm_layout(G_old, G_new, n_old, n_delta, sign, &l) || workspace_bytes < l.total) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  char* w = (char*)workspace;
  int* cnt = (int*)(w + l.cnt);
  int* ntile = (int*)(w + l.ntile);
  int* bsum = (int*)(w + l.bsum);
  const int Go = (int)G_old, Gn = (int)G_new, rows = Gn + 1, sb = pert_cdiv(rows, SCAN_TILE);
  const long long n_out = n_old + sign * n_delta;
  k_cpd_merge_count<<<pert_cdiv(rows, 256), 256, 0, st>>>(ptr, Go, d_ptr, Gn, sign, cnt, ntile, status);
  k_scan_tile_sums<<<dim3(sb, 2), SCAN_THREADS, 0, st>>>(cnt, ntile, rows, bsum, sb);
  k_scan_block_sums<<<dim3(1, 2), SCAN_THREADS, 0, st>>>(bsum, sb);
  k_scan_apply<<<dim3(sb, 2), SCAN_THREADS, 0, st>>>(cnt, ntile, rows, bsum, sb);
  k_cpd_merge_ptr<<<pert_cdiv(rows, 256), 256, 0, st>>>(cnt, Gn, out_ptr);
  if (sign > 0) {
    k_cpd_merge_insert<<<(unsigned)l.tiles_max, CPD_THREADS, 0, st>>>(scores, ptr, Go, d_scores, d_ptr, Gn, ntile,
                                                                     out_scores, out_ptr, n_out);
  } else {
    k_cpd_merge_check<<<pert_cdiv(n_delta, 256), 256, 0, st>>>(scores, ptr, Go, d_scores, d_ptr, Gn, (int)n_delta,
                                                               status);
    k_cpd_merge_remove<<<(unsigned)l.tiles_max, CPD_THREADS, 0, st>>>(scores, ptr, Go, d_scores, d_ptr, Gn, ntile,
                                                                     out_scores, out_ptr, n_out, status);
  }
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_cpd_tail(const float* scores, const long long* ptr, long long n_groups, long long min_count,
                  const float* yhat, long long ld, int col, const int64_t* group, long long Q, const float* x, int S,
                  const int64_t* y, int* ge, int* gt, int* row, int* status, void* stream) {
  if (!cpd_query_args(scores, ptr, n_groups, min_count, yhat, ld, col, Q, S, status)) return PERT_ERR_BADARG;
  if ((x == nullptr) == (y == nullptr) || (y && S != 1)) return PERT_ERR_BADARG;
  if (Q == 0) return PERT_OK;
  if (!ge || !gt || !row) return PERT_ERR_BADARG;
  const int R = (int)(Q * S);
  k_cpd_tail<<<pert_cdiv(R, 256), 256, 0, (cudaStream_t)stream>>>(scores, ptr, (int)n_groups, min_count, yhat + col, ld,
                                                                 group, (int)Q, x, S, y, ge, gt, row, status);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_cpd_quantile(const float* scores, const long long* ptr, long long n_groups, long long min_count,
                      const float* yhat, long long ld, int col, const int64_t* group, long long Q, const double* taus,
                      int L, float* out, int* status, void* stream) {
  CalibTaus tv;
  if (load_calib_taus(taus, L, &tv)) return PERT_ERR_BADARG;
  if (!cpd_query_args(scores, ptr, n_groups, min_count, yhat, ld, col, Q, L, status)) return PERT_ERR_BADARG;
  if (Q == 0) return PERT_OK;
  if (!out) return PERT_ERR_BADARG;
  const int R = (int)(Q * L);
  k_cpd_quantile<<<pert_cdiv(R, 256), 256, 0, (cudaStream_t)stream>>>(scores, ptr, (int)n_groups, min_count,
                                                                     yhat + col, ld, group, (int)Q, L, tv, out, status);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
