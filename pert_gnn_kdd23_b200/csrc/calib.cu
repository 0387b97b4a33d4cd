// Split-conformal calibration of the quantile head (pert_calib_offsets, pert_calib_apply).
//
// Fit: the scores s = (float)y - yhat of n labelled graphs at T levels are counting-sorted by group (entry id), then for
// every (group, level) the k-th smallest score, k = max(1, ceil((n_g + 1) tau)), is selected by an MSB radix select
// over order-preserving uint32 keys: 4 passes of 8-bit digits with integer histograms, so the result is independent of
// scheduling and is an element of the score array, bit for bit.  Two tiers: a segment of at most CB_SMALL graphs is
// selected by one CTA from shared memory (k_cb_small, one CTA per (segment, level)); a larger one -- the global row of
// any real set, and a hot entry -- is cut into CB_TILE-key tiles whose CTAs add into one 256-bin global histogram per
// (segment, level) and pass (k_cb_hist), followed by one small CTA per (segment, level) that picks the digit
// (k_cb_pick).  No segment above CB_SMALL is handled by a single CTA, so a set where one entry holds 90 % of the
// graphs spreads over the whole GPU.  The host never reads the device: the large-tier grids are sized from n.
#include <limits.h>

#include <algorithm>

#include "calib.cuh"

#define CB_THREADS 256

namespace {

// One thread per segment: the large segments get a slot, their tiles and, per level, the select state {prefix, k}
// (k = 0: the level keeps the global offset, nothing to select).
__global__ void k_cb_plan(const int* __restrict__ ptr, int G, int n, int T, CalibTaus taus, long long min_count,
                          int* __restrict__ meta, int* __restrict__ large_seg, int2* __restrict__ tiles,
                          uint2* __restrict__ state) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > G) return;
  int start, len;
  calib_seg(ptr, G, n, s, &start, &len);
  if (len <= CB_SMALL) return;
  const int slot = atomicAdd(meta, 1);
  large_seg[slot] = s;
  const int nt = (len + CB_TILE - 1) / CB_TILE;
  const int base = atomicAdd(meta + 1, nt);
  for (int j = 0; j < nt; ++j) tiles[base + j] = make_int2(slot, j * CB_TILE);
  for (int t = 0; t < T; ++t) {
    const bool own = calib_own(len, taus.v[t], min_count, s == G);
    state[(long long)slot * T + t] = make_uint2(0u, own ? (uint32_t)calib_k(len, taus.v[t]) : 0u);
  }
}

// Warp 0: the digit d of a 256-bin histogram h where the running count reaches k, and the count below it.
__device__ __forceinline__ void pick_digit(const int* h, int k, int* digit, int* below) {
  const int lane = threadIdx.x & 31;
  int c[8], sum = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    c[j] = h[lane * 8 + j];
    sum += c[j];
  }
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  int run = incl - sum;
  if (run < k && k <= incl) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (run + c[j] >= k) {
        *digit = lane * 8 + j;
        *below = run;
        break;
      }
      run += c[j];
    }
  }
}

// Small tier: one CTA per (segment, level) with at most CB_SMALL keys, staged in shared memory.
__global__ void __launch_bounds__(CB_THREADS) k_cb_small(const uint32_t* __restrict__ keys, const int* __restrict__ ptr,
                                                         int G, int n, int T, CalibTaus taus, long long min_count,
                                                         uint32_t* __restrict__ sel) {
  __shared__ uint32_t sk[CB_SMALL];
  __shared__ int hist[256];
  __shared__ int s_digit, s_below;
  const int s = blockIdx.x, t = blockIdx.y;
  int start, len;
  calib_seg(ptr, G, n, s, &start, &len);
  if (len == 0 || len > CB_SMALL || !calib_own(len, taus.v[t], min_count, s == G)) return;
  int k = (int)calib_k(len, taus.v[t]);
  const uint32_t* src = keys + (long long)t * n + start;
  for (int i = threadIdx.x; i < len; i += CB_THREADS) sk[i] = src[i];
  uint32_t prefix = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    const uint32_t hi = shift == 24 ? 0u : ~0u << (shift + 8);
    hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < len; i += CB_THREADS) {
      const uint32_t key = sk[i];
      if (((key ^ prefix) & hi) == 0) atomicAdd(hist + ((key >> shift) & 255u), 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) pick_digit(hist, k, &s_digit, &s_below);
    __syncthreads();
    prefix |= (uint32_t)s_digit << shift;
    k -= s_below;
    __syncthreads();                          // s_digit / s_below are rewritten by the next pass
  }
  if (threadIdx.x == 0) sel[(long long)s * T + t] = prefix;
}

// Large tier, one pass: every tile CTA adds the digit counts of its keys that match the prefix into the global
// histogram of its (segment, level).
__global__ void __launch_bounds__(CB_THREADS) k_cb_hist(const uint32_t* __restrict__ keys, const int* __restrict__ ptr,
                                                        int G, int n, int T, const int* __restrict__ meta,
                                                        const int* __restrict__ large_seg,
                                                        const int2* __restrict__ tiles,
                                                        const uint2* __restrict__ state, int* __restrict__ hist,
                                                        int shift) {
  __shared__ int h[256];
  const int tile = blockIdx.x, t = blockIdx.y;
  if (tile >= meta[1]) return;
  const int2 tl = tiles[tile];
  const uint2 st = state[(long long)tl.x * T + t];
  if (st.y == 0) return;
  int start, len;
  calib_seg(ptr, G, n, large_seg[tl.x], &start, &len);
  const int end = min(tl.y + CB_TILE, len);
  const uint32_t hi = shift == 24 ? 0u : ~0u << (shift + 8);
  h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t* src = keys + (long long)t * n + start;
  for (int i = tl.y + threadIdx.x; i < end; i += CB_THREADS) {
    const uint32_t key = __ldg(src + i);
    if (((key ^ st.x) & hi) == 0) atomicAdd(h + ((key >> shift) & 255u), 1);
  }
  __syncthreads();
  const int c = h[threadIdx.x];
  if (c) atomicAdd(hist + ((long long)tl.x * T + t) * 256 + threadIdx.x, c);
}

// Large tier, one pass: the digit of every (segment, level), its histogram cleared for the next pass; after the last
// pass the selected key.
__global__ void __launch_bounds__(CB_THREADS) k_cb_pick(const int* __restrict__ meta, const int* __restrict__ large_seg,
                                                        int T, uint2* __restrict__ state, int* __restrict__ hist,
                                                        uint32_t* __restrict__ sel, int shift) {
  __shared__ int h[256];
  __shared__ int s_digit, s_below;
  const int slot = blockIdx.x, t = blockIdx.y;
  if (slot >= meta[0]) return;
  const long long at = (long long)slot * T + t;
  const uint2 st = state[at];
  if (st.y == 0) return;
  int* hp = hist + at * 256;
  h[threadIdx.x] = hp[threadIdx.x];
  hp[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x < 32) pick_digit(h, (int)st.y, &s_digit, &s_below);
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint2 nx = make_uint2(st.x | ((uint32_t)s_digit << shift), st.y - (uint32_t)s_below);
    state[at] = nx;
    if (shift == 0) sel[(long long)large_seg[slot] * T + t] = nx.x;
  }
}

__global__ void k_cb_final(const int* __restrict__ ptr, int G, int n, int T, CalibTaus taus, long long min_count,
                           const uint32_t* __restrict__ sel, float* __restrict__ off, int* __restrict__ count,
                           int8_t* __restrict__ own) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)(G + 1) * T) return;
  const int s = (int)(i / T), t = (int)(i % T);
  int start, len;
  calib_seg(ptr, G, n, s, &start, &len);
  const bool mine = calib_own(len, taus.v[t], min_count, s == G);
  off[i] = calib_value(sel[mine ? i : (long long)G * T + t]);
  own[i] = mine ? 1 : 0;
  if (t == 0) count[s] = len;
}

// In place on yhat [Q, T]: + off[g, t] (g outside [0, n_rows - 1): the global row n_rows - 1), then the running max.
template <int TM>
__global__ void k_cb_apply(float* __restrict__ yhat, const int64_t* __restrict__ group, int Q, int T_,
                           const float* __restrict__ off, int n_rows, int monotone,
                           const long long* __restrict__ live) {
  const int T = TM == 1 ? 1 : T_;
  int Ql = Q;
  if (live) Ql = (int)min((long long)Q, live[1]);
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Ql) return;
  float v[TM];
  float* row = yhat + (long long)q * T;
#pragma unroll
  for (int t = 0; t < TM; ++t)
    if (t < T) v[t] = row[t];
  if (off) {
    long long g = group ? group[q] : -1;
    if (g < 0 || g >= n_rows - 1) g = n_rows - 1;
    const float* o = off + g * T;
#pragma unroll
    for (int t = 0; t < TM; ++t)
      if (t < T) v[t] = __fadd_rn(v[t], o[t]);
  }
  if (monotone) {
#pragma unroll
    for (int t = 1; t < TM; ++t)
      if (t < T) v[t] = fmaxf(v[t], v[t - 1]);
  }
#pragma unroll
  for (int t = 0; t < TM; ++t)
    if (t < T) row[t] = v[t];
}

struct CalibLayout {
  long long ptr, fill, bsum, keys, sel, meta, large_seg, tiles, state, hist, total;
  long long L_max, tiles_max;
};

bool calib_layout(long long n, int T, long long G, CalibLayout* l) {
  if (n < 1 || T < 1 || T > PERT_MAX_QUANTILES || n * T >= (1LL << 31) || G < 0 || G > INT_MAX - 1) return false;
  l->L_max = n / (CB_SMALL + 1) + 1;
  l->tiles_max = 2 * ((n + CB_TILE - 1) / CB_TILE) + l->L_max;
  long long o = 0;
  auto take = [&](long long bytes) {
    const long long at = o;
    o += al256(bytes);
    return at;
  };
  l->ptr = take(4 * (G + 1));
  l->fill = take(4 * std::max(G, 1LL));
  l->bsum = take(2LL * pert_cdiv(std::max(G, 1LL), SCAN_TILE) * 4 + 16);
  l->keys = take(4 * n * T);
  l->sel = take(4 * (G + 1) * T);
  l->meta = take(16);
  l->large_seg = take(4 * l->L_max);
  l->tiles = take(8 * l->tiles_max);
  l->state = take(8 * l->L_max * T);
  l->hist = take(4 * 256 * l->L_max * T);
  l->total = o;
  return true;
}

}  // namespace

extern "C" {

long long pert_calib_workspace_bytes(long long n, int T, long long n_groups) {
  CalibLayout l;
  if (!calib_layout(n, T, n_groups, &l)) return PERT_ERR_BADARG;
  return l.total;
}

int pert_calib_offsets(const int64_t* y, const float* yhat, const int64_t* group, long long n, int T,
                       const double* taus, long long n_groups, long long min_count, float* off, int* count,
                       int8_t* own, void* workspace, long long workspace_bytes, int* status, void* stream) {
  CalibTaus tv;
  CalibLayout l;
  if (!y || !yhat || !off || !count || !own || !workspace || !status) return PERT_ERR_BADARG;
  if (load_calib_taus(taus, T, &tv) || min_count < 1 || !calib_layout(n, T, n_groups, &l)) return PERT_ERR_BADARG;
  if (workspace_bytes < l.total) return PERT_ERR_BADARG;
  for (int t = 0; t < T; ++t)
    if (calib_k(n, tv.v[t]) > n) return PERT_ERR_BADARG;        // the global row cannot be formed at this level
  cudaStream_t st = (cudaStream_t)stream;
  char* w = (char*)workspace;
  int* ptr = (int*)(w + l.ptr);
  int* fill = (int*)(w + l.fill);
  uint32_t* keys = (uint32_t*)(w + l.keys);
  uint32_t* sel = (uint32_t*)(w + l.sel);
  int* meta = (int*)(w + l.meta);
  int* large_seg = (int*)(w + l.large_seg);
  int2* tiles = (int2*)(w + l.tiles);
  uint2* state = (uint2*)(w + l.state);
  int* hist = (int*)(w + l.hist);
  const int N = (int)n, G = (int)n_groups;
  cudaError_t e;
  // ptr, fill and bsum are adjacent; meta .. hist are the plan and the large-tier histograms
  if ((e = cudaMemsetAsync(w + l.ptr, 0, l.keys - l.ptr, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(w + l.meta, 0, 16, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(w + l.hist, 0, l.total - l.hist, st)) != cudaSuccess) return (int)e;
  calib_group_scatter(y, yhat, T, group, N, T, G, ptr, fill, (int*)(w + l.bsum), keys, status, st);
  k_cb_plan<<<pert_cdiv(G + 1, 256), 256, 0, st>>>(ptr, G, N, T, tv, min_count, meta, large_seg, tiles, state);
  k_cb_small<<<dim3(G + 1, T), CB_THREADS, 0, st>>>(keys, ptr, G, N, T, tv, min_count, sel);
  for (int shift = 24; shift >= 0; shift -= 8) {
    k_cb_hist<<<dim3((unsigned)l.tiles_max, T), CB_THREADS, 0, st>>>(keys, ptr, G, N, T, meta, large_seg, tiles, state,
                                                                      hist, shift);
    k_cb_pick<<<dim3((unsigned)l.L_max, T), CB_THREADS, 0, st>>>(meta, large_seg, T, state, hist, sel, shift);
  }
  const long long R = (long long)(G + 1) * T;
  k_cb_final<<<pert_cdiv(R, 256), 256, 0, st>>>(ptr, G, N, T, tv, min_count, sel, off, count, own);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_calib_apply(float* yhat, const int64_t* group, long long Q, int T, const float* off, long long n_rows,
                     int monotone, const long long* live, void* stream) {
  if (Q < 0 || T < 1 || T > PERT_MAX_QUANTILES || Q * T >= (1LL << 31) || (Q > 0 && !yhat)) return PERT_ERR_BADARG;
  if (off && (n_rows < 1 || n_rows > INT_MAX)) return PERT_ERR_BADARG;
  if (Q == 0 || (!off && !monotone)) return PERT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = pert_cdiv(Q, 256), q = (int)Q, r = (int)n_rows, m = monotone ? 1 : 0;
  if (T == 1) k_cb_apply<1><<<grid, 256, 0, st>>>(yhat, group, q, T, off, r, m, live);
  else if (T == 2) k_cb_apply<2><<<grid, 256, 0, st>>>(yhat, group, q, T, off, r, m, live);
  else if (T <= 4) k_cb_apply<4><<<grid, 256, 0, st>>>(yhat, group, q, T, off, r, m, live);
  else k_cb_apply<8><<<grid, 256, 0, st>>>(yhat, group, q, T, off, r, m, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
