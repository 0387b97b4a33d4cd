// The parts of the conformal fit shared by the calibration offsets (calib.cu) and the conformal predictive
// distribution (cpd.cu): the score and its order-preserving uint32 key, the k rule and the own-row rule, the segments
// of the group-sorted keys, and the counting sort of the scores by group (entry id).
#pragma once
#include <string.h>

#include "common.cuh"
#include "scan.cuh"

#define CB_SMALL 4096                  // largest segment one CTA handles (16 KB of keys in shared memory)
#define CB_TILE 8192                   // keys per CTA of the large tier

namespace {

struct CalibTaus {
  double v[PERT_MAX_QUANTILES];
};

__host__ __device__ __forceinline__ long long calib_k(long long m, double tau) {
#ifdef __CUDA_ARCH__
  const double x = __dmul_rn((double)(m + 1), tau);
#else
  const double x = (double)(m + 1) * tau;
#endif
  const long long k = (long long)ceil(x);
  return k < 1 ? 1 : k;
}

// The group's own offset is used iff k <= n_g and n_g >= min_count; the global row (s == G) only needs k <= n.
__device__ __forceinline__ bool calib_own(long long m, double tau, long long min_count, bool global) {
  return m > 0 && calib_k(m, tau) <= m && (global || m >= min_count);
}

__device__ __forceinline__ uint32_t calib_key(float s) {
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float calib_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// segment s of the group-sorted keys: groups 0 .. G-1 from the scanned counts, the global row G = all n
__device__ __forceinline__ void calib_seg(const int* __restrict__ ptr, int G, int n, int s, int* start, int* len) {
  if (s == G) {
    *start = 0;
    *len = n;
  } else {
    *start = ptr[s];
    *len = ptr[s + 1] - ptr[s];
  }
}

// atomicAdd(ctr + g, 1) for every calling lane, one atomic per distinct g in the warp: a hot entry (90 % of the graphs)
// would otherwise serialise on one address.  Returns the calling lane's old value, as its own atomicAdd would.
__device__ __forceinline__ int warp_counter_add(int* ctr, int g) {
  const unsigned peers = __match_any_sync(__activemask(), g);
  const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(ctr + g, __popc(peers));
  return __shfl_sync(peers, base, leader) + __popc(peers & ((1u << lane) - 1));
}

__global__ void k_cb_count(const int64_t* __restrict__ group, int n, int G, int* __restrict__ cnt,
                           int* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t g = group[i];
  if (g < 0 || g >= G) *status = PERT_ERR_RANGE;
  else warp_counter_add(cnt, (int)g);
}

// the T keys of graph i (predictions yhat[i ld + t]) at its slot of the group order (slot i without groups); level
// t's keys are keys[t n ..)
__global__ void k_cb_scatter(const int64_t* __restrict__ y, const float* __restrict__ yhat, long long ld,
                             const int64_t* __restrict__ group, int n, int T, int G, const int* __restrict__ ptr,
                             int* __restrict__ fill, uint32_t* __restrict__ keys, int* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int pos = i;
  if (group) {
    const int64_t g = group[i];
    if (g < 0 || g >= G) return;            // k_cb_count has set the status
    pos = ptr[g] + warp_counter_add(fill, (int)g);
  }
  const float yt = (float)y[i];             // the conversion k_eval_metrics_q's coverage test uses
  for (int t = 0; t < T; ++t) {
    float s = __fsub_rn(yt, yhat[(long long)i * ld + t]);
    if (!isfinite(s)) *status = PERT_ERR_RANGE;
    if (s == 0.f) s = 0.f;                  // -0 -> +0: one key per value
    keys[(long long)t * n + pos] = calib_key(s);
  }
}

// The counting sort of the scores by group: ptr [G + 1] (zeroed by the caller) gets the scanned group counts from
// ptr[1], fill [G] (zeroed) the per-group cursors, bsum the scan's tile sums; then the keys of every level in group
// order.  Without groups the keys stay in graph order.
void calib_group_scatter(const int64_t* y, const float* yhat, long long ld, const int64_t* group, int N, int T, int G,
                         int* ptr, int* fill, int* bsum, uint32_t* keys, int* status, cudaStream_t st) {
  const int nb = pert_cdiv(N, 256);
  if (group && G > 0) {
    k_cb_count<<<nb, 256, 0, st>>>(group, N, G, ptr + 1, status);
    const int sb = pert_cdiv(G, SCAN_TILE);
    k_scan_tile_sums<<<dim3(sb, 1), SCAN_THREADS, 0, st>>>(ptr + 1, nullptr, G, bsum, sb);
    k_scan_block_sums<<<dim3(1, 1), SCAN_THREADS, 0, st>>>(bsum, sb);
    k_scan_apply<<<dim3(sb, 1), SCAN_THREADS, 0, st>>>(ptr + 1, nullptr, G, bsum, sb);
  } else if (group) {
    k_cb_count<<<nb, 256, 0, st>>>(group, N, G, ptr + 1, status);       // every id is out of range
  }
  k_cb_scatter<<<nb, 256, 0, st>>>(y, yhat, ld, group, N, T, G, ptr, fill, keys, status);
}

inline long long al256(long long b) { return (b + 255) / 256 * 256; }

int load_calib_taus(const double* taus, int T, CalibTaus* out) {
  if (T < 1 || T > PERT_MAX_QUANTILES || !taus) return PERT_ERR_BADARG;
  memset(out, 0, sizeof(*out));
  for (int t = 0; t < T; ++t) {
    if (!(taus[t] >= 0.0 && taus[t] <= 1.0)) return PERT_ERR_BADARG;
    if (t > 0 && !(taus[t] > taus[t - 1])) return PERT_ERR_BADARG;
    out->v[t] = taus[t];
  }
  return PERT_OK;
}

}  // namespace
