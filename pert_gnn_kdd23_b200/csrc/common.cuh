// Shared device/host helpers for libpertgnn (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pertgnn.h"  // prototypes + PERT_ERR_* (keeps definitions and ABI header in sync)

// SM count of the current device (H100 SXM: 132, H100 PCIe: 114), read once per device.  Persistent grids are sized
// to it, and the peer all-reduce needs all of its CTAs co-resident, so it must not be a compile-time guess.
static inline int pert_num_sms() {
  static int sms[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 1;
  if (sms[dev] <= 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 1;
    sms[dev] = n;
  }
  return sms[dev];
}
#define PERT_NUM_SMS pert_num_sms()

#define PERT_LAUNCH_CHECK()                          \
  do {                                               \
    cudaError_t e__ = cudaPeekAtLastError();         \
    if (e__ != cudaSuccess) return (int)e__;         \
  } while (0)

static inline int pert_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Time bucket of a timestamp (ms): floor(ts / 30000) * 30000 with floor division (pandas //), so -1 -> -30000
// (preprocess.py:39 get_tr2ts_map).  The trace grouping labels traces with it; request assembly joins resources on it.
constexpr int64_t TG_BUCKET = 30000;
__host__ __device__ __forceinline__ int64_t pert_time_bucket(int64_t ts) {
  int64_t q = ts / TG_BUCKET;
  if (ts % TG_BUCKET != 0 && ts < 0) --q;
  return q * TG_BUCKET;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ float4 ld4(const float* p) {
  return *reinterpret_cast<const float4*>(p);
}
__device__ __forceinline__ void st4(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}
__device__ __forceinline__ float4 f4add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4fma(float s, float4 a, float4 acc) {
  return make_float4(fmaf(s, a.x, acc.x), fmaf(s, a.y, acc.y), fmaf(s, a.z, acc.z), fmaf(s, a.w, acc.w));
}
__device__ __forceinline__ float f4dot(float4 a, float4 b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ float4 f4max(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4scale(float s, float4 a) {
  return make_float4(s * a.x, s * a.y, s * a.z, s * a.w);
}
// 16-byte vector reduction to global memory (REDG.E.ADD.F32x4, sm_90+).
__device__ __forceinline__ void red4(float* p, float4 v) {
  atomicAdd(reinterpret_cast<float4*>(p), v);
}
// butterfly sum over a sub-warp group of LPR lanes; every lane of the group gets the sum.
template <int LPR>
__device__ __forceinline__ float group_sum(float v, unsigned gmask) {
#pragma unroll
  for (int off = LPR >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(gmask, v, off);
  return v;
}

// engine-internal entry points (not part of the C-ABI)
// PERT_GEMM_TC=0: the exact-fp32 SIMT GEMMs of gemm.cu instead of the tensor-core kernels (csrc/gemm_tc.cu), read once
bool pert_gemm_tc_enabled();
// live: optional device {N, B} of a padded batch (pert_batch_pad); the BatchNorm sums then count the rows below live[0].
// C: the logical width whose 1/sqrt(C) scales the logits (pert_tconv_fwd_c; C = H for an unpadded model)
int pert_tconv_fwd_stats(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                         const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if,
                         const float* t_rpc, float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E,
                         long long B_hint, int H, int C, double* bn_acc, const long long* live, int* fused,
                         void* stream);
int pert_bn_fwd_ex(const float* x, int ld_x, const float* gamma, const float* beta, float* running_mean,
                   float* running_var, long long* num_batches_tracked, float eps, float momentum, int training,
                   int relu, float* mean, float* rstd, float* y, int ld_y, long long N, int H, void* workspace,
                   long long workspace_bytes, int stats_ready, float dropout, const long long* drop_ctr,
                   int drop_layer, const long long* live, void* stream);
int pert_bn_fwd_stats(const float* x, int ld_x, const float* running_mean, const float* running_var, float eps,
                      int training, float* mean, float* rstd, long long N, int H, void* workspace,
                      long long workspace_bytes, int stats_ready, const long long* live, cudaStream_t st,
                      double** acc);
int pert_bn_bwd_ex(const float* dy, int ld_dy, const float* y, int ld_y, const float* x, int ld_x, const float* mean,
                   const float* rstd, const float* gamma, int relu, float relu_scale, int training, float* dx,
                   int ld_dx, float* dgamma, float* dbeta, float* sums, long long N, int H, const long long* live,
                   void* stream);
// pert_bn_linear_fwd_planes with the live word of a padded batch (BatchNorm statistics over the rows below live[0])
int pert_bn_linear_fwd_planes_ex(const float* A, int lda, int bn, const float* gamma, const float* beta,
                                 float* running_mean, float* running_var, long long* num_batches_tracked, float eps,
                                 float momentum, int training, float* mean, float* rstd, float* x_out, int ld_x_out,
                                 void* workspace, long long workspace_bytes, int stats_ready, float dropout,
                                 const long long* drop_ctr, int drop_layer, const long long* live, const float* W4,
                                 int ldw, const float* b4, float* planes, long long plane_stride, long long N, int H,
                                 int K, void* stream);
