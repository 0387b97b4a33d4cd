// Shared device/host helpers for libpertgnn (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
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

// ---- programmatic dependent launch (sm_90).  A kernel launched through launch_pdl may start while its predecessor in
// the stream (or captured graph) is still draining, and runs its set-up (weight staging, index staging, barrier init)
// before pdl_wait(), which returns once the predecessor has completed and its memory is visible.  Ordering rule, for
// every kernel launched this way:
//   - it calls pdl_wait() on every path that touches data its predecessor writes, and pdl_trigger() only after
//     pdl_wait(), so that kernel n's set-up can start only once kernel n - 2 has completed;
//   - before pdl_wait() it reads only data written by kernel n - 2 or earlier (packed parameters, the graph index, edge
//     tables, forward activations in the backward) and writes no global memory at all: no read-after-write and no
//     write-after-read race with kernel n - 1;
//   - where unsure, pdl_wait() is its first statement.
// The step engine launches its conv chain this way (node-linear forward, conv forward, conv backward target and source
// passes, node-linear backward), so each kernel's set-up overlaps its predecessor's drain and launch.
// tests/test_pdl_contract.py checks the textual form of these rules over csrc/*.cu.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// The attribute is set only while the step engine issues its chain (PdlChain, engine.cu), where every predecessor is
// known.  Called on its own, a kernel keeps plain stream order: the caller's last kernel may have written what its
// set-up reads.  (griddepcontrol.wait returns at once in a kernel launched without the attribute.)  The same flag turns
// on the chain's L2 eviction hints and its discards of dead scratch (sm90.cuh, DESIGN section 1).
inline thread_local bool pert_pdl_chain = false;
struct PdlChain {
  bool prev;
  explicit PdlChain(bool on) : prev(pert_pdl_chain) { pert_pdl_chain = on; }
  ~PdlChain() { pert_pdl_chain = prev; }
};

// cudaLaunchKernelEx with programmatic stream serialisation (inside a PdlChain), and with a (cluster_x, 1, 1) cluster
// when cluster_x > 0.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl_cluster(int cluster_x, void (*kernel)(KArgs...), dim3 grid, dim3 block,
                                             size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pert_pdl_chain) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (cluster_x > 0) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n++].val.clusterDim.z = 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, ((KArgs)args)...);
}
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
  return launch_pdl_cluster(0, kernel, grid, block, smem, st, args...);
}

// Time bucket of a timestamp (ms): floor(ts / 30000) * 30000 with floor division (pandas //), so -1 -> -30000
// (preprocess.py:39 get_tr2ts_map).  The trace grouping labels traces with it; request assembly joins resources on it.
constexpr int64_t TG_BUCKET = 30000;
__host__ __device__ __forceinline__ int64_t pert_time_bucket(int64_t ts) {
  int64_t q = ts / TG_BUCKET;
  if (ts % TG_BUCKET != 0 && ts < 0) --q;
  return q * TG_BUCKET;
}

// Largest b in [0, n) with off[b] <= v, for an exclusive prefix sum off (non-decreasing, off[0] = 0 <= v): the segment
// that holds item v.  The compares run in the type of v, so an int item costs 32-bit compares.
template <typename V>
__device__ __forceinline__ int upper_seg(const int* __restrict__ off, int n, V v) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= v) lo = mid;
    else hi = mid;
  }
  return lo;
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
// Host side of one torch.optim.Adam step t: step_size = lr / (1 - beta1^t) and bc2_sqrt = sqrt(1 - beta2^t), computed
// in double as torch does and rounded once to float.  In float, 1 - beta^t cancels: at t = 2 the rounding of
// powf(0.999f, 2) alone is up to 1.5e-5 of 1 - beta2^t.
struct PertAdamScalars {
  float step_size, bc2_sqrt;
};
static inline PertAdamScalars pert_adam_scalars(float lr, float beta1, float beta2, long long step) {
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
  return {(float)((double)lr / bc1), (float)sqrt(bc2)};
}
// One element of torch.optim.Adam (amsgrad = False, maximize = False): L2 weight decay added to the scaled gradient
// (not AdamW's decoupled decay), m by lerp as torch's foreach path, then p -= step_size * m / (sqrt(v) / bc2_sqrt + eps).
// k_adam and the vector bodies and scalar tails of both peer kernels (peer.cu) run this one function, every rounding
// spelled out, so that they agree bit for bit whatever the compiler contracts around it.
__device__ __forceinline__ void adam_elem(float g, float& p, float& m, float& v, float grad_scale, float wd, float b1,
                                          float b2, float eps, float step_size, float bc2_sqrt) {
  float gi = __fmul_rn(g, grad_scale);
  if (wd != 0.f) gi = fmaf(wd, p, gi);
  m = fmaf(__fsub_rn(gi, m), __fsub_rn(1.f, b1), m);
  v = fmaf(__fmul_rn(__fsub_rn(1.f, b2), gi), gi, __fmul_rn(b2, v));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
  p = fmaf(-step_size, __fdiv_rn(m, denom), p);
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
