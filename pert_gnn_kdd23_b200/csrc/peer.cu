// Gradient all-reduce fused with Adam over NVLink peer memory: ONE kernel per step on every rank, no NCCL call on
// the step path (the reference is single-GPU: pert_gnn.py:343,247 `Adam.step`; this is its data-parallel form).
//
// Every rank owns an "exchange" allocation (cudaMalloc, exported with cudaIpcGetMemHandle and mapped by the peers):
//   [ n_al floats  G : this rank's flat gradient of the current step (read by the peers)            ]
//   [ n_al floats  P : updated parameters, slice q written by rank q                                 ]
//   [ PEER_MAX u64 f1: f1[src] = last step for which rank `src` has published its gradient          ]
//   [ PEER_MAX u64 f2: f2[src] = last step for which rank `src` has written its parameter slice here ]
//   [ 2 x u32        : grid arrival counters of this rank's own kernel (phase 1 / phase 4)           ]
// Step t on rank r (k_reduce_scatter_adam; default for more than 4 ranks): reduce-scatter + Adam on the owned slice + all-gather of the
// updated parameters, so every rank pulls 1/W of every peer's gradient instead of all of it (W = 8: 1.4 MB instead of
// 11 MB per rank and step at cfg2) and runs Adam on 1/W of the parameters (ZeRO-1: m, v are only maintained for the
// owned slice):
//   1. publish: copy the local gradient into G (float4, whole grid); __threadfence_system; the LAST CTA to arrive
//      (monotonic counter) stores t into f1[r] of EVERY rank (st.release.sys over NVLink).
//   2. wait until f1[*] >= t locally (ld.acquire.sys; bounded spin: a lost peer sets `status` instead of hanging).
//   3. slice r of the parameters: sum the world's G in rank order 0..W-1 (cache-bypassing peer loads, all issued before
//      the first add), apply torch.optim.Adam's update, store the new parameters locally and into P of every peer.
//   4. __threadfence_system; the last CTA stores t into f2[r] of every rank.
//   5. wait until f2[*] >= t, copy the other ranks' slices P -> parameters (local).
// Replicas are bit-identical by construction (every element is computed once).  Buffer reuse needs no extra barrier:
// G of step t+1 is written after this rank's step-t kernel ended, i.e. after f2[*] >= t, which every peer set after
// its last read of G; P of step t+1 is written by peers only after f1[r] >= t+1, set after this rank's step-t copy.
// Up to 4 ranks (or PERT_PEER_MODE=ag) the first-generation kernel runs instead (k_allreduce_adam: G and P are the two
// halves of a double-buffered gradient copy, every rank pulls every peer's whole gradient and applies the full Adam;
// one flag exchange instead of two -- cheaper while the pulled volume is small).
#include "common.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int PEER_MAX = 8;

struct PeerArgs {
  float* p;
  const float* g;
  float* m;
  float* v;
  long long n, n_al;
  float lr, b1, b2, eps, wd, bc1, bc2_sqrt, grad_scale;
  float* xbuf[PEER_MAX];
  int rank, world;
  unsigned long long step;     // 1, 2, 3, ... (same on every rank)
  unsigned int arrive_target;  // value of the grid counter that identifies the last CTA of this launch
  int* status;
  long long* timing;           // optional [5]: += ns of CTA 0 in publish / wait / reduce+Adam / gather, += 1 (calls)
};

__device__ __forceinline__ unsigned long long* flags_of(float* xbuf, long long n_al) {
  return reinterpret_cast<unsigned long long*>(xbuf + 2 * n_al);     // f1[PEER_MAX] | f2[PEER_MAX] | ctr1 | ctr2
}
__device__ __forceinline__ unsigned int* ctrs_of(float* xbuf, long long n_al) {
  return reinterpret_cast<unsigned int*>(flags_of(xbuf, n_al) + 2 * PEER_MAX);
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ long long gtime_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__global__ void __launch_bounds__(256) k_allreduce_adam(PeerArgs a) {
  __shared__ int s_last;
  const bool stamp = a.timing && blockIdx.x == 0 && threadIdx.x == 0;
  long long ts0 = 0, ts1 = 0, ts2 = 0;
  if (stamp) ts0 = gtime_ns();
  const long long n4 = a.n >> 2;                 // n is padded to a multiple of 4 by the caller's layout (n_al)
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float* mine = a.xbuf[a.rank] + (a.step & 1ull) * a.n_al;
  // ---- 1. publish
  for (long long i = t0; i < n4; i += stride) st4(mine + i * 4, ldg4(a.g + i * 4));
  for (long long i = (n4 << 2) + t0; i < a.n; i += stride) mine[i] = a.g[i];
  __threadfence_system();
  __syncthreads();
  unsigned long long* my_flags = flags_of(a.xbuf[a.rank], a.n_al);
  unsigned int* ctr = ctrs_of(a.xbuf[a.rank], a.n_al);
  if (threadIdx.x == 0) s_last = (atomicAdd(ctr, 1u) == a.arrive_target);
  __syncthreads();
  if (s_last && threadIdx.x < a.world) {
    __threadfence_system();
    st_release_sys(flags_of(a.xbuf[threadIdx.x], a.n_al) + a.rank, a.step);
  }
  if (stamp) ts1 = gtime_ns();
  // ---- 2. wait for every rank's gradient of this step
  if (threadIdx.x < a.world) {
    const long long t_start = clock64();
    while (ld_acquire_sys(my_flags + threadIdx.x) < a.step) {
      if (clock64() - t_start > 6000000000LL) {   // ~3 s: a peer is gone; report instead of hanging the device
        if (a.status) atomicExch(a.status, PERT_ERR_PEER_TIMEOUT);
        break;
      }
    }
  }
  __syncthreads();
  if (stamp) ts2 = gtime_ns();
  // ---- 3. reduce in rank order + Adam
  const long long off = (a.step & 1ull) * a.n_al;
  for (long long i = t0; i < n4; i += stride) {
    // all peers' loads are issued before the first add (one NVLink round trip per element instead of `world`; r2 at 8
    // GPUs: this phase took 22 us with the loads chained through the running sum); the sum keeps the rank order
    float4 pv_r[PEER_MAX];
#pragma unroll
    for (int r = 0; r < PEER_MAX; ++r)
      pv_r[r] = r < a.world ? __ldcv(reinterpret_cast<const float4*>(a.xbuf[r] + off) + i) : f4zero();
    const float4 pv = ld4(a.p + i * 4), mv = ld4(a.m + i * 4), vv = ld4(a.v + i * 4);
    float4 s = f4zero();
#pragma unroll
    for (int r = 0; r < PEER_MAX; ++r)
      if (r < a.world) s = f4add(s, pv_r[r]);
    float gs[4] = {s.x, s.y, s.z, s.w}, pp[4] = {pv.x, pv.y, pv.z, pv.w}, mm[4] = {mv.x, mv.y, mv.z, mv.w},
          vs[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float gi = gs[k] * a.grad_scale;
      if (a.wd != 0.f) gi = fmaf(a.wd, pp[k], gi);
      mm[k] = mm[k] + (1.f - a.b1) * (gi - mm[k]);
      vs[k] = a.b2 * vs[k] + (1.f - a.b2) * gi * gi;
      pp[k] = pp[k] - (a.lr / a.bc1) * (mm[k] / (sqrtf(vs[k]) / a.bc2_sqrt + a.eps));
    }
    st4(a.p + i * 4, make_float4(pp[0], pp[1], pp[2], pp[3]));
    st4(a.m + i * 4, make_float4(mm[0], mm[1], mm[2], mm[3]));
    st4(a.v + i * 4, make_float4(vs[0], vs[1], vs[2], vs[3]));
  }
  for (long long i = (n4 << 2) + t0; i < a.n; i += stride) {
    float s = 0.f;
    for (int r = 0; r < a.world; ++r) s += __ldcv(a.xbuf[r] + off + i);
    float gi = s * a.grad_scale;
    const float pi = a.p[i];
    if (a.wd != 0.f) gi = fmaf(a.wd, pi, gi);
    const float mi = a.m[i] + (1.f - a.b1) * (gi - a.m[i]);
    const float vi = a.b2 * a.v[i] + (1.f - a.b2) * gi * gi;
    a.m[i] = mi;
    a.v[i] = vi;
    a.p[i] = pi - (a.lr / a.bc1) * (mi / (sqrtf(vi) / a.bc2_sqrt + a.eps));
  }
  if (stamp) {   // phase times of CTA 0 (publish incl. the grid arrival; wait = slowest rank's skew + flag latency)
    const long long ts3 = gtime_ns();
    a.timing[0] += ts1 - ts0;
    a.timing[1] += ts2 - ts1;
    a.timing[2] += ts3 - ts2;
    a.timing[4] += 1;
  }
}

__device__ __forceinline__ void adam4(const PeerArgs& a, float4 s, float4& pv, float4& mv, float4& vv) {
  float gs[4] = {s.x, s.y, s.z, s.w}, pp[4] = {pv.x, pv.y, pv.z, pv.w}, mm[4] = {mv.x, mv.y, mv.z, mv.w},
        vs[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float gi = gs[k] * a.grad_scale;
    if (a.wd != 0.f) gi = fmaf(a.wd, pp[k], gi);
    mm[k] = mm[k] + (1.f - a.b1) * (gi - mm[k]);
    vs[k] = a.b2 * vs[k] + (1.f - a.b2) * gi * gi;
    pp[k] = pp[k] - (a.lr / a.bc1) * (mm[k] / (sqrtf(vs[k]) / a.bc2_sqrt + a.eps));
  }
  pv = make_float4(pp[0], pp[1], pp[2], pp[3]);
  mv = make_float4(mm[0], mm[1], mm[2], mm[3]);
  vv = make_float4(vs[0], vs[1], vs[2], vs[3]);
}

// grid-wide arrival: true in the last CTA of this launch to get here (after every thread's earlier writes are visible
// system-wide)
__device__ __forceinline__ bool grid_arrive_last(unsigned int* ctr, unsigned int target, int* s_last) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) *s_last = (atomicAdd(ctr, 1u) == target);
  __syncthreads();
  return *s_last != 0;
}
__device__ __forceinline__ void wait_flags(const PeerArgs& a, unsigned long long* flags) {
  if (threadIdx.x < a.world) {
    const long long t_start = clock64();
    while (ld_acquire_sys(flags + threadIdx.x) < a.step) {
      if (clock64() - t_start > 6000000000LL) {   // ~3 s: a peer is gone; report instead of hanging the device
        if (a.status) atomicExch(a.status, PERT_ERR_PEER_TIMEOUT);
        break;
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) k_reduce_scatter_adam(PeerArgs a) {
  __shared__ int s_last;
  const bool stamp = a.timing && blockIdx.x == 0 && threadIdx.x == 0;
  long long ts[6] = {0, 0, 0, 0, 0, 0};
  if (stamp) ts[0] = gtime_ns();
  const long long n4 = a.n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float* G = a.xbuf[a.rank];
  float* P = G + a.n_al;
  unsigned long long* f1 = flags_of(G, a.n_al);
  unsigned long long* f2 = f1 + PEER_MAX;
  unsigned int* ctr = ctrs_of(G, a.n_al);
  // ---- 1. publish
  for (long long i = t0; i < n4; i += stride) st4(G + i * 4, ldg4(a.g + i * 4));
  for (long long i = (n4 << 2) + t0; i < a.n; i += stride) G[i] = a.g[i];
  if (grid_arrive_last(ctr, a.arrive_target, &s_last) && threadIdx.x < a.world) {
    __threadfence_system();
    st_release_sys(flags_of(a.xbuf[threadIdx.x], a.n_al) + a.rank, a.step);
  }
  if (stamp) ts[1] = gtime_ns();
  // ---- 2. every rank's gradient of this step is visible
  wait_flags(a, f1);
  if (stamp) ts[2] = gtime_ns();
  // ---- 3. owned slice: rank-ordered sum + Adam, new parameters to every rank
  const long long chunk4 = (n4 + a.world - 1) / a.world;
  const long long lo4 = (long long)a.rank * chunk4;
  const long long hi4 = lo4 + chunk4 < n4 ? lo4 + chunk4 : n4;
  for (long long i = lo4 + t0; i < hi4; i += stride) {
    float4 gv[PEER_MAX];
#pragma unroll
    for (int r = 0; r < PEER_MAX; ++r)
      gv[r] = r < a.world ? __ldcv(reinterpret_cast<const float4*>(a.xbuf[r]) + i) : f4zero();
    float4 pv = ld4(a.p + i * 4), mv = ld4(a.m + i * 4), vv = ld4(a.v + i * 4);
    float4 s = f4zero();
#pragma unroll
    for (int r = 0; r < PEER_MAX; ++r)
      if (r < a.world) s = f4add(s, gv[r]);
    adam4(a, s, pv, mv, vv);
    st4(a.p + i * 4, pv);
    st4(a.m + i * 4, mv);
    st4(a.v + i * 4, vv);
#pragma unroll
    for (int r = 0; r < PEER_MAX; ++r)
      if (r < a.world && r != a.rank) st4(a.xbuf[r] + a.n_al + i * 4, pv);
  }
  if (a.rank == a.world - 1) {   // scalar tail (n % 4 elements) belongs to the last rank
    for (long long i = (n4 << 2) + t0; i < a.n; i += stride) {
      float s = 0.f;
      for (int r = 0; r < a.world; ++r) s += __ldcv(a.xbuf[r] + i);
      float gi = s * a.grad_scale;
      const float pi = a.p[i];
      if (a.wd != 0.f) gi = fmaf(a.wd, pi, gi);
      const float mi = a.m[i] + (1.f - a.b1) * (gi - a.m[i]);
      const float vi = a.b2 * a.v[i] + (1.f - a.b2) * gi * gi;
      const float pn = pi - (a.lr / a.bc1) * (mi / (sqrtf(vi) / a.bc2_sqrt + a.eps));
      a.m[i] = mi;
      a.v[i] = vi;
      a.p[i] = pn;
      for (int r = 0; r < a.world; ++r)
        if (r != a.rank) a.xbuf[r][a.n_al + i] = pn;
    }
  }
  // ---- 4. this rank's slice has landed everywhere
  if (grid_arrive_last(ctr + 1, a.arrive_target, &s_last) && threadIdx.x < a.world) {
    __threadfence_system();
    st_release_sys(flags_of(a.xbuf[threadIdx.x], a.n_al) + PEER_MAX + a.rank, a.step);
  }
  if (stamp) ts[3] = gtime_ns();
  // ---- 5. collect the other ranks' slices
  wait_flags(a, f2);
  for (long long i = t0; i < n4; i += stride)
    if (i < lo4 || i >= hi4) st4(a.p + i * 4, __ldcv(reinterpret_cast<const float4*>(P) + i));
  if (a.rank != a.world - 1)
    for (long long i = (n4 << 2) + t0; i < a.n; i += stride) a.p[i] = __ldcv(P + i);
  if (stamp) {
    ts[4] = gtime_ns();
    a.timing[0] += ts[1] - ts[0];
    a.timing[1] += ts[2] - ts[1];
    a.timing[2] += ts[3] - ts[2];
    a.timing[3] += ts[4] - ts[3];
    a.timing[4] += 1;
  }
}

inline long long al64(long long n) { return (n + 63) / 64 * 64; }

}  // namespace

extern "C" {

long long pert_peer_exchange_bytes(long long n) {
  if (n < 0) return 0;
  return 2 * al64(n) * 4 + 2 * PEER_MAX * 8 + 64;
}

// Allocates + zeroes this rank's exchange buffer and returns its 64-byte CUDA IPC handle.
int pert_peer_alloc(long long bytes, void** ptr, unsigned char* handle64) {
  if (bytes <= 0 || !ptr || !handle64) return PERT_ERR_BADARG;
  cudaError_t e = cudaMalloc(ptr, (size_t)bytes);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemset(*ptr, 0, (size_t)bytes)) != cudaSuccess) return (int)e;
  cudaIpcMemHandle_t h;
  if ((e = cudaIpcGetMemHandle(&h, *ptr)) != cudaSuccess) return (int)e;
  static_assert(sizeof(h) == 64, "CUDA IPC handle size");
  memcpy(handle64, &h, 64);
  return PERT_OK;
}
int pert_peer_open(const unsigned char* handle64, void** ptr) {
  if (!handle64 || !ptr) return PERT_ERR_BADARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? PERT_OK : (int)e;
}
int pert_peer_close(void* ptr) {
  if (!ptr) return PERT_OK;
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  return e == cudaSuccess ? PERT_OK : (int)e;
}
int pert_peer_free(void* ptr) {
  if (!ptr) return PERT_OK;
  cudaError_t e = cudaFree(ptr);
  return e == cudaSuccess ? PERT_OK : (int)e;
}

// xbufs: HOST array of `world` device pointers (index = rank; xbufs[rank] = own allocation, the others peer-mapped),
// every allocation sized pert_peer_exchange_bytes(n).  `step` = 1, 2, ... identical on all ranks and equal to the
// number of calls so far (it also is Adam's bias-correction step).  All ranks must call once per step.
int pert_allreduce_adam(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                        float eps, float weight_decay, long long step, float grad_scale, void* const* xbufs, int rank,
                        int world, int* status, long long* timing, void* stream) {
  if (!p || !g || !m || !v || n < 0 || step < 1 || !xbufs || world < 1 || world > PEER_MAX || rank < 0 || rank >= world)
    return PERT_ERR_BADARG;
  if (((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) return PERT_ERR_BADARG;
  if (n == 0) return PERT_OK;
  PeerArgs a;
  a.p = p; a.g = g; a.m = m; a.v = v; a.n = n; a.n_al = al64(n);
  a.lr = lr; a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.wd = weight_decay;
  a.bc1 = 1.f - powf(beta1, (float)step);
  a.bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  a.grad_scale = grad_scale;
  for (int r = 0; r < PEER_MAX; ++r) a.xbuf[r] = r < world ? (float*)xbufs[r] : nullptr;
  for (int r = 0; r < world; ++r)
    if (!a.xbuf[r]) return PERT_ERR_BADARG;
  a.rank = rank; a.world = world; a.step = (unsigned long long)step; a.status = status; a.timing = timing;
  long long blocks = pert_cdiv(n / 4 + 1, 256);
  if (blocks > PERT_NUM_SMS) blocks = PERT_NUM_SMS;   // all CTAs co-resident: they wait on each other's arrival
  if (blocks < 1) blocks = 1;
  // the grid counter is monotonic: after `step` launches of `blocks` CTAs the last arrival reads step*blocks - 1
  a.arrive_target = (unsigned int)((unsigned long long)step * (unsigned long long)blocks - 1ull);
  // the reduce-scatter form pays a second flag round and wins it back only when the pulled volume shrinks enough,
  // i.e. at more than 4 ranks.  PERT_PEER_MODE=ag|rs overrides (same value on every rank).
  static int mode = -1;   // 0 auto, 1 all-gather form, 2 reduce-scatter form
  if (mode < 0) {
    const char* e = getenv("PERT_PEER_MODE");
    mode = (e && e[0] == 'a') ? 1 : ((e && e[0] == 'r') ? 2 : 0);
  }
  const bool rs = mode == 2 || (mode == 0 && world > 4);
  if (rs) k_reduce_scatter_adam<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a);
  else k_allreduce_adam<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
