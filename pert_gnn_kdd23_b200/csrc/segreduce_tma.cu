// Streaming variant of the segmented reduce (the BASELINE "level-wise scatter-max" metric kernel) for messages that
// are already in CSR (target-sorted) order: out[i,:] = max|sum over rows [rowptr[i], rowptr[i+1]) of msg.
//
// The rows of consecutive segments are contiguous, so a tile of TN consecutive segments is ONE contiguous byte range.
// Persistent CTAs (one per SM) run a 3- or 4-stage (see Ring) mbarrier pipeline: a producer warp issues one TMA bulk copy
// (cp.async.bulk, complete_tx on the stage's mbarrier) per tile -- no per-thread loads, no registers, tens of KB
// in flight per SM independent of occupancy -- and 8 consumer warps reduce the staged rows from shared memory with
// 16-byte accesses and write the [TN,H] result with streaming stores.  Segment boundaries travel with the tile
// (the producer warp prefetches the rowptr slice of the NEXT tile while the current copy is in flight).
// Algorithmic bytes: 4*E*H (msg, read once) + 4*(N+1) (rowptr) + 4*N*H (out).  A tile whose rows exceed the stage
// capacity (very high in-degree) is reduced straight from global memory instead.
#include "common.cuh"
#include <type_traits>

namespace {

constexpr int TN = 32;        // segments (nodes) per tile
// ring geometry by row width: a tile of 32 segments at ~3 rows each is 12 / 24 / 48 KB for H = 32 / 64 / 128; the stage
// must hold a tile with headroom (an oversized tile falls back to global loads), and 4 stages of 48 KB fit next to
// each other in the 227 KB of shared memory an H100 block may use
template <int LPR>
struct Ring {
  static constexpr int STAGES = (LPR >= 32) ? 3 : 4;
  static constexpr int STAGE_BYTES = (LPR >= 32) ? 72 * 1024 : 48 * 1024;
};
constexpr int CONS_WARPS = 8;
constexpr int THREADS = (CONS_WARPS + 1) * 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

struct StageHdr {
  int ptr[TN + 1];   // rowptr slice of the tile
  int staged;        // 1: rows are in the stage buffer; 0: read them from global (tile larger than the stage)
  int pad[2];
};

template <int LPR, bool IS_MAX>
__global__ void __launch_bounds__(THREADS, 1) k_segreduce_stream(const float* __restrict__ msg,
                                                                 const int* __restrict__ rowptr,
                                                                 float* __restrict__ out, int N, int ntiles) {
  constexpr int H = 4 * LPR;
  constexpr int STAGES = Ring<LPR>::STAGES;
  constexpr int STAGE_BYTES = Ring<LPR>::STAGE_BYTES;
  constexpr int CAP = STAGE_BYTES / (H * 4);
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ __align__(8) uint64_t full[STAGES], empty[STAGES];
  __shared__ StageHdr hdr[STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == CONS_WARPS) {
    // ================= producer warp =================
    uint32_t stage = 0, ph = 0;
    int t = blockIdx.x;
    // rowptr slice of the first tile
    int v0 = 0, v1 = 0;
    if (t < ntiles) {
      const int n0 = t * TN;
      v0 = __ldg(rowptr + min(n0 + lane, N));
      v1 = __ldg(rowptr + min(n0 + TN, N));
    }
    for (; t < ntiles; t += gridDim.x) {
      const int tn = t + gridDim.x;
      int nv0 = 0, nv1 = 0;
      if (tn < ntiles) {   // prefetch the next tile's boundaries while this tile's copy is in flight
        const int nn0 = tn * TN;
        nv0 = __ldg(rowptr + min(nn0 + lane, N));
        nv1 = __ldg(rowptr + min(nn0 + TN, N));
      }
      mbar_wait(&empty[stage], ph ^ 1);
      hdr[stage].ptr[lane] = v0;
      const int e0 = __shfl_sync(0xffffffffu, v0, 0);
      const int rows = v1 - e0;
      if (lane == 0) {
        hdr[stage].ptr[TN] = v1;
        hdr[stage].staged = rows <= CAP;
      }
      __syncwarp();
      if (lane == 0) {
        if (rows > 0 && rows <= CAP) {
          const uint32_t bytes = (uint32_t)rows * H * 4;
          mbar_arrive_tx(&full[stage], bytes);
          bulk_g2s(smem + (size_t)stage * STAGE_BYTES, msg + (size_t)e0 * H, bytes, &full[stage]);
        } else {
          mbar_arrive(&full[stage]);
        }
      }
      v0 = nv0;
      v1 = nv1;
      if (++stage == STAGES) {
        stage = 0;
        ph ^= 1;
      }
    }
  } else {
    // ================= consumers: lane groups of LPR lanes, one segment at a time =================
    constexpr int GPC = CONS_WARPS * 32 / LPR;
    const int lig = lane % LPR;
    const int grp = warp * (32 / LPR) + lane / LPR;
    uint32_t stage = 0, ph = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int n0 = t * TN;
      mbar_wait(&full[stage], ph);
      const StageHdr& h = hdr[stage];
      const int e0 = h.ptr[0];
      const bool staged = h.staged != 0;
      const float* srows = reinterpret_cast<const float*>(smem + (size_t)stage * STAGE_BYTES);
      for (int loc = grp; loc < TN; loc += GPC) {
        const int i = n0 + loc;
        if (i >= N) break;
        const int p0 = h.ptr[loc], p1 = h.ptr[loc + 1];
        const float init = IS_MAX ? -INFINITY : 0.f;
        float4 acc = make_float4(init, init, init, init);
        if (staged) {
          const float* p = srows + (size_t)(p0 - e0) * H + lig * 4;
          for (int r = p0; r < p1; ++r, p += H) {
            const float4 v = *reinterpret_cast<const float4*>(p);
            acc = IS_MAX ? f4max(acc, v) : f4add(acc, v);
          }
        } else {
          const float* p = msg + (size_t)p0 * H + lig * 4;
          for (int r = p0; r < p1; ++r, p += H) {
            const float4 v = __ldcs(reinterpret_cast<const float4*>(p));
            acc = IS_MAX ? f4max(acc, v) : f4add(acc, v);
          }
        }
        if (IS_MAX && p0 == p1) acc = f4zero();
        __stcs(reinterpret_cast<float4*>(out + (size_t)i * H + lig * 4), acc);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == STAGES) {
        stage = 0;
        ph ^= 1;
      }
    }
  }
}

template <int LPR>
int launch(const float* msg, const int* rowptr, float* out, long long N, int op, cudaStream_t st) {
  const int ntiles = (int)((N + TN - 1) / TN);
  const size_t smem = (size_t)Ring<LPR>::STAGES * Ring<LPR>::STAGE_BYTES;
  int grid = PERT_NUM_SMS < ntiles ? PERT_NUM_SMS : ntiles;
  cudaError_t e;
  if (op == 1) {
    e = cudaFuncSetAttribute(k_segreduce_stream<LPR, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    k_segreduce_stream<LPR, true><<<grid, THREADS, smem, st>>>(msg, rowptr, out, (int)N, ntiles);
  } else {
    e = cudaFuncSetAttribute(k_segreduce_stream<LPR, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    k_segreduce_stream<LPR, false><<<grid, THREADS, smem, st>>>(msg, rowptr, out, (int)N, ntiles);
  }
  return PERT_OK;
}

}  // namespace

// PERT_ERR_UNSUPPORTED => caller uses the per-row kernels of segreduce.cu
int pert_segreduce_stream(const float* msg, const int* rowptr, float* out, long long N, int H, int op,
                          cudaStream_t st) {
  if ((((uintptr_t)msg | (uintptr_t)out) & 15) != 0 || N < 4096) return PERT_ERR_UNSUPPORTED;
  switch (H) {
    case 32: return launch<8>(msg, rowptr, out, N, op, st);
    case 64: return launch<16>(msg, rowptr, out, N, op, st);
    case 128: return launch<32>(msg, rowptr, out, N, op, st);
    default: return PERT_ERR_UNSUPPORTED;
  }
}
