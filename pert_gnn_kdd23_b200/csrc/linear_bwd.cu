// Fused backward of the plane-blocked node linear (q|k|v|skip = X . W4^T + b4, W4 [4H, K]) in ONE pass over the
// gradient planes dY = [dq|dk|dv|ds] (4 planes of [N, H], row stride H, plane stride pz):
//   dW4[4H, K] += dY^T . X        db4[4H] += colsum(dY)        dX[:, 0:Kd] = dY . W4[:, 0:Kd]
// The two-kernel path (k_gemm_tn_wg + k_gemm_nt_wg) reads the 52 MB of dY twice at the flagship shape, more than L2
// holds; here dY and X are read from HBM once and dX written once.
//
// Layout: a cluster of 4 CTAs, CTA r owns plane r (r = 0 q, 1 k, 2 v, 3 skip), persistent over a contiguous range of
// 64-row tiles.  Per CTA:
//   - thread 0 streams the tile's plane-r block of dY (64 x H, one contiguous 16 KB) and X block (64 x K, contiguous)
//     with bulk copies into a 3-stage ring (2 at Kd = 80; one mbarrier per stage, completion counted in bytes);
//   - warpgroup 0, data gradient: A = the dY tile (shared -> registers -> hi / lo), B = the plane's slice of W4^T
//     [Kd, H], hi / lo, resident in shared memory; the [64, Kd] fp32 partial goes to a double-buffered shared slot;
//   - warpgroup 1, weight and bias gradient: A = dY^T gathered from the same staged tile, B = the X block transposed
//     and split into the K-major layout, 32 rows at a time (the second chunk is split while the first is multiplied).
//     Every 32-row tensor-core sum is added (round to nearest) into per-thread fp32 partials (no running tensor-core
//     sum spans more than 32 rows, as in k_gemm_tn_wg); the bias gradient is summed from the same A values.  At the
//     end the partials go to dW4 / db4 with vector red.global;
//   - after a cluster barrier, warpgroup 0 of CTA r sums rows 16r..16r+15 of the four partials in the fixed order q,
//     k, v, skip through distributed shared memory and writes them to dX with 16-byte stores: no memset, no global
//     atomics, and dX is bit-identical from run to run.  It does so for tile i - 1 right after its data gradient of
//     tile i, while warpgroup 1 is still busy with the longer weight gradient.
// Optional BatchNorm-backward reduction (bn_sums != null, K = Kd = H): X is y = relu(bn(x)) [dropout-masked] of the
// previous conv, and the dX rows just summed are dy of that BatchNorm.  Warpgroup 0 also reads those rows of y (X) and
// x from global memory (the stage of the tile has been refilled by then), requested before the data gradient of the
// next tile so that they arrive while it runs, and accumulates sum dz and sum dz*xhat per column in registers (bn.cuh,
// the expressions of k_bn_bwd_reduce) over the rows below live[0]; at the end one fp64 atomic per column and CTA adds
// them to bn_sums.  This replaces the k_bn_bwd_reduce pass over dx, y and x; the apply runs in the conv backward target
// pass (tconv_tile.cu).
// Accuracy: 3xTF32 (hi*hi + lo*hi + hi*lo, round-to-nearest split); the data gradient is four K = H tensor-core sums
// added in fp32.
#include "common.cuh"
#include "bn.cuh"
#include "sm90.cuh"
#include <stdlib.h>

namespace {

constexpr int LB_THREADS = 256;   // warpgroup 0: data gradient, warpgroup 1: weight / bias gradient
constexpr int LB_H = 64;          // plane width
constexpr int LB_TM = 64;         // rows per tile
constexpr int LB_RC = 32;         // rows per weight-gradient tensor-core sum

template <int K, int KD>
struct LbLayout {
  static constexpr int STAGES = KD == 80 ? 2 : 3;                   // (80, 80): the ring gives way to the X stages
  static constexpr uint32_t W_HALF = KD * LB_H * 4;                 // W4^T slice, one of hi / lo
  static constexpr uint32_t W_SBO = (LB_H / 4) * 128;
  static constexpr uint32_t Y_BYTES = LB_TM * LB_H * 4;
  static constexpr uint32_t STAGE = Y_BYTES + LB_TM * K * 4;
  static constexpr uint32_t XT_HALF = K * LB_RC * 4;                // transposed X chunk, one of hi / lo
  static constexpr uint32_t XT_SBO = (LB_RC / 4) * 128;
  static constexpr int PLD = KD + 8;                                // padded partial row: conflict-free float2 stores
  static constexpr uint32_t P_BYTES = LB_TM * PLD * 4;
  static constexpr uint32_t OFF_STAGE = 2 * W_HALF;
  static constexpr uint32_t OFF_XT = OFF_STAGE + STAGES * STAGE;
  static constexpr uint32_t OFF_P = OFF_XT + 4 * XT_HALF;           // two 32-row X chunks, hi / lo
  static constexpr uint32_t OFF_BAR = OFF_P + 2 * P_BYTES;
  static constexpr uint32_t SMEM = OFF_BAR + STAGES * 8;
};

struct LbArgs {
  const float* dY;
  long long pz;
  const float* X;      // [N, K], row stride K
  const float* W4t;    // [>= Kd, ldw]: W4^T
  int ldw;
  float* dW4;
  int ldw4;
  float* db4;
  float* dX;
  int ldxo;
  int N, tiles_per_cluster;
  // BatchNorm-backward reduction (see the top): bn_sums != null turns it on
  const float* bn_x;                  // [N, H]: the BatchNorm input
  const float *bn_mean, *bn_rstd;
  float relu_scale;
  const long long* live;              // rows >= live[0] are left out (null: all N)
  double* bn_sums;                    // [2H] += sum dz | sum dz*xhat
  int l2;   // the step engine's chain (PdlChain, common.cuh): L2 hints, and dY is discarded once staged (see the loop)
};

template <int K, int KD>
__global__ void __launch_bounds__(LB_THREADS, 1) k_linear_bwd_planes(LbArgs g) {
  using Lay = LbLayout<K, KD>;
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Lay::OFF_BAR);
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warp-uniform as far as the compiler can tell
  const int w = (tid >> 5) & 3, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  const uint32_t rank = cluster_rank();
  const int ntiles = (g.N + LB_TM - 1) / LB_TM;
  const int t0 = (blockIdx.x >> 2) * g.tiles_per_cluster;
  const int nt = max(0, min(ntiles, t0 + g.tiles_per_cluster) - t0);
  const float* Yp = g.dY + (size_t)rank * g.pz;

  auto issue = [&](int i) {   // tile t0 + i -> stage i % Lay::STAGES
    const int row0 = (t0 + i) * LB_TM, rows = min(LB_TM, g.N - row0);
    unsigned char* st = smem + Lay::OFF_STAGE + (i % Lay::STAGES) * Lay::STAGE;
    uint64_t* bar = &full[i % Lay::STAGES];
    mbar_arrive_tx(bar, (uint32_t)rows * (LB_H + K) * 4);
    // dY: its last read.  X (and bn_x below): streamed as well, although with the BatchNorm sums the next kernel, the
    // target pass of the conv before, reads X and bn_x again as y and x.  Keeping those 26 MB (evict_last) or leaving
    // them at the default policy measured no faster at cfg2 (DESIGN section 7), and L2 then holds dX and the backward
    // planes this kernel reads instead.
    const uint64_t pol = l2_stream(g.l2);
    bulk_g2s_hint(st, Yp + (size_t)row0 * LB_H, (uint32_t)rows * LB_H * 4, bar, pol);
    bulk_g2s_hint(st + Lay::Y_BYTES, g.X + (size_t)row0 * K, (uint32_t)rows * K * 4, bar, pol);
  };
  if (tid == 0) {
    for (int s = 0; s < Lay::STAGES; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  // Set-up before pdl_wait (common.cuh): W4^T comes from the parameter pack.  dY is the conv backward's output, so the
  // ring is filled after the wait.
  // W4^T slice [KD, H] of this plane -> shared memory, split hi / lo, K permuted as in k_gemm_nt_wg (nt_logical_k)
  for (int i = tid; i < KD * LB_H; i += LB_THREADS) {
    const int n = i / LB_H, p = i - n * LB_H;
    const float v = __ldg(g.W4t + (size_t)n * g.ldw + rank * LB_H + p);
    const int L = nt_logical_k(p, LB_H);
    const uint32_t off = (uint32_t)(n >> 3) * Lay::W_SBO + (n & 7) * 16 + (L >> 2) * 128 + (L & 3) * 4;
    const uint32_t h = tf32_hi(v);
    *reinterpret_cast<uint32_t*>(smem + off) = h;
    *reinterpret_cast<uint32_t*>(smem + Lay::W_HALF + off) = tf32_lo(v, h);
  }
  pdl_wait();
  pdl_trigger();
  if (tid == 0)
    for (int i = 0; i < Lay::STAGES && i < nt; ++i) issue(i);
  fence_async_smem();
  __syncthreads();

  const uint32_t s0 = smem_u32(smem);
  const int mb = w * 16 + 2 * gq;   // weight gradient: plane columns of fragment rows g / g + 8
  float part[K / 2];
#pragma unroll
  for (int j = 0; j < K / 2; ++j) part[j] = 0.f;
  float cs0 = 0.f, cs1 = 0.f;
  // BatchNorm-backward reduction (K = KD = H only): this thread always handles column group tid % 16 of its rows
  const bool bn = K == LB_H && KD == LB_H && g.bn_sums != nullptr;
  float4 bs1 = f4zero(), bs2 = f4zero(), bmu = f4zero(), brs = f4zero();
  int n_live = 0;
  if (bn && wg == 0) {
    bmu = ldg4(g.bn_mean + (tid & 15) * 4);
    brs = ldg4(g.bn_rstd + (tid & 15) * 4);
    n_live = g.live ? (int)min((long long)g.N, *g.live) : g.N;
  }
  // BatchNorm: the y (X) and x rows this thread reduces for tile i, requested one data gradient ahead of reduce(i)
  // (the rows of thread tid: 16 rank + tid / 16 + 8 j, column group tid % 16)
  float4 by[2], bx[2];
  auto bn_fetch = [&](int i) {
    const int row0 = (t0 + i) * LB_TM;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = row0 + 16 * (int)rank + (tid >> 4) + 8 * j;
      const uint64_t pol = l2_stream(g.l2);
      by[j] = n < n_live ? ldg4_hint(g.X + (size_t)n * K + (tid & 15) * 4, pol) : f4zero();
      bx[j] = n < n_live ? ldg4_hint(g.bn_x + (size_t)n * LB_H + (tid & 15) * 4, pol) : f4zero();
    }
  };
  // dX rows 16 rank .. 16 rank + 15 of tile i = q + k + v + skip partials (warpgroup 0).  The slot of tile i is written
  // before the cluster barrier of tile i, read after it and before the barrier of tile i + 1, and rewritten for tile
  // i + 2 only after that barrier.
  auto reduce = [&](int i) {
    constexpr int V = KD / 4;
    const int row0 = (t0 + i) * LB_TM, rows = min(LB_TM, g.N - row0);
    const float* P = reinterpret_cast<const float*>(smem + Lay::OFF_P + (i & 1) * Lay::P_BYTES);
    auto one = [&](int e, float4 y, float4 x) {
      const int r = 16 * (int)rank + e / V, c4 = e - (e / V) * V;
      if (r >= rows) return;
      const uint32_t a = smem_u32(P + r * Lay::PLD + c4 * 4);
      float4 acc = ld_cluster4(map_rank(a, 0));
      acc = f4add(acc, ld_cluster4(map_rank(a, 1)));
      acc = f4add(acc, ld_cluster4(map_rank(a, 2)));
      acc = f4add(acc, ld_cluster4(map_rank(a, 3)));
      // with the BatchNorm sums the target pass reads dX next and demotes it; else (dX0, which the embedding
      // backward reads, or the eval backward) the default policy
      st4_hint(g.dX + (size_t)(row0 + r) * g.ldxo + c4 * 4, acc, l2_keep(g.l2 && g.bn_sums));
      if (bn && row0 + r < n_live) bn_bwd_acc4(bs1, bs2, bn_bwd_dz4(acc, y, g.relu_scale), x, bmu, brs);
    };
    if constexpr (K == LB_H && KD == LB_H) {   // 16 V = 256: the two rows of bn_fetch
#pragma unroll
      for (int j = 0; j < 2; ++j) one(tid + 128 * j, by[j], bx[j]);
    } else {
      for (int e = tid; e < 16 * V; e += 128) one(e, f4zero(), f4zero());
    }
  };

  for (int i = 0; i < nt; ++i) {
    const int row0 = (t0 + i) * LB_TM, rows = min(LB_TM, g.N - row0);
    const uint32_t so = Lay::OFF_STAGE + (i % Lay::STAGES) * Lay::STAGE;
    const float* sY = reinterpret_cast<const float*>(smem + so);
    const float* sX = reinterpret_cast<const float*>(smem + so + Lay::Y_BYTES);
    float* P = reinterpret_cast<float*>(smem + Lay::OFF_P + (i & 1) * Lay::P_BYTES);
    mbar_wait(&full[i % Lay::STAGES], (i / Lay::STAGES) & 1);
    // The tile's dY block (this CTA's plane) is in shared memory and nothing reads it from global memory again in the
    // step: drop its lines from L2 without a write-back, one 128-byte line per thread of warpgroup 0.
    if (g.l2 && wg == 0 && tid * 128 < rows * LB_H * 4) discard_l2(Yp + (size_t)row0 * LB_H + tid * 32);
    if (wg == 0) {
      // ---- data gradient of this plane: [64, H] . [H, KD]; rows past the end are computed and not stored
      const int r0 = w * 16 + gq, r1 = r0 + 8;
      if (bn && i > 0) bn_fetch(i - 1);   // in flight during this tile's data gradient
      uint32_t ah[LB_H / 8][4], al[LB_H / 8][4];
#pragma unroll
      for (int q = 0; q < LB_H / 16; ++q) {
        const float4 v0 = ld4(sY + r0 * LB_H + q * 16 + tq * 4), v1 = ld4(sY + r1 * LB_H + q * 16 + tq * 4);
        split4({v0.x, v1.x, v0.y, v1.y}, ah[2 * q], al[2 * q]);
        split4({v0.z, v1.z, v0.w, v1.w}, ah[2 * q + 1], al[2 * q + 1]);
      }
      float d[KD / 2];
#pragma unroll
      for (int j = 0; j < KD / 2; ++j) d[j] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < LB_H / 8; ++k)
        mma_step_wide<KD>(d, ah[k], al[k], s0 + k * 256, s0 + Lay::W_HALF + k * 256, Lay::W_SBO);
      wgmma_commit();
      wgmma_wait0();
#pragma unroll
      for (int j = 0; j < KD / 2; j += 2) {
        const int col = (j / 16) * 32 + acc_col(j & 15, tq);
        const int row = (j & 2) ? r1 : r0;
        *reinterpret_cast<float2*>(P + row * Lay::PLD + col) = make_float2(d[j], d[j + 1]);
      }
      if (i > 0) reduce(i - 1);
      // partials of tile i complete in all four CTAs; every thread of this CTA is done with stage i % STAGES
      cluster_sync();
      if (tid == 0 && i + Lay::STAGES < nt) issue(i + Lay::STAGES);
    } else {
      // ---- weight and bias gradient of this plane: [H, 64 rows] . [64 rows, K], in two 32-row sums.  X chunk c goes
      // to its own K-major stage; both were last read by the wgmmas of the previous tile, complete before its cluster
      // barrier.
      unsigned char* xt = smem + Lay::OFF_XT;
      // X rows 32c.. -> B operand (hi / lo), rows past the end as zeros.  A thread takes column n of four adjacent
      // rows 4q..4q+3, which is one 16-byte row of a core matrix: adjacent lanes read adjacent columns and write
      // adjacent core-matrix rows, both free of bank conflicts.
      auto stage_x = [&](int c) {
#pragma unroll
        for (int j = 0; j < K / 16; ++j) {
          const int idx = (tid - 128) + 128 * j, q = idx / K, n = idx - q * K, r = c * LB_RC + 4 * q;
          float v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) v[u] = r + u < rows ? sX[(r + u) * K + n] : 0.f;
          uint4 h, l;
          h.x = tf32_hi(v[0]), h.y = tf32_hi(v[1]), h.z = tf32_hi(v[2]), h.w = tf32_hi(v[3]);
          l.x = tf32_lo(v[0], h.x), l.y = tf32_lo(v[1], h.y), l.z = tf32_lo(v[2], h.z), l.w = tf32_lo(v[3], h.w);
          const uint32_t off = (uint32_t)(n >> 3) * Lay::XT_SBO + (n & 7) * 16 + q * 128;
          *reinterpret_cast<uint4*>(xt + c * 2 * Lay::XT_HALF + off) = h;
          *reinterpret_cast<uint4*>(xt + c * 2 * Lay::XT_HALF + Lay::XT_HALF + off) = l;
        }
        fence_async_smem();
        bar_sync(1, 128);
      };
      float d[K / 2];
      auto mma_chunk = [&](int c) {   // A = dY^T rows 32c.. (rows past the end as zeros); column sums on the way
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int ra = c * LB_RC + s * 8 + tq, rb = ra + 4;
          const float2 u0 = ra < rows ? *reinterpret_cast<const float2*>(sY + ra * LB_H + mb) : make_float2(0.f, 0.f);
          const float2 u1 = rb < rows ? *reinterpret_cast<const float2*>(sY + rb * LB_H + mb) : make_float2(0.f, 0.f);
          split4({u0.x, u0.y, u1.x, u1.y}, ah[s], al[s]);
          cs0 += u0.x + u1.x;
          cs1 += u0.y + u1.y;
        }
#pragma unroll
        for (int j = 0; j < K / 2; ++j) d[j] = 0.f;
        const uint32_t xhi = smem_u32(xt + c * 2 * Lay::XT_HALF), xlo = xhi + Lay::XT_HALF;
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 4; ++s) mma_step_wide<K>(d, ah[s], al[s], xhi + s * 256, xlo + s * 256, Lay::XT_SBO);
        wgmma_commit();
      };
      stage_x(0);
      mma_chunk(0);
      stage_x(1);                      // while chunk 0 is multiplied
      wgmma_wait0();
#pragma unroll
      for (int j = 0; j < K / 2; ++j) part[j] += d[j];
      mma_chunk(1);
      wgmma_wait0();
#pragma unroll
      for (int j = 0; j < K / 2; ++j) part[j] += d[j];
      // This warpgroup only has to tell the cluster that it is done with stage i % STAGES; it does not wait for the
      // barrier of tile i (the wait of tile i - 1 only keeps arrive / wait alternating) and goes on with tile i + 1.
      if (i > 0) cluster_wait();
      cluster_arrive();
    }
  }
  if (wg == 1 && nt > 0) cluster_wait();
  if (wg == 0 && nt > 0) {
    if (bn) bn_fetch(nt - 1);
    reduce(nt - 1);
  }
  cluster_sync();   // no CTA exits while another may still read its partials
  if (bn && wg == 0 && nt > 0) {
    // the 8 threads of a column group (lanes l, l + 16 of the four warps) -> one fp64 atomic per column.  The partial
    // slots are free: no CTA of the cluster reads them after the barrier above.
    float* red = reinterpret_cast<float*>(smem + Lay::OFF_P);   // [4 warps][2H]
    float v[8] = {bs1.x, bs1.y, bs1.z, bs1.w, bs2.x, bs2.y, bs2.z, bs2.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], 16);
    if (lane < 16) {
      st4(red + w * 2 * LB_H + lane * 4, make_float4(v[0], v[1], v[2], v[3]));
      st4(red + w * 2 * LB_H + LB_H + lane * 4, make_float4(v[4], v[5], v[6], v[7]));
    }
    bar_sync(2, 128);
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) t += (double)red[k * 2 * LB_H + tid];
    atomicAdd(g.bn_sums + tid, t);
  }
  if (wg == 1 && nt > 0) {
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 1);
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 2);
    cs1 += __shfl_xor_sync(0xffffffffu, cs1, 1);
    cs1 += __shfl_xor_sync(0xffffffffu, cs1, 2);
    const int m = (int)rank * LB_H + mb;
    if (tq == 0) {
      atomicAdd(g.db4 + m, cs0);
      atomicAdd(g.db4 + m + 1, cs1);
    }
#pragma unroll
    for (int j = 0; j < K / 2; j += 2) {
      const int col = (j / 16) * 32 + acc_col(j & 15, tq);
      atomicAdd(reinterpret_cast<float2*>(g.dW4 + (size_t)(m + ((j & 2) ? 1 : 0)) * g.ldw4 + col),
                make_float2(part[j], part[j + 1]));
    }
  }
}

bool fused_enabled() {   // PERT_LINEAR_BWD_FUSED=0: the two-kernel path (A/B); the kernel is tensor-core only
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("PERT_LINEAR_BWD_FUSED");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on == 1 && pert_gemm_tc_enabled();
}

bool shape_ok(long long N, int H, int K, int Kd) {
  return fused_enabled() && H == LB_H && (K == 64 || K == 80) && (Kd == 64 || Kd == K) && N >= 4096 &&
         N <= 0x7fffffffLL - LB_TM;
}

template <int K, int KD>
cudaLaunchConfig_t cluster_config(cudaLaunchAttribute* attr, cudaStream_t st) {
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 4;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(LB_THREADS);
  cfg.dynamicSmemBytes = LbLayout<K, KD>::SMEM;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

// Clusters of 4 CTAs of k_linear_bwd_planes<K, KD> that the current device holds at once, queried once per device;
// <= 0: none can be placed (or there is no device).
template <int K, int KD>
int clusters_that_fit() {
  static_assert(LbLayout<K, KD>::SMEM <= 227 * 1024, "shared memory");
  static int clusters[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    (void)cudaGetLastError();
    return 0;
  }
  if (clusters[dev] == 0) {
    auto kern = k_linear_bwd_planes<K, KD>;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = cluster_config<K, KD>(attr, nullptr);
    cfg.gridDim = dim3(4 * PERT_NUM_SMS);
    int n = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.dynamicSmemBytes) !=
            cudaSuccess ||
        cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
      (void)cudaGetLastError();
      n = -1;
    }
    clusters[dev] = n > 0 ? n : -1;
  }
  return clusters[dev];
}

int clusters_for(int K, int Kd) {
  if (K == 64) return clusters_that_fit<64, 64>();
  return Kd == 64 ? clusters_that_fit<80, 64>() : clusters_that_fit<80, 80>();
}

template <int K, int KD>
int launch(const LbArgs& a0, int clusters, cudaStream_t st) {
  LbArgs a = a0;
  a.l2 = pert_pdl_chain;
  const int ntiles = (a.N + LB_TM - 1) / LB_TM;
  a.tiles_per_cluster = (ntiles + clusters - 1) / clusters;
  const dim3 grid(4 * ((ntiles + a.tiles_per_cluster - 1) / a.tiles_per_cluster));
  const cudaError_t e =
      launch_pdl_cluster(4, k_linear_bwd_planes<K, KD>, grid, LB_THREADS, LbLayout<K, KD>::SMEM, st, a);
  return e == cudaSuccess ? PERT_OK : (int)e;
}

inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" {

int pert_linear_bwd_planes_supported(long long N, int H, int K, int Kd) {
  return shape_ok(N, H, K, Kd) && clusters_for(K, Kd) > 0 ? 1 : 0;
}

int pert_linear_bwd_planes(const float* dY, long long plane_stride, const float* X, int ldx, const float* W4t, int ldw,
                           float* dW4, int ldw4, float* db4, float* dX, int ldx_out, long long N, int H, int K, int Kd,
                           void* stream) {
  return pert_linear_bwd_planes_ex(dY, plane_stride, X, ldx, W4t, ldw, dW4, ldw4, db4, dX, ldx_out, N, H, K, Kd,
                                   nullptr, nullptr, nullptr, 1.f, nullptr, nullptr, stream);
}

int pert_linear_bwd_planes_ex(const float* dY, long long plane_stride, const float* X, int ldx, const float* W4t,
                              int ldw, float* dW4, int ldw4, float* db4, float* dX, int ldx_out, long long N, int H,
                              int K, int Kd, const float* bn_x, const float* bn_mean, const float* bn_rstd,
                              float relu_scale, const long long* live, double* bn_sums, void* stream) {
  if (!dY || !X || !W4t || !dW4 || !db4 || !dX || N < 0 || H <= 0 || K <= 0 || Kd <= 0 || Kd > K || ldx < K ||
      ldw < 4 * H || ldw4 < K || ldx_out < Kd || plane_stride < N * H)
    return PERT_ERR_BADARG;
  if (bn_sums && (!bn_x || !bn_mean || !bn_rstd || K != H || Kd != K || !al16(bn_x) || !al16(bn_mean) ||
                  !al16(bn_rstd) || ((uintptr_t)bn_sums & 7)))
    return PERT_ERR_BADARG;
  if (!shape_ok(N, H, K, Kd)) return PERT_ERR_UNSUPPORTED;
  // bulk copies of whole tiles (contiguous X rows, 16-byte aligned blocks), 16-byte dX stores, 8-byte dW4 reductions
  if (ldx != K || plane_stride % 4 || ldx_out % 4 || ldw4 % 2 || !al16(dY) || !al16(X) || !al16(dX) ||
      ((uintptr_t)dW4 & 7))
    return PERT_ERR_UNSUPPORTED;
  const int clusters = clusters_for(K, Kd);
  if (clusters <= 0) return PERT_ERR_UNSUPPORTED;   // a cluster of 4 such CTAs cannot be placed
  LbArgs a{dY, plane_stride, X, W4t, ldw, dW4, ldw4, db4, dX, ldx_out, (int)N, 0,
           bn_x, bn_mean, bn_rstd, relu_scale, live, bn_sums};
  cudaStream_t st = (cudaStream_t)stream;
  if (K == 64) return launch<64, 64>(a, clusters, st);
  if (Kd == 64) return launch<80, 64>(a, clusters, st);
  return launch<80, 80>(a, clusters, st);
}

}  // extern "C"
