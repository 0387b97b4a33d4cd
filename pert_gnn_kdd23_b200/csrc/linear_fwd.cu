// Forward of the plane-blocked node linear at H = 64 (q|k|v|skip = A . W4^T + b4, W4 [4H, K]) in ONE pass over A,
// optionally with the BatchNorm + ReLU (+ dropout) of the previous conv applied while A is loaded:
//   plain mode (conv 0):   A = x[0] [N, K]                                           planes[4][N][H] = A . W4^T + b4
//   BN mode (conv l >= 1): A = dropout(relu(bn(out[l-1]))), also written to x[l]     (K = H)
// The two-launch path (k_bn_apply, then k_gemm_nt_wg in two N blocks of 128) writes x[l] and reads it straight back,
// and reads it twice more, once per N block; here out[l-1] is read once, x[l] written once and the planes written once.
//
// Layout: persistent CTAs, one per SM, each owning the 64-row tiles blockIdx.x, blockIdx.x + gridDim.x, ...
//   - each tile (64 x K fp32, one contiguous 16 / 20 KB block) arrives by one bulk copy in a ring of STAGES stages
//     (one mbarrier each, completion counted in bytes).  Thread 0 fills the ring; after that, the warpgroup that has
//     read a stage (a 128-thread named barrier) refills it with tile i + STAGES at once, so no thread waits for a free
//     stage and the block stays at 256 threads (a separate producer warp would cap ptxas at 168 registers);
//   - the whole [4H, K] weight block is resident in shared memory, split hi / lo, K permuted as in k_gemm_nt_wg
//     (nt_logical_k), so A is read from HBM once;
//   - two consumer warpgroups take alternate tiles, so one warpgroup's epilogue overlaps the other's wgmmas.  A thread
//     reads its fragment rows' four contiguous columns of each 16-column chunk from the stage (one 16-byte load per
//     row and chunk), in BN mode applies the affine, the ReLU and the dropout (its float4 is exactly one Philox group)
//     and stores the float4 to x[l], then splits hi / lo and issues the chunk's m64n128k8 wgmmas (two N halves x
//     hi*hi, lo*hi, hi*lo x two K-steps).  The A registers are double-buffered over chunks: chunk q waits only for the
//     wgmmas of chunk q - 2, never for all of them, until the tile's epilogue;
//   - epilogue: bias from shared memory, sector-complete float2 stores into the four planes.
// BatchNorm semantics are those of k_bn_apply, through the same helpers (bn.cuh): mean / rstd from the fp64 sums (CTA 0
// stores them and updates the running statistics and num_batches_tracked) or, in eval mode, the arrays
// k_bn_eval_stats wrote; x[l] is bit-identical to pert_bn_fwd_ex's output.
// Accuracy: 3xTF32 (hi*hi + lo*hi + hi*lo, round-to-nearest split), one K-long tensor-core sum per output, as
// k_gemm_nt_wg.
#include "common.cuh"
#include "bn.cuh"
#include "sm90.cuh"

namespace {

constexpr int LF_THREADS = 256;                     // two warpgroups
constexpr int LF_H = 64;                            // plane width
constexpr int LF_NC = 4 * LF_H;                     // q | k | v | skip
constexpr int LF_TM = 64;                           // rows per tile
enum { LF_PLAIN = 0, LF_BN = 1, LF_BN_DROP = 2 };

template <int K>
struct LfLayout {
  // Even, so that the tiles of one stage (i, i + STAGES, ...) all belong to one warpgroup, which waits for each of
  // its phases in turn: a warpgroup that waited for a stage's next phase while an earlier one was still pending
  // would see that parity as complete and read a stale tile.  (K = 80: 3 stages do not fit beside the weights.)
  static constexpr int STAGES = K == 64 ? 4 : 2;
  static constexpr uint32_t W_HALF = LF_NC * K * 4;               // W4, one of hi / lo
  static constexpr uint32_t W_SBO = (K / 4) * 128;
  static constexpr uint32_t STAGE = LF_TM * K * 4;
  static constexpr uint32_t OFF_STAGE = 2 * W_HALF;
  static constexpr uint32_t OFF_PAR = OFF_STAGE + STAGES * STAGE;  // bias [4H] | mean | rstd | gamma | beta [H]
  static constexpr uint32_t OFF_BAR = OFF_PAR + (LF_NC + 4 * LF_H) * 4;
  static constexpr uint32_t SMEM = OFF_BAR + STAGES * 8;
  static_assert(STAGES % 2 == 0, "one warpgroup per stage");
};

struct LfArgs {
  const float* A;      // [N, K], row stride K
  const float* W4;     // [4H, K] (ldw)
  int ldw;
  const float* b4;     // [4H]
  float* planes;       // 4 planes [N, H] (row stride H, plane stride pz)
  long long pz;
  // BN mode
  float* x_out;        // [N, H]: the BatchNorm output, the conv's input
  const double* acc;   // training: fp64 column sums | sums of squares; NULL: eval (mean / rstd are read)
  float *mean, *rstd;
  const float *gamma, *beta;
  float eps, momentum;
  float *running_mean, *running_var;
  long long* num_batches_tracked;
  BnDropout drop;
  const long long* live;   // training on a padded batch: {N, B} of the real part (statistics over live[0] rows)
  int N;
  int l2;              // the step engine's chain (PdlChain, common.cuh): L2 hints, see the epilogue
};

template <int K, int MODE>
__global__ void __launch_bounds__(LF_THREADS, 1) k_bn_linear_fwd_planes(LfArgs g) {
  using Lay = LfLayout<K>;
  constexpr bool BN = MODE != LF_PLAIN, DROP = MODE == LF_BN_DROP;
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Lay::OFF_BAR);
  float* par = reinterpret_cast<float*>(smem + Lay::OFF_PAR);
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warp-uniform as far as the compiler can tell
  const int ntiles = (g.N + LF_TM - 1) / LF_TM;
  const int nt = ((int)blockIdx.x < ntiles) ? (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  auto issue = [&](int i) {   // tile i of this CTA -> stage i % STAGES
    const int s = i % Lay::STAGES;
    const int row0 = ((int)blockIdx.x + i * (int)gridDim.x) * LF_TM, rows = min(LF_TM, g.N - row0);
    mbar_arrive_tx(&full[s], (uint32_t)rows * K * 4);
    bulk_g2s_hint(smem + Lay::OFF_STAGE + s * Lay::STAGE, g.A + (size_t)row0 * K, (uint32_t)rows * K * 4, &full[s],
                  l2_stream(g.l2));   // out[l - 1] (x[0]): last read in the forward
  };
  if (tid == 0) {
    for (int s = 0; s < Lay::STAGES; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  // Set-up before pdl_wait (common.cuh): W4 / b4 come from the parameter pack and gamma / beta from the parameters, none
  // of them written by the preceding conv.  A and the BatchNorm sums are its output and are read after the wait.
  // W4 [4H, K] -> shared memory, split hi / lo, K permuted (nt_logical_k).  K loads per thread, issued 16 at a time
  // before any is used: one at a time, the L2 latency of each would add up to most of the kernel's time.
  constexpr int WB = 16;
  static_assert(LF_NC * K % (LF_THREADS * WB) == 0, "weight batches");
  for (int j0 = 0; j0 < LF_NC * K / LF_THREADS; j0 += WB) {
    float v[WB];
#pragma unroll
    for (int u = 0; u < WB; ++u) {
      const int i = tid + (j0 + u) * LF_THREADS, n = i / K, p = i - n * K;
      v[u] = __ldg(g.W4 + (size_t)n * g.ldw + p);
    }
#pragma unroll
    for (int u = 0; u < WB; ++u) {
      const int i = tid + (j0 + u) * LF_THREADS, n = i / K, p = i - n * K;
      const int L = nt_logical_k(p, K);
      const uint32_t off = (uint32_t)(n >> 3) * Lay::W_SBO + (n & 7) * 16 + (L >> 2) * 128 + (L & 3) * 4;
      const uint32_t h = tf32_hi(v[u]);
      *reinterpret_cast<uint32_t*>(smem + off) = h;
      *reinterpret_cast<uint32_t*>(smem + Lay::W_HALF + off) = tf32_lo(v[u], h);
    }
  }
  for (int c = tid; c < LF_NC; c += LF_THREADS) par[c] = __ldg(g.b4 + c);
  if (BN)
    for (int c = tid; c < LF_H; c += LF_THREADS) {
      par[LF_NC + 2 * LF_H + c] = g.gamma[c];
      par[LF_NC + 3 * LF_H + c] = g.beta[c];
    }
  pdl_wait();
  pdl_trigger();
  if (tid == 0)
    for (int i = 0; i < Lay::STAGES && i < nt; ++i) issue(i);
  if (BN)
    for (int c = tid; c < LF_H; c += LF_THREADS) {
      float mu, rs;
      if (g.acc) {
        const long long n_stat = g.live ? g.live[0] : g.N;   // read here only, never in the tile loop
        bn_batch_stats(g.acc, n_stat, LF_H, c, g.eps, g.momentum, blockIdx.x == 0, g.mean, g.rstd, g.running_mean,
                       g.running_var, g.num_batches_tracked, mu, rs);
      } else {
        mu = g.mean[c];
        rs = g.rstd[c];
      }
      par[LF_NC + c] = mu;
      par[LF_NC + LF_H + c] = rs;
    }
  fence_async_smem();   // generic-proxy weight stores -> visible to the wgmmas
  __syncthreads();

  // ---- warpgroup wg takes the CTA's tiles wg, wg + 2, ...
  const int w = (tid >> 5) & 3, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  const int r0 = w * 16 + gq, r1 = r0 + 8;   // fragment rows inside the tile
  const uint32_t bhi = smem_u32(smem), blo = bhi + Lay::W_HALF;
  BnDropKey key{};
  if (DROP) key = bn_drop_key(g.drop);
  for (int i = wg; i < nt; i += 2) {
    const int s = i % Lay::STAGES;
    const int row0 = ((int)blockIdx.x + i * (int)gridDim.x) * LF_TM, rows = min(LF_TM, g.N - row0);
    const float* sA = reinterpret_cast<const float*>(smem + Lay::OFF_STAGE + s * Lay::STAGE);
    mbar_wait(&full[s], (i / Lay::STAGES) & 1);
    float d[LF_NC / 2];   // the first wgmma of each N half overwrites it
    uint32_t ah[2][2][4], al[2][2][4];   // [chunk parity][K-step of the chunk]
#pragma unroll
    for (int q = 0; q < K / 16; ++q) {
      if (q >= 2) wgmma_wait1();       // chunk q - 2, the last reader of this register set, is complete
      const int c = q * 16 + tq * 4;
      float4 v0 = ld4(sA + r0 * K + c), v1 = ld4(sA + r1 * K + c);
      if (BN) {
        const float* P = par + LF_NC;
        const float4 mu = ld4(P + c), rs = ld4(P + LF_H + c), ga = ld4(P + 2 * LF_H + c), be = ld4(P + 3 * LF_H + c);
        v0 = bn_affine4(v0, mu, rs, ga, be, true);
        v1 = bn_affine4(v1, mu, rs, ga, be, true);
        if (DROP) {   // float4 group = row * (H/4) + col/4
          v0 = bn_dropout4(v0, (uint32_t)(row0 + r0) * (LF_H / 4) + (uint32_t)(c >> 2), g.drop, key);
          v1 = bn_dropout4(v1, (uint32_t)(row0 + r1) * (LF_H / 4) + (uint32_t)(c >> 2), g.drop, key);
        }
        const uint64_t pol = l2_stream(g.l2);   // x[l]: next read by the backward
        if (r0 < rows) st4_hint(g.x_out + (size_t)(row0 + r0) * LF_H + c, v0, pol);
        if (r1 < rows) st4_hint(g.x_out + (size_t)(row0 + r1) * LF_H + c, v1, pol);
      }
      split4({v0.x, v1.x, v0.y, v1.y}, ah[q & 1][0], al[q & 1][0]);   // K-step 2q:     columns 4t, 4t+1
      split4({v0.z, v1.z, v0.w, v1.w}, ah[q & 1][1], al[q & 1][1]);   // K-step 2q + 1: columns 4t+2, 4t+3
      if (q == K / 16 - 1) {
        // The warpgroup's last read of the stage: refill it.  The refill comes after the loaded values were used (a
        // barrier alone does not wait for loads in flight) and after a proxy fence, so the bulk copy (async proxy)
        // cannot overtake a shared-memory read of this tile.
        fence_async_smem();
        bar_sync(1 + wg, 128);
        if ((tid & 127) == 0 && i + Lay::STAGES < nt) issue(i + Lay::STAGES);
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int nh = 0; nh < 2; ++nh) {
          const uint32_t o = (2 * q + ks) * 256 + nh * 16 * Lay::W_SBO;
          const uint64_t dh = make_desc(bhi + o, 128, Lay::W_SBO), dl = make_desc(blo + o, 128, Lay::W_SBO);
          wgmma_n128(d + 64 * nh, ah[q & 1][ks], dh, q + ks > 0);
          wgmma_n128(d + 64 * nh, al[q & 1][ks], dh);
          wgmma_n128(d + 64 * nh, ah[q & 1][ks], dl);
        }
      wgmma_commit();
    }
    wgmma_wait0();
    // ---- epilogue: + bias, two adjacent columns per store (four lanes cover one 32-byte sector of a row).  In the
    // chain the k and v planes are kept in L2: the conv forward copies their tiles before it computes anything, while
    // it reads the q and skip rows one node at a time.  All four (52 MB at cfg2) would not fit the 50 MB L2.
    const uint64_t keep = l2_keep(g.l2), norm = l2_evict_normal();
#pragma unroll
    for (int j = 0; j < LF_NC / 2; j += 2) {
      const int col = (j / 16) * 32 + acc_col(j & 15, tq);
      const int r = (j & 2) ? r1 : r0;
      if (r >= rows) continue;
      const float2 b = *reinterpret_cast<const float2*>(par + col);
      const int plane = col >> 6;
      st2_hint(g.planes + (size_t)plane * g.pz + (size_t)(row0 + r) * LF_H + (col & 63),
               make_float2(d[j] + b.x, d[j + 1] + b.y), plane == 1 || plane == 2 ? keep : norm);
    }
  }
}

bool shape_ok(long long N, int H, int K) {
  return pert_gemm_tc_enabled() && H == LF_H && (K == 64 || K == 80) && N >= 4096 && N <= 0x7fffffffLL - LF_TM;
}

// CTAs of k_bn_linear_fwd_planes<K, MODE> one SM holds (the shared-memory attribute is set on the way), queried once
// per device; <= 0: the kernel cannot be placed (or there is no device).
template <int K, int MODE>
int ctas_per_sm() {
  static_assert(LfLayout<K>::SMEM <= 227 * 1024, "shared memory");
  static int per_sm[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    (void)cudaGetLastError();
    return 0;
  }
  if (per_sm[dev] == 0) {
    auto kern = k_bn_linear_fwd_planes<K, MODE>;
    int n = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LfLayout<K>::SMEM) !=
            cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, LF_THREADS, LfLayout<K>::SMEM) != cudaSuccess) {
      (void)cudaGetLastError();
      n = -1;
    }
    per_sm[dev] = n > 0 ? n : -1;
  }
  return per_sm[dev];
}

template <int K, int MODE>
int launch(const LfArgs& a, cudaStream_t st) {
  const int per_sm = ctas_per_sm<K, MODE>();
  if (per_sm <= 0) return PERT_ERR_UNSUPPORTED;
  const int ntiles = (a.N + LF_TM - 1) / LF_TM;
  const int grid = min(ntiles, PERT_NUM_SMS * per_sm);
  LfArgs b = a;
  b.l2 = pert_pdl_chain;
  const cudaError_t e = launch_pdl(k_bn_linear_fwd_planes<K, MODE>, grid, LF_THREADS, LfLayout<K>::SMEM, st, b);
  return e == cudaSuccess ? PERT_OK : (int)e;
}

inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" {

int pert_bn_linear_fwd_planes_supported(long long N, int H, int K) {
  if (!shape_ok(N, H, K)) return 0;
  return (K == 64 ? ctas_per_sm<64, LF_PLAIN>() : ctas_per_sm<80, LF_PLAIN>()) > 0 ? 1 : 0;
}

int pert_bn_linear_fwd_planes(const float* A, int lda, int bn, const float* gamma, const float* beta,
                              float* running_mean, float* running_var, long long* num_batches_tracked, float eps,
                              float momentum, int training, float* mean, float* rstd, float* x_out, int ld_x_out,
                              void* workspace, long long workspace_bytes, int stats_ready, float dropout,
                              const long long* drop_ctr, int drop_layer, const float* W4, int ldw, const float* b4,
                              float* planes, long long plane_stride, long long N, int H, int K, void* stream) {
  return pert_bn_linear_fwd_planes_ex(A, lda, bn, gamma, beta, running_mean, running_var, num_batches_tracked, eps,
                                      momentum, training, mean, rstd, x_out, ld_x_out, workspace, workspace_bytes,
                                      stats_ready, dropout, drop_ctr, drop_layer, nullptr, W4, ldw, b4, planes,
                                      plane_stride, N, H, K, stream);
}

}  // extern "C"

int pert_bn_linear_fwd_planes_ex(const float* A, int lda, int bn, const float* gamma, const float* beta,
                                 float* running_mean, float* running_var, long long* num_batches_tracked, float eps,
                                 float momentum, int training, float* mean, float* rstd, float* x_out, int ld_x_out,
                                 void* workspace, long long workspace_bytes, int stats_ready, float dropout,
                                 const long long* drop_ctr, int drop_layer, const long long* live, const float* W4,
                                 int ldw, const float* b4, float* planes, long long plane_stride, long long N, int H,
                                 int K, void* stream) {
  if (!A || !W4 || !b4 || !planes || N < 0 || H <= 0 || K <= 0 || lda < K || ldw < K || plane_stride < N * H)
    return PERT_ERR_BADARG;
  const bool drop = bn && training && dropout > 0.f;
  if (bn) {
    if (!gamma || !beta || !mean || !rstd || !x_out || ld_x_out < K) return PERT_ERR_BADARG;
    if (!al16(gamma) || !al16(beta) || !al16(mean) || !al16(rstd)) return PERT_ERR_BADARG;
    if (!(dropout >= 0.f && dropout <= 1.f)) return PERT_ERR_BADARG;
    if (drop && (!drop_ctr || N * (H / 4) >= (1LL << 32))) return PERT_ERR_BADARG;
    if (training && (!workspace || workspace_bytes < pert_bn_workspace_bytes(N, H) || ((uintptr_t)workspace & 7)))
      return PERT_ERR_BADARG;
    if (!training && (!running_mean || !running_var)) return PERT_ERR_BADARG;
  }
  if (!shape_ok(N, H, K) || (bn && K != H)) return PERT_ERR_UNSUPPORTED;
  // one bulk copy per contiguous 64-row tile, 16-byte x[l] stores, 8-byte plane stores
  if (lda != K || (bn && ld_x_out != K) || plane_stride % 4 || !al16(A) || !al16(planes) || (bn && !al16(x_out)))
    return PERT_ERR_UNSUPPORTED;
  const int per_sm = K == 64 ? ctas_per_sm<64, LF_PLAIN>() : ctas_per_sm<80, LF_PLAIN>();
  if (per_sm <= 0) return PERT_ERR_UNSUPPORTED;   // nothing launched yet
  cudaStream_t st = (cudaStream_t)stream;
  LfArgs a{};
  a.A = A;
  a.W4 = W4;
  a.ldw = ldw;
  a.b4 = b4;
  a.planes = planes;
  a.pz = plane_stride;
  a.N = (int)N;
  if (!bn) return K == 64 ? launch<64, LF_PLAIN>(a, st) : launch<80, LF_PLAIN>(a, st);
  if ((drop ? ctas_per_sm<64, LF_BN_DROP>() : ctas_per_sm<64, LF_BN>()) <= 0) return PERT_ERR_UNSUPPORTED;
  double* acc = nullptr;
  const int rc = pert_bn_fwd_stats(A, lda, running_mean, running_var, eps, training, mean, rstd, N, H, workspace,
                                   workspace_bytes, stats_ready, training ? live : nullptr, st, &acc);
  if (rc != PERT_OK) return rc;
  a.x_out = x_out;
  a.acc = acc;
  a.mean = mean;
  a.rstd = rstd;
  a.gamma = gamma;
  a.beta = beta;
  a.eps = eps;
  a.momentum = momentum;
  if (training) {
    a.running_mean = running_mean;
    a.running_var = running_var;
    a.num_batches_tracked = num_batches_tracked;
    a.live = live;
  }
  if (!drop) return launch<64, LF_BN>(a, st);
  a.drop = bn_dropout_params(dropout, drop_ctr, drop_layer);
  return launch<64, LF_BN_DROP>(a, st);
}
