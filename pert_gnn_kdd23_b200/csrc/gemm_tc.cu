// Tensor-core path of the dense node linears on Hopper: wgmma (m64nNk8, kind tf32) with 3xTF32 split accumulation.
//
// The linears need fp32-level accuracy (1e-4 after 3-5 layers + BatchNorm), which single-pass TF32 (10-bit
// mantissa) does not give.  Every fp32 operand x is split into hi = nearest tf32 of x and lo = x - hi (see tf32_hi);
// the product is accumulated in fp32 registers as  hi*hi + lo*hi + hi*lo  (the dropped lo*lo term is ~2^-22
// relative), three wgmmas per K-step (tests: test_linear_* at 2e-6).
//
// Operand staging:
//   A (activations / the transposed operand of the weight gradient): global -> registers in the wgmma A-fragment
//       layout -> split.  A thread of warp w holds rows 16w + g and 16w + g + 8 (g = lane / 4) and K columns t, t + 4
//       (t = lane % 4) of every K-step of 8.  The K order inside a step is free as long as B uses the same one, so the
//       forward kernel gives thread t the four CONTIGUOUS columns 4t..4t+3 of a 16-column chunk (one 16-byte load per
//       row and chunk: columns 4t, 4t+1 feed step 0, 4t+2, 4t+3 step 1) and permutes the weights to match
//       (nt_logical_k).  The weight-gradient kernel permutes M instead: fragment rows g / g + 8 are the adjacent
//       output rows 2g / 2g + 1, so a thread reads two of them with one 8-byte load.
//   B:  shared memory, no-swizzle K-major canonical layout (8-row x 16-byte core matrices, LBO = 128 B between
//       K-adjacent core matrices, SBO between N-adjacent ones), split hi/lo.
//   D:  fp32 accumulators in registers (fragment: row g / g + 8, columns 8j + 2t, 8j + 2t + 1).
//
//   k_gemm_nt_wg (forward / data gradient, C[M,Nc] = A[M,K] . B[Nc,K]^T (+bias)): persistent, two warpgroups per
//       CTA, each owns 64-row tiles; the [BN, K] weight block is resident in shared memory (hi + lo), the next
//       16-column A chunk is in flight while the current one is multiplied.
//   k_gemm_tn_wg (weight gradient, C[Mc,Nc] += A[R,Mc]^T . B[R,Nc], split over R, vector red.global accumulation):
//       two warpgroups cover 128 output rows; the CTA transposes 32-row chunks of B into a double-buffered K-major
//       stage while the previous chunk is multiplied.  The tensor-core accumulation truncates, an error that grows
//       with the length of the running sum, so every TN_FLUSH chunks the register accumulators are added (round to
//       nearest) into per-thread partial sums in shared memory and restarted from zero.
// These GEMMs are memory-bound by shape (K <= 256): A read once, C written once.
#include "common.cuh"
#include "sm90.cuh"
#include <stdlib.h>

namespace {

constexpr int WG_THREADS = 256;   // two warpgroups
constexpr int SMEM_MAX = 226 * 1024;

struct NtArgs {
  const float* A;
  int lda, a_cb;
  long long a_cbs;
  long long a_pz;      // plane stride of A (gridDim.z > 1: plane z multiplies A + z * a_pz by columns z*K.. of B)
  const float* B;
  int ldb;
  const float* bias;
  float* C;
  int ldc, c_cb;
  long long c_cbs;
  int M, Nc, K, relu;
  int reduce;          // 1: accumulate into C with vector red.global (planes), bias from plane 0 only
};

// grid: (persistent over 128-row tile pairs, Nc / BN, planes)
template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1) k_gemm_nt_wg(NtArgs g) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  const int K = g.K, Kp = (K + 7) & ~7, K16 = K & ~15;
  const int n0 = blockIdx.y * BN, kz = blockIdx.z;
  const uint32_t SBO = (uint32_t)(Kp / 4) * 128;
  unsigned char* sBhi = smem;
  unsigned char* sBlo = smem + (size_t)BN * Kp * 4;
  const float* Bp = g.B + (size_t)kz * K;
  const float* Ap = g.A + (size_t)kz * g.a_pz;

  // ---- weights [BN, K] -> shared memory once per CTA, split hi / lo, permuted K (nt_logical_k)
  for (int i = tid; i < BN * Kp; i += WG_THREADS) {
    const int n = i / Kp, p = i - n * Kp;
    const float v = p < K ? __ldg(Bp + (size_t)(n0 + n) * g.ldb + p) : 0.f;
    const int L = nt_logical_k(p, K16);
    const uint32_t off = (uint32_t)(n >> 3) * SBO + (n & 7) * 16 + (L >> 2) * 128 + (L & 3) * 4;
    const uint32_t h = tf32_hi(v);
    *reinterpret_cast<uint32_t*>(sBhi + off) = h;
    *reinterpret_cast<uint32_t*>(sBlo + off) = tf32_lo(v, h);
  }
  fence_async_smem();                                // generic-proxy smem writes -> visible to wgmma (async proxy)
  __syncthreads();

  const uint32_t bhi0 = smem_u32(sBhi), blo0 = smem_u32(sBlo);
  const int mtiles = (g.M + 63) / 64, nq = K16 / 16;
  const bool add_bias = g.bias && kz == 0;
  for (int mt = blockIdx.x * 2 + wg; mt < mtiles; mt += gridDim.x * 2) {
    const int r0 = mt * 64 + w * 16 + gq, r1 = r0 + 8;
    const bool ok0 = r0 < g.M, ok1 = r1 < g.M;
    float d[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
    auto load = [&](int q, float4& v0, float4& v1) {
      const int c = q * 16 + tq * 4;               // a 16-column chunk never straddles two column blocks
      const float* base = Ap + (size_t)(c / g.a_cb) * g.a_cbs + (c % g.a_cb);
      v0 = ok0 ? ldg4(base + (size_t)r0 * g.lda) : f4zero();
      v1 = ok1 ? ldg4(base + (size_t)r1 * g.lda) : f4zero();
    };
    float4 v0, v1;
    if (nq > 0) load(0, v0, v1);
    for (int q = 0; q < nq; ++q) {
      uint32_t ah0[4], al0[4], ah1[4], al1[4];
      split4({v0.x, v1.x, v0.y, v1.y}, ah0, al0);  // step 2q:     columns 4t, 4t+1 of rows g, g+8
      split4({v0.z, v1.z, v0.w, v1.w}, ah1, al1);  // step 2q + 1: columns 4t+2, 4t+3
      if (q + 1 < nq) load(q + 1, v0, v1);         // in flight while this chunk is multiplied
      wgmma_fence();
      mma_step<BN>(d, ah0, al0, bhi0 + (2 * q) * 256, blo0 + (2 * q) * 256, SBO);
      mma_step<BN>(d, ah1, al1, bhi0 + (2 * q + 1) * 256, blo0 + (2 * q + 1) * 256, SBO);
      wgmma_commit();
      wgmma_wait0();                               // the A registers are rewritten next iteration
    }
    if (K16 < K) {                                 // trailing K-step of 8
      const int c = K16 + tq * 2;
      const float* base = Ap + (size_t)(c / g.a_cb) * g.a_cbs + (c % g.a_cb);
      const float2 u0 = ok0 ? __ldg(reinterpret_cast<const float2*>(base + (size_t)r0 * g.lda)) : make_float2(0.f, 0.f);
      const float2 u1 = ok1 ? __ldg(reinterpret_cast<const float2*>(base + (size_t)r1 * g.lda)) : make_float2(0.f, 0.f);
      uint32_t ah[4], al[4];
      split4({u0.x, u1.x, u0.y, u1.y}, ah, al);
      wgmma_fence();
      mma_step<BN>(d, ah, al, bhi0 + (K16 / 8) * 256, blo0 + (K16 / 8) * 256, SBO);
      wgmma_commit();
      wgmma_wait0();
    }
    // ---- epilogue: registers (+bias, relu) -> global, two adjacent columns per store
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int col = n0 + (i / 16) * 32 + acc_col(i & 15, tq);
      const int row = (i & 2) ? r1 : r0;
      if (row >= g.M) continue;
      float2 o = make_float2(d[i], d[i + 1]);
      if (add_bias) {
        o.x += __ldg(g.bias + col);
        o.y += __ldg(g.bias + col + 1);
      }
      if (g.relu) o = make_float2(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f));
      float2* p = reinterpret_cast<float2*>(g.C + (size_t)(col / g.c_cb) * g.c_cbs + (col % g.c_cb) + (size_t)row * g.ldc);
      if (g.reduce) atomicAdd(p, o);
      else *p = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
constexpr int RC = 32;   // reduction rows (nodes) per chunk == K of one stage
constexpr int TN_FLUSH = 1;   // chunks per register partial sum of the weight gradient

struct TnArgs {
  const float* A;   // [R, Mc] blocked
  int lda, a_cb;
  long long a_cbs;
  const float* B;   // [R, Nc] plain
  int ldb;
  float* C;         // [Mc, Nc], ldc
  int ldc;
  float* colsum;    // optional [Mc]: += column sums of A (bias gradient)
  int R, Mc, Nc, rows_per_split;
};

// grid: (splits over R, Mc / 128).  NCP = Nc rounded up to 16 (<= 160)
template <int NCP>
__global__ void __launch_bounds__(WG_THREADS, 1) k_gemm_tn_wg(TnArgs g) {
  constexpr uint32_t SBO = (RC / 4) * 128;            // N-adjacent core-matrix groups of a stage
  constexpr uint32_t HALF = (uint32_t)NCP * RC * 4;   // one of hi / lo of one stage
  constexpr int NP = NCP / 8;                         // B items per thread: a warp item is 4 rows x 8 columns
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, tq = lane & 3;
  const int r_begin = blockIdx.x * g.rows_per_split;
  const int r_end = min(g.R, r_begin + g.rows_per_split);
  const int nch = (r_end - r_begin + RC - 1) / RC;
  // fragment rows g / g + 8 of this warp are output rows mb / mb + 1
  const int mb = blockIdx.y * 128 + wg * 64 + w * 16 + 2 * gq;
  const bool mok = mb < g.Mc;
  const float* acol = g.A + (size_t)((mok ? mb : 0) / g.a_cb) * g.a_cbs + ((mok ? mb : 0) % g.a_cb);
  const uint32_t s0 = smem_u32(smem);
  float* part = reinterpret_cast<float*>(smem + 4 * HALF);   // [NCP / 2][256]: this thread's partial sums
  bool parted = false;

  float2 av[4][2];                                    // [K-step][row t / t + 4] x (row mb, mb + 1)
  float bv[NP];
  auto load = [&](int c) {
    const int r0 = r_begin + c * RC;
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + s * 8 + tq + 4 * h;
        av[s][h] = (mok && r < r_end) ? __ldg(reinterpret_cast<const float2*>(acol + (size_t)r * g.lda))
                                      : make_float2(0.f, 0.f);
      }
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      const int it = warp + 8 * i, r = (it & 7) * 4 + (lane & 3), n = (it >> 3) * 8 + (lane >> 2);
      bv[i] = (r0 + r < r_end && n < g.Nc) ? __ldg(g.B + (size_t)(r0 + r) * g.ldb + n) : 0.f;
    }
  };
  float d[NCP / 2];
#pragma unroll
  for (int i = 0; i < NCP / 2; ++i) d[i] = 0.f;
  float cs0 = 0.f, cs1 = 0.f;
  if (nch > 0) load(0);
  for (int c = 0; c < nch; ++c) {
    // stage c & 1 was last read by the wgmmas of chunk c - 2, which every warpgroup waited for before the barrier of
    // chunk c - 1
    unsigned char* sh = smem + (size_t)(c & 1) * 2 * HALF;
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      const int it = warp + 8 * i;
      const uint32_t off = (uint32_t)(it >> 3) * SBO + (lane >> 2) * 16 + (it & 7) * 128 + (lane & 3) * 4;
      const uint32_t h = tf32_hi(bv[i]);
      *reinterpret_cast<uint32_t*>(sh + off) = h;
      *reinterpret_cast<uint32_t*>(sh + HALF + off) = tf32_lo(bv[i], h);
    }
    fence_async_smem();
    __syncthreads();
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      split4({av[s][0].x, av[s][0].y, av[s][1].x, av[s][1].y}, ah[s], al[s]);
      cs0 += av[s][0].x + av[s][1].x;
      cs1 += av[s][0].y + av[s][1].y;
    }
    if (c + 1 < nch) load(c + 1);                     // in flight while this chunk is multiplied
    const uint32_t bhi = s0 + (uint32_t)(c & 1) * 2 * HALF, blo = bhi + HALF;
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < 4; ++s) mma_step<NCP>(d, ah[s], al[s], bhi + s * 256, blo + s * 256, SBO);
    wgmma_commit();
    wgmma_wait0();
    if (c % TN_FLUSH == TN_FLUSH - 1 && c + 1 < nch) {
#pragma unroll
      for (int i = 0; i < NCP / 2; ++i) {
        part[i * WG_THREADS + tid] = parted ? part[i * WG_THREADS + tid] + d[i] : d[i];
        d[i] = 0.f;
      }
      parted = true;
    }
  }
  if (nch == 0 || !mok) return;
  if (parted)
#pragma unroll
    for (int i = 0; i < NCP / 2; ++i) d[i] += part[i * WG_THREADS + tid];
  if (g.colsum) {
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 1);
    cs0 += __shfl_xor_sync(0xffffffffu, cs0, 2);
    cs1 += __shfl_xor_sync(0xffffffffu, cs1, 1);
    cs1 += __shfl_xor_sync(0xffffffffu, cs1, 2);
    if (tq == 0) {
      atomicAdd(g.colsum + mb, cs0);
      atomicAdd(g.colsum + mb + 1, cs1);
    }
  }
#pragma unroll
  for (int i = 0; i < NCP / 2; i += 2) {
    const int col = (i / 16) * 32 + acc_col(i & 15, tq);
    if (col < g.Nc)
      atomicAdd(reinterpret_cast<float2*>(g.C + (size_t)(mb + ((i & 2) ? 1 : 0)) * g.ldc + col),
                make_float2(d[i], d[i + 1]));
  }
}

// ---------------------------------------------------------------------------------------------------------
inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }
inline bool al8(const void* p) { return ((uintptr_t)p & 7) == 0; }

// grid size of a persistent launch: as many CTAs as fit on the device, shared by `parts` independent grid columns
template <typename Kern>
static int persistent_ctas(Kern kern, size_t smem, int parts, int* out) {
  int occ = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, WG_THREADS, smem);
  if (e != cudaSuccess) return (int)e;
  const int n = PERT_NUM_SMS * (occ > 0 ? occ : 1) / parts;
  *out = n > 0 ? n : 1;
  return PERT_OK;
}

template <int BN>
static int launch_nt(const NtArgs& g, int nblk, int kplanes, cudaStream_t st) {
  const size_t smem = (size_t)BN * ((g.K + 7) & ~7) * 8;
  auto kern = k_gemm_nt_wg<BN>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  int gx = 0;
  int rc = persistent_ctas(kern, smem, nblk * kplanes, &gx);
  if (rc) return rc;
  const int pairs = (g.M + 127) / 128;
  if (gx > pairs) gx = pairs;
  kern<<<dim3(gx, nblk, kplanes), WG_THREADS, smem, st>>>(g);
  return PERT_OK;
}

}  // namespace

bool pert_gemm_tc_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("PERT_GEMM_TC");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

// Returns PERT_ERR_UNSUPPORTED when the shape / layout is outside what the tensor-core kernels handle (the caller
// then uses the exact-fp32 SIMT kernels of gemm.cu).
static int gemm_nt_tc_impl(const float* A, int lda, int a_cb, long long a_cbs, long long a_pz, const float* B, int ldb,
                           const float* bias, float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K,
                           int relu, int kplanes, cudaStream_t st);

// Layout requirements of k_gemm_nt_wg, on the arguments of gemm_nt_tc_impl (K is the K of one plane).  A column block
// that covers all of A or C is a plain matrix.
static bool nt_tc_layout_ok(const float* A, int lda, int a_cb, long long a_cbs, long long a_pz, const float* C,
                            int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K) {
  if (a_cb <= 0 || a_cb >= K) { a_cb = K; a_cbs = 0; }
  if (c_cb <= 0) { c_cb = Nc; c_cbs = 0; }
  if (K % 8 || K > 1024 || Nc % 16 || lda % 4 || ldc % 2 || c_cb % 16 || a_cbs % 4 || a_pz % 4 || c_cbs % 2 ||
      !al16(A) || !al8(C) || M > 0x7fffffff)
    return false;
  return a_cb == K || a_cb % 16 == 0;   // a 16-column chunk must not straddle two column blocks
}

int pert_gemm_nt_tc(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, const float* bias,
                    float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K, int relu,
                    cudaStream_t st) {
  if (!pert_gemm_tc_enabled() || M < 1024) return PERT_ERR_UNSUPPORTED;
  // Deep K over a column-blocked A (the data gradient dX = [dq|dk|dv|ds] . W4 at H = 128: K = 512): the whole [BN, K]
  // weight block (hi + lo) does not fit in shared memory unless BN is narrowed, which re-reads A once per N block.
  // Instead every column block of A is a plane (gridDim.z) with its own resident K-slice of the weights; C is zeroed
  // first and every plane accumulates into it (vector red.global), so A is read once.  The per-plane layout is checked
  // before C is cleared: a layout the planes cannot take (Nc = 100, say) goes to the SIMT kernel like any other.
  if (a_cb > 0 && a_cb < K && K % a_cb == 0 && !relu && Nc <= 128 && (size_t)Nc * K * 8 > SMEM_MAX &&
      (size_t)Nc * a_cb * 8 <= SMEM_MAX && K / a_cb <= 8 && (c_cb <= 0 || c_cb >= Nc) &&
      nt_tc_layout_ok(A, lda, a_cb, 0, a_cbs, C, ldc, c_cb, c_cbs, M, Nc, a_cb)) {
    cudaError_t me = (ldc == Nc) ? cudaMemsetAsync(C, 0, (size_t)M * Nc * sizeof(float), st)
                                 : cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)Nc * 4, (size_t)M, st);
    if (me != cudaSuccess) return (int)me;
    int rc = gemm_nt_tc_impl(A, lda, a_cb, 0, a_cbs, B, ldb, bias, C, ldc, c_cb, c_cbs, M, Nc, a_cb, 0, K / a_cb, st);
    return rc == PERT_ERR_UNSUPPORTED ? PERT_ERR_BADARG : rc;   // cannot happen after nt_tc_layout_ok; C is cleared
  }
  return gemm_nt_tc_impl(A, lda, a_cb, a_cbs, 0, B, ldb, bias, C, ldc, c_cb, c_cbs, M, Nc, K, relu, 1, st);
}

static int gemm_nt_tc_impl(const float* A, int lda, int a_cb, long long a_cbs, long long a_pz, const float* B, int ldb,
                           const float* bias, float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K,
                           int relu, int kplanes, cudaStream_t st) {
  if (a_cb <= 0 || a_cb >= K) { a_cb = K; a_cbs = 0; }
  if (c_cb <= 0) { c_cb = Nc; c_cbs = 0; }
  if (!nt_tc_layout_ok(A, lda, a_cb, a_cbs, a_pz, C, ldc, c_cb, c_cbs, M, Nc, K)) return PERT_ERR_UNSUPPORTED;
  // N block: <= 128 accumulator columns per warpgroup, Nc split into equal multiples of 16 (the whole [BN, K] weight
  // block is resident in shared memory, hi and lo: for a deep K it is narrowed until it fits, at the price of
  // re-reading A once per N block)
  const size_t Kp = (size_t)((K + 7) & ~7);
  int nblk = (Nc + 127) / 128, BN = 0;
  for (;; ++nblk) {
    if (nblk > Nc / 16) return PERT_ERR_UNSUPPORTED;
    if (Nc % nblk || (Nc / nblk) % 16) continue;
    BN = Nc / nblk;
    if ((size_t)BN * Kp * 8 <= SMEM_MAX) break;
  }
  NtArgs g{A, lda, a_cb, a_cbs, a_pz, B, ldb, bias, C, ldc, c_cb, c_cbs, (int)M, Nc, K, relu, kplanes > 1 ? 1 : 0};
  switch (BN) {
    case 16: return launch_nt<16>(g, nblk, kplanes, st);
    case 32: return launch_nt<32>(g, nblk, kplanes, st);
    case 48: return launch_nt<48>(g, nblk, kplanes, st);
    case 64: return launch_nt<64>(g, nblk, kplanes, st);
    case 80: return launch_nt<80>(g, nblk, kplanes, st);
    case 96: return launch_nt<96>(g, nblk, kplanes, st);
    case 112: return launch_nt<112>(g, nblk, kplanes, st);
    case 128: return launch_nt<128>(g, nblk, kplanes, st);
  }
  return PERT_ERR_UNSUPPORTED;
}

template <int NCP>
static int launch_tn(TnArgs g, int mblk, cudaStream_t st) {
  const size_t smem = (size_t)NCP * RC * 4 * 2 * 2 + (size_t)NCP / 2 * WG_THREADS * 4;   // two stages (hi + lo), partials
  auto kern = k_gemm_tn_wg<NCP>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  int splits = 0;
  int rc = persistent_ctas(kern, smem, mblk, &splits);
  if (rc) return rc;
  int rps = (g.R + splits - 1) / splits;
  rps = (rps + RC - 1) / RC * RC;
  splits = (g.R + rps - 1) / rps;
  g.rows_per_split = rps;
  kern<<<dim3(splits, mblk), WG_THREADS, smem, st>>>(g);
  return PERT_OK;
}

int pert_gemm_tn_tc(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, int b_cb,
                    long long b_cbs, float* C, int ldc, float* a_colsum, long long R, int Mc, int Nc,
                    cudaStream_t st) {
  if (!pert_gemm_tc_enabled() || R < 4096) return PERT_ERR_UNSUPPORTED;
  if (a_cb <= 0) { a_cb = Mc; a_cbs = 0; }
  if (b_cb > 0 && b_cb < Nc) return PERT_ERR_UNSUPPORTED;   // B must be a plain matrix
  // two adjacent output rows per thread (8-byte loads of A), two adjacent columns per vector reduction into C
  if (Nc % 4 || Nc > 160 || Mc % 2 || a_cb % 2 || lda % 2 || a_cbs % 2 || ldc % 2 || !al8(A) || !al8(C) ||
      R > 0x7fffffff)
    return PERT_ERR_UNSUPPORTED;
  (void)b_cbs;
  TnArgs g{A, lda, a_cb, a_cbs, B, ldb, C, ldc, a_colsum, (int)R, Mc, Nc, 0};
  const int mblk = (Mc + 127) / 128;
  switch ((Nc + 15) / 16) {
    case 1: return launch_tn<16>(g, mblk, st);
    case 2: return launch_tn<32>(g, mblk, st);
    case 3: return launch_tn<48>(g, mblk, st);
    case 4: return launch_tn<64>(g, mblk, st);
    case 5: return launch_tn<80>(g, mblk, st);
    case 6: return launch_tn<96>(g, mblk, st);
    case 7: return launch_tn<112>(g, mblk, st);
    case 8: return launch_tn<128>(g, mblk, st);
    case 9: return launch_tn<144>(g, mblk, st);
    case 10: return launch_tn<160>(g, mblk, st);
  }
  return PERT_ERR_UNSUPPORTED;
}
