// Dense fp32 linears of the hot path (reference model.py:26-55 Linear / lin_{query,key,value,skip,edge};
// PyG Linear == x W^T + b).  Exact-fp32 SIMT kernels: the 1e-4 parity bar of BASELINE.json rules out
// single-pass TF32 (SURVEY.md 7 "hard parts").  K is tiny (<= a few hundred) and M = #nodes is huge, so
// these are streaming GEMMs: A read once, C written once.
//
//  NT : C[M,Nc]  = A[M,K] . B[Nc,K]^T (+ bias[Nc]) (relu)      forward and data-gradient
//  TN : C[Mc,Nc] += A[R,Mc]^T . B[R,Nc]                         weight gradient (split over R, atomics)
//  colsum: out[c] += sum_r A[r,c]                                bias gradient
//
// "Column-block" addressing lets one GEMM write/read the 4 node planes (q|k|v|skip stored as
// [4][M][H]) as if they were one [M,4H] matrix: element (m, c) of a blocked matrix lives at
//   base + (c / cb) * cbs + m * ld + (c % cb).      (cb = c-extent of a block, cbs = block stride)
#include "common.cuh"

namespace {

struct Blocked {
  int ld;         // row stride (floats)
  int cb;         // columns per block (>= total columns => plain matrix)
  long long cbs;  // stride between column blocks (floats)
};
__device__ __forceinline__ size_t baddr(const Blocked& b, int row, int col) {
  int blk = col / b.cb;
  return (size_t)blk * b.cbs + (size_t)row * b.ld + (col - blk * b.cb);
}

constexpr int BM = 128, BN = 64, BK = 16, NT_THREADS = 256;
constexpr int APAD = 4;

// requires: K % 4 == 0, a.cb % 4 == 0, 16-byte aligned rows (checked on host)
__global__ void __launch_bounds__(NT_THREADS) k_gemm_nt(const float* __restrict__ A, Blocked a,
                                                         const float* __restrict__ B, int ldb,
                                                         const float* __restrict__ bias, float* __restrict__ C,
                                                         Blocked c, int M, int Nc, int K, int relu, int accumulate,
                                                         int vec_a, int vec_b) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN + APAD];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int ty = tid / 16, tx = tid % 16;  // 16 x 16 threads, 8 x 4 outputs each
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // global->register staging: A tile 128x16 = 512 float4 (2 per thread), B tile 64x16 = 256 float4 (1 per thread)
  const int a_row = tid / 4, a_k = (tid % 4) * 4;
  const int b_row = tid / 4, b_k = (tid % 4) * 4;
  float4 ra[2], rb;
  auto gload = [&](int k0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      int m = m0 + a_row + 64 * r, k = k0 + a_k;
      if (vec_a) {
        ra[r] = (m < M && k < K) ? ldg4(A + baddr(a, m, k)) : f4zero();
      } else {
        ra[r] = f4zero();
        if (m < M)
          for (int j = 0; j < 4; ++j)
            if (k + j < K) (&ra[r].x)[j] = __ldg(A + baddr(a, m, k + j));
      }
    }
    int n = n0 + b_row, k = k0 + b_k;
    if (vec_b) {
      rb = (n < Nc && k < K) ? ldg4(B + (size_t)n * ldb + k) : f4zero();
    } else {
      rb = f4zero();
      if (n < Nc)
        for (int j = 0; j < 4; ++j)
          if (k + j < K) (&rb.x)[j] = __ldg(B + (size_t)n * ldb + k + j);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      int row = a_row + 64 * r;
      As[buf][a_k + 0][row] = ra[r].x;
      As[buf][a_k + 1][row] = ra[r].y;
      As[buf][a_k + 2][row] = ra[r].z;
      As[buf][a_k + 3][row] = ra[r].w;
    }
    Bs[buf][b_k + 0][b_row] = rb.x;
    Bs[buf][b_k + 1][b_row] = rb.y;
    Bs[buf][b_k + 2][b_row] = rb.z;
    Bs[buf][b_k + 3][b_row] = rb.w;
  };
  const int nk = (K + BK - 1) / BK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8 + 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }
  // epilogue: 4 consecutive columns per thread -> one float4 store when the block layout allows
  const int n = n0 + tx * 4;
  if (n >= Nc) return;
  float bb[4] = {0.f, 0.f, 0.f, 0.f};
  if (bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (n + j < Nc) bb[j] = __ldg(bias + n + j);
  }
  const bool vec = (n + 3 < Nc) && (c.cb % 4 == 0) && (c.ld % 4 == 0) && (c.cbs % 4 == 0) &&
                   ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + ty * 8 + i;
    if (m >= M) break;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = acc[i][j] + bb[j];
      if (relu) v[j] = fmaxf(v[j], 0.f);
    }
    if (vec) {
      float* p = C + baddr(c, m, n);
      if (accumulate) {
        float4 o = ld4(p);
        v[0] += o.x; v[1] += o.y; v[2] += o.z; v[3] += o.w;
      }
      st4(p, make_float4(v[0], v[1], v[2], v[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < Nc) {
          float* p = C + baddr(c, m, n + j);
          *p = accumulate ? (*p + v[j]) : v[j];
        }
    }
  }
}

// ---- TN: C[Mc,Nc] += A[R,Mc]^T B[R,Nc]; grid (Mc/64, Nc/64, splits over R) ----------------------
constexpr int TM = 64, TN_ = 64, TR = 16, TN_THREADS = 256;

__global__ void __launch_bounds__(TN_THREADS) k_gemm_tn(const float* __restrict__ A, Blocked a,
                                                         const float* __restrict__ B, Blocked b,
                                                         float* __restrict__ C, int ldc, int R, int Mc, int Nc,
                                                         int rows_per_split, int vec_a, int vec_b) {
  __shared__ __align__(16) float As[TR][TM + 4];
  __shared__ __align__(16) float Bs[TR][TN_ + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN_;
  const int r_begin = blockIdx.z * rows_per_split;
  const int r_end = min(R, r_begin + rows_per_split);
  const int ty = tid / 16, tx = tid % 16;  // 4 x 4 outputs each
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int l_row = tid / 16, l_col = (tid % 16) * 4;  // 16 rows x 16 float4
  for (int r0 = r_begin; r0 < r_end; r0 += TR) {
    int r = r0 + l_row;
    float4 va = f4zero(), vb = f4zero();
    if (r < r_end) {
      int mc = m0 + l_col, nc = n0 + l_col;
      if (vec_a && mc + 3 < Mc) va = ldg4(A + baddr(a, r, mc));
      else
        for (int j = 0; j < 4; ++j)
          if (mc + j < Mc) (&va.x)[j] = __ldg(A + baddr(a, r, mc + j));
      if (vec_b && nc + 3 < Nc) vb = ldg4(B + baddr(b, r, nc));
      else
        for (int j = 0; j < 4; ++j)
          if (nc + j < Nc) (&vb.x)[j] = __ldg(B + baddr(b, r, nc + j));
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&As[l_row][l_col]) = va;
    *reinterpret_cast<float4*>(&Bs[l_row][l_col]) = vb;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TR; ++kk) {
      float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      float av[4] = {a4.x, a4.y, a4.z, a4.w};
      float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= Mc) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < Nc) atomicAdd(C + (size_t)m * ldc + n, acc[i][j]);
    }
  }
}

// out[c] += sum_r A[r,c];  block = 32 columns x 8 row-lanes, grid (cols/32, row splits)
__global__ void __launch_bounds__(256) k_colsum(const float* __restrict__ A, Blocked a, float* __restrict__ out,
                                                 int R, int Cc, int rows_per_split) {
  __shared__ float part[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  const int r_begin = blockIdx.y * rows_per_split, r_end = min(R, r_begin + rows_per_split);
  float s = 0.f;
  if (col < Cc)
    for (int r = r_begin + ry; r < r_end; r += 8) s += __ldg(A + baddr(a, r, col));
  part[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && col < Cc) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += part[i][cx];
    atomicAdd(out + col, t);
  }
}

inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

// tensor-core (wgmma, 3xTF32) kernels of gemm_tc.cu; PERT_ERR_UNSUPPORTED => exact-fp32 SIMT kernels below
int pert_gemm_nt_tc(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, const float* bias,
                    float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K, int relu,
                    cudaStream_t st);
int pert_gemm_tn_tc(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, int b_cb,
                    long long b_cbs, float* C, int ldc, float* a_colsum, long long R, int Mc, int Nc,
                    cudaStream_t st);

extern "C" {

int pert_gemm_nt(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, const float* bias,
                 float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K, int relu, int accumulate,
                 void* stream) {
  if (M < 0 || Nc <= 0 || K <= 0 || !A || !B || !C) return PERT_ERR_BADARG;
  if (a_cb <= 0) a_cb = K;
  if (c_cb <= 0) c_cb = Nc;
  if (M == 0) return PERT_OK;
  if (!accumulate) {
    int rt = pert_gemm_nt_tc(A, lda, a_cb, a_cbs, B, ldb, bias, C, ldc, c_cb, c_cbs, M, Nc, K, relu,
                             (cudaStream_t)stream);
    if (rt != PERT_ERR_UNSUPPORTED) {
      if (rt) return rt;
      PERT_LAUNCH_CHECK();
      return PERT_OK;
    }
  }
  const int vec_a = !(K % 4 || lda % 4 || a_cb % 4 || a_cbs % 4 || !al16(A));
  const int vec_b = !(K % 4 || ldb % 4 || !al16(B));
  Blocked a{lda, a_cb, a_cbs}, c{ldc, c_cb, c_cbs};
  dim3 grid(pert_cdiv(M, BM), pert_cdiv(Nc, BN));
  k_gemm_nt<<<grid, NT_THREADS, 0, (cudaStream_t)stream>>>(A, a, B, ldb, bias, C, c, (int)M, Nc, K, relu,
                                                          accumulate, vec_a, vec_b);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_gemm_tn(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, int b_cb,
                 long long b_cbs, float* C, int ldc, float* a_colsum, long long R, int Mc, int Nc, void* stream) {
  if (R < 0 || Mc <= 0 || Nc <= 0 || !A || !B || !C) return PERT_ERR_BADARG;
  if (a_cb <= 0) a_cb = Mc;
  if (b_cb <= 0) b_cb = Nc;
  if (R == 0) return PERT_OK;
  {
    int rt = pert_gemm_tn_tc(A, lda, a_cb, a_cbs, B, ldb, b_cb, b_cbs, C, ldc, a_colsum, R, Mc, Nc,
                             (cudaStream_t)stream);
    if (rt != PERT_ERR_UNSUPPORTED) {
      if (rt) return rt;
      PERT_LAUNCH_CHECK();
      return PERT_OK;
    }
  }
  if (a_colsum) {
    int rc = pert_colsum(A, lda, a_cb, a_cbs, a_colsum, R, Mc, stream);
    if (rc) return rc;
  }
  const int vec_a = !(lda % 4 || a_cb % 4 || a_cbs % 4 || !al16(A));
  const int vec_b = !(ldb % 4 || b_cb % 4 || b_cbs % 4 || !al16(B));
  Blocked a{lda, a_cb, a_cbs}, b{ldb, b_cb, b_cbs};
  int tiles = pert_cdiv(Mc, TM) * pert_cdiv(Nc, TN_);
  int splits = (2 * PERT_NUM_SMS + tiles - 1) / tiles;
  int max_splits = pert_cdiv(R, 4 * TR);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int rps = pert_cdiv(R, splits);
  rps = (rps + TR - 1) / TR * TR;
  splits = pert_cdiv(R, rps);
  dim3 grid(pert_cdiv(Mc, TM), pert_cdiv(Nc, TN_), splits);
  k_gemm_tn<<<grid, TN_THREADS, 0, (cudaStream_t)stream>>>(A, a, B, b, C, ldc, (int)R, Mc, Nc, rps, vec_a,
                                                          vec_b);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_colsum(const float* A, int lda, int a_cb, long long a_cbs, float* out, long long R, int Cc, void* stream) {
  if (R < 0 || Cc <= 0 || !A || !out) return PERT_ERR_BADARG;
  if (a_cb <= 0) a_cb = Cc;
  if (R == 0) return PERT_OK;
  Blocked a{lda, a_cb, a_cbs};
  int cblocks = pert_cdiv(Cc, 32);
  int splits = (2 * PERT_NUM_SMS + cblocks - 1) / cblocks;
  int max_splits = pert_cdiv(R, 64);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int rps = pert_cdiv(R, splits);
  splits = pert_cdiv(R, rps);
  k_colsum<<<dim3(cblocks, splits), 256, 0, (cudaStream_t)stream>>>(A, a, out, (int)R, Cc, rps);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
