// Node-/graph-level pieces of the hot path around the fused conv (all HBM-bound elementwise / reduction work):
//   embedding gather / scatter-add           reference model.py:87-97,108  (nn.Embedding fwd / dense bwd)
//   feature concat                           model.py:90
//   BatchNorm1d (+ReLU) fwd / bwd            model.py:101-102 (training: batch stats, eps 1e-5, momentum 0.1)
//   local head + prob-weighted add-pool      model.py:105-107 (local_linear, x*probs/num_nodes, global_add_pool)
//   pinball loss, Adam                       pert_gnn.py:191-193,245-247
#include "common.cuh"
#include "bn.cuh"
#include <limits.h>
#include <string.h>
#include <type_traits>

namespace {

// ---------------------------------------------------------------- embeddings
// out[n, 0:H] (+)= table[ids[n*id_stride], :]
__global__ void k_embedding_fwd(const float* __restrict__ table, int n_rows, const int64_t* __restrict__ ids,
                                int id_stride, float* __restrict__ out, int ld_out, long long N, int H,
                                int accumulate, int* status) {
  const int vec_per_row = H >> 2;
  long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= N * vec_per_row) return;
  long long n = id / vec_per_row;
  int c = (int)(id % vec_per_row) * 4;
  int64_t r = ids[n * id_stride];
  if (r < 0 || r >= n_rows) {
    if (status) atomicExch(status, PERT_ERR_RANGE);
    r = 0;
  }
  float4 v = ldg4(table + (size_t)r * H + c);
  float* o = out + (size_t)n * ld_out + c;
  if (accumulate) v = f4add(v, ld4(o));
  st4(o, v);
}

// dtable[ids[n*id_stride], :] += dy[n, 0:H]      (REDG.128; nn.Embedding dense backward)
// One thread owns one float4 column of EB_RUN consecutive rows and merges equal ids before the atomic: the stage nodes
// of a microservice are consecutive in a PERT graph (misc.py:238-250: 2c+1 nodes per caller share cat_X), so real
// batches send runs of rows to the same table row.
constexpr int EB_RUN = 8;
__global__ void k_embedding_bwd(const float* __restrict__ dy, int ld_dy, const int64_t* __restrict__ ids,
                                int id_stride, float* __restrict__ dtable, int n_rows, long long N, int H) {
  const int vec_per_row = H >> 2;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long chunks = (N + EB_RUN - 1) / EB_RUN;
  if (id >= chunks * vec_per_row) return;
  const long long n0 = (id / vec_per_row) * EB_RUN;
  const int c = (int)(id % vec_per_row) * 4;
  int64_t cur = -1;
  float4 acc = f4zero();
#pragma unroll
  for (int k = 0; k < EB_RUN; ++k) {
    const long long n = n0 + k;
    if (n >= N) break;
    const int64_t r = ids[n * id_stride];
    if (r != cur) {
      if (cur >= 0 && cur < n_rows) red4(dtable + (size_t)cur * H + c, acc);
      cur = r;
      acc = f4zero();
    }
    acc = f4add(acc, ldg4(dy + (size_t)n * ld_dy + c));
  }
  if (cur >= 0 && cur < n_rows) red4(dtable + (size_t)cur * H + c, acc);
}

// out[n, col0 : col0+F] = x[n, 0:F]; out[n, col0+F : ld_out) = 0
__global__ void k_copy_cols(const float* __restrict__ x, int F, float* __restrict__ out, int ld_out, int col0,
                            long long N) {
  const int w = ld_out - col0;
  long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= N * w) return;
  long long n = id / w;
  int c = (int)(id % w);
  out[(size_t)n * ld_out + col0 + c] = (c < F) ? x[(size_t)n * F + c] : 0.f;
}

// ---------------------------------------------------------------- batch norm
constexpr int BN_ROWS = 128;      // rows per CTA chunk (forward statistics)
constexpr int BN_BWD_ROWS = 64;   // rows per CTA (backward reductions: atomics, so the chunk count is free)

// per-chunk (mean, M2) with a two-pass centred sum in fp32; the chunks are combined in double precision by
// bn_acc_chunk (bn.cuh: acc[c] += n_b mean_b,  acc[H + c] += M2_b + n_b mean_b^2, fp64 atomics), so no finalize kernel
// is needed -- k_bn_apply derives mean / rstd from acc in its prologue.
// live != null (padded batch, see pert_batch_pad): only the rows below live[0] are counted.
__global__ void __launch_bounds__(256) k_bn_partial(const float* __restrict__ x, int ld, long long N, int H,
                                                     double* __restrict__ acc /*[2][H], zeroed*/,
                                                     const long long* __restrict__ live) {
  extern __shared__ float sm[];  // [rl][H] scratch, then mean[H]
  const int vpr = H >> 2;              // float4 lanes per row
  const int rl_n = blockDim.x / vpr;   // row lanes
  const int cl = threadIdx.x % vpr, rl = threadIdx.x / vpr;
  const long long r0 = (long long)blockIdx.x * BN_ROWS;
  if (live) N = min(N, live[0]);
  if (r0 >= N) return;                 // a chunk of ghost rows only (block-uniform)
  const int rows = (int)min((long long)BN_ROWS, N - r0);
  float* s_red = sm;             // [rl_n][H]
  float* s_mean = sm + rl_n * H; // [H]
  float4 s = f4zero();
  if (rl < rl_n)
    for (int rb = rl; rb < rows; rb += 8 * rl_n) {   // 8 independent row loads in flight per thread
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int r = rb + u * rl_n;
        v[u] = (r < rows) ? ldg4(x + (size_t)(r0 + r) * ld + cl * 4) : f4zero();
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) s = f4add(s, v[u]);
    }
  if (rl < rl_n) st4(s_red + rl * H + cl * 4, s);
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += blockDim.x) {   // H > 256: a thread owns several columns
    float t = 0.f;
    for (int i = 0; i < rl_n; ++i) t += s_red[i * H + c];
    s_mean[c] = t / (float)rows;
  }
  __syncthreads();
  float4 mu = (rl < rl_n) ? ld4(s_mean + cl * 4) : f4zero();
  float4 q = f4zero();
  if (rl < rl_n)
    for (int rb = rl; rb < rows; rb += 8 * rl_n) {
      float4 vv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int r = rb + u * rl_n;
        vv[u] = (r < rows) ? ldg4(x + (size_t)(r0 + r) * ld + cl * 4) : mu;   // mu => contributes 0
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float4 v = vv[u];
        float dx = v.x - mu.x, dy = v.y - mu.y, dz = v.z - mu.z, dw = v.w - mu.w;
        q.x = fmaf(dx, dx, q.x); q.y = fmaf(dy, dy, q.y); q.z = fmaf(dz, dz, q.z); q.w = fmaf(dw, dw, q.w);
      }
    }
  __syncthreads();
  if (rl < rl_n) st4(s_red + rl * H + cl * 4, q);
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float t = 0.f;
    for (int i = 0; i < rl_n; ++i) t += s_red[i * H + c];
    bn_acc_chunk(acc, H, c, (double)rows, (double)s_mean[c], (double)t);
  }
}

// eval mode: mean = running_mean, rstd = 1/sqrt(running_var + eps)
__global__ void k_bn_eval_stats(const float* __restrict__ rm, const float* __restrict__ rv, float eps, int H,
                                float* __restrict__ mean, float* __restrict__ rstd) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  mean[c] = rm[c];
  rstd[c] = 1.0f / sqrtf(rv[c] + eps);
}

// y = (relu)((x - mean) rstd gamma + beta) [* keep * scale].  acc != null (training): mean / rstd come from the fp64
// sums of k_bn_partial (every CTA derives them in its prologue; CTA 0 also stores them for the backward pass and
// updates the running statistics); acc == null (eval): mean / rstd arrays are read.  DROP (training + ReLU only):
// inverted dropout of the ReLU output, one Philox call per float4.
template <bool DROP>
__global__ void __launch_bounds__(256) k_bn_apply(const float* __restrict__ x, int ld_x, float* __restrict__ mean,
                                                   float* __restrict__ rstd, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* __restrict__ y, int ld_y,
                                                   long long N, int H, int relu, const double* __restrict__ acc,
                                                   float eps, float momentum, float* running_mean,
                                                   float* running_var, long long* num_batches_tracked,
                                                   BnDropout drop, const long long* __restrict__ live) {
  extern __shared__ float s_par[];   // mean | rstd | gamma | beta
  const long long n_stat = live ? live[0] : N;   // rows the statistics count (every row is normalised)
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float mu, rs;
    if (acc) {
      bn_batch_stats(acc, n_stat, H, c, eps, momentum, blockIdx.x == 0, mean, rstd, running_mean, running_var,
                     num_batches_tracked, mu, rs);
    } else {
      mu = mean[c];
      rs = rstd[c];
    }
    s_par[c] = mu;
    s_par[H + c] = rs;
    s_par[2 * H + c] = gamma[c];
    s_par[3 * H + c] = beta[c];
  }
  __syncthreads();
  const int vpr = H >> 2;
  const long long total = N * vpr;
  const BnDropKey key = DROP ? bn_drop_key(drop) : BnDropKey{};
  for (long long id0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; id0 < total;
       id0 += 4LL * gridDim.x * blockDim.x) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {       // 4 independent row loads in flight
      const long long id = id0 + (long long)u * gridDim.x * blockDim.x;
      v[u] = id < total ? ldg4(x + (size_t)(id / vpr) * ld_x + (int)(id % vpr) * 4) : f4zero();
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long id = id0 + (long long)u * gridDim.x * blockDim.x;
      if (id >= total) break;
      const int c = (int)(id % vpr) * 4;
      const float4 mu = ld4(s_par + c), rs = ld4(s_par + H + c), ga = ld4(s_par + 2 * H + c), be = ld4(s_par + 3 * H + c);
      float4 o = bn_affine4(v[u], mu, rs, ga, be, relu);
      if (DROP) o = bn_dropout4(o, (uint32_t)id, drop, key);   // id = row * (H/4) + col/4 is the float4 group
      st4(y + (size_t)(id / vpr) * ld_y + c, o);
    }
  }
}

// sums[0:H] += sum_n dz,  sums[H:2H] += sum_n dz*xhat   with dz = dy * (y > 0 if relu) * scale (bn_bwd_dz4).
__global__ void __launch_bounds__(256) k_bn_bwd_reduce(const float* __restrict__ dy, int ld_dy,
                                                        const float* __restrict__ y, int ld_y,
                                                        const float* __restrict__ x, int ld_x,
                                                        const float* __restrict__ mean,
                                                        const float* __restrict__ rstd, long long N, int H, int relu,
                                                        float scale, float* __restrict__ sums,
                                                        const long long* __restrict__ live) {
  extern __shared__ float sm[];  // [rl_n][2H]
  const int vpr = H >> 2;
  const int rl_n = blockDim.x / vpr;
  const int cl = threadIdx.x % vpr, rl = threadIdx.x / vpr;
  const long long r0 = (long long)blockIdx.x * BN_BWD_ROWS;
  if (live) N = min(N, live[0]);
  if (r0 >= N) return;                 // ghost rows only (block-uniform)
  const int rows = (int)min((long long)BN_BWD_ROWS, N - r0);
  float4 s1 = f4zero(), s2 = f4zero();
  if (rl < rl_n) {
    const float4 mu = ldg4(mean + cl * 4), rs = ldg4(rstd + cl * 4);
    for (int rb = rl; rb < rows; rb += 4 * rl_n) {   // 4 rows x 3 operands = 12 independent loads in flight
      float4 gg[4], yy4[4], vv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = rb + u * rl_n;
        const bool ok = r < rows;
        gg[u] = ok ? ldg4(dy + (size_t)(r0 + r) * ld_dy + cl * 4) : f4zero();
        yy4[u] = (ok && relu) ? ldg4(y + (size_t)(r0 + r) * ld_y + cl * 4) : make_float4(1.f, 1.f, 1.f, 1.f);
        vv[u] = ok ? ldg4(x + (size_t)(r0 + r) * ld_x + cl * 4) : mu;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) bn_bwd_acc4(s1, s2, bn_bwd_dz4(gg[u], yy4[u], scale), vv[u], mu, rs);
    }
    st4(sm + rl * 2 * H + cl * 4, s1);
    st4(sm + rl * 2 * H + H + cl * 4, s2);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) {
    float t = 0.f;
    for (int i = 0; i < rl_n; ++i) t += sm[i * 2 * H + c];
    atomicAdd(sums + c, t);
  }
}

// training: dx = gamma*rstd*(dz - sum_dz/N - xhat*sum_dzxhat/N); eval: dx = gamma*rstd*dz.
// live != null (padded batch): N in the mean terms is live[0], and the ghost rows n >= live[0] get dx = 0 -- the mean
// terms would otherwise hand them a gradient that flows on into the weights and the embedding row of the ghosts.
__global__ void k_bn_bwd_apply(const float* __restrict__ dy, int ld_dy, const float* __restrict__ y, int ld_y,
                               const float* __restrict__ x, int ld_x, const float* __restrict__ mean,
                               const float* __restrict__ rstd, const float* __restrict__ gamma,
                               const float* __restrict__ sums, float* __restrict__ dx, int ld_dx, long long N, int H,
                               int relu, float scale, int training, float* dgamma, float* dbeta,
                               const long long* __restrict__ live) {
  const int vpr = H >> 2;
  long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0)  // parameter grads accumulate (+=) like autograd
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      if (dbeta) dbeta[c] += sums[c];
      if (dgamma) dgamma[c] += sums[H + c];
    }
  if (id >= N * vpr) return;
  long long n = id / vpr;
  int c = (int)(id % vpr) * 4;
  const long long n_live = live ? live[0] : N;
  if (n >= n_live) {
    st4(dx + (size_t)n * ld_dx + c, f4zero());
    return;
  }
  float4 g = ldg4(dy + (size_t)n * ld_dy + c);
  if (relu) g = bn_bwd_dz4(g, ldg4(y + (size_t)n * ld_y + c), scale);
  const float4 rs = ldg4(rstd + c), ga = ldg4(gamma + c);
  float4 o;
  if (training) {
    const float invn = 1.0f / (float)n_live;
    const float4 v = ldg4(x + (size_t)n * ld_x + c), mu = ldg4(mean + c);
    o = bn_bwd_dx4(g, v, mu, rs, ga, ldg4(sums + c), ldg4(sums + H + c), invn);
  } else {
    o = make_float4(ga.x * rs.x * g.x, ga.y * rs.y * g.y, ga.z * rs.z * g.z, ga.w * rs.w * g.w);
  }
  st4(dx + (size_t)n * ld_dx + c, o);
}

// ---------------------------------------------------------------- local head + weighted add-pool
constexpr int POOL_ROWS = 8;  // consecutive rows per lane group (run-length pre-aggregation of the pool atomics)

template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_pool_fwd(const float* __restrict__ x, int ld, const float* __restrict__ probs,
                                                   const float* __restrict__ pnn, const int64_t* __restrict__ batch,
                                                   const float* __restrict__ w_local, const float* __restrict__ b_local,
                                                   float* __restrict__ local, float* __restrict__ pool, long long N,
                                                   int B, int* status) {
  constexpr int H = 4 * LPR * VPL;
  const int lane = threadIdx.x & 31, lig = lane % LPR, grp = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (grp * LPR));
  const long long gid = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * (32 / LPR) + grp;
  const long long r0 = gid * POOL_ROWS;
  if (r0 >= N) return;
  float4 w[VPL], acc[VPL];
#pragma unroll
  for (int u = 0; u < VPL; ++u) {
    w[u] = w_local ? ldg4(w_local + lig * 4 + u * LPR * 4) : f4zero();
    acc[u] = f4zero();
  }
  const float bl = b_local ? __ldg(b_local) : 0.f;
  long long cur = -1;
  const int rows = (int)min((long long)POOL_ROWS, N - r0);
  for (int r = 0; r < rows; ++r) {
    const long long n = r0 + r;
    float4 v[VPL];
    float d = 0.f;
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      v[u] = ldg4(x + (size_t)n * ld + lig * 4 + u * LPR * 4);
      d += f4dot(v[u], w[u]);
    }
    if (local) {
      d = group_sum<LPR>(d, gmask);
      if (lig == 0) local[n] = d + bl;
    }
    long long g = batch[n];
    if (g < 0 || g >= B) {
      if (status) atomicExch(status, PERT_ERR_RANGE);
      continue;
    }
    if (g != cur) {
      if (cur >= 0) {
#pragma unroll
        for (int u = 0; u < VPL; ++u) red4(pool + (size_t)cur * H + lig * 4 + u * LPR * 4, acc[u]);
      }
#pragma unroll
      for (int u = 0; u < VPL; ++u) acc[u] = f4zero();
      cur = g;
    }
    const float pr = __ldg(probs + n), nn = __ldg(pnn + n);
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      // reference order: (x * p) / n  (model.py:106) -- keep the two roundings
      acc[u].x += (v[u].x * pr) / nn;
      acc[u].y += (v[u].y * pr) / nn;
      acc[u].z += (v[u].z * pr) / nn;
      acc[u].w += (v[u].w * pr) / nn;
    }
  }
  if (cur >= 0) {
#pragma unroll
    for (int u = 0; u < VPL; ++u) red4(pool + (size_t)cur * H + lig * 4 + u * LPR * 4, acc[u]);
  }
}

// dx[n] = dlocal[n]*w_local + dpool[batch[n]] * probs[n]/pnn[n];  dw_local += sum dlocal[n]*x[n]; db_local += sum dlocal
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_pool_bwd(const float* __restrict__ dpool, const float* __restrict__ dlocal,
                                                   const float* __restrict__ x, int ld,
                                                   const float* __restrict__ probs, const float* __restrict__ pnn,
                                                   const int64_t* __restrict__ batch,
                                                   const float* __restrict__ w_local, float* __restrict__ dx,
                                                   int ld_dx, float* __restrict__ dw_local,
                                                   float* __restrict__ db_local, long long N, int B) {
  constexpr int H = 4 * LPR * VPL;
  __shared__ float s_dw[H];
  __shared__ float s_db;
  const bool has_local = dlocal != nullptr;
  if (has_local) {
    for (int c = threadIdx.x; c < H; c += blockDim.x) s_dw[c] = 0.f;
    if (threadIdx.x == 0) s_db = 0.f;
    __syncthreads();
  }
  const int lane = threadIdx.x & 31, lig = lane % LPR, grp = lane / LPR;
  const long long gid = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * (32 / LPR) + grp;
  const long long r0 = gid * POOL_ROWS;
  float4 w[VPL], dw[VPL];
  float db = 0.f;
#pragma unroll
  for (int u = 0; u < VPL; ++u) {
    w[u] = (has_local && w_local) ? ldg4(w_local + lig * 4 + u * LPR * 4) : f4zero();
    dw[u] = f4zero();
  }
  if (r0 < N) {
    const int rows = (int)min((long long)POOL_ROWS, N - r0);
    for (int r = 0; r < rows; ++r) {
      const long long n = r0 + r;
      const long long g = batch[n];
      const float sc = __ldg(probs + n) / __ldg(pnn + n);
      const float dl = has_local ? __ldg(dlocal + n) : 0.f;
      db += dl;
#pragma unroll
      for (int u = 0; u < VPL; ++u) {
        float4 o = f4zero();
        if (dpool && g >= 0 && g < B) o = f4scale(sc, ldg4(dpool + (size_t)g * H + lig * 4 + u * LPR * 4));
        if (has_local) {
          o = f4fma(dl, w[u], o);
          dw[u] = f4fma(dl, ldg4(x + (size_t)n * ld + lig * 4 + u * LPR * 4), dw[u]);
        }
        st4(dx + (size_t)n * ld_dx + lig * 4 + u * LPR * 4, o);
      }
    }
  }
  if (has_local) {
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      float* p = s_dw + lig * 4 + u * LPR * 4;
      atomicAdd(p + 0, dw[u].x); atomicAdd(p + 1, dw[u].y); atomicAdd(p + 2, dw[u].z); atomicAdd(p + 3, dw[u].w);
    }
    if (lig == 0) atomicAdd(&s_db, db);
    __syncthreads();
    if (dw_local)
      for (int c = threadIdx.x; c < H; c += blockDim.x) atomicAdd(dw_local + c, s_dw[c]);
    if (db_local && threadIdx.x == 0) atomicAdd(db_local, s_db);
  }
}

template <typename F>
int dispatch_h(int H, F&& f) {
  switch (H) {
    case 4: return f(std::integral_constant<int, 1>{}, std::integral_constant<int, 1>{});
    case 8: return f(std::integral_constant<int, 2>{}, std::integral_constant<int, 1>{});
    case 16: return f(std::integral_constant<int, 4>{}, std::integral_constant<int, 1>{});
    case 32: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 1>{});
    case 64: return f(std::integral_constant<int, 16>{}, std::integral_constant<int, 1>{});
    case 96: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 3>{});
    case 128: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 1>{});
    case 192: return f(std::integral_constant<int, 16>{}, std::integral_constant<int, 3>{});
    case 256: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 2>{});
    default: return PERT_ERR_UNSUPPORTED;
  }
}

// ---------------------------------------------------------------- small elementwise
__global__ void k_relu_bwd(const float* __restrict__ y, float* __restrict__ dy, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(y[i] > 0.f)) dy[i] = 0.f;
}

// pinball loss (pert_gnn.py:191-193): loss = mean(max(tau*e, (tau-1)*e)), e = y - yhat; dyhat = dloss/dyhat.
// live != null (padded batch): the mean runs over the graphs i < live[1]; the ghost graphs above get dyhat = 0.
__global__ void k_pinball(const int64_t* __restrict__ y, const float* __restrict__ yhat, float tau, int B,
                          float grad_scale, float* __restrict__ loss, float* __restrict__ dyhat,
                          const long long* __restrict__ live) {
  __shared__ float red[32];
  const int Bl = live ? (int)min((long long)B, live[1]) : B;
  float s = 0.f;
  for (long long i = threadIdx.x; i < B; i += blockDim.x) {   // 64-bit: i + 256 passes INT_MAX at B near it
    if (i >= Bl) {
      if (dyhat) dyhat[i] = 0.f;
      continue;
    }
    float e = (float)y[i] - yhat[i];
    float a = tau * e, b = (tau - 1.f) * e;
    s += fmaxf(a, b);
    if (dyhat) {
      // torch.maximum backward: ties split the gradient evenly
      float d = (a > b) ? -tau : ((a < b) ? (1.f - tau) : 0.5f * (1.f - 2.f * tau));
      dyhat[i] = grad_scale * d / (float)Bl;
    }
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0 && loss) *loss = t / (float)Bl;
  }
}

// T quantile levels, passed by value (a captured graph keeps them)
struct Taus {
  float v[PERT_MAX_QUANTILES];
};

// pinball loss over [B, T] (pert_pinball_loss_q): loss = mean over the B*T terms, element i = b*T + t at level t; the
// terms, the tie rule and the reduction are k_pinball's.  Ghost graphs (b >= live[1]) get dyhat = 0 in every column.
__global__ void k_pinball_q(const int64_t* __restrict__ y, const float* __restrict__ yhat, Taus taus, int T, int B,
                            float grad_scale, float* __restrict__ loss, float* __restrict__ dyhat,
                            const long long* __restrict__ live) {
  __shared__ float red[32];
  const int Bl = live ? (int)min((long long)B, live[1]) : B;
  const long long n = (long long)B * T, nl = (long long)Bl * T;
  const float inv = (float)nl;
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    if (i >= nl) {
      if (dyhat) dyhat[i] = 0.f;
      continue;
    }
    const long long b = i / T;
    const int lt = (int)(i - b * T);
    float tau = taus.v[0];
#pragma unroll
    for (int t = 1; t < PERT_MAX_QUANTILES; ++t)   // select, not index: the levels stay in parameter space
      if (t == lt) tau = taus.v[t];
    float e = (float)y[b] - yhat[i];
    float a = tau * e, c = (tau - 1.f) * e;
    s += fmaxf(a, c);
    if (dyhat) {
      float d = (a > c) ? -tau : ((a < c) ? (1.f - tau) : 0.5f * (1.f - 2.f * tau));
      dyhat[i] = grad_scale * d / inv;
    }
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0 && loss) *loss = t / inv;
  }
}

// torch.optim.Adam over one flat buffer (adam_elem, common.cuh)
__global__ void k_adam(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                       float* __restrict__ v, long long n, float b1, float b2, float eps, float wd, float step_size,
                       float bc2_sqrt, float grad_scale) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float pi = p[i], mi = m[i], vi = v[i];
  adam_elem(g[i], pi, mi, vi, grad_scale, wd, b1, b2, eps, step_size, bc2_sqrt);
  m[i] = mi;
  v[i] = vi;
  p[i] = pi;
}

inline bool al16(const void* p) { return p == nullptr || ((uintptr_t)p & 15) == 0; }

}  // namespace


// ---- eval metrics (reference pert_gnn.py:284-289, :249): block sums in double, one atomic per block and metric
__global__ void __launch_bounds__(256) k_eval_metrics(const int64_t* __restrict__ y, const float* __restrict__ yhat,
                                                      float tau, int B, double* __restrict__ acc,
                                                      const long long* __restrict__ live) {
  if (live) B = (int)min((long long)B, live[1]);   // padded batch: the real graphs only
  double mae = 0.0, mape = 0.0, q = 0.0;
  for (long long b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    const float yt = (float)y[b];                 // y.float() / int64 -> float32 promotion of the reference
    const float e = yt - yhat[b];
    const float ae = fabsf(yhat[b] - yt);
    mae += (double)ae;
    mape += (double)(ae / yt);
    q += (double)fmaxf(tau * e, (tau - 1.0f) * e);
  }
  __shared__ double red[3][8];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    mae += __shfl_xor_sync(0xffffffffu, mae, off);
    mape += __shfl_xor_sync(0xffffffffu, mape, off);
    q += __shfl_xor_sync(0xffffffffu, q, off);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = mae; red[1][w] = mape; red[2][w] = q; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
    atomicAdd(acc + threadIdx.x, t);
  }
}

// ---- eval metrics of T quantile levels (pert_eval_metrics_q): per level the sums of k_eval_metrics (same arithmetic)
// and the coverage count, then the count of graphs whose levels cross.  TM (1, 2, 4, 8) bounds T.
template <int TM>
__global__ void __launch_bounds__(256) k_eval_metrics_q(const int64_t* __restrict__ y, const float* __restrict__ yhat,
                                                        Taus taus, int T_, int B, double* __restrict__ acc,
                                                        const long long* __restrict__ live) {
  constexpr int NV = 4 * TM + 1;
  const int T = TM == 1 ? 1 : T_;
  if (live) B = (int)min((long long)B, live[1]);
  double v[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) v[k] = 0.0;
  for (long long b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    const float yt = (float)y[b];
    float prev = 0.f;
    bool cross = false;
#pragma unroll
    for (int t = 0; t < TM; ++t) {
      if (t >= T) continue;
      const float yh = yhat[b * T + t];
      const float tau = taus.v[t];
      const float e = yt - yh;
      const float ae = fabsf(yh - yt);
      v[4 * t + 0] += (double)ae;
      v[4 * t + 1] += (double)(ae / yt);
      v[4 * t + 2] += (double)fmaxf(tau * e, (tau - 1.0f) * e);
      v[4 * t + 3] += yt <= yh ? 1.0 : 0.0;
      if (t > 0 && prev > yh) cross = true;
      prev = yh;
    }
    v[4 * TM] += cross ? 1.0 : 0.0;
  }
  __shared__ double red[NV][8];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], off);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) red[k][w] = v[k];
  }
  __syncthreads();
  // value k of the 4T + 1: level sums at 4t + j (t < T), the crossing count last (slot 4 TM of red)
  if (threadIdx.x < 4 * T + 1) {
    const int k = threadIdx.x < 4 * T ? threadIdx.x : 4 * TM;
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[k][i];
    atomicAdd(acc + threadIdx.x, t);
  }
}

namespace {
// T in 1..PERT_MAX_QUANTILES, taus a host array of T levels in [0, 1], strictly increasing (NaN fails every test)
int load_taus(const float* taus, int T, Taus* out) {
  if (T < 1 || T > PERT_MAX_QUANTILES || !taus) return PERT_ERR_BADARG;
  memset(out, 0, sizeof(*out));
  for (int t = 0; t < T; ++t) {
    if (!(taus[t] >= 0.f && taus[t] <= 1.f)) return PERT_ERR_BADARG;
    if (t > 0 && !(taus[t] > taus[t - 1])) return PERT_ERR_BADARG;
    out->v[t] = taus[t];
  }
  return PERT_OK;
}
}  // namespace

extern "C" {

int pert_embedding_fwd(const float* table, int n_rows, const int64_t* ids, int id_stride, float* out, int ld_out,
                       long long N, int H, int accumulate, int* status, void* stream) {
  if (N < 0 || H <= 0 || H % 4 || ld_out % 4 || !table || !out || n_rows <= 0 || !al16(table) || !al16(out))
    return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  long long total = N * (H / 4);
  k_embedding_fwd<<<pert_cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(table, n_rows, ids, id_stride, out,
                                                                         ld_out, N, H, accumulate, status);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_embedding_bwd(const float* dy, int ld_dy, const int64_t* ids, int id_stride, float* dtable, int n_rows,
                       long long N, int H, void* stream) {
  if (N < 0 || H <= 0 || H % 4 || ld_dy % 4 || !dy || !dtable || !al16(dy) || !al16(dtable)) return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  long long total = ((N + EB_RUN - 1) / EB_RUN) * (H / 4);
  k_embedding_bwd<<<pert_cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(dy, ld_dy, ids, id_stride, dtable,
                                                                         n_rows, N, H);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_copy_cols(const float* x, int F, float* out, int ld_out, int col0, long long N, void* stream) {
  if (N < 0 || F < 0 || !out || col0 < 0 || col0 + F > ld_out) return PERT_ERR_BADARG;
  if (N == 0 || ld_out == col0) return PERT_OK;
  long long total = N * (ld_out - col0);
  k_copy_cols<<<pert_cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, F, out, ld_out, col0, N);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_bn_workspace_bytes(long long N, int H) {
  (void)N;
  return 2LL * H * 8 + 64;   // fp64 (sum, sum of squares) per column
}

// training != 0: batch statistics (and running-stat update when running_* given); else running statistics.
// Writes mean[H], rstd[H] (saved for backward) and y = (relu)(xhat*gamma + beta).
int pert_bn_fwd(const float* x, int ld_x, const float* gamma, const float* beta, float* running_mean,
                float* running_var, long long* num_batches_tracked, float eps, float momentum, int training,
                int relu, float* mean, float* rstd, float* y, int ld_y, long long N, int H, void* workspace,
                long long workspace_bytes, void* stream) {
  return pert_bn_fwd_ex(x, ld_x, gamma, beta, running_mean, running_var, num_batches_tracked, eps, momentum, training,
                        relu, mean, rstd, y, ld_y, N, H, workspace, workspace_bytes, 0, 0.f, nullptr, 0, nullptr,
                        stream);
}

}  // extern "C"

// The statistics half of a BatchNorm forward, shared by pert_bn_fwd_ex and the node-linear forward that applies
// BatchNorm to its input (csrc/linear_fwd.cu).  Training: *acc = the fp64 column sums / sums of squares in `workspace`
// (computed here by k_bn_partial unless stats_ready, i.e. the producer of x already left them there); the apply derives
// mean / rstd from them.  Eval: mean / rstd = the running statistics (k_bn_eval_stats), *acc = NULL.
// live != null (padded batch): the sums cover the rows below live[0] only.
int pert_bn_fwd_stats(const float* x, int ld_x, const float* running_mean, const float* running_var, float eps,
                      int training, float* mean, float* rstd, long long N, int H, void* workspace,
                      long long workspace_bytes, int stats_ready, const long long* live, cudaStream_t st,
                      double** acc) {
  *acc = nullptr;
  if (training) {
    if (!workspace || workspace_bytes < pert_bn_workspace_bytes(N, H)) return PERT_ERR_BADARG;
    int chunks = pert_cdiv(N, BN_ROWS);
    // 256 threads at every width (the kernel's launch bound): H <= 1024 gives H/4 <= 256 float4 lanes, so rl_n >= 1
    const int vpr = H / 4;
    const int threads = 256;
    const int rl_n = threads / vpr;
    if (rl_n < 1) return PERT_ERR_UNSUPPORTED;
    size_t smem = ((size_t)rl_n * H + H) * sizeof(float);
    if (smem > 48 * 1024) return PERT_ERR_UNSUPPORTED;
    if ((uintptr_t)workspace & 7) return PERT_ERR_BADARG;
    *acc = (double*)workspace;
    if (!stats_ready) {
      cudaError_t e = cudaMemsetAsync(*acc, 0, (size_t)2 * H * sizeof(double), st);
      if (e != cudaSuccess) return (int)e;
      k_bn_partial<<<chunks, threads, smem, st>>>(x, ld_x, N, H, *acc, live);
    }
  } else {
    if (!running_mean || !running_var) return PERT_ERR_BADARG;
    k_bn_eval_stats<<<pert_cdiv(H, 128), 128, 0, st>>>(running_mean, running_var, eps, H, mean, rstd);
  }
  return PERT_OK;
}

// stats_ready != 0 (training): the fp64 column sums / sums of squares already sit in `workspace` (written by the producer
// of x, csrc/tconv_tile.cu) -- only the apply pass runs.  dropout > 0 (training + ReLU): inverted dropout of the output
// with the mask of layer `drop_layer` at the device {seed, step} `drop_ctr` (see philox4x32_10 for the contract).
// live != null (training on a padded batch): the statistics count the rows below live[0]; every row is normalised.
int pert_bn_fwd_ex(const float* x, int ld_x, const float* gamma, const float* beta, float* running_mean,
                   float* running_var, long long* num_batches_tracked, float eps, float momentum, int training,
                   int relu, float* mean, float* rstd, float* y, int ld_y, long long N, int H, void* workspace,
                   long long workspace_bytes, int stats_ready, float dropout, const long long* drop_ctr,
                   int drop_layer, const long long* live, void* stream) {
  if (N < 0 || H <= 0 || H % 4 || H > 1024 || ld_x % 4 || ld_y % 4 || !x || !gamma || !beta || !mean || !rstd || !y)
    return PERT_ERR_BADARG;
  if (!al16(x) || !al16(gamma) || !al16(beta) || !al16(mean) || !al16(rstd) || !al16(y)) return PERT_ERR_BADARG;
  if (!(dropout >= 0.f && dropout <= 1.f)) return PERT_ERR_BADARG;
  const bool drop = dropout > 0.f && training;
  if (drop && (!relu || !drop_ctr || N * (H / 4) >= (1LL << 32))) return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  double* acc = nullptr;
  int rc = pert_bn_fwd_stats(x, ld_x, running_mean, running_var, eps, training, mean, rstd, N, H, workspace,
                             workspace_bytes, stats_ready, live, st, &acc);
  if (rc != PERT_OK) return rc;
  long long total = N * (H / 4);
  long long blocks = pert_cdiv(total, 256 * 4);
  if (blocks > 8LL * PERT_NUM_SMS) blocks = 8LL * PERT_NUM_SMS;
  const BnDropout dp = drop ? bn_dropout_params(dropout, drop_ctr, drop_layer) : BnDropout{nullptr, 0ull, 1.f, 0};
  auto apply = drop ? k_bn_apply<true> : k_bn_apply<false>;
  apply<<<(int)blocks, 256, (size_t)4 * H * sizeof(float), st>>>(x, ld_x, mean, rstd, gamma, beta, y, ld_y, N, H, relu,
                                                                 acc, eps, momentum,
                                                                 training ? running_mean : nullptr,
                                                                 training ? running_var : nullptr,
                                                                 training ? num_batches_tracked : nullptr, dp,
                                                                 training ? live : nullptr);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

extern "C" {

// sums: [2H] scratch (zeroed here).  dgamma/dbeta accumulate (+=).
int pert_bn_bwd(const float* dy, int ld_dy, const float* y, int ld_y, const float* x, int ld_x, const float* mean,
                const float* rstd, const float* gamma, int relu, int training, float* dx, int ld_dx, float* dgamma,
                float* dbeta, float* sums, long long N, int H, void* stream) {
  return pert_bn_bwd_ex(dy, ld_dy, y, ld_y, x, ld_x, mean, rstd, gamma, relu, 1.f, training, dx, ld_dx, dgamma, dbeta,
                        sums, N, H, nullptr, stream);
}

}  // extern "C"

// relu_scale: factor applied to the ReLU-masked gradient (1 / (1 - p) after inverted dropout, see bn_bwd_dz4);
// anything but 1 needs relu.  live != null (training on a padded batch): see k_bn_bwd_apply.
int pert_bn_bwd_ex(const float* dy, int ld_dy, const float* y, int ld_y, const float* x, int ld_x, const float* mean,
                   const float* rstd, const float* gamma, int relu, float relu_scale, int training, float* dx,
                   int ld_dx, float* dgamma, float* dbeta, float* sums, long long N, int H, const long long* live,
                   void* stream) {
  if (N < 0 || H <= 0 || H % 4 || H > 1024 || !dy || !x || !mean || !rstd || !gamma || !dx || !sums)
    return PERT_ERR_BADARG;
  if (relu && !y) return PERT_ERR_BADARG;
  if (!relu && relu_scale != 1.f) return PERT_ERR_BADARG;
  if (ld_dy % 4 || ld_x % 4 || ld_dx % 4 || (relu && ld_y % 4)) return PERT_ERR_BADARG;
  if (!al16(dy) || !al16(y) || !al16(x) || !al16(mean) || !al16(rstd) || !al16(gamma) || !al16(dx) || !al16(sums))
    return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, sizeof(float) * 2 * H, st);
  if (e != cudaSuccess) return (int)e;
  int vpr = H / 4;
  int threads = 256;
  if (threads < vpr) threads = (vpr + 31) / 32 * 32;
  int rl_n = threads / vpr;
  size_t smem = (size_t)rl_n * 2 * H * sizeof(float);
  if (smem > 48 * 1024) return PERT_ERR_UNSUPPORTED;
  if (!training) live = nullptr;
  k_bn_bwd_reduce<<<pert_cdiv(N, BN_BWD_ROWS), threads, smem, st>>>(dy, ld_dy, y, ld_y, x, ld_x, mean, rstd, N, H, relu,
                                                              relu_scale, sums, live);
  long long total = N * vpr;
  k_bn_bwd_apply<<<pert_cdiv(total, 256), 256, 0, st>>>(dy, ld_dy, y, ld_y, x, ld_x, mean, rstd, gamma, sums, dx,
                                                       ld_dx, N, H, relu, relu_scale, training, dgamma, dbeta, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

extern "C" {

// local[n] = <x_n, w_local> + b_local (optional);  pool[batch[n]] += x_n * probs[n] / pnn[n]  (pool zeroed here)
int pert_pool_fwd(const float* x, int ld, const float* probs, const float* pnn, const int64_t* batch,
                  const float* w_local, const float* b_local, float* local, float* pool, long long N, long long B,
                  int H, int* status, void* stream) {
  // an empty batch (N = 0) or pool (B = 0) may come with NULL pointers (empty tensors)
  if (N < 0 || B < 0 || (N > 0 && (!x || !probs || !pnn || !batch)) || (B > 0 && !pool) || ld % 4 || !al16(x) ||
      !al16(w_local) || !al16(pool))
    return PERT_ERR_BADARG;
  if (dispatch_h(H, [](auto, auto) { return PERT_OK; }) != PERT_OK) return PERT_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  if (B > 0) {
    cudaError_t e = cudaMemsetAsync(pool, 0, sizeof(float) * B * H, st);
    if (e != cudaSuccess) return (int)e;
  }
  if (N == 0) return PERT_OK;
  int rc = dispatch_h(H, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    long long groups = (N + POOL_ROWS - 1) / POOL_ROWS;
    long long threads = groups * LPR;
    k_pool_fwd<LPR, VPL><<<pert_cdiv(threads, 256), 256, 0, st>>>(x, ld, probs, pnn, batch, w_local, b_local, local,
                                                                 pool, N, (int)B, status);
    return PERT_OK;
  });
  if (rc) return rc;
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_pool_bwd(const float* dpool, const float* dlocal, const float* x, int ld, const float* probs,
                  const float* pnn, const int64_t* batch, const float* w_local, float* dx, int ld_dx,
                  float* dw_local, float* db_local, long long N, long long B, int H, void* stream) {
  if (N < 0 || B < 0 || (N > 0 && (!probs || !pnn || !batch || !dx)) || ld % 4 || ld_dx % 4 || !al16(dpool) ||
      !al16(x) || !al16(w_local) || !al16(dx))
    return PERT_ERR_BADARG;
  if (dlocal && (!x || !w_local)) return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  int rc = dispatch_h(H, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    long long groups = (N + POOL_ROWS - 1) / POOL_ROWS;
    long long threads = groups * LPR;
    k_pool_bwd<LPR, VPL><<<pert_cdiv(threads, 256), 256, 0, (cudaStream_t)stream>>>(
        dpool, dlocal, x, ld, probs, pnn, batch, w_local, dx, ld_dx, dw_local, db_local, N, (int)B);
    return PERT_OK;
  });
  if (rc) return rc;
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_relu_bwd(const float* y, float* dy, long long n, void* stream) {
  if (n < 0 || !y || !dy) return PERT_ERR_BADARG;
  if (n == 0) return PERT_OK;
  k_relu_bwd<<<pert_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(y, dy, n);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_pinball_loss(const int64_t* y, const float* yhat, float tau, long long B, float grad_scale, float* loss,
                      float* dyhat, void* stream) {
  return pert_pinball_loss_live(y, yhat, tau, B, grad_scale, loss, dyhat, nullptr, stream);
}

int pert_pinball_loss_live(const int64_t* y, const float* yhat, float tau, long long B, float grad_scale, float* loss,
                           float* dyhat, const long long* live, void* stream) {
  if (B <= 0 || B > INT_MAX || !y || !yhat) return PERT_ERR_BADARG;
  k_pinball<<<1, 256, 0, (cudaStream_t)stream>>>(y, yhat, tau, (int)B, grad_scale, loss, dyhat, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_pinball_loss_q(const int64_t* y, const float* yhat, const float* taus, int T, long long B, float grad_scale,
                        float* loss, float* dyhat, const long long* live, void* stream) {
  Taus tv;
  if (load_taus(taus, T, &tv)) return PERT_ERR_BADARG;
  if (T == 1) return pert_pinball_loss_live(y, yhat, tv.v[0], B, grad_scale, loss, dyhat, live, stream);
  if (B <= 0 || B > INT_MAX || !y || !yhat) return PERT_ERR_BADARG;
  k_pinball_q<<<1, 256, 0, (cudaStream_t)stream>>>(y, yhat, tv, T, (int)B, grad_scale, loss, dyhat, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                   float eps, float weight_decay, long long step, float grad_scale, void* stream) {
  if (n < 0 || step < 1 || !p || !g || !m || !v) return PERT_ERR_BADARG;
  if (n == 0) return PERT_OK;
  const PertAdamScalars s = pert_adam_scalars(lr, beta1, beta2, step);
  k_adam<<<pert_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, beta1, beta2, eps, weight_decay,
                                                             s.step_size, s.bc2_sqrt, grad_scale);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_eval_metrics(const int64_t* y, const float* yhat, float tau, long long B, double* acc, void* stream) {
  return pert_eval_metrics_live(y, yhat, tau, B, acc, nullptr, stream);
}

int pert_eval_metrics_live(const int64_t* y, const float* yhat, float tau, long long B, double* acc,
                           const long long* live, void* stream) {
  if (B < 0 || B > INT_MAX || !y || !yhat || !acc) return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  int grid = pert_cdiv(B, 256);
  if (grid > 64) grid = 64;
  k_eval_metrics<<<grid, 256, 0, (cudaStream_t)stream>>>(y, yhat, tau, (int)B, acc, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_eval_metrics_q(const int64_t* y, const float* yhat, const float* taus, int T, long long B, double* acc,
                        const long long* live, void* stream) {
  Taus tv;
  if (load_taus(taus, T, &tv)) return PERT_ERR_BADARG;
  if (B < 0 || B > INT_MAX || !y || !yhat || !acc) return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  int grid = pert_cdiv(B, 256);
  if (grid > 64) grid = 64;
  cudaStream_t st = (cudaStream_t)stream;
  if (T == 1) k_eval_metrics_q<1><<<grid, 256, 0, st>>>(y, yhat, tv, T, (int)B, acc, live);
  else if (T == 2) k_eval_metrics_q<2><<<grid, 256, 0, st>>>(y, yhat, tv, T, (int)B, acc, live);
  else if (T <= 4) k_eval_metrics_q<4><<<grid, 256, 0, st>>>(y, yhat, tv, T, (int)B, acc, live);
  else k_eval_metrics_q<8><<<grid, 256, 0, st>>>(y, yhat, tv, T, (int)B, acc, live);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
