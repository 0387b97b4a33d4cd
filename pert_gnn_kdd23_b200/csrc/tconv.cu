// Fused TransformerConv(heads=1, edge_dim, root_weight) message passing over CSR rows.
//
// Replaces, per layer, PyG 2.4.0's __collect__ gathers, lin_edge, logits, utils.softmax
// (scatter-max + scatter-add), message and aggr='add' scatter (reference call sites
// model.py:100,104; ~30 ATen launches and ~22 passes over [E,H] temporaries, SURVEY.md 2.2
// K2..K10) with ONE launch forward and TWO launches backward, no [E,H] temporary at all.
//
// Semantics (SURVEY.md 8c), for target node i with incoming edges t (source j, ids a,b):
//   e_t = T_if[a] + T_rpc[b]                (== lin_edge(cat(if_emb[a], rpc_emb[b])): lin_edge has no bias,
//                                             so it distributes over the concat; tables are [n,H] GEMM outputs)
//   s_t = <q_i, k_j + e_t> / sqrt(H);  m_i = max_t s_t;  p_t = exp(s_t - m_i)
//   Z_i = sum_t p_t + 1e-16;  alpha_t = p_t / Z_i;  out_i = sum_t alpha_t (v_j + e_t) + r_i
// Backward (g = dL/dout):
//   dalpha_t = <g_i, v_j + e_t>;  ds_t = alpha_t (dalpha_t - sum_t' alpha_t' dalpha_t')
//   dq_i = sum_t ds_t (k_j + e_t)/sqrt(H)            (target-CSR pass)
//   dk_j = sum_t ds_t q_i/sqrt(H);  dv_j = sum_t alpha_t g_i;  de_t = alpha_t g_i + ds_t q_i/sqrt(H)
//                                                      (source-CSC pass; de_t reduced into dT_if / dT_rpc)
//
// Mapping: a group of LPR lanes owns one node row (H = 4*LPR*VPL floats, one or more float4 per
// lane, 16-byte coalesced row reads); 32/LPR nodes per warp; dot products reduce with sub-warp
// butterfly shuffles.  HBM-bound by bytes (forward 16*N*H + 12*E + 4*(N+1), SURVEY.md 8d) but
// LATENCY-bound in practice: call-graph nodes have 1-4 in-edges and every gather is a dependent
// chain rowptr -> index -> row.  The kernels therefore take a register fast path for degree <= FAST_DEG:
// all indices, then ALL neighbour rows (k, v, the two edge-table rows) are issued before the first use,
// so a node costs 3 dependent memory latencies instead of ~3 per edge per pass (r1 ncu: 50 % warps
// active, 36 % issue-active, DRAM at 10 % with bytes == algorithmic bytes).
#include "common.cuh"
#include <type_traits>

namespace {

constexpr int FAST_DEG = 4;

template <int VPL>
struct Row {
  float4 v[VPL];
};

template <int LPR, int VPL>
__device__ __forceinline__ Row<VPL> load_row(const float* __restrict__ base, int ld, int row, int lig) {
  Row<VPL> r;
  const float* p = base + (size_t)row * ld + lig * 4;
#pragma unroll
  for (int u = 0; u < VPL; ++u) r.v[u] = ldg4(p + u * LPR * 4);
  return r;
}
// predicated (branch-free) row load: @P LDG.128, zeros when !pred -- keeps all of a node's loads in one basic block
template <int LPR, int VPL>
__device__ __forceinline__ Row<VPL> load_row_if(bool pred, const float* __restrict__ base, int ld, int row, int lig) {
  Row<VPL> r;
  const float* p = base + (size_t)row * ld + lig * 4;
#pragma unroll
  for (int u = 0; u < VPL; ++u) r.v[u] = pred ? ldg4(p + u * LPR * 4) : f4zero();
  return r;
}
template <int LPR, int VPL>
__device__ __forceinline__ void store_row(float* __restrict__ base, int ld, int row, int lig, const Row<VPL>& r) {
  float* p = base + (size_t)row * ld + lig * 4;
#pragma unroll
  for (int u = 0; u < VPL; ++u) st4(p + u * LPR * 4, r.v[u]);
}
template <int VPL>
__device__ __forceinline__ Row<VPL> row_add(const Row<VPL>& a, const Row<VPL>& b) {
  Row<VPL> r;
#pragma unroll
  for (int u = 0; u < VPL; ++u) r.v[u] = f4add(a.v[u], b.v[u]);
  return r;
}
template <int VPL>
__device__ __forceinline__ float row_dot(const Row<VPL>& a, const Row<VPL>& b) {
  float s = 0.f;
#pragma unroll
  for (int u = 0; u < VPL; ++u) s += f4dot(a.v[u], b.v[u]);
  return s;
}
template <int VPL>
__device__ __forceinline__ void row_fma(float s, const Row<VPL>& a, Row<VPL>& acc) {
#pragma unroll
  for (int u = 0; u < VPL; ++u) acc.v[u] = f4fma(s, a.v[u], acc.v[u]);
}
template <int VPL>
__device__ __forceinline__ Row<VPL> row_zero() {
  Row<VPL> r;
#pragma unroll
  for (int u = 0; u < VPL; ++u) r.v[u] = f4zero();
  return r;
}

struct TconvArgs {
  const float *q, *k, *v, *s;  // node planes, row stride ld
  int ld;
  const int *rowptr, *csr_src, *csr_if, *csr_rpc;
  const float *t_if, *t_rpc;  // [n_if,H], [n_rpc,H] (may be null => no edge term)
  float* out;
  int ld_out;
  float* alpha;  // [E] CSR order
  int N;
  float inv_sqrt_c;
};

template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_tconv_fwd(TconvArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int lig = lane % LPR;
  const int grp = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (grp * LPR));
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int i = warp * GPW + grp;
  if (i >= a.N) return;
  const bool has_e = a.t_if != nullptr;
  const int p0 = __ldg(a.rowptr + i), p1 = __ldg(a.rowptr + i + 1);
  const bool staged = (p1 - p0) > FAST_DEG;   // degree > chunk: raw logits staged in alpha[], normalised at the end
  const Row<VPL> q = load_row<LPR, VPL>(a.q, a.ld, i, lig);
  const Row<VPL> skip = a.s ? load_row<LPR, VPL>(a.s, a.ld, i, lig) : row_zero<VPL>();
  // Edges are consumed in chunks of FAST_DEG: per chunk, all indices, then every neighbour row (k, v, two edge-table
  // rows) are in flight before the first use (branch-free predicated loads); chunks are merged with the online
  // softmax recurrence, so k/v/e rows are read exactly once for any degree.
  Row<VPL> acc = row_zero<VPL>();
  float m = -INFINITY, Z = 0.f;
  for (int c0 = p0; c0 < p1; c0 += FAST_DEG) {
    const int deg = p1 - c0;  // edges left (>= 1)
    int j[FAST_DEG], ia[FAST_DEG], ib[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      j[x] = on ? __ldg(a.csr_src + c0 + x) : 0;
      ia[x] = (on && has_e) ? __ldg(a.csr_if + c0 + x) : 0;
      ib[x] = (on && has_e) ? __ldg(a.csr_rpc + c0 + x) : 0;
    }
    Row<VPL> kj[FAST_DEG], vj[FAST_DEG], ei[FAST_DEG], er[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      kj[x] = load_row_if<LPR, VPL>(on, a.k, a.ld, j[x], lig);
      vj[x] = load_row_if<LPR, VPL>(on, a.v, a.ld, j[x], lig);
      ei[x] = load_row_if<LPR, VPL>(on && has_e, a.t_if, H, ia[x], lig);
      er[x] = load_row_if<LPR, VPL>(on && has_e, a.t_rpc, H, ib[x], lig);
    }
    float s[FAST_DEG];
    float m_new = m;
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const Row<VPL> e = row_add(ei[x], er[x]);
      kj[x] = row_add(kj[x], e);
      vj[x] = row_add(vj[x], e);
      s[x] = group_sum<LPR>(row_dot(q, kj[x]), gmask) * a.inv_sqrt_c;
      if (x < deg) m_new = fmaxf(m_new, s[x]);
    }
    const float scale = expf(m - m_new);   // 0 on the first chunk (m = -inf), 1 when the max did not move
    Z *= scale;
#pragma unroll
    for (int u = 0; u < VPL; ++u) acc.v[u] = f4scale(scale, acc.v[u]);
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const float pz = (x < deg) ? expf(s[x] - m_new) : 0.f;
      Z += pz;
      row_fma(pz, vj[x], acc);
      if (lig == 0 && x < deg) a.alpha[c0 + x] = staged ? s[x] : pz;   // un-normalised for now
    }
    m = m_new;
  }
  const float invZ = 1.0f / (Z + 1e-16f);   // PyG: sum(exp(s - max)) + 1e-16
#pragma unroll
  for (int u = 0; u < VPL; ++u) acc.v[u] = f4scale(invZ, acc.v[u]);
  store_row<LPR, VPL>(a.out, a.ld_out, i, lig, row_add(acc, skip));
  // normalise alpha (saved for backward)
  __syncwarp(gmask);
  for (int p = p0 + lig; p < p1; p += LPR) {
    const float v = a.alpha[p];
    a.alpha[p] = (staged ? expf(v - m) : v) * invZ;
  }
}


struct TconvBwdDstArgs {
  const float *g;   // dL/dout [N,H], row stride ld_g
  int ld_g;
  const float *q, *k, *v;
  int ld;
  const int *rowptr, *csr_src, *csr_if, *csr_rpc;
  const float *t_if, *t_rpc;
  const float* alpha;
  float* dq;  // [N,H] row stride ld_d
  int ld_d;
  float* dsp;  // [E] ds/sqrt(C), CSR order
  int N;
  float inv_sqrt_c;
};

template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_tconv_bwd_dst(TconvBwdDstArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int lig = lane % LPR;
  const int grp = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (grp * LPR));
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int i = warp * GPW + grp;
  if (i >= a.N) return;
  const bool has_e = a.t_if != nullptr;
  const int p0 = __ldg(a.rowptr + i), p1 = __ldg(a.rowptr + i + 1);
  const Row<VPL> g = load_row<LPR, VPL>(a.g, a.ld_g, i, lig);
  Row<VPL> dq = row_zero<VPL>();
  if (p1 - p0 <= FAST_DEG) {
    // ---- whole neighbourhood in registers: every k/v/e row read once, all loads in flight together
    const int deg = p1 - p0;
    int j[FAST_DEG], ia[FAST_DEG], ib[FAST_DEG];
    float al[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      j[x] = on ? __ldg(a.csr_src + p0 + x) : 0;
      al[x] = on ? __ldg(a.alpha + p0 + x) : 0.f;
      ia[x] = (on && has_e) ? __ldg(a.csr_if + p0 + x) : 0;
      ib[x] = (on && has_e) ? __ldg(a.csr_rpc + p0 + x) : 0;
    }
    Row<VPL> kj[FAST_DEG], vj[FAST_DEG], ei[FAST_DEG], er[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      kj[x] = load_row_if<LPR, VPL>(on, a.k, a.ld, j[x], lig);
      vj[x] = load_row_if<LPR, VPL>(on, a.v, a.ld, j[x], lig);
      ei[x] = load_row_if<LPR, VPL>(on && has_e, a.t_if, H, ia[x], lig);
      er[x] = load_row_if<LPR, VPL>(on && has_e, a.t_rpc, H, ib[x], lig);
    }
    float da[FAST_DEG];
    float dot = 0.f;
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const Row<VPL> e = row_add(ei[x], er[x]);
      kj[x] = row_add(kj[x], e);
      vj[x] = row_add(vj[x], e);
      da[x] = group_sum<LPR>(row_dot(g, vj[x]), gmask);
      dot = fmaf(al[x], da[x], dot);       // al = 0 beyond deg
    }
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const float ds = al[x] * (da[x] - dot) * a.inv_sqrt_c;
      row_fma(ds, kj[x], dq);
      if (lig == 0 && x < deg) a.dsp[p0 + x] = ds;
    }
    store_row<LPR, VPL>(a.dq, a.ld_d, i, lig, dq);
    return;
  }
  // ---- any degree: two chunked passes (dalpha needs the full-segment dot before ds), FAST_DEG rows in flight
  float dot = 0.f;
  for (int c0 = p0; c0 < p1; c0 += FAST_DEG) {
    const int deg = p1 - c0;
    int j[FAST_DEG], ia[FAST_DEG], ib[FAST_DEG];
    float al[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      j[x] = on ? __ldg(a.csr_src + c0 + x) : 0;
      al[x] = on ? __ldg(a.alpha + c0 + x) : 0.f;
      ia[x] = (on && has_e) ? __ldg(a.csr_if + c0 + x) : 0;
      ib[x] = (on && has_e) ? __ldg(a.csr_rpc + c0 + x) : 0;
    }
    Row<VPL> vj[FAST_DEG], ei[FAST_DEG], er[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      vj[x] = load_row_if<LPR, VPL>(on, a.v, a.ld, j[x], lig);
      ei[x] = load_row_if<LPR, VPL>(on && has_e, a.t_if, H, ia[x], lig);
      er[x] = load_row_if<LPR, VPL>(on && has_e, a.t_rpc, H, ib[x], lig);
    }
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      vj[x] = row_add(vj[x], row_add(ei[x], er[x]));
      const float da = group_sum<LPR>(row_dot(g, vj[x]), gmask);
      dot = fmaf(al[x], da, dot);
      if (lig == 0 && x < deg) a.dsp[c0 + x] = da;
    }
  }
  __syncwarp(gmask);
  for (int c0 = p0; c0 < p1; c0 += FAST_DEG) {
    const int deg = p1 - c0;
    int j[FAST_DEG], ia[FAST_DEG], ib[FAST_DEG];
    float ds[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      j[x] = on ? __ldg(a.csr_src + c0 + x) : 0;
      ds[x] = on ? __ldg(a.alpha + c0 + x) * (a.dsp[c0 + x] - dot) * a.inv_sqrt_c : 0.f;
      ia[x] = (on && has_e) ? __ldg(a.csr_if + c0 + x) : 0;
      ib[x] = (on && has_e) ? __ldg(a.csr_rpc + c0 + x) : 0;
    }
    Row<VPL> kj[FAST_DEG], ei[FAST_DEG], er[FAST_DEG];
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      const bool on = x < deg;
      kj[x] = load_row_if<LPR, VPL>(on, a.k, a.ld, j[x], lig);
      ei[x] = load_row_if<LPR, VPL>(on && has_e, a.t_if, H, ia[x], lig);
      er[x] = load_row_if<LPR, VPL>(on && has_e, a.t_rpc, H, ib[x], lig);
    }
    __syncwarp(gmask);   // all lanes have read the staged dalpha of this chunk before lane 0 overwrites it
#pragma unroll
    for (int x = 0; x < FAST_DEG; ++x) {
      kj[x] = row_add(kj[x], row_add(ei[x], er[x]));
      row_fma(ds[x], kj[x], dq);
      if (lig == 0 && x < deg) a.dsp[c0 + x] = ds[x];
    }
  }
  store_row<LPR, VPL>(a.dq, a.ld_d, i, lig, dq);
}


struct TconvBwdSrcArgs {
  const float *g;
  int ld_g;
  const float* q;
  int ld;
  const int *colptr, *csc_pos, *csc_dst, *csr_if, *csr_rpc;
  const float *alpha, *dsp;
  float *dk, *dv;  // [N,H] row stride ld_d
  int ld_d;
  float *dt_if, *dt_rpc;  // [n_if,H], [n_rpc,H] accumulated with atomics (caller zeroes); may be null
  int n_rpc;
  int N;
};

// Interface id 0 is what the reference writes on every chain and return edge of a PERT graph (3 of 4 edges).  Its
// table-gradient row is summed per thread, then per CTA, then added once per CTA, as the staged kernels do
// (tconv_tile.cu, hot_if): per-edge atomics into that one row would chain ~E fp32 additions of mixed-sign terms whose
// sum cancels ~100-fold, and serialise every edge on one address.
constexpr int HOT_IF = 0;

template <int LPR, int VPL, bool SMEM_RPC>
__device__ __forceinline__ void edge_table_grad(const TconvBwdSrcArgs& a, float* s_rpc, float al, float ds,
                                                const Row<VPL>& gi, const Row<VPL>& qi, int ia, int ib, int lig,
                                                Row<VPL>& hot) {
  constexpr int H = 4 * LPR * VPL;
  Row<VPL> de = row_zero<VPL>();
  row_fma(al, gi, de);
  row_fma(ds, qi, de);
  float* pif = a.dt_if + (size_t)ia * H + lig * 4;
#pragma unroll
  for (int u = 0; u < VPL; ++u) {
    if (ia == HOT_IF) hot.v[u] = f4add(hot.v[u], de.v[u]);
    else red4(pif + u * LPR * 4, de.v[u]);
    if (SMEM_RPC) {
      float* ps = s_rpc + ib * H + lig * 4 + u * LPR * 4;
      atomicAdd(ps + 0, de.v[u].x);
      atomicAdd(ps + 1, de.v[u].y);
      atomicAdd(ps + 2, de.v[u].z);
      atomicAdd(ps + 3, de.v[u].w);
    } else {
      red4(a.dt_rpc + (size_t)ib * H + lig * 4 + u * LPR * 4, de.v[u]);
    }
  }
}

// dynamic smem: n_rpc*H floats when the rpc-type table is privatised per CTA (few, hot rows)
template <int LPR, int VPL, bool SMEM_RPC>
__global__ void __launch_bounds__(256) k_tconv_bwd_src(TconvBwdSrcArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  extern __shared__ float s_rpc[];
  __shared__ float s_hot[H];
  const bool has_e = a.dt_if != nullptr;
  if (has_e) {
    for (int x = threadIdx.x; x < H; x += blockDim.x) s_hot[x] = 0.f;
    if (SMEM_RPC)
      for (int x = threadIdx.x; x < a.n_rpc * H; x += blockDim.x) s_rpc[x] = 0.f;
    __syncthreads();
  }
  Row<VPL> hot = row_zero<VPL>();   // this thread's part of table-gradient row HOT_IF
  const int lane = threadIdx.x & 31;
  const int lig = lane % LPR;
  const int grp = lane / LPR;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  for (int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; warp * GPW < a.N; warp += warps_total) {
    const int j = warp * GPW + grp;
    if (j >= a.N) continue;
    const int c0 = __ldg(a.colptr + j), c1 = __ldg(a.colptr + j + 1);
    Row<VPL> dk = row_zero<VPL>(), dv = row_zero<VPL>();
    for (int cc = c0; cc < c1; cc += FAST_DEG) {   // chunks of FAST_DEG out-edges, all loads of a chunk in flight
      const int deg = c1 - cc;
      int p[FAST_DEG], i[FAST_DEG];
#pragma unroll
      for (int x = 0; x < FAST_DEG; ++x) {
        const bool on = x < deg;
        p[x] = on ? __ldg(a.csc_pos + cc + x) : 0;
        i[x] = on ? __ldg(a.csc_dst + cc + x) : 0;
      }
      float al[FAST_DEG], ds[FAST_DEG];
      int ia[FAST_DEG], ib[FAST_DEG];
      Row<VPL> gi[FAST_DEG], qi[FAST_DEG];
#pragma unroll
      for (int x = 0; x < FAST_DEG; ++x) {
        const bool on = x < deg;
        al[x] = on ? __ldg(a.alpha + p[x]) : 0.f;
        ds[x] = on ? __ldg(a.dsp + p[x]) : 0.f;
        ia[x] = (on && has_e) ? __ldg(a.csr_if + p[x]) : 0;
        ib[x] = (on && has_e) ? __ldg(a.csr_rpc + p[x]) : 0;
        gi[x] = load_row_if<LPR, VPL>(on, a.g, a.ld_g, i[x], lig);
        qi[x] = load_row_if<LPR, VPL>(on, a.q, a.ld, i[x], lig);
      }
#pragma unroll
      for (int x = 0; x < FAST_DEG; ++x) {
        row_fma(ds[x], qi[x], dk);
        row_fma(al[x], gi[x], dv);
        if (has_e && x < deg)
          edge_table_grad<LPR, VPL, SMEM_RPC>(a, s_rpc, al[x], ds[x], gi[x], qi[x], ia[x], ib[x], lig, hot);
      }
    }
    store_row<LPR, VPL>(a.dk, a.ld_d, j, lig, dk);
    store_row<LPR, VPL>(a.dv, a.ld_d, j, lig, dv);
  }
  if (has_e) {
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      float* hp = s_hot + lig * 4 + u * LPR * 4;
      if (hot.v[u].x != 0.f) atomicAdd(hp + 0, hot.v[u].x);
      if (hot.v[u].y != 0.f) atomicAdd(hp + 1, hot.v[u].y);
      if (hot.v[u].z != 0.f) atomicAdd(hp + 2, hot.v[u].z);
      if (hot.v[u].w != 0.f) atomicAdd(hp + 3, hot.v[u].w);
    }
    __syncthreads();
    for (int x = threadIdx.x; x < H; x += blockDim.x) {
      const float v = s_hot[x];
      if (v != 0.f) atomicAdd(a.dt_if + (size_t)HOT_IF * H + x, v);
    }
    if (SMEM_RPC)
      for (int x = threadIdx.x; x < a.n_rpc * H; x += blockDim.x) {
        float v = s_rpc[x];
        if (v != 0.f) atomicAdd(a.dt_rpc + x, v);
      }
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

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

// shared-memory-staged kernels (tconv_tile.cu); PERT_ERR_UNSUPPORTED => use the per-row gather kernels below
int pert_tile_fwd(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                  const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                  int n_rpc, float* out, int ld_out, float* alpha, long long N, long long E, long long B, int H, int C,
                  double* bn_acc, const long long* live, cudaStream_t st);
int pert_tile_bwd(const float* g_, int ld_g, const float* q, const float* k, const float* v, int ld, const int* rowptr,
                  const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                  const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha, float* dq, float* dk,
                  float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc, int n_rpc, long long N,
                  long long E, long long B, int H, int C, const PertBnBwd* bn, cudaStream_t st);

namespace {

// argument checks shared by pert_tconv_bwd_c and pert_tconv_bwd_bn
int bwd_args_ok(const float* g, int ld_g, const float* q, const float* k, const float* v, int ld, const int* rowptr,
                const int* csr_if, const int* csr_rpc, const int* colptr, const float* t_if, const float* t_rpc,
                const float* dq, const float* dk, const float* dv, int ld_d, const float* dt_if, const float* dt_rpc,
                long long N, long long E, int H, int C) {
  if (N < 0 || E < 0 || !g || !q || !k || !v || !rowptr || !colptr || !dq || !dk || !dv || C < 1 || C > H) return 0;
  if (ld % 4 || ld_g % 4 || ld_d % 4 || !aligned16(g) || !aligned16(q) || !aligned16(k) || !aligned16(v) ||
      !aligned16(dq) || !aligned16(dk) || !aligned16(dv))
    return 0;
  if (t_if && (!t_rpc || !dt_if || !dt_rpc || !aligned16(dt_if) || !aligned16(dt_rpc))) return 0;
  if (t_if && E > 0 && (!csr_if || !csr_rpc)) return 0;   // an edgeless batch may pass null edge arrays
  return 1;
}

}  // namespace

extern "C" {

int pert_tconv_supported_width(int H) {
  return dispatch_h(H, [](auto, auto) { return 1; }) == 1 ? 1 : 0;
}

// pert_tconv_fwd_c with the BatchNorm statistics of `out` fused into the staged tile kernel (include/pertgnn.h)
int pert_tconv_fwd_stats(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                         const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if,
                         const float* t_rpc, float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E,
                         long long B_hint, int H, int C, double* bn_acc, const long long* live, int* fused,
                         void* stream) {
  *fused = 0;
  if (bn_acc && N > 0 && ld_out == H && q && k && v && rowptr && out && !(ld % 4) && aligned16(q) &&
      aligned16(k) && aligned16(v) && aligned16(out) && (!s || aligned16(s)) &&
      (!t_if || (aligned16(t_if) && t_rpc && aligned16(t_rpc) && (E == 0 || (csr_if && csr_rpc))))) {   // as _c
    int rt = pert_tile_fwd(q, k, v, s, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, n_rpc, out, ld_out, alpha, N, E,
                           B_hint, H, C, bn_acc, live, (cudaStream_t)stream);
    if (rt == PERT_OK) {
      *fused = 1;
      PERT_LAUNCH_CHECK();
      return PERT_OK;
    }
    if (rt != PERT_ERR_UNSUPPORTED) return rt;
  }
  return pert_tconv_fwd_c(q, k, v, s, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, out, ld_out, alpha, n_rpc, N,
                          E, B_hint, H, C, stream);
}

int pert_tconv_fwd(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                   const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                   float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E, long long B_hint, int H,
                   void* stream) {
  return pert_tconv_fwd_c(q, k, v, s, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, out, ld_out, alpha, n_rpc, N,
                          E, B_hint, H, H, stream);
}

int pert_tconv_fwd_c(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                     const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                     float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E, long long B_hint, int H,
                     int C, void* stream) {
  if (N < 0 || E < 0 || !q || !k || !v || !rowptr || !out || C < 1 || C > H) return PERT_ERR_BADARG;
  if (ld % 4 || ld_out % 4 || !aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(out) ||
      (s && !aligned16(s)) || (t_if && (!aligned16(t_if) || !aligned16(t_rpc) || !t_rpc)) ||
      (t_if && E > 0 && (!csr_if || !csr_rpc)))   // an edgeless batch may pass null edge arrays
    return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  if (ld_out == H) {
    int rt = pert_tile_fwd(q, k, v, s, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, n_rpc, out, ld_out, alpha, N, E,
                           B_hint, H, C, nullptr, nullptr, (cudaStream_t)stream);
    if (rt != PERT_ERR_UNSUPPORTED) {
      if (rt) return rt;
      PERT_LAUNCH_CHECK();
      return PERT_OK;
    }
  }
  TconvArgs a{q, k, v, s, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, out, ld_out, alpha, (int)N,
              1.0f / sqrtf((float)C)};
  int rc = dispatch_h(H, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    const int gpw = 32 / LPR;
    const long long warps = (N + gpw - 1) / gpw;
    k_tconv_fwd<LPR, VPL><<<pert_cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(a);
    return PERT_OK;
  });
  if (rc) return rc;
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_tconv_bwd(const float* g, int ld_g, const float* q, const float* k, const float* v, int ld,
                   const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr,
                   const int* csc_pos, const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha,
                   float* dq, float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                   int n_rpc, long long N, long long E, long long B_hint, int H, void* stream) {
  return pert_tconv_bwd_c(g, ld_g, q, k, v, ld, rowptr, csr_src, csr_if, csr_rpc, colptr, csc_pos, csc_dst, t_if, t_rpc,
                          alpha, dq, dk, dv, ld_d, dsp, rpc_ws, dt_if, dt_rpc, n_rpc, N, E, B_hint, H, H, stream);
}

int pert_tconv_bwd_c(const float* g, int ld_g, const float* q, const float* k, const float* v, int ld,
                     const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr,
                     const int* csc_pos, const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha,
                     float* dq, float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                     int n_rpc, long long N, long long E, long long B_hint, int H, int C, void* stream) {
  if (!bwd_args_ok(g, ld_g, q, k, v, ld, rowptr, csr_if, csr_rpc, colptr, t_if, t_rpc, dq, dk, dv, ld_d, dt_if, dt_rpc,
                   N, E, H, C))
    return PERT_ERR_BADARG;
  if (N == 0) return PERT_OK;
  if (ld_d == H) {
    int rt = pert_tile_bwd(g, ld_g, q, k, v, ld, rowptr, csr_src, csr_if, csr_rpc, colptr, csc_pos, csc_dst, t_if, t_rpc,
                           alpha, dq, dk, dv, ld_d, dsp, rpc_ws, dt_if, dt_rpc, n_rpc, N, E, B_hint, H, C, nullptr,
                           (cudaStream_t)stream);
    if (rt != PERT_ERR_UNSUPPORTED) {
      if (rt) return rt;
      PERT_LAUNCH_CHECK();
      return PERT_OK;
    }
  }
  const float isc = 1.0f / sqrtf((float)C);
  TconvBwdDstArgs ad{g, ld_g, q, k, v, ld, rowptr, csr_src, csr_if, csr_rpc, t_if, t_rpc, alpha, dq, ld_d, dsp,
                     (int)N, isc};
  TconvBwdSrcArgs as{g, ld_g, q, ld, colptr, csc_pos, csc_dst, csr_if, csr_rpc, alpha, dsp, dk, dv, ld_d,
                     t_if ? dt_if : nullptr, t_if ? dt_rpc : nullptr, n_rpc, (int)N};
  int rc = dispatch_h(H, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    constexpr int HH = 4 * LPR * VPL;
    const int gpw = 32 / LPR;
    const long long warps = (N + gpw - 1) / gpw;
    cudaStream_t st = (cudaStream_t)stream;
    k_tconv_bwd_dst<LPR, VPL><<<pert_cdiv(warps * 32, 256), 256, 0, st>>>(ad);
    const size_t smem = t_if ? (size_t)n_rpc * HH * sizeof(float) : 0;
    // persistent-ish grid (multiple of the SM count) so the privatised rpc table is flushed few times
    const long long blocks = (warps * 32 + 255) / 256;
    const int grid = (int)(blocks < (long long)PERT_NUM_SMS * 8 ? blocks : (long long)PERT_NUM_SMS * 8);
    if (smem > 0 && smem <= 32 * 1024)
      k_tconv_bwd_src<LPR, VPL, true><<<grid, 256, smem, st>>>(as);
    else
      k_tconv_bwd_src<LPR, VPL, false><<<grid, 256, 0, st>>>(as);
    return PERT_OK;
  });
  if (rc) return rc;
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_tconv_bwd_bn_supported(int H, int n_rpc) {
  return H == 64 && n_rpc >= 0 && (size_t)n_rpc * H * 4 <= 16 * 1024 ? 1 : 0;
}

int pert_tconv_bwd_bn(float* g, int ld_g, const float* q, const float* k, const float* v, int ld, const int* rowptr,
                      const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                      const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha, float* dq,
                      float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                      int n_rpc, long long N, long long E, long long B_hint, int H, int C, const PertBnBwd* bn,
                      void* stream) {
  if (!bwd_args_ok(g, ld_g, q, k, v, ld, rowptr, csr_if, csr_rpc, colptr, t_if, t_rpc, dq, dk, dv, ld_d, dt_if, dt_rpc,
                   N, E, H, C))
    return PERT_ERR_BADARG;
  if (!bn || !bn->dx || !bn->y || !bn->x || !bn->mean || !bn->rstd || !bn->gamma || !bn->sums || !bn->dgamma ||
      !bn->dbeta || !aligned16(bn->dx) || !aligned16(bn->y) || !aligned16(bn->x) || !aligned16(bn->mean) ||
      !aligned16(bn->rstd) || !aligned16(bn->gamma) || !aligned16(bn->sums))
    return PERT_ERR_BADARG;
  if (!pert_tconv_bwd_bn_supported(H, n_rpc) || ld != H || ld_g != H || ld_d != H) return PERT_ERR_UNSUPPORTED;
  if (N == 0) return PERT_OK;
  int rt = pert_tile_bwd(g, ld_g, q, k, v, ld, rowptr, csr_src, csr_if, csr_rpc, colptr, csc_pos, csc_dst, t_if, t_rpc,
                         alpha, dq, dk, dv, ld_d, dsp, rpc_ws, dt_if, dt_rpc, n_rpc, N, E, B_hint, H, C, bn,
                         (cudaStream_t)stream);
  if (rt) return rt;
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
