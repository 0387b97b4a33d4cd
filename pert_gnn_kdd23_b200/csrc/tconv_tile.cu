// Shared-memory-staged variant of the fused TransformerConv kernels (see tconv.cu for the math).
//
// Why: the per-row gather kernels are bound by L2->SM traffic, latency and instruction issue, not by HBM: every
// k/v row is fetched once per out-edge (~3x), L1 catches only ~35-50 % of that, and the predicated 4-edge register
// blocks cost 19 M instructions per launch at cfg2 (r1 ncu: 70 % of issue cycles without an eligible warp, DRAM at
// 10 % with bytes == algorithmic bytes).  Batched call graphs are graph-major: all neighbours of a node live within a
// few hundred rows of it.  So a CTA takes a TILE of consecutive nodes, pulls the tile's two operand planes (k and v
// forward / target pass, g and q in the source pass -- contiguous in the plane layout) into shared memory with two
// TMA bulk copies (cp.async.bulk + mbarrier complete_tx: no per-thread loads, no register staging), stages the
// tile's CSR (or CSC) index slices and per-edge scalars next to them, and walks each node's edges one by one
// against shared memory (~30-cycle latency, 32-bit addressing, no padding slots), with the one remaining global
// gather (the interface-table row) prefetched one edge ahead.  Each operand row is read from L2/HBM once per tile;
// neighbours outside the tile (a graph cut by a tile boundary, graphs larger than a tile) fall back to the global
// gather.  Same semantics, same outputs as tconv.cu.
//
// Tile size (nodes) is chosen by the host so that two CTAs of 512 threads fit one SM; when the batch holds equally
// sized graphs the tile is a whole number of graphs (no cut edges).
#include "common.cuh"
#include <type_traits>

namespace {

// CTA size: 512 threads when two CTAs share an SM (tiles <= ~113 KB), 1024 when a tile needs the whole SM's shared memory
// (the same 32 resident warps per SM either way; 64 registers per thread in both)

// ---------------------------------------------------------------- mbarrier / bulk-copy PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
  } while (!ok);
}
// global -> shared bulk copy (TMA, 1-D): dst/src 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct TileArgs {
  const float *q, *k, *v, *s;   // planes, dense rows (ld == H)
  const float* g;               // backward: dL/dout, dense rows
  const int *rowptr, *csr_src, *csr_if, *csr_rpc;
  const int *colptr, *csc_pos, *csc_dst;
  const float *t_if, *t_rpc;
  int n_rpc;
  float* out;       // fwd: out rows; bwd_dst: dq rows (dense)
  float *dk, *dv;   // bwd_src
  float* alpha;     // fwd: written; bwd: read
  float* dsp;       // bwd_dst: written; bwd_src: read
  float *dt_if, *dt_rpc;
  double* bn_acc;   // fwd: optional [2][H] column sums / sums of squares of `out` (BatchNorm statistics), +=
  const long long* live;   // fwd, padded batch: bn_acc counts the nodes below live[0] only (null: all N)
  float* rpc_ws;    // [N][2][RPC_FAST] per-target sums over in-edges of (alpha, ds) by rpc type, or null (see bwd_src)
  int N, tile_nodes, edge_cap;
  int hot_if;          // interface id whose table-gradient row is accumulated per CTA instead of per edge (source pass)
  float inv_sqrt_c;
};

// Gradient of the (tiny, hot) rpc-type table without per-edge atomics: for an edge t -> i of rpc type b the table row
// receives de = alpha_t g_i + ds_t q_i, so  dT_rpc[b] = sum_i (A_ib g_i + S_ib q_i)  with the per-target scalars
// A_ib = sum_{t in in(i), rpc(t)=b} alpha_t and S_ib likewise over ds_t.  The target pass accumulates A, S in the lanes
// (lane b of the node's group owns type b) and writes 2 x RPC_FAST floats per node; the source pass -- which has the
// g and q tiles in shared memory anyway -- finishes with a [RPC_FAST x T] x [T x H] product per tile.  With the
// per-edge shared-memory atomics the source pass took 52 us at the BASELINE cfg2 shape, without them 28 us.
constexpr int RPC_FAST = 8;   // fast path for n_rpc <= 8 (the reference data has a handful of rpc types)

// dynamic smem layout shared by the three kernels (NA per-edge 4-byte arrays, kernel specific):
//   [bar 16 B][tile A: T*H][tile B: T*H][rpc table (source pass only): n_rpc*H][row/col ptr slice: T+1][NA x ecap]
// attribute ids are staged packed: interface id | rpc id << 22.  Ids that do not fit (interface id >= 2^22, rpc id >=
// 2^10) are seen while a tile is staged; that tile then ignores its staged edges and runs the global-gather variant, which
// reads the two ids separately (so any int32 interface id is right, the common tile pays one compare per edge).
#define PACK_ID(a, b) ((a) | ((b) << 22))
#define ID_IF(x) ((x) & 0x3fffff)
#define ID_RPC(x) ((int)((unsigned)(x) >> 22))
__device__ __forceinline__ bool packable(int ia, int ib) { return (unsigned)ia < (1u << 22) && (unsigned)ib < (1u << 10); }
struct Smem {
  uint64_t* bar;
  float *ta, *tb, *rpc;
  int *ptr, *e0, *e1;
  unsigned short* ord;   // node slots in descending-degree order (tile-local ids, T <= 65535)
  float *f0, *f1;
};
__device__ __forceinline__ Smem carve_smem(unsigned char* base, int T, int H, int n_rpc, int ecap) {
  Smem s;
  s.bar = reinterpret_cast<uint64_t*>(base);
  float* f = reinterpret_cast<float*>(base + 16);
  s.ta = f; f += (size_t)T * H;
  s.tb = f; f += (size_t)T * H;
  s.rpc = f; f += (size_t)n_rpc * H;
  s.ptr = reinterpret_cast<int*>(f); f += ((T + 1 + 3) / 4) * 4;
  s.ord = reinterpret_cast<unsigned short*>(f); f += ((T + 7) / 8) * 4;
  s.e0 = reinterpret_cast<int*>(f); f += ecap;
  s.e1 = reinterpret_cast<int*>(f); f += ecap;
  s.f0 = f; f += ecap;       // only the first NA arrays are backed by memory (see smem_bytes)
  s.f1 = f;
  return s;
}
static size_t smem_bytes(int T, int H, int n_rpc, int ecap, int n_edge_arrays) {
  return 16 + sizeof(float) * ((size_t)2 * T * H + (size_t)n_rpc * H + ((T + 1 + 3) / 4) * 4 + ((T + 7) / 8) * 4 +
                               (size_t)n_edge_arrays * ecap);
}

// This CTA's tile: nodes [n0, n0 + nt), tiles of tile_nodes consecutive nodes, one per CTA.  The empty asm hides where
// the two values come from.  Without it the compiler works with blockIdx.x * tile_nodes itself, and ptxas gives the
// 1024-thread forward kernels with edge attributes 228-256 bytes of spill stores instead of 156-168 (nvcc 12.9,
// -Xptxas -v).  Whether it still helps depends on the compiler: re-check those spill counts after an nvcc upgrade.
__device__ __forceinline__ void cta_tile(const TileArgs& a, int& n0, int& nt) {
  n0 = blockIdx.x * a.tile_nodes;
  nt = min(a.tile_nodes, a.N - n0);
  asm volatile("" : "+r"(n0), "+r"(nt));
}

// stage the two operand tiles + the node-pointer slice + the degree-sorted node order; returns after the pointers and
// the order are visible (tiles: the caller's mbar_wait).  The mbarrier is initialised by the caller.
// Lane groups of a warp walk their nodes' edges in lockstep (trip count = the largest degree in the warp): handing the
// nodes out in DESCENDING DEGREE order puts equal degrees side by side (no idle lockstep iterations: E[max of 2 degrees]
// is 3.8 against a mean of 3.0 at cfg2) and starts the long rows first.  Counting sort over degrees clamped to 32.
template <int H, int NT>
__device__ __forceinline__ void stage_tiles(const Smem& S, const float* pa, const float* pb, const int* nodeptr,
                                            int n0, int nt, int tid) {
  __shared__ int s_hist[34];
  if (tid == 0) {
    const uint32_t tile_bytes = (uint32_t)nt * H * 4;
    mbar_expect_tx(S.bar, 2 * tile_bytes);
    bulk_g2s(S.ta, pa + (size_t)n0 * H, tile_bytes, S.bar);
    bulk_g2s(S.tb, pb + (size_t)n0 * H, tile_bytes, S.bar);
  }
  if (tid < 34) s_hist[tid] = 0;
  for (int x = tid; x <= nt; x += NT) S.ptr[x] = __ldg(nodeptr + n0 + x);
  __syncthreads();
  for (int x = tid; x < nt; x += NT) atomicAdd(&s_hist[32 - min(S.ptr[x + 1] - S.ptr[x], 32)], 1);
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int b = 0; b < 33; ++b) {
      const int c = s_hist[b];
      s_hist[b] = run;
      run += c;
    }
  }
  __syncthreads();
  for (int x = tid; x < nt; x += NT)
    S.ord[atomicAdd(&s_hist[32 - min(S.ptr[x + 1] - S.ptr[x], 32)], 1)] = (unsigned short)x;
  __syncthreads();
}
__device__ __forceinline__ void tile_barrier_init(const Smem& S, int tid) {
  if (tid == 0) {
    mbar_init(S.bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
}

// ---------------------------------------------------------------- explicit shared-space accessors (32-bit addresses:
// keeps the compiler from falling back to generic loads + cluster-address checks inside the edge loops)
__device__ __forceinline__ float4 lds4s(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ int ldsi(uint32_t a) {
  int v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ int ldsu16(uint32_t a) {
  unsigned short v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a));
  return (int)v;
}
__device__ __forceinline__ float ldsf(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void stsf(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
template <int LPR>
__device__ __forceinline__ float gsum_full(float v) {   // butterfly inside each LPR-lane group, whole warp converged
#pragma unroll
  for (int off = LPR >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
struct SAddr {   // shared-space byte addresses of the staged arrays
  uint32_t ta, tb, rpc, ptr, ord, e0, e1, f0, f1;
};
__device__ __forceinline__ SAddr saddr_of(const Smem& S) {
  SAddr s;
  s.ta = smem_u32(S.ta); s.tb = smem_u32(S.tb); s.rpc = smem_u32(S.rpc); s.ptr = smem_u32(S.ptr);
  s.ord = smem_u32(S.ord);
  s.e0 = smem_u32(S.e0); s.e1 = smem_u32(S.e1); s.f0 = smem_u32(S.f0); s.f1 = smem_u32(S.f1);
  return s;
}

// All lane groups of a warp walk their nodes' edges in lockstep (trip count = the warp's max degree, finished groups
// contribute zeros), so shuffles use the full mask and no per-group branch divergence bookkeeping is generated.

// ============================================================== forward
// VPL = float4 vectors per lane: a node row of H = 4 * LPR * VPL floats is owned by LPR lanes, lane `lig` holding the
// float4 pieces lig, lig + LPR, ... (each piece index is contiguous across the group's lanes: conflict-free shared-memory
// rows, coalesced global rows).  VPL = 1: one warp walks 32 / LPR nodes; VPL = 2 halves the lanes per node, so a warp
// walks twice as many nodes per instruction stream (fewer instructions per edge: the per-edge bookkeeping, the shuffle
// tree and the per-node prologue / epilogue are shared by twice the data) at twice the registers per thread.
template <int LPR, int VPL, bool HAS_E, int NT>
__global__ void __launch_bounds__(NT, NT == 1024 ? 1 : 2) k_tile_fwd(TileArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  constexpr int GPC = NT / LPR;  // lane groups per CTA
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const Smem S = carve_smem(smem_raw, a.tile_nodes, H, 0, a.edge_cap);
  const SAddr sa = saddr_of(S);
  const int tid = threadIdx.x;
  const int lane = tid & 31, lig = lane % LPR, grp = lane / LPR;
  const float qscale = a.inv_sqrt_c * 1.4426950408889634f;   // logits kept in log2 units: exp(x) = 2^(x*log2 e)
  const int g0 = (tid >> 5) * GPW;          // first group slot of this warp
  float4 bsum[VPL], bsq[VPL];               // this lane's columns over its nodes (fused BatchNorm statistics)
#pragma unroll
  for (int u = 0; u < VPL; ++u) bsum[u] = bsq[u] = f4zero();
  auto ldrow = [&](const float* base, size_t row, float4 (&v)[VPL]) {
#pragma unroll
    for (int u = 0; u < VPL; ++u) v[u] = ldg4(base + row * H + (lig + u * LPR) * 4);
  };
  int n0, nt;
  cta_tile(a, n0, nt);
  if (nt <= 0) return;                         // uniform across the CTA
  tile_barrier_init(S, tid);
  stage_tiles<H, NT>(S, a.k, a.v, a.rowptr, n0, nt, tid);
  const int e_lo = S.ptr[0];
  const int ne_c = min(S.ptr[nt] - e_lo, a.edge_cap);
  int bad = 0, wide = 0;   // a staged neighbour outside this tile / staged ids that do not pack
  for (int x = tid; x < ne_c; x += NT) {
    const int nb_id = __ldg(a.csr_src + e_lo + x);
    S.e0[x] = nb_id;
    bad |= (unsigned)(nb_id - n0) >= (unsigned)nt;
    if (HAS_E) {
      const int ia = __ldg(a.csr_if + e_lo + x), ib = __ldg(a.csr_rpc + e_lo + x);
      wide |= !packable(ia, ib);
      S.e1[x] = PACK_ID(ia, ib);
    }
  }
  // fast variant of the edge loops when every edge of the tile is staged and every neighbour row is in the tile
  // (whole-graph tiles): no global-memory fallbacks are compiled into it
  // (one barrier in the common case; a second one tells unpackable ids from neighbours outside the tile)
  const bool any = __syncthreads_or(bad | wide) != 0;
  const bool narrow = !(HAS_E && any && __syncthreads_or(wide));   // else every edge takes the global path
  const int ne_s = narrow ? ne_c : 0;
  const bool all_in = !any && (S.ptr[nt] - e_lo <= a.edge_cap);
  mbar_wait(S.bar, 0);

  // node slots are handed out in descending-degree order (S.ord); the q row is requested one node ahead, the skip row
  // at the start of its own node (it is consumed after the edge loop, which hides its latency)
  int slot = g0 + grp;
  int loc = slot < nt ? ldsu16(sa.ord + slot * 2) : 0;
  float4 q_n[VPL];
#pragma unroll
  for (int u = 0; u < VPL; ++u) q_n[u] = f4zero();
  if (slot < nt) ldrow(a.q, (size_t)(n0 + loc), q_n);
  auto run = [&](auto fast_c) {
    constexpr bool FAST = decltype(fast_c)::value;
    for (; slot - grp < nt; slot += GPC) {   // warp-uniform: the warp's first group still has a node
      const bool valid = slot < nt;
      const int i = n0 + loc;
      float4 q[VPL], skip[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) {
        q[u] = f4scale(qscale, q_n[u]);
        skip[u] = f4zero();
      }
      if (valid && a.s) ldrow(a.s, (size_t)i, skip);
      const int p0 = valid ? ldsi(sa.ptr + loc * 4) : 0;
      const int p1 = valid ? ldsi(sa.ptr + loc * 4 + 4) : 0;
      if (slot + GPC < nt) {
        loc = ldsu16(sa.ord + (slot + GPC) * 2);
        ldrow(a.q, (size_t)(n0 + loc), q_n);
      }
      const int deg = p1 - p0;
      const int degmax = __reduce_max_sync(0xffffffffu, deg);
      float4 acc[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) acc[u] = f4zero();
      float m = -INFINITY, Z = 0.f;
      // software pipeline over edges: ids + table rows of edge t+1 are requested before edge t is consumed
      int j = n0;
      float4 eif[VPL], erp[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) eif[u] = erp[u] = f4zero();
      auto fetch = [&](int p, bool on) {
        j = n0;
        int ia = 0, ib = 0;
        if (on) {
          const int le = p - e_lo;
          if (FAST || le < ne_s) {
            j = ldsi(sa.e0 + le * 4);
            if (HAS_E) {
              const int id = ldsi(sa.e1 + le * 4);
              ia = ID_IF(id);
              ib = ID_RPC(id);
            }
          } else {
            j = __ldg(a.csr_src + p);
            if (HAS_E) {
              ia = __ldg(a.csr_if + p);
              ib = __ldg(a.csr_rpc + p);
            }
          }
        }
        if (HAS_E) {
          ldrow(a.t_if, (size_t)ia, eif);
          ldrow(a.t_rpc, (size_t)ib, erp);
        }
      };
      fetch(p0, 0 < deg);
      for (int t = 0; t < degmax; ++t) {
        const bool on = t < deg;
        const int p = p0 + t;
        const int cj = j;
        float4 e[VPL];
#pragma unroll
        for (int u = 0; u < VPL; ++u) e[u] = f4add(eif[u], erp[u]);
        fetch(p + 1, t + 1 < deg);
        float4 kk[VPL], vv[VPL];
        const unsigned sl = (unsigned)(cj - n0);
        if (FAST || sl < (unsigned)nt) {
#pragma unroll
          for (int u = 0; u < VPL; ++u) {
            kk[u] = lds4s(sa.ta + sl * (H * 4) + (lig + u * LPR) * 16);
            vv[u] = lds4s(sa.tb + sl * (H * 4) + (lig + u * LPR) * 16);
          }
        } else {
          ldrow(a.k, (size_t)cj, kk);
          ldrow(a.v, (size_t)cj, vv);
        }
        float part = 0.f;
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          if (HAS_E) {
            kk[u] = f4add(kk[u], e[u]);
            vv[u] = f4add(vv[u], e[u]);
          }
          part += f4dot(q[u], kk[u]);
        }
        const float s = gsum_full<LPR>(part);
        if (on && lig == 0) {
          const int le = p - e_lo;
          if (FAST || le < ne_s) stsf(sa.f0 + le * 4, s);
          else a.alpha[p] = s;
        }
        const float mn = on ? fmaxf(m, s) : m;
        const float sc = on ? ex2(m - mn) : 1.f;
        const float pz = on ? ex2(s - mn) : 0.f;
        Z = fmaf(Z, sc, pz);
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          acc[u].x = fmaf(pz, vv[u].x, acc[u].x * sc);
          acc[u].y = fmaf(pz, vv[u].y, acc[u].y * sc);
          acc[u].z = fmaf(pz, vv[u].z, acc[u].z * sc);
          acc[u].w = fmaf(pz, vv[u].w, acc[u].w * sc);
        }
        m = mn;
      }
      const float invZ = 1.0f / (Z + 1e-16f);
      if (valid) {
        // padded batch: only the real nodes (below live[0]) enter the statistics.  Read per node, not kept in a
        // register across the edge loop (a volatile load is not hoisted; it hits L1 after the first node)
        const bool counted = !a.live || i < *reinterpret_cast<const volatile long long*>(a.live);
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          const float4 o = f4add(f4scale(invZ, acc[u]), skip[u]);
          st4(a.out + (size_t)i * H + (lig + u * LPR) * 4, o);
          if (!counted) continue;
          bsum[u] = f4add(bsum[u], o);
          bsq[u].x = fmaf(o.x, o.x, bsq[u].x); bsq[u].y = fmaf(o.y, o.y, bsq[u].y);
          bsq[u].z = fmaf(o.z, o.z, bsq[u].z); bsq[u].w = fmaf(o.w, o.w, bsq[u].w);
        }
      }
      __syncwarp();
      for (int p = p0 + lig; p < p1; p += LPR) {
        const int le = p - e_lo;
        const float s = (FAST || le < ne_s) ? ldsf(sa.f0 + le * 4) : a.alpha[p];
        a.alpha[p] = ex2(s - m) * invZ;
      }
    }
  };
  if (all_in) run(std::true_type{});
  else run(std::false_type{});
  if (a.bn_acc) {
    // BatchNorm statistics of this layer's output, fused: column sums and sums of squares over the CTA's tile (per-lane
    // fp32 partials, combined in fp64) -> one fp64 atomic per column and CTA into bn_acc, the accumulator k_bn_apply
    // derives mean / rstd from (nodeops.cu).  Saves the separate statistics pass over `out`.
    __syncthreads();                                   // every warp is done with the staged tiles
    double* sc = reinterpret_cast<double*>(S.ta);
    for (int x = tid; x < 2 * H; x += NT) sc[x] = 0.0;
    __syncthreads();
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      float vals[8] = {bsum[u].x, bsum[u].y, bsum[u].z, bsum[u].w, bsq[u].x, bsq[u].y, bsq[u].z, bsq[u].w};
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        float v = vals[kk];
#pragma unroll
        for (int off = LPR; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);   // the warp's groups
        if (grp == 0) atomicAdd(&sc[(kk < 4 ? 0 : H) + (lig + u * LPR) * 4 + (kk & 3)], (double)v);
      }
    }
    __syncthreads();
    for (int x = tid; x < 2 * H; x += NT)
      if (sc[x] != 0.0) atomicAdd(a.bn_acc + x, sc[x]);
  }
}

// ============================================================== backward, target pass (dq, ds)
template <int LPR, int VPL, bool HAS_E, int NT>
__global__ void __launch_bounds__(NT, NT == 1024 ? 1 : 2) k_tile_bwd_dst(TileArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int GPC = NT / LPR;
  const Smem S = carve_smem(smem_raw, a.tile_nodes, H, 0, a.edge_cap);
  const SAddr sa = saddr_of(S);
  const int tid = threadIdx.x;
  const int lane = tid & 31, lig = lane % LPR, grp = lane / LPR;
  const int g0 = (tid >> 5) * GPW;
  auto ldrow = [&](const float* base, size_t row, float4 (&v)[VPL]) {
#pragma unroll
    for (int u = 0; u < VPL; ++u) v[u] = ldg4(base + row * H + (lig + u * LPR) * 4);
  };
  int n0, nt;
  cta_tile(a, n0, nt);
  if (nt <= 0) return;                         // uniform across the CTA
  tile_barrier_init(S, tid);
  stage_tiles<H, NT>(S, a.k, a.v, a.rowptr, n0, nt, tid);
  const int e_lo = S.ptr[0];
  const int ne_c = min(S.ptr[nt] - e_lo, a.edge_cap);
  int bad = 0, wide = 0;   // a staged neighbour outside this tile / staged ids that do not pack
  for (int x = tid; x < ne_c; x += NT) {
    const int nb_id = __ldg(a.csr_src + e_lo + x);
    S.e0[x] = nb_id;
    bad |= (unsigned)(nb_id - n0) >= (unsigned)nt;
    S.f0[x] = __ldg(a.alpha + e_lo + x);
    if (HAS_E) {
      const int ia = __ldg(a.csr_if + e_lo + x), ib = __ldg(a.csr_rpc + e_lo + x);
      wide |= !packable(ia, ib);
      S.e1[x] = PACK_ID(ia, ib);
    }
  }
  // fast variant of the edge loops when every edge of the tile is staged and every neighbour row is in the tile
  // (whole-graph tiles): no global-memory fallbacks are compiled into it
  // (one barrier in the common case; a second one tells unpackable ids from neighbours outside the tile)
  const bool any = __syncthreads_or(bad | wide) != 0;
  const bool narrow = !(HAS_E && any && __syncthreads_or(wide));   // else every edge takes the global path
  const int ne_s = narrow ? ne_c : 0;
  const bool all_in = !any && (S.ptr[nt] - e_lo <= a.edge_cap);
  mbar_wait(S.bar, 0);

  int slot = g0 + grp;
  int loc = slot < nt ? ldsu16(sa.ord + slot * 2) : 0;
  float4 g_n[VPL];
#pragma unroll
  for (int u = 0; u < VPL; ++u) g_n[u] = f4zero();
  if (slot < nt) ldrow(a.g, (size_t)(n0 + loc), g_n);
  auto run = [&](auto fast_c) {
    constexpr bool FAST = decltype(fast_c)::value;
    for (; slot - grp < nt; slot += GPC) {
      const bool valid = slot < nt;
      const int i = n0 + loc;
      float4 g[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) g[u] = g_n[u];
      const int p0 = valid ? ldsi(sa.ptr + loc * 4) : 0;
      const int p1 = valid ? ldsi(sa.ptr + loc * 4 + 4) : 0;
      if (slot + GPC < nt) {
        loc = ldsu16(sa.ord + (slot + GPC) * 2);
        ldrow(a.g, (size_t)(n0 + loc), g_n);
      }
      const int deg = p1 - p0;
      const int degmax = __reduce_max_sync(0xffffffffu, deg);
      // one edge record: source row offsets + e = T_if[a] + T_rpc[b]
      auto edge = [&](int p, bool on, int& j, float& al, float4 (&e)[VPL], int& rid) {
        j = n0;
        al = 0.f;
        int ia = 0, ib = 0;
        if (on) {
          const int le = p - e_lo;
          if (FAST || le < ne_s) {
            j = ldsi(sa.e0 + le * 4);
            al = ldsf(sa.f0 + le * 4);
            if (HAS_E) {
              const int id = ldsi(sa.e1 + le * 4);
              ia = ID_IF(id);
              ib = ID_RPC(id);
            }
          } else {
            j = __ldg(a.csr_src + p);
            al = __ldg(a.alpha + p);
            if (HAS_E) {
              ia = __ldg(a.csr_if + p);
              ib = __ldg(a.csr_rpc + p);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          e[u] = f4zero();
          if (HAS_E)
            e[u] = f4add(ldg4(a.t_if + (size_t)ia * H + (lig + u * LPR) * 4),
                         ldg4(a.t_rpc + ib * H + (lig + u * LPR) * 4));
        }
        rid = ib;
      };
      // ONE pass over the in-edges.  With d_t = <g_i, v_j + e_t> (shifted by the first edge's value c, which cancels
      // exactly: sum_t ds_t = 0), w_t = alpha_t (d_t - c) and dot = sum_t w_t:
      //   ds_t = alpha_t (d_t - c - dot) / sqrt(C)
      //   dq_i = sum_t ds_t (k_j + e_t) = (P - dot Q) / sqrt(C),   P = sum_t w_t (k_j + e_t),  Q = sum_t alpha_t (k_j + e_t)
      // so k_j, v_j and the table rows of an edge are fetched once (the two-pass form fetched the edge record and
      // its table rows twice); ds_t is written by a scalar post-pass with the lanes spread over the node's edges.
      float dot = 0.f, c_shift = 0.f;
      float4 P[VPL], Q[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) P[u] = Q[u] = f4zero();
      float sumA = 0.f, sumW = 0.f;          // lane b: sums of alpha / w over this node's in-edges of rpc type b
      for (int t = 0; t < degmax; ++t) {
        const bool on = t < deg;
        const int p = p0 + t;
        int j, rid;
        float al;
        float4 e[VPL];
        edge(p, on, j, al, e, rid);
        float4 kk[VPL], vv[VPL];
        const unsigned sl = (unsigned)(j - n0);
        if (FAST || sl < (unsigned)nt) {
#pragma unroll
          for (int u = 0; u < VPL; ++u) {
            kk[u] = lds4s(sa.ta + sl * (H * 4) + (lig + u * LPR) * 16);
            vv[u] = lds4s(sa.tb + sl * (H * 4) + (lig + u * LPR) * 16);
          }
        } else {
          ldrow(a.k, (size_t)j, kk);
          ldrow(a.v, (size_t)j, vv);
        }
        float part = 0.f;
#pragma unroll
        for (int u = 0; u < VPL; ++u) part += f4dot(g[u], f4add(vv[u], e[u]));
        const float da = gsum_full<LPR>(part);
        if (t == 0) c_shift = da;
        const float dc = da - c_shift;
        const float w = al * dc;             // alpha is 0 on finished groups
        dot += w;
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          const float4 ke = f4add(kk[u], e[u]);
          P[u] = f4fma(w, ke, P[u]);
          Q[u] = f4fma(al, ke, Q[u]);
        }
        if (HAS_E && on && lig == rid) { sumA += al; sumW += w; }
        if (on && lig == 0) {
          const int le = p - e_lo;
          if (FAST || le < ne_s) stsf(sa.f1 + le * 4, dc);
          else a.dsp[p] = dc;
        }
      }
      const float sumS = (sumW - dot * sumA) * a.inv_sqrt_c;
      __syncwarp();
      for (int p = p0 + lig; p < p1; p += LPR) {
        const int le = p - e_lo;
        const float dc = (FAST || le < ne_s) ? ldsf(sa.f1 + le * 4) : a.dsp[p];
        const float al = (FAST || le < ne_s) ? ldsf(sa.f0 + le * 4) : __ldg(a.alpha + p);
        a.dsp[p] = al * (dc - dot) * a.inv_sqrt_c;
      }
      if (valid) {
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          float4 dq;
          dq.x = (P[u].x - dot * Q[u].x) * a.inv_sqrt_c; dq.y = (P[u].y - dot * Q[u].y) * a.inv_sqrt_c;
          dq.z = (P[u].z - dot * Q[u].z) * a.inv_sqrt_c; dq.w = (P[u].w - dot * Q[u].w) * a.inv_sqrt_c;
          st4(a.out + (size_t)i * H + (lig + u * LPR) * 4, dq);
        }
      }
      if (HAS_E && a.rpc_ws && valid && lig < RPC_FAST) {
        a.rpc_ws[(size_t)i * 2 * RPC_FAST + lig] = sumA;
        a.rpc_ws[(size_t)i * 2 * RPC_FAST + RPC_FAST + lig] = sumS;
      }
    }
  };
  if (all_in) run(std::true_type{});
  else run(std::false_type{});
}

// ============================================================== backward, source pass (dk, dv, table grads)
template <int LPR, int VPL, bool HAS_E, int NT>
__global__ void __launch_bounds__(NT, NT == 1024 ? 1 : 2) k_tile_bwd_src(TileArgs a) {
  constexpr int H = 4 * LPR * VPL;
  constexpr int GPW = 32 / LPR;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int GPC = NT / LPR;
  const Smem S = carve_smem(smem_raw, a.tile_nodes, H, HAS_E ? a.n_rpc : 0, a.edge_cap);
  const SAddr sa = saddr_of(S);
  const int tid = threadIdx.x;
  const int lane = tid & 31, lig = lane % LPR, grp = lane / LPR;
  const int g0 = (tid >> 5) * GPW;
  float* s_drpc = S.rpc;   // privatised gradient of the rpc-type table (few hot rows), flushed once per CTA
  if (HAS_E)
    for (int x = tid; x < a.n_rpc * H; x += NT) s_drpc[x] = 0.f;
  // Interface id `hot_if` (0: what the reference writes on every chain and return edge of a PERT graph, misc.py:247,289,
  // i.e. 3 of 4 edges of real data) would serialise tens of thousands of REDG.128 on ONE 4H-byte row per layer.  Its
  // contributions stay in registers
  // and leave once per CTA (through the first row of tile A, which is dead after the edge loops: the geometry of cfg2
  // fits its 200-node graphs into a two-CTA tile with less than 256 bytes to spare).
  float4 hot[VPL];
#pragma unroll
  for (int u = 0; u < VPL; ++u) hot[u] = f4zero();
  int n0, nt;
  cta_tile(a, n0, nt);
  if (nt <= 0) return;                         // uniform across the CTA
  tile_barrier_init(S, tid);
  stage_tiles<H, NT>(S, a.g, a.q, a.colptr, n0, nt, tid);   // targets of a node's out-edges live in the same graph
  const int c_lo = S.ptr[0];
  const int ne_c = min(S.ptr[nt] - c_lo, a.edge_cap);
  // per out-edge (CSC order): target, and through the CSR slot its alpha, ds and attribute ids
  int bad = 0, wide = 0;   // a staged neighbour outside this tile / staged ids that do not pack
  for (int x = tid; x < ne_c; x += NT) {
    const int p = __ldg(a.csc_pos + c_lo + x);
    const int nb_id = __ldg(a.csc_dst + c_lo + x);
    S.e0[x] = nb_id;
    bad |= (unsigned)(nb_id - n0) >= (unsigned)nt;
    S.f0[x] = __ldg(a.alpha + p);
    S.f1[x] = __ldg(a.dsp + p);
    if (HAS_E) {
      const int ia = __ldg(a.csr_if + p), ib = __ldg(a.csr_rpc + p);
      wide |= !packable(ia, ib);
      S.e1[x] = PACK_ID(ia, ib);
    }
  }
  // fast variant of the edge loops when every edge of the tile is staged and every neighbour row is in the tile
  // (whole-graph tiles): no global-memory fallbacks are compiled into it
  // (one barrier in the common case; a second one tells unpackable ids from neighbours outside the tile)
  const bool any = __syncthreads_or(bad | wide) != 0;
  const bool narrow = !(HAS_E && any && __syncthreads_or(wide));   // else every edge takes the global path
  const int ne_s = narrow ? ne_c : 0;
  const bool all_in = !any && (S.ptr[nt] - c_lo <= a.edge_cap);
  mbar_wait(S.bar, 0);

  auto run = [&](auto fast_c) {
    constexpr bool FAST = decltype(fast_c)::value;
    for (int slot = g0 + grp; slot - grp < nt; slot += GPC) {
      const bool valid = slot < nt;
      const int loc = valid ? ldsu16(sa.ord + slot * 2) : 0;
      const int jn = n0 + loc;
      const int c0 = valid ? ldsi(sa.ptr + loc * 4) : 0;
      const int c1 = valid ? ldsi(sa.ptr + loc * 4 + 4) : 0;
      const int deg = c1 - c0;
      const int degmax = __reduce_max_sync(0xffffffffu, deg);
      float4 dk[VPL], dv[VPL];
#pragma unroll
      for (int u = 0; u < VPL; ++u) dk[u] = dv[u] = f4zero();
#pragma unroll 2
      for (int t = 0; t < degmax; ++t) {
        const bool on = t < deg;
        const int c = c0 + t;
        int i = n0, ia = 0, ib = 0;
        float al = 0.f, ds = 0.f;
        if (on) {
          const int le = c - c_lo;
          if (FAST || le < ne_s) {
            i = ldsi(sa.e0 + le * 4); al = ldsf(sa.f0 + le * 4); ds = ldsf(sa.f1 + le * 4);
            if (HAS_E) {
              const int id = ldsi(sa.e1 + le * 4);
              ia = ID_IF(id);
              ib = ID_RPC(id);
            }
          } else {
            const int p = __ldg(a.csc_pos + c);
            i = __ldg(a.csc_dst + c); al = __ldg(a.alpha + p); ds = __ldg(a.dsp + p);
            if (HAS_E) {
              ia = __ldg(a.csr_if + p);
              ib = __ldg(a.csr_rpc + p);
            }
          }
        }
        const unsigned sl = (unsigned)(i - n0);
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          float4 gi, qi;
          if (FAST || sl < (unsigned)nt) {
            gi = lds4s(sa.ta + sl * (H * 4) + (lig + u * LPR) * 16);
            qi = lds4s(sa.tb + sl * (H * 4) + (lig + u * LPR) * 16);
          } else {
            gi = ldg4(a.g + (size_t)i * H + (lig + u * LPR) * 4);
            qi = ldg4(a.q + (size_t)i * H + (lig + u * LPR) * 4);
          }
          dk[u] = f4fma(ds, qi, dk[u]);
          dv[u] = f4fma(al, gi, dv[u]);
          if (HAS_E && on) {
            const float4 de = f4fma(ds, qi, f4scale(al, gi));
            if (ia == a.hot_if) hot[u] = f4add(hot[u], de);
            else red4(a.dt_if + (size_t)ia * H + (lig + u * LPR) * 4, de);
            if (!a.rpc_ws) {                 // general path (n_rpc > RPC_FAST): privatised table, per-edge atomics
              float* prp = s_drpc + ib * H + (lig + u * LPR) * 4;
              atomicAdd(prp + 0, de.x);
              atomicAdd(prp + 1, de.y);
              atomicAdd(prp + 2, de.z);
              atomicAdd(prp + 3, de.w);
            }
          }
        }
      }
      if (valid) {
#pragma unroll
        for (int u = 0; u < VPL; ++u) {
          st4(a.dk + (size_t)jn * H + (lig + u * LPR) * 4, dk[u]);
          st4(a.dv + (size_t)jn * H + (lig + u * LPR) * 4, dv[u]);
        }
      }
    }
  };
  if (all_in) run(std::true_type{});
  else run(std::false_type{});
  if (HAS_E && a.rpc_ws) {
    // dT_rpc tile contribution: thread = (column, node slice); the per-target scalars are warp-uniform loads
    constexpr int NSL = NT / H;
    const int col = tid % H, slc = tid / H;
    float acc[RPC_FAST];
#pragma unroll
    for (int b = 0; b < RPC_FAST; ++b) acc[b] = 0.f;
#pragma unroll 2
    for (int loc = slc; loc < nt; loc += NSL) {
      const float4* wp = reinterpret_cast<const float4*>(a.rpc_ws + (size_t)(n0 + loc) * 2 * RPC_FAST);
      const float4 A0 = __ldg(wp), A1 = __ldg(wp + 1), S0 = __ldg(wp + 2), S1 = __ldg(wp + 3);
      const float gv = S.ta[(size_t)loc * H + col], qv = S.tb[(size_t)loc * H + col];
      acc[0] = fmaf(A0.x, gv, fmaf(S0.x, qv, acc[0])); acc[1] = fmaf(A0.y, gv, fmaf(S0.y, qv, acc[1]));
      acc[2] = fmaf(A0.z, gv, fmaf(S0.z, qv, acc[2])); acc[3] = fmaf(A0.w, gv, fmaf(S0.w, qv, acc[3]));
      acc[4] = fmaf(A1.x, gv, fmaf(S1.x, qv, acc[4])); acc[5] = fmaf(A1.y, gv, fmaf(S1.y, qv, acc[5]));
      acc[6] = fmaf(A1.z, gv, fmaf(S1.z, qv, acc[6])); acc[7] = fmaf(A1.w, gv, fmaf(S1.w, qv, acc[7]));
    }
#pragma unroll
    for (int b = 0; b < RPC_FAST; ++b)
      if (b < a.n_rpc && acc[b] != 0.f) atomicAdd(s_drpc + b * H + col, acc[b]);
  }
  if (HAS_E) {
    __syncthreads();                       // every warp is done with the staged tiles
    float* s_hot = S.ta;
    for (int x = tid; x < H; x += NT) s_hot[x] = 0.f;
    __syncthreads();
#pragma unroll
    for (int u = 0; u < VPL; ++u) {
      float* hp = s_hot + (lig + u * LPR) * 4;
      if (hot[u].x != 0.f) atomicAdd(hp + 0, hot[u].x);
      if (hot[u].y != 0.f) atomicAdd(hp + 1, hot[u].y);
      if (hot[u].z != 0.f) atomicAdd(hp + 2, hot[u].z);
      if (hot[u].w != 0.f) atomicAdd(hp + 3, hot[u].w);
    }
    __syncthreads();
    for (int x = tid; x < a.n_rpc * H; x += NT) {
      const float v = s_drpc[x];
      if (v != 0.f) atomicAdd(a.dt_rpc + x, v);
    }
    for (int x = tid; x < H; x += NT) {
      const float v = s_hot[x];
      if (v != 0.f) atomicAdd(a.dt_if + (size_t)a.hot_if * H + x, v);
    }
  }
}

// Tile geometry: nodes per tile (T) and staged-edge capacity (ecap) within the per-CTA shared-memory budget -- two CTAs
// per SM ((233472 / 2) - 1024 reserved each) unless the average graph does not fit, then one.  ONE geometry serves the
// three kernels of a layer (sized for the most demanding one: 4 per-edge arrays + the privatised rpc table).  Tiles are
// T consecutive nodes, one per CTA.  N % B == 0 is a hint, not a proof: should the graphs differ after all, the tiles
// cut some of them and those CTAs run the global-gather variant of the edge loops (same results, slower).
struct TileGeom {
  int T, ecap;
};
// Room kept for the kernels' static shared memory (s_hist[34]: 136 B).  T, ecap and the CTAs per SM depend on this
// value, and with them the order of every tile sum, so it is not tightened to the bytes in use.
constexpr int STATIC_SMEM = 160;
TileGeom tile_geom(int H, int n_rpc, long long N, long long E, long long B) {
  const double budget2 = 115712.0 - STATIC_SMEM, budget1 = 231424.0 - STATIC_SMEM;
  const double deg = N > 0 ? (double)E / (double)N : 1.0;
  const double per_node = 4.0 * (2.0 * H + 1.0 + 0.5 + 4.0 * deg);
  const double fixed = 64.0 + 4.0 * n_rpc * H + 4.0 * 4.0 * 12.0;
  auto fit = [&](double b) { return (long long)((b - fixed) / per_node); };
  long long T = fit(budget2);
  const double avg = B > 0 ? (double)N / (double)B : 0.0;
  const bool uniform = B > 0 && N % B == 0;                 // equally sized graphs (a hint, see above)
  // two CTAs per SM when the graphs fit such a tile (exactly, if they are uniform; comfortably -- average <= 60 % of the
  // tile -- if their sizes vary: larger ones would be cut); else whole-SM tiles that pack one or two graphs
  const bool two = T >= 64 && (avg == 0.0 || (uniform ? avg <= (double)T : avg <= 0.6 * (double)T));
  if (!two) T = fit(budget1);
  if (uniform && avg <= (double)T) T = T / (N / B) * (N / B);   // fixed tiles hold whole graphs
  if (T > N) T = N;
  if (T > 65535) T = 65535;
  if (T < 1) T = 1;
  int ecap = (int)(deg * (double)T + 0.999) + 8;
  ecap = (ecap + 3) / 4 * 4;
  return TileGeom{(int)T, ecap};
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e == cudaSuccess ? 0 : (int)e;
}

// grid + tile fields of a launch: one T-node tile per CTA.  Returns the CTAs per SM the shared-memory footprint allows
// (2 -> 512-thread CTAs, 256 for the VPL = 2 forward; 1 -> 1024-thread CTAs).
int plan_launch(TileArgs& a, const TileGeom& g, size_t bytes, long long N, int& grid) {
  a.tile_nodes = g.T;
  a.edge_cap = g.ecap;
  grid = pert_cdiv(N, g.T);
  return bytes + STATIC_SMEM + 1024 <= 233472 / 2 ? 2 : 1;
}

template <typename K>
int launch_k(K kernel, int grid, int threads, size_t bytes, const TileArgs& a, cudaStream_t st) {
  int rc = set_smem(kernel, bytes);
  if (rc) return rc;
  kernel<<<grid, threads, bytes, st>>>(a);
  return PERT_OK;
}

// forward launch for row width H: the VPL = 2 variant (LPR = H / 8 lanes per node, 256-thread CTAs with up to 128
// registers, still two CTAs per SM) when two CTAs fit an SM, else VPL = 1 with 1024-thread CTAs.
template <int H>
int launch_fwd(const TileArgs& a0, long long N, long long E, long long B, bool has_e, cudaStream_t st) {
  const TileGeom g = tile_geom(H, a0.n_rpc, N, E, B);
  const size_t bytes = smem_bytes(g.T, H, 0, g.ecap, 3);   // src, packed ids, logit staging
  TileArgs a = a0;
  int grid = 0;
  if (plan_launch(a, g, bytes, N, grid) == 2)
    return has_e ? launch_k(k_tile_fwd<H / 8, 2, true, 256>, grid, 256, bytes, a, st)
                 : launch_k(k_tile_fwd<H / 8, 2, false, 256>, grid, 256, bytes, a, st);
  return has_e ? launch_k(k_tile_fwd<H / 4, 1, true, 1024>, grid, 1024, bytes, a, st)
               : launch_k(k_tile_fwd<H / 4, 1, false, 1024>, grid, 1024, bytes, a, st);
}
// backward launches for row width H: one vector per lane (LPR = H / 4), 512-thread CTAs when two CTAs fit an SM, else
// 1024.  (The backward pair's REDG and shared-memory atomics want the resident warps more than the fewer instructions
// of two vectors per lane.)
template <int H>
int launch_bwd(const TileArgs& a0, long long N, long long E, long long B, bool has_e, cudaStream_t st) {
  const TileGeom g = tile_geom(H, a0.n_rpc, N, E, B);
  const size_t bd = smem_bytes(g.T, H, 0, g.ecap, 4);                      // src, ids, alpha, dalpha staging
  const size_t bs = smem_bytes(g.T, H, has_e ? a0.n_rpc : 0, g.ecap, 4);   // dst, ids, alpha, ds
  TileArgs ad = a0, as = a0;
  int gd = 0, gs = 0;
  const int pd = plan_launch(ad, g, bd, N, gd), ps = plan_launch(as, g, bs, N, gs);
  constexpr int L1 = H / 4;
  // per-target rpc sums (see RPC_FAST) live in caller scratch; without it the general atomics path runs
  const int nthr = ps == 2 ? 512 : 1024;
  float* ws = (has_e && a0.n_rpc <= RPC_FAST && L1 >= RPC_FAST && nthr % H == 0) ? a0.rpc_ws : nullptr;
  ad.rpc_ws = as.rpc_ws = ws;
  int rc;
  if (pd == 2)
    rc = has_e ? launch_k(k_tile_bwd_dst<L1, 1, true, 512>, gd, 512, bd, ad, st)
               : launch_k(k_tile_bwd_dst<L1, 1, false, 512>, gd, 512, bd, ad, st);
  else
    rc = has_e ? launch_k(k_tile_bwd_dst<L1, 1, true, 1024>, gd, 1024, bd, ad, st)
               : launch_k(k_tile_bwd_dst<L1, 1, false, 1024>, gd, 1024, bd, ad, st);
  if (rc) return rc;
  if (ps == 2)
    return has_e ? launch_k(k_tile_bwd_src<L1, 1, true, 512>, gs, 512, bs, as, st)
                 : launch_k(k_tile_bwd_src<L1, 1, false, 512>, gs, 512, bs, as, st);
  return has_e ? launch_k(k_tile_bwd_src<L1, 1, true, 1024>, gs, 1024, bs, as, st)
               : launch_k(k_tile_bwd_src<L1, 1, false, 1024>, gs, 1024, bs, as, st);
}

}  // namespace

// Entry points used by tconv.cu's C-ABI functions: return PERT_ERR_UNSUPPORTED when the tile path does not apply
// (width, strided planes, oversized rpc table) so the caller falls through to the per-row gather kernels.
int pert_tile_fwd(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                  const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                  int n_rpc, float* out, int ld_out, float* alpha, long long N, long long E, long long B, int H,
                  int C, double* bn_acc, const long long* live, cudaStream_t st) {
  if (ld != H || ld_out != H || (t_if && (size_t)n_rpc * H * 4 > 16 * 1024))
    return PERT_ERR_UNSUPPORTED;
  TileArgs a{};
  a.q = q; a.k = k; a.v = v; a.s = s;
  a.rowptr = rowptr; a.csr_src = csr_src; a.csr_if = csr_if; a.csr_rpc = csr_rpc;
  a.t_if = t_if; a.t_rpc = t_rpc; a.n_rpc = n_rpc; a.out = out; a.alpha = alpha; a.bn_acc = bn_acc;
  a.live = bn_acc ? live : nullptr;
  a.N = (int)N; a.inv_sqrt_c = 1.0f / sqrtf((float)C);
  switch (H) {
    case 32: return launch_fwd<32>(a, N, E, B, t_if != nullptr, st);
    case 64: return launch_fwd<64>(a, N, E, B, t_if != nullptr, st);
    case 128: return launch_fwd<128>(a, N, E, B, t_if != nullptr, st);
    default: return PERT_ERR_UNSUPPORTED;
  }
}

int pert_tile_bwd(const float* g_, int ld_g, const float* q, const float* k, const float* v, int ld, const int* rowptr,
                  const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                  const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha, float* dq, float* dk,
                  float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc, int n_rpc, long long N,
                  long long E, long long B, int H, int C, cudaStream_t st) {
  if (ld != H || ld_g != H || ld_d != H || (t_if && (size_t)n_rpc * H * 4 > 16 * 1024))
    return PERT_ERR_UNSUPPORTED;
  TileArgs a{};
  a.q = q; a.k = k; a.v = v; a.g = g_;
  a.rowptr = rowptr; a.csr_src = csr_src; a.csr_if = csr_if; a.csr_rpc = csr_rpc;
  a.colptr = colptr; a.csc_pos = csc_pos; a.csc_dst = csc_dst;
  a.t_if = t_if; a.t_rpc = t_rpc; a.n_rpc = n_rpc;
  a.out = dq; a.dk = dk; a.dv = dv; a.alpha = const_cast<float*>(alpha); a.dsp = dsp;
  a.dt_if = dt_if; a.dt_rpc = dt_rpc; a.rpc_ws = rpc_ws; a.hot_if = 0;
  a.N = (int)N; a.inv_sqrt_c = 1.0f / sqrtf((float)C);
  switch (H) {
    case 32: return launch_bwd<32>(a, N, E, B, t_if != nullptr, st);
    case 64: return launch_bwd<64>(a, N, E, B, t_if != nullptr, st);
    case 128: return launch_bwd<128>(a, N, E, B, t_if != nullptr, st);
    default: return PERT_ERR_UNSUPPORTED;
  }
}
