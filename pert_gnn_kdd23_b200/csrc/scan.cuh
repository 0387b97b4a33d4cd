// Device-wide inclusive scan of one or two int32 arrays in place (3 launches: tile sums, a one-CTA scan of the tile
// sums, apply).  Used by the CSR build (index.cu) and the trace grouping (tracegroup.cu).  Integer sums: exact and
// independent of scheduling.
#pragma once
#include "common.cuh"

#define SCAN_THREADS 1024
#define SCAN_ITEMS 4
#define SCAN_TILE (SCAN_THREADS * SCAN_ITEMS)

namespace {

__device__ __forceinline__ int block_scan_inclusive(int v, int* smem_warp /*32*/) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) smem_warp[w] = v;
  __syncthreads();
  if (w == 0) {
    int x = smem_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += u;
    }
    smem_warp[lane] = x;
  }
  __syncthreads();
  int base = (w == 0) ? 0 : smem_warp[w - 1];
  __syncthreads();
  return v + base;
}

// blockIdx.y selects the array
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tile_sums(const int* a0, const int* a1, int L,
                                                                  int* bsum, int nb) {
  __shared__ int sw[32];
  const int* a = blockIdx.y ? a1 : a0;
  int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i)
    if (base + i < L) s += a[base + i];
  int incl = block_scan_inclusive(s, sw);
  if (threadIdx.x == SCAN_THREADS - 1) bsum[blockIdx.y * nb + blockIdx.x] = incl;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block_sums(int* bsum, int nb) {
  __shared__ int sw[32];
  __shared__ int carry_s;
  int* b = bsum + blockIdx.y * nb;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += SCAN_THREADS) {
    int i = base + threadIdx.x;
    int v = (i < nb) ? b[i] : 0;
    int incl = block_scan_inclusive(v, sw);
    int carry = carry_s;
    __syncthreads();
    if (i < nb) b[i] = carry + incl - v;   // exclusive prefix of tile sums
    if (threadIdx.x == SCAN_THREADS - 1) carry_s = carry + incl;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(int* a0, int* a1, int L, const int* bsum,
                                                              int nb) {
  __shared__ int sw[32];
  int* a = blockIdx.y ? a1 : a0;
  int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int v[SCAN_ITEMS];
  int s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    v[i] = (base + i < L) ? a[base + i] : 0;
    s += v[i];
  }
  int incl = block_scan_inclusive(s, sw);
  int run = incl - s + bsum[blockIdx.y * nb + blockIdx.x];
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    run += v[i];
    if (base + i < L) a[base + i] = run;
  }
}

}  // namespace
