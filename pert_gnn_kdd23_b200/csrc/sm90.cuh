// Hopper (sm_90a) building blocks shared by the tensor-core GEMMs (gemm_tc.cu, linear_bwd.cu, linear_fwd.cu) and the
// bulk-copy kernels (tconv_tile.cu, segreduce_tma.cu): wgmma (m64nNk8, kind tf32) with the 3xTF32 hi / lo split,
// shared-memory matrix descriptors, mbarriers, bulk copies, L2 eviction policies and cluster barriers.
//
// Operand conventions (see gemm_tc.cu for how each kernel stages its operands):
//   A: registers in the wgmma A-fragment layout: a thread of warp w holds rows 16w + g and 16w + g + 8 (g = lane / 4)
//      and K columns t, t + 4 (t = lane % 4) of every K-step of 8.
//   B: shared memory, no-swizzle K-major canonical layout (8-row x 16-byte core matrices, LBO = 128 B between
//      K-adjacent core matrices, SBO between N-adjacent ones), split hi / lo.
//   D: fp32 accumulators in registers (fragment: row g / g + 8, columns 8j + 2t, 8j + 2t + 1).
#pragma once
#include <stdint.h>

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// wgmma shared-memory matrix descriptor (sm_90): start address, LBO, SBO in 16-byte units; base offset 0,
// layout type 0 (no swizzle)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3fff) << 32;
  return d;
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed group complete
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// D[64 x 32] += A[64 x 8] (registers) . B[32 x 8]^T (descriptor)
__device__ __forceinline__ void wgmma_n32(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
      : "memory");
}
// D[64 x 16] += A[64 x 8] . B[16 x 8]^T
__device__ __forceinline__ void wgmma_n16(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
      : "memory");
}

// D[64 x 64] += A[64 x 8] . B[64 x 8]^T
__device__ __forceinline__ void wgmma_n64(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
      : "memory");
}
// D[64 x 80] += A[64 x 8] . B[80 x 8]^T
__device__ __forceinline__ void wgmma_n80(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39"
      "}, {%40, %41, %42, %43}, %44, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b)
      : "memory");
}

// D[64 x 128] (+)= A[64 x 8] . B[128 x 8]^T; accumulate = 0 overwrites D (a sum starts without zeroed registers)
__device__ __forceinline__ void wgmma_n128(float* d, const uint32_t* a, uint64_t b, int accumulate = 1) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate)
      : "memory");
}

// One K-step of 8 over all BN in {64, 80} columns as single wgmmas (the accumulator layout equals mma_step's):
// hi*hi + lo*hi + hi*lo
template <int BN>
__device__ __forceinline__ void mma_step_wide(float* d, const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t bhi,
                                              uint32_t blo, uint32_t sbo) {
  static_assert(BN == 64 || BN == 80, "mma_step_wide: N = 64 or 80");
  const uint64_t dh = make_desc(bhi, 128, sbo), dl = make_desc(blo, 128, sbo);
  if (BN == 64) {
    wgmma_n64(d, ah, dh);
    wgmma_n64(d, al, dh);
    wgmma_n64(d, ah, dl);
  } else {
    wgmma_n80(d, ah, dh);
    wgmma_n80(d, al, dh);
    wgmma_n80(d, ah, dl);
  }
}

// Round-to-nearest split with integer ops: hi = (bits + 0x1000) & 0xffffe000 (nearest tf32, ties away from zero; two
// full-rate ALU instructions instead of the quarter-rate cvt.rna.tf32.f32), lo = x - hi (exact in fp32,
// |lo| <= 2^-11 |x|, either sign; the tensor core drops its low 13 bits: <= 2^-21 |x|, sign-symmetric).  A truncating
// hi (x & 0xffffe000) makes lo one-signed and the dropped bits a one-sided residual that does not average out over
// 10^4..10^5-term sums.
__device__ __forceinline__ uint32_t tf32_hi(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ uint32_t tf32_lo(float x, uint32_t hi) { return __float_as_uint(x - __uint_as_float(hi)); }

__device__ __forceinline__ void split4(const float (&v)[4], uint32_t (&h)[4], uint32_t (&l)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = tf32_hi(v[i]);
    l[i] = tf32_lo(v[i], h[i]);
  }
}

// One K-step of 8 over all BN columns: hi*hi + lo*hi + hi*lo.  bhi / blo: shared addresses of the step's first core
// matrix; 32 columns (four 8-row core-matrix groups) further is 4 * SBO.
template <int BN>
__device__ __forceinline__ void mma_step(float* d, const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t bhi,
                                         uint32_t blo, uint32_t sbo) {
  constexpr int N32 = BN / 32;
#pragma unroll
  for (int j = 0; j < N32; ++j) {
    const uint64_t dh = make_desc(bhi + j * 4 * sbo, 128, sbo), dl = make_desc(blo + j * 4 * sbo, 128, sbo);
    wgmma_n32(d + 16 * j, ah, dh);
    wgmma_n32(d + 16 * j, al, dh);
    wgmma_n32(d + 16 * j, ah, dl);
  }
  if (BN % 32) {
    const uint64_t dh = make_desc(bhi + N32 * 4 * sbo, 128, sbo), dl = make_desc(blo + N32 * 4 * sbo, 128, sbo);
    wgmma_n16(d + 16 * N32, ah, dh);
    wgmma_n16(d + 16 * N32, al, dh);
    wgmma_n16(d + 16 * N32, ah, dl);
  }
}

// Local column of accumulator register i (fragment of the n32 / n16 pieces: 4 registers per 8 columns)
__device__ __forceinline__ int acc_col(int i, int t) { return (i >> 2) * 8 + 2 * t + (i & 1); }

// Logical K position (inside the weight operand) of physical column p when thread t of an A fragment holds the four
// CONTIGUOUS columns 4t..4t+3 of every 16-column chunk (columns 4t, 4t+1 feed K-step 0 of the chunk, 4t+2, 4t+3
// step 1); K16 = K rounded down to 16, the trailing 8 columns give thread t columns 2t, 2t + 1.
__device__ __forceinline__ int nt_logical_k(int p, int K16) {
  if (p < K16) {
    const int r = p & 15;
    return (p & ~15) + ((r >> 1) & 1) * 8 + (r >> 2) + (r & 1) * 4;
  }
  const int r = p - K16;
  return K16 + (r >> 1) + (r & 1) * 4;
}

// ---- mbarriers and bulk copies (global -> shared, completion counted in bytes on an mbarrier)
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
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
// dst / src 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- L2 eviction priority.  A policy (createpolicy) gives the lines an access touches an eviction priority in L2:
// evict_last lines are replaced after every other line, evict_first lines before them, evict_normal is what an access
// without a hint gets.  A fraction f < 1 marks only that share of the lines (chosen by address).  A hinted access
// re-marks a line that is already in L2, so a consumer's last read of a handoff demotes it again.
__device__ __forceinline__ uint64_t l2_evict_last(float f = 1.f) {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, %1;" : "=l"(p) : "f"(f));
  return p;
}
__device__ __forceinline__ uint64_t l2_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// the policy of a hinted access in a kernel whose hints are switched on by `on`, else the default policy
__device__ __forceinline__ uint64_t l2_keep(int on, float f = 1.f) { return on ? l2_evict_last(f) : l2_evict_normal(); }
__device__ __forceinline__ uint64_t l2_stream(int on) { return on ? l2_evict_first() : l2_evict_normal(); }
// hinted forms of the accesses of the conv chain: 16-byte read-only load, 16- and 8-byte stores, 1-D bulk copy
__device__ __forceinline__ float4 ldg4_hint(const float* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st4_hint(float* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void st2_hint(float* p, float2 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
// Drops the 128-byte L2 line that starts at p without writing it back: its contents are undefined afterwards.  Only for
// dead scratch, after its last read has completed.  It counts as a global write (pdl_wait first, common.cuh).  A p that
// is not 128-byte aligned does nothing: the line would hold bytes of a live neighbour (a workspace the caller aligned to
// 16 bytes only).
__device__ __forceinline__ void discard_l2(const void* p) {
  if (((uintptr_t)p & 127) == 0) asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory");
}

// ---- thread-block clusters and distributed shared memory
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster: shared-memory writes before it are visible to the cluster after it
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the two halves of cluster_sync, for threads that have work to do in between (each thread alternates them)
__device__ __forceinline__ void cluster_arrive() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t map_rank(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 ld_cluster4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(addr)
               : "memory");
  return v;
}
// named barrier over `count` threads (a multiple of 32)
__device__ __forceinline__ void bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

}  // namespace
