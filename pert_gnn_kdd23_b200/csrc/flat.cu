// Relayout of the flat parameter buffers when parameters grow (train.FlatParams.grow): one launch copies every
// parameter segment of params / Adam m / Adam v into the new layout, zeroes the new tails and the padding, and zeroes
// the new gradient buffer.
#include "common.cuh"

namespace {

// The segment table travels as a kernel argument (3 KB, under the 4 KB parameter limit): no device copy of it, no host
// synchronisation, nothing to allocate.
struct FlatSegs {
  long long new_off[PERT_FLAT_MAX_SEGS];
  long long old_off[PERT_FLAT_MAX_SEGS];
  long long old_len[PERT_FLAT_MAX_SEGS];
};

struct FlatBufs {
  const float* src[3];     // params, m, v of the old layout (NULL: pair absent)
  float* dst[3];           // the same three in the new layout
  float* grad;             // new gradient buffer: zeroed
};

// One float4 of the new layout per thread and step.  Its segment is the last one starting at or before it (binary
// search over the segment starts, staged in shared memory); the float4 holds old data up to the segment's old length
// and zero past it (new rows, alignment padding, the gap before the first segment).  Offsets are multiples of
// PERT_FLAT_ALIGN, so a float4 never straddles two segments, and the old float4 read lies inside the old segment's
// padded slot.
__global__ void __launch_bounds__(256) k_flat_grow(const __grid_constant__ FlatSegs segs, int n_seg,
                                                   const __grid_constant__ FlatBufs bufs, long long n4) {
  __shared__ long long s_new[PERT_FLAT_MAX_SEGS];
  for (int i = threadIdx.x; i < n_seg; i += blockDim.x) s_new[i] = segs.new_off[i];
  __syncthreads();
  const float4 zero = f4zero();
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
    const long long j = q * 4;
    int lo = 0, hi = n_seg;                          // first segment with new_off > j
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_new[mid] <= j) lo = mid + 1;
      else hi = mid;
    }
    const int s = lo - 1;
    long long r = 0, len = 0, src = 0;
    if (s >= 0) {
      r = j - s_new[s];
      len = segs.old_len[s];
      src = segs.old_off[s] + r;
    }
    const bool any = s >= 0 && r < len;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      if (!bufs.dst[b]) continue;
      float4 v = zero;
      if (any) {
        v = ld4(bufs.src[b] + src);
        if (r + 1 >= len) v.y = 0.f;
        if (r + 2 >= len) v.z = 0.f;
        if (r + 3 >= len) v.w = 0.f;
      }
      st4(bufs.dst[b] + j, v);
    }
    st4(bufs.grad + j, zero);
  }
}

bool overlap(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + (uintptr_t)nb * 4 && y < x + (uintptr_t)na * 4;
}

}  // namespace

extern "C" {

int pert_flat_grow(const long long* segs, int n_seg, long long n_old, long long n_new, const float* p_old,
                   float* p_new, const float* m_old, float* m_new, const float* v_old, float* v_new, float* g_new,
                   void* stream) {
  const long long A = PERT_FLAT_ALIGN;
  if (n_seg < 0 || n_seg > PERT_FLAT_MAX_SEGS || (n_seg > 0 && !segs)) return PERT_ERR_BADARG;
  if (n_old < 0 || n_new < n_old || n_old % A || n_new % A) return PERT_ERR_BADARG;
  if (!p_old || !p_new || !g_new) return PERT_ERR_BADARG;
  if (!m_old != !m_new || !v_old != !v_new) return PERT_ERR_BADARG;
  // segments: in order, aligned, non-overlapping in both layouts, never shrinking
  FlatSegs t;
  long long end_old = 0, end_new = 0;
  for (int s = 0; s < n_seg; ++s) {
    const long long oo = segs[4 * s], no = segs[4 * s + 1], ol = segs[4 * s + 2], nl = segs[4 * s + 3];
    if (ol < 0 || nl < ol || oo % A || no % A) return PERT_ERR_BADARG;
    if (oo < end_old || no < end_new) return PERT_ERR_BADARG;
    end_old = oo + ol;
    end_new = no + nl;
    if (end_old > n_old || end_new > n_new) return PERT_ERR_BADARG;
    t.old_off[s] = oo;
    t.new_off[s] = no;
    t.old_len[s] = ol;
  }
  // no buffer may alias another: the kernel reads the old ones while it writes the new ones
  const void* ptrs[7] = {p_old, p_new, m_old, m_new, v_old, v_new, g_new};
  const long long lens[7] = {n_old, n_new, n_old, n_new, n_old, n_new, n_new};
  for (int a = 0; a < 7; ++a) {
    if (((uintptr_t)ptrs[a] & 15) != 0) return PERT_ERR_BADARG;
    for (int b = a + 1; b < 7; ++b)
      if (ptrs[a] && ptrs[b] && lens[a] > 0 && lens[b] > 0 && overlap(ptrs[a], lens[a], ptrs[b], lens[b])) return PERT_ERR_BADARG;
  }
  if (n_new == 0) return PERT_OK;
  FlatBufs bufs = {{p_old, m_old, v_old}, {p_new, m_new, v_new}, g_new};
  const long long n4 = n_new / 4;
  int grid = pert_cdiv(n4, 256);
  if (grid > 16 * PERT_NUM_SMS) grid = 16 * PERT_NUM_SMS;
  k_flat_grow<<<grid, 256, 0, (cudaStream_t)stream>>>(t, n_seg, bufs, n4);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
