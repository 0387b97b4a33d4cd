// BatchNorm forward pieces shared by the stand-alone apply (k_bn_apply, nodeops.cu) and the node-linear forward that
// applies BatchNorm while it loads its A operand (k_bn_linear_fwd_planes, linear_fwd.cu).  Both kernels call these
// helpers, so the activations they write are bit-identical by construction.
#pragma once
#include <math.h>

#include "common.cuh"

namespace {

// ---------------------------------------------------------------- dropout mask (Philox4x32-10, Random123)
// Counter-based: the mask of an element is a pure function of (seed, step, layer, position), so nothing is stored
// between forward and backward and a replayed CUDA graph draws a new mask whenever the step word in memory moved.
// Contract (include/pertgnn.h, pert_model_forward): key = (seed lo, seed hi), counter = (float4 group g = row*(H/4) +
// col/4, layer, step lo, step hi); output word j decides column col + j: kept iff word >= T.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

struct BnDropout {
  const long long* ctr;   // device {seed, step} of this forward
  unsigned long long T;   // keep iff word >= T; T = 2^32 (p = 1) drops everything
  float scale;            // 1 / (1 - p), 0 at p = 1
  int layer;
};

// the Philox key and step words of one forward, read once per thread
struct BnDropKey {
  uint2 key;
  uint32_t step_lo, step_hi;
};
__device__ __forceinline__ BnDropKey bn_drop_key(const BnDropout& drop) {
  const unsigned long long seed = (unsigned long long)drop.ctr[0], step = (unsigned long long)drop.ctr[1];
  return BnDropKey{make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)), (uint32_t)step, (uint32_t)(step >> 32)};
}

// Training: mean / rstd of column c from the fp64 sums acc = [sum | sum of squares] (k_bn_partial or the conv
// epilogue).  The CTA that passes `owner` also stores them for the backward pass and updates the running statistics
// (unbiased variance) and num_batches_tracked.
__device__ __forceinline__ void bn_batch_stats(const double* acc, long long N, int H, int c, float eps, float momentum,
                                               bool owner, float* mean, float* rstd, float* running_mean,
                                               float* running_var, long long* num_batches_tracked, float& mu,
                                               float& rs) {
  const double n = (double)N;
  const double m = acc[c] / n;
  double m2 = acc[H + c] - n * m * m;
  if (m2 < 0.0) m2 = 0.0;
  const double var = m2 / n;       // biased, used to normalise
  mu = (float)m;
  rs = (float)(1.0 / sqrt(var + (double)eps));
  if (owner) {
    mean[c] = mu;
    rstd[c] = rs;
    if (running_mean) {
      const double unbiased = (N > 1) ? m2 / (n - 1.0) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
    }
    if (c == 0 && num_batches_tracked) *num_batches_tracked += 1;
  }
}

// (relu)((x - mean) rstd gamma + beta) of one float4
__device__ __forceinline__ float4 bn_affine4(float4 v, float4 mu, float4 rs, float4 ga, float4 be, bool relu) {
  float4 o;
  o.x = fmaf((v.x - mu.x) * rs.x, ga.x, be.x);
  o.y = fmaf((v.y - mu.y) * rs.y, ga.y, be.y);
  o.z = fmaf((v.z - mu.z) * rs.z, ga.z, be.z);
  o.w = fmaf((v.w - mu.w) * rs.w, ga.w, be.w);
  return relu ? f4max(o, f4zero()) : o;
}

// inverted dropout of float4 group g = row * (H/4) + col/4 (< 2^32, checked by the host)
__device__ __forceinline__ float4 bn_dropout4(float4 o, uint32_t g, const BnDropout& drop, const BnDropKey& k) {
  const uint4 r = philox4x32_10(make_uint4(g, (uint32_t)drop.layer, k.step_lo, k.step_hi), k.key);
  o.x = r.x >= drop.T ? o.x * drop.scale : 0.f;
  o.y = r.y >= drop.T ? o.y * drop.scale : 0.f;
  o.z = r.z >= drop.T ? o.z * drop.scale : 0.f;
  o.w = r.w >= drop.T ? o.w * drop.scale : 0.f;
  return o;
}

// host: the mask parameters of rate p (0 < p <= 1)
inline BnDropout bn_dropout_params(float p, const long long* ctr, int layer) {
  BnDropout dp;
  dp.ctr = ctr;
  dp.T = (unsigned long long)floor((double)p * 4294967296.0);   // exact: p is a float, 2^32 a power of two
  dp.scale = p >= 1.f ? 0.f : (float)(1.0 / (1.0 - (double)p));
  dp.layer = layer;
  return dp;
}

}  // namespace
