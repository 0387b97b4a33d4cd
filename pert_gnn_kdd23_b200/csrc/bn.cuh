// BatchNorm forward pieces shared by the stand-alone apply (k_bn_apply, nodeops.cu) and the node-linear forward that
// applies BatchNorm while it loads its A operand (k_bn_linear_fwd_planes, linear_fwd.cu).  Both kernels call these
// helpers, so the activations they write are bit-identical by construction.  Likewise the backward pieces: the
// stand-alone passes (k_bn_bwd_reduce / k_bn_bwd_apply) and their fold into the node-linear backward (linear_bwd.cu)
// and the conv backward target pass (tconv_tile.cu).
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

// One chunk of n rows of column c into the fp64 statistics accumulator acc = [2][H] (k_bn_partial's 128-row chunks,
// the conv epilogue's node tiles): acc[c] += n mu,  acc[H + c] += M2 + n mu^2, where M2 is the chunk's sum of squares
// CENTRED on mu.  Raw fp32 sums of squares would lose the variance to cancellation once |mean| >> std (a column of
// mean 1e3 / std 1 keeps about 3 correct digits, a constant column gets a variance of rounding noise); with centred
// chunks, acc[H + c] - acc[c]^2 / N in fp64 cancels only the n mu^2 terms, which fp64 carries exactly enough.
__device__ __forceinline__ void bn_acc_chunk(double* acc, int H, int c, double n, double mu, double m2) {
  atomicAdd(acc + c, n * mu);
  atomicAdd(acc + H + c, m2 + n * mu * mu);
}

// Training: mean / rstd of column c from the fp64 sums acc = [sum | sum of squares] (bn_acc_chunk: k_bn_partial or
// the conv epilogue).  The CTA that passes `owner` also stores them for the backward pass and updates the running
// statistics (unbiased variance) and num_batches_tracked.
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

// dz = dy * (y > 0) * scale of one float4.  With inverted dropout after the ReLU, y > 0 <=> (ReLU active and kept), so
// the saved output is the whole mask and only the 1/(1-p) factor is applied (scale = 1 without dropout; __fmul_rn keeps
// that product exact and uncontracted).
__device__ __forceinline__ float4 bn_bwd_dz4(float4 g, float4 y, float scale) {
  g.x = y.x > 0.f ? __fmul_rn(g.x, scale) : 0.f; g.y = y.y > 0.f ? __fmul_rn(g.y, scale) : 0.f;
  g.z = y.z > 0.f ? __fmul_rn(g.z, scale) : 0.f; g.w = y.w > 0.f ? __fmul_rn(g.w, scale) : 0.f;
  return g;
}

// s1 += dz,  s2 += dz * xhat  (xhat = (x - mean) rstd): the two column sums of the training backward
__device__ __forceinline__ void bn_bwd_acc4(float4& s1, float4& s2, float4 dz, float4 x, float4 mu, float4 rs) {
  s1 = f4add(s1, dz);
  s2.x = fmaf(dz.x, (x.x - mu.x) * rs.x, s2.x); s2.y = fmaf(dz.y, (x.y - mu.y) * rs.y, s2.y);
  s2.z = fmaf(dz.z, (x.z - mu.z) * rs.z, s2.z); s2.w = fmaf(dz.w, (x.w - mu.w) * rs.w, s2.w);
}

// training: dx = gamma rstd (dz - sum_dz / n - xhat sum_dzxhat / n), a = sum_dz, b = sum_dzxhat, invn = 1 / n
__device__ __forceinline__ float4 bn_bwd_dx4(float4 g, float4 v, float4 mu, float4 rs, float4 ga, float4 a, float4 b,
                                             float invn) {
  float4 o;
  o.x = ga.x * rs.x * (g.x - a.x * invn - (v.x - mu.x) * rs.x * b.x * invn);
  o.y = ga.y * rs.y * (g.y - a.y * invn - (v.y - mu.y) * rs.y * b.y * invn);
  o.z = ga.z * rs.z * (g.z - a.z * invn - (v.z - mu.z) * rs.z * b.z * invn);
  o.w = ga.w * rs.w * (g.w - a.w * invn - (v.w - mu.w) * rs.w * b.w * invn);
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
