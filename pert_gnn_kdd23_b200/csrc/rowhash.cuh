// The runtime key of a trace: its (um, dm, interface) rows in file order.  Two traces share a runtime iff these
// sequences are equal (order and length included).  Shared by the trace grouping (tracegroup.cu), which hashes every
// trace of a table, and the trace ingest (ingest.cu), which matches a chunk's runtimes against a live store's: both
// use the same two order-sensitive 64-bit hashes, the same slot of an open-addressing table and a row-by-row
// comparison before accepting a match, so a hash collision costs a comparison and never merges two runtimes.
#pragma once
#include "common.cuh"

namespace {

constexpr unsigned long long RT_SEED1 = 0x243f6a8885a308d3ull;
constexpr unsigned long long RT_SEED2 = 0x13198a2e03707344ull;

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {   // splitmix64 finaliser
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// one row's term of a runtime hash: the hash is the sum of these over the rows, pos = the row's position in the trace
__device__ __forceinline__ unsigned long long row_mix(unsigned long long seed, int pos, int64_t um, int64_t dm,
                                                      int64_t itf) {
  unsigned long long h = mix64(seed ^ (unsigned long long)pos);
  h = mix64(h ^ (unsigned long long)um);
  h = mix64(h ^ (unsigned long long)dm);
  return mix64(h ^ (unsigned long long)itf);
}

// the hashes keep their low hash_bits bits (tests narrow them to force collisions)
__device__ __forceinline__ unsigned long long hash_mask(int hash_bits) {
  return hash_bits >= 64 ? ~0ull : ((1ull << hash_bits) - 1);
}

// first probe of a runtime in a power-of-two table of S slots
__device__ __forceinline__ long long runtime_slot(unsigned long long h1, unsigned long long h2, int len, long long S) {
  return (long long)(mix64(h1 ^ mix64(h2 ^ (unsigned long long)len)) & (unsigned long long)(S - 1));
}

// Warp-wide comparison of two row sequences of length len; A and B give um(i), dm(i), itf(i) of row i.  Every lane
// returns the same answer.
template <class A, class B>
__device__ __forceinline__ bool warp_same_rows(const A& a, const B& b, int len, int lane) {
  bool eq = true;
  for (int i = lane; i < len && eq; i += 32) eq = a.um(i) == b.um(i) && a.dm(i) == b.dm(i) && a.itf(i) == b.itf(i);
  return __all_sync(0xffffffffu, eq);
}

}  // namespace
