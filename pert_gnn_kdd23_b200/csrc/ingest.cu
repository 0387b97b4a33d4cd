// Appending traces to a live pattern store (PatternStore.append_traces).
//
// A chunk of span rows is grouped by the trace grouping (tracegroup.cu) on its own: chunk-local runtimes with their
// representatives' rows, chunk-local (entry, runtime) pairs with counts.  The store then needs two things from the
// device, both computed here without touching the store's arrays (the results go to fresh arrays the caller swaps in):
//   1. match: which chunk runtimes the store already has.  The store keeps the (um, dm, interface) rows of every
//      pattern's representative (its runtime key) and a persistent open-addressing table over them, keyed by the two
//      hashes and the length tracegroup.cu uses (rowhash.cuh).  One warp per chunk runtime hashes its representative,
//      probes the table and compares row by row before it accepts a match.  Chunk runtimes are distinct from each
//      other, so a chunk runtime matches at most one pattern and no two chunk runtimes match the same one.  Unmatched
//      runtimes become patterns n_pat + (rank in chunk insertion order), with runtime ids n_rt + (rank in chunk runtime
//      id order, i.e. by smallest traceid): two scans of "new" flags.
//   2. merge: the entry mixes.  An (entry, pattern) table over the store's pairs decides, for every chunk pair,
//      whether it adds to an old pair or is new to its entry.  Entry e keeps its old pairs in their order and appends
//      its new ones in chunk order; its pointer comes from a scan of the per-entry lengths.  Every output slot is
//      written by one thread, once: an old pair receives at most one chunk pair (the chunk's pairs of one entry have
//      distinct patterns), so the result does not depend on scheduling.  Probabilities are (old count + chunk count) /
//      (old total + chunk total) in fp64, rounded to fp32.
// The table only grows; the caller rebuilds it (pert_ingest_table_insert from 0) into a larger one when the load
// would pass 1/2.
#include "rowhash.cuh"
#include "scan.cuh"

namespace {

constexpr int IG_WARPS = 8;
constexpr int IG_THREADS = 256;
constexpr int IG_EMPTY = -1;
constexpr unsigned long long IG_NOKEY = ~0ull;

// the key rows of runtime k of a PertRuntimeKeys: rows [3][ld], runtime k owns ptr[k] .. ptr[k+1]-1
struct KeyRows {
  const int64_t* r;
  long long ld;
  __device__ int64_t um(int i) const { return r[i]; }
  __device__ int64_t dm(int i) const { return r[ld + i]; }
  __device__ int64_t itf(int i) const { return r[2 * ld + i]; }
};

__device__ __forceinline__ KeyRows key_rows(const PertRuntimeKeys& k, long long j) {
  return KeyRows{k.rows + k.ptr[j], k.ld};
}

__device__ __forceinline__ void warp_hash(const KeyRows& a, int len, int lane, int hash_bits, unsigned long long& h1,
                                          unsigned long long& h2) {
  unsigned long long s1 = 0, s2 = 0;
  for (int i = lane; i < len; i += 32) {
    const int64_t um = a.um(i), dm = a.dm(i), itf = a.itf(i);
    s1 += row_mix(RT_SEED1, i, um, dm, itf);
    s2 += row_mix(RT_SEED2, i, um, dm, itf);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  const unsigned long long mask = hash_mask(hash_bits);
  h1 = s1 & mask;
  h2 = s2 & mask;
}

// warp per runtime j in [first, n): hash its key rows and claim an empty slot (the keys are distinct)
__global__ void __launch_bounds__(IG_WARPS * 32) k_table_insert(PertRuntimeKeys keys, long long first,
                                                                PertRuntimeTable tab) {
  const long long j = first + (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= keys.n) return;
  const int len = keys.ptr[j + 1] - keys.ptr[j];
  unsigned long long h1, h2;
  warp_hash(key_rows(keys, j), len, lane, tab.hash_bits, h1, h2);
  if (lane) return;
  tab.h1[j] = h1;
  tab.h2[j] = h2;
  long long s = runtime_slot(h1, h2, len, tab.S);
  while (atomicCAS(&tab.slot[s], IG_EMPTY, (int)j) != IG_EMPTY) s = (s + 1) & (tab.S - 1);
}

// warp per chunk runtime k (chunk insertion order): the store's pattern with the same key rows, or -1; flags[k+1] = new
__global__ void __launch_bounds__(IG_WARPS * 32) k_match(PertRuntimeKeys keys, PertRuntimeTable tab,
                                                         PertRuntimeKeys chunk, int* pat_of, int* flags) {
  const long long k = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= chunk.n) return;
  const KeyRows a = key_rows(chunk, k);
  const int len = chunk.ptr[k + 1] - chunk.ptr[k];
  unsigned long long h1, h2;
  warp_hash(a, len, lane, tab.hash_bits, h1, h2);
  long long s = runtime_slot(h1, h2, len, tab.S);
  int found = IG_EMPTY;
  for (;;) {
    const int o = tab.slot[s];
    if (o == IG_EMPTY) break;
    if (tab.h1[o] == h1 && tab.h2[o] == h2 && keys.ptr[o + 1] - keys.ptr[o] == len &&
        warp_same_rows(a, key_rows(keys, o), len, lane)) {
      found = o;
      break;
    }
    s = (s + 1) & (tab.S - 1);
  }
  if (lane == 0) {
    pat_of[k] = found;
    flags[k + 1] = found == IG_EMPTY;
  }
}

// rflags[r+1] = chunk runtime id r is new (runtime_ins: insertion index of every chunk runtime id)
__global__ void k_rid_flags(long long n, const int* runtime_ins, const int* flags, int* rflags) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) rflags[r + 1] = flags[runtime_ins[r] + 1];
}

// after the scans: new chunk runtime k becomes pattern n_pat + flags[k]; new_rep / new_rt list the new patterns
__global__ void k_new_assign(long long n, long long n_pat, const int* runtime_ins, const int* flags,
                             const int* rflags, int* pat_of, int* new_rep, int* new_rt, long long* n_new) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x == 0) *n_new = flags[n];
  if (x >= n) return;
  if (flags[x + 1] != flags[x]) {                           // x as an insertion index
    pat_of[x] = (int)(n_pat + flags[x]);
    new_rep[flags[x]] = (int)x;
  }
  if (rflags[x + 1] != rflags[x]) {                         // x as a chunk runtime id
    new_rt[flags[runtime_ins[x]]] = (int)(n_pat + rflags[x]);
  }
}

// largest e in [0, n) with ptr[e] <= v (ptr non-decreasing, ptr[0] = 0 <= v)
__device__ __forceinline__ int seg_of(const int* __restrict__ ptr, long long n, long long v) {
  int lo = 0, hi = (int)n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (ptr[mid] <= v) lo = mid;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ unsigned long long pair_key(int e, int pat) {
  return ((unsigned long long)(unsigned)e << 32) | (unsigned)pat;
}

// thread per old pair i: (entry, pattern) -> i
__global__ void k_pair_table(PertStore s, long long n_pairs, long long S, unsigned long long* pkey, int* pval) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int e = seg_of(s.ent_ptr, s.n_ent, i);
  const unsigned long long key = pair_key(e, s.ent_pat[i]);
  long long j = (long long)(mix64(key) & (unsigned long long)(S - 1));
  while (atomicCAS(&pkey[j], IG_NOKEY, key) != IG_NOKEY) j = (j + 1) & (S - 1);
  pval[j] = (int)i;
}

// thread per chunk pair j: its entry, global pattern and count; adds to the old pair it extends (add[i]) or flags
// itself new (nf[j+1])
__global__ void k_chunk_pairs(PertStore s, PertChunkMix c, long long S, const unsigned long long* pkey,
                              const int* pval, int* add, int* nf, int* jent, int* jpat, int* jcnt) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c.n_pairs) return;
  const int e = seg_of(c.ent_pair_ptr, c.n_ent, j);
  const int pat = c.pat_of[c.runtime_ins[c.pair_runtime[j]]];
  // pair_prob = count / total, correctly rounded, with count <= total < 2^31: prob * total is within 2^-22 of count
  const int cnt = (int)llrint(c.pair_prob[j] * (double)(c.ent_trace_ptr[e + 1] - c.ent_trace_ptr[e]));
  int old = IG_EMPTY;
  if (e < s.n_ent && s.ent_ptr[e + 1] > s.ent_ptr[e]) {
    const unsigned long long key = pair_key(e, pat);
    long long q = (long long)(mix64(key) & (unsigned long long)(S - 1));
    for (;;) {
      const unsigned long long o = pkey[q];
      if (o == IG_NOKEY) break;
      if (o == key) {
        old = pval[q];
        break;
      }
      q = (q + 1) & (S - 1);
    }
  }
  if (old != IG_EMPTY) add[old] = cnt;
  nf[j + 1] = old == IG_EMPTY;
  jent[j] = e;
  jpat[j] = pat;
  jcnt[j] = cnt;
}

// thread per output entry e: its pair count (into ent_ptr[e+1], scanned afterwards), node / edge totals and trace total
__global__ void k_entry_sizes(PertStore s, const int* tot, PertChunkMix c, const int* pat_nptr, const int* pat_eptr,
                              const int* nf, const int* jpat, long long n_ent_out, PertMixOut out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e == 0) out.ent_ptr[0] = 0;
  if (e >= n_ent_out) return;
  const bool in_old = e < s.n_ent, in_chunk = e < c.n_ent;
  int len = in_old ? s.ent_ptr[e + 1] - s.ent_ptr[e] : 0;
  int nodes = in_old ? s.ent_nodes[e] : 0, edges = in_old ? s.ent_edges[e] : 0;
  int total = in_old ? tot[e] : 0;
  if (in_chunk) {
    const int lo = c.ent_pair_ptr[e], hi = c.ent_pair_ptr[e + 1];
    len += nf[hi] - nf[lo];
    for (int j = lo; j < hi; ++j) {
      if (nf[j + 1] == nf[j]) continue;
      const int p = jpat[j];
      nodes += pat_nptr[p + 1] - pat_nptr[p];
      edges += pat_eptr[p + 1] - pat_eptr[p];
    }
    total += c.ent_trace_ptr[e + 1] - c.ent_trace_ptr[e];
  }
  out.ent_ptr[e + 1] = len;
  out.ent_nodes[e] = nodes;
  out.ent_edges[e] = edges;
  out.tot[e] = total;
}

__device__ __forceinline__ void emit(const PertMixOut& out, long long slot, int pat, int cnt, int total) {
  out.ent_pat[slot] = pat;
  out.cnt[slot] = cnt;
  out.ent_prob[slot] = (float)((double)cnt / (double)total);
}

// thread per old pair i: same rank inside its entry, count grown by the chunk's
__global__ void k_emit_old(PertStore s, const int* cnt, const int* add, long long n_pairs, PertMixOut out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int e = seg_of(s.ent_ptr, s.n_ent, i);
  emit(out, out.ent_ptr[e] + (i - s.ent_ptr[e]), s.ent_pat[i], cnt[i] + add[i], out.tot[e]);
}

// thread per chunk pair j new to its entry: after the entry's old pairs, in chunk order
__global__ void k_emit_new(PertStore s, PertChunkMix c, const int* nf, const int* jent, const int* jpat,
                           const int* jcnt, PertMixOut out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c.n_pairs || nf[j + 1] == nf[j]) return;
  const int e = jent[j];
  const int old_len = e < s.n_ent ? s.ent_ptr[e + 1] - s.ent_ptr[e] : 0;
  emit(out, (long long)out.ent_ptr[e] + old_len + (nf[j] - nf[c.ent_pair_ptr[e]]), jpat[j], jcnt[j], out.tot[e]);
}

bool keys_ok(const PertRuntimeKeys* k) {
  return k && k->n >= 0 && k->n <= 0x7ffffff0LL && k->ld >= 0 && k->ptr && (k->ld == 0 || k->rows);
}

bool table_ok(const PertRuntimeTable* t) {
  return t && t->S >= 64 && (t->S & (t->S - 1)) == 0 && t->S <= 0x40000000LL && t->hash_bits >= 1 &&
         t->hash_bits <= 64 && t->slot && t->h1 && t->h2;
}

long long pow2_slots(long long n) {            // power of two >= 2n (>= 64): every probe sequence ends at an empty slot
  long long S = 64;
  while (S < 2 * n) S <<= 1;
  return S;
}

long long scan_ws(long long L) { return 2LL * pert_cdiv(L, SCAN_TILE) * 4 + 16; }

void scan_launch(int* a0, int* a1, long long L, int* bsum, cudaStream_t st) {   // inclusive, in place
  const int nb = pert_cdiv(L, SCAN_TILE), ny = a1 ? 2 : 1;
  k_scan_tile_sums<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
  k_scan_block_sums<<<dim3(1, ny), SCAN_THREADS, 0, st>>>(bsum, nb);
  k_scan_apply<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
}

}  // namespace

extern "C" {

int pert_ingest_table_insert(const PertRuntimeKeys* keys, long long first, const PertRuntimeTable* table,
                             void* stream) {
  if (!keys_ok(keys) || !table_ok(table) || first < 0 || first > keys->n || 2 * keys->n > table->S)
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if (first == 0 && (e = cudaMemsetAsync(table->slot, 0xff, sizeof(int) * table->S, st)) != cudaSuccess)
    return (int)e;
  const long long n = keys->n - first;
  if (n == 0) return PERT_OK;
  const int WB = IG_WARPS * 32;
  k_table_insert<<<pert_cdiv(n * 32, WB), WB, 0, st>>>(*keys, first, *table);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_ingest_match_workspace_bytes(long long n_chunk) {
  if (n_chunk < 0 || n_chunk > 0x7ffffff0LL) return PERT_ERR_BADARG;
  return 2 * (n_chunk + 1) * 4 + scan_ws(n_chunk + 1) + 64;
}

int pert_ingest_match(const PertRuntimeKeys* keys, const PertRuntimeTable* table, const PertRuntimeKeys* chunk,
                      const int32_t* chunk_runtime_ins, int32_t* pat_of, int32_t* new_rep, int32_t* new_rt,
                      long long* n_new, void* workspace, long long workspace_bytes, void* stream) {
  if (!keys_ok(keys) || !table_ok(table) || !keys_ok(chunk) || 2 * keys->n > table->S || !n_new || !workspace ||
      (chunk->n > 0 && (!chunk_runtime_ins || !pat_of || !new_rep || !new_rt)))
    return PERT_ERR_BADARG;
  const long long n = chunk->n;
  if (workspace_bytes < pert_ingest_match_workspace_bytes(n)) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  int* flags = (int*)workspace;
  int* rflags = flags + (n + 1);
  int* bsum = rflags + (n + 1);
  cudaError_t e;
  if ((e = cudaMemsetAsync(flags, 0, 2 * sizeof(int) * (n + 1), st)) != cudaSuccess) return (int)e;
  const int WB = IG_WARPS * 32, B = IG_THREADS;
  if (n > 0) {
    k_match<<<pert_cdiv(n * 32, WB), WB, 0, st>>>(*keys, *table, *chunk, pat_of, flags);
    k_rid_flags<<<pert_cdiv(n, B), B, 0, st>>>(n, chunk_runtime_ins, flags, rflags);
    scan_launch(flags, rflags, n + 1, bsum, st);
  }
  k_new_assign<<<pert_cdiv(n + 1, B), B, 0, st>>>(n, keys->n, chunk_runtime_ins, flags, rflags, pat_of, new_rep,
                                                  new_rt, n_new);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_ingest_merge_workspace_bytes(long long n_pairs, long long n_chunk_pairs, long long n_ent_out) {
  if (n_pairs < 0 || n_chunk_pairs < 0 || n_ent_out < 0 || n_pairs > 0x7ffffff0LL || n_chunk_pairs > 0x7ffffff0LL ||
      n_ent_out > 0x7ffffff0LL)
    return PERT_ERR_BADARG;
  const long long S = pow2_slots(n_pairs);
  const long long L = n_chunk_pairs + 1 > n_ent_out + 1 ? n_chunk_pairs + 1 : n_ent_out + 1;
  return 8 * S + 4 * (S + n_pairs + (n_chunk_pairs + 1) + 3 * n_chunk_pairs) + scan_ws(L) + 64;
}

int pert_ingest_merge(const PertStore* store, const int32_t* cnt, const int32_t* tot, long long n_pairs,
                      const PertChunkMix* chunk, const int32_t* pat_nptr, const int32_t* pat_eptr, long long n_ent_out,
                      const PertMixOut* out, void* workspace, long long workspace_bytes, void* stream) {
  if (!store || !chunk || !out || !workspace || !pat_nptr || !pat_eptr || n_pairs < 0 || store->n_ent < 0 ||
      chunk->n_ent < 0 || chunk->n_pairs < 0 || n_ent_out < store->n_ent || n_ent_out < chunk->n_ent ||
      !store->ent_ptr || !store->ent_nodes || !store->ent_edges || (store->n_ent > 0 && !tot))
    return PERT_ERR_BADARG;
  if ((n_pairs > 0 && (!store->ent_pat || !cnt)) || !chunk->ent_pair_ptr || !chunk->ent_trace_ptr ||
      (chunk->n_pairs > 0 && (!chunk->pair_runtime || !chunk->pair_prob || !chunk->runtime_ins || !chunk->pat_of)))
    return PERT_ERR_BADARG;
  if (!out->ent_ptr || !out->ent_nodes || !out->ent_edges || !out->tot ||
      (n_pairs + chunk->n_pairs > 0 && (!out->ent_pat || !out->ent_prob || !out->cnt)))
    return PERT_ERR_BADARG;
  if (n_pairs + chunk->n_pairs > 0x7fffffffLL) return PERT_ERR_BADARG;
  const long long need = pert_ingest_merge_workspace_bytes(n_pairs, chunk->n_pairs, n_ent_out);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long S = pow2_slots(n_pairs), np = chunk->n_pairs;
  unsigned long long* pkey = (unsigned long long*)workspace;
  int* w = (int*)(pkey + S);
  int* pval = w;  w += S;
  int* add = w;   w += n_pairs;
  int* nf = w;    w += np + 1;
  int* jent = w;  w += np;
  int* jpat = w;  w += np;
  int* jcnt = w;  w += np;
  int* bsum = w;
  cudaError_t e;
  if ((e = cudaMemsetAsync(pkey, 0xff, 8 * S, st)) || (e = cudaMemsetAsync(add, 0, 4 * n_pairs, st)) ||
      (e = cudaMemsetAsync(nf, 0, 4 * (np + 1), st)))
    return (int)e;
  const int B = IG_THREADS;
  if (n_pairs > 0) k_pair_table<<<pert_cdiv(n_pairs, B), B, 0, st>>>(*store, n_pairs, S, pkey, pval);
  if (np > 0) {
    k_chunk_pairs<<<pert_cdiv(np, B), B, 0, st>>>(*store, *chunk, S, pkey, pval, add, nf, jent, jpat, jcnt);
    scan_launch(nf, nullptr, np + 1, bsum, st);
  }
  k_entry_sizes<<<pert_cdiv(n_ent_out + 1, B), B, 0, st>>>(*store, tot, *chunk, pat_nptr, pat_eptr, nf, jpat,
                                                           n_ent_out, *out);
  scan_launch(out->ent_ptr, nullptr, n_ent_out + 1, bsum, st);
  if (n_pairs > 0) k_emit_old<<<pert_cdiv(n_pairs, B), B, 0, st>>>(*store, cnt, add, n_pairs, *out);
  if (np > 0) k_emit_new<<<pert_cdiv(np, B), B, 0, st>>>(*store, *chunk, nf, jent, jpat, jcnt, *out);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
