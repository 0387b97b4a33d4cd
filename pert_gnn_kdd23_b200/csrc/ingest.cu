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
//
// Evicting old traces (PatternStore.evict_traces) is split like the resource update into a count and an apply, so the
// caller allocates every output at its exact new size (an eviction exists to free memory):
//   1. count: one thread per trace flags keep = bucket >= before; an evicted trace probes the (entry, pattern) pair
//      table with its entry and pattern (the store keeps the pattern of every trace) and adds 1 to that pair's evicted
//      count (integer atomics: the sums do not depend on scheduling).  One thread per pair keeps it while its count
//      stays above 0 and marks its pattern alive; one thread per pattern takes the node / edge / key-row lengths of the
//      alive ones; one warp per entry sums its surviving nodes, edges and traces.  scan.cuh scans of the trace, pair
//      and pattern flags and of the surviving lengths give every new position; the sizes word holds their totals.
//   2. apply: stable compaction, every output slot written once by one thread, no atomics.  Traces and pairs move to
//      their scanned positions (a pair's pattern renumbered, its probability recomputed as emit() rounds it); the nodes,
//      edges and key rows of a surviving pattern move as one segment (pat_src / pat_dst are pattern-local).
// A pattern that keeps any trace keeps its representative's graph and key rows even when that trace was evicted.
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

__device__ __forceinline__ unsigned long long pair_key(int e, int pat) {
  return ((unsigned long long)(unsigned)e << 32) | (unsigned)pat;
}

// thread per old pair i: (entry, pattern) -> i
__global__ void k_pair_table(PertStore s, long long n_pairs, long long S, unsigned long long* pkey, int* pval) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int e = upper_seg(s.ent_ptr, s.n_ent, i);
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
  const int e = upper_seg(c.ent_pair_ptr, c.n_ent, j);
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
  const int e = upper_seg(s.ent_ptr, s.n_ent, i);
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

// ---- eviction -------------------------------------------------------------------------------------------------------

// the eviction workspace, shared by the count (which fills it) and the apply (which reads it).  Flag arrays are
// [n+1] with the flag of item i at [i+1]; after the inclusive scan [i] is the item's new position.
struct EvictWs {
  long long S;
  unsigned long long* pkey;   // [S] pair table keys
  int* pval;                  // [S] pair table values (old pair index)
  int* ev;                    // [P] evicted traces per old pair
  int* tkeep;                 // [T+1] trace kept
  int* pkeep;                 // [P+1] pair kept
  int* pa;                    // [n_pat+1] pattern kept
  int* pn;                    // [n_pat+1] nodes of a kept pattern (0 otherwise)
  int* pe;                    // [n_pat+1] edges of a kept pattern
  int* pk;                    // [n_pat+1] key rows of a kept pattern
  int* e_nodes;               // [n_ent] surviving nodes, edges and traces of every entry
  int* e_edges;
  int* e_tot;
  int* bsum;
};

long long evict_scan_len(long long T, long long P, long long n_pat) {
  long long L = T > P ? T : P;
  return (L > n_pat ? L : n_pat) + 1;
}

long long evict_ws_bytes(long long T, long long P, long long n_pat, long long n_ent) {
  const long long S = pow2_slots(P);
  return 8 * S + 4 * (S + P + (T + 1) + (P + 1) + 4 * (n_pat + 1) + 3 * n_ent) + scan_ws(evict_scan_len(T, P, n_pat)) +
         64;
}

EvictWs evict_ws(void* w, long long T, long long P, long long n_pat, long long n_ent) {
  EvictWs a;
  a.S = pow2_slots(P);
  a.pkey = (unsigned long long*)w;
  int* p = (int*)(a.pkey + a.S);
  a.pval = p;     p += a.S;
  a.ev = p;       p += P;
  a.tkeep = p;    p += T + 1;
  a.pkeep = p;    p += P + 1;
  a.pa = p;       p += n_pat + 1;
  a.pn = p;       p += n_pat + 1;
  a.pe = p;       p += n_pat + 1;
  a.pk = p;       p += n_pat + 1;
  a.e_nodes = p;  p += n_ent;
  a.e_edges = p;  p += n_ent;
  a.e_tot = p;    p += n_ent;
  a.bsum = p;
  return a;
}

// thread per trace t: tkeep[t+1] = bucket >= before; an evicted trace adds 1 to its (entry, pattern) pair's count
__global__ void k_evict_traces(PertStore s, const int* trace_pat, long long before, EvictWs w) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= s.n_traces) return;
  const bool keep = s.trace_ts[t] >= before;
  w.tkeep[t + 1] = keep;
  if (keep) return;
  const unsigned long long key = pair_key(s.trace_entry[t], trace_pat[t]);
  long long q = (long long)(mix64(key) & (unsigned long long)(w.S - 1));
  for (;;) {                                              // every trace's pair is in the table
    const unsigned long long o = w.pkey[q];
    if (o == key) {
      atomicAdd(&w.ev[w.pval[q]], 1);
      return;
    }
    if (o == IG_NOKEY) return;
    q = (q + 1) & (w.S - 1);
  }
}

// thread per pair i: kept while traces remain; a kept pair keeps its pattern (pa[pat+1] = 1, the same value from
// every pair of the pattern)
__global__ void k_evict_pairs(PertStore s, const int* cnt, long long n_pairs, EvictWs w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const bool alive = cnt[i] - w.ev[i] > 0;
  w.pkeep[i + 1] = alive;
  if (alive) w.pa[s.ent_pat[i] + 1] = 1;
}

// thread per pattern p: the node / edge / key-row lengths of a kept pattern, 0 for a dropped one
__global__ void k_evict_pat_lens(PertStore s, const int* key_ptr, EvictWs w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= s.n_pat) return;
  const bool alive = w.pa[p + 1];
  w.pn[p + 1] = alive ? s.pat_nptr[p + 1] - s.pat_nptr[p] : 0;
  w.pe[p + 1] = alive ? s.pat_eptr[p + 1] - s.pat_eptr[p] : 0;
  w.pk[p + 1] = alive ? key_ptr[p + 1] - key_ptr[p] : 0;
}

// warp per entry e: the nodes, edges and traces of its surviving pairs (integer sums)
__global__ void __launch_bounds__(IG_WARPS * 32) k_evict_entries(PertStore s, const int* cnt, EvictWs w) {
  const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= s.n_ent) return;
  int nodes = 0, edges = 0, traces = 0;
  for (int i = s.ent_ptr[e] + lane; i < s.ent_ptr[e + 1]; i += 32) {
    const int c = cnt[i] - w.ev[i];
    if (c <= 0) continue;
    const int p = s.ent_pat[i];
    nodes += s.pat_nptr[p + 1] - s.pat_nptr[p];
    edges += s.pat_eptr[p + 1] - s.pat_eptr[p];
    traces += c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nodes += __shfl_xor_sync(0xffffffffu, nodes, o);
    edges += __shfl_xor_sync(0xffffffffu, edges, o);
    traces += __shfl_xor_sync(0xffffffffu, traces, o);
  }
  if (lane) return;
  w.e_nodes[e] = nodes;
  w.e_edges[e] = edges;
  w.e_tot[e] = traces;
}

__global__ void k_evict_sizes(long long T, long long P, long long n_pat, EvictWs w, long long* sizes) {
  sizes[0] = w.tkeep[T];
  sizes[1] = w.pkeep[P];
  sizes[2] = w.pa[n_pat];
  sizes[3] = w.pn[n_pat];
  sizes[4] = w.pe[n_pat];
  sizes[5] = w.pk[n_pat];
}

// thread per old trace t: moves to tkeep[t] if kept; remap[t] = its new index or -1
__global__ void k_evict_apply_traces(PertStore s, PertIngestState g, EvictWs w, PertEvictOut o) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= s.n_traces) return;
  const int j = w.tkeep[t];
  const bool keep = w.tkeep[t + 1] != j;
  o.remap[t] = keep ? j : -1;
  if (!keep) return;
  o.trace_entry[j] = s.trace_entry[t];
  o.trace_ts[j] = s.trace_ts[t];
  o.trace_y[j] = s.trace_y[t];
  o.trace_pat[j] = w.pa[g.trace_pat[t]];
  o.trace_tid[j] = g.trace_tid[t];
}

// thread per old pair i: a kept pair moves to pkeep[i] with its pattern renumbered and its probability recomputed
__global__ void k_evict_apply_pairs(PertStore s, PertIngestState g, EvictWs w, PertMixOut out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n_pairs || w.pkeep[i + 1] == w.pkeep[i]) return;
  const int e = upper_seg(s.ent_ptr, s.n_ent, i);
  emit(out, w.pkeep[i], w.pa[s.ent_pat[i]], g.cnt[i] - w.ev[i], w.e_tot[e]);
}

// thread per entry e <= n_ent: its new pair offset (the kept pairs before it) and totals
__global__ void k_evict_apply_entries(PertStore s, EvictWs w, PertMixOut out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e > s.n_ent) return;
  out.ent_ptr[e] = w.pkeep[s.ent_ptr[e]];
  if (e == s.n_ent) return;
  out.ent_nodes[e] = w.e_nodes[e];
  out.ent_edges[e] = w.e_edges[e];
  out.tot[e] = w.e_tot[e];
}

// thread per old pattern p <= n_pat: the offsets of a kept pattern (and the totals at p = n_pat); pat_new[p]
__global__ void k_evict_apply_pats(PertStore s, EvictWs w, PertEvictOut o) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p > s.n_pat) return;
  const int j = w.pa[p];
  const bool alive = p < s.n_pat && w.pa[p + 1] != j;
  if (p < s.n_pat) o.pat_new[p] = alive ? j : -1;
  if (p < s.n_pat && !alive) return;
  o.pat_nptr[j] = w.pn[p];
  o.pat_eptr[j] = w.pe[p];
  o.key_ptr[j] = w.pk[p];
}

// thread per old node v: the nodes of a kept pattern move as one segment
__global__ void k_evict_apply_nodes(PertStore s, long long n_nodes, EvictWs w, PertEvictOut o) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_nodes) return;
  const int p = upper_seg(s.pat_nptr, s.n_pat, v);
  if (w.pa[p + 1] == w.pa[p]) return;
  const long long j = w.pn[p] + (v - s.pat_nptr[p]);
  o.pat_ms[j] = s.pat_ms[v];
  o.pat_depth[j] = s.pat_depth[v];
  o.pat_last[j] = s.pat_last[v];
}

// thread per old edge x: pattern-local endpoints, so a pure segment move
__global__ void k_evict_apply_edges(PertStore s, long long n_edges, EvictWs w, PertEvictOut o) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n_edges) return;
  const int p = upper_seg(s.pat_eptr, s.n_pat, x);
  if (w.pa[p + 1] == w.pa[p]) return;
  const long long j = w.pe[p] + (x - s.pat_eptr[p]);
  o.pat_src[j] = s.pat_src[x];
  o.pat_dst[j] = s.pat_dst[x];
  for (int c = 0; c < s.attr_cols; ++c) o.pat_attr[j * s.attr_cols + c] = s.pat_attr[x * s.attr_cols + c];
}

// thread per old key row r: the runtime keys move like the nodes
__global__ void k_evict_apply_keys(PertStore s, PertIngestState g, EvictWs w, PertEvictOut o) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= g.n_key_rows) return;
  const int p = upper_seg(g.keys.ptr, s.n_pat, r);
  if (w.pa[p + 1] == w.pa[p]) return;
  const long long j = w.pk[p] + (r - g.keys.ptr[p]);
  const long long ld = g.keys.ld, nld = o.key_ld;
  o.key_rows[j] = g.keys.rows[r];
  o.key_rows[nld + j] = g.keys.rows[ld + r];
  o.key_rows[2 * nld + j] = g.keys.rows[2 * ld + r];
}

constexpr long long IG_MAX = 0x7ffffff0LL;

// the argument checks both eviction calls share
bool evict_args_ok(const PertStore* s, const PertIngestState* g) {
  if (!s || !g || s->n_traces < 0 || s->n_traces > IG_MAX || s->n_pat < 0 || s->n_ent < 0 || g->n_pairs < 0 ||
      g->n_pairs > IG_MAX || g->n_nodes < 0 || g->n_nodes > IG_MAX || g->n_edges < 0 || g->n_edges > IG_MAX ||
      g->n_key_rows < 0 || g->n_key_rows > g->keys.ld || s->attr_cols < 0 || !keys_ok(&g->keys) ||
      g->keys.n != s->n_pat)
    return false;
  if (!s->ent_ptr || !s->pat_nptr || !s->pat_eptr || (s->n_ent > 0 && !g->tot) ||
      (s->n_traces > 0 && (!s->trace_entry || !s->trace_ts || !g->trace_pat)) ||
      (g->n_pairs > 0 && (!s->ent_pat || !g->cnt)))
    return false;
  return true;
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

long long pert_ingest_evict_workspace_bytes(long long n_traces, long long n_pairs, long long n_pat, long long n_ent) {
  if (n_traces < 0 || n_pairs < 0 || n_pat < 0 || n_ent < 0 || n_traces > IG_MAX || n_pairs > IG_MAX ||
      n_pat > IG_MAX || n_ent > IG_MAX)
    return PERT_ERR_BADARG;
  return evict_ws_bytes(n_traces, n_pairs, n_pat, n_ent);
}

int pert_ingest_evict_count(const PertStore* store, const PertIngestState* ing, long long before, void* workspace,
                            long long workspace_bytes, long long* sizes, void* stream) {
  if (!evict_args_ok(store, ing) || !workspace || !sizes) return PERT_ERR_BADARG;
  const long long T = store->n_traces, P = ing->n_pairs, n_pat = store->n_pat, n_ent = store->n_ent;
  if (workspace_bytes < evict_ws_bytes(T, P, n_pat, n_ent)) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const EvictWs w = evict_ws(workspace, T, P, n_pat, n_ent);
  cudaError_t e;
  if ((e = cudaMemsetAsync(w.pkey, 0xff, 8 * w.S, st)) ||
      (e = cudaMemsetAsync(w.pval, 0, (char*)w.bsum - (char*)w.pval, st)))
    return (int)e;
  const int B = IG_THREADS, WB = IG_WARPS * 32;
  if (P > 0) k_pair_table<<<pert_cdiv(P, B), B, 0, st>>>(*store, P, w.S, w.pkey, w.pval);
  if (T > 0) k_evict_traces<<<pert_cdiv(T, B), B, 0, st>>>(*store, ing->trace_pat, before, w);
  if (P > 0) k_evict_pairs<<<pert_cdiv(P, B), B, 0, st>>>(*store, ing->cnt, P, w);
  if (n_pat > 0) k_evict_pat_lens<<<pert_cdiv(n_pat, B), B, 0, st>>>(*store, ing->keys.ptr, w);
  if (n_ent > 0) k_evict_entries<<<pert_cdiv(n_ent * 32, WB), WB, 0, st>>>(*store, ing->cnt, w);
  if (T > 0) scan_launch(w.tkeep, nullptr, T + 1, w.bsum, st);
  if (P > 0) scan_launch(w.pkeep, nullptr, P + 1, w.bsum, st);
  if (n_pat > 0) {
    scan_launch(w.pa, w.pn, n_pat + 1, w.bsum, st);
    scan_launch(w.pe, w.pk, n_pat + 1, w.bsum, st);
  }
  k_evict_sizes<<<1, 1, 0, st>>>(T, P, n_pat, w, sizes);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_ingest_evict_apply(const PertStore* store, const PertIngestState* ing, const long long* sizes,
                            const void* workspace, long long workspace_bytes, const PertEvictOut* out, void* stream) {
  if (!evict_args_ok(store, ing) || !workspace || !sizes || !out) return PERT_ERR_BADARG;
  const long long T = store->n_traces, P = ing->n_pairs, n_pat = store->n_pat, n_ent = store->n_ent;
  if (workspace_bytes < evict_ws_bytes(T, P, n_pat, n_ent)) return PERT_ERR_BADARG;
  const long long T2 = sizes[0], P2 = sizes[1], n_pat2 = sizes[2], N2 = sizes[3], E2 = sizes[4], K2 = sizes[5];
  if (T2 < 0 || T2 > T || P2 < 0 || P2 > P || n_pat2 < 0 || n_pat2 > n_pat || N2 < 0 || N2 > ing->n_nodes ||
      E2 < 0 || E2 > ing->n_edges || K2 < 0 || K2 > ing->n_key_rows || out->key_ld < K2)
    return PERT_ERR_BADARG;
  const PertMixOut& m = out->mix;
  if ((T > 0 && (!ing->trace_tid || !out->remap)) ||
      (T2 > 0 && (!out->trace_entry || !out->trace_ts || !out->trace_y || !out->trace_pat || !out->trace_tid)) ||
      (T > 0 && !store->trace_y) || !m.ent_ptr || (n_ent > 0 && (!m.ent_nodes || !m.ent_edges || !m.tot)) ||
      (P2 > 0 && (!m.ent_pat || !m.ent_prob || !m.cnt)) || (n_pat > 0 && !out->pat_new) || !out->pat_nptr ||
      !out->pat_eptr || !out->key_ptr)
    return PERT_ERR_BADARG;
  if ((ing->n_nodes > 0 && (!store->pat_ms || !store->pat_depth || !store->pat_last)) ||
      (N2 > 0 && (!out->pat_ms || !out->pat_depth || !out->pat_last)) ||
      (ing->n_edges > 0 && (!store->pat_src || !store->pat_dst || (store->attr_cols > 0 && !store->pat_attr))) ||
      (E2 > 0 && (!out->pat_src || !out->pat_dst || (store->attr_cols > 0 && !out->pat_attr))) ||
      (K2 > 0 && !out->key_rows))
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const EvictWs w = evict_ws((void*)workspace, T, P, n_pat, n_ent);
  const int B = IG_THREADS;
  if (T > 0) k_evict_apply_traces<<<pert_cdiv(T, B), B, 0, st>>>(*store, *ing, w, *out);
  if (P > 0) k_evict_apply_pairs<<<pert_cdiv(P, B), B, 0, st>>>(*store, *ing, w, m);
  k_evict_apply_entries<<<pert_cdiv(n_ent + 1, B), B, 0, st>>>(*store, w, m);
  k_evict_apply_pats<<<pert_cdiv(n_pat + 1, B), B, 0, st>>>(*store, w, *out);
  if (ing->n_nodes > 0) k_evict_apply_nodes<<<pert_cdiv(ing->n_nodes, B), B, 0, st>>>(*store, ing->n_nodes, w, *out);
  if (ing->n_edges > 0) k_evict_apply_edges<<<pert_cdiv(ing->n_edges, B), B, 0, st>>>(*store, ing->n_edges, w, *out);
  if (ing->n_key_rows > 0) k_evict_apply_keys<<<pert_cdiv(ing->n_key_rows, B), B, 0, st>>>(*store, *ing, w, *out);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
