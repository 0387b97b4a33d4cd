// Raw call-graph and resource rows -> the processed span and resource tables: the else-branch of the reference's
// preprocess.py get_df() (:191-266) on dictionary-encoded columns.
//
// The host reads the CSV files and gives every string (and every rpcid value) a dictionary code; everything after that
// is integer and float work over the whole table, restated here step by step:
//   1. drop_duplicates (:212): an open-addressing table over a 64-bit row hash; a slot matches only after a column-by-
//      column comparison with its owner, so a collision costs a comparison and never merges two rows.  atomicMin of the
//      row index per slot keeps the first row in concatenation order;
//   2. sort_values("timestamp") (:213): done by the caller as a stable sort of the kept rows' timestamps (ties keep
//      concatenation order); ``order`` maps sorted position -> row;
//   3. map_consecutive_ids (:216-221): for every dictionary code, atomicMin of its first position, then a scan of the
//      "first position" flags numbers the codes by first appearance (Series.factorize).  traceid and interface over the
//      whole sorted table, entryid / rpcid / rpctype over the rows of traces that keep an entry, so the later filters
//      leave gaps in the codes exactly as in the reference;
//   4. filter_traces_with_missing_entry_and_get_delay (:99-149): per trace (atomics on its dictionary code) the minimum
//      timestamp is the timestamp at its first sorted position, max |rt| an atomicMax; candidates are the http rows at
//      that timestamp with that |rt|; one candidate is the entry, several are narrowed to um == "(?)" and kept only if
//      exactly one is left.  The entry key (dm, interface code) is factorised through a second hash table;
//   5. filter_traces_with_missing_features (:155-177): the distinct {um, dm} of a trace are the first claims of
//      (trace, ms) pairs in a third table; kept iff (double) resourced / (double) distinct >= 0.6;
//   6. filter_traces_by_occurence_per_entry (:180-188): traces surviving 5 counted per entry, kept iff > min_occurence;
//   7. microservice ids (:248-254): the union of the surviving um / dm and every resource msname, numbered by a scan of
//      presence flags over the dictionary, whose codes are in lexicographic name order;
//   8. compaction of the surviving rows into the nine processed columns;
//   9. the resource groupby(["timestamp", "msname"]).agg([max, min, mean, median]) (:227-242): a thread per group walks
//      its rows in concatenation order (the caller's stable key sort) with pandas' group_max / group_min / group_mean
//      (Kahan-compensated sum over the non-NaN count) and reads the median from the caller's per-group value sort.
// Every atomic is a min, a max, an add or a slot claim whose winner changes no output, so results do not depend on
// scheduling.
// The chunks of a stream (pert_raw_stream_*, rawtable.RawStream) run the same passes, instantiated with S = true: every
// chunk code is read through its map to a stream code, only values without an id are flagged at their first position
// (so the scans rank the new ones), entries are looked up in a persistent (dm, interface) table, coverage and the
// occurrence counts are cumulative, and the new ids go into fresh state arrays the host swaps in.
#include "common.cuh"
#include "rowhash.cuh"
#include "scan.cuh"

#include <algorithm>

namespace {

constexpr int RW_NONE = 0x7f7f7f7f;                     // "no position yet": the 0x7f byte fill of every atomicMin
constexpr long long RW_MAX_ROWS = 1LL << 30;            // rows and traceids: every table slot fits an int
constexpr unsigned long long RW_NOKEY = ~0ull;
constexpr long long RW_WIN_MAX = 0x7ffffff0LL;          // window keys, samples and batch sizes: int32 offsets and scans
constexpr unsigned long long RW_SEED = 0x452821e638d01377ull;

__device__ __forceinline__ bool in_dict(int64_t v, long long n) { return v >= 0 && v < n; }

__device__ __forceinline__ bool codes_ok(const PertRawCalls& c, long long r) {
  return in_dict(c.traceid[r], c.n_trace) && in_dict(c.interface[r], c.n_iface) && in_dict(c.rpcid[r], c.n_rpcid) &&
         in_dict(c.rpctype[r], c.n_rpctype) && in_dict(c.um[r], c.n_ms) && in_dict(c.dm[r], c.n_ms);
}

__device__ __forceinline__ unsigned long long row_hash(const PertRawCalls& c, long long r) {
  unsigned long long h = mix64(RW_SEED ^ (unsigned long long)c.traceid[r]);
  h = mix64(h ^ (unsigned long long)c.timestamp[r]);
  h = mix64(h ^ (unsigned long long)c.rpcid[r]);
  h = mix64(h ^ (unsigned long long)c.um[r]);
  h = mix64(h ^ (unsigned long long)c.rpctype[r]);
  h = mix64(h ^ (unsigned long long)c.dm[r]);
  h = mix64(h ^ (unsigned long long)c.interface[r]);
  return mix64(h ^ (unsigned long long)c.rt[r]);
}

__device__ __forceinline__ bool same_row(const PertRawCalls& c, long long a, long long b) {
  return c.traceid[a] == c.traceid[b] && c.timestamp[a] == c.timestamp[b] && c.rpcid[a] == c.rpcid[b] &&
         c.um[a] == c.um[b] && c.rpctype[a] == c.rpctype[b] && c.dm[a] == c.dm[b] &&
         c.interface[a] == c.interface[b] && c.rt[a] == c.rt[b];
}

__device__ __forceinline__ int64_t abs64(int64_t v) { return v < 0 ? -v : v; }

// ---- 1. drop_duplicates ----------------------------------------------------------------------------------------------
__global__ void k_dedup_insert(PertRawCalls c, long long S, int hash_bits, int* owner, int* first, int* slot_of,
                               int* status) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= c.R) return;
  if (!codes_ok(c, r)) {                                 // reported, and the row is left out
    atomicExch(status, PERT_ERR_RANGE);
    slot_of[r] = -1;
    return;
  }
  long long s = (long long)(mix64(row_hash(c, r) & hash_mask(hash_bits)) & (unsigned long long)(S - 1));
  for (;;) {
    const int o = atomicCAS(&owner[s], -1, (int)r);
    if (o == -1 || same_row(c, o, r)) break;
    s = (s + 1) & (S - 1);
  }
  atomicMin(&first[s], (int)r);
  slot_of[r] = (int)s;
}

__global__ void k_dedup_flags(long long R, const int* slot_of, const int* first, int* flags) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int s = slot_of[r];
  flags[r + 1] = s >= 0 && first[s] == r;
}

__global__ void k_dedup_compact(PertRawCalls c, const int* flags, int* rows, int64_t* keys, int64_t* n_kept) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= c.R) return;
  const int q = flags[r];
  if (flags[r + 1] != q) {
    rows[q] = (int)r;
    keys[q] = c.timestamp[r];
  }
  if (r == c.R - 1) *n_kept = flags[c.R];
}

// ---- 3.-8. over the sorted kept rows: position p holds row order[p] ----------------------------------------------------
struct Work {                 // carved from the caller's workspace by layout()
  int *fl_tr, *fl_if, *fl_ent, *fl_rpc, *fl_rty, *fl_row;           // [N+1] first-position / survivor flags, scanned
  int *first_tr, *first_if, *first_rpc, *first_rty;                 // [dictionary] first position of every code
  int *fl_ms;                                                       // [n_ms+1] microservice presence, scanned
  int *ncand, *nq, *cand_pos, *q_pos, *epos, *eslot, *ndist, *nres, *covered;   // [n_trace] per trace
  int64_t* amax;                                                    // [n_trace] max |rt|
  unsigned long long *ekey, *pkey;                                  // [SE], [SP] entry / (trace, ms) tables
  int *efirst, *ecnt;                                               // [SE]
  int* bsum;
  int64_t *cid_ms, *cid_if, *cid_rpc, *cid_rty;                    // stream only: [dictionary] id so far, -1 none
  int64_t* eid;                                                     // stream only: [SE] entry id of a slot's key, -1
  long long SE, SP;
};

long long pow2_at_least(long long n) {
  long long S = 64;
  while (S < n) S <<= 1;
  return S;
}

long long scan_bytes(long long L) { return 2LL * pert_cdiv(L, SCAN_TILE) * 4 + 16; }

// bytes of the workspace of pert_raw_process / pert_raw_emit (stream: of the _stream_ pair); w != NULL also carves it
long long layout(const PertRawCalls& c, long long N, void* base, Work* w, bool stream = false) {
  const long long SE = pow2_at_least(2 * c.n_trace), SP = pow2_at_least(4 * N);
  long long off = 0;
  auto take = [&](long long bytes) {
    char* p = base ? (char*)base + off : nullptr;
    off += (bytes + 15) / 16 * 16;
    return (void*)p;
  };
  Work x;
  x.SE = SE;
  x.SP = SP;
  x.ekey = (unsigned long long*)take(8 * SE);
  x.pkey = (unsigned long long*)take(8 * SP);
  x.amax = (int64_t*)take(8 * c.n_trace);
  int** flags[] = {&x.fl_tr, &x.fl_if, &x.fl_ent, &x.fl_rpc, &x.fl_rty, &x.fl_row};
  for (int** f : flags) *f = (int*)take(4 * (N + 1));
  x.first_tr = (int*)take(4 * c.n_trace);
  x.first_if = (int*)take(4 * c.n_iface);
  x.first_rpc = (int*)take(4 * c.n_rpcid);
  x.first_rty = (int*)take(4 * c.n_rpctype);
  x.fl_ms = (int*)take(4 * (c.n_ms + 1));
  int** per_trace[] = {&x.ncand, &x.nq, &x.cand_pos, &x.q_pos, &x.epos, &x.eslot, &x.ndist, &x.nres, &x.covered};
  for (int** f : per_trace) *f = (int*)take(4 * c.n_trace);
  x.efirst = (int*)take(4 * SE);
  x.ecnt = (int*)take(4 * SE);
  x.bsum = (int*)take(scan_bytes(std::max(N, c.n_ms) + 1));
  x.cid_ms = x.cid_if = x.cid_rpc = x.cid_rty = x.eid = nullptr;
  if (stream) {
    x.cid_ms = (int64_t*)take(8 * c.n_ms);
    x.cid_if = (int64_t*)take(8 * c.n_iface);
    x.cid_rpc = (int64_t*)take(8 * c.n_rpcid);
    x.cid_rty = (int64_t*)take(8 * c.n_rpctype);
    x.eid = (int64_t*)take(8 * SE);
  }
  if (w) *w = x;
  return off;
}

__global__ void k_first_codes(PertRawCalls c, long long N, const int64_t* order, Work w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int64_t tr = c.traceid[r];
  atomicMin(&w.first_tr[tr], (int)p);
  atomicMin(&w.first_if[c.interface[r]], (int)p);
  atomicMax((long long*)&w.amax[tr], (long long)abs64(c.rt[r]));
}

// stream (S): the id a chunk code already has (-1: none), and the id of a code: its old one, or next + rank
template <bool S>
__device__ __forceinline__ int64_t id_of(const int64_t* cid, long long next, const int* fl, const int* first,
                                         int64_t code) {
  if (S) {
    const int64_t k = cid[code];
    if (k >= 0) return k;
    return next + fl[first[code]];
  }
  return fl[first[code]];
}

// the entry table of a stream: open addressing, linear probing, load <= 1/2
__device__ __forceinline__ int64_t ent_find(const unsigned long long* keys, const int64_t* ids, long long cap,
                                            unsigned long long key) {
  long long s = (long long)(mix64(key) & (unsigned long long)(cap - 1));
  for (;;) {
    const unsigned long long o = keys[s];
    if (o == key) return ids[s];
    if (o == RW_NOKEY) return -1;
    s = (s + 1) & (cap - 1);
  }
}

__device__ __forceinline__ void ent_insert(unsigned long long* keys, int64_t* ids, long long cap,
                                           unsigned long long key, int64_t id) {
  long long s = (long long)(mix64(key) & (unsigned long long)(cap - 1));
  while (atomicCAS(&keys[s], RW_NOKEY, key) != RW_NOKEY) s = (s + 1) & (cap - 1);   // keys inserted are distinct
  ids[s] = id;
}

// stream: every chunk code's id so far through its map (a stream code past the id array is new), and has_res OR-ed
// with the stream's
__global__ void k_stream_gather(PertRawCalls c, PertRawState s, int* has_res, Work w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto old = [](const int64_t* map, const int64_t* id, long long n, long long k) -> int64_t {
    const int64_t v = map[k];
    return v >= 0 && v < n ? id[v] : -1;
  };
  if (i < c.n_ms) {
    w.cid_ms[i] = old(s.ms_map, s.ms_id, s.n_ms_codes, i);
    const int64_t v = s.ms_map[i];
    if (v >= 0 && v < s.n_ms_codes && s.has_res[v]) has_res[i] = 1;
  }
  if (i < c.n_iface) w.cid_if[i] = old(s.if_map, s.if_id, s.n_if_codes, i);
  if (i < c.n_rpcid) w.cid_rpc[i] = old(s.rpc_map, s.rpc_id, s.n_rpc_codes, i);
  if (i < c.n_rpctype) w.cid_rty[i] = old(s.rty_map, s.rty_id, s.n_rty_codes, i);
}

// first-position flags of traceid / interface (S: interfaces without an id only); entry candidates: http, the trace's
// first timestamp, its max |rt|
template <bool S>
__global__ void k_candidates(PertRawCalls c, long long N, const int64_t* order, Work w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int64_t tr = c.traceid[r];
  const int f = w.first_tr[tr];
  w.fl_tr[p + 1] = f == p;
  w.fl_if[p + 1] = w.first_if[c.interface[r]] == p && (!S || w.cid_if[c.interface[r]] < 0);
  const int64_t ts = c.timestamp[r];
  if (c.rpctype[r] == c.http && ts == c.timestamp[order[f]] && abs64(c.rt[r]) == w.amax[tr]) {
    atomicAdd(&w.ncand[tr], 1);
    atomicMin(&w.cand_pos[tr], (int)p);
    if (c.um[r] == c.unknown) {
      atomicAdd(&w.nq[tr], 1);
      atomicMin(&w.q_pos[tr], (int)p);
    }
  }
}

// per trace (dictionary code): its entry row, and the slot of its (dm, interface) key in the entry table (S: stream
// codes, and the id the stream's table holds for the key)
template <bool S>
__global__ void k_entries(PertRawCalls c, const int64_t* order, PertRawState st, Work w) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= c.n_trace) return;
  int e = -1;
  if (w.first_tr[k] != RW_NONE) {
    const int n = w.ncand[k];
    e = n == 1 ? w.cand_pos[k] : (n > 1 && w.nq[k] == 1 ? w.q_pos[k] : -1);
  }
  w.epos[k] = e;
  w.eslot[k] = -1;
  if (e < 0) return;
  const long long r = order[e];
  const unsigned long long key =
      S ? ((unsigned long long)st.ms_map[c.dm[r]] << 32) | (unsigned long long)st.if_map[c.interface[r]]
        : ((unsigned long long)c.dm[r] << 32) | (unsigned long long)c.interface[r];
  long long s = (long long)(mix64(key) & (unsigned long long)(w.SE - 1));
  for (;;) {
    const unsigned long long o = atomicCAS(&w.ekey[s], RW_NOKEY, key);
    if (o == RW_NOKEY || o == key) break;
    s = (s + 1) & (w.SE - 1);
  }
  w.eslot[k] = (int)s;
  if (S) w.eid[s] = ent_find(st.ent_key, st.ent_id, st.ent_cap, key);   // every trace of the key writes the same
}

__device__ __forceinline__ void claim_pair(const Work& w, int64_t tr, int64_t ms, const int* has_res) {
  const unsigned long long key = ((unsigned long long)tr << 32) | (unsigned long long)ms;
  long long s = (long long)(mix64(key) & (unsigned long long)(w.SP - 1));
  for (;;) {
    const unsigned long long o = atomicCAS(&w.pkey[s], RW_NOKEY, key);
    if (o == key) return;                                // the trace already counted this microservice
    if (o == RW_NOKEY) break;
    s = (s + 1) & (w.SP - 1);
  }
  atomicAdd(&w.ndist[tr], 1);
  if (has_res[ms]) atomicAdd(&w.nres[tr], 1);
}

// rows of traces with an entry: first positions of entryid / rpcid / rpctype, and the distinct (trace, ms) pairs
__global__ void k_entry_rows(PertRawCalls c, long long N, const int64_t* order, const int* has_res, Work w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int64_t tr = c.traceid[r];
  const int s = w.eslot[tr];
  if (s < 0) return;
  atomicMin(&w.efirst[s], (int)p);
  atomicMin(&w.first_rpc[c.rpcid[r]], (int)p);
  atomicMin(&w.first_rty[c.rpctype[r]], (int)p);
  claim_pair(w, tr, c.um[r], has_res);
  claim_pair(w, tr, c.dm[r], has_res);
}

template <bool S>
__global__ void k_entry_flags(PertRawCalls c, long long N, const int64_t* order, Work w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int s = w.eslot[c.traceid[r]];
  const bool ok = s >= 0;
  w.fl_ent[p + 1] = ok && w.efirst[s] == p && (!S || w.eid[s] < 0);
  w.fl_rpc[p + 1] = ok && w.first_rpc[c.rpcid[r]] == p && (!S || w.cid_rpc[c.rpcid[r]] < 0);
  w.fl_rty[p + 1] = ok && w.first_rty[c.rpctype[r]] == p && (!S || w.cid_rty[c.rpctype[r]] < 0);
}

// resource coverage (IEEE double quotient, as Python's int / int) and the per-entry trace count of the survivors
__global__ void k_coverage(long long n_trace, Work w) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_trace) return;
  const int s = w.eslot[k];
  const bool cov = s >= 0 && (double)w.nres[k] / (double)w.ndist[k] >= 0.6;
  w.covered[k] = cov;
  if (cov) atomicAdd(&w.ecnt[s], 1);
}

template <bool S>
__global__ void k_ms_init(long long n_ms, const int* has_res, Work w) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m < n_ms) w.fl_ms[m + 1] = has_res[m] != 0 && (!S || w.cid_ms[m] < 0);
}

// S: an entry's count is the stream's so far plus this chunk's, and only microservices without an id are flagged
template <bool S>
__global__ void k_survivors(PertRawCalls c, long long N, const int64_t* order, long long min_occurence,
                            PertRawState st, Work w) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int64_t tr = c.traceid[r];
  const int s = w.eslot[tr];
  long long cnt = s >= 0 ? w.ecnt[s] : 0;
  if (S && s >= 0 && w.eid[s] >= 0) cnt += st.ent_cnt[w.eid[s]];
  const bool keep = s >= 0 && w.covered[tr] && cnt > min_occurence;
  w.fl_row[p + 1] = keep;
  if (keep) {
    if (!S || w.cid_ms[c.um[r]] < 0) w.fl_ms[c.um[r] + 1] = 1;
    if (!S || w.cid_ms[c.dm[r]] < 0) w.fl_ms[c.dm[r] + 1] = 1;
  }
}

__global__ void k_sizes(long long N, long long n_ms, Work w, int64_t* sizes) {
  sizes[0] = w.fl_row[N];
  sizes[1] = w.fl_ms[n_ms];
  sizes[2] = w.fl_tr[N];
  sizes[3] = w.fl_if[N];
  sizes[4] = w.fl_ent[N];
  sizes[5] = w.fl_rpc[N];
  sizes[6] = w.fl_rty[N];
}

// S: ids continue the stream's counters, new ones are written into the fresh state (so), and every entry of the chunk
// (new or not) adds its covered traces to its count
template <bool S>
__global__ void k_emit_rows(PertRawCalls c, long long N, const int64_t* order, Work w, PertRawOut o, PertRawState st,
                            PertRawStateOut so) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const long long r = order[p];
  const int64_t tr = c.traceid[r], itf = c.interface[r];
  // dictionaries: the code each new id was given at its first position
  if (w.fl_tr[p + 1] != w.fl_tr[p]) o.tr_code[w.fl_tr[p]] = tr;
  if (w.fl_if[p + 1] != w.fl_if[p]) {
    o.if_code[w.fl_if[p]] = itf;
    if (S) so.if_id[st.if_map[itf]] = st.n_if + w.fl_if[p];
  }
  if (w.fl_rpc[p + 1] != w.fl_rpc[p]) {
    o.rpc_code[w.fl_rpc[p]] = c.rpcid[r];
    if (S) so.rpc_id[st.rpc_map[c.rpcid[r]]] = st.n_rpc + w.fl_rpc[p];
  }
  if (w.fl_rty[p + 1] != w.fl_rty[p]) {
    o.rty_code[w.fl_rty[p]] = c.rpctype[r];
    if (S) so.rty_id[st.rty_map[c.rpctype[r]]] = st.n_rty + w.fl_rty[p];
  }
  if (w.fl_ent[p + 1] != w.fl_ent[p]) {
    const long long er = order[w.epos[tr]];
    o.ent_dm[w.fl_ent[p]] = c.dm[er];
    o.ent_if[w.fl_ent[p]] = id_of<S>(w.cid_if, st.n_if, w.fl_if, w.first_if, c.interface[er]);
  }
  const int es = w.eslot[tr];
  if (S && es >= 0 && w.efirst[es] == p) {
    const int64_t known = w.eid[es];
    const int64_t e = known >= 0 ? known : st.n_ent + w.fl_ent[p];
    so.ent_cnt[e] = (known >= 0 ? st.ent_cnt[known] : 0) + w.ecnt[es];
    if (known < 0) ent_insert(so.ent_key, so.ent_id, so.ent_cap2, w.ekey[es], e);
  }
  const int q = w.fl_row[p];
  if (w.fl_row[p + 1] == q) return;
  o.traceid[q] = (S ? st.n_tr : 0) + w.fl_tr[w.first_tr[tr]];
  o.timestamp[q] = c.timestamp[r];
  o.rpcid[q] = id_of<S>(w.cid_rpc, st.n_rpc, w.fl_rpc, w.first_rpc, c.rpcid[r]);
  o.um[q] = S ? (w.cid_ms[c.um[r]] >= 0 ? w.cid_ms[c.um[r]] : st.n_ms + w.fl_ms[c.um[r]]) : w.fl_ms[c.um[r]];
  o.dm[q] = S ? (w.cid_ms[c.dm[r]] >= 0 ? w.cid_ms[c.dm[r]] : st.n_ms + w.fl_ms[c.dm[r]]) : w.fl_ms[c.dm[r]];
  o.interface[q] = id_of<S>(w.cid_if, st.n_if, w.fl_if, w.first_if, itf);
  o.rpctype[q] = id_of<S>(w.cid_rty, st.n_rty, w.fl_rty, w.first_rty, c.rpctype[r]);
  o.rt[q] = c.rt[r];
  o.entryid[q] = S && w.eid[es] >= 0 ? w.eid[es] : (S ? st.n_ent : 0) + w.fl_ent[w.efirst[es]];
  o.row[q] = r;
}

// microservice id of a valid chunk code (S: the stream's, or next + rank among the chunk's new names)
template <bool S>
__device__ __forceinline__ int64_t ms_id_of(const Work& w, const PertRawState& st, int64_t m) {
  return S && w.cid_ms[m] >= 0 ? w.cid_ms[m] : (S ? st.n_ms : 0) + w.fl_ms[m];
}

template <bool S>
__global__ void k_emit_ms(long long n_ms, Work w, int64_t* ms_code, const int* has_res, PertRawState st,
                          PertRawStateOut so) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_ms) return;
  if (w.fl_ms[m + 1] != w.fl_ms[m]) {
    ms_code[w.fl_ms[m]] = m;
    if (S) so.ms_id[st.ms_map[m]] = st.n_ms + w.fl_ms[m];
  }
  if (S && has_res[m]) so.has_res[st.ms_map[m]] = 1;
}

template <bool S>
__global__ void k_emit_res(long long G, long long n_ms, const int64_t* g_ts, const int64_t* g_ms, Work w,
                           int64_t* res_index, PertRawState st) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int64_t m = g_ms[g];
  res_index[2 * g] = g_ts[g];
  res_index[2 * g + 1] = in_dict(m, n_ms) ? ms_id_of<S>(w, st, m) : -1;   // groups hold valid codes only; guarded
}

// stream: the microservice id of every raw resource row (-1: an ms outside the chunk dictionary, left out)
__global__ void k_resource_ms(long long K, long long n_ms, const int64_t* r_ms, Work w, PertRawState st,
                              int64_t* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K) return;
  const int64_t m = r_ms[i];
  out[i] = in_dict(m, n_ms) ? ms_id_of<true>(w, st, m) : -1;
}

// stream: the old entry table into a larger fresh one
__global__ void k_ent_rehash(const unsigned long long* keys, const int64_t* ids, long long cap, unsigned long long* keys2,
                             int64_t* ids2, long long cap2) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < cap && keys[s] != RW_NOKEY) ent_insert(keys2, ids2, cap2, keys[s], ids[s]);
}

// ---- 9. resource groups ----------------------------------------------------------------------------------------------
__global__ void k_res_flags(long long K, const int64_t* ts, const int64_t* ms, const int64_t* perm, long long n_ms,
                            int* gflag, int* has_res, int* status) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  const long long r = perm[p];
  const int64_t m = ms[r];
  if (!in_dict(m, n_ms)) {                               // reported, and the row is left out of every group
    atomicExch(status, PERT_ERR_RANGE);
    gflag[p + 1] = 0;
    return;
  }
  has_res[m] = 1;
  bool start = p == 0;
  if (!start) {
    const long long q = perm[p - 1];
    start = ts[q] != ts[r] || ms[q] != m;
  }
  gflag[p + 1] = start;
}

// valid rows come first in perm (rows with an ms outside [0, n_ms) last), so the groups are the valid prefix
__global__ void k_res_groups(long long K, long long n_ms, const int64_t* ts, const int64_t* ms, const int64_t* perm,
                             const int* gflag, int* gptr, int64_t* g_ts, int64_t* g_ms, int64_t* n_groups) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  if (p == K - 1) *n_groups = gflag[K];
  const long long r = perm[p];
  if (!in_dict(ms[r], n_ms)) return;
  const int g = gflag[p];
  if (gflag[p + 1] != g) {
    gptr[g] = (int)p;
    g_ts[g] = ts[r];
    g_ms[g] = ms[r];
  }
  if (p == K - 1 || !in_dict(ms[perm[p + 1]], n_ms)) gptr[gflag[p + 1]] = (int)(p + 1);   // end of the last group
}

struct GroupStats {
  double mx = -INFINITY, mn = INFINITY, sum = 0.0, comp = 0.0;
  long long nobs = 0;
  // pandas group_max / group_min (strict compare, first value kept on ties) and group_mean (Kahan, :GH#50367 reset of
  // a NaN compensation after an infinite value)
  __device__ __forceinline__ void add(double v) {
    if (v != v) return;
    ++nobs;
    if (v > mx) mx = v;
    if (v < mn) mn = v;
    const double y = __dsub_rn(v, comp);
    const double t = __dadd_rn(sum, y);
    comp = __dsub_rn(__dsub_rn(t, sum), y);
    if (comp != comp) comp = 0.0;
    sum = t;
  }
};

// median of the nobs non-NaN values at the front of a group's ascending sort (NaN sorts last)
__device__ __forceinline__ double median_of(const double* sorted, long long nobs) {
  if (nobs == 0) return NAN;
  const long long h = nobs / 2;
  if (nobs % 2) return sorted[h];
  return __ddiv_rn(__dadd_rn(sorted[h], sorted[h - 1]), 2.0);
}

// the 8 statistics of one group from its folds and its ascending value runs (NaN last)
__device__ __forceinline__ void put_stats(const GroupStats& a, const GroupStats& m, const double* cpu_sorted,
                                          const double* mem_sorted, double* out) {
  const GroupStats* st[2] = {&a, &m};
  const double* sorted[2] = {cpu_sorted, mem_sorted};
  for (int j = 0; j < 2; ++j) {
    const GroupStats& s = *st[j];
    const bool none = s.nobs == 0;
    out[4 * j + 0] = none ? NAN : s.mx;
    out[4 * j + 1] = none ? NAN : s.mn;
    out[4 * j + 2] = none ? NAN : __ddiv_rn(s.sum, (double)s.nobs);
    out[4 * j + 3] = median_of(sorted[j], s.nobs);
  }
}

__global__ void k_res_stats(long long G, const int64_t* perm, const int* gptr, const double* cpu, const double* mem,
                            const double* cpu_sorted, const double* mem_sorted, double* vals) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int b = gptr[g], e = gptr[g + 1];
  GroupStats a, m;
  for (int p = b; p < e; ++p) {
    const long long r = perm[p];
    a.add(cpu[r]);
    m.add(mem[r]);
  }
  put_stats(a, m, cpu_sorted + b, mem_sorted + b, vals + 8 * g);
}

// ---- the open-bucket sample window (ResourceSampleWindow) ---------------------------------------------------------
// Window state: keys[U] (sorted unique ts * n_ms + ms), off[U+1] (run offsets), st[U][2] (the GroupStats fold of cpu
// and memory) and the runs cpu_run / mem_run [S]: every key's values ascending in the order of vo_lt, ties in arrival
// order.  A batch is given sorted by key (stable, so arrival order within a key), and each column also as bsorted[k]:
// the batch's values of each key ascending (ties in arrival order) at the key's positions.
static_assert(sizeof(GroupStats) == 40, "the window stores GroupStats as 5 doubles per column");

// value order of the runs: NaN above every number and equal to NaN; -0.0 == 0.0 (IEEE compare)
__device__ __forceinline__ bool vo_lt(double a, double b) { return a < b || (b != b && a == a); }

__device__ __forceinline__ int64_t floor_div(int64_t a, long long n) {
  int64_t q = a / n;
  return (a % n != 0 && a < 0) ? q - 1 : q;
}

__device__ __forceinline__ long long lower_bound(const int64_t* a, long long n, int64_t v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// #values of the ascending run a[0, n) that are below v (le = false) or not above v (le = true)
__device__ __forceinline__ int count_below(const double* a, int n, double v, bool le) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (le ? !vo_lt(v, a[mid]) : vo_lt(a[mid], v)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// flags[0..k] / flags[k+1..2k+1]: 1 at p + 1 if batch position p starts a key that is not late (fu), and one that is
// also absent from the window (fn); slot 0 of each is 0.  Scanned, fu[p] / fn[p] count such starts before p.
__global__ void k_win_flags(long long k, const int64_t* bkeys, long long n_ms, long long seal, long long U,
                            const int64_t* keys, int* fu, int* fn) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= k) return;
  if (p == 0) fu[0] = fn[0] = 0;
  const int64_t key = bkeys[p];
  const bool first = floor_div(key, n_ms) >= seal && (p == 0 || bkeys[p - 1] != key);
  bool fresh = false;
  if (first) {
    const long long j = lower_bound(keys, U, key);
    fresh = j == U || keys[j] != key;
  }
  fu[p + 1] = first;
  fn[p + 1] = fresh;
}

// sizes = {late samples (a prefix of the sorted batch), keys the batch touches, keys after the merge}
__global__ void k_win_sizes(long long k, const int64_t* bkeys, long long n_ms, long long seal, long long U,
                            const int* fu, const int* fn, int64_t* sizes) {
  long long lo = 0, hi = k;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (floor_div(bkeys[mid], n_ms) < seal) lo = mid + 1; else hi = mid;
  }
  sizes[0] = lo;
  sizes[1] = k ? fu[k] : 0;
  sizes[2] = U + (k ? fn[k] : 0);
}

// the key merge: every old key and every touched key finds its slot of the merged table; each slot field is written
// once.  src[s]: old index or -1; bsrc[s]: touched key index or -1; opos[j]: slot of old key j; ustart[b]: first batch
// position of touched key b (ustart[u] = k); upos[b]: its slot.
__global__ void k_win_keys(long long U, const int64_t* keys, long long k, const int64_t* bkeys, const int* fu,
                           const int* fn, int64_t* keys2, int* src, int* bsrc, int* opos, int* ustart, int* upos) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < U) {
    const int64_t key = keys[t];
    const long long lb = lower_bound(bkeys, k, key);
    const int pos = (int)(t + fn[lb]);
    keys2[pos] = key;
    src[pos] = (int)t;
    opos[t] = pos;
    if (lb == k || bkeys[lb] != key) bsrc[pos] = -1;
  }
  if (t < k) {
    if (t == k - 1) ustart[fu[k]] = (int)k;
    if (fu[t + 1] == fu[t]) return;                      // late, or not the first sample of its key
    const int64_t key = bkeys[t];
    const int b = fu[t];
    const long long j = lower_bound(keys, U, key);
    const int pos = (int)(j + fn[t]);
    ustart[b] = (int)t;
    upos[b] = pos;
    bsrc[pos] = b;
    if (j == U || keys[j] != key) {
      keys2[pos] = key;
      src[pos] = -1;
    }
  }
}

// the fold: each slot continues its key's GroupStats over the key's batch samples in arrival order (untouched keys
// copy theirs) and writes its run length at cnt[s + 1]
__global__ void k_win_fold(long long U2, const int* src, const int* bsrc, const int* ustart, const int* off,
                           const GroupStats* st, const int64_t* perm, const double* cpu, const double* mem,
                           GroupStats* st2, int* cnt) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= U2) return;
  if (s == 0) cnt[0] = 0;
  const int j = src[s], b = bsrc[s];
  GroupStats a, m;
  int n = 0;
  if (j >= 0) {
    a = st[2 * j];
    m = st[2 * j + 1];
    n = off[j + 1] - off[j];
  }
  if (b >= 0) {
    const int e = ustart[b + 1];
    for (int p = ustart[b]; p < e; ++p) {
      const long long r = perm[p];
      a.add(cpu[r]);
      m.add(mem[r]);
    }
    n += e - ustart[b];
  }
  st2[2 * s] = a;
  st2[2 * s + 1] = m;
  cnt[s + 1] = n;
}

// the run merge, one thread per value: old value i of key K goes to off2(K) + i + #(batch values of K below it), batch
// value i to off2(K) + i + #(old values of K not above it), so ties keep arrival order
__global__ void k_win_runs(long long U, long long S, const int* off, const double* cpu_run, const double* mem_run,
                           long long n_late, long long n_new, const int* fu, const int* ustart, const int* upos,
                           const double* cpu_sorted, const double* mem_sorted, const int* src, const int* bsrc,
                           const int* opos, const int* off2, double* cpu_run2, double* mem_run2) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < S) {
    int lo = 0, hi = (int)U - 1;                         // the key j with off[j] <= t < off[j + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const int pos = opos[lo], b = bsrc[pos];
    const long long dst = off2[pos] + (t - off[lo]);
    const double c = cpu_run[t], m = mem_run[t];
    if (b < 0) {
      cpu_run2[dst] = c;
      mem_run2[dst] = m;
    } else {
      const int bb = ustart[b], bn = ustart[b + 1] - bb;
      cpu_run2[dst + count_below(cpu_sorted + bb, bn, c, false)] = c;
      mem_run2[dst + count_below(mem_sorted + bb, bn, m, false)] = m;
    }
  } else if (t < S + n_new) {
    const long long p = n_late + (t - S);
    const int b = fu[p + 1] - 1, pos = upos[b], j = src[pos];
    const long long dst = off2[pos] + (p - ustart[b]);
    const double c = cpu_sorted[p], m = mem_sorted[p];
    if (j < 0) {
      cpu_run2[dst] = c;
      mem_run2[dst] = m;
    } else {
      const int ob = off[j], on = off[j + 1] - ob;
      cpu_run2[dst + count_below(cpu_run + ob, on, c, true)] = c;
      mem_run2[dst + count_below(mem_run + ob, on, m, true)] = m;
    }
  }
}

// (timestamp, ms) and the 8 statistics of n slots: slot[i], or slot i itself when slot is NULL
__global__ void k_win_emit(long long n, const int* slot, const int64_t* keys, const int* off, const GroupStats* st,
                           const double* cpu_run, const double* mem_run, long long n_ms, int64_t* index,
                           double* vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long s = slot ? slot[i] : i;
  const int64_t key = keys[s], ts = floor_div(key, n_ms);
  index[2 * i] = ts;
  index[2 * i + 1] = key - ts * n_ms;
  const int b = off[s];
  put_stats(st[2 * s], st[2 * s + 1], cpu_run + b, mem_run + b, vals + 8 * i);
}

bool calls_ok(const PertRawCalls* c) {
  return c && c->R >= 0 && c->R <= RW_MAX_ROWS && c->n_trace >= 0 && c->n_trace <= RW_MAX_ROWS &&
         c->n_iface >= 0 && c->n_iface <= 0x7fffffffLL && c->n_rpcid >= 0 && c->n_rpcid <= 0x7fffffffLL &&
         c->n_rpctype >= 0 && c->n_rpctype <= 0x7fffffffLL && c->n_ms >= 0 && c->n_ms <= 0x7ffffff0LL &&
         (c->R == 0 || (c->traceid && c->timestamp && c->rpcid && c->um && c->rpctype && c->dm && c->interface &&
                        c->rt));
}

int scan(int* a0, int* a1, long long L, int* bsum, cudaStream_t st) {   // inclusive, in place; a1 may be NULL
  const int nb = pert_cdiv(L, SCAN_TILE), ny = a1 ? 2 : 1;
  k_scan_tile_sums<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
  k_scan_block_sums<<<dim3(1, ny), SCAN_THREADS, 0, st>>>(bsum, nb);
  k_scan_apply<<<dim3(nb, ny), SCAN_THREADS, 0, st>>>(a0, a1, (int)L, bsum, nb);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long dedup_table(long long R) { return pow2_at_least(2 * R); }

}  // namespace

extern "C" {

long long pert_raw_dedup_workspace_bytes(long long R) {
  if (R < 0 || R > RW_MAX_ROWS) return PERT_ERR_BADARG;
  const long long S = dedup_table(R);
  return 4 * (2 * S + R + (R + 1)) + scan_bytes(R + 1) + 64;
}

int pert_raw_dedup(const PertRawCalls* calls, int hash_bits, int* rows, int64_t* keys, int64_t* n_kept,
                   void* workspace, long long workspace_bytes, int* status, void* stream_) {
  if (!calls_ok(calls) || hash_bits < 1 || hash_bits > 64 || !rows || !keys || !n_kept || !workspace || !status)
    return PERT_ERR_BADARG;
  const long long R = calls->R;
  if (workspace_bytes < pert_raw_dedup_workspace_bytes(R)) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  cudaError_t e;
  if ((e = cudaMemsetAsync(n_kept, 0, sizeof(int64_t), st)) != cudaSuccess) return (int)e;
  if (R == 0) return PERT_OK;
  const long long S = dedup_table(R);
  int* owner = (int*)workspace;
  int* first = owner + S;
  int* slot_of = first + S;
  int* flags = slot_of + R;
  int* bsum = flags + R + 1;
  if ((e = cudaMemsetAsync(owner, 0xff, 4 * S, st)) || (e = cudaMemsetAsync(first, 0x7f, 4 * S, st)) ||
      (e = cudaMemsetAsync(flags, 0, 4, st)))
    return (int)e;
  const int B = 256, gR = pert_cdiv(R, B);
  k_dedup_insert<<<gR, B, 0, st>>>(*calls, S, hash_bits, owner, first, slot_of, status);
  k_dedup_flags<<<gR, B, 0, st>>>(R, slot_of, first, flags);
  PERT_LAUNCH_CHECK();
  int rc;
  if ((rc = scan(flags, nullptr, R + 1, bsum, st)) != PERT_OK) return rc;
  k_dedup_compact<<<gR, B, 0, st>>>(*calls, flags, rows, keys, n_kept);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

long long pert_raw_process_workspace_bytes(const PertRawCalls* calls, long long N) {
  if (!calls_ok(calls) || N < 0 || N > calls->R) return PERT_ERR_BADARG;
  return layout(*calls, N, nullptr, nullptr) + 64;
}

}  // extern "C"

namespace {

// pert_raw_process (S = false, ps unused) and pert_raw_stream_process (S = true) after their argument checks
template <bool S>
int process_chunk(const PertRawCalls& c, long long N, const int64_t* order, int* has_res, long long min_occurence,
                  const PertRawState& ps, int64_t* sizes, void* workspace, cudaStream_t st) {
  Work w;
  layout(c, N, workspace, &w, S);
  cudaError_t e;
  auto fill = [&](void* p, long long bytes, int v) { return cudaMemsetAsync(p, v, (size_t)bytes, st); };
  if ((e = fill(w.ekey, 8 * w.SE, 0xff)) || (e = fill(w.pkey, 8 * w.SP, 0xff)) ||
      (e = fill(w.amax, 8 * c.n_trace, 0)) || (e = fill(w.first_tr, 4 * c.n_trace, 0x7f)) ||
      (e = fill(w.first_if, 4 * c.n_iface, 0x7f)) || (e = fill(w.first_rpc, 4 * c.n_rpcid, 0x7f)) ||
      (e = fill(w.first_rty, 4 * c.n_rpctype, 0x7f)) || (e = fill(w.fl_ms, 4 * (c.n_ms + 1), 0)) ||
      (e = fill(w.ncand, 4 * c.n_trace, 0)) || (e = fill(w.nq, 4 * c.n_trace, 0)) ||
      (e = fill(w.cand_pos, 4 * c.n_trace, 0x7f)) || (e = fill(w.q_pos, 4 * c.n_trace, 0x7f)) ||
      (e = fill(w.ndist, 4 * c.n_trace, 0)) || (e = fill(w.nres, 4 * c.n_trace, 0)) ||
      (e = fill(w.efirst, 4 * w.SE, 0x7f)) || (e = fill(w.ecnt, 4 * w.SE, 0)) ||
      (e = fill(sizes, 7 * sizeof(int64_t), 0)))
    return (int)e;
  int* flags[] = {w.fl_tr, w.fl_if, w.fl_ent, w.fl_rpc, w.fl_rty, w.fl_row};
  for (int* f : flags)
    if ((e = fill(f, 4, 0))) return (int)e;
  const int B = 256, gN = pert_cdiv(std::max(N, 1LL), B), gT = pert_cdiv(std::max(c.n_trace, 1LL), B);
  const int gM = pert_cdiv(std::max(c.n_ms, 1LL), B);
  int rc;
  if (S) {                                               // the stream's ids of the chunk codes, its has_res
    const long long n = std::max(std::max(c.n_ms, c.n_iface), std::max(c.n_rpcid, c.n_rpctype));
    if (n > 0) k_stream_gather<<<pert_cdiv(n, B), B, 0, st>>>(c, ps, has_res, w);
  }
  if (N > 0) {
    // 3. + 4. traceid / interface codes, entry candidates, entry keys
    k_first_codes<<<gN, B, 0, st>>>(c, N, order, w);
    k_candidates<S><<<gN, B, 0, st>>>(c, N, order, w);
    PERT_LAUNCH_CHECK();
    if ((rc = scan(w.fl_tr, w.fl_if, N + 1, w.bsum, st)) != PERT_OK) return rc;
    k_entries<S><<<gT, B, 0, st>>>(c, order, ps, w);
    // entryid / rpcid / rpctype codes over the rows of traces with an entry; 5. coverage; 6. occurrences
    k_entry_rows<<<gN, B, 0, st>>>(c, N, order, has_res, w);
    k_entry_flags<S><<<gN, B, 0, st>>>(c, N, order, w);
    PERT_LAUNCH_CHECK();
    if ((rc = scan(w.fl_ent, w.fl_rpc, N + 1, w.bsum, st)) != PERT_OK) return rc;
    if ((rc = scan(w.fl_rty, nullptr, N + 1, w.bsum, st)) != PERT_OK) return rc;
    k_coverage<<<gT, B, 0, st>>>(c.n_trace, w);
  }
  // 7. microservice presence (every resource msname, the surviving rows' um / dm); 8. survivor positions
  k_ms_init<S><<<gM, B, 0, st>>>(c.n_ms, has_res, w);
  if (N > 0) k_survivors<S><<<gN, B, 0, st>>>(c, N, order, min_occurence, ps, w);
  PERT_LAUNCH_CHECK();
  if ((rc = scan(w.fl_ms, nullptr, c.n_ms + 1, w.bsum, st)) != PERT_OK) return rc;
  if ((rc = scan(w.fl_row, nullptr, N + 1, w.bsum, st)) != PERT_OK) return rc;
  k_sizes<<<1, 1, 0, st>>>(N, c.n_ms, w, sizes);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

// pert_raw_emit (S = false) and pert_raw_stream_emit (S = true) after their argument checks
template <bool S>
int emit_chunk(const PertRawCalls& c, long long N, const int64_t* order, long long G, const int64_t* g_ts,
               const int64_t* g_ms, long long K, const int64_t* r_ms, const int* has_res, const PertRawOut& o,
               const PertRawState& ps, const PertRawStateOut& so, void* workspace, cudaStream_t st) {
  Work w;
  layout(c, N, workspace, &w, S);
  const int B = 256;
  if (S) {                                               // the fresh entry table: a copy, or the old keys rehashed
    cudaError_t e;
    if (so.ent_cap2 == ps.ent_cap) {
      if ((e = cudaMemcpyAsync(so.ent_key, ps.ent_key, 8 * ps.ent_cap, cudaMemcpyDeviceToDevice, st)) ||
          (e = cudaMemcpyAsync(so.ent_id, ps.ent_id, 8 * ps.ent_cap, cudaMemcpyDeviceToDevice, st)))
        return (int)e;
    } else {
      if ((e = cudaMemsetAsync(so.ent_key, 0xff, 8 * so.ent_cap2, st))) return (int)e;
      k_ent_rehash<<<pert_cdiv(ps.ent_cap, B), B, 0, st>>>(ps.ent_key, ps.ent_id, ps.ent_cap, so.ent_key, so.ent_id,
                                                         so.ent_cap2);
    }
  }
  if (N > 0) k_emit_rows<S><<<pert_cdiv(N, B), B, 0, st>>>(c, N, order, w, o, ps, so);
  if (c.n_ms > 0) k_emit_ms<S><<<pert_cdiv(c.n_ms, B), B, 0, st>>>(c.n_ms, w, o.ms_code, has_res, ps, so);
  if (G > 0) k_emit_res<S><<<pert_cdiv(G, B), B, 0, st>>>(G, c.n_ms, g_ts, g_ms, w, o.res_index, ps);
  if (S && K > 0) k_resource_ms<<<pert_cdiv(K, B), B, 0, st>>>(K, c.n_ms, r_ms, w, ps, so.resource_ms);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

bool out_ok(const PertRawOut& o) {
  return o.traceid && o.timestamp && o.rpcid && o.um && o.dm && o.interface && o.rpctype && o.rt && o.entryid &&
         o.row && o.res_index && o.ms_code && o.tr_code && o.if_code && o.rpc_code && o.rty_code && o.ent_dm && o.ent_if;
}

bool pow2(long long n) { return n > 0 && (n & (n - 1)) == 0; }

constexpr long long RW_MAX_IDS = 0x7ffffff0LL;           // ids and stream codes of every column

bool state_ok(const PertRawCalls& c, const PertRawState* s) {
  if (!s) return false;
  const long long codes[] = {s->n_ms_codes, s->n_if_codes, s->n_rpc_codes, s->n_rty_codes};
  const long long ids[] = {s->n_tr, s->n_if, s->n_rpc, s->n_rty, s->n_ent, s->n_ms};
  for (long long n : codes)
    if (n < 0 || n > RW_MAX_IDS) return false;
  for (long long n : ids)
    if (n < 0 || n > RW_MAX_IDS) return false;
  return (c.n_ms == 0 || s->ms_map) && (c.n_iface == 0 || s->if_map) && (c.n_rpcid == 0 || s->rpc_map) &&
         (c.n_rpctype == 0 || s->rty_map) && (s->n_ms_codes == 0 || (s->ms_id && s->has_res)) &&
         (s->n_if_codes == 0 || s->if_id) && (s->n_rpc_codes == 0 || s->rpc_id) && (s->n_rty_codes == 0 || s->rty_id) &&
         s->ent_cap >= 64 && s->ent_cap <= (1LL << 40) && pow2(s->ent_cap) && s->ent_key && s->ent_id &&
         (s->n_ent == 0 || s->ent_cnt) && 2 * s->n_ent <= s->ent_cap;
}

}  // namespace

extern "C" {

int pert_raw_process(const PertRawCalls* calls, long long N, const int64_t* order, const int* has_res,
                     long long min_occurence, int64_t* sizes, void* workspace, long long workspace_bytes,
                     void* stream_) {
  if (!calls_ok(calls) || N < 0 || N > calls->R || (N > 0 && !order) || !has_res || !sizes || !workspace)
    return PERT_ERR_BADARG;
  const long long need = pert_raw_process_workspace_bytes(calls, N);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  return process_chunk<false>(*calls, N, order, const_cast<int*>(has_res), min_occurence, PertRawState{}, sizes,
                              workspace, (cudaStream_t)stream_);
}

int pert_raw_emit(const PertRawCalls* calls, long long N, const int64_t* order, long long G, const int64_t* g_ts,
                  const int64_t* g_ms, const PertRawOut* out, void* workspace, long long workspace_bytes,
                  void* stream_) {
  if (!calls_ok(calls) || N < 0 || N > calls->R || (N > 0 && !order) || G < 0 || (G > 0 && (!g_ts || !g_ms)) ||
      !out || !workspace || !out_ok(*out))
    return PERT_ERR_BADARG;
  const long long need = pert_raw_process_workspace_bytes(calls, N);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  return emit_chunk<false>(*calls, N, order, G, g_ts, g_ms, 0, nullptr, nullptr, *out, PertRawState{},
                           PertRawStateOut{}, workspace, (cudaStream_t)stream_);
}

long long pert_raw_stream_workspace_bytes(const PertRawCalls* calls, long long N) {
  if (!calls_ok(calls) || N < 0 || N > calls->R) return PERT_ERR_BADARG;
  return layout(*calls, N, nullptr, nullptr, true) + 64;
}

int pert_raw_stream_process(const PertRawCalls* calls, long long N, const int64_t* order, int* has_res,
                            long long min_occurence, const PertRawState* state, int64_t* sizes, void* workspace,
                            long long workspace_bytes, void* stream_) {
  if (!calls_ok(calls) || N < 0 || N > calls->R || (N > 0 && !order) || !has_res || !sizes || !workspace ||
      !state_ok(*calls, state))
    return PERT_ERR_BADARG;
  const long long need = pert_raw_stream_workspace_bytes(calls, N);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  return process_chunk<true>(*calls, N, order, has_res, min_occurence, *state, sizes, workspace,
                             (cudaStream_t)stream_);
}

int pert_raw_stream_emit(const PertRawCalls* calls, long long N, const int64_t* order, long long G,
                         const int64_t* g_ts, const int64_t* g_ms, long long K, const int64_t* r_ms,
                         const int* has_res, const PertRawState* state, const PertRawOut* out,
                         const PertRawStateOut* state_out, void* workspace, long long workspace_bytes, void* stream_) {
  if (!calls_ok(calls) || N < 0 || N > calls->R || (N > 0 && !order) || G < 0 || (G > 0 && (!g_ts || !g_ms)) ||
      K < 0 || K > 0x7ffffff0LL || !out || !workspace || !out_ok(*out) || !state_ok(*calls, state) || !state_out)
    return PERT_ERR_BADARG;
  const PertRawCalls& c = *calls;
  const PertRawStateOut& so = *state_out;
  if ((c.n_ms > 0 && (!has_res || !so.ms_id || !so.has_res)) || (c.n_iface > 0 && !so.if_id) ||
      (c.n_rpcid > 0 && !so.rpc_id) || (c.n_rpctype > 0 && !so.rty_id) || !so.ent_key || !so.ent_id ||
      !so.ent_cnt || so.ent_cap2 < state->ent_cap || so.ent_cap2 > (1LL << 40) || !pow2(so.ent_cap2) ||
      (K > 0 && (!r_ms || !so.resource_ms)))
    return PERT_ERR_BADARG;
  const long long need = pert_raw_stream_workspace_bytes(calls, N);
  if (need < 0 || workspace_bytes < need) return PERT_ERR_BADARG;
  return emit_chunk<true>(c, N, order, G, g_ts, g_ms, K, r_ms, has_res, *out, *state, so, workspace,
                          (cudaStream_t)stream_);
}

long long pert_raw_resource_workspace_bytes(long long K) {
  if (K < 0 || K > 0x7ffffff0LL) return PERT_ERR_BADARG;
  return scan_bytes(K + 1) + 64;
}

int pert_raw_resource_groups(long long K, const int64_t* ts, const int64_t* ms, const int64_t* perm, long long n_ms,
                             int* gflag, int* has_res, int* gptr, int64_t* g_ts, int64_t* g_ms, int64_t* n_groups,
                             void* workspace, long long workspace_bytes, int* status, void* stream_) {
  if (K < 0 || K > 0x7ffffff0LL || n_ms < 0 || (K > 0 && (!ts || !ms || !perm)) || !gflag || !has_res || !gptr ||
      !g_ts || !g_ms || !n_groups || !workspace || !status)
    return PERT_ERR_BADARG;
  if (workspace_bytes < pert_raw_resource_workspace_bytes(K)) return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  cudaError_t e;
  if ((e = cudaMemsetAsync(n_groups, 0, sizeof(int64_t), st)) || (e = cudaMemsetAsync(gflag, 0, 4, st)) ||
      (e = cudaMemsetAsync(gptr, 0, 4, st)) || (n_ms > 0 && (e = cudaMemsetAsync(has_res, 0, 4 * n_ms, st))))
    return (int)e;
  if (K == 0) return PERT_OK;
  const int B = 256, gK = pert_cdiv(K, B);
  k_res_flags<<<gK, B, 0, st>>>(K, ts, ms, perm, n_ms, gflag, has_res, status);
  PERT_LAUNCH_CHECK();
  int rc;
  if ((rc = scan(gflag, nullptr, K + 1, (int*)workspace, st)) != PERT_OK) return rc;
  k_res_groups<<<gK, B, 0, st>>>(K, n_ms, ts, ms, perm, gflag, gptr, g_ts, g_ms, n_groups);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_raw_resource_stats(long long G, const int64_t* perm, const int* gptr, const double* cpu, const double* mem,
                            const double* cpu_sorted, const double* mem_sorted, double* vals, void* stream_) {
  if (G < 0 || (G > 0 && (!perm || !gptr || !cpu || !mem || !cpu_sorted || !mem_sorted || !vals)))
    return PERT_ERR_BADARG;
  if (G == 0) return PERT_OK;
  k_res_stats<<<pert_cdiv(G, 128), 128, 0, (cudaStream_t)stream_>>>(G, perm, gptr, cpu, mem, cpu_sorted, mem_sorted,
                                                                   vals);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

// ---- the open-bucket sample window ----------------------------------------------------------------------------------
static bool win_count_ok(long long n) { return n >= 0 && n <= RW_WIN_MAX; }

long long pert_raw_window_workspace_bytes(long long U, long long k, long long U2) {
  if (!win_count_ok(U) || !win_count_ok(k) || !win_count_ok(U2)) return PERT_ERR_BADARG;
  return 4 * (2 * (U2 + 16) + (U + 16)) + scan_bytes(std::max(k, U2) + 1) + 64;
}

int pert_raw_window_count(long long k, const int64_t* bkeys, long long n_ms, long long seal, long long U,
                          const int64_t* keys, int* flags, int64_t* sizes, void* workspace, long long workspace_bytes,
                          void* stream_) {
  if (!win_count_ok(k) || !win_count_ok(U) || n_ms < 1 || (k > 0 && (!bkeys || !flags)) || (U > 0 && !keys) ||
      !sizes || !workspace || workspace_bytes < pert_raw_window_workspace_bytes(U, k, 0))
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  int* fu = flags;
  int* fn = flags ? flags + k + 1 : nullptr;
  if (k > 0) {
    k_win_flags<<<pert_cdiv(k, 256), 256, 0, st>>>(k, bkeys, n_ms, seal, U, keys, fu, fn);
    PERT_LAUNCH_CHECK();
    int rc;
    if ((rc = scan(fu, fn, k + 1, (int*)workspace, st)) != PERT_OK) return rc;
  }
  k_win_sizes<<<1, 1, 0, st>>>(k, bkeys, n_ms, seal, U, fu, fn, sizes);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

int pert_raw_window_merge(long long U, long long S, const int64_t* keys, const int* off, const void* state,
                          const double* cpu_run, const double* mem_run, long long k, const int64_t* bkeys, const int64_t* perm,
                          const double* cpu, const double* mem, const double* cpu_sorted, const double* mem_sorted,
                          const int* flags, long long n_late, long long u, long long U2, int64_t* keys2, int* off2,
                          void* state2, double* cpu_run2, double* mem_run2, int* ustart, int* upos, void* workspace,
                          long long workspace_bytes, void* stream_) {
  if (!win_count_ok(U) || !win_count_ok(S) || S < U || (U == 0 && S > 0) || !win_count_ok(k) || !win_count_ok(U2) ||
      S + k > RW_WIN_MAX || n_late < 0 || n_late > k || u < 0 ||
      u > k - n_late || U2 < U || U2 > U + u || !off || !off2 || !ustart ||
      (U > 0 && (!keys || !state || !cpu_run || !mem_run)) ||
      (k > 0 && (!bkeys || !perm || !cpu || !mem || !cpu_sorted || !mem_sorted || !flags)) ||
      (U2 > 0 && (!keys2 || !state2 || !cpu_run2 || !mem_run2)) || (u > 0 && !upos) || !workspace ||
      workspace_bytes < pert_raw_window_workspace_bytes(U, k, U2))
    return PERT_ERR_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  int* src = (int*)workspace;
  int* bsrc = src + U2 + 16;
  int* opos = bsrc + U2 + 16;
  int* bsum = opos + U + 16;
  const int* fu = flags;
  const int* fn = flags ? flags + k + 1 : nullptr;
  const int B = 256;
  if (U > 0 || k > 0) {
    k_win_keys<<<pert_cdiv(std::max(U, k), B), B, 0, st>>>(U, keys, k, bkeys, fu, fn, keys2, src, bsrc, opos, ustart,
                                                           upos);
    PERT_LAUNCH_CHECK();
  }
  if (U2 == 0) return (int)cudaMemsetAsync(off2, 0, 4, st);
  k_win_fold<<<pert_cdiv(U2, 128), 128, 0, st>>>(U2, src, bsrc, ustart, off, (const GroupStats*)state, perm, cpu, mem,
                                                 (GroupStats*)state2, off2);
  PERT_LAUNCH_CHECK();
  int rc;
  if ((rc = scan(off2, nullptr, U2 + 1, bsum, st)) != PERT_OK) return rc;
  const long long n_new = k - n_late;
  if (S + n_new > 0) {
    k_win_runs<<<pert_cdiv(S + n_new, B), B, 0, st>>>(U, S, off, cpu_run, mem_run, n_late, n_new, fu, ustart, upos,
                                                      cpu_sorted, mem_sorted, src, bsrc, opos, off2, cpu_run2,
                                                      mem_run2);
    PERT_LAUNCH_CHECK();
  }
  return PERT_OK;
}

int pert_raw_window_emit(long long n, const int* slot, long long U, const int64_t* keys, const int* off,
                         const void* state, const double* cpu_run, const double* mem_run, long long n_ms,
                         int64_t* index, double* vals, void* stream_) {
  if (!win_count_ok(n) || !win_count_ok(U) || (!slot && n > U) || n_ms < 1 ||
      (n > 0 && (!keys || !off || !state || !cpu_run || !mem_run || !index || !vals)))
    return PERT_ERR_BADARG;
  if (n == 0) return PERT_OK;
  k_win_emit<<<pert_cdiv(n, 128), 128, 0, (cudaStream_t)stream_>>>(n, slot, keys, off, (const GroupStats*)state,
                                                                   cpu_run, mem_run, n_ms, index, vals);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
