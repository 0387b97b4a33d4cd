// Device-side batch assembly from a resident pattern store (SURVEY.md section 8f rows N1 + N4).
//
// The reference builds every sample on the host, per trace, from Python dicts and a pandas MultiIndex:
//   get_entry_data (pert_gnn.py:134-173): for the trace's entry, concatenate ALL runtime-pattern graphs of that entry --
//     get_x (:40-67, the (timestamp, msname) -> 8 resource statistics join, missing-indicator column),
//     get_cat_X (:97-99), get_node_depth (:102-104), get_edge_index (:107-119, pattern node offsets),
//     get_edge_attr (:77-82), get_pattern_num_nodes (:85-94), pattern_probs (:170) --
//   then PyG's DataLoader collates B samples (:201-209: concatenate, offset edge_index by the cumulative node count,
//   batch vector, ptr), and the train loop rebuilds the per-node pattern probability on the host every step with B
//   tiny H2D copies (:220-230, transform_pattern_probs :122-131).
// Here the patterns (CSR-like concatenation), the entry -> (pattern, probability) lists, the resource table (sorted
// (timestamp, ms) keys) and the trace table live in HBM; a batch is a list of trace ids (8 B each) and two kernels
// (one thread per output node / per output edge) write the collated Batch tensors -- bit-identical to what
// get_entry_data + Batch.from_data_list + transform_pattern_probs produce (tests/golden/ref_loop.npz holds the
// reference's own outputs).
//
// Reference quirk reproduced: get_x maps ms -> node id through a dict (ms2nid), so when a microservice occurs several
// times in one pattern only its LAST node receives the resource statistics; earlier duplicates keep [0 x 8, 1]
// (`last_occ` flag, computed when the store is built).  A resourced microservice whose (timestamp, ms) row is missing
// raises KeyError in the reference; here it sets PERT_ERR_RANGE in `status` and the node keeps the missing indicator.
//
// Serving (pert_store_assemble_requests): the same kernels, with graph b taken from a request (entry, timestamp) instead
// of a trace row -- the source is a template parameter -- and optionally the as-of resource join: the newest row of the
// microservice at or before the request's time bucket, through a per-microservice index of the sorted rows.
#include "common.cuh"

namespace {

constexpr int NF = 8;   // resource statistics per (timestamp, ms) row; x has NF + 1 columns (pert_gnn.py:44-52)

// Where graph b of a batch takes its entry, time bucket, label and pattern mix from: a row of the store's trace table
// (pert_store_assemble), a request (pert_store_assemble_requests) or a what-if request (pert_store_assemble_whatif).
// entry() flags a bad id in `bad` and falls back to trace 0 / entry 0; the other reads repeat the fallback, so every
// kernel sees the same graph.  The mix of graph b is the slot range slots() returns, pattern pat(k) with probability
// prob(k) in slot k; sizes() gives the graph's node, edge and slot counts.
struct OwnMix {                       // the entry's stored mix: ent_ptr / ent_pat / ent_prob
  using Slot = int;
  static constexpr bool kWhatIf = false;
  __device__ __forceinline__ void slots(const PertStore& s, int, int ent, Slot& k0, Slot& k1) const {
    k0 = s.ent_ptr[ent];
    k1 = s.ent_ptr[ent + 1];
  }
  __device__ __forceinline__ int pat(const PertStore& s, Slot k) const { return s.ent_pat[k]; }
  __device__ __forceinline__ float prob(const PertStore& s, Slot k) const { return s.ent_prob[k]; }
  __device__ __forceinline__ void sizes(const PertStore& s, int, int ent, int v[3], bool&) const {
    v[0] = s.ent_nodes[ent];
    v[1] = s.ent_edges[ent];
    v[2] = s.ent_ptr[ent + 1] - s.ent_ptr[ent];
  }
};

struct TraceRows : OwnMix {
  const int64_t* __restrict__ ids;
  static constexpr bool kLabel = true;
  __device__ __forceinline__ int64_t row(const PertStore& s, int b, bool& bad) const {
    const int64_t t = ids[b];
    bad = t < 0 || t >= s.n_traces;
    return bad ? 0 : t;
  }
  __device__ __forceinline__ int entry(const PertStore& s, int b, bool& bad) const {
    return s.trace_entry[row(s, b, bad)];
  }
  __device__ __forceinline__ int64_t bucket(const PertStore& s, int b) const {
    bool bad;
    return s.trace_ts[row(s, b, bad)];
  }
  __device__ __forceinline__ int64_t label(const PertStore& s, int b) const {
    bool bad;
    return s.trace_y[row(s, b, bad)];
  }
};

struct Requests : OwnMix {
  const int64_t* __restrict__ entry_ids;
  const int64_t* __restrict__ timestamps;
  static constexpr bool kLabel = false;
  __device__ __forceinline__ int entry(const PertStore& s, int b, bool& bad) const {
    const int64_t e = entry_ids[b];
    bad = e < 0 || e >= s.n_ent || s.ent_ptr[e + 1] == s.ent_ptr[e];
    return bad ? 0 : (int)e;
  }
  __device__ __forceinline__ int64_t bucket(const PertStore&, int b) const { return pert_time_bucket(timestamps[b]); }
};

// A request with its own pattern mix (w.mix_ptr != NULL: slots mix_ptr[b] .. mix_ptr[b+1]-1 of mix_pat / mix_prob,
// absolute offsets) and / or a resource scenario (w.scenario[b] >= 0: the override rows (scenario, ms)).  A pattern
// index outside [0, n_pat) reads pattern 0 and an empty or inverted mix gives an empty graph; sizes() flags both.
struct WhatIfRequests {
  const int64_t* __restrict__ entry_ids;
  const int64_t* __restrict__ timestamps;
  PertWhatIf w;
  using Slot = int64_t;
  static constexpr bool kLabel = false;
  static constexpr bool kWhatIf = true;
  __device__ __forceinline__ int entry(const PertStore& s, int b, bool& bad) const {
    const int64_t e = entry_ids[b];
    bad = e < 0 || e >= s.n_ent || (!w.mix_ptr && s.ent_ptr[e + 1] == s.ent_ptr[e]);   // own mix: not read if given
    return bad ? 0 : (int)e;
  }
  __device__ __forceinline__ int64_t bucket(const PertStore&, int b) const { return pert_time_bucket(timestamps[b]); }
  __device__ __forceinline__ void slots(const PertStore& s, int b, int ent, Slot& k0, Slot& k1) const {
    if (w.mix_ptr) {
      k0 = w.mix_ptr[b];
      k1 = max(k0, w.mix_ptr[b + 1]);
    } else {
      k0 = s.ent_ptr[ent];
      k1 = s.ent_ptr[ent + 1];
    }
  }
  __device__ __forceinline__ int pat(const PertStore& s, Slot k) const {
    if (!w.mix_ptr) return s.ent_pat[k];
    const int p = w.mix_pat[k];
    return (p < 0 || p >= s.n_pat) ? 0 : p;
  }
  __device__ __forceinline__ float prob(const PertStore& s, Slot k) const {
    return w.mix_ptr ? w.mix_prob[k] : s.ent_prob[k];
  }
  __device__ __forceinline__ void sizes(const PertStore& s, int b, int ent, int v[3], bool& bad) const {
    if (!w.mix_ptr) {
      v[0] = s.ent_nodes[ent];
      v[1] = s.ent_edges[ent];
      v[2] = s.ent_ptr[ent + 1] - s.ent_ptr[ent];
      return;
    }
    const int64_t k0 = w.mix_ptr[b], k1 = w.mix_ptr[b + 1];
    if (k1 <= k0) bad = true;
    v[0] = v[1] = v[2] = 0;
    for (int64_t k = k0; k < k1; ++k) {
      const int q = w.mix_pat[k];
      if (q < 0 || q >= s.n_pat) bad = true;
      const int p = (q < 0 || q >= s.n_pat) ? 0 : q;
      v[0] += s.pat_nptr[p + 1] - s.pat_nptr[p];
      v[1] += s.pat_eptr[p + 1] - s.pat_eptr[p];
      v[2] += 1;
    }
  }
  // the first override row of key (scenario[b], ms) -- ov_keys sorted ascending, nonnegative -- into f; false if none.
  // A scenario above the largest one in the table has no rows (and its key could overflow int64: compared unsigned).
  __device__ __forceinline__ bool override_row(const PertStore& s, int b, int64_t ms, float* f) const {
    if (!w.scenario || w.n_ov == 0) return false;
    const int64_t sc = w.scenario[b];
    if (sc < 0 || sc > w.ov_keys[w.n_ov - 1] / s.n_ms) return false;
    const uint64_t key = (uint64_t)sc * (uint64_t)s.n_ms + (uint64_t)ms;
    long long lo = 0, hi = w.n_ov;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if ((uint64_t)w.ov_keys[mid] < key) lo = mid + 1;
      else hi = mid;
    }
    if (lo == w.n_ov || (uint64_t)w.ov_keys[lo] != key) return false;
    const float4* v = reinterpret_cast<const float4*>(w.ov_vals + (size_t)lo * NF);
    const float4 a = v[0], c = v[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = c.x; f[5] = c.y; f[6] = c.z; f[7] = c.w;
    return true;
  }
};

// exclusive prefix sums of the per-graph node / edge / pattern counts (one CTA; B is a batch size)
template <class Src>
__global__ void __launch_bounds__(1024) k_store_offsets(PertStore s, Src src, int B, int* __restrict__ node_off,
                                                        int* __restrict__ edge_off, int* __restrict__ pat_off,
                                                        int* status) {
  __shared__ int carry[3];
  __shared__ int wsum[3][32];
  if (threadIdx.x < 3) carry[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int base = 0; base < B; base += blockDim.x) {
    const int b = base + threadIdx.x;
    int v[3] = {0, 0, 0};
    if (b < B) {
      bool bad;
      const int ent = src.entry(s, b, bad);
      src.sizes(s, b, ent, v, bad);
      if (bad && status) atomicExch(status, PERT_ERR_RANGE);
    }
    int incl[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      int x = v[k];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += u;
      }
      incl[k] = x;
      if (lane == 31) wsum[k][w] = x;
    }
    __syncthreads();
    if (w == 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int x = wsum[k][lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int u = __shfl_up_sync(0xffffffffu, x, o);
          if (lane >= o) x += u;
        }
        wsum[k][lane] = x;
      }
    }
    __syncthreads();
    int* outs[3] = {node_off, edge_off, pat_off};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int excl = carry[k] + (w ? wsum[k][w - 1] : 0) + incl[k] - v[k];
      if (b < B) outs[k][b] = excl;
      if (b == B - 1) outs[k][B] = excl + v[k];
    }
    __syncthreads();
    if (threadIdx.x < 3) carry[threadIdx.x] += wsum[threadIdx.x][31];
    __syncthreads();
  }
  if (B == 0 && threadIdx.x == 0) node_off[0] = edge_off[0] = pat_off[0] = 0;
}

// pattern instance of local node / edge index l inside graph b (entry `ent`): returns the mix slot k and the offsets
// of that pattern inside the graph
template <class Src>
__device__ __forceinline__ typename Src::Slot find_pattern(const PertStore& s, const Src& src, int b, int ent, int l,
                                                           bool edges, int& node_base, int& local) {
  using Slot = typename Src::Slot;
  int nb = 0, acc = 0;
  Slot k0, k1;
  src.slots(s, b, ent, k0, k1);
  for (Slot k = k0; k < k1; ++k) {
    const int p = src.pat(s, k);
    const int nn = s.pat_nptr[p + 1] - s.pat_nptr[p];
    const int sz = edges ? s.pat_eptr[p + 1] - s.pat_eptr[p] : nn;
    if (l < acc + sz || k == k1 - 1) {
      node_base = nb;
      local = l - acc;
      return k;
    }
    acc += sz;
    nb += nn;
  }
  node_base = 0;
  local = 0;
  return k0;
}

// exact join: the sorted row of key (bucket, ms) (the lower bound over res_keys), -1 if there is none
__device__ __forceinline__ int exact_row(const PertStore& s, int64_t bucket, int64_t ms) {
  const int64_t key = bucket * (int64_t)s.n_ms + ms;
  int lo = 0, hi = s.n_res;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s.res_keys[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return (lo < s.n_res && s.res_keys[lo] == key) ? lo : -1;
}

// as-of join: the row of ms with the largest timestamp <= bucket, the first of the rows sharing that timestamp (the one
// exact_row returns for it); -1 if every row of ms is later than bucket
__device__ __forceinline__ int asof_row(const PertResourceAsOf& a, int64_t bucket, int64_t ms) {
  const int first = a.ms_ptr[ms];
  int lo = first, hi = a.ms_ptr[ms + 1];
  while (lo < hi) {                               // first k with ts[k] > bucket
    const int mid = (lo + hi) >> 1;
    if (a.ts[mid] <= bucket) lo = mid + 1;
    else hi = mid;
  }
  if (lo == first) return -1;
  const int64_t t = a.ts[lo - 1];
  hi = lo - 1;
  lo = first;
  while (lo < hi) {                               // first k with ts[k] == t
    const int mid = (lo + hi) >> 1;
    if (a.ts[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  return a.row[lo];
}

// asof.ms_ptr == NULL: exact join (a missing row sets status)
template <class Src>
__global__ void __launch_bounds__(256) k_store_nodes(PertStore s, Src src, PertResourceAsOf asof, int B,
                                                     const int* __restrict__ node_off, PertBatchOut o, int* status) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = node_off[B];
  if (n >= N) return;
  const int b = upper_seg(node_off, B, n);
  bool bad;
  const int ent = src.entry(s, b, bad);
  int node_base, local;
  const auto k = find_pattern(s, src, b, ent, n - node_off[b], false, node_base, local);
  const int p = src.pat(s, k);
  const int g = s.pat_nptr[p] + local;
  const int64_t ms = s.pat_ms[g];
  o.cat_X[n] = ms;
  o.node_depth[n] = s.pat_depth[g];
  o.pattern_num_nodes[n] = (float)(s.pat_nptr[p + 1] - s.pat_nptr[p]);
  o.rt_probs[n] = src.prob(s, k);
  o.batch[n] = b;
  // ---- feature join (get_x): statistics of (timestamp, ms) for the LAST node of a resourced ms, else missing indicator
  float f[NF + 1];
#pragma unroll
  for (int c = 0; c < NF; ++c) f[c] = 0.f;
  f[NF] = 1.f;
  bool overridden = false;                       // what-if: an override row of (scenario, ms) replaces the store's join
  if constexpr (Src::kWhatIf) {
    if (s.pat_last[g] && ms >= 0 && ms < s.n_ms && src.override_row(s, b, ms, f)) {
      f[NF] = 0.f;
      overridden = true;
    }
  }
  if (!overridden && s.pat_last[g] && ms >= 0 && ms < s.n_ms && s.ms_has_res[ms]) {
    const int64_t bucket = src.bucket(s, b);
    const int r = asof.ms_ptr ? asof_row(asof, bucket, ms) : exact_row(s, bucket, ms);
    if (r >= 0) {
#pragma unroll
      for (int c = 0; c < NF; ++c) f[c] = s.res_vals[(size_t)r * NF + c];
      f[NF] = 0.f;
    } else if (!asof.ms_ptr && status) {
      atomicExch(status, PERT_ERR_RANGE);      // the reference raises KeyError here (resource_df.loc)
    }
  }
#pragma unroll
  for (int c = 0; c <= NF; ++c) o.x[(size_t)n * (NF + 1) + c] = f[c];
}

template <class Src>
__global__ void __launch_bounds__(256) k_store_edges(PertStore s, Src src, int B, const int* __restrict__ node_off,
                                                     const int* __restrict__ edge_off, PertBatchOut o) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int E = edge_off[B];
  if (e >= E) return;
  const int b = upper_seg(edge_off, B, e);
  bool bad;
  const int ent = src.entry(s, b, bad);
  int node_base, local;
  const auto k = find_pattern(s, src, b, ent, e - edge_off[b], true, node_base, local);
  const int p = src.pat(s, k);
  const size_t ge = (size_t)s.pat_eptr[p] + local;
  const int64_t off = (int64_t)node_off[b] + node_base;
  o.edge_index[e] = s.pat_src[ge] + off;
  o.edge_index[(size_t)E + e] = s.pat_dst[ge] + off;
  for (int c = 0; c < s.attr_cols; ++c) o.edge_attr[(size_t)e * s.attr_cols + c] = s.pat_attr[ge * s.attr_cols + c];
}

// per-graph outputs: entry_id, y (trace rows only), ptr (int64), and the concatenated per-pattern probabilities
template <class Src>
__global__ void __launch_bounds__(256) k_store_traces(PertStore s, Src src, int B, const int* __restrict__ node_off,
                                                      const int* __restrict__ pat_off, PertBatchOut o) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  o.ptr[b] = node_off[b];
  if (b == B) return;
  bool bad;
  const int ent = src.entry(s, b, bad);
  o.entry_id[b] = ent;
  if constexpr (Src::kLabel) o.y[b] = src.label(s, b);
  typename Src::Slot k0, k1;
  src.slots(s, b, ent, k0, k1);
  for (auto k = k0; k < k1; ++k) o.pattern_probs[pat_off[b] + (k - k0)] = src.prob(s, k);
}

// one thread per (timestamp, ms) query: the row the exact or the as-of join of assembly reads (pert_store_lookup_resources)
__global__ void __launch_bounds__(256) k_store_lookup(PertStore s, PertResourceAsOf asof, const int64_t* __restrict__ ts,
                                                      const int64_t* __restrict__ ms, int k, float* __restrict__ values,
                                                      uint8_t* __restrict__ found) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int64_t m = ms[i];
  int r = -1;
  if (m >= 0 && m < s.n_ms) {
    const int64_t bucket = pert_time_bucket(ts[i]);
    r = asof.ms_ptr ? asof_row(asof, bucket, m) : exact_row(s, bucket, m);
  }
#pragma unroll
  for (int c = 0; c < NF; ++c) values[(size_t)i * NF + c] = r >= 0 ? s.res_vals[(size_t)r * NF + c] : 0.f;
  found[i] = r >= 0;
}

bool entries_ok(const PertStore* s) { return s->ent_ptr && s->ent_pat && s->ent_prob && s->pat_nptr && s->pat_eptr; }

template <class Src>
int assemble(const PertStore& s, const Src& src, const PertResourceAsOf& asof, long long B, long long N, long long E,
             int* offsets, const PertBatchOut& out, int* status, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int* node_off = offsets;
  int* edge_off = offsets + (B + 1);
  int* pat_off = offsets + 2 * (B + 1);
  k_store_offsets<<<1, 1024, 0, st>>>(s, src, (int)B, node_off, edge_off, pat_off, status);
  k_store_traces<<<pert_cdiv(B + 1, 256), 256, 0, st>>>(s, src, (int)B, node_off, pat_off, out);
  if (N > 0) k_store_nodes<<<pert_cdiv(N, 256), 256, 0, st>>>(s, src, asof, (int)B, node_off, out, status);
  if (E > 0) k_store_edges<<<pert_cdiv(E, 256), 256, 0, st>>>(s, src, (int)B, node_off, edge_off, out);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // namespace

extern "C" {

int pert_store_assemble(const PertStore* s, const int64_t* trace_ids, long long B, long long N, long long E,
                        int* offsets, const PertBatchOut* out, int* status, void* stream) {
  if (!s || !out || B < 0 || N < 0 || E < 0 || (B > 0 && (!trace_ids || !offsets))) return PERT_ERR_BADARG;
  if (!entries_ok(s) || !s->trace_entry) return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  return assemble(*s, TraceRows{{}, trace_ids}, PertResourceAsOf{}, B, N, E, offsets, *out, status, stream);
}

int pert_store_assemble_requests(const PertStore* s, const PertResourceAsOf* asof, const int64_t* entry_ids,
                                 const int64_t* timestamps, long long B, long long N, long long E, int* offsets,
                                 const PertBatchOut* out, int* status, void* stream) {
  if (!s || !out || B < 0 || N < 0 || E < 0 || (B > 0 && (!entry_ids || !timestamps || !offsets)))
    return PERT_ERR_BADARG;
  if (!entries_ok(s) || (asof && (!asof->ms_ptr || (s->n_res > 0 && (!asof->ts || !asof->row)))))
    return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  return assemble(*s, Requests{{}, entry_ids, timestamps}, asof ? *asof : PertResourceAsOf{}, B, N, E, offsets, *out,
                  status, stream);
}

int pert_store_assemble_whatif(const PertStore* s, const PertResourceAsOf* asof, const PertWhatIf* w,
                               const int64_t* entry_ids, const int64_t* timestamps, long long B, long long N,
                               long long E, int* offsets, const PertBatchOut* out, int* status, void* stream) {
  if (!s || !out || !w || B < 0 || N < 0 || E < 0 || (B > 0 && (!entry_ids || !timestamps || !offsets)))
    return PERT_ERR_BADARG;
  if (!entries_ok(s) || (asof && (!asof->ms_ptr || (s->n_res > 0 && (!asof->ts || !asof->row)))))
    return PERT_ERR_BADARG;
  if (w->mix_ptr && (!w->mix_pat || !w->mix_prob)) return PERT_ERR_BADARG;
  if (w->n_ov < 0 || (w->n_ov > 0 && (!w->ov_keys || !w->ov_vals || s->n_ms < 1 ||
                                      reinterpret_cast<uintptr_t>(w->ov_vals) % 16)))
    return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  WhatIfRequests src{entry_ids, timestamps, *w};
  return assemble(*s, src, asof ? *asof : PertResourceAsOf{}, B, N, E, offsets, *out, status, stream);
}

int pert_store_lookup_resources(const PertStore* s, const PertResourceAsOf* asof, const int64_t* timestamps,
                                const int64_t* ms, long long k, float* values, uint8_t* found, void* stream) {
  if (!s || k < 0 || k > INT32_MAX || (k > 0 && (!timestamps || !ms || !values || !found))) return PERT_ERR_BADARG;
  if (s->n_ms < 1 || (s->n_res > 0 && (!s->res_keys || !s->res_vals)) ||
      (asof && (!asof->ms_ptr || (s->n_res > 0 && (!asof->ts || !asof->row)))))
    return PERT_ERR_BADARG;
  if (k == 0) return PERT_OK;
  k_store_lookup<<<pert_cdiv(k, 256), 256, 0, (cudaStream_t)stream>>>(*s, asof ? *asof : PertResourceAsOf{}, timestamps,
                                                                     ms, (int)k, values, found);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
