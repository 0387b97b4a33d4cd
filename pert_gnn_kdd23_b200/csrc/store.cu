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

__device__ __forceinline__ int upper_seg(const int* __restrict__ off, int n, int v) {
  // largest b in [0, n) with off[b] <= v   (off is an exclusive prefix sum, off[n] = total)
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= v) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Where graph b of a batch takes its entry, time bucket and label from: a row of the store's trace table
// (pert_store_assemble) or a request (pert_store_assemble_requests).  entry() flags a bad id in `bad` and falls back to
// trace 0 / entry 0; the other reads repeat the fallback, so every kernel sees the same graph.
struct TraceRows {
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

struct Requests {
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
      if (bad && status) atomicExch(status, PERT_ERR_RANGE);
      v[0] = s.ent_nodes[ent];
      v[1] = s.ent_edges[ent];
      v[2] = s.ent_ptr[ent + 1] - s.ent_ptr[ent];
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

// pattern instance of local node / edge index l inside entry `ent`: returns slot k (into ent_pat / ent_prob) and the
// offsets of that pattern inside the graph
__device__ __forceinline__ int find_pattern(const PertStore& s, int ent, int l, bool edges, int& node_base,
                                            int& local) {
  int nb = 0, acc = 0;
  const int k0 = s.ent_ptr[ent], k1 = s.ent_ptr[ent + 1];
  for (int k = k0; k < k1; ++k) {
    const int p = s.ent_pat[k];
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
  const int k = find_pattern(s, ent, n - node_off[b], false, node_base, local);
  const int p = s.ent_pat[k];
  const int g = s.pat_nptr[p] + local;
  const int64_t ms = s.pat_ms[g];
  o.cat_X[n] = ms;
  o.node_depth[n] = s.pat_depth[g];
  o.pattern_num_nodes[n] = (float)(s.pat_nptr[p + 1] - s.pat_nptr[p]);
  o.rt_probs[n] = s.ent_prob[k];
  o.batch[n] = b;
  // ---- feature join (get_x): statistics of (timestamp, ms) for the LAST node of a resourced ms, else missing indicator
  float f[NF + 1];
#pragma unroll
  for (int c = 0; c < NF; ++c) f[c] = 0.f;
  f[NF] = 1.f;
  if (s.pat_last[g] && ms >= 0 && ms < s.n_ms && s.ms_has_res[ms]) {
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
  const int k = find_pattern(s, ent, e - edge_off[b], true, node_base, local);
  const int p = s.ent_pat[k];
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
  const int k0 = s.ent_ptr[ent], k1 = s.ent_ptr[ent + 1];
  for (int k = k0; k < k1; ++k) o.pattern_probs[pat_off[b] + (k - k0)] = s.ent_prob[k];
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
  return assemble(*s, TraceRows{trace_ids}, PertResourceAsOf{}, B, N, E, offsets, *out, status, stream);
}

int pert_store_assemble_requests(const PertStore* s, const PertResourceAsOf* asof, const int64_t* entry_ids,
                                 const int64_t* timestamps, long long B, long long N, long long E, int* offsets,
                                 const PertBatchOut* out, int* status, void* stream) {
  if (!s || !out || B < 0 || N < 0 || E < 0 || (B > 0 && (!entry_ids || !timestamps || !offsets)))
    return PERT_ERR_BADARG;
  if (!entries_ok(s) || (asof && (!asof->ms_ptr || (s->n_res > 0 && (!asof->ts || !asof->row)))))
    return PERT_ERR_BADARG;
  if (B == 0) return PERT_OK;
  return assemble(*s, Requests{entry_ids, timestamps}, asof ? *asof : PertResourceAsOf{}, B, N, E, offsets, *out,
                  status, stream);
}

}  // extern "C"
