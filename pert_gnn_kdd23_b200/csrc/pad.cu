// Padding of a batch into the persistent buffers of a capacity bucket (N_cap, E_cap, B_cap), so that one captured CUDA
// graph per bucket serves every batch that fits it (train.BucketedTrainStep).  The real part is copied bit for bit; the
// tail is filled with ghost graphs that change no real result:
//   ghost node j = N + j' (j' = 0 .. N_cap - N - 1) belongs to graph B + min(j', B_cap - B - 1): the batch vector stays
//   sorted and every ghost graph owns at least one node;
//   ghost edge k = E + k' is a self-loop on ghost node N + k' mod (N_cap - N): no edge joins a ghost to a real node;
//   x = 0, every id (cat_X, edge_attr, entry_id) = 0, rt_probs = 0 (a ghost node adds nothing to any pool),
//   pattern_num_nodes = 1 (a divisor in the pool), y = 1.
// The kernels then run at the capacity sizes; live = {N, B} tells the few places where a count enters the arithmetic
// (BatchNorm statistics and backward, the loss, the eval metrics) how many rows and graphs are real.
#include "common.cuh"

namespace {

struct PadArgs {
  const float *x, *probs, *pnn;
  const int64_t *cat_X, *edge_index, *edge_attr, *batch, *entry_id, *y;
  float *x_cap, *probs_cap, *pnn_cap;
  int64_t *cat_X_cap, *edge_index_cap, *edge_attr_cap, *batch_cap, *entry_id_cap, *y_cap;
  long long* live;
  long long N, E, B, N_cap, E_cap, B_cap;
  int F, n_cat, attr_cols;
  // element offsets of the segments of the flat work range (exclusive ends)
  long long s_x, s_cat, s_src, s_dst, s_attr, s_batch, s_probs, s_pnn, s_ent, s_y;
};

__global__ void __launch_bounds__(256) k_batch_pad(PadArgs a) {
  const long long ng = a.N_cap - a.N, bg = a.B_cap - a.B;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.live[0] = a.N;
    a.live[1] = a.B;
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < a.s_y; t += stride) {
    if (t < a.s_x) {                               // x [N_cap, F]
      const long long n = t / a.F;
      a.x_cap[t] = n < a.N ? a.x[t] : 0.f;
    } else if (t < a.s_cat) {                      // cat_X [N_cap, n_cat]
      const long long i = t - a.s_x;
      a.cat_X_cap[i] = i / a.n_cat < a.N ? a.cat_X[i] : 0;
    } else if (t < a.s_dst) {                      // edge_index [2, E_cap]: both rows
      const long long i = t - a.s_cat, r = i / a.E_cap, e = i - r * a.E_cap;
      a.edge_index_cap[i] = e < a.E ? a.edge_index[r * a.E + e] : a.N + (e - a.E) % ng;
    } else if (t < a.s_attr) {                     // edge_attr [E_cap, attr_cols]
      const long long i = t - a.s_dst;
      a.edge_attr_cap[i] = i / a.attr_cols < a.E ? a.edge_attr[i] : 0;
    } else if (t < a.s_batch) {                    // batch [N_cap]
      const long long n = t - a.s_attr;
      a.batch_cap[n] = n < a.N ? a.batch[n] : a.B + min(n - a.N, bg - 1);
    } else if (t < a.s_probs) {                    // rt_probs [N_cap]
      const long long n = t - a.s_batch;
      a.probs_cap[n] = n < a.N ? a.probs[n] : 0.f;
    } else if (t < a.s_pnn) {                      // pattern_num_nodes [N_cap]
      const long long n = t - a.s_probs;
      a.pnn_cap[n] = n < a.N ? a.pnn[n] : 1.f;
    } else if (t < a.s_ent) {                      // entry_id [B_cap]
      const long long b = t - a.s_pnn;
      a.entry_id_cap[b] = b < a.B ? a.entry_id[b] : 0;
    } else {                                       // y [B_cap]
      const long long b = t - a.s_ent;
      a.y_cap[b] = b < a.B ? a.y[b] : 1;
    }
  }
}

int pad_check(long long N, long long E, long long B, long long N_cap, long long E_cap, long long B_cap) {
  if (N < 0 || E < 0 || B < 1 || N_cap < N || E_cap < E || B_cap < B) return PERT_ERR_BADARG;
  const long long ng = N_cap - N, bg = B_cap - B;
  if (bg < 1 || ng < bg) return PERT_ERR_BADARG;                 // >= 1 ghost graph, each with >= 1 node
  if (E_cap - E > PERT_PAD_MAX_GHOST_DEGREE * ng) return PERT_ERR_BADARG;   // ghost in-degree <= 4
  if (N_cap > 0x7fffffffLL || E_cap > 0x7fffffffLL) return PERT_ERR_BADARG;
  return PERT_OK;
}

}  // namespace

extern "C" {

int pert_batch_pad(const float* x, const int64_t* cat_X, const int64_t* edge_index, const int64_t* edge_attr,
                   const int64_t* batch, const int64_t* entry_id, const int64_t* y, const float* rt_probs,
                   const float* pattern_num_nodes, long long N, long long E, long long B, int F, int n_cat,
                   int attr_cols, float* x_cap, int64_t* cat_X_cap, int64_t* edge_index_cap, int64_t* edge_attr_cap,
                   int64_t* batch_cap, int64_t* entry_id_cap, int64_t* y_cap, float* rt_probs_cap,
                   float* pattern_num_nodes_cap, long long N_cap, long long E_cap, long long B_cap, long long* live,
                   void* stream) {
  if (F < 1 || n_cat < 1 || attr_cols < 1) return PERT_ERR_BADARG;
  const int rc = pad_check(N, E, B, N_cap, E_cap, B_cap);
  if (rc) return rc;
  if (!x_cap || !cat_X_cap || !edge_index_cap || !edge_attr_cap || !batch_cap || !entry_id_cap || !y_cap ||
      !rt_probs_cap || !pattern_num_nodes_cap || !live || !entry_id || !y)
    return PERT_ERR_BADARG;
  if (N > 0 && (!x || !cat_X || !batch || !rt_probs || !pattern_num_nodes)) return PERT_ERR_BADARG;
  if (E > 0 && (!edge_index || !edge_attr)) return PERT_ERR_BADARG;
  PadArgs a{};
  a.x = x; a.probs = rt_probs; a.pnn = pattern_num_nodes;
  a.cat_X = cat_X; a.edge_index = edge_index; a.edge_attr = edge_attr; a.batch = batch; a.entry_id = entry_id; a.y = y;
  a.x_cap = x_cap; a.probs_cap = rt_probs_cap; a.pnn_cap = pattern_num_nodes_cap;
  a.cat_X_cap = cat_X_cap; a.edge_index_cap = edge_index_cap; a.edge_attr_cap = edge_attr_cap;
  a.batch_cap = batch_cap; a.entry_id_cap = entry_id_cap; a.y_cap = y_cap; a.live = live;
  a.N = N; a.E = E; a.B = B; a.N_cap = N_cap; a.E_cap = E_cap; a.B_cap = B_cap;
  a.F = F; a.n_cat = n_cat; a.attr_cols = attr_cols;
  a.s_x = N_cap * F;
  a.s_cat = a.s_x + N_cap * n_cat;
  a.s_src = a.s_cat + E_cap;
  a.s_dst = a.s_src + E_cap;
  a.s_attr = a.s_dst + E_cap * attr_cols;
  a.s_batch = a.s_attr + N_cap;
  a.s_probs = a.s_batch + N_cap;
  a.s_pnn = a.s_probs + N_cap;
  a.s_ent = a.s_pnn + B_cap;
  a.s_y = a.s_ent + B_cap;
  long long blocks = pert_cdiv(a.s_y, 256);
  if (blocks > 8LL * PERT_NUM_SMS) blocks = 8LL * PERT_NUM_SMS;
  k_batch_pad<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a);
  PERT_LAUNCH_CHECK();
  return PERT_OK;
}

}  // extern "C"
