/* libpertgnn -- C-ABI of the H100 (sm_90a) hot path of PERT-GNN.
 *
 * The reference (handasontam/PERT-GNN-KDD23) is pure Python on top of torch_geometric 2.4.0 and has no
 * FFI of its own; the "interface each entry point replaces" is therefore the Python/PyG call the
 * reference makes at the cited file:line.  INTEGRATION.md shows the ctypes binding (the one this
 * repository ships in pert_gnn_kdd23_b200/_lib.py) a maintainer of the reference would add.
 *
 * Conventions (all entry points):
 *   - every data buffer (inputs, outputs, workspaces, scratch) is a CALLER-OWNED DEVICE pointer: the library
 *     allocates no device memory for data (the one exception is pert_peer_alloc, whose purpose is to allocate the
 *     IPC-shareable exchange buffer);  fp32 row-major, `ld*` = row stride in floats; indices int32 inside the library,
 *     int64 where the reference's tensors are int64 (edge_index, edge_attr, batch, ids);
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous, nothing synchronises; every call acts on the
 *     CURRENT CUDA device, which must be the device that owns the buffers and the stream (the Python binding enters
 *     torch.cuda.device(tensor.device) around each call);
 *   - return value: 0 = ok; > 0 = cudaError_t of a failed launch/memset; < 0 = library code
 *     (PERT_ERR_*).  Never throws, never exits.  Out-of-range indices found ON THE DEVICE are
 *     reported by writing PERT_ERR_RANGE into the optional device word `status`;
 *   - library-owned state (all of it; none of it is data): (1) per device, one auxiliary non-blocking stream and
 *     two events the step engine (pert_model_forward/backward) uses to run independent small kernels beside the main
 *     chain (fork/join by events, capture-safe); the host-side issue of engine calls on
 *     one device is serialised by a mutex, so engines driven from several host threads / streams stay correct (their
 *     side work shares that one auxiliary stream); (2) the SM count of
 *     each device, read once; (3) environment switches read once (debug / measurement A/B only):
 *     PERT_GEMM_TC, PERT_LINEAR_BWD_FUSED, PERT_PEER_MODE.
 *     With that, operator-level calls are re-entrant and thread-safe across streams;
 *   - rows of float matrices must be 16-byte aligned (ld % 4 == 0, base pointer 16-byte aligned)
 *     unless stated otherwise.
 */
#ifndef PERTGNN_H_
#define PERTGNN_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PERT_OK 0
#define PERT_ERR_BADARG (-1)
#define PERT_ERR_UNSUPPORTED (-2)
#define PERT_ERR_RANGE (-3)
#define PERT_ERR_PEER_TIMEOUT (-4)

/* ABI version (major*1000 + minor).  2000: pert_tconv_bwd takes rpc_ws; node_depth / eval-metric entry points.
 * 2001: pert_pert_graph_count / pert_pert_graph_build.  2002: pert_allreduce_adam timing[5], reduce-scatter form.
 * 2003: pert_span_graph_count / pert_span_graph_build.  2004: pert_linear_bwd_planes(_supported).
 * 2005: pert_model_forward takes dropout + dropout_state, pert_model_backward takes dropout; later, and additive (no
 * existing signature changed): pert_bn_linear_fwd_planes(_supported); pert_batch_pad, pert_model_forward_live,
 * pert_model_backward_live, pert_pinball_loss_live, pert_eval_metrics_live; pert_tconv_fwd_c, pert_tconv_bwd_c,
 * pert_model_width (the step engine accepts every hidden width 1..256); pert_trace_group_* (trace grouping);
 * pert_store_assemble_requests (request assembly with the exact or as-of resource join); pert_store_resources_count /
 * _merge (appending and evicting resource rows of a live store), pert_store_resources_update_count / _update_merge
 * (replacing and deleting them by key); pert_ingest_* (appending traces to a live store);
 * pert_ingest_evict_* (evicting traces from a live store); pert_store_assemble_whatif (per-request pattern mixes and
 * resource overrides), pert_store_lookup_resources; pert_raw_* (processed tables from raw rows); pert_raw_window_*
 * (raw resource samples aggregated into the open buckets' statistics); pert_linear_bwd_planes_ex, pert_tconv_bwd_bn
 * (_supported) (the BatchNorm backward folded into the node-linear and conv backward passes); pert_tconv_fwd_stats
 * (the conv forward with the BatchNorm statistics of its output); pert_flat_grow (relayout of the flat parameter and
 * optimizer buffers when embedding tables grow); pert_model_workspace_bytes_q, pert_model_packed_bytes_q,
 * pert_model_workspace_offset_q, pert_model_forward_q, pert_model_backward_q, pert_pinball_loss_q, pert_eval_metrics_q
 * (a global head with several quantile outputs); pert_calib_workspace_bytes, pert_calib_offsets, pert_calib_apply
 * (conformal calibration of the quantile levels); pert_cpd_workspace_bytes, pert_cpd_fit, pert_cpd_tail,
 * pert_cpd_quantile (the conformal predictive distribution: tail probabilities, p-values and quantiles at any level);
 * pert_cpd_merge_workspace_bytes, pert_cpd_merge (inserting scores into and removing them from a fitted table).
 * An additive entry point leaves the version as it is. */
int pert_version(void);

/* ---- index construction (integer, bit-exact) ---------------------------------------------------
 * Replaces the COO handling PyG MessagePassing does implicitly for TransformerConv.propagate
 * (reference model.py:100,104) and the edge_index offsetting/collation of pert_gnn.py:107-119,
 * 201-209: builds, once per batch, a STABLE CSR by target and CSC by source.
 *   edge_index int64 [2,E] (row 0 source, row 1 target);  edge_attr int64 [E,attr_cols] or NULL
 *   (columns 0,1 = interface id, rpctype id -- reference model.py:93-94), ids checked < n_if/n_rpc.
 * out (int32): rowptr[N+1], perm[E] (original edge id at CSR slot), csr_src[E], csr_if[E], csr_rpc[E],
 *              colptr[N+1], csc_pos[E] (CSR slot of the edge at CSC slot), csc_dst[E].
 * Definition of the layout: oracle/index_oracle.py:build_index. */
long long pert_index_workspace_bytes(long long N, long long E);
int pert_build_index(const int64_t* edge_index, const int64_t* edge_attr, int attr_cols, long long N, long long E,
                     int n_if, int n_rpc, int* rowptr, int* perm, int* csr_src, int* csr_if, int* csr_rpc,
                     int* colptr, int* csc_pos, int* csc_dst, void* workspace, long long workspace_bytes,
                     int* status, void* stream);

/* ptr[B+1] int32 from the PyG `batch` vector (Batch.ptr; pert_gnn.py:201-209 collation).
 * workspace >= 64 KiB is always enough for B < 2^22. */
int pert_graph_ptr(const int64_t* batch, long long N, long long B, int* ptr, void* workspace,
                   long long workspace_bytes, int* status, void* stream);

/* Level index: min hop depth from roots[g] over out-edges inside graph g, -1 if unreachable.
 * Replaces misc.py:52-63 (DFS.dfs_min_node_depth) + :107-136.  gptr[B+1], colptr/csc_dst from
 * pert_build_index, roots[B] global node ids, depth[N] int32 out. */
int pert_min_depth(const int* gptr, long long B, const int* colptr, const int* csc_dst, const int* roots,
                   int* depth, void* stream);

/* The tensor the reference stores as Data.node_depth (misc.py:159-175: unreachable -> 0, divide by the graph's max
 * depth or 1; misc.py:215,368: torch.tensor(float, dtype=long) truncation -> {0,1}) from pert_min_depth's output.
 * gptr[B+1], depth[N] int32 (-1 unreachable), node_depth[N] int64 (viewed [N,1] by the caller). */
int pert_node_depth(const int* gptr, long long B, const int* depth, int64_t* node_depth, void* stream);

/* Level-major node order inside each graph (BASELINE north_star "per-level index layout for coalescing"):
 * order[N] int32 = node ids sorted by (graph, level, id), unreachable nodes last inside their graph
 * (definition: oracle/index_oracle.py:level_order).  The reference has no counterpart (its model never reads
 * node_depth, SURVEY.md fact 3); it is a layout key for collation. */
int pert_level_order(const int* gptr, long long B, const int* depth, int* order, void* stream);

/* ---- segmented reduce (the scatter-max / scatter-add metric kernel) -----------------------------
 * out[i,:] = reduce over CSR segment i of msg rows; op 0 = sum, 1 = max; empty segment -> 0.
 * Replaces torch_geometric.utils.scatter(reduce='max'|'sum') as used by utils.softmax and
 * aggr='add' (call sites model.py:100,104) and global_add_pool (model.py:107).
 * perm NULL: msg rows already in CSR order; else row of slot p is perm[p]. */
int pert_segment_reduce_fwd(const float* msg, const int* rowptr, const int* perm, float* out, long long N, int H,
                            int op, void* stream);
int pert_segment_reduce_bwd(const float* dout, const float* msg, const float* out, const int* rowptr,
                            const int* perm, float* dmsg, long long N, int H, int op, void* stream);

/* ---- fused TransformerConv message passing -------------------------------------------------------
 * Replaces torch_geometric.nn.TransformerConv.propagate/message/aggregate (heads=1, edge_dim set,
 * root_weight) -- reference model.py:26-51 (construction), :100,:104 (calls).  q,k,v,s: [N,H] planes with
 * row stride ld (s = lin_skip(x), may be NULL); t_if [n_if,H], t_rpc [n_rpc,H] = embedding tables already
 * multiplied by the two halves of lin_edge.weight (NULL,NULL = no edge features).  out [N,H];
 * alpha [E] (CSR order) is saved for backward.  H in {4,8,16,32,64,96,128,192,256}.
 * E = number of edges, B_hint = number of graphs in the batch (0 if unknown): only used to size the shared-memory
 * node tiles of the staged kernels (csrc/tconv_tile.cu); n_rpc = rows of t_rpc. */
int pert_tconv_supported_width(int H);
int pert_tconv_fwd(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                   const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                   float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E, long long B_hint, int H,
                   void* stream);
/* g = dL/dout [N,H] (stride ld_g).  Writes dq,dk,dv [N,H] (stride ld_d), dsp [E] scratch; ACCUMULATES
 * (+=, atomics) into dt_if [n_if,H] and dt_rpc [n_rpc,H] (caller zeroes them once per step).
 * rpc_ws: caller scratch of PERT_TCONV_RPC_WS_FLOATS * N floats (per-target sums of alpha / ds by rpc type, written by
 * the target pass and consumed by the source pass of the same call) or NULL; with NULL, or n_rpc > 8, the rpc-table
 * gradient falls back to per-edge shared-memory atomics (same result, slower). */
#define PERT_TCONV_RPC_WS_FLOATS 16
int pert_tconv_bwd(const float* g, int ld_g, const float* q, const float* k, const float* v, int ld,
                   const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr,
                   const int* csc_pos, const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha,
                   float* dq, float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                   int n_rpc, long long N, long long E, long long B_hint, int H, void* stream);
/* The same two for a conv of logical width C run at a kernel width H >= C (1 <= C <= H, else PERT_ERR_BADARG): the
 * planes, tables and outputs are [*, H] with columns [C, H) zero, and the logits are scaled by 1/sqrt(C) instead of
 * 1/sqrt(H), so the first C columns are those of the width-C conv and the rest stay 0.  pert_tconv_fwd / _bwd are these
 * with C = H. */
int pert_tconv_fwd_c(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                     const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if, const float* t_rpc,
                     float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E, long long B_hint, int H,
                     int C, void* stream);
int pert_tconv_bwd_c(const float* g, int ld_g, const float* q, const float* k, const float* v, int ld,
                     const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr,
                     const int* csc_pos, const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha,
                     float* dq, float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                     int n_rpc, long long N, long long E, long long B_hint, int H, int C, void* stream);
/* pert_tconv_fwd_c that also leaves the BatchNorm statistics of `out` (the training forward of the step engine):
 * bn_acc [2][H] doubles (+=; the caller zeroes it) receives, per node tile, n_b mean_b and M2_b + n_b mean_b^2 of each
 * column, M2_b the tile's sum of squares centred on its mean_b (so mean = bn_acc[c] / n and the biased variance
 * (bn_acc[H + c] - n mean^2) / n, n = live[0], or N without live), counting the rows below live[0] (live: optional
 * device {N, B} of a padded batch; NULL: all N).  *fused = 1 when the staged tile kernel ran and bn_acc holds the
 * statistics; *fused = 0 (bn_acc untouched) when the shape takes the per-row kernels, or bn_acc is NULL: the caller
 * then computes the statistics with its own pass.  `out` is bit-identical to pert_tconv_fwd_c's. */
int pert_tconv_fwd_stats(const float* q, const float* k, const float* v, const float* s, int ld, const int* rowptr,
                         const int* csr_src, const int* csr_if, const int* csr_rpc, const float* t_if,
                         const float* t_rpc, float* out, int ld_out, float* alpha, int n_rpc, long long N, long long E,
                         long long B_hint, int H, int C, double* bn_acc, const long long* live, int* fused,
                         void* stream);
/* The backward of the BatchNorm(+ReLU, +dropout) that feeds a conv, folded into that conv's backward (training): the
 * conv's output gradient g is not read but computed row by row where the target pass loads it, and written to g (the
 * node-linear backward of the conv reads it as its skip plane; pert_bn_bwd semantics):
 *   dz = dx * (y > 0) * relu_scale,  g = gamma rstd (dz - sums[0:H] / n - xhat sums[H:2H] / n),  xhat = (x - mean) rstd,
 *   n = live[0] (NULL: N), rows >= n get g = 0;  dbeta += sums[0:H], dgamma += sums[H:2H]  (as float).
 * sums: the fp64 column sums of dz and dz * xhat over the rows below n, as pert_linear_bwd_planes_ex leaves them.
 * dx, y, x are dense [N, H] rows. */
typedef struct PertBnBwd {
  const float* dx;        /* gradient w.r.t. y */
  const float* y;         /* relu(bn(x)) [* keep * scale]: the forward's output of the BatchNorm */
  const float* x;         /* BatchNorm input */
  const float* mean;      /* [H] batch statistics of the forward */
  const float* rstd;
  const float* gamma;
  const double* sums;     /* [2H] */
  float* dgamma;          /* [H], += */
  float* dbeta;
  const long long* live;  /* optional {N, B} of a padded batch */
  float relu_scale;       /* 1 / (1 - p) after inverted dropout, else 1 */
} PertBnBwd;
/* pert_tconv_bwd_c with g = BN backward of bn (written, not read).  PERT_ERR_BADARG as pert_tconv_bwd_c, and for NULL or
 * misaligned BatchNorm operands.  PERT_ERR_UNSUPPORTED (nothing launched: use pert_bn_bwd + pert_tconv_bwd_c) unless
 * H = 64 and the shared-memory-staged conv kernels take the shape: ld = ld_g = ld_d = H and an rpc table of at most
 * 16 KiB.  pert_tconv_bwd_bn_supported: 1 if H and n_rpc qualify, else 0. */
int pert_tconv_bwd_bn(float* g, int ld_g, const float* q, const float* k, const float* v, int ld, const int* rowptr,
                      const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                      const int* csc_dst, const float* t_if, const float* t_rpc, const float* alpha, float* dq,
                      float* dk, float* dv, int ld_d, float* dsp, float* rpc_ws, float* dt_if, float* dt_rpc,
                      int n_rpc, long long N, long long E, long long B_hint, int H, int C, const PertBnBwd* bn,
                      void* stream);
int pert_tconv_bwd_bn_supported(int H, int n_rpc);

/* ---- dense linears (exact fp32) --------------------------------------------------------------------
 * Replace torch_geometric.nn.Linear / the lin_* of TransformerConv (model.py:26-55,105,110-112).
 * "Blocked" matrices: element (r,c) at base + (c / cb)*cbs + r*ld + (c % cb); cb <= 0 means a plain matrix.
 *   NT: C[M,Nc] (=|+=) A[M,K] . B[Nc,K]^T (+ bias) (relu)
 *   TN: C[Mc,Nc] += A[R,Mc]^T . B[R,Nc]      (atomic accumulation; weight gradients)
 *   colsum: out[c] += sum_r A[r,c]            (bias gradients) */
int pert_gemm_nt(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, const float* bias,
                 float* C, int ldc, int c_cb, long long c_cbs, long long M, int Nc, int K, int relu, int accumulate,
                 void* stream);
/* a_colsum (optional, [Mc]): also accumulates a_colsum[m] += sum_r A[r,m] (the bias gradient of the same linear,
 * fused into the producer of the tensor-core kernel: A is read once for both). */
int pert_gemm_tn(const float* A, int lda, int a_cb, long long a_cbs, const float* B, int ldb, int b_cb,
                 long long b_cbs, float* C, int ldc, float* a_colsum, long long R, int Mc, int Nc, void* stream);
int pert_colsum(const float* A, int lda, int a_cb, long long a_cbs, float* out, long long R, int Cc, void* stream);
/* Backward of the plane-blocked node linear [q|k|v|skip] = X . W4^T + b4 in one pass over the gradient planes
 * (tensor cores, 3xTF32; dY and X are read once):
 *   dY: 4 planes [N, H] (row stride H, plane stride plane_stride);  X [N, K] (ldx);  W4t = W4^T [K, 4H] (ldw);
 *   dW4 [4H, K] (ldw4) += dY^T . X;   db4 [4H] += colsum(dY);   dX[:, 0:Kd] (ldx_out) = dY . W4[:, 0:Kd] (written,
 *   columns Kd.. untouched; bit-identical from run to run).
 * PERT_ERR_BADARG for NULL pointers, negative sizes, Kd > K, a leading dimension shorter than its row or
 * overlapping planes.  PERT_ERR_UNSUPPORTED (nothing launched: use pert_gemm_tn + pert_gemm_nt) unless H = 64,
 * K in {64, 80}, Kd in {64, K}, N >= 4096, ldx == K, 16-byte aligned dY / X / dX rows, 8-byte aligned dW4 rows, and a
 * cluster of 4 CTAs fits on the device; also with PERT_LINEAR_BWD_FUSED=0 or PERT_GEMM_TC=0.
 * pert_linear_bwd_planes_supported: 1 if the shape, the switches and the current device qualify, else 0; operand
 * alignment and ldx == K are the caller's to ensure (the engine's workspace always meets them). */
int pert_linear_bwd_planes(const float* dY, long long plane_stride, const float* X, int ldx, const float* W4t, int ldw,
                           float* dW4, int ldw4, float* db4, float* dX, int ldx_out, long long N, int H, int K, int Kd,
                           void* stream);
int pert_linear_bwd_planes_supported(long long N, int H, int K, int Kd);
/* The same with the column sums of the BatchNorm backward of the previous conv (bn_sums != NULL; K = Kd = H), for
 * pert_tconv_bwd_bn: X is that BatchNorm's output y, dX its gradient dx, and
 *   bn_sums[0:H] += sum dz,  bn_sums[H:2H] += sum dz * (bn_x - bn_mean) bn_rstd,  dz = dX * (X > 0) * relu_scale
 * over the rows below live[0] (NULL: all N); bn_x dense [N, H].  dX and the weight gradients are those of
 * pert_linear_bwd_planes (dX bit-identical).  bn_sums = NULL: pert_linear_bwd_planes. */
int pert_linear_bwd_planes_ex(const float* dY, long long plane_stride, const float* X, int ldx, const float* W4t,
                              int ldw, float* dW4, int ldw4, float* db4, float* dX, int ldx_out, long long N, int H,
                              int K, int Kd, const float* bn_x, const float* bn_mean, const float* bn_rstd,
                              float relu_scale, const long long* live, double* bn_sums, void* stream);
/* Forward of the same node linear in one pass over A (tensor cores, 3xTF32), optionally with the BatchNorm(+ReLU,
 * +dropout) of the previous conv applied while A is loaded:
 *   planes: 4 planes [N, H] (row stride H, plane stride plane_stride) = A' . W4^T + b4,  W4 [4H, K] (ldw), b4 [4H];
 *   bn = 0: A' = A [N, K] (lda);
 *   bn != 0 (K = H): A' = y = relu(bn(A)) [* keep * scale], with exactly the semantics and arguments of pert_bn_fwd_ex
 *     (training: batch statistics from `workspace`, computed here unless stats_ready; running statistics and
 *     num_batches_tracked updated; eval: running statistics; dropout > 0 in training: the mask of layer drop_layer at
 *     drop_ctr), and y is also written to x_out (ld_x_out), bit-identical to pert_bn_fwd_ex's output.
 * PERT_ERR_BADARG for NULL pointers, negative sizes, a leading dimension shorter than its row, overlapping planes and
 * the BatchNorm argument errors of pert_bn_fwd_ex.  PERT_ERR_UNSUPPORTED (nothing launched: use pert_bn_fwd_ex +
 * pert_gemm_nt) unless H = 64, K in {64, 80} (bn: K = H), N >= 4096, lda == K, ld_x_out == K, 16-byte aligned A,
 * x_out and plane rows, and the kernel fits on the device; also with PERT_GEMM_TC=0.
 * pert_bn_linear_fwd_planes_supported: 1 if the shape, the switch and the current device qualify, else 0. */
int pert_bn_linear_fwd_planes(const float* A, int lda, int bn, const float* gamma, const float* beta,
                              float* running_mean, float* running_var, long long* num_batches_tracked, float eps,
                              float momentum, int training, float* mean, float* rstd, float* x_out, int ld_x_out,
                              void* workspace, long long workspace_bytes, int stats_ready, float dropout,
                              const long long* drop_ctr, int drop_layer, const float* W4, int ldw, const float* b4,
                              float* planes, long long plane_stride, long long N, int H, int K, void* stream);
int pert_bn_linear_fwd_planes_supported(long long N, int H, int K);

/* ---- embeddings / concat (model.py:87-97,108) -------------------------------------------------------
 * fwd: out[n,0:H] (=|+=) table[ids[n*id_stride]];  bwd: dtable[ids[n*id_stride]] += dy[n,0:H]. */
int pert_embedding_fwd(const float* table, int n_rows, const int64_t* ids, int id_stride, float* out, int ld_out,
                       long long N, int H, int accumulate, int* status, void* stream);
int pert_embedding_bwd(const float* dy, int ld_dy, const int64_t* ids, int id_stride, float* dtable, int n_rows,
                       long long N, int H, void* stream);
/* out[n, col0:col0+F] = x[n,0:F] (x dense [N,F], any F), out[n, col0+F:ld_out] = 0. */
int pert_copy_cols(const float* x, int F, float* out, int ld_out, int col0, long long N, void* stream);

/* ---- BatchNorm1d (+ fused ReLU) (model.py:33,43,101-102) ---------------------------------------------
 * training: batch statistics (biased var), running stats updated with `momentum` (unbiased var),
 * num_batches_tracked += 1; eval: running statistics.  mean/rstd [H] are outputs saved for backward. */
long long pert_bn_workspace_bytes(long long N, int H);
int pert_bn_fwd(const float* x, int ld_x, const float* gamma, const float* beta, float* running_mean,
                float* running_var, long long* num_batches_tracked, float eps, float momentum, int training,
                int relu, float* mean, float* rstd, float* y, int ld_y, long long N, int H, void* workspace,
                long long workspace_bytes, void* stream);
/* dy = grad wrt the (post-ReLU) output y; sums = [2H] scratch; dgamma/dbeta (+=) may be NULL. */
int pert_bn_bwd(const float* dy, int ld_dy, const float* y, int ld_y, const float* x, int ld_x, const float* mean,
                const float* rstd, const float* gamma, int relu, int training, float* dx, int ld_dx, float* dgamma,
                float* dbeta, float* sums, long long N, int H, void* stream);

/* ---- local head + probability-weighted add-pool (model.py:105-107) -----------------------------------
 * local[n] = <x_n, w_local> + b_local (skipped when local NULL);
 * pool[batch[n], :] += (x_n * probs[n]) / pnn[n]   (pool [B,H] is zeroed by the call). */
int pert_pool_fwd(const float* x, int ld, const float* probs, const float* pnn, const int64_t* batch,
                  const float* w_local, const float* b_local, float* local, float* pool, long long N, long long B,
                  int H, int* status, void* stream);
int pert_pool_bwd(const float* dpool, const float* dlocal, const float* x, int ld, const float* probs,
                  const float* pnn, const int64_t* batch, const float* w_local, float* dx, int ld_dx,
                  float* dw_local, float* db_local, long long N, long long B, int H, void* stream);

/* dy[i] = 0 where y[i] <= 0 (F.relu backward, model.py:111). */
int pert_relu_bwd(const float* y, float* dy, long long n, void* stream);

/* Pinball loss (pert_gnn.py:191-193): loss[0] = mean(max(tau*e,(tau-1)*e)), e = y - yhat;
 * dyhat[B] = grad_scale * dloss/dyhat (either output may be NULL); a tie (e = 0) gets torch.maximum's even split,
 * grad_scale * 0.5 * (1 - 2 tau) / B.  B is at most INT_MAX: a larger B is PERT_ERR_BADARG before any launch, as it
 * is for the other three loss and metric entries below. */
int pert_pinball_loss(const int64_t* y, const float* yhat, float tau, long long B, float grad_scale, float* loss,
                      float* dyhat, void* stream);

/* Eval / epoch metrics without host syncs (pert_gnn.py:249, :284-289): acc[0] += sum|yhat - y|, acc[1] += sum(|yhat - y| / y),
 * acc[2] += B * pinball_tau(y, yhat)  (= sum of the per-graph pinball terms).  acc: 3 doubles on the device, zeroed by
 * the caller at the start of an epoch and read back once at its end. */
int pert_eval_metrics(const int64_t* y, const float* yhat, float tau, long long B, double* acc, void* stream);
/* The same two on a batch padded by pert_batch_pad: y / yhat hold B (capacity) graphs, the device word live = {N, B_real}
 * says how many are real.  The loss is the mean over the real graphs and dyhat = 0 for the ghost graphs; the metrics sum
 * over the real graphs only.  live = NULL is exactly pert_pinball_loss / pert_eval_metrics. */
int pert_pinball_loss_live(const int64_t* y, const float* yhat, float tau, long long B, float grad_scale, float* loss,
                           float* dyhat, const long long* live, void* stream);
int pert_eval_metrics_live(const int64_t* y, const float* yhat, float tau, long long B, double* acc,
                           const long long* live, void* stream);
/* The same two for a head with T quantile outputs: yhat [B, T] (row-major), column t the taus[t]-quantile.  taus is a
 * HOST array of T levels, read during the call and passed to the kernel by value (a captured graph keeps them).
 *   loss[0] = 1/(B T) sum_b sum_t max(tau_t e_bt, (tau_t - 1) e_bt), e_bt = y_b - yhat_bt; dyhat [B, T] its gradient
 *   times grad_scale, ties split evenly as in pert_pinball_loss.
 *   acc: 4T + 1 doubles; for level t, acc[4t + 0..3] += sum |yhat_t - y|, sum |yhat_t - y| / y, sum of the pinball
 *   terms at tau_t and the count of graphs with y <= yhat_t (coverage); acc[4T] += the count of graphs whose levels
 *   cross (yhat_t > yhat_{t+1} for some t).
 * live as above (NULL: every graph is real; ghost graphs get dyhat = 0 in every column and are not counted).  At T = 1
 * the loss runs pert_pinball_loss's kernel, and the metric sums acc[0..2] follow pert_eval_metrics's arithmetic.
 * PERT_ERR_BADARG, before any CUDA call, for T outside 1..PERT_MAX_QUANTILES, taus NULL, NaN, outside [0, 1] or not
 * strictly increasing, and everything the plain forms refuse. */
#define PERT_MAX_QUANTILES 8
int pert_pinball_loss_q(const int64_t* y, const float* yhat, const float* taus, int T, long long B, float grad_scale,
                        float* loss, float* dyhat, const long long* live, void* stream);
int pert_eval_metrics_q(const int64_t* y, const float* yhat, const float* taus, int T, long long B, double* acc,
                        const long long* live, void* stream);

/* ---- conformal calibration of the quantile levels (csrc/calib.cu) ------------------------------------------------
 * Split-conformal offsets per group (entry id) and level from n held-out graphs: labels y [n] int64, predictions
 * yhat [n, T] fp32 row-major, group [n] int64 (NULL: every graph in the global group only).  taus is a HOST array of T
 * doubles, read during the call.  Outputs, G + 1 rows (G = n_groups), row G the global group of all n graphs:
 *   off [(G+1) T] fp32, count [G+1] int32 (graphs per group), own [(G+1) T] int8 (1: the group's own offset).
 * Score s = (float)y - yhat in fp32 (the conversion of pert_eval_metrics_q's coverage test), -0 canonicalised to +0.
 * For a group of n_g graphs at level tau, k = max(1, ceil((n_g + 1) tau)) in double; the group's own offset is used iff
 * k <= n_g and n_g >= min_count, and is then exactly the k-th smallest score of the group (an element of the score
 * array, bit for bit); otherwise the group gets row G's offset.  Row G follows the rule over all n graphs (min_count
 * does not apply to it).  Deterministic: integer histograms only, no device-to-host read inside the call.
 * On the device, a NaN or infinite score or a group id outside [0, G) writes PERT_ERR_RANGE to status (the outputs
 * are then undefined).  PERT_ERR_BADARG, before any CUDA call, for NULL pointers (group excepted), n < 1, n T >= 2^31,
 * T outside 1..PERT_MAX_QUANTILES, taus NaN, outside [0, 1] or not strictly increasing, n_groups < 0 or >= INT_MAX,
 * min_count < 1, a level at which row G cannot be formed (k > n, e.g. tau = 1) and a workspace below
 * pert_calib_workspace_bytes(n, T, n_groups) (-1 for sizes the fit refuses). */
long long pert_calib_workspace_bytes(long long n, int T, long long n_groups);
int pert_calib_offsets(const int64_t* y, const float* yhat, const int64_t* group, long long n, int T,
                       const double* taus, long long n_groups, long long min_count, float* off, int* count,
                       int8_t* own, void* workspace, long long workspace_bytes, int* status, void* stream);
/* In place on yhat [Q, T]: yhat[q, t] += off[g, t] in fp32, g = group[q]; an id outside [0, n_rows - 1) (an entry the
 * calibration never saw) or group = NULL reads the global row n_rows - 1.  off = NULL adds nothing.  monotone != 0 then
 * replaces each row by its running max over t (removes crossing levels; it only raises predictions).  live as in
 * pert_eval_metrics_q: rows q >= live[1] (ghost graphs of a padded batch) are left untouched.  PERT_ERR_BADARG, before
 * any CUDA call, for Q < 0, Q T >= 2^31, T outside 1..PERT_MAX_QUANTILES, yhat NULL with Q > 0, and off with n_rows
 * outside 1..INT_MAX.  Nothing is launched when Q = 0 or when off = NULL and monotone = 0. */
int pert_calib_apply(float* yhat, const int64_t* group, long long Q, int T, const float* off, long long n_rows,
                     int monotone, const long long* live, void* stream);

/* ---- conformal predictive distribution (csrc/cpd.cu) -------------------------------------------------------------
 * The sorted split-conformal scores of n held-out graphs per group (entry id), around one prediction column: labels
 * y [n] int64, predictions yhat[i ld + col] fp32 (a [n, ld] head output needs no copy), group [n] int64 (NULL: the
 * global row only).  Score s = fl((float)y - yhat) in fp32, -0 canonicalised to +0 (the score of pert_calib_offsets).
 * Outputs, G = n_groups:
 *   ptr [G + 2] int64: row g (0 <= g < G) holds the scores of group g at scores[ptr[g] .. ptr[g+1]), ascending; row G,
 *     all n scores ascending, is scores[ptr[G] .. ptr[G+1]).  ptr[G+1] = 2n with groups, n without.
 *   scores [ptr[G+1]] fp32.
 * Only values are kept, so the table is unique: bit-identical to a sort of every row, run to run.  No device-to-host
 * read inside the call.  On the device, a NaN or infinite score or a group id outside [0, G) writes PERT_ERR_RANGE to
 * status (the outputs are then undefined).  PERT_ERR_BADARG, before any CUDA call, for NULL pointers (group
 * excepted), n < 1, n >= 2^30, n_groups < 0 or > INT_MAX - 2, ld < 1, col outside [0, ld) and a workspace below
 * pert_cpd_workspace_bytes(n, n_groups) (-1 for sizes the fit refuses). */
long long pert_cpd_workspace_bytes(long long n, long long n_groups);
int pert_cpd_fit(const int64_t* y, const float* yhat, long long ld, int col, const int64_t* group, long long n,
                 long long n_groups, float* scores, long long* ptr, void* workspace, long long workspace_bytes,
                 int* status, void* stream);
/* Queries of a fitted table (scores, ptr, n_groups as written by pert_cpd_fit) for Q requests with predictions
 * yhat[q ld + col] and group ids group[q] (NULL: every request reads row G).
 * pert_cpd_tail: request q reads row r = g iff 0 <= g < G and n_g >= min_count (>= 1), else row G (so an id outside
 * [0, G) reads row G).  For each of its S thresholds x[q S + j] (x [Q, S] fp32), or for its label y[q] (y [Q] int64,
 * S = 1; exactly one of x and y is non-NULL), with c = fl(x - yhat) (-0 -> +0) and m the row's size it writes
 * ge[q S + j] = #{s >= c} and gt[q S + j] = #{s > c} (int32), and row[q] = r.  Then gt / (m + 1) and (ge + 1) / (m + 1)
 * bracket P(latency > x) under the conformal predictive distribution, and (ge + 1) / (m + 1) at x = y is the
 * conformal p-value of the label.
 * pert_cpd_quantile: for each of L levels taus (a HOST array of doubles, 1 <= L <= PERT_MAX_QUANTILES, in [0, 1] and
 * strictly increasing), k = max(1, ceil((m + 1) tau)) in double; row g iff 0 <= g < G, k <= n_g and n_g >= min_count,
 * else row G; out[q L + l] = fl(yhat + s_(k)) fp32, the k-th smallest score of the row, or +inf where k exceeds even
 * row G's size.  At a level pert_calib_offsets can fit, this is that offset added as pert_calib_apply adds it.
 * Both: a NaN c (a NaN threshold or prediction, or inf - inf) or a NaN prediction writes PERT_ERR_RANGE to status.
 * PERT_ERR_BADARG, before any CUDA call, for Q < 0, Q S (Q L) >= 2^31, n_groups < 0 or > INT_MAX - 2, min_count < 1,
 * ld < 1, col outside [0, ld), NULL table, yhat, status or outputs with Q > 0, and for pert_cpd_tail S < 1, both or
 * neither of x and y, or y with S != 1.  Nothing is launched when Q = 0. */
int pert_cpd_tail(const float* scores, const long long* ptr, long long n_groups, long long min_count,
                  const float* yhat, long long ld, int col, const int64_t* group, long long Q, const float* x, int S,
                  const int64_t* y, int* ge, int* gt, int* row, int* status, void* stream);
int pert_cpd_quantile(const float* scores, const long long* ptr, long long n_groups, long long min_count,
                      const float* yhat, long long ld, int col, const int64_t* group, long long Q, const double* taus,
                      int L, float* out, int* status, void* stream);
/* Updates of a fitted table: the old table (scores [n_old], ptr [G_old + 2], n_old = ptr[G_old + 1]) plus (sign = +1)
 * or minus (sign = -1) a delta table written by pert_cpd_fit (d_scores [n_delta], d_ptr [G_new + 2], n_delta =
 * d_ptr[G_new + 1], G_new >= G_old) gives out_scores [n_old + sign n_delta] and out_ptr [G_new + 2].  Output row r is
 * old row r (r < G_old), an empty old row (G_old <= r < G_new) or old row G_old (r = G_new), merged with delta row r:
 * a sorted merge, or the multiset difference (each value v loses c(v) copies, c(v) its count in the delta row).  The
 * result is the table pert_cpd_fit writes for the union or difference of the two scored sets, bit for bit.  A delta
 * row of a removal that holds a value more often than its old row (so also one longer than its old row) writes
 * PERT_ERR_RANGE to status (out_scores is then undefined; no write leaves it).  No device-to-host read inside the
 * call.  PERT_ERR_BADARG, before any CUDA call, for NULL pointers, G_old < 0, G_new < G_old or > INT_MAX - 2, a sign
 * other than +-1, n_old < 1, n_delta < 1, a result below 1 or at 2^31 scores (the fit's n < 2^30 graphs) and a
 * workspace below pert_cpd_merge_workspace_bytes(G_old, G_new, n_old, n_delta) (-1 for sizes neither sign accepts). */
long long pert_cpd_merge_workspace_bytes(long long G_old, long long G_new, long long n_old, long long n_delta);
int pert_cpd_merge(const float* scores, const long long* ptr, long long G_old, long long n_old, const float* d_scores,
                   const long long* d_ptr, long long G_new, long long n_delta, int sign, float* out_scores,
                   long long* out_ptr, void* workspace, long long workspace_bytes, int* status, void* stream);

/* torch.optim.Adam step (pert_gnn.py:343,247) over one flat parameter buffer; g is scaled by grad_scale, weight_decay
 * is L2 added to the scaled gradient (not AdamW's decoupled decay).  The bias corrections lr / (1 - beta1^step) and
 * sqrt(1 - beta2^step) are computed in double on the host, as torch does, and passed to the kernel as floats. */
int pert_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                   float eps, float weight_decay, long long step, float grad_scale, void* stream);

/* ---- relayout of the flat parameter buffers when parameters grow (csrc/flat.cu) -----------------------------------
 * train.FlatParams keeps every trainable parameter in one flat fp32 buffer, each starting on a PERT_FLAT_ALIGN-float
 * boundary; Adam's m and v share that layout.  Growing a parameter (new embedding rows) moves every one after it.
 * `segs` is a HOST array [n_seg][4] of (old_off, new_off, old_len, new_len) in floats, one row per parameter.  One
 * launch, in stream order and without a host synchronisation:
 *   - copies old_len floats of each segment of p_old, m_old and v_old bit for bit to new_off of p_new, m_new, v_new;
 *   - writes 0 to every other float of the new buffers (the new tail of each segment and all padding);
 *   - writes 0 to the whole new gradient buffer g_new.
 * m_old / m_new and v_old / v_new may be NULL (as a pair: no optimizer state to carry).  PERT_ERR_BADARG, before any
 * CUDA call, for n_seg outside [0, PERT_FLAT_MAX_SEGS], sizes that are negative, not multiples of PERT_FLAT_ALIGN or with
 * n_new < n_old, offsets that are not multiples of PERT_FLAT_ALIGN, segments out of order or overlapping in either
 * layout or running past n_old / n_new, new_len < old_len, NULL p_old / p_new / g_new or one half of a pair, pointers
 * not 16-byte aligned, and any two buffers that overlap. */
#define PERT_FLAT_ALIGN 64
#define PERT_FLAT_MAX_SEGS 128
int pert_flat_grow(const long long* segs, int n_seg, long long n_old, long long n_new, const float* p_old,
                   float* p_new, const float* m_old, float* m_new, const float* v_old, float* v_new, float* g_new,
                   void* stream);

/* ---- gradient all-reduce fused with Adam over NVLink peer memory (csrc/peer.cu) ---------------------------
 * Data-parallel form of pert_adam_step, one kernel per step and no NCCL on the step path: every rank publishes its
 * flat gradient in an IPC-shared exchange buffer and signals the peers; rank r then sums slice r of all gradients in
 * rank order (1/world of each peer's buffer over NVLink), applies Adam to that slice (m, v are only maintained for the
 * owned slice, ZeRO-1 style) and stores the new parameters into every peer's buffer; a second flag round collects the
 * other slices (replicas bit-identical by construction).  That form runs for world > 4; up to 4 ranks every rank pulls
 * whole gradients and runs the full Adam with ONE flag round (cheaper while the volume is small; measured both ways at
 * 2 and 8 GPUs).  PERT_PEER_MODE=ag|rs (environment, same on all ranks) forces one form.
 * path.  Setup: pert_peer_alloc on every rank, exchange the 64-byte handles out of band (torch.distributed
 * all_gather), pert_peer_open the peers'.  `xbufs` is a HOST array of `world` device pointers (index = rank).
 * `step` = 1, 2, ... must equal the number of calls so far on every rank (the arrival counter is monotonic).
 * A peer that never arrives makes the kernel write PERT_ERR_PEER_TIMEOUT to `status` after ~3 s instead of hanging. */
long long pert_peer_exchange_bytes(long long n);
int pert_peer_alloc(long long bytes, void** ptr, unsigned char* handle64);
int pert_peer_open(const unsigned char* handle64, void** ptr);
int pert_peer_close(void* ptr);
int pert_peer_free(void* ptr);
int pert_allreduce_adam(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                        float eps, float weight_decay, long long step, float grad_scale, void* const* xbufs, int rank,
                        int world, int* status, long long* timing, void* stream);
/* timing (optional device int64[5]): CTA 0 adds the nanoseconds (%globaltimer) it spent in (0) publishing the gradient
 * + grid arrival, (1) waiting for the peers' flags -- the slowest rank's skew plus the flag round trip --, (2) the
 * rank-ordered reduce + Adam of its slice + parameter push + second arrival, (3) waiting for the peers' slices and
 * copying them, and (4) += 1 per call: the per-phase evidence behind the scaling curve (bench.py `peer`). */

/* ---- whole-model step engine --------------------------------------------------------------------------
 * SAGEDeterministic.forward (model.py:76-114) and its backward as one call each: the same kernels as above,
 * issued back-to-back from C++ (no interpreter between launches).  Parameters live in ONE flat fp32 buffer in
 * the reference's own tensor shapes; PertModelDesc gives the offset (in floats, each 16-byte aligned) of every
 * tensor, named after the reference's state_dict keys.  Gradients go to a second flat buffer with the same
 * offsets and are ACCUMULATED (+=), like autograd.  The workspace holds packed operands, saved activations and
 * temporaries; its first pert_model_packed_bytes() bytes must be zero when first used (padding columns).
 *
 * Any hidden width 1 <= H <= 256 runs: the engine runs a model of width H at the internal width Hp =
 * pert_model_width(H), the smallest attention-kernel width >= H (one of 4, 8, 16, 32, 64, 96, 128, 192, 256; Hp = H
 * at those).  Every parameter is copied into zero-padded Hp-wide packs each step, and columns [H, Hp) of every
 * activation and gradient stay exactly 0; the parameters, gradients and outputs are those of the width-H model (the
 * attention logits are scaled by 1/sqrt(H)), at the cost of a width-Hp step.  Workspace sizes and the layouts below are
 * at Hp. */
#define PERT_MAX_CONVS 8
#define PERT_MAX_CAT 4
typedef struct PertModelDesc {
  int32_t F;        /* in_channels of the model (raw node features, 9)             model.py:13  */
  int32_t H;        /* hidden_channels                                              model.py:18  */
  int32_t n_convs;  /* max(2, num_layers)                                           model.py:24-52 */
  int32_t n_cat;    /* len(cat_dims)                                                model.py:57-60 */
  int32_t cat_rows[PERT_MAX_CAT];
  int32_t n_entry, n_if, n_rpc; /* rows of entry_embeds / interface_embeds / rpctype_embeds  model.py:63-67 */
  int32_t k0;       /* padded input width of conv 0: round_up(F + Hp, 8), Hp = pert_model_width(H) */
  float bn_eps, bn_momentum;
  long long off_cat[PERT_MAX_CAT];                 /* cat_embedding.{i}.weight [rows,H] */
  long long off_entry, off_if, off_rpc;            /* *_embeds.weight                   */
  long long off_wq[PERT_MAX_CONVS], off_bq[PERT_MAX_CONVS]; /* convs.{l}.lin_query.{weight [H,Din],bias} */
  long long off_wk[PERT_MAX_CONVS], off_bk[PERT_MAX_CONVS]; /* lin_key   */
  long long off_wv[PERT_MAX_CONVS], off_bv[PERT_MAX_CONVS]; /* lin_value */
  long long off_ws[PERT_MAX_CONVS], off_bs[PERT_MAX_CONVS]; /* lin_skip  */
  long long off_we[PERT_MAX_CONVS];                         /* lin_edge.weight [H,2H] */
  long long off_bn_g[PERT_MAX_CONVS], off_bn_b[PERT_MAX_CONVS]; /* bns.{l}.weight / bias */
  long long off_local_w, off_local_b;              /* local_linear   [1,H],[1]  */
  long long off_g1_w, off_g1_b;                    /* global_linear1 [H,2H],[H] */
  long long off_g2_w, off_g2_b;                    /* global_linear2 [1,H],[1]  */
} PertModelDesc;

/* Hp for a model of hidden width H (see above), PERT_ERR_UNSUPPORTED outside 1..256. */
int pert_model_width(int H);
long long pert_model_workspace_bytes(const PertModelDesc* desc, long long N, long long E, long long B);
long long pert_model_packed_bytes(const PertModelDesc* desc);
/* Test / debug aid: offset (in floats) inside the workspace of a saved activation of the last forward:
 * which = 0: input of conv `layer` (>= 1) = post-BatchNorm-ReLU activations [N,Hp]; which = 1: relu(global_linear1)
 * [B,Hp] (Hp = pert_model_width(H); columns [H, Hp) are 0).
 * Lets a reference be differentiated on the same linear piece of the network (which ReLUs were active).
 * The engine's own intermediates, so that each of its kernels can be checked on its own inputs:
 *   which = 2: z = [pool | entry_embeds[entry_id]] [B,2Hp], the global head's input (valid after a forward);
 *   which = 3: dpool [B,Hp], the head's gradient with respect to pool (valid after a backward);
 *   which = 4 / 5: t_if / t_rpc of conv `layer` [n_if / n_rpc, Hp] = interface / rpc embeddings . lin_edge half^T
 *                  (forward);
 *   which = 6 / 7: their gradients dt_if / dt_rpc, same shapes (backward);
 *   which = 8..11: the packed gradients of conv `layer` before they are added into the flat gradient buffer (backward):
 *                  dW4 [4Hp,K] (rows q|k|v|skip, K = k0 for conv 0 with columns [emb | x | pad], else Hp), db4 [4Hp],
 *                  and the two lin_edge halves dWeA / dWeB [Hp,Hp] (row = output feature).
 * which 4..11 need 0 <= layer < n_convs, else PERT_ERR_BADARG; which 1..3 ignore `layer`. */
long long pert_model_workspace_offset(const PertModelDesc* desc, long long N, long long E, long long B, int which,
                                      int layer);
/* bn_running: [n_convs-1][2][Hp] (running_mean | running_var; the first H of each Hp are the model's, the others belong
 * to padding columns, whose outputs are 0 whatever they hold, and only need to be finite and >= 0 for the variance), bn_nbt: [n_convs-1] int64 (either may be NULL in
 * training mode); index arrays from pert_build_index (built with edge_attr); probs/pnn [N] fp32.
 * Outputs: global_pred [B], local_pred [N] (NULL to skip). */
/* Optional measurement probe: the engine records the two caller-created cudaEvent_t around ONE kernel family of ONE
 * layer, on the launching stream (bench.py: in-step duration of the dominant kernel).  kernel: 1 = fused conv forward,
 * 2 = fused conv backward (target + source pass), 3 = node-linear forward GEMM, 4 = weight-gradient GEMM (where the
 * node-linear backward runs fused, pert_linear_bwd_planes: the whole backward, weight and data gradient),
 * 5 = data-gradient GEMM (an empty interval right after 4 when fused).  NULL = no probe. */
typedef struct PertProbe {
  int32_t kernel, layer;
  void* ev_start;
  void* ev_stop;
} PertProbe;
int pert_model_forward(const PertModelDesc* desc, const float* params, float* bn_running, long long* bn_nbt,
                       const float* x, const int64_t* cat_X, const int64_t* entry_id, const float* probs,
                       const float* pnn, const int64_t* batch, long long N, long long E, long long B,
                       const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc, void* workspace,
                       long long workspace_bytes, int training, float dropout, long long* dropout_state,
                       float* global_pred, float* local_pred, int* status, const PertProbe* probe, void* index_ready,
                       void* stream);
/* index_ready: optional cudaEvent_t recorded (on another stream) after the graph index was built: the forward waits
 * for it only right before the first attention kernel, so the index build overlaps the parameter pack, the input
 * prologue and the first GEMM.  NULL = the index is already complete in `stream` order.
 *
 * dropout: F.dropout(x, p=dropout, training) after every BatchNorm + ReLU (model.py:103), fused into the BatchNorm
 * apply.  Used only when training; p = 0 runs exactly the kernels of a model without dropout.  dropout_state: caller
 * device memory, two int64 {seed, step}; a training forward with p > 0 reads it in stream order and adds 1 to step, so
 * a captured graph draws a new mask on every replay.  The mask is a pure function of (seed, step, layer, position):
 *   Philox4x32-10 (Random123), key = (seed & 0xffffffff, seed >> 32),
 *   counter = (g, l, step & 0xffffffff, step >> 32), g = row*(Hp/4) + col/4 (the float4 group), l = the conv whose
 *   BatchNorm output is dropped (0 .. n_convs-2); output word j of the group decides column col + j.
 *   Element kept iff word >= T, T = floor(p * 2^32) in fp64 (p = 1: all dropped); kept values are multiplied by
 *   (float)(1 / (1 - p)), 0 at p = 1.
 * PERT_ERR_BADARG, before any CUDA call, when p is NaN or outside [0, 1], or when training with p > 0 and
 * dropout_state is NULL or N*Hp/4 >= 2^32.
 *
 * Must follow pert_model_forward on the same workspace, with the same training flag and dropout (the backward applies
 * the 1/(1-p) factor; the mask is read back from the saved activations).  d_global [B], d_local [N] or NULL. */
int pert_model_backward(const PertModelDesc* desc, const float* params, float* grads, const int64_t* cat_X,
                        const int64_t* entry_id, const float* probs, const float* pnn, const int64_t* batch,
                        long long N, long long E, long long B, const int* rowptr, const int* csr_src,
                        const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                        const int* csc_dst, void* workspace, long long workspace_bytes, int training, float dropout,
                        const float* d_global, const float* d_local, const PertProbe* probe, void* stream);

/* ---- capacity buckets: padded batches for CUDA-graph replay (csrc/pad.cu) ------------------------------------------
 * pert_batch_pad copies a batch of N nodes, E edges and B graphs bit for bit into caller buffers of the capacity sizes
 * (N_cap, E_cap, B_cap) -- x [N,F] fp32, cat_X [N,n_cat], edge_index [2,E], edge_attr [E,attr_cols], batch [N],
 * entry_id [B], y [B] int64, rt_probs [N], pattern_num_nodes [N] fp32 -- fills the tail with ghost graphs and stores
 * live = {N, B} (two int64 on the device).  Ghost node j = N + j' belongs to graph B + min(j', B_cap - B - 1) (the batch
 * vector stays sorted, every ghost graph owns a node); ghost edge E + k' is a self-loop on ghost node
 * N + k' mod (N_cap - N); x = 0, every id = 0, rt_probs = 0, pattern_num_nodes = 1, y = 1.  No edge joins a ghost to
 * a real node and ghost graphs pool nothing, so a step on the padded batch that reads `live` where a count enters the
 * arithmetic (pert_model_forward_live / backward_live, pert_pinball_loss_live, pert_eval_metrics_live) computes what
 * the unpadded step computes for the real graphs.  One grid-stride launch; its source pointers change with every
 * batch, so it runs eagerly in front of a replayed graph.
 * PERT_ERR_BADARG, before any CUDA call, for NULL pointers, negative sizes, B < 1, F / n_cat / attr_cols < 1, a
 * capacity below the real size, N_cap - N < max(1, B_cap - B), E_cap - E > PERT_PAD_MAX_GHOST_DEGREE * (N_cap - N)
 * (a ghost in-degree above 4) or a capacity above 2^31 - 1. */
#define PERT_PAD_MAX_GHOST_DEGREE 4
int pert_batch_pad(const float* x, const int64_t* cat_X, const int64_t* edge_index, const int64_t* edge_attr,
                   const int64_t* batch, const int64_t* entry_id, const int64_t* y, const float* rt_probs,
                   const float* pattern_num_nodes, long long N, long long E, long long B, int F, int n_cat,
                   int attr_cols, float* x_cap, int64_t* cat_X_cap, int64_t* edge_index_cap, int64_t* edge_attr_cap,
                   int64_t* batch_cap, int64_t* entry_id_cap, int64_t* y_cap, float* rt_probs_cap,
                   float* pattern_num_nodes_cap, long long N_cap, long long E_cap, long long B_cap, long long* live,
                   void* stream);
/* pert_model_forward / pert_model_backward on a padded batch: N, E, B and every array are those of the capacity
 * buffers, live the word pert_batch_pad wrote.  In training the BatchNorm statistics (mean, variance, the running
 * statistics with the unbiased factor of the real N) count the real rows only, and the BatchNorm backward divides by
 * the real N and gives the ghost rows a zero gradient.  The backward's d_global must be 0 for the ghost graphs
 * (pert_pinball_loss_live).  The dropout mask of a real row does not depend on the padding.  live = NULL is exactly
 * pert_model_forward / pert_model_backward. */
int pert_model_forward_live(const PertModelDesc* desc, const float* params, float* bn_running, long long* bn_nbt,
                            const float* x, const int64_t* cat_X, const int64_t* entry_id, const float* probs,
                            const float* pnn, const int64_t* batch, long long N, long long E, long long B,
                            const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc,
                            void* workspace, long long workspace_bytes, int training, float dropout,
                            long long* dropout_state, float* global_pred, float* local_pred, int* status,
                            const PertProbe* probe, void* index_ready, const long long* live, void* stream);
int pert_model_backward_live(const PertModelDesc* desc, const float* params, float* grads, const int64_t* cat_X,
                             const int64_t* entry_id, const float* probs, const float* pnn, const int64_t* batch,
                             long long N, long long E, long long B, const int* rowptr, const int* csr_src,
                             const int* csr_if, const int* csr_rpc, const int* colptr, const int* csc_pos,
                             const int* csc_dst, void* workspace, long long workspace_bytes, int training,
                             float dropout, const float* d_global, const float* d_local, const PertProbe* probe,
                             const long long* live, void* stream);
/* A global head with n_out outputs (1 <= n_out <= PERT_MAX_QUANTILES): global_linear2 is [n_out, H] / [n_out] at
 * off_g2_w / off_g2_b, global_pred and d_global are [B, n_out] (row-major).  Everything else is as in the _live forms
 * (live may be NULL); at n_out = 1 these are exactly those calls.  At Hp > H the padded copy of global_linear2.weight
 * (and its gradient) is [n_out, Hp], so the workspace layout depends on n_out: size, offsets and packed bytes come from
 * the _q forms.  PERT_ERR_BADARG, before any CUDA call, for n_out outside 1..PERT_MAX_QUANTILES and everything the
 * plain forms refuse. */
long long pert_model_workspace_bytes_q(const PertModelDesc* desc, int n_out, long long N, long long E, long long B);
long long pert_model_packed_bytes_q(const PertModelDesc* desc, int n_out);
long long pert_model_workspace_offset_q(const PertModelDesc* desc, int n_out, long long N, long long E, long long B,
                                        int which, int layer);
int pert_model_forward_q(const PertModelDesc* desc, int n_out, const float* params, float* bn_running,
                         long long* bn_nbt, const float* x, const int64_t* cat_X, const int64_t* entry_id,
                         const float* probs, const float* pnn, const int64_t* batch, long long N, long long E,
                         long long B, const int* rowptr, const int* csr_src, const int* csr_if, const int* csr_rpc,
                         void* workspace, long long workspace_bytes, int training, float dropout,
                         long long* dropout_state, float* global_pred, float* local_pred, int* status,
                         const PertProbe* probe, void* index_ready, const long long* live, void* stream);
int pert_model_backward_q(const PertModelDesc* desc, int n_out, const float* params, float* grads,
                          const int64_t* cat_X, const int64_t* entry_id, const float* probs, const float* pnn,
                          const int64_t* batch, long long N, long long E, long long B, const int* rowptr,
                          const int* csr_src, const int* csr_if, const int* csr_rpc, const int* colptr,
                          const int* csc_pos, const int* csc_dst, void* workspace, long long workspace_bytes,
                          int training, float dropout, const float* d_global, const float* d_local,
                          const PertProbe* probe, const long long* live, void* stream);

/* ---- device-side batch assembly from a resident pattern store (csrc/store.cu) ---------------------------------------
 * Replaces the host-side sample assembly + collation + per-step probability expansion of the reference:
 * get_entry_data / get_x / get_cat_X / get_node_depth / get_edge_index / get_edge_attr / get_pattern_num_nodes
 * (pert_gnn.py:40-173), torch_geometric DataLoader collation (:201-209) and transform_pattern_probs (:122-131,
 * :220-230).  All pointers are caller-owned device arrays, built once from the reference's artefacts
 * (runtime2graph, entry2runtimes, resource_df, tr2data -- pert_gnn.py:297-305) by pert_gnn_kdd23_b200/store.py.
 *   patterns p = 0..n_pat-1 (the runtime ids in the order the store assigned):
 *     pat_nptr/pat_eptr [n_pat+1] node / edge offsets into the concatenated arrays;  pat_ms [sum n] = ms_id (cat_X);
 *     pat_depth [sum n] = node_depth;  pat_last [sum n] = 1 iff the node is the LAST one of its ms inside the pattern
 *     (get_x's ms2nid dict, pert_gnn.py:54-65);  pat_src/pat_dst [sum e] pattern-local edge_index;  pat_attr [sum e, attr_cols]
 *   entries: ent_ptr [n_ent+1] into ent_pat (pattern index) / ent_prob (float32 probability), in the dict order of
 *     entry2runtimes[entry];  ent_nodes / ent_edges [n_ent] totals over the entry's patterns
 *   resources: res_keys [n_res] sorted int64 = timestamp * n_ms + ms, res_vals [n_res, 8] float32,
 *     ms_has_res [n_ms] = 1 iff ms has a row at ANY timestamp (pert_gnn.py:138)
 *   traces: trace_entry [n_traces] int32, trace_ts [n_traces] int64, trace_y [n_traces] int64. */
typedef struct PertStore {
  int32_t n_pat, n_ent, n_res, n_ms, attr_cols;
  long long n_traces;
  const int32_t *pat_nptr, *pat_eptr;
  const int64_t *pat_ms, *pat_depth;
  const uint8_t* pat_last;
  const int32_t *pat_src, *pat_dst;
  const int64_t* pat_attr;
  const int32_t *ent_ptr, *ent_pat;
  const float* ent_prob;
  const int32_t *ent_nodes, *ent_edges;
  const int64_t* res_keys;
  const float* res_vals;
  const uint8_t* ms_has_res;
  const int32_t* trace_entry;
  const int64_t *trace_ts, *trace_y;
} PertStore;
/* Output = the collated Batch of pert_gnn.py:163-173 + PyG collate + the per-node probability of :220-230. */
typedef struct PertBatchOut {
  float* x;                  /* [N, 9]  */
  int64_t* cat_X;            /* [N, 1]  */
  int64_t* node_depth;       /* [N, 1]  */
  float* pattern_num_nodes;  /* [N, 1]  */
  float* rt_probs;           /* [N, 1]  per-node pattern probability (transform_pattern_probs) */
  int64_t* batch;            /* [N]     */
  int64_t* edge_index;       /* [2, E]  */
  int64_t* edge_attr;        /* [E, attr_cols] */
  int64_t* entry_id;         /* [B]     */
  int64_t* y;                /* [B]     */
  int64_t* ptr;              /* [B+1]   */
  float* pattern_probs;      /* [sum_b patterns(entry_b), 1] */
} PertBatchOut;
/* trace_ids [B] int64 (device): which traces form the batch.  N, E = node / edge totals of the batch (the caller sizes
 * the outputs from its host copy of ent_nodes / ent_edges -- no device sync); offsets: int32 scratch of 3 * (B + 1).
 * status: PERT_ERR_RANGE for a trace id out of range or a (timestamp, ms) row missing for a resourced ms (the
 * reference raises KeyError there). */
int pert_store_assemble(const PertStore* store, const int64_t* trace_ids, long long B, long long N, long long E,
                        int* offsets, const PertBatchOut* out, int* status, void* stream);

/* ---- request assembly: batches for prediction, keyed by (entry, time) instead of a trace id ---------------------------
 * Graph b is entry entry_ids[b] at the time bucket floor(timestamps[b] / 30000) * 30000 (floor division: -1 maps to
 * -30000, preprocess.py:39).  The outputs are those of pert_store_assemble for a trace of that entry and bucket, except
 * y, which is not written (out->y may be NULL): a request has no label.  Entries, patterns and resources come from
 * `store`; its trace table is not read.  N, E and the sum of the entries' pattern counts size the outputs as above.
 * Resource join, for the node that receives statistics (the last node of a resourced microservice in its pattern):
 *   asof == NULL (exact): the (bucket, ms) row; a missing row sets PERT_ERR_RANGE in status (as pert_store_assemble);
 *   asof != NULL (as-of): the row of that ms with the largest timestamp <= bucket; among rows sharing that timestamp the
 *     one the exact join picks (the first in the store's sorted order), so an exact hit gives identical features in both
 *     modes.  No such row: the node keeps the missing indicator [0 x 8, 1]; this is not an error.
 * PertResourceAsOf indexes the store's resource rows by microservice: rows of ms m are k = ms_ptr[m] .. ms_ptr[m+1]-1,
 * ts[k] (int64) ascending, and row[k] (int32) is the row's index into res_keys / res_vals (ascending among equal ts).
 * 12 bytes per resource row (ts and row may be NULL when n_res = 0); PatternStore builds it on the device with the store.
 * On the device, an entry < 0, >= n_ent or without patterns sets PERT_ERR_RANGE and the graph is assembled as entry 0
 * (as a bad trace id reads trace 0).  PERT_ERR_BADARG, before any CUDA call, for NULL pointers and negative sizes;
 * B = 0 returns PERT_OK and launches nothing. */
typedef struct PertResourceAsOf {
  const int32_t* ms_ptr;  /* [n_ms+1] */
  const int64_t* ts;      /* [n_res]  */
  const int32_t* row;     /* [n_res]  */
} PertResourceAsOf;
int pert_store_assemble_requests(const PertStore* store, const PertResourceAsOf* asof, const int64_t* entry_ids,
                                 const int64_t* timestamps, long long B, long long N, long long E, int* offsets,
                                 const PertBatchOut* out, int* status, void* stream);

/* ---- what-if request assembly: per-request pattern mixes and resource overrides ------------------------------------
 * pert_store_assemble_requests with two optional replacements, read from `w`:
 *   mix_ptr [B+1] int64 (NULL: every request uses its entry's stored mix): graph b is the concatenation, in slot order,
 *     of patterns mix_pat[k] (int32 pattern index) for k = mix_ptr[b] .. mix_ptr[b+1]-1, with probabilities
 *     mix_prob[k] (float32) as pattern_probs and per-node rt_probs, instead of entry_ids[b]'s stored mix.  The offsets
 *     are absolute, so a caller may pass a slice of a longer CSR without rebasing.  entry_ids[b] still selects the
 *     entry embedding and is written to entry_id; its own mix is not read, so it may be empty.  Probabilities are used
 *     as given (they need not sum to 1).
 *   scenario [B] int64 (NULL: none), with n_ov override rows: ov_keys [n_ov] int64 = scenario * n_ms + ms, sorted
 *     ascending (>= 0), and ov_vals [n_ov, 8] float32 (16-byte aligned).  At the node that receives statistics (the last
 *     node of a microservice m in its pattern, as in pert_store_assemble), a request with scenario s >= 0 reads the
 *     first row of key s * n_ms + m if there is one: the node gets its values and indicator 0, whether or not m has
 *     resource rows, and no store join runs for it (so the exact join flags no missing row there).  Without such a
 *     row (scenario -1, or no row of that key) the exact or as-of join runs as in pert_store_assemble_requests.
 * N, E and the pattern total size the outputs as there: sums over the requests' mixes of the patterns' node / edge
 * counts and the mixes' lengths.  On the device, an entry < 0 or >= n_ent (or, without mix_ptr, with no patterns), a
 * pattern index outside [0, n_pat) or an empty mix sets PERT_ERR_RANGE in status; the graph then reads entry 0 /
 * pattern 0 (an empty mix gives an empty graph).  PERT_ERR_BADARG, before any CUDA call, for NULL pointers with
 * non-zero sizes (including w, and mix_pat / mix_prob when mix_ptr is set), negative sizes and ov_vals not 16-byte
 * aligned; B = 0 returns PERT_OK and launches nothing. */
typedef struct PertWhatIf {
  const int64_t* mix_ptr;   /* [B+1] or NULL */
  const int32_t* mix_pat;   /* [mix_ptr[B]]  */
  const float* mix_prob;    /* [mix_ptr[B]]  */
  const int64_t* scenario;  /* [B] or NULL   */
  long long n_ov;
  const int64_t* ov_keys;   /* [n_ov]        */
  const float* ov_vals;     /* [n_ov, 8]     */
} PertWhatIf;
int pert_store_assemble_whatif(const PertStore* store, const PertResourceAsOf* asof, const PertWhatIf* w,
                               const int64_t* entry_ids, const int64_t* timestamps, long long B, long long N,
                               long long E, int* offsets, const PertBatchOut* out, int* status, void* stream);

/* The resource row each join of request assembly reads, for k (timestamp, ms) queries: values [k, 8] float32 get the
 * row of (floor(timestamps[i] / 30000) * 30000, ms[i]) -- the exact join (asof == NULL) or the as-of join -- and
 * found [k] uint8 is 1; with no such row, or ms outside [0, n_ms), values are 0 and found is 0.  Only the resource
 * fields of `store` are read.  PERT_ERR_BADARG, before any CUDA call, for NULL pointers with k > 0, k < 0 or
 * k > 2^31 - 1; k = 0 returns PERT_OK and launches nothing. */
int pert_store_lookup_resources(const PertStore* store, const PertResourceAsOf* asof, const int64_t* timestamps,
                                const int64_t* ms, long long k, float* values, uint8_t* found, void* stream);

/* ---- resource updates of a live store (csrc/resources.cu) -----------------------------------------------------------
 * Append k resource rows to a store's sorted resource table and its as-of index, and drop every row whose timestamp is
 * < evict_before (LLONG_MIN: none), old rows and appended rows alike.  The results are fresh arrays whose contents
 * equal, bit for bit, what the store's constructor builds from the surviving rows in arrival order (the old rows first,
 * in their table order, then the batch in input order): res_keys sorted with equal keys in arrival order, res_vals,
 * ms_has_res [n_ms] = 1 iff ms keeps a row, and the as-of index of those keys.  No old row is re-sorted; equal keys are
 * all kept (the joins read the first), so a later row never replaces an earlier one: that is the update pair below.
 * Inputs, all device arrays:
 *   store, asof: the current table (store->res_keys, res_vals, n_res, n_ms >= 1) and its index (ts / row may be NULL
 *     when n_res = 0); only these fields of the store are read;
 *   new_keys [k] int64: the batch's keys timestamp * n_ms + ms (0 <= ms < n_ms, no overflow: the caller checks),
 *     sorted ascending by a STABLE sort; new_perm [k] int64: input row of every sorted key;
 *   new_vals [k, 8] float32 in input order (16-byte aligned);
 *   new_group [k] int32: positions into new_keys ordered by (ms, position) -- a stable regrouping of the sorted keys by
 *     microservice, as the as-of index regroups the table.
 * Two calls, the caller reading `sizes` from the device between them:
 *   pert_store_resources_count writes ms_ptr_out [n_ms+1] int32 (the new index offsets: the surviving rows per
 *     microservice, scanned), seg [2*n_ms] int32 (per microservice: the first surviving entry of its old index segment,
 *     i.e. asof->ms_ptr[m] + its evicted entries, then the first surviving position of its rows in new_group) and
 *     sizes [3] int64 = {p, q, n_out}: the evicted prefix of the table, the evicted prefix of new_keys, the rows after
 *     the update.  It changes nothing else.
 *   pert_store_resources_merge takes p, q, n_out from sizes and ms_ptr_out / seg unchanged, and writes keys_out
 *     [n_out] int64, vals_out [n_out, 8] float32 (16-byte aligned), has_out [n_ms] uint8, ts_out [n_out] int64 and
 *     row_out [n_out] int32 (the new as-of index with ms_ptr_out).  Outputs may not overlap the inputs.
 * PERT_ERR_BADARG, before any CUDA call, for NULL pointers (output arrays may be NULL when n_out = 0, batch arrays when
 * k = 0), negative sizes, k or n_out above 2^31 - 1, sizes the count cannot have produced, and (merge) new_vals,
 * vals_out or store->res_vals not 16-byte aligned. */
int pert_store_resources_count(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                               const int32_t* new_group, long long k, long long evict_before, int32_t* ms_ptr_out,
                               int32_t* seg, long long* sizes, void* stream);
int pert_store_resources_merge(const PertStore* store, const PertResourceAsOf* asof, const int64_t* new_keys,
                               const int64_t* new_perm, const float* new_vals, const int32_t* new_group, long long k,
                               const int32_t* ms_ptr_out, const int32_t* seg, long long p, long long q,
                               long long n_out, int64_t* keys_out, float* vals_out, uint8_t* has_out, int64_t* ts_out,
                               int32_t* row_out, void* stream);

/* Replacing and deleting resource rows by key (PatternStore.append_resources(replace=True), delete_resources): the same
 * two calls with a drop set, whose keys' old rows all leave the table before the batch goes in.  With L the rows in
 * arrival order and D the drop set, the result is what the constructor builds from [r in L : key(r) not in D and
 * timestamp(r) >= evict_before] followed by the surviving batch rows in input order.  A replace passes its batch's
 * keys as D and the last row of each key as the batch, a delete passes D and no batch, and D empty is the plain append.
 *   drop_keys [n_drop] int64: sorted ascending, unique (0 <= ms < n_ms); drop_group [n_drop] int32: positions into
 *     drop_keys ordered by (ms, position), as new_group;
 *   drop_cnt [2 * (n_drop + 1)] int32: written by the count, read by the merge: the old rows at or above the cut each
 *     drop key removes, as exclusive scans in key order and in drop_group order, each followed by its total;
 *   seg [3 * n_ms + 1] int32: pert_store_resources_count's two parts, then the first drop_group position of every
 *     microservice and n_drop;
 *   sizes [4] int64 = {p, q, n_out, n_dropped}: n_dropped = the old rows the drop set removes (rows it names below
 *     the cut are counted in p), n_out = (n_res - p - n_dropped) + (k - q).
 * The merge takes drop_cnt, seg, p, q, n_dropped and n_out as the count left them.  Arguments, outputs and refusals
 * as pert_store_resources_count / _merge; also PERT_ERR_BADARG for n_drop < 0 or >= 2^31 - 1, NULL drop arrays with
 * n_drop > 0, a NULL drop_cnt, and n_dropped outside [0, n_res - p] or above 0 with n_drop = 0. */
int pert_store_resources_update_count(const PertStore* store, const PertResourceAsOf* asof, const int64_t* drop_keys,
                                      const int32_t* drop_group, long long n_drop, const int64_t* new_keys,
                                      const int32_t* new_group, long long k, long long evict_before,
                                      int32_t* drop_cnt, int32_t* ms_ptr_out, int32_t* seg, long long* sizes,
                                      void* stream);
int pert_store_resources_update_merge(const PertStore* store, const PertResourceAsOf* asof, const int64_t* drop_keys,
                                      const int32_t* drop_group, const int32_t* drop_cnt, long long n_drop,
                                      const int64_t* new_keys, const int64_t* new_perm, const float* new_vals,
                                      const int32_t* new_group, long long k, const int32_t* ms_ptr_out,
                                      const int32_t* seg, long long p, long long q, long long n_dropped,
                                      long long n_out, int64_t* keys_out, float* vals_out, uint8_t* has_out,
                                      int64_t* ts_out, int32_t* row_out, void* stream);

/* ---- trace ingest: appending traces to a live store (csrc/ingest.cu) ------------------------------------------------
 * A chunk of span rows, grouped on its own by pert_trace_group_*, is taken into a store whose patterns are runtimes
 * with known key rows (PatternStore.from_trace_groups).  Pattern j of the store is runtime j's representative; the
 * runtime ids of a store built that way are 0 .. n_pat-1, so a new runtime's id is n_pat + its rank (after an
 * eviction has dropped patterns, the caller shifts these ids to the next unissued one: ids are not reused).
 * Runtime keys: the (um, dm, interface) rows of every representative, file order: rows [3][ld] int64 (um at rows[0..],
 * dm at rows[ld..], interface at rows[2*ld..]), runtime k owning ptr[k] .. ptr[k+1]-1 of each ([n+1] int32).  The
 * runtime table is an open-addressing table over them with the hashes of the trace grouping (2 x hash_bits bits, the
 * same function): slot [S] int32 (runtime index or -1; S a power of two, 64 <= S <= 2^30, n <= S / 2), h1 / h2 [>= n]
 * uint64 the hashes of every runtime. */
typedef struct PertRuntimeKeys {
  long long n;             /* runtimes */
  long long ld;            /* row stride of rows */
  const int32_t* ptr;      /* [n+1] */
  const int64_t* rows;     /* [3][ld] */
} PertRuntimeKeys;
typedef struct PertRuntimeTable {
  long long S;
  int32_t hash_bits;       /* 1..64 (64 except in tests that force collisions) */
  int32_t* slot;           /* [S] */
  uint64_t *h1, *h2;       /* [capacity >= n] */
} PertRuntimeTable;
/* Inserts runtimes first .. keys->n - 1 (their key rows must differ from every other runtime's) and writes their
 * hashes; first = 0 empties the table first (a build or a rebuild into a larger table). */
int pert_ingest_table_insert(const PertRuntimeKeys* keys, long long first, const PertRuntimeTable* table,
                             void* stream);
/* Match of a chunk's runtimes against the store's.  chunk: the chunk's representatives' key rows in the chunk's
 * insertion order (the first three rows of pert_trace_group_gather's output, with its rep_ptr); chunk_runtime_ins
 * [chunk->n]: the insertion index of every chunk runtime id (PertTraceGroups.runtime_ins).  The chunk's runtimes must be
 * distinct (as the grouping makes them).  A chunk runtime matches a store runtime only when the hashes, the length
 * and every row agree.  Outputs: pat_of [chunk->n] = the store pattern of every chunk runtime, insertion order; a new
 * runtime gets n_pat + its rank in insertion order; new_rep [chunk->n] lists the insertion indices of the new runtimes
 * and new_rt [chunk->n] their runtime ids n_pat + rank by chunk runtime id (smallest traceid); n_new [1] int64 their
 * count.  The table is not changed.  workspace: pert_ingest_match_workspace_bytes(chunk->n). */
long long pert_ingest_match_workspace_bytes(long long n_chunk);
int pert_ingest_match(const PertRuntimeKeys* keys, const PertRuntimeTable* table, const PertRuntimeKeys* chunk,
                      const int32_t* chunk_runtime_ins, int32_t* pat_of, int32_t* new_rep, int32_t* new_rt,
                      long long* n_new, void* workspace, long long workspace_bytes, void* stream);
/* Entry-mix merge.  Old mixes: store->n_ent, ent_ptr, ent_pat, ent_nodes, ent_edges (only these fields are read),
 * cnt [n_pairs] the count of every pair, tot [n_ent] the trace total of every entry.  The chunk's mixes (PertChunkMix,
 * from its grouping): ent_pair_ptr / ent_trace_ptr [n_ent+1], pair_runtime / pair_prob [n_pairs], runtime_ins, and
 * pat_of from pert_ingest_match.  pat_nptr / pat_eptr: node / edge offsets of every pattern after the append.
 * Outputs (PertMixOut), n_ent_out = max(store->n_ent, chunk->n_ent) entries: ent_ptr [n_ent_out+1]; ent_pat, ent_prob
 * (fp32), cnt [>= n_pairs + chunk->n_pairs, the first ent_ptr[n_ent_out] written]; ent_nodes, ent_edges, tot
 * [n_ent_out].  Entry e keeps its old pairs in order, then the pairs new to it in chunk order; probability =
 * (old + chunk count) / (old + chunk total) in fp64, rounded to fp32.  Outputs may not overlap the inputs.
 * workspace: pert_ingest_merge_workspace_bytes(n_pairs, chunk->n_pairs, n_ent_out).  PERT_ERR_BADARG, before any CUDA
 * call, for NULL pointers, negative sizes, n_ent_out below either entry count and more than 2^31 - 1 pairs. */
typedef struct PertChunkMix {
  long long n_ent, n_pairs;
  const int32_t *ent_pair_ptr, *ent_trace_ptr, *pair_runtime;
  const double* pair_prob;
  const int32_t *runtime_ins, *pat_of;
} PertChunkMix;
typedef struct PertMixOut {
  int32_t *ent_ptr, *ent_pat;
  float* ent_prob;
  int32_t *cnt, *ent_nodes, *ent_edges, *tot;
} PertMixOut;
long long pert_ingest_merge_workspace_bytes(long long n_pairs, long long n_chunk_pairs, long long n_ent_out);
int pert_ingest_merge(const PertStore* store, const int32_t* cnt, const int32_t* tot, long long n_pairs,
                      const PertChunkMix* chunk, const int32_t* pat_nptr, const int32_t* pat_eptr, long long n_ent_out,
                      const PertMixOut* out, void* workspace, long long workspace_bytes, void* stream);
/* Trace eviction: drops every trace whose bucket (trace_ts) is < before, with the (entry, pattern) pairs left without
 * a trace and the patterns left without a pair.  What the store keeps beside PertStore (PertIngestState): the runtime
 * keys (keys.n = n_pat), trace_pat [n_traces] the pattern of every trace, trace_tid [n_traces] its traceid, cnt
 * [n_pairs] / tot [n_ent] as for pert_ingest_merge, and the totals of pattern nodes, edges and key rows.  The store
 * fields read: n_traces, trace_entry, trace_ts, trace_y, n_ent, ent_ptr, ent_pat, n_pat, pat_nptr, pat_eptr, pat_ms,
 * pat_depth, pat_last, pat_src, pat_dst, pat_attr, attr_cols.
 * Two calls with one host read between them, so that every output is allocated at its exact new size:
 *   pert_ingest_evict_count -> sizes [6] int64 (device): traces T', pairs P', patterns n_pat', nodes N', edges E',
 *                              key rows K' that survive; fills the workspace.
 *   pert_ingest_evict_apply  -> with those sizes (host) and the same workspace: stable compaction into PertEvictOut.
 * Traces keep their order (remap [n_traces] int64: new index or -1, monotone on the survivors); entry e keeps its
 * surviving pairs in order, probability = surviving count / surviving total in fp64 rounded to fp32 (an entry with no
 * trace left gets no pairs and tot 0; n_ent is kept); patterns keep their order (pat_new [n_pat] int32: new index or
 * -1), their nodes, edges and key rows unchanged; ent_pat and trace_pat are renumbered.  Output sizes: mix.ent_ptr
 * [n_ent+1], mix.ent_nodes / ent_edges / tot [n_ent], mix.ent_pat / ent_prob / cnt [P'], trace_* [T'], pat_nptr /
 * pat_eptr / key_ptr [n_pat'+1], pat_ms / pat_depth / pat_last [N'], pat_src / pat_dst [E'], pat_attr [E'][attr_cols],
 * key_rows [3][key_ld] with key_ld >= K'.  Outputs may not overlap the inputs.  The integer atomics of the count
 * make no output depend on scheduling.  workspace: pert_ingest_evict_workspace_bytes(n_traces, n_pairs, n_pat, n_ent).
 * PERT_ERR_BADARG, before any CUDA call, for NULL pointers, negative sizes or sizes above 2^31 - 16, keys.n != n_pat,
 * an undersized workspace, and (apply) sizes outside [0, old size]. */
typedef struct PertIngestState {
  PertRuntimeKeys keys;
  const int32_t* trace_pat;  /* [n_traces] */
  const int64_t* trace_tid;  /* [n_traces] (read by the apply only) */
  const int32_t *cnt, *tot;  /* [n_pairs], [n_ent] */
  long long n_pairs, n_nodes, n_edges, n_key_rows;
} PertIngestState;
typedef struct PertEvictOut {
  PertMixOut mix;
  int64_t* remap;            /* [n_traces] */
  int32_t* trace_entry;      /* [T'] */
  int64_t *trace_ts, *trace_y;
  int32_t* trace_pat;
  int64_t* trace_tid;
  int32_t *pat_new;          /* [n_pat] */
  int32_t *pat_nptr, *pat_eptr;
  int64_t *pat_ms, *pat_depth;
  uint8_t* pat_last;
  int32_t *pat_src, *pat_dst;
  int64_t* pat_attr;
  int32_t* key_ptr;
  int64_t* key_rows;
  long long key_ld;
} PertEvictOut;
long long pert_ingest_evict_workspace_bytes(long long n_traces, long long n_pairs, long long n_pat, long long n_ent);
int pert_ingest_evict_count(const PertStore* store, const PertIngestState* ing, long long before, void* workspace,
                            long long workspace_bytes, long long* sizes, void* stream);
int pert_ingest_evict_apply(const PertStore* store, const PertIngestState* ing, const long long* sizes,
                            const void* workspace, long long workspace_bytes, const PertEvictOut* out, void* stream);

/* ---- PERT-graph construction (SURVEY 8f row N2) ---------------------------------------------------------------
 * Replaces misc.py:221-319 (GraphConstruct.get_pert_edge_index) for T traces at once.  Input: the cleaned span rows
 * (what misc.py:87-105 drop_wrong_edges leaves) of all traces concatenated, row_ptr[T+1]; per row um, dm, interface,
 * rpctype, t_start (= timestamp), t_end (= endTimestamp), all int64 [R]; root_ms[T] (misc.py:138-142).
 * Output per trace: nodes = 2*rows + distinct microservices, edges = 4*rows (edge slots of trace t start at
 * 4*row_ptr[t]); ms_id[N] = sorted_span_id; edge_index[2,4R] with trace-local node ids (global_ids = 0, the
 * per-pattern tensors the reference stores) or batch-global ids (global_ids = 1); edge_attr[4R,4] =
 * [interface, rpctype, call, same_ms]; root_nid[T] = GLOBAL id of stage 0 of the root microservice (-1 + PERT_ERR_RANGE
 * in status if the root is absent; the reference raises KeyError).  Node numbering is the canonical order documented
 * in csrc/pertgraph.cu (the reference's is pandas / set iteration order); edge order is the reference's.
 * Two passes so the caller can size the outputs: _count writes node_cnt[T]; the caller scans it into node_ptr[T+1].
 * max_rows >= the longest trace (<= PERT_PERT_GRAPH_MAX_ROWS); a longer trace sets PERT_ERR_RANGE. */
#define PERT_PERT_GRAPH_MAX_ROWS 2048
int pert_pert_graph_count(const int64_t* row_ptr, long long T, const int64_t* um, const int64_t* dm, int max_rows,
                          int64_t* node_cnt, int* status, void* stream);
int pert_pert_graph_build(const int64_t* row_ptr, long long T, long long R, const int64_t* um, const int64_t* dm,
                          const int64_t* interface, const int64_t* rpctype, const int64_t* t_start,
                          const int64_t* t_end, const int64_t* root_ms, const int64_t* node_ptr, int max_rows,
                          int global_ids, int64_t* ms_id, int64_t* edge_index, int64_t* edge_attr, int64_t* root_nid,
                          int* status, void* stream);
/* Span graph of T traces (misc.py:190-219 get_span_edge_index; `--graph_type span` is pert_gnn.py's default): nodes =
 * the trace's sorted unique microservice ids (ms_id[N], N from pert_span_graph_count), edge_index[2,R] = positions of
 * um / dm in that list (one edge per row, table order; edge slots of trace t start at row_ptr[t]), edge_attr[R,2] =
 * [interface, rpctype], root_nid[T] as above.  Bit-identical to the reference's tensors. */
int pert_span_graph_count(const int64_t* row_ptr, long long T, const int64_t* um, const int64_t* dm, int max_rows,
                          int64_t* node_cnt, int* status, void* stream);
int pert_span_graph_build(const int64_t* row_ptr, long long T, long long R, const int64_t* um, const int64_t* dm,
                          const int64_t* interface, const int64_t* rpctype, const int64_t* root_ms,
                          const int64_t* node_ptr, int max_rows, int global_ids, int64_t* ms_id, int64_t* edge_index,
                          int64_t* edge_attr, int64_t* root_nid, int* status, void* stream);

/* ---- trace grouping: runtime patterns, entry mixes, trace labels (csrc/tracegroup.cu) ------------------------------
 * Replaces the body of preprocess.py main() after get_df() (:269-381): get_tr2ts_map (:32-41, bucket = floor(min
 * timestamp / 30000) * 30000), the label tr2delay (:290-292, y = max |rt|), the runtime id of every trace (:280-293:
 * factorize of the " ".join of its um_dm_interface strings), the entry x trace iteration (:295-316) with its
 * representative trace per runtime (:317-367) and the normalised entry mixes (:371-375).
 * Input: the processed span table, one row per span in file order, int64 device columns of R rows.  Traces are the
 * distinct traceids (ascending, t = 0..T-1); a trace's rows keep file order.  traceid and entryid must lie in
 * [0, 2^31) (else PERT_ERR_RANGE in status and the row / trace is left out); every row of a trace must carry the same
 * entryid (else PERT_ERR_RANGE).  Four calls, the caller reading a size from the device between them:
 *   pert_trace_group_range  -> maxes[2] = {max traceid, max entryid} (-1: none)   => n_keys = maxes[0] + 1
 *   pert_trace_group_keys   -> key_ptr[n_keys+1] (first row slot of every traceid), key_trace[n_keys+1] (trace index of
 *                              every traceid; key_trace[n_keys] = T)             => T
 *   pert_trace_group_build  -> every per-trace / per-runtime / per-entry array, sizes[3] = {n_runtimes, n_pairs, R'}
 *   pert_trace_group_gather -> the rows of the representatives (R'), the only rows the host needs (GraphConstruct).
 * Runtime ids: two traces share one iff their (um, dm, interface) sequences are equal (order and length included);
 * ids count from 0 in order of the smallest traceid of each runtime (Series.factorize over ascending traceids).  The
 * grouping hashes every trace (order-sensitive, 2 x hash_bits bits) into an open-addressing table and merges two traces
 * only after a row-by-row comparison, so hash collisions cost time and never a wrong merge; hash_bits (1..64) is 64
 * except in tests that force collisions.  Iteration order = entries ascending, traceids ascending inside an entry
 * (tr2data's key order).  Outputs do not depend on thread scheduling. */
typedef struct PertSpanTable {
  long long R;
  const int64_t *traceid, *timestamp, *rpcid, *um, *dm, *interface, *rpctype, *rt, *entryid;
} PertSpanTable;
/* Outputs of pert_trace_group_build.  Sizes T (traces), n_ent = max entryid + 1.  Arrays marked [T*] are sized T and
 * hold n_runtimes or n_pairs valid entries (sizes[]); ids are int32 unless stated. */
typedef struct PertTraceGroups {
  int32_t *row_ptr;                  /* [T+1] trace t owns perm[row_ptr[t] .. row_ptr[t+1])                     */
  int32_t *perm;                     /* [R]   row ids grouped by trace, file order inside a trace               */
  int64_t *trace_id, *bucket, *y;    /* [T]   traceid, timestamp bucket (:39), label (:290-292)                 */
  int32_t *entry, *runtime;          /* [T]   entry id, runtime id                                              */
  int32_t *order;                    /* [T]   iteration order: trace index at position p (tr2data key order)    */
  int32_t *ent_trace_ptr;            /* [n_ent+1] entry e owns positions ent_trace_ptr[e] .. [e+1] of `order`   */
  int32_t *ent_pair_ptr;             /* [n_ent+1] entry e owns pairs ent_pair_ptr[e] .. [e+1]                   */
  int32_t *pair_runtime;             /* [T*]  runtime of every (entry, runtime) pair, entry-major, first met first */
  double *pair_prob;                 /* [T*]  count / entry total in fp64 (entry2runtimes, :371-375)            */
  int32_t *occurrences;              /* [T*]  traces per runtime id (:336, :342)                                */
  int32_t *ins_runtime;              /* [T*]  runtime id at insertion index k (runtime2*graph_map key order)    */
  int32_t *rep_trace;                /* [T*]  representative trace (first in iteration order) at insertion index */
  int32_t *runtime_ins;              /* [T*]  insertion index of every runtime id                               */
  int32_t *rep_ptr;                  /* [T+1] row offsets of the representatives' rows, insertion order         */
  int64_t *sizes;                    /* [3]   n_runtimes, n_pairs, R' = rep_ptr[n_runtimes]                      */
} PertTraceGroups;
int pert_trace_group_range(const PertSpanTable* table, int* maxes, int* status, void* stream);
int pert_trace_group_keys(const PertSpanTable* table, long long n_keys, int* key_ptr, int* key_trace, void* workspace,
                          long long workspace_bytes, void* stream);
/* workspace bytes of pert_trace_group_keys (n_traces < 0) or pert_trace_group_build; -1 for bad sizes. */
long long pert_trace_group_workspace_bytes(long long R, long long n_keys, long long n_traces, long long n_ent);
int pert_trace_group_build(const PertSpanTable* table, long long n_keys, long long n_traces, long long n_ent,
                           int hash_bits, const int* key_ptr, const int* key_trace, const PertTraceGroups* out,
                           void* workspace, long long workspace_bytes, int* status, void* stream);
/* rows[8][R'] int64: um, dm, interface, rpctype, timestamp, endTimestamp (= timestamp + |rt|, :263), rpcid, rt of the
 * representatives' rows, representative k at rep_ptr[k], file order inside it. */
int pert_trace_group_gather(const PertSpanTable* table, const int* perm, const int* row_ptr, const int* rep_trace,
                            const int* rep_ptr, long long n_runtimes, long long R_rep, int64_t* rows, void* stream);

/* ---- raw tables: the processed span and resource tables from raw rows (csrc/rawtable.cu) ---------------------------
 * Replaces the else-branch of preprocess.py get_df() (:201-261) after the CSV read: drop_duplicates (:212), the sort by
 * timestamp (:213), map_consecutive_ids of traceid / interface / entryid / rpcid / rpctype (:216-221), the entry
 * detection of filter_traces_with_missing_entry_and_get_delay (:99-149), the resource-coverage filter (:155-177), the
 * per-entry occurrence filter (:180-188), the microservice ids (:248-254) and the resource groupby(["timestamp",
 * "msname"]).agg([max, min, mean, median]) (:227-242).
 * Input: dictionary-encoded device columns.  Every call-graph column but timestamp and rt holds codes into a host
 * dictionary of n_* entries; um, dm and the resource msname share ONE dictionary whose codes are in lexicographic name
 * order.  A row with a code outside its dictionary sets PERT_ERR_RANGE in status and is left out.  At most 2^30
 * call-graph rows and traceid codes (every hash-table slot is an int32), else PERT_ERR_BADARG.  The calls, in order
 * (the caller reads a size between them):
 *   pert_raw_resource_groups -> groups of the resource rows sorted (stable) by (timestamp, ms), has_res[n_ms] => G
 *   pert_raw_resource_stats  -> vals[G, 8]: cpu max, min, mean, median, memory max, min, mean, median (pandas' NaN
 *                               skipping group_max / group_min / Kahan group_mean / median, bit for bit)
 *   pert_raw_dedup           -> rows[n_kept] (the first of every set of equal rows, concatenation order) and their
 *                               timestamps keys[n_kept]                         => n_kept; the caller sorts keys stably
 *   pert_raw_process         -> sizes[7] = {M rows, n_ms ids, traceid, interface, entryid, rpcid, rpctype codes}
 *   pert_raw_emit            -> the nine processed columns [M], res_index[G, 2] = (timestamp, ms id) and the code
 *                               dictionaries of PertRawOut.
 * Codes count from 0 by first appearance in sorted order (Series.factorize); entryid / rpcid / rpctype over the rows of
 * traces with an entry, so later filters leave gaps as in the reference.  Microservice ids number the union of the
 * surviving um / dm and every resource msname in dictionary (lexicographic) order; the reference numbers that set in
 * Python set order, which is hash-randomised.  The duplicate table compares rows column by column before merging, so
 * a hash collision costs time and never a wrong merge; hash_bits (1..64) is 64 except in tests.  Outputs do not depend
 * on thread scheduling. */
typedef struct PertRawCalls {
  long long R;                                         /* rows, concatenation order                         */
  long long n_trace, n_iface, n_rpcid, n_rpctype, n_ms; /* dictionary sizes                                 */
  long long http, unknown;                             /* codes of rpctype "http" and microservice "(?)", -1: none */
  const int64_t *traceid, *timestamp, *rpcid, *um, *rpctype, *dm, *interface, *rt;
} PertRawCalls;
/* Outputs of pert_raw_emit, all int64, sized by pert_raw_process's sizes[] (and G). */
typedef struct PertRawOut {
  int64_t *traceid, *timestamp, *rpcid, *um, *dm, *interface, *rpctype, *rt, *entryid;   /* [M] processed rows   */
  int64_t *row;                                        /* [M] concatenation index of every processed row */
  int64_t *res_index;                                  /* [G, 2] (timestamp, ms id)                          */
  int64_t *ms_code;                                    /* [n_ms ids] dictionary code of every ms id          */
  int64_t *tr_code, *if_code, *rpc_code, *rty_code;    /* dictionary code of every traceid / interface / rpcid / rpctype id */
  int64_t *ent_dm, *ent_if;                            /* [entryid ids] the entry's dm code and interface id  */
} PertRawOut;
long long pert_raw_resource_workspace_bytes(long long K);
/* K resource rows ts / ms, perm[K] = row at sorted position, rows with an ms outside [0, n_ms) after all others (they
 * set PERT_ERR_RANGE and join no group); gflag[K+1], gptr[K+1], g_ts[K], g_ms[K] (group g: positions gptr[g] ..
 * gptr[g+1], key (g_ts, g_ms)), n_groups[1] = G; has_res[n_ms] = ms has a row. */
int pert_raw_resource_groups(long long K, const int64_t* ts, const int64_t* ms, const int64_t* perm, long long n_ms,
                             int* gflag, int* has_res, int* gptr, int64_t* g_ts, int64_t* g_ms, int64_t* n_groups,
                             void* workspace, long long workspace_bytes, int* status, void* stream);
/* cpu / mem [K] by row; cpu_sorted / mem_sorted [K]: every group's values ascending (NaN last) at its positions. */
int pert_raw_resource_stats(long long G, const int64_t* perm, const int* gptr, const double* cpu, const double* mem,
                            const double* cpu_sorted, const double* mem_sorted, double* vals, void* stream);
long long pert_raw_dedup_workspace_bytes(long long R);
int pert_raw_dedup(const PertRawCalls* calls, int hash_bits, int* rows, int64_t* keys, int64_t* n_kept,
                   void* workspace, long long workspace_bytes, int* status, void* stream);
/* workspace of pert_raw_process and pert_raw_emit (one buffer, passed to both); order[N] = row at sorted position */
long long pert_raw_process_workspace_bytes(const PertRawCalls* calls, long long N);
int pert_raw_process(const PertRawCalls* calls, long long N, const int64_t* order, const int* has_res,
                     long long min_occurence, int64_t* sizes, void* workspace, long long workspace_bytes,
                     void* stream);
int pert_raw_emit(const PertRawCalls* calls, long long N, const int64_t* order, long long G, const int64_t* g_ts,
                  const int64_t* g_ms, const PertRawOut* out, void* workspace, long long workspace_bytes,
                  void* stream);

/* ---- Raw chunks of a stream: ids that stay fixed from chunk to chunk (rawtable.RawStream) ------------------------
 * pert_raw_stream_process / pert_raw_stream_emit run pert_raw_process / pert_raw_emit over one chunk (its own
 * dictionaries, as PertRawCalls) and continue the stream described by PertRawState: every chunk dictionary code is read
 * through map[code] -> stream code (the host's dictionary of every value seen, one per coded column, microservices
 * shared), and a stream code with id[code] >= 0 keeps that id.  Only values without an id are flagged at their first
 * position, and get next + their rank (first sorted position; microservices: dictionary (name) order).  Traceid ids
 * continue n_tr (the caller refuses a chunk repeating a traceid).  Entries are keyed by (dm, interface) stream codes
 * (dm << 32 | interface) in an open-addressing table of ent_cap (a power of two >= 64) slots, ent_key ~0 = empty.
 * The coverage filter reads has_res of the chunk OR the stream's has_res; the occurrence filter keeps a chunk's covered
 * traces of entry e iff ent_cnt[e] + (this chunk's covered traces of e) > min_occurence.
 * sizes[7] are those of pert_raw_process with every id count counting NEW ids only.  The state is only read; emit
 * writes the new ids into PertRawStateOut, whose arrays the caller allocated fresh: ms_id / if_id / rpc_id / rty_id /
 * has_res / ent_cnt hold the old contents followed by -1 (ids) or 0 (has_res, ent_cnt) for stream codes / entries
 * the chunk adds; the entry table (ent_cap2 >= ent_cap, a power of two) is filled here, copied or rehashed from the
 * old one, and gets the new keys.  resource_ms[K]: the id of every raw resource row's microservice (-1: outside the
 * chunk dictionary).  The PertRawOut code arrays of new ids hold chunk codes; ent_if holds interface ids.
 * has_res (chunk, from pert_raw_resource_groups) is OR-ed with the stream's in place.  One workspace of
 * pert_raw_stream_workspace_bytes serves both calls. */
typedef struct PertRawState {
  const int64_t *ms_map, *if_map, *rpc_map, *rty_map;  /* [chunk dictionary] stream code of every chunk code     */
  const int64_t *ms_id, *if_id, *rpc_id, *rty_id;      /* [n_*_codes] id of every stream code, -1: none          */
  long long n_ms_codes, n_if_codes, n_rpc_codes, n_rty_codes;   /* lengths of the id arrays (and of has_res)   */
  const int* has_res;                                  /* [n_ms_codes] a resource row in some earlier chunk      */
  const unsigned long long* ent_key;                   /* [ent_cap] (dm << 32 | interface) stream codes, ~0 empty */
  const int64_t* ent_id;                               /* [ent_cap] entry id of every key                        */
  const int64_t* ent_cnt;                              /* [n_ent] covered traces of every entry so far            */
  long long ent_cap;
  long long n_tr, n_if, n_rpc, n_rty, n_ent, n_ms;     /* ids issued so far                                      */
} PertRawState;
typedef struct PertRawStateOut {
  int64_t *ms_id, *if_id, *rpc_id, *rty_id;            /* fresh id arrays (old ids, then -1), new ids written    */
  int* has_res;                                        /* fresh (old flags, then 0), this chunk's flags OR-ed in  */
  unsigned long long* ent_key;                         /* [ent_cap2] fresh entry table, filled here               */
  int64_t* ent_id;
  int64_t* ent_cnt;                                    /* [n_ent + new] old counts then 0; this chunk's added    */
  long long ent_cap2;
  int64_t* resource_ms;                                /* [K] ms id of every raw resource row, -1: left out      */
} PertRawStateOut;
long long pert_raw_stream_workspace_bytes(const PertRawCalls* calls, long long N);
int pert_raw_stream_process(const PertRawCalls* calls, long long N, const int64_t* order, int* has_res,
                            long long min_occurence, const PertRawState* state, int64_t* sizes, void* workspace,
                            long long workspace_bytes, void* stream);
int pert_raw_stream_emit(const PertRawCalls* calls, long long N, const int64_t* order, long long G,
                         const int64_t* g_ts, const int64_t* g_ms, long long K, const int64_t* r_ms,
                         const int* has_res, const PertRawState* state, const PertRawOut* out,
                         const PertRawStateOut* state_out, void* workspace, long long workspace_bytes, void* stream);

/* ---- the open-bucket sample window: raw resource samples -> running statistics (csrc/rawtable.cu) -------------------
 * Continues preprocess.py:237-242 (groupby(["timestamp", "msname"]).agg([max, min, mean, median])) sample batch by
 * sample batch: after any sequence of batches every open key's 8 statistics are bit for bit those
 * pert_raw_resource_stats gives for the concatenation of the key's samples in arrival order.  The window is caller
 * memory: keys[U] int64 (sorted unique ts * n_ms + ms), off[U+1] int32 run offsets (off[0] = 0, off[U] = S),
 * state[U] of 80 bytes (the cpu and the memory fold: max, min, Kahan sum, compensation as doubles and the non-NaN count
 * as int64) and cpu_run / mem_run [S] float64: each key's values ascending, NaN last (NaN equal to NaN, -0.0 == 0.0),
 * ties in arrival order.  A batch of k samples comes as bkeys[k] sorted stably (arrival order within a key), perm[k]
 * (sorted position -> input row of cpu / mem [k]) and cpu_sorted / mem_sorted [k]: every key's batch values ascending
 * in that order at the key's positions of bkeys.  Samples with floor(key / n_ms) < seal are late: a prefix of bkeys,
 * counted and skipped.  At most 2^31 - 16 keys, samples and batch samples.  The calls of one batch, in order:
 *   pert_raw_window_count -> flags[2(k+1)] (scanned first-of-key flags), sizes[3] = {late samples, keys the batch
 *                            touches u, keys after the merge U2}; the caller reads sizes and allocates the new window
 *   pert_raw_window_merge -> the new window (U2 keys, S + k - late samples), ustart[u+1] (first batch position of each
 *                            touched key, ustart[u] = k) and upos[u] (its slot in the new window), ascending by key
 *   pert_raw_window_emit  -> index[n, 2] (timestamp, ms) and vals[n, 8] (STATS order) of slot[0..n) (or slots 0..n-1
 *                            when slot is NULL).
 * One workspace of pert_raw_window_workspace_bytes(U, k, U2) serves both count and merge (U2 <= U + k bounds it).
 * Integer merge positions only: no atomics, every output written once, results independent of scheduling. */
long long pert_raw_window_workspace_bytes(long long U, long long k, long long U2);
int pert_raw_window_count(long long k, const int64_t* bkeys, long long n_ms, long long seal, long long U,
                          const int64_t* keys, int* flags, int64_t* sizes, void* workspace, long long workspace_bytes,
                          void* stream);
int pert_raw_window_merge(long long U, long long S, const int64_t* keys, const int* off, const void* state,
                          const double* cpu_run, const double* mem_run, long long k, const int64_t* bkeys,
                          const int64_t* perm, const double* cpu, const double* mem, const double* cpu_sorted,
                          const double* mem_sorted, const int* flags, long long n_late, long long u, long long U2,
                          int64_t* keys2, int* off2, void* state2, double* cpu_run2, double* mem_run2, int* ustart,
                          int* upos, void* workspace, long long workspace_bytes, void* stream);
int pert_raw_window_emit(long long n, const int* slot, long long U, const int64_t* keys, const int* off,
                         const void* state, const double* cpu_run, const double* mem_run, long long n_ms,
                         int64_t* index, double* vals, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PERTGNN_H_ */
