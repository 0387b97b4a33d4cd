"""ctypes binding of libpertgnn.so (the C-ABI declared in include/pertgnn.h).

There is NO fallback: if the shared library is missing or a call fails the
product path raises.  The library is built in-tree by ``__graft_entry__.build()``
(or ``make -C pert_gnn_kdd23_b200/csrc``).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpertgnn.so")

P, I, LL, F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
I32 = C.c_int32

# name -> (restype, argtypes); must mirror include/pertgnn.h
SIGNATURES = {
    "pert_version": (I, []),
    "pert_index_workspace_bytes": (LL, [LL, LL]),
    "pert_build_index": (I, [P, P, I, LL, LL, I, I, P, P, P, P, P, P, P, P, P, LL, P, P]),
    "pert_graph_ptr": (I, [P, LL, LL, P, P, LL, P, P]),
    "pert_min_depth": (I, [P, LL, P, P, P, P, P]),
    "pert_node_depth": (I, [P, LL, P, P, P]),
    "pert_level_order": (I, [P, LL, P, P, P]),
    "pert_segment_reduce_fwd": (I, [P, P, P, P, LL, I, I, P]),
    "pert_segment_reduce_bwd": (I, [P, P, P, P, P, P, LL, I, I, P]),
    "pert_tconv_supported_width": (I, [I]),
    "pert_tconv_fwd": (I, [P, P, P, P, I, P, P, P, P, P, P, P, I, P, I, LL, LL, LL, I, P]),
    "pert_tconv_bwd": (I, [P, I, P, P, P, I, P, P, P, P, P, P, P, P, P, P, P, P, P, I, P, P, P, P, I, LL, LL, LL, I,
                           P]),
    "pert_tconv_fwd_c": (I, [P, P, P, P, I, P, P, P, P, P, P, P, I, P, I, LL, LL, LL, I, I, P]),
    "pert_tconv_bwd_c": (I, [P, I, P, P, P, I, P, P, P, P, P, P, P, P, P, P, P, P, P, I, P, P, P, P, I, LL, LL, LL, I,
                             I, P]),
    "pert_tconv_fwd_stats": (I, [P, P, P, P, I, P, P, P, P, P, P, P, I, P, I, LL, LL, LL, I, I, P, P, P, P]),
    "pert_tconv_bwd_bn": (I, [P, I, P, P, P, I, P, P, P, P, P, P, P, P, P, P, P, P, P, I, P, P, P, P, I, LL, LL, LL, I,
                              I, P, P]),
    "pert_tconv_bwd_bn_supported": (I, [I, I]),
    "pert_gemm_nt": (I, [P, I, I, LL, P, I, P, P, I, I, LL, LL, I, I, I, I, P]),
    "pert_gemm_tn": (I, [P, I, I, LL, P, I, I, LL, P, I, P, LL, I, I, P]),
    "pert_colsum": (I, [P, I, I, LL, P, LL, I, P]),
    "pert_linear_bwd_planes": (I, [P, LL, P, I, P, I, P, I, P, P, I, LL, I, I, I, P]),
    "pert_linear_bwd_planes_supported": (I, [LL, I, I, I]),
    "pert_linear_bwd_planes_ex": (I, [P, LL, P, I, P, I, P, I, P, P, I, LL, I, I, I, P, P, P, F, P, P, P]),
    "pert_bn_linear_fwd_planes": (I, [P, I, I, P, P, P, P, P, F, F, I, P, P, P, I, P, LL, I, F, P, I, P, I, P, P, LL,
                                      LL, I, I, P]),
    "pert_bn_linear_fwd_planes_supported": (I, [LL, I, I]),
    "pert_embedding_fwd": (I, [P, I, P, I, P, I, LL, I, I, P, P]),
    "pert_embedding_bwd": (I, [P, I, P, I, P, I, LL, I, P]),
    "pert_copy_cols": (I, [P, I, P, I, I, LL, P]),
    "pert_bn_workspace_bytes": (LL, [LL, I]),
    "pert_bn_fwd": (I, [P, I, P, P, P, P, P, F, F, I, I, P, P, P, I, LL, I, P, LL, P]),
    "pert_bn_bwd": (I, [P, I, P, I, P, I, P, P, P, I, I, P, I, P, P, P, LL, I, P]),
    "pert_pool_fwd": (I, [P, I, P, P, P, P, P, P, P, LL, LL, I, P, P]),
    "pert_pool_bwd": (I, [P, P, P, I, P, P, P, P, P, I, P, P, LL, LL, I, P]),
    "pert_relu_bwd": (I, [P, P, LL, P]),
    "pert_pinball_loss": (I, [P, P, F, LL, F, P, P, P]),
    "pert_eval_metrics": (I, [P, P, F, LL, P, P]),
    "pert_pinball_loss_live": (I, [P, P, F, LL, F, P, P, P, P]),
    "pert_eval_metrics_live": (I, [P, P, F, LL, P, P, P]),
    "pert_adam_step": (I, [P, P, P, P, LL, F, F, F, F, F, LL, F, P]),
    # relayout of the flat parameter / Adam buffers when parameters grow (csrc/flat.cu; first argument: host table)
    "pert_flat_grow": (I, [P, I, LL, LL, P, P, P, P, P, P, P, P]),
    # fused all-reduce + Adam over peer memory (csrc/peer.cu)
    "pert_peer_exchange_bytes": (LL, [LL]),
    "pert_peer_alloc": (I, [LL, P, P]),
    "pert_peer_open": (I, [P, P]),
    "pert_peer_close": (I, [P]),
    "pert_peer_free": (I, [P]),
    "pert_allreduce_adam": (I, [P, P, P, P, LL, F, F, F, F, F, LL, F, P, I, I, P, P, P]),
    # device-side batch assembly from the pattern store (first / 7th argument: struct pointers, see store.py)
    "pert_store_assemble": (I, [P, P, LL, LL, LL, P, P, P, P]),
    # request assembly (second argument: const PertResourceAsOf* or NULL for the exact join)
    "pert_store_assemble_requests": (I, [P, P, P, P, LL, LL, LL, P, P, P, P]),
    # what-if request assembly (third argument: const PertWhatIf*) and the joined resource rows of (timestamp, ms)
    "pert_store_assemble_whatif": (I, [P, P, P, P, P, LL, LL, LL, P, P, P, P]),
    "pert_store_lookup_resources": (I, [P, P, P, P, LL, P, P, P]),
    # resource updates of a live store (csrc/resources.cu; first two arguments: PertStore*, PertResourceAsOf*)
    "pert_store_resources_count": (I, [P, P, P, P, LL, LL, P, P, P, P]),
    "pert_store_resources_merge": (I, [P, P, P, P, P, P, LL, P, P, LL, LL, LL, P, P, P, P, P, P]),
    "pert_store_resources_update_count": (I, [P, P, P, P, LL, P, P, LL, LL, P, P, P, P, P]),
    "pert_store_resources_update_merge": (I, [P, P, P, P, P, LL, P, P, P, P, LL, P, P, LL, LL, LL, LL, P, P, P, P, P,
                                              P]),
    # trace ingest of a live store (csrc/ingest.cu; struct pointers, see store.py)
    "pert_ingest_table_insert": (I, [P, LL, P, P]),
    "pert_ingest_match_workspace_bytes": (LL, [LL]),
    "pert_ingest_match": (I, [P, P, P, P, P, P, P, P, P, LL, P]),
    "pert_ingest_merge_workspace_bytes": (LL, [LL, LL, LL]),
    "pert_ingest_merge": (I, [P, P, P, LL, P, P, P, LL, P, P, LL, P]),
    "pert_ingest_evict_workspace_bytes": (LL, [LL, LL, LL, LL]),
    "pert_ingest_evict_count": (I, [P, P, LL, P, LL, P, P]),
    "pert_ingest_evict_apply": (I, [P, P, P, P, LL, P, P]),
    # PERT-graph construction (pertgraph.py)
    "pert_pert_graph_count": (I, [P, LL, P, P, I, P, P, P]),
    "pert_pert_graph_build": (I, [P, LL, LL, P, P, P, P, P, P, P, P, I, I, P, P, P, P, P, P]),
    "pert_span_graph_count": (I, [P, LL, P, P, I, P, P, P]),
    "pert_span_graph_build": (I, [P, LL, LL, P, P, P, P, P, P, I, I, P, P, P, P, P, P]),
    # trace grouping (tracegroup.py; first argument: const PertSpanTable*)
    "pert_trace_group_range": (I, [P, P, P, P]),
    "pert_trace_group_keys": (I, [P, LL, P, P, P, LL, P]),
    "pert_trace_group_workspace_bytes": (LL, [LL, LL, LL, LL]),
    "pert_trace_group_build": (I, [P, LL, LL, LL, I, P, P, P, P, LL, P, P]),
    "pert_trace_group_gather": (I, [P, P, P, P, P, LL, LL, P, P]),
    # processed tables from raw rows (rawtable.py; PertRawCalls* / PertRawOut* arguments)
    "pert_raw_resource_workspace_bytes": (LL, [LL]),
    "pert_raw_resource_groups": (I, [LL, P, P, P, LL, P, P, P, P, P, P, P, LL, P, P]),
    "pert_raw_resource_stats": (I, [LL, P, P, P, P, P, P, P, P]),
    "pert_raw_dedup_workspace_bytes": (LL, [LL]),
    "pert_raw_dedup": (I, [P, I, P, P, P, P, LL, P, P]),
    "pert_raw_process_workspace_bytes": (LL, [P, LL]),
    "pert_raw_process": (I, [P, LL, P, P, LL, P, P, LL, P]),
    "pert_raw_emit": (I, [P, LL, P, LL, P, P, P, P, LL, P]),
    "pert_raw_stream_workspace_bytes": (LL, [P, LL]),
    "pert_raw_stream_process": (I, [P, LL, P, P, LL, P, P, P, LL, P]),
    "pert_raw_stream_emit": (I, [P, LL, P, LL, P, P, LL, P, P, P, P, P, P, LL, P]),
    # the open-bucket sample window (rawtable.ResourceSampleWindow)
    "pert_raw_window_workspace_bytes": (LL, [LL, LL, LL]),
    "pert_raw_window_count": (I, [LL, P, LL, LL, LL, P, P, P, P, LL, P]),
    "pert_raw_window_merge": (I, [LL, LL, P, P, P, P, P, LL, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, P, P, P,
                                  LL, P]),
    "pert_raw_window_emit": (I, [LL, P, LL, P, P, P, P, P, LL, P, P, P]),
    # whole-model engine (first argument: const PertModelDesc*, see engine.py)
    "pert_model_width": (I, [I]),
    "pert_model_workspace_bytes": (LL, [P, LL, LL, LL]),
    "pert_model_packed_bytes": (LL, [P]),
    "pert_model_workspace_offset": (LL, [P, LL, LL, LL, I, I]),
    "pert_model_forward": (I, [P, P, P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, LL, I, F, P, P, P, P, P, P,
                               P]),
    "pert_model_backward": (I, [P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, P, P, P, LL, I, F, P, P, P, P]),
    # padded batches for per-bucket graph replay (csrc/pad.cu; the *_live entries read the {N, B} word it writes)
    "pert_model_forward_live": (I, [P, P, P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, LL, I, F, P, P, P, P, P,
                                    P, P, P]),
    "pert_model_backward_live": (I, [P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, P, P, P, LL, I, F, P, P, P,
                                     P, P]),
    "pert_batch_pad": (I, [P, P, P, P, P, P, P, P, P, LL, LL, LL, I, I, I, P, P, P, P, P, P, P, P, P, LL, LL, LL, P,
                           P]),
    # a global head with n_out quantile outputs (int n_out after the descriptor; the _live argument lists)
    "pert_model_workspace_bytes_q": (LL, [P, I, LL, LL, LL]),
    "pert_model_packed_bytes_q": (LL, [P, I]),
    "pert_model_workspace_offset_q": (LL, [P, I, LL, LL, LL, I, I]),
    "pert_model_forward_q": (I, [P, I, P, P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, LL, I, F, P, P, P, P, P,
                                 P, P, P]),
    "pert_model_backward_q": (I, [P, I, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P, P, P, P, P, LL, I, F, P, P, P,
                                  P, P]),
    "pert_pinball_loss_q": (I, [P, P, P, I, LL, F, P, P, P, P]),
    "pert_eval_metrics_q": (I, [P, P, P, I, LL, P, P, P]),
    # conformal calibration of the quantile levels (csrc/calib.cu; taus: host array of doubles)
    "pert_calib_workspace_bytes": (LL, [LL, I, LL]),
    "pert_calib_offsets": (I, [P, P, P, LL, I, P, LL, LL, P, P, P, P, LL, P, P]),
    "pert_calib_apply": (I, [P, P, LL, I, P, LL, I, P, P]),
    # the conformal predictive distribution (csrc/cpd.cu; taus: host array of doubles)
    "pert_cpd_workspace_bytes": (LL, [LL, LL]),
    "pert_cpd_fit": (I, [P, P, LL, I, P, LL, LL, P, P, P, LL, P, P]),
    "pert_cpd_tail": (I, [P, P, LL, LL, P, LL, I, P, LL, P, I, P, P, P, P, P, P]),
    "pert_cpd_quantile": (I, [P, P, LL, LL, P, LL, I, P, LL, P, I, P, P, P]),
    "pert_cpd_merge_workspace_bytes": (LL, [LL, LL, LL, LL]),
    "pert_cpd_merge": (I, [P, P, LL, LL, P, P, LL, LL, I, P, P, P, LL, P, P]),
}
MAX_QUANTILES = 8                                       # PERT_MAX_QUANTILES

_lib = None


class PertGnnError(RuntimeError):
    pass


# ---- the structs of include/pertgnn.h, field for field, checked against the header by tests/test_abi_structs.py; the
# header documents every field
MAX_CONVS, MAX_CAT = 8, 4                               # PERT_MAX_CONVS, PERT_MAX_CAT
FLAT_ALIGN, FLAT_MAX_SEGS = 64, 128                      # PERT_FLAT_ALIGN, PERT_FLAT_MAX_SEGS


class PertModelDesc(C.Structure):
    _fields_ = [
        ("F", I32), ("H", I32), ("n_convs", I32), ("n_cat", I32), ("cat_rows", I32 * MAX_CAT), ("n_entry", I32),
        ("n_if", I32), ("n_rpc", I32), ("k0", I32), ("bn_eps", F), ("bn_momentum", F),
        ("off_cat", LL * MAX_CAT), ("off_entry", LL), ("off_if", LL), ("off_rpc", LL),
        ("off_wq", LL * MAX_CONVS), ("off_bq", LL * MAX_CONVS), ("off_wk", LL * MAX_CONVS), ("off_bk", LL * MAX_CONVS),
        ("off_wv", LL * MAX_CONVS), ("off_bv", LL * MAX_CONVS), ("off_ws", LL * MAX_CONVS), ("off_bs", LL * MAX_CONVS),
        ("off_we", LL * MAX_CONVS), ("off_bn_g", LL * MAX_CONVS), ("off_bn_b", LL * MAX_CONVS),
        ("off_local_w", LL), ("off_local_b", LL), ("off_g1_w", LL), ("off_g1_b", LL), ("off_g2_w", LL),
        ("off_g2_b", LL),
    ]


class PertProbe(C.Structure):
    _fields_ = [("kernel", I32), ("layer", I32), ("ev_start", P), ("ev_stop", P)]


class PertBnBwd(C.Structure):
    _fields_ = [(k, P) for k in ("dx", "y", "x", "mean", "rstd", "gamma", "sums", "dgamma", "dbeta", "live")] + \
        [("relu_scale", F)]


class PertStore(C.Structure):
    _fields_ = [("n_pat", I32), ("n_ent", I32), ("n_res", I32), ("n_ms", I32), ("attr_cols", I32), ("n_traces", LL)] + \
        [(k, P) for k in ("pat_nptr", "pat_eptr", "pat_ms", "pat_depth", "pat_last", "pat_src", "pat_dst", "pat_attr",
                          "ent_ptr", "ent_pat", "ent_prob", "ent_nodes", "ent_edges", "res_keys", "res_vals",
                          "ms_has_res", "trace_entry", "trace_ts", "trace_y")]


class PertBatchOut(C.Structure):
    _fields_ = [(k, P) for k in ("x", "cat_X", "node_depth", "pattern_num_nodes", "rt_probs", "batch", "edge_index",
                                 "edge_attr", "entry_id", "y", "ptr", "pattern_probs")]


class PertResourceAsOf(C.Structure):
    """The as-of index of a store's resource rows: device pointers ms_ptr [n_ms+1] int32, ts [n_res] int64, row [n_res]
    int32."""
    _fields_ = [("ms_ptr", P), ("ts", P), ("row", P)]


class PertWhatIf(C.Structure):
    """Per-request mixes and resource overrides of what-if assembly: device pointers mix_ptr [B+1] int64 (absolute
    offsets) into mix_pat int32 / mix_prob float32, scenario [B] int64, and n_ov override rows, ov_keys [n_ov] int64
    sorted and ov_vals [n_ov, 8] float32 (16-byte aligned); NULL mix_ptr / scenario: none."""
    _fields_ = [("mix_ptr", P), ("mix_pat", P), ("mix_prob", P), ("scenario", P), ("n_ov", LL), ("ov_keys", P),
                ("ov_vals", P)]


class PertRuntimeKeys(C.Structure):
    _fields_ = [("n", LL), ("ld", LL), ("ptr", P), ("rows", P)]


class PertRuntimeTable(C.Structure):
    _fields_ = [("S", LL), ("hash_bits", I32), ("slot", P), ("h1", P), ("h2", P)]


class PertChunkMix(C.Structure):
    _fields_ = [("n_ent", LL), ("n_pairs", LL)] + [(k, P) for k in ("ent_pair_ptr", "ent_trace_ptr", "pair_runtime",
                                                                   "pair_prob", "runtime_ins", "pat_of")]


class PertMixOut(C.Structure):
    _fields_ = [(k, P) for k in ("ent_ptr", "ent_pat", "ent_prob", "cnt", "ent_nodes", "ent_edges", "tot")]


class PertIngestState(C.Structure):
    _fields_ = [("keys", PertRuntimeKeys)] + [(k, P) for k in ("trace_pat", "trace_tid", "cnt", "tot")] + \
        [(k, LL) for k in ("n_pairs", "n_nodes", "n_edges", "n_key_rows")]


EVICT_ARRAYS = ("remap", "trace_entry", "trace_ts", "trace_y", "trace_pat", "trace_tid", "pat_new", "pat_nptr",
                "pat_eptr", "pat_ms", "pat_depth", "pat_last", "pat_src", "pat_dst", "pat_attr", "key_ptr", "key_rows")


class PertEvictOut(C.Structure):
    _fields_ = [("mix", PertMixOut)] + [(k, P) for k in EVICT_ARRAYS] + [("key_ld", LL)]


class PertSpanTable(C.Structure):
    _fields_ = [("R", LL)] + [(k, P) for k in ("traceid", "timestamp", "rpcid", "um", "dm", "interface", "rpctype",
                                               "rt", "entryid")]


class PertTraceGroups(C.Structure):
    _fields_ = [(k, P) for k in ("row_ptr", "perm", "trace_id", "bucket", "y", "entry", "runtime", "order",
                                 "ent_trace_ptr", "ent_pair_ptr", "pair_runtime", "pair_prob", "occurrences",
                                 "ins_runtime", "rep_trace", "runtime_ins", "rep_ptr", "sizes")]


class PertRawCalls(C.Structure):
    _fields_ = [(k, LL) for k in ("R", "n_trace", "n_iface", "n_rpcid", "n_rpctype", "n_ms", "http", "unknown")] + \
        [(k, P) for k in ("traceid", "timestamp", "rpcid", "um", "rpctype", "dm", "interface", "rt")]


RAW_OUT = ("traceid", "timestamp", "rpcid", "um", "dm", "interface", "rpctype", "rt", "entryid", "row", "res_index",
           "ms_code", "tr_code", "if_code", "rpc_code", "rty_code", "ent_dm", "ent_if")


class PertRawOut(C.Structure):
    _fields_ = [(k, P) for k in RAW_OUT]


class PertRawState(C.Structure):
    _fields_ = [(k, P) for k in ("ms_map", "if_map", "rpc_map", "rty_map", "ms_id", "if_id", "rpc_id", "rty_id")] + \
        [(k, LL) for k in ("n_ms_codes", "n_if_codes", "n_rpc_codes", "n_rty_codes")] + \
        [(k, P) for k in ("has_res", "ent_key", "ent_id", "ent_cnt")] + \
        [(k, LL) for k in ("ent_cap", "n_tr", "n_if", "n_rpc", "n_rty", "n_ent", "n_ms")]


class PertRawStateOut(C.Structure):
    _fields_ = [(k, P) for k in ("ms_id", "if_id", "rpc_id", "rty_id", "has_res", "ent_key", "ent_id", "ent_cnt")] + \
        [("ent_cap2", LL), ("resource_ms", P)]


def lib():
    """Load (once) and return the ctypes handle; raises if the CUDA library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PertGnnError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the hot path)")
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        if rc > 0:
            raise PertGnnError(f"{what}: CUDA error {rc}")
        names = {-1: "bad argument", -2: "unsupported width/mode", -3: "index out of range",
                 -4: "a data-parallel peer never arrived (timeout)"}
        raise PertGnnError(f"{what}: {names.get(rc, rc)}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def on_device_of(fn):
    """Decorator: run ``fn`` with the CUDA device of its first CUDA-tensor argument current.  The C library launches
    on the current device and ``stream()`` returns that device's current stream, so every binding that takes tensors
    must pin the device (reference loop: ``--device N`` + ``model.to(f'cuda:{N}')`` never calls ``set_device``)."""
    import functools

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        dev = None
        for a in args:
            if torch.is_tensor(a) and a.is_cuda:
                dev = a.device
                break
            d = getattr(a, "device", None)             # objects that carry a device (Engine, GraphIndex, FlatParams)
            if isinstance(d, torch.device) and d.type == "cuda":
                dev = d
                break
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)

    return wrapped


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    check(rc, name)
