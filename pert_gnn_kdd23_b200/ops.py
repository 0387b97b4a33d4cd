"""torch.autograd.Function wrappers over the libpertgnn C-ABI (include/pertgnn.h).

Each Function allocates inputs/outputs/workspaces with torch and passes raw device
pointers + the current CUDA stream to the library; nothing here computes on the CPU
and nothing falls back to PyTorch kernels.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import call, ptr, stream

# launches issued through the C-ABI (bench.py reports it as `gpu_launches`)
LAUNCHES = {"n": 0}


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.PertGnnError("pert_gnn_kdd23_b200 ops need CUDA tensors: there is no CPU fallback")


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


def _pad_cols(t, width):
    """t [..., H] -> [..., width], columns H.. zero (t itself when H == width)."""
    return t if t is None or t.size(-1) == width else torch.nn.functional.pad(t, (0, width - t.size(-1)))


def _round4(H):
    """The embedding and BatchNorm kernels take rows of whole float4s: a width H % 4 != 0 runs zero-padded."""
    return (H + 3) // 4 * 4


def _kernel_width(H):
    """The attention and pool kernels run at the widths of pert_model_width: H runs zero-padded to the next one."""
    Hp = _lib.lib().pert_model_width(H)
    _lib.check(min(Hp, 0), f"pert_model_width({H})")
    return Hp


# ---------------------------------------------------------------------------------- GEMM
def _blocked(t):
    """tensor -> (ptr-holder, ld, cb, cbs, rows, cols): 2-D [M,K] or 3-D blocked [nb,M,cb] (logical [M,nb*cb])."""
    if t.dim() == 2:
        return t, t.stride(0), 0, 0, t.size(0), t.size(1)
    nb, M, cb = t.shape
    return t, t.stride(1), cb, t.stride(0), M, nb * cb


def gemm_nt_raw(A, B, bias, out, relu=False, accumulate=False):
    """out (=|+=) A . B^T (+bias)(relu);  A, out 2-D or 3-D blocked;  B [Nc,K]."""
    _, lda, a_cb, a_cbs, M, K = _blocked(A)
    _, ldc, c_cb, c_cbs, M2, Nc = _blocked(out)
    assert M == M2 and B.size(0) == Nc and B.size(1) == K, (A.shape, B.shape, out.shape)
    call("pert_gemm_nt", ptr(A), lda, a_cb, a_cbs, ptr(B), B.stride(0), ptr(bias), ptr(out), ldc, c_cb, c_cbs,
         M, Nc, K, int(relu), int(accumulate), stream())
    LAUNCHES["n"] += 1
    return out


def gemm_tn_raw(A, B, out):
    """out[Mc,Nc] += A[R,Mc]^T . B[R,Nc]  (A, B 2-D or blocked)."""
    _, lda, a_cb, a_cbs, R, Mc = _blocked(A)
    _, ldb, b_cb, b_cbs, R2, Nc = _blocked(B)
    assert R == R2 and out.shape == (Mc, Nc) and out.is_contiguous()
    call("pert_gemm_tn", ptr(A), lda, a_cb, a_cbs, ptr(B), ldb, b_cb, b_cbs, ptr(out), out.stride(0), None, R, Mc,
         Nc, stream())
    LAUNCHES["n"] += 1
    return out


def colsum_raw(A, out):
    _, lda, a_cb, a_cbs, R, Cc = _blocked(A)
    assert out.numel() == Cc
    call("pert_colsum", ptr(A), lda, a_cb, a_cbs, ptr(out), R, Cc, stream())
    LAUNCHES["n"] += 1
    return out


class _LinearFn(torch.autograd.Function):
    """y = x W^T + b (relu).  x: [M,K] or blocked [nb,M,cb]; y: [M,Nc] or blocked [out_blocks,M,Nc/out_blocks]."""

    @staticmethod
    @_lib.on_device_of
    def forward(ctx, x, weight, bias, relu, out_blocks):
        _need_cuda(x, weight, bias)
        x, weight = _c(x), _c(weight)
        bias = _c(bias) if bias is not None else None
        M = x.size(-2)
        Nc = weight.size(0)
        if out_blocks > 1:
            y = torch.empty(out_blocks, M, Nc // out_blocks, device=x.device, dtype=torch.float32)
        else:
            y = torch.empty(M, Nc, device=x.device, dtype=torch.float32)
        gemm_nt_raw(x, weight, bias, y, relu=relu)
        ctx.relu = relu
        ctx.out_blocks = out_blocks
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, weight, y if relu else None)
        return y

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dy):
        x, weight, y = ctx.saved_tensors
        dy = _c(dy)
        if ctx.relu:
            dy = dy.clone()
            call("pert_relu_bwd", ptr(y), ptr(dy), dy.numel(), stream())
            LAUNCHES["n"] += 1
        dx = dw = db = None
        M, K = x.size(-2), weight.size(1)
        if (ctx.out_blocks == 4 and not ctx.relu and ctx.has_bias and all(ctx.needs_input_grad[:3]) and x.dim() == 2
                and _lib.lib().pert_linear_bwd_planes_supported(M, weight.size(0) // 4, K, K)):
            # one pass over the four gradient planes for dX, dW and db (csrc/linear_bwd.cu)
            dx = torch.empty_like(x)
            dw = torch.zeros_like(weight)
            db = torch.zeros(weight.size(0), device=dy.device, dtype=torch.float32)
            wt = weight.t().contiguous()
            rc = _lib.lib().pert_linear_bwd_planes(ptr(dy), dy.stride(0), ptr(x), x.stride(0), ptr(wt), wt.stride(0),
                                                   ptr(dw), dw.stride(0), ptr(db), ptr(dx), dx.stride(0), M,
                                                   weight.size(0) // 4, K, K, stream())
            if rc == 0:
                LAUNCHES["n"] += 1
                return dx, dw, db, None, None
            if rc != -2:                                      # -2: nothing launched, the GEMM pair below does it
                _lib.check(rc, "pert_linear_bwd_planes")
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            wt = weight.t().contiguous()                      # [K,Nc]: B operand of dX = dY . W
            gemm_nt_raw(dy, wt, None, dx)
        if ctx.needs_input_grad[1]:
            dw = torch.zeros_like(weight)
            gemm_tn_raw(dy, x, dw)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = torch.zeros(weight.size(0), device=dy.device, dtype=torch.float32)
            colsum_raw(dy, db)
        return dx, dw, db, None, None


def linear(x, weight, bias=None, relu=False, out_blocks=1):
    return _LinearFn.apply(x, weight, bias, relu, out_blocks)


# ---------------------------------------------------------------------------------- embeddings
class _EmbeddingFn(torch.autograd.Function):
    @staticmethod
    @_lib.on_device_of
    def forward(ctx, table, ids, col):
        """table [R,H]; ids int64 [N] or [N,C] (column ``col``) -> [N,H]."""
        _need_cuda(table, ids)
        ids = _c(ids)
        stride = 1 if ids.dim() == 1 else ids.size(1)
        N = ids.size(0)
        H = table.size(1)
        table = _c(_pad_cols(table, _round4(H)))
        H4 = table.size(1)
        out = torch.empty(N, H4, device=table.device, dtype=torch.float32)
        base = ids.data_ptr() + 8 * col
        call("pert_embedding_fwd", ptr(table), table.size(0), base, stride, ptr(out), H4, N, H4, 0, None, stream())
        LAUNCHES["n"] += 1
        ctx.save_for_backward(ids)
        ctx.meta = (table.shape, col, stride, H)
        return out[:, :H] if H4 != H else out

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        shape, col, stride, H = ctx.meta
        dy = _c(_pad_cols(dy, shape[1]))
        dt = torch.zeros(shape, device=dy.device, dtype=torch.float32)
        call("pert_embedding_bwd", ptr(dy), dy.stride(0), ids.data_ptr() + 8 * col, stride, ptr(dt), shape[0],
             ids.size(0), shape[1], stream())
        LAUNCHES["n"] += 1
        return dt[:, :H] if shape[1] != H else dt, None, None


def embedding(table, ids, col=0):
    return _EmbeddingFn.apply(table, ids, col)


class _EmbedConcatFn(torch.autograd.Function):
    """X0 = [ sum_i table_i[cat_X[:, i]]  (H) | x (F) | 0-pad ]  -> [N, ld] with ld = round_up(H+F, 8).

    The reference concatenates [x | cat_embeds] (model.py:90); the internal column order is permuted so the
    embedding block is 16-byte aligned -- the first conv's weights are permuted to match (nn.py).  At H % 4 != 0 the
    sum is built in a [N, round4(H)] buffer from zero-padded tables and copied into the block."""

    @staticmethod
    @_lib.on_device_of
    def forward(ctx, x, cat_X, *tables):
        _need_cuda(x, cat_X, *tables)
        x, cat_X = _c(x), _c(cat_X)
        N, F = x.shape
        H = tables[0].size(1)
        H4 = _round4(H)
        ld = (H + F + 7) // 8 * 8
        out = torch.empty(N, ld, device=x.device, dtype=torch.float32)
        emb, ld_emb = (out, ld) if H4 == H else (torch.empty(N, H4, device=x.device, dtype=torch.float32), H4)
        ncat = cat_X.size(1)
        for i, t in enumerate(tables):
            t = _c(_pad_cols(t, H4))
            call("pert_embedding_fwd", ptr(t), t.size(0), cat_X.data_ptr() + 8 * i, ncat, ptr(emb), ld_emb, N, H4,
                 int(i > 0), None, stream())
        if H4 != H:
            out[:, :H].copy_(emb[:, :H])
        call("pert_copy_cols", ptr(x), F, ptr(out), ld, H, N, stream())
        LAUNCHES["n"] += len(tables) + 1
        ctx.save_for_backward(cat_X)
        ctx.meta = ([tuple(t.shape) for t in tables], F, H, ld)
        return out

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dout):
        (cat_X,) = ctx.saved_tensors
        shapes, F, H, ld = ctx.meta
        dout = _c(dout)
        N, ncat = cat_X.shape
        grads = []
        H4 = _round4(H)
        demb = dout if H4 == H else _c(_pad_cols(dout[:, :H], H4))
        for i, shp in enumerate(shapes):
            if ctx.needs_input_grad[2 + i]:
                dt = torch.zeros(shp[0], H4, device=dout.device, dtype=torch.float32)
                call("pert_embedding_bwd", ptr(demb), demb.stride(0), cat_X.data_ptr() + 8 * i, ncat, ptr(dt), shp[0], N,
                     H4, stream())
                LAUNCHES["n"] += 1
                grads.append(dt[:, :H] if H4 != H else dt)
            else:
                grads.append(None)
        dx = dout[:, H:H + F].contiguous() if ctx.needs_input_grad[0] else None
        return (dx, None, *grads)


def embed_concat(x, cat_X, tables):
    return _EmbedConcatFn.apply(x, cat_X, *tables)


# ---------------------------------------------------------------------------------- fused conv
class _TConvFn(torch.autograd.Function):
    """planes [4,N,H] (q,k,v,skip) or [3,N,H] (no skip), t_if [n_if,H], t_rpc [n_rpc,H] (or None) -> out [N,H].

    Any H up to 256: a width the attention kernels lack runs at Hp = pert_model_width(H) on zero-padded planes and
    tables, with the logits scaled by 1/sqrt(H) (pert_tconv_fwd_c); the output is the first H columns."""

    @staticmethod
    @_lib.on_device_of
    def forward(ctx, planes, t_if, t_rpc, index):
        _need_cuda(planes, t_if, t_rpc)
        C = planes.size(2)
        Hp = _kernel_width(C)
        planes = _c(_pad_cols(planes, Hp))
        P_, N, H = planes.shape
        assert index.N == N
        has_e = t_if is not None
        if has_e:
            t_if, t_rpc = _c(_pad_cols(t_if, Hp)), _c(_pad_cols(t_rpc, Hp))
            assert index.has_attr, "edge tables given but the index was built without edge_attr"
        out = torch.empty(N, H, device=planes.device, dtype=torch.float32)
        alpha = torch.empty(max(index.E, 1), device=planes.device, dtype=torch.float32)
        q, k, v = planes[0], planes[1], planes[2]
        s = planes[3] if P_ == 4 else None
        call("pert_tconv_fwd_c", ptr(q), ptr(k), ptr(v), ptr(s), H, ptr(index.rowptr), ptr(index.csr_src),
             ptr(index.csr_if) if has_e else None, ptr(index.csr_rpc) if has_e else None,
             ptr(t_if), ptr(t_rpc), ptr(out), H, ptr(alpha), t_rpc.size(0) if has_e else 0, N, index.E,
             getattr(index, "num_graphs", 0), H, C, stream())
        LAUNCHES["n"] += 1
        ctx.index = index
        ctx.has_e = has_e
        ctx.C = C
        ctx.save_for_backward(planes, t_if, t_rpc, alpha)
        return out[:, :C] if C != H else out

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, g):
        planes, t_if, t_rpc, alpha = ctx.saved_tensors
        index, C = ctx.index, ctx.C
        P_, N, H = planes.shape
        g = _c(_pad_cols(g, H))
        dplanes = torch.empty_like(planes)
        dsp = torch.empty_like(alpha)
        rpc_ws = torch.empty(16 * N, device=g.device, dtype=torch.float32) if ctx.has_e else None
        dt_if = dt_rpc = None
        if ctx.has_e:
            dt_if = torch.zeros_like(t_if)
            dt_rpc = torch.zeros_like(t_rpc)
        call("pert_tconv_bwd_c", ptr(g), g.stride(0), ptr(planes[0]), ptr(planes[1]), ptr(planes[2]), H,
             ptr(index.rowptr), ptr(index.csr_src), ptr(index.csr_if) if ctx.has_e else None,
             ptr(index.csr_rpc) if ctx.has_e else None, ptr(index.colptr), ptr(index.csc_pos),
             ptr(index.csc_dst), ptr(t_if), ptr(t_rpc), ptr(alpha), ptr(dplanes[0]), ptr(dplanes[1]),
             ptr(dplanes[2]), H, ptr(dsp), ptr(rpc_ws), ptr(dt_if), ptr(dt_rpc), t_rpc.size(0) if ctx.has_e else 0, N,
             index.E, getattr(index, "num_graphs", 0), H, C, stream())
        LAUNCHES["n"] += 2
        if P_ == 4:
            dplanes[3].copy_(g)
        if C != H:
            dplanes = dplanes[:, :, :C]
            dt_if, dt_rpc = (dt_if[:, :C], dt_rpc[:, :C]) if ctx.has_e else (None, None)
        return dplanes, dt_if, dt_rpc, None


def tconv(planes, t_if, t_rpc, index):
    return _TConvFn.apply(planes, t_if, t_rpc, index)


# ---------------------------------------------------------------------------------- batch norm (+relu)
class _BatchNormFn(torch.autograd.Function):
    @staticmethod
    @_lib.on_device_of
    def forward(ctx, x, gamma, beta, running_mean, running_var, nbt, training, eps, momentum, relu):
        _need_cuda(x, gamma, beta)
        H0 = x.size(1)
        H4 = _round4(H0)
        x, gamma, beta = _c(_pad_cols(x, H4)), _c(_pad_cols(gamma, H4)), _c(_pad_cols(beta, H4))
        rm, rv = running_mean, running_var
        if H4 != H0 and running_mean is not None:
            # padding columns: mean 0, variance 1 (finite rstd); their statistics are dropped again below
            rm, rv = _pad_cols(running_mean, H4), torch.nn.functional.pad(running_var, (0, H4 - H0), value=1.0)
        N, H = x.shape
        y = torch.empty_like(x)
        stats = torch.empty(2, H, device=x.device, dtype=torch.float32)
        wsb = _lib.lib().pert_bn_workspace_bytes(N, H)
        ws = torch.empty(wsb, device=x.device, dtype=torch.uint8)
        call("pert_bn_fwd", ptr(x), H, ptr(gamma), ptr(beta), ptr(rm), ptr(rv), ptr(nbt),
             float(eps), float(momentum), int(training), int(relu), ptr(stats[0]), ptr(stats[1]), ptr(y), H, N, H,
             ptr(ws), wsb, stream())
        LAUNCHES["n"] += 2
        if rm is not running_mean:
            running_mean.copy_(rm[:H0])
            running_var.copy_(rv[:H0])
        ctx.cfg = (bool(training), bool(relu), H0)
        ctx.save_for_backward(x, y, stats, gamma)
        return y[:, :H0] if H != H0 else y

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dy):
        x, y, stats, gamma = ctx.saved_tensors
        training, relu, H0 = ctx.cfg
        N, H = x.shape
        dy = _c(_pad_cols(dy, H))
        dx = torch.empty_like(x)
        # a scale / shift that is no parameter (BatchNorm1d(affine=False)) gets no gradient
        dgamma = torch.zeros(H, device=x.device, dtype=torch.float32) if ctx.needs_input_grad[1] else None
        dbeta = torch.zeros(H, device=x.device, dtype=torch.float32) if ctx.needs_input_grad[2] else None
        sums = torch.empty(2 * H, device=x.device, dtype=torch.float32)
        call("pert_bn_bwd", ptr(dy), dy.stride(0), ptr(y), H, ptr(x), H, ptr(stats[0]), ptr(stats[1]), ptr(gamma),
             int(relu), int(training), ptr(dx), H, ptr(dgamma), ptr(dbeta), ptr(sums), N, H, stream())
        LAUNCHES["n"] += 2
        if H != H0:
            dx = dx[:, :H0]
            dgamma = dgamma[:H0] if dgamma is not None else None
            dbeta = dbeta[:H0] if dbeta is not None else None
        return dx, dgamma, dbeta, None, None, None, None, None, None, None


def batch_norm(x, gamma, beta, running_mean, running_var, num_batches_tracked, training, eps=1e-5, momentum=0.1,
               relu=False):
    return _BatchNormFn.apply(x, gamma, beta, running_mean, running_var, num_batches_tracked, training, eps,
                              momentum, relu)


# ---------------------------------------------------------------------------------- local head + pool
class _PoolFn(torch.autograd.Function):
    @staticmethod
    @_lib.on_device_of
    def forward(ctx, x, probs, pnn, batch, w_local, b_local, num_graphs):
        _need_cuda(x, probs, pnn, batch)
        H0 = x.size(1)
        x = _c(_pad_cols(x, _kernel_width(H0)))
        w_pad = _c(_pad_cols(w_local, x.size(1))) if w_local is not None else None
        N, H = x.shape
        probs = _c(probs.reshape(-1).float())
        pnn = _c(pnn.reshape(-1).float())
        batch = _c(batch)
        B = int(num_graphs)
        pool = torch.empty(B, H, device=x.device, dtype=torch.float32)
        local = torch.empty(N, 1, device=x.device, dtype=torch.float32) if w_local is not None else None
        call("pert_pool_fwd", ptr(x), H, ptr(probs), ptr(pnn), ptr(batch), ptr(w_pad), ptr(b_local), ptr(local),
             ptr(pool), N, B, H, None, stream())
        LAUNCHES["n"] += 1
        ctx.B = B
        ctx.H0 = H0
        ctx.save_for_backward(x, probs, pnn, batch, w_pad)
        if local is None:
            local = torch.zeros(N, 1, device=x.device)
        return (pool[:, :H0] if H != H0 else pool), local

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dpool, dlocal):
        x, probs, pnn, batch, w_local = ctx.saved_tensors
        N, H = x.shape
        H0 = ctx.H0
        dx = torch.empty_like(x)
        has_local = w_local is not None and dlocal is not None
        dw = db = None
        if has_local:
            dlocal = _c(dlocal.reshape(-1))
            dw = torch.zeros_like(w_local)
            db = torch.zeros(1, device=x.device, dtype=torch.float32)
        dpool = _c(_pad_cols(dpool, H)) if dpool is not None else None
        call("pert_pool_bwd", ptr(dpool), ptr(dlocal) if has_local else None, ptr(x), H, ptr(probs), ptr(pnn),
             ptr(batch), ptr(_c(w_local)) if has_local else None, ptr(dx), H, ptr(dw), ptr(db), N, ctx.B, H,
             stream())
        LAUNCHES["n"] += 1
        if H != H0:
            dx, dw = dx[:, :H0], (dw[..., :H0] if dw is not None else None)
        return dx, None, None, None, dw, db, None


def pool_local(x, probs, pnn, batch, w_local, b_local, num_graphs):
    """-> (pool [B,H], local [N,1]) : local = x w^T + b ; pool = add-pool of (x*probs)/pnn  (model.py:105-107)."""
    return _PoolFn.apply(x, probs, pnn, batch, w_local, b_local, num_graphs)


# ---------------------------------------------------------------------------------- segmented reduce
class _SegReduceFn(torch.autograd.Function):
    @staticmethod
    @_lib.on_device_of
    def forward(ctx, msg, rowptr, perm, op):
        _need_cuda(msg, rowptr)
        msg = _c(msg)
        N = rowptr.numel() - 1
        H = msg.size(1) if msg.dim() == 2 else 1
        out = torch.empty((N, H) if msg.dim() == 2 else (N,), device=msg.device, dtype=torch.float32)
        call("pert_segment_reduce_fwd", ptr(msg), ptr(rowptr), ptr(perm), ptr(out), N, H, op, stream())
        LAUNCHES["n"] += 1
        ctx.op = op
        ctx.save_for_backward(msg, out, rowptr, perm)
        return out

    @staticmethod
    @_lib.on_device_of
    def backward(ctx, dout):
        msg, out, rowptr, perm = ctx.saved_tensors
        dout = _c(dout)
        N = rowptr.numel() - 1
        H = msg.size(1) if msg.dim() == 2 else 1
        dmsg = torch.zeros_like(msg)
        call("pert_segment_reduce_bwd", ptr(dout), ptr(msg), ptr(out), ptr(rowptr), ptr(perm), ptr(dmsg), N, H,
             ctx.op, stream())
        LAUNCHES["n"] += 1
        return dmsg, None, None, None


def segment_reduce(msg, rowptr, perm=None, reduce="max"):
    """out[i] = reduce over CSR segment i of msg rows (row of slot p = p, or perm[p]); empty segments -> 0."""
    return _SegReduceFn.apply(msg, rowptr, perm, {"sum": 0, "add": 0, "max": 1}[reduce])
