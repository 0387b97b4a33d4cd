"""Python side of the whole-model step engine (csrc/engine.cu): builds the ``PertModelDesc`` from a
``SAGEDeterministic`` module, owns the workspace, and exposes
  * ``Engine.forward`` / ``Engine.backward``  -- raw calls (no autograd), used by the fused train step;
  * ``engine_forward``                        -- a single autograd.Function for ``model.forward`` (drop-in path).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, ops
from ._lib import MAX_CAT, MAX_CONVS, PertModelDesc
from .index import GraphIndex


def _bind():
    return _lib.lib()


class PertProbe(_lib.PertProbe):
    """Measurement probe (include/pertgnn.h): two CUDA events recorded around one kernel family of one layer."""

    KERNELS = {"tconv_fwd": 1, "tconv_bwd": 2, "gemm_fwd": 3, "gemm_wgrad": 4, "gemm_dgrad": 5}
    _rt = None

    @classmethod
    def _cudart(cls):
        if cls._rt is None:
            import glob
            import os

            cands = glob.glob(os.path.join(os.path.dirname(torch.__file__), "lib", "libcudart*.so*")) + \
                glob.glob("/usr/local/cuda/lib64/libcudart.so*")
            if not cands:
                import nvidia.cuda_runtime as _n   # pip layout

                cands = glob.glob(os.path.join(os.path.dirname(_n.__file__), "lib", "libcudart.so*"))
            cls._rt = C.CDLL(sorted(cands)[0])
            cls._rt.cudaEventCreate.argtypes = [C.POINTER(C.c_void_p)]
            cls._rt.cudaEventElapsedTime.argtypes = [C.POINTER(C.c_float), C.c_void_p, C.c_void_p]
            cls._rt.cudaEventDestroy.argtypes = [C.c_void_p]
        return cls._rt

    @classmethod
    def create(cls, kernel, layer):
        rt = cls._cudart()
        a, b = C.c_void_p(), C.c_void_p()
        assert rt.cudaEventCreate(C.byref(a)) == 0 and rt.cudaEventCreate(C.byref(b)) == 0
        return cls(cls.KERNELS[kernel], layer, a, b)

    def elapsed_ms(self):
        ms = C.c_float()
        rc = self._cudart().cudaEventElapsedTime(C.byref(ms), self.ev_start, self.ev_stop)
        return ms.value if rc == 0 else float("nan")

    def destroy(self):
        rt = self._cudart()
        rt.cudaEventDestroy(self.ev_start)
        rt.cudaEventDestroy(self.ev_stop)


class Engine:
    """Owns flat parameters / gradients / BN buffers of one model replica and the engine workspace."""

    # launches per call (for the gpu_launches accounting of bench.py)
    def __init__(self, model, flat=None):
        from .train import FlatParams

        self.model = model
        self.fp = flat if flat is not None else FlatParams(model)
        self.lib = _bind()
        dev = self.fp.flat.device
        H = model.hidden_channels
        # the engine runs the width-H model at the kernel width Hp >= H, columns [H, Hp) zero (include/pertgnn.h)
        Hp = self.lib.pert_model_width(H)
        _lib.check(min(Hp, 0), f"pert_model_width({H})")
        self.Hp = Hp
        n_convs = len(model.convs)
        assert n_convs <= MAX_CONVS and len(model.cat_embedding) <= MAX_CAT
        # BN running statistics as one flat buffer [n_bn, 2, Hp]; the module buffers become views of its first H columns
        # (the padding columns start at mean 0, variance 1 and never reach an output)
        n_bn = n_convs - 1
        self.bn_running = torch.zeros(n_bn, 2, Hp, device=dev, dtype=torch.float32)
        self.bn_running[:, 1] = 1.0
        self.bn_nbt = torch.zeros(n_bn, device=dev, dtype=torch.int64)
        for l, bn in enumerate(model.bns):
            self.bn_running[l, 0, :H].copy_(bn.running_mean)
            self.bn_running[l, 1, :H].copy_(bn.running_var)
            self.bn_nbt[l] = bn.num_batches_tracked
            bn._buffers["running_mean"] = self.bn_running[l, 0, :H]
            bn._buffers["running_var"] = self.bn_running[l, 1, :H]
            bn._buffers["num_batches_tracked"] = self.bn_nbt[l]
        d = PertModelDesc()
        d.F, d.H, d.n_convs, d.n_cat = model.in_channels, H, n_convs, len(model.cat_embedding)
        d.n_entry = model.entry_embeds.num_embeddings
        d.n_if = model.interface_embeds.num_embeddings
        d.n_rpc = model.rpctype_embeds.num_embeddings
        d.k0 = (model.in_channels + Hp + 7) // 8 * 8
        d.bn_eps = model.bns[0].eps
        d.bn_momentum = model.bns[0].momentum if model.bns[0].momentum is not None else 0.0
        base = self.fp.flat.data_ptr()

        def off(p):
            o = p.data_ptr() - base
            assert o % 16 == 0 and 0 <= o < self.fp.flat.numel() * 4, "parameter is not an aligned view of the flat buffer"
            return o // 4

        for i, e in enumerate(model.cat_embedding):
            d.cat_rows[i] = e.num_embeddings
            d.off_cat[i] = off(e.weight)
        d.off_entry, d.off_if, d.off_rpc = off(model.entry_embeds.weight), off(model.interface_embeds.weight), \
            off(model.rpctype_embeds.weight)
        for l, c in enumerate(model.convs):
            d.off_wq[l], d.off_bq[l] = off(c.lin_query.weight), off(c.lin_query.bias)
            d.off_wk[l], d.off_bk[l] = off(c.lin_key.weight), off(c.lin_key.bias)
            d.off_wv[l], d.off_bv[l] = off(c.lin_value.weight), off(c.lin_value.bias)
            d.off_ws[l], d.off_bs[l] = off(c.lin_skip.weight), off(c.lin_skip.bias)
            d.off_we[l] = off(c.lin_edge.weight)
        for l, bn in enumerate(model.bns):
            d.off_bn_g[l], d.off_bn_b[l] = off(bn.weight), off(bn.bias)
        d.off_local_w, d.off_local_b = off(model.local_linear.weight), off(model.local_linear.bias)
        d.off_g1_w, d.off_g1_b = off(model.global_linear1.weight), off(model.global_linear1.bias)
        d.off_g2_w, d.off_g2_b = off(model.global_linear2.weight), off(model.global_linear2.bias)
        self.desc = d
        # outputs of the global head (quantile levels); a one-output head calls the plain entry points
        self.n_out = int(model.global_linear2.weight.size(0))
        self.n_convs = n_convs
        self.ws = None
        self.ws_key = (0, 0, 0)
        self.ws_generation = 0
        self._saved = None

    # ------------------------------------------------------------------------------------------
    @property
    def device(self):
        return self.fp.flat.device

    def reserve(self, N, E, B):
        """Pre-size the workspace (growth only).  ``ws_generation`` changes whenever the buffer is re-allocated: a CUDA
        graph captured over the old buffer must not be replayed any more (train._GraphCache checks it, and calls this
        before every capture so that no capture allocates the workspace)."""
        return self._workspace(int(N), int(E), int(B))

    def _workspace(self, N, E, B):
        if self.ws is None or N > self.ws_key[0] or E > self.ws_key[1] or B > self.ws_key[2]:
            key = (max(N, self.ws_key[0]), max(E, self.ws_key[1]), max(B, self.ws_key[2]))
            if self.n_out == 1:
                nbytes = self.lib.pert_model_workspace_bytes(C.byref(self.desc), *key)
            else:
                nbytes = self.lib.pert_model_workspace_bytes_q(C.byref(self.desc), self.n_out, *key)
            if nbytes < 0:
                _lib.check(int(nbytes), "pert_model_workspace_bytes")
            with torch.cuda.device(self.fp.flat.device):
                self.ws = torch.zeros(nbytes // 4, device=self.fp.flat.device, dtype=torch.float32)
            self.ws_key = key
            self.ws_generation += 1
        return self.ws

    def workspace_offset(self, which, layer, N, E, B):
        """pert_model_workspace_offset(_q) of this engine's head: where an intermediate lives in ``ws`` (floats)."""
        if self.n_out == 1:
            off = self.lib.pert_model_workspace_offset(C.byref(self.desc), N, E, B, which, layer)
        else:
            off = self.lib.pert_model_workspace_offset_q(C.byref(self.desc), self.n_out, N, E, B, which, layer)
        _lib.check(int(min(off, 0)), "pert_model_workspace_offset")
        return off

    def active_relus(self):
        """{'bn{i}': [N,H] bool, 'head': [B,H] bool}: the entries > 0 of the saved activations of the LAST forward,
        i.e. which ReLUs were active -- with dropout, active AND kept.  Test aid: lets a reference be differentiated on
        the same linear piece."""
        x, cat_X, entry_id, probs, pnn, batch, index, training, N, E, B, p = self._saved
        H, Hp = self.desc.H, self.Hp
        out = {}
        for l in range(1, self.n_convs):
            off = self.workspace_offset(0, l, N, E, B)
            out[f"bn{l - 1}"] = self.ws[off:off + N * Hp].view(N, Hp)[:, :H] > 0
        off = self.workspace_offset(1, 0, N, E, B)
        out["head"] = self.ws[off:off + B * Hp].view(B, Hp)[:, :H] > 0
        return out

    def _pack_launches(self):
        # mirrors engine.cu: conv 0 contributes 24 segments, the others 16; a launch holds at most 96.  A padded width
        # (Hp > H) adds one launch for the zero-padded copies of the other tensors.
        n, count = int(self.Hp != self.desc.H), 0
        for l in range(self.n_convs):
            count += 24 if l == 0 else 16
            if count + 24 > 96 or l == self.n_convs - 1:
                n, count = n + 1, 0
        return n

    def launches_forward(self):
        """Kernels pert_model_forward launches (memsets not counted): pack, edge tables (6 layers per launch),
        embeddings + copy, per conv GEMM + attention (whose epilogue also produces the BatchNorm statistics), per
        BatchNorm one apply kernel unless pert_bn_linear_fwd_planes takes the shape (the next conv's GEMM then applies
        it), pool, head."""
        L, H, N = self.n_convs, self.Hp, self._saved[8]
        applies = 0 if self.lib.pert_bn_linear_fwd_planes_supported(N, H, H) else L - 1
        return self._pack_launches() + (L + 5) // 6 + self.desc.n_cat + 1 + 2 * L + applies + 1 + 1

    def launches_backward(self):
        """head, pool, per conv (target pass, source pass, node-linear backward: one fused launch where
        pert_linear_bwd_planes takes the shape, else weight GEMM + data GEMM), per BatchNorm reduce + apply unless the
        training backward folds them into the node-linear backward and the target pass (pert_tconv_bwd_bn), embedding
        scatters, edge-table gradients (3 layers per launch), unpack."""
        L, H, N, training = self.n_convs, self.Hp, self._saved[8], self._saved[7]
        linear = sum(1 if self.lib.pert_linear_bwd_planes_supported(N, H, self.desc.k0 if l == 0 else H,
                                                                     H) else 2 for l in range(L))
        fold = training and self.lib.pert_linear_bwd_planes_supported(N, H, H, H) and \
            self.lib.pert_tconv_bwd_bn_supported(H, self.desc.n_rpc)
        bn = 0 if fold else 2 * (L - 1)
        return 1 + 1 + 2 * L + linear + bn + self.desc.n_cat + (L + 2) // 3 + self._pack_launches()

    @_lib.on_device_of
    def forward(self, x, cat_X, entry_id, probs, pnn, batch, index: GraphIndex, training, probe=None,
                index_ready=None, live=None):
        """-> (global_pred [B, n_out], local_pred [N,1]); keeps what backward needs in the workspace.  In training the
        BatchNorm outputs are dropped with ``model.dropout`` (mask drawn from ``model.dropout_state()``, whose step
        this call advances on the device).  ``live``: device int64 [2] {N, B} of a batch padded by
        ``pert_batch_pad`` (the inputs are the capacity buffers); the BatchNorm statistics then count the real rows
        only (``pert_model_forward_live``)."""
        N, E, B = x.size(0), index.E, entry_id.numel()
        p_drop = float(self.model.dropout) if training else 0.0
        state = self.model.dropout_state() if p_drop > 0 else None
        ws = self._workspace(N, E, B)
        dev = x.device
        x = x.contiguous().float()
        cat_X = cat_X.contiguous()
        entry_id = entry_id.contiguous().reshape(-1)
        probs = probs.reshape(-1).contiguous().float()
        pnn = pnn.reshape(-1).contiguous().float()
        batch = batch.contiguous()
        gpred = torch.empty(B, self.n_out, device=dev, dtype=torch.float32)
        lpred = torch.empty(N, 1, device=dev, dtype=torch.float32)
        p = _lib.ptr
        args = (C.byref(self.desc), p(self.fp.flat), p(self.bn_running), p(self.bn_nbt), p(x), p(cat_X), p(entry_id),
                p(probs), p(pnn), p(batch), N, E, B, p(index.rowptr), p(index.csr_src), p(index.csr_if),
                p(index.csr_rpc), p(ws), ws.numel() * 4, int(training), p_drop, p(state), p(gpred), p(lpred),
                p(index.status), C.byref(probe) if probe is not None else None,
                C.c_void_p(index_ready.cuda_event) if index_ready is not None else None)
        if self.n_out > 1:
            rc = self.lib.pert_model_forward_q(args[0], self.n_out, *args[1:], p(live), _lib.stream())
        elif live is None:
            rc = self.lib.pert_model_forward(*args, _lib.stream())
        else:
            rc = self.lib.pert_model_forward_live(*args, p(live), _lib.stream())
        _lib.check(rc, "pert_model_forward")
        self._saved = (x, cat_X, entry_id, probs, pnn, batch, index, bool(training), N, E, B, p_drop)
        ops.LAUNCHES["n"] += self.launches_forward()
        return gpred, lpred

    @_lib.on_device_of
    def backward(self, d_global, d_local=None, grads=None, probe=None, live=None):
        """Accumulates (+=) parameter gradients into ``grads`` (default: the flat gradient buffer).  ``live``: the
        word the forward got (padded batch); ``d_global`` [B, n_out] must then be 0 for the ghost graphs."""
        x, cat_X, entry_id, probs, pnn, batch, index, training, N, E, B, p_drop = self._saved
        grads = self.fp.grad if grads is None else grads
        d_global = d_global.reshape(-1).contiguous().float()
        if d_local is not None:
            d_local = d_local.reshape(-1).contiguous().float()
        p = _lib.ptr
        ws = self.ws
        args = (C.byref(self.desc), p(self.fp.flat), p(grads), p(cat_X), p(entry_id), p(probs), p(pnn), p(batch), N,
                E, B, p(index.rowptr), p(index.csr_src), p(index.csr_if), p(index.csr_rpc), p(index.colptr),
                p(index.csc_pos), p(index.csc_dst), p(ws), ws.numel() * 4, int(training), p_drop, p(d_global),
                p(d_local), C.byref(probe) if probe is not None else None)
        if self.n_out > 1:
            rc = self.lib.pert_model_backward_q(args[0], self.n_out, *args[1:], p(live), _lib.stream())
        elif live is None:
            rc = self.lib.pert_model_backward(*args, _lib.stream())
        else:
            rc = self.lib.pert_model_backward_live(*args, p(live), _lib.stream())
        _lib.check(rc, "pert_model_backward")
        ops.LAUNCHES["n"] += self.launches_backward()


class _EngineFn(torch.autograd.Function):
    """model.forward as ONE autograd node: inputs are the parameters (so autograd routes their gradients),
    outputs (global_pred, local_pred)."""

    @staticmethod
    def forward(ctx, engine, x, cat_X, entry_id, probs, pnn, batch, index, training, *params):
        g, l = engine.forward(x, cat_X, entry_id, probs, pnn, batch, index, training)
        ctx.engine = engine
        ctx.token = engine._saved
        return g, l

    @staticmethod
    def backward(ctx, dg, dl):
        eng = ctx.engine
        if eng._saved is not ctx.token:
            raise RuntimeError("engine workspace was overwritten by a later forward before this backward ran "
                               "(one in-flight forward per model replica)")
        gbuf = torch.zeros_like(eng.fp.flat)
        eng.backward(dg, dl, grads=gbuf)
        eng.last_grad_buffer = gbuf      # every parameter gradient is a view of this buffer (one all-reduce in DP)
        views = eng.fp.views_of(gbuf)
        params = eng.fp.params
        # The reference loop calls optimizer.zero_grad() (set_to_none) before every backward (pert_gnn.py:232): every
        # .grad is None and autograd's AccumulateGrad would just install the 42 views one by one (~0.25 ms of host time
        # per step, a third of this loop's budget).  In exactly that state -- no gradient to accumulate into, no hooks
        # registered on any parameter -- the views are attached directly and autograd gets no parameter gradients to
        # route.  Any other state takes the regular autograd path below.
        direct = True
        for p in params:
            if p.grad is not None or p._backward_hooks or getattr(p, "_post_accumulate_grad_hooks", None):
                direct = False
                break
        if direct:
            for p, v in zip(params, views):
                p.grad = v
            return (None,) * (9 + len(params))
        return (None,) * 9 + tuple(views)


def engine_forward(engine, x, cat_X, entry_id, probs, pnn, batch, index, training):
    return _EngineFn.apply(engine, x, cat_X, entry_id, probs, pnn, batch, index, training, *engine.fp.params)
