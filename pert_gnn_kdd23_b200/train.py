"""Train / eval step mirroring reference pert_gnn.py:191-193 (pinball loss), :213-251 (train), :254-294 (test),
plus the data-parallel wrapper the reference lacks (SURVEY.md 8e: shard independent graphs over GPUs, ONE
flat-buffer gradient all-reduce per step).

Every step, metric and evaluation takes ``tau=None``: the levels of a quantile model (``model.quantiles``; an explicit
``tau`` must equal them), else 0.5.  A model with T > 1 levels trains on the mean pinball loss over its T outputs.
"""
from __future__ import annotations

import ctypes as C
import math
import operator
import weakref

import numpy as np
import torch
import torch.distributed as dist

from . import _lib, ops


def torch_quantile_loss(y_test, y_hat, tau=None):
    """reference pert_gnn.py:191-193 (tau None: 0.5).  With a sequence of T levels, y_hat is [B, T] and the loss is the
    mean over the B T pinball terms, column t at level tau[t]."""
    if tau is None:
        tau = 0.5
    if isinstance(tau, (tuple, list)):
        taus = torch.tensor(tau, dtype=y_hat.dtype, device=y_hat.device)
        e = y_test.reshape(-1, 1) - y_hat
        return torch.mean(torch.maximum(taus * e, (taus - 1) * e))
    e = y_test - y_hat
    return torch.mean(torch.maximum(tau * e, (tau - 1) * e))


def _as_levels(tau):
    try:
        return (float(tau),)
    except TypeError:
        return tuple(float(t) for t in tau)


def resolve_tau(model, tau=None):
    """-> the quantile levels a step or evaluation of ``model`` uses, as a tuple.  ``tau`` None: ``model.quantiles``,
    else (0.5,).  On a quantile model an explicit ``tau`` (a level or a sequence) must equal its levels; a model without
    quantiles takes one level.  ``ValueError`` otherwise."""
    q = getattr(model, "quantiles", None)
    if tau is None:
        return q if q is not None else (0.5,)
    given = _as_levels(tau)
    if q is not None and given != q:
        raise ValueError(f"tau {given} differs from the model's quantile levels {q}")
    if q is None and len(given) != 1:
        raise ValueError(f"a model without quantiles has one output, got {len(given)} levels")
    return given


def _c_levels(levels):
    """The levels as the host float array the _q entry points read (by value, so a captured graph keeps them)."""
    return (C.c_float * len(levels))(*levels)


def model_inputs(data):
    """Argument tuple of SAGEDeterministic.forward from a Batch (pert_gnn.py:233-243); the per-node pattern
    probability ``rt_probs`` is precomputed at collation instead of rebuilt on the host every step (:220-230)."""
    probs = data.rt_probs if "rt_probs" in data else data.pattern_probs
    return (data.x, data.cat_X, data.edge_index, data.edge_attr, data.pattern_num_nodes, probs, data.entry_id,
            data.batch)


def flat_layout(sizes):
    """Offsets (floats) of parameters of ``sizes`` floats in one flat buffer, each on a ``_lib.FLAT_ALIGN``-float
    (256-byte: float4 / TMA) boundary, and the buffer's length -> (offsets, n)."""
    a = _lib.FLAT_ALIGN
    offs, n = [], 0
    for k in sizes:
        offs.append(n)
        n += (int(k) + a - 1) // a * a
    return offs, n


class FlatParams:
    """All parameters (and their gradients) of a module as views into two flat fp32 buffers, so that the
    gradient all-reduce and the Adam update are ONE collective and ONE kernel (payload <= 4.8 MB, latency-bound)."""

    def __init__(self, module, bind_grads=True):
        params = [p for p in module.parameters() if p.requires_grad]
        offs, n = flat_layout([p.numel() for p in params])
        dev = params[0].device
        self.flat = torch.zeros(n, device=dev, dtype=torch.float32)
        self.grad = torch.zeros(n, device=dev, dtype=torch.float32)
        self._layout = []                              # (offset, shape, contiguous strides) of every parameter
        for p, off in zip(params, offs):
            k = p.numel()
            self.flat[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + k].view_as(p)
            if bind_grads:
                p.grad = self.grad[off:off + k].view_as(p)
            self._layout.append((off, tuple(p.shape), tuple(p.stride())))
        self.params = params
        self.numel = n
        self._optimizers = []      # weak references to the FusedAdams over this object, whose m and v grow() relays
        # ONE FlatParams per module: model.engine() adopts this one instead of re-pointing p.data into a second flat
        # buffer (which would silently detach an optimizer built over this one)
        if isinstance(module, torch.nn.Module):
            module.__dict__["_flat_params"] = self

    @property
    def device(self):
        return self.flat.device

    def owns(self, module):
        """True while every trainable parameter of ``module`` is still a view into this flat buffer."""
        lo = self.flat.data_ptr()
        hi = lo + self.flat.numel() * 4
        ps = [p for p in module.parameters() if p.requires_grad]
        return len(ps) == len(self.params) and all(lo <= p.data_ptr() < hi for p in ps)

    def owns_fast(self):
        """Cheap form of ``owns`` for the per-step path: the first and the last parameter still live in the flat buffer
        (``module.to()`` / re-flattening moves all of them; ``load_state_dict`` copies in place)."""
        lo = self.flat.data_ptr()
        hi = lo + self.flat.numel() * 4
        return lo <= self.params[0].data_ptr() < hi and lo <= self.params[-1].data_ptr() < hi

    def views_of(self, buf):
        """One view per parameter (its shape) into ``buf``, a flat tensor laid out like ``flat`` / ``grad``."""
        return [buf.as_strided(shape, stride, off) for off, shape, stride in self._layout]

    def zero_grad(self):
        self.grad.zero_()

    def grow_plan(self, new_shapes):
        """The layout ``grow(new_shapes)`` moves to, host only: (shapes, offsets, length, segment table [n, 4] int64 of
        (old_off, new_off, old_len, new_len) per parameter).  ``PertGnnError`` for a shape ``grow`` refuses."""
        shapes = [tuple(int(d) for d in s) for s in new_shapes]
        if len(shapes) != len(self.params):
            raise _lib.PertGnnError(f"FlatParams.grow: {len(shapes)} shapes for {len(self.params)} parameters")
        for i, (p, s) in enumerate(zip(self.params, shapes)):
            old = tuple(p.shape)
            if len(s) != len(old) or s[1:] != old[1:] or (old and s[0] < old[0]):
                raise _lib.PertGnnError(f"FlatParams.grow: parameter {i} of shape {old} cannot become {s} (only the "
                                        "first dimension may grow)")
        if len(self.params) > _lib.FLAT_MAX_SEGS:
            raise _lib.PertGnnError(f"FlatParams.grow: {len(self.params)} parameters, at most {_lib.FLAT_MAX_SEGS}")
        sizes = [int(np.prod(s, dtype=np.int64)) for s in shapes]
        offs, n = flat_layout(sizes)
        segs = np.array([(o, no, p.numel(), k) for (o, _, _), no, p, k in zip(self._layout, offs, self.params, sizes)],
                        dtype=np.int64).reshape(-1, 4)
        return shapes, offs, n, segs

    def _live_optimizers(self):
        self._optimizers = [r for r in self._optimizers if r() is not None]
        return [r() for r in self._optimizers]

    @_lib.on_device_of
    def grow(self, new_shapes):
        """Grows parameters in place.  ``new_shapes``: one shape per parameter, in ``params`` order, equal to its
        current shape except for the first dimension, which may only grow (new embedding rows).

        The new layout follows the constructor's rule (``flat_layout``).  Every new buffer is allocated before anything
        changes; then one launch (``pert_flat_grow``) copies each parameter, and each parameter's slot of the m and v
        of the ``FusedAdam`` over this object (every one registers itself here), bit for bit to its new offset, writes 0
        to the new rows and the padding, and zeroes the new gradient buffer.  So no optimizer over this object is left
        with buffers of the old length, whether or not the caller names it.  Every parameter is re-pointed at the new
        buffer.  A gradient bound to ``grad`` is bound to the new one; any other ``p.grad`` is stale and set to None.
        This object stays the one the model, the optimizer and ``DataParallel`` hold.  ``PertGnnError``, before anything
        changes, for host buffers, for more than one live FusedAdam over this object and for a ``PeerAdam`` over more
        than one rank (its m and v cover its own slice)."""
        shapes, offs, n, segs = self.grow_plan(new_shapes)
        opts = self._live_optimizers()
        if len(opts) > 1:
            raise _lib.PertGnnError(f"FlatParams.grow: {len(opts)} FusedAdams hold this FlatParams; one can be relaid")
        if opts and getattr(opts[0], "world", 1) > 1:
            raise _lib.PertGnnError("FlatParams.grow: PeerAdam over more than one rank keeps m and v for its own slice "
                                    "only; growing it is not supported")
        carry = [b for o in opts for b in (o.m, o.v)]
        if any(c.shape != self.flat.shape for c in carry):
            raise _lib.PertGnnError("FlatParams.grow: the optimizer's m / v are not laid out like this FlatParams")
        if not self.flat.is_cuda:
            raise _lib.PertGnnError("FlatParams.grow needs CUDA buffers (no CPU fallback for the relayout)")
        sizes = segs[:, 3].tolist()
        dev = self.device
        flat, grad = (torch.empty(n, device=dev, dtype=torch.float32) for _ in range(2))
        out = [torch.empty(n, device=dev, dtype=torch.float32) for _ in carry]
        src, dst = carry + [None] * (2 - len(carry)), out + [None] * (2 - len(out))
        p = _lib.ptr
        _lib.call("pert_flat_grow", segs.ctypes.data, segs.shape[0], self.numel, n, p(self.flat), p(flat), p(src[0]),
                  p(dst[0]), p(src[1]), p(dst[1]), p(grad), _lib.stream())
        ops.LAUNCHES["n"] += 1
        st = torch.cuda.current_stream()
        for t in (self.flat, self.grad, *carry):        # the launch still reads them: no reuse before it is done
            t.record_stream(st)
        lo, hi = self.grad.data_ptr(), self.grad.data_ptr() + self.grad.numel() * 4
        layout = []
        for q, off, s, k in zip(self.params, offs, shapes, sizes):
            bound = q.grad is not None and lo <= q.grad.data_ptr() < hi
            q.grad = None
            q.data = flat[off:off + k].view(s)
            if bound:
                q.grad = grad[off:off + k].view(s)
            layout.append((off, s, tuple(q.stride())))
        self.flat, self.grad, self._layout, self.numel = flat, grad, layout, n
        if opts:
            opts[0].m, opts[0].v = out


class FusedAdam:
    """torch.optim.Adam(params, lr) semantics (reference pert_gnn.py:343) in one kernel over FlatParams."""

    def __init__(self, flat: FlatParams, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.fp = flat
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.m = torch.zeros_like(flat.flat)
        self.v = torch.zeros_like(flat.flat)
        self.t = 0
        flat._optimizers.append(weakref.ref(self))

    @property
    def device(self):
        return self.fp.flat.device

    def zero_grad(self, set_to_none=False):
        self.fp.zero_grad()

    def _check_layout(self):
        # m and v must cover the flat buffer: the kernel runs over fp.numel floats of each
        if self.m.numel() != self.fp.numel or self.v.numel() != self.fp.numel:
            raise _lib.PertGnnError(f"{type(self).__name__}.step: m / v hold {self.m.numel()} / {self.v.numel()} floats "
                                    f"but the FlatParams {self.fp.numel}")

    @_lib.on_device_of
    def step(self, grad_scale=1.0):
        self._check_layout()
        self.t += 1
        _lib.call("pert_adam_step", _lib.ptr(self.fp.flat), _lib.ptr(self.fp.grad), _lib.ptr(self.m),
                  _lib.ptr(self.v), self.fp.numel, self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.t,
                  float(grad_scale), _lib.stream())
        ops.LAUNCHES["n"] += 1


class PeerAdam(FusedAdam):
    """FusedAdam whose step also averages the gradient over the data-parallel ranks: ONE kernel per step
    (csrc/peer.cu) that publishes the flat gradient in a CUDA-IPC exchange buffer, reduces + updates ITS 1/world slice
    of the parameters from the peers' buffers over NVLink and pushes the result to every rank (m, v are maintained
    for the owned slice only) -- no NCCL call on the step path.  ``DataParallel`` skips its own
    all-reduce when the optimiser is a PeerAdam.  Needs one process per GPU on one node (``torch.distributed``
    initialised, used once to exchange the 64-byte IPC handles); with a single rank it degenerates to FusedAdam."""

    fused_allreduce = True

    def __init__(self, flat: FlatParams, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, group=None):
        super().__init__(flat, lr, betas, eps, weight_decay)
        import ctypes

        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self._own = None
        self._peers = []
        self.status = torch.zeros(1, dtype=torch.int32, device=flat.flat.device)
        self.timing = torch.zeros(5, dtype=torch.int64, device=flat.flat.device)   # ns publish/wait/reduce/gather, calls
        if self.world == 1:
            return
        if self.world > 8:
            raise _lib.PertGnnError("PeerAdam supports up to 8 ranks on one node")
        L = _lib.lib()
        dev = flat.flat.device

        def all_ok(ok):
            # every rank takes part in every collective of the setup, whatever happened locally: a rank that failed
            # must not leave the others waiting in a different collective
            t = torch.tensor([1.0 if ok else 0.0], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            return float(t) > 0.0

        err = None
        handle = (ctypes.c_ubyte * 64)()
        try:
            nbytes = L.pert_peer_exchange_bytes(flat.numel)
            own = ctypes.c_void_p()
            _lib.check(L.pert_peer_alloc(nbytes, ctypes.byref(own), handle), "pert_peer_alloc")
            self._own = own.value
        except Exception as e:  # noqa: BLE001
            err = e
        if not all_ok(err is None):
            self.close(collective=False)
            raise _lib.PertGnnError(f"PeerAdam setup failed on some rank (local error: {err!r})")
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=dev)
        gathered = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(gathered, mine, group=group)
        ptrs = []
        try:
            for r in range(self.world):
                if r == self.rank:
                    ptrs.append(self._own)
                    continue
                hb = (ctypes.c_ubyte * 64)(*gathered[r].cpu().tolist())
                pp = ctypes.c_void_p()
                _lib.check(L.pert_peer_open(hb, ctypes.byref(pp)), "pert_peer_open")
                self._peers.append(pp.value)
                ptrs.append(pp.value)
        except Exception as e:  # noqa: BLE001
            err = e
        if not all_ok(err is None):
            self.close(collective=False)
            raise _lib.PertGnnError(f"PeerAdam peer mapping failed on some rank (local error: {err!r})")
        self._xbufs = (ctypes.c_void_p * self.world)(*ptrs)
        dist.barrier(group=group)      # every rank has mapped every buffer before the first step touches them

    @_lib.on_device_of
    def step(self, grad_scale=1.0):
        if self.world == 1:
            return super().step(grad_scale)
        self._check_layout()
        self.t += 1
        _lib.call("pert_allreduce_adam", _lib.ptr(self.fp.flat), _lib.ptr(self.fp.grad), _lib.ptr(self.m),
                  _lib.ptr(self.v), self.fp.numel, self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.t,
                  float(grad_scale), self._xbufs, self.rank, self.world, _lib.ptr(self.status), _lib.ptr(self.timing),
                  _lib.stream())
        ops.LAUNCHES["n"] += 1

    def phase_times_us(self, reset=True):
        """Mean microseconds CTA 0 of the fused kernel spent publishing, waiting for the peers' gradients, reducing +
        Adam on its slice + pushing the parameters, and gathering the peers' slices (synchronising read; the wait phase
        is the slowest rank's skew plus the flag round trip over NVLink)."""
        t = self.timing.cpu().tolist()
        if reset:
            self.timing.zero_()
        n = max(t[4], 1)
        return {"publish_us": t[0] / n / 1e3, "wait_us": t[1] / n / 1e3, "reduce_adam_us": t[2] / n / 1e3,
                "gather_us": t[3] / n / 1e3, "calls": t[4]}

    def check(self):
        """Synchronising check of the device status word (a peer that never arrived sets PERT_ERR_PEER_TIMEOUT)."""
        code = int(self.status.item())
        if code != 0:
            _lib.check(code, "pert_allreduce_adam")

    def close(self, collective=True):
        L = _lib.lib()
        for pp in self._peers:
            L.pert_peer_close(pp)
        self._peers = []
        if self._own:
            if collective and dist.is_initialized() and self.world > 1:
                torch.cuda.synchronize()
                dist.barrier(group=self.group)     # nobody still reads this buffer
            L.pert_peer_free(self._own)
            self._own = None


class DataParallel:
    """One process per GPU; each rank owns a shard of the graphs; gradients are averaged with a single
    all-reduce of the flat gradient buffer (NCCL over NVLink on the box, gloo in the CPU tests).
    BatchNorm statistics stay per-replica (like DDP); parity claims are per shard (DESIGN.md)."""

    def __init__(self, flat: FlatParams, group=None):
        self.fp = flat
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1

    def all_reduce_grads(self, optimizer=None):
        """Sums the flat gradient over the ranks (unless ``optimizer`` does it itself, see PeerAdam) and returns the
        scale that turns the sum into the mean."""
        if self.world > 1 and not getattr(optimizer, "fused_allreduce", False):
            dist.all_reduce(self.fp.grad, op=dist.ReduceOp.SUM, group=self.group)
        return 1.0 / self.world


    def all_reduce_module_grads(self, model):
        """Averages the gradients ATTACHED to the parameters (``p.grad``) over the ranks -- the torch-optimizer branch
        of ``train_step``: ``torch.optim``'s ``zero_grad()`` defaults to ``set_to_none=True``, so the views FlatParams
        bound to ``fp.grad`` are gone and autograd installs views of the engine's last gradient buffer instead.  One
        all-reduce of that buffer when every gradient is a view of it, else flatten -> reduce -> scatter back."""
        if self.world <= 1:
            return
        gs = [p.grad for p in model.parameters() if p.grad is not None]
        if not gs:
            return
        gb = getattr(getattr(model, "_engine", None), "last_grad_buffer", None)
        if gb is not None:
            lo, hi = gb.data_ptr(), gb.data_ptr() + gb.numel() * gb.element_size()
            if all(lo <= g.data_ptr() < hi for g in gs):
                dist.all_reduce(gb, op=dist.ReduceOp.SUM, group=self.group)
                gb.mul_(1.0 / self.world)
                return
        flat = torch.cat([g.reshape(-1) for g in gs])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
        flat.mul_(1.0 / self.world)
        o = 0
        for g in gs:
            g.copy_(flat[o:o + g.numel()].view_as(g))
            o += g.numel()


GROWN_TABLES = ("cat", "entry", "interface", "rpctype")


def _tables(model):
    return dict(zip(GROWN_TABLES, (model.cat_embedding[0], model.entry_embeds, model.interface_embeds,
                                   model.rpctype_embeds)))


def grow_embeddings(model, optimizer=None, store=None, *, entry=None, interface=None, rpctype=None, cat=None,
                    seed=None):
    """Appends rows to the embedding tables of a trained ``SAGEDeterministic`` so that it covers the ids a live
    ``PatternStore`` has gained (``append_traces``), keeping every trained value and the optimizer state.  Returns the
    row counts {"cat", "entry", "interface", "rpctype"} after the call; "cat" is ``cat_embedding[0]``, the microservice
    table that ``cat_X`` column 0 indexes.

    The target of each table is the largest of its current rows, the explicit argument and, with ``store``, the
    store's ``id_bounds()``.  An explicit count below the current one is refused: tables never shrink.  When no table
    grows, nothing is touched (no relayout; the engine and every captured graph stay).

    New rows are drawn N(0, 1), as ``nn.Embedding`` initialises them, table by table in the order above, from
    ``torch.Generator(device).manual_seed(seed)`` when ``seed`` is given, else from torch's default generator of the
    device: data-parallel replicas given one seed grow identically, with no collective (as ``seed_dropout``).

    The parameters move through ``FlatParams.grow`` (one relayout launch, ``pert_flat_grow``): the ``FlatParams`` of
    ``optimizer`` (``FusedAdam``), else the one registered on the model (a new one if none holds it).  Optimizer state:
    the m and v of the ``FusedAdam`` over that ``FlatParams`` are relaid by the same launch -- also when ``optimizer``
    is omitted, as the FlatParams knows its optimizer -- with m = v = 0 in the new rows, and its step count stays.
    That is the state of a row present from the start that never received a gradient; with weight_decay = 0 Adam
    leaves such a row bit-unchanged (its update is 0 / (0 + eps)) until a batch uses it.  A ``torch.optim`` optimizer
    (the drop-in loop) gets every state tensor of a grown table padded with zero rows (Adam's exp_avg, exp_avg_sq),
    ``step`` kept.  ``PeerAdam`` over more than one rank is refused: its m and v cover the rank's own slice and its
    exchange buffers are mapped into the other processes.

    ``num_embeddings`` follows on the modules, so ``state_dict`` has the grown shapes and loads into a model built at
    them.  The step engine is dropped and built again on next use (its descriptor carries the row counts and the
    offsets); the BatchNorm running statistics, ``num_batches_tracked`` and the dropout counter carry over.  Every
    captured graph (``GraphedTrainStep``, ``BucketedTrainStep``, ``evaluate_bucketed``, ``predict``) was captured over
    the old engine and is captured again on its next visit (``_GraphCache.invalidations``).  Refused during CUDA-graph
    capture and for a model that is not on a CUDA device."""
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise _lib.PertGnnError("grow_embeddings cannot run during CUDA-graph capture")
    if isinstance(optimizer, PeerAdam) and optimizer.world > 1:
        raise _lib.PertGnnError("grow_embeddings: PeerAdam over more than one rank keeps m and v for its own slice "
                                "only and maps its exchange buffers across processes; growing it is not supported")
    if optimizer is not None and not isinstance(optimizer, (FusedAdam, torch.optim.Optimizer)):
        raise _lib.PertGnnError(f"grow_embeddings: unsupported optimizer {type(optimizer).__name__}")
    tables = _tables(model)
    rows = {k: int(e.num_embeddings) for k, e in tables.items()}
    want = dict(rows)
    for k, v in zip(GROWN_TABLES, (cat, entry, interface, rpctype)):
        if v is None:
            continue
        v = operator.index(v)
        if v < rows[k]:
            raise _lib.PertGnnError(f"grow_embeddings: {k} = {v} is below the table's {rows[k]} rows (tables never "
                                    "shrink)")
        want[k] = v
    if store is not None:
        for k, v in store.id_bounds().items():
            want[k] = max(want[k], v)
    if want == rows:
        return want
    if isinstance(optimizer, FusedAdam) and not optimizer.fp.owns(model):
        raise _lib.PertGnnError("grow_embeddings: the optimizer's FlatParams does not hold this model's parameters")
    if not model.entry_embeds.weight.is_cuda:
        raise _lib.PertGnnError("grow_embeddings needs the model on a CUDA device (the relayout runs there)")
    if isinstance(optimizer, FusedAdam):
        fp = optimizer.fp
    else:
        reg = model.__dict__.get("_flat_params")
        fp = reg if reg is not None and reg.owns(model) else FlatParams(model, bind_grads=False)
    dev = fp.device
    gen = None
    if seed is not None:
        gen = torch.Generator(dev)
        gen.manual_seed(int(seed))
    fresh = {k: torch.randn(want[k] - rows[k], e.embedding_dim, generator=gen, device=dev)
             for k, e in tables.items() if want[k] > rows[k]}
    grown = {id(tables[k].weight): (want[k],) + tuple(tables[k].weight.shape[1:]) for k in fresh}
    shapes = [grown.get(id(p), tuple(p.shape)) for p in fp.params]
    old_shapes = {k: tuple(tables[k].weight.shape) for k in fresh}
    fp.grow(shapes)
    with torch.no_grad():
        for k, r in fresh.items():
            tables[k].weight[rows[k]:].copy_(r)
            tables[k].num_embeddings = want[k]
    if isinstance(optimizer, torch.optim.Optimizer):
        for k in fresh:
            st = optimizer.state.get(tables[k].weight)
            for name, s in (st or {}).items():
                if torch.is_tensor(s) and tuple(s.shape) == old_shapes[k]:
                    st[name] = torch.cat([s, s.new_zeros((want[k] - rows[k],) + old_shapes[k][1:])])
    model.reset_engine()
    return want


def train_step(model, optimizer, data, tau=None, dp: DataParallel | None = None):
    """One iteration of the loop body of reference pert_gnn.py:231-247 on a device-resident Batch.
    Returns the (device) loss tensor; no host sync."""
    levels = resolve_tau(model, tau)
    fused = isinstance(optimizer, FusedAdam)
    if fused and hasattr(model, "engine"):
        # the model must read the SAME flat buffer the optimizer updates, and its p.grad must be the views of fp.grad
        eng = model.engine(optimizer.fp)
        lo, hi = optimizer.fp.grad.data_ptr(), optimizer.fp.grad.data_ptr() + optimizer.fp.grad.numel() * 4
        for p in optimizer.fp.params:
            if p.grad is None or not (lo <= p.grad.data_ptr() < hi):
                base = optimizer.fp.flat.data_ptr()
                o = (p.data_ptr() - base) // 4
                p.grad = optimizer.fp.grad[o:o + p.numel()].view_as(p)
    optimizer.zero_grad()
    global_pred, _ = model(*model_inputs(data))
    if len(levels) == 1:
        loss = torch_quantile_loss(data.y.float(), global_pred.flatten(), levels[0])
    else:
        loss = torch_quantile_loss(data.y.float(), global_pred, levels)
    loss.backward()
    if fused:
        scale = dp.all_reduce_grads(optimizer) if dp is not None else 1.0
        optimizer.step(grad_scale=scale)
    else:
        if dp is not None:
            dp.all_reduce_module_grads(model)
        optimizer.step()
    return loss


_SIDE_STREAMS = {}


def _side_stream(device):
    key = torch.device(device).index
    st = _SIDE_STREAMS.get(key)
    if st is None:
        st = _SIDE_STREAMS[key] = torch.cuda.Stream(device)
    return st


@_lib.on_device_of
def _fused_fwd_bwd(model, optimizer: FusedAdam, data, tau, index, probe, use_index_cache=True, live=None):
    """Device work of one step up to the gradients: (index build) -> zero grads -> engine forward -> pinball loss +
    its gradient -> engine backward into the flat gradient buffer.  Returns (loss [1], index).  ``live``: the {N, B}
    word of a padded batch (``PaddedBatch``), read by the engine and the loss.  ``tau``: as in ``resolve_tau``."""
    from .index import build_index, cached_index

    tau = resolve_tau(model, tau)
    eng = _engine_of(model, optimizer)
    x, cat_X, edge_index, edge_attr, pnn, probs, entry_id, batch = model_inputs(data)
    index_ready = None
    if index is None:
        n_if, n_rpc = model.interface_embeds.num_embeddings, model.rpctype_embeds.num_embeddings
        if use_index_cache:
            index = cached_index(edge_index, x.size(0), edge_attr, n_if, n_rpc)
        else:
            # build the index on a side stream: the forward only waits for it right before the first attention
            # kernel, so it overlaps the parameter pack, the input prologue and the first GEMM
            main = torch.cuda.current_stream(x.device)
            side = _side_stream(x.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                index = build_index(edge_index, x.size(0), edge_attr, n_if, n_rpc, check=False)
                index_ready = torch.cuda.Event()
                index_ready.record(side)
    optimizer.zero_grad()
    with torch.no_grad():
        gpred, _ = eng.forward(x, cat_X, entry_id, probs, pnn, batch, index, model.training, probe=probe,
                               index_ready=index_ready, live=live)
        B, T = gpred.size(0), len(tau)
        if gpred.size(1) != T:
            raise ValueError(f"{T} quantile levels for a head of {gpred.size(1)} outputs")
        loss = torch.empty(1, device=gpred.device, dtype=torch.float32)
        dy = torch.empty((B, T) if T > 1 else (B,), device=gpred.device, dtype=torch.float32)
        if T > 1:
            _lib.call("pert_pinball_loss_q", _lib.ptr(data.y), _lib.ptr(gpred), _c_levels(tau), T, B, 1.0,
                      _lib.ptr(loss), _lib.ptr(dy), _lib.ptr(live), _lib.stream())
        elif live is None:
            _lib.call("pert_pinball_loss", _lib.ptr(data.y), _lib.ptr(gpred), float(tau[0]), B, 1.0, _lib.ptr(loss),
                      _lib.ptr(dy), _lib.stream())
        else:
            _lib.call("pert_pinball_loss_live", _lib.ptr(data.y), _lib.ptr(gpred), float(tau[0]), B, 1.0,
                      _lib.ptr(loss), _lib.ptr(dy), _lib.ptr(live), _lib.stream())
        ops.LAUNCHES["n"] += 1
        eng.backward(dy, None, probe=probe, live=live)
    return loss, index


def _engine_of(model, optimizer: FusedAdam):
    """The step engine of ``model`` over ``optimizer``'s FlatParams (``model.engine`` is only asked when the current
    engine is over another one: the per-step path makes no ownership check)."""
    eng = model._engine
    return model.engine(optimizer.fp) if eng is None or eng.fp is not optimizer.fp else eng


def _reduce_and_step(optimizer: FusedAdam, dp: DataParallel | None, loss):
    """The end of a fused step once the gradients are in the flat buffer: (gradient all-reduce) -> fused Adam, issued
    eagerly (the Adam step count is a by-value kernel argument).  Returns ``loss``."""
    with torch.no_grad():
        scale = dp.all_reduce_grads(optimizer) if dp is not None else 1.0
        optimizer.step(grad_scale=scale)
    return loss


def fused_train_step(model, optimizer: FusedAdam, data, tau=None, dp: DataParallel | None = None, index=None,
                     probe=None):
    """Same step as ``train_step`` but without autograd: engine forward -> pinball loss + its gradient (one
    kernel) -> engine backward into the flat gradient buffer -> (all-reduce) -> fused Adam.  5 C calls per step.
    Returns the device loss tensor [1]."""
    loss, _ = _fused_fwd_bwd(model, optimizer, data, tau, index, probe)
    return _reduce_and_step(optimizer, dp, loss)


def _batch_sizes(data):
    return int(data.x.size(0)), int(data.edge_index.size(1)), int(data.num_graphs)


class _GraphCache:
    """One CUDA graph per key, for the steps below that replay their device work.

    ``cache(key, eng, sizes, fn, pin)`` returns what ``fn()`` returns.  A key's first visit runs ``fn`` eagerly (it also
    does the library's one-time initialisation), the second captures it and every visit from then on replays it; a
    replay returns the tensors of the capture, which it has just rewritten.  ``eng.reserve(*sizes)`` comes first, so
    the workspace is never allocated inside a capture.  A graph captured over another engine (re-created after the
    parameters moved) or over a workspace the engine has since re-allocated points into freed memory: that key's graph
    is dropped and captured again on the visit that finds it (``invalidations``).  At most ``max_graphs`` keys hold a
    graph; a key past that, or one whose capture raised (``capture_error``), runs ``fn`` eagerly on every visit.
    ``ops.LAUNCHES`` counts the launches a replay runs, not the ones a capture records.  An entry keeps alive what its
    graph points into: the outputs, the engine and its workspace, and ``pin`` (the caller's input buffers).  The
    callers that pad a batch into its capacity bucket (``pad``) key on the bucket and keep its ``PaddedBatch`` here."""

    def __init__(self, max_graphs=32):
        self.max_graphs = max_graphs
        self.buckets = {}    # key -> {"state": "ran-once" | "eager" | "graph", and with a graph what it keeps alive}
        self.bufs = {}       # capacity bucket -> its PaddedBatch (``pad``)
        self.capture_error = None
        self.replays = 0
        self.captures = 0
        self.invalidations = 0

    def pad(self, data):
        """Copies ``data`` into the ``PaddedBatch`` of its capacity bucket (made on the bucket's first visit).
        -> (bucket: the capacities and the edge-attribute width, the filled PaddedBatch)."""
        caps = bucket_caps(*_batch_sizes(data))
        bucket = caps + (int(data.edge_attr.size(1)),)
        buf = self.bufs.get(bucket)
        if buf is None:
            buf = self.bufs[bucket] = PaddedBatch(caps, data)
        return bucket, buf.fill(data)

    def cache(self, key, eng, sizes, fn, pin=None):
        eng.reserve(*sizes)
        ent = self.buckets.get(key)
        if ent is None:
            self.buckets[key] = {"state": "ran-once"}
            return fn()
        if ent["state"] == "graph" and (ent["engine"] is not eng or ent["ws_gen"] != eng.ws_generation):
            ent = self.buckets[key] = {"state": "ran-once"}
            self.invalidations += 1
        if ent["state"] == "ran-once":
            held = sum(e["state"] == "graph" for e in self.buckets.values())
            if held >= self.max_graphs or not self._capture(ent, eng, fn, pin):
                ent["state"] = "eager"
        if ent["state"] == "eager":
            return fn()
        ent["graph"].replay()
        ops.LAUNCHES["n"] += ent["launches"]
        self.replays += 1
        return ent["out"]

    def _capture(self, ent, eng, fn, pin):
        g = torch.cuda.CUDAGraph()
        l0 = ops.LAUNCHES["n"]
        try:
            with torch.cuda.graph(g):
                out = fn()
        except Exception as e:  # noqa: BLE001 - any capture failure leaves this key on the eager path
            self.capture_error = repr(e)
            torch.cuda.synchronize()
            return False
        finally:
            launches, ops.LAUNCHES["n"] = ops.LAUNCHES["n"] - l0, l0      # a capture runs nothing
        ent.update(state="graph", graph=g, out=out, launches=launches, engine=eng, ws_gen=eng.ws_generation,
                   ws=eng.ws, pin=pin)
        self.captures += 1
        return True


class GraphedTrainStep(_GraphCache):
    """``fused_train_step`` with the device work up to the gradients replayed from a CUDA graph.

    One graph per (input buffers, shapes) key -- e.g. one per slab of ``data.DevicePrefetcher``'s ring, or one per
    resident batch.  The graph holds: index build, gradient zeroing, engine forward, pinball loss, engine backward
    (~45 kernel launches become one ``cudaGraphLaunch``: no per-kernel launch gaps on the GPU, ~0.5 ms less host
    work per step).  The gradient all-reduce and Adam (its step count is a by-value kernel argument) are issued
    eagerly after the replay.  Eager first visit, capture, replays, invalidation and ``max_graphs`` as in
    ``_GraphCache``.  The reference has no counterpart (its loop body, pert_gnn.py:231-247, launches every operator
    from Python each step)."""

    def __init__(self, model, optimizer: FusedAdam, tau=None, dp: DataParallel | None = None, max_graphs=32):
        super().__init__(max_graphs)
        self.model, self.opt, self.tau, self.dp = model, optimizer, resolve_tau(model, tau), dp

    @staticmethod
    def _key(data):
        # every tensor the captured kernels read must sit where it sat at capture time
        ptrs = tuple(t.data_ptr() for t in model_inputs(data) if torch.is_tensor(t)) + (data.y.data_ptr(),)
        return ptrs + (tuple(data.x.shape), int(data.edge_index.size(1)), int(data.num_graphs))

    def __call__(self, data):
        # the training flag and the dropout rate are by-value arguments of the captured engine calls: a change of
        # either needs its own graph instead of a replay of the old ones
        key = self._key(data) + (self.model.training, float(self.model.dropout))
        # the index is built inside the step: the same buffers may hold another batch at replay time
        loss, _ = self.cache(key, _engine_of(self.model, self.opt), _batch_sizes(data),
                             lambda: _fused_fwd_bwd(self.model, self.opt, data, self.tau, None, None,
                                                    use_index_cache=False), pin=data)
        return _reduce_and_step(self.opt, self.dp, loss)


# ------------------------------------------------------------------------------------------ capacity buckets
def ladder(x):
    """x up to 16, else x rounded up to 4 significant bits (m * 2^k, m in 8..15): less than 1/8 wasted."""
    x = int(x)
    if x <= 16:
        return x
    k = x.bit_length() - 4
    m = -(-x >> k)                     # ceil(x / 2^k), in 8..16
    return m << k


def bucket_caps(N, E, B):
    """Capacity bucket (N_cap, E_cap, B_cap) of a batch of N nodes, E edges and B graphs: at least one ghost graph
    (B_cap > B), at least one ghost node per ghost graph and at most 4 ghost edges per ghost node (a single ghost hub
    with thousands of self-loops would stall a warp of the attention kernels)."""
    B_cap = ladder(B + 1)
    E_cap = ladder(E)
    return ladder(N + max(B_cap - B, -(-(E_cap - E) // 4))), E_cap, B_cap


def bucket_bound(N, E, B):
    """Componentwise upper bound of ``bucket_caps(n, e, b)`` over all n <= N, e <= E, b <= B (monotone in each
    argument, which ``bucket_caps`` is not in N_cap): ``ladder`` adds less than 1/8, so a batch has at most
    ceil((b + 1) / 8) + 1 ghost graphs and ceil(e / 8) ghost edges."""
    return (ladder(N + max(-(-(B + 1) // 8) + 1, -(-(-(-E // 8)) // 4))), ladder(E), ladder(B + 1))


class PaddedBatch:
    """Persistent device buffers of one capacity bucket.  ``fill(data)`` copies a batch into them and writes the
    ghost tail and the {N, B} word ``live`` (``pert_batch_pad``, one launch); the object then serves as the batch of
    the padded step (``model_inputs`` works on it)."""

    def __init__(self, caps, like):
        N_cap, E_cap, B_cap = caps
        dev = like.x.device
        f32, i64 = torch.float32, torch.int64
        self.caps = caps
        self.x = torch.empty(N_cap, like.x.size(1), dtype=f32, device=dev)
        self.cat_X = torch.empty(N_cap, like.cat_X.size(1), dtype=i64, device=dev)
        self.edge_index = torch.empty(2, E_cap, dtype=i64, device=dev)
        self.edge_attr = torch.empty(E_cap, like.edge_attr.size(1), dtype=i64, device=dev)
        self.batch = torch.empty(N_cap, dtype=i64, device=dev)
        self.entry_id = torch.empty(B_cap, dtype=i64, device=dev)
        self.y = torch.empty(B_cap, dtype=i64, device=dev)
        self.rt_probs = torch.empty(N_cap, 1, dtype=f32, device=dev)
        self.pattern_num_nodes = torch.empty(N_cap, 1, dtype=f32, device=dev)
        self.live = torch.zeros(2, dtype=i64, device=dev)
        self.num_graphs = B_cap

    def __contains__(self, key):
        return key == "rt_probs"

    @property
    def device(self):
        return self.x.device

    @staticmethod
    def accepts(data):
        """True if ``fill`` can pad ``data``: per-node ``rt_probs`` and ``pattern_num_nodes``, edge attributes, at
        least one graph.  A batch with per-pattern ``pattern_probs`` only is not padded (the callers run it eagerly)."""
        if "rt_probs" not in data or data.edge_attr is None or data.num_graphs < 1:
            return False
        N = data.x.size(0)
        return data.rt_probs.numel() == N and data.pattern_num_nodes.numel() == N

    @_lib.on_device_of
    def fill(self, data):
        if not self.accepts(data):
            raise _lib.PertGnnError("PaddedBatch needs per-node rt_probs and pattern_num_nodes and edge attributes")
        x, cat_X, edge_index, edge_attr, pnn, probs, entry_id, batch = model_inputs(data)
        N, E, B = x.size(0), edge_index.size(1), entry_id.numel()
        c = lambda t: t.contiguous()
        x, cat_X, edge_index, edge_attr = c(x.float()), c(cat_X), c(edge_index), c(edge_attr)
        pnn, probs, entry_id, batch, y = c(pnn.float()), c(probs.float()), c(entry_id), c(batch), c(data.y)
        p = _lib.ptr
        _lib.call("pert_batch_pad", p(x), p(cat_X), p(edge_index), p(edge_attr), p(batch), p(entry_id), p(y),
                  p(probs), p(pnn), N, E, B, x.size(1), cat_X.size(1), edge_attr.size(1), p(self.x), p(self.cat_X),
                  p(self.edge_index), p(self.edge_attr), p(self.batch), p(self.entry_id), p(self.y),
                  p(self.rt_probs), p(self.pattern_num_nodes), *self.caps, p(self.live), _lib.stream())
        ops.LAUNCHES["n"] += 1
        return self


class BucketedTrainStep(_GraphCache):
    """``fused_train_step`` replayed from one CUDA graph per capacity bucket, for batches whose sizes and buffers
    change every step (a shuffled ``StoreLoader``: ``GraphedTrainStep`` keys on both and never replays there).

    Each batch is padded into the persistent buffers of its bucket ``bucket_caps(N, E, B)`` (``PaddedBatch``, one
    eager launch); the kernels run at the capacity sizes and read the real {N, B} from a device word where a count
    enters the arithmetic (BatchNorm statistics and backward, the loss), so the step computes what the unpadded step
    computes for the real graphs.  Eager first visit, capture, replays and ``max_graphs`` as in ``_GraphCache``: past
    ``max_graphs`` buckets and after a failed capture the padded step runs eagerly.  A graph captured over an engine or
    workspace that has since been replaced (a re-allocation for a bigger bucket, a re-created engine) is captured again
    (``invalidations``; ``reserve(*loader.max_sizes())`` sizes the workspace once up front).  A batch ``PaddedBatch``
    cannot pad (per-pattern probabilities only) runs eager ``fused_train_step``.  ``pad_ratio`` = sum of N_cap / sum
    of N over the padded steps."""

    def __init__(self, model, optimizer: FusedAdam, tau=None, dp: DataParallel | None = None, max_graphs=32):
        super().__init__(max_graphs)
        self.model, self.opt, self.tau, self.dp = model, optimizer, resolve_tau(model, tau), dp
        self._n_real = 0
        self._n_cap = 0

    @property
    def pad_ratio(self):
        return self._n_cap / max(self._n_real, 1)

    def reserve(self, N, E, B):
        """Sizes the engine workspace for every bucket of a batch of at most N nodes, E edges and B graphs."""
        _engine_of(self.model, self.opt).reserve(*bucket_bound(N, E, B))

    def __call__(self, data):
        if not PaddedBatch.accepts(data):
            return fused_train_step(self.model, self.opt, data, self.tau, self.dp)
        bucket, buf = self.pad(data)
        self._n_real += int(data.x.size(0))
        self._n_cap += buf.caps[0]
        # training flag and dropout rate are by-value arguments of the captured calls: each needs its own graph
        key = bucket + (self.model.training, float(self.model.dropout))
        loss, _ = self.cache(key, _engine_of(self.model, self.opt), buf.caps,
                             lambda: _fused_fwd_bwd(self.model, self.opt, buf, self.tau, None, None,
                                                    use_index_cache=False, live=buf.live), pin=buf)
        return _reduce_and_step(self.opt, self.dp, loss)


class AsyncLossReader:
    """Per-step loss read-back that does not drain the stream: ``push(loss)`` enqueues a 4-byte D2H copy into a pinned
    slot + an event right behind the step that produced ``loss`` and returns the value of the PREVIOUS push (whose
    copy has long finished while the current step was being enqueued); ``flush()`` returns the last one.  The
    reference reads ``loss.item()`` synchronously every step (pert_gnn.py:248); the running sum is identical, the GPU
    just never waits for the host between steps."""

    def __init__(self, device):
        self.buf = torch.zeros(2, dtype=torch.float32).pin_memory()
        self.ev = [torch.cuda.Event(), torch.cuda.Event()]
        self.pending = None
        self.n = 0
        self.device = device

    def push(self, loss):
        slot = self.n & 1
        self.n += 1
        self.buf[slot:slot + 1].copy_(loss.detach().reshape(1), non_blocking=True)
        self.ev[slot].record()
        prev = self.flush() if self.pending is not None else None
        self.pending = slot
        return prev

    def flush(self):
        if self.pending is None:
            return None
        self.ev[self.pending].synchronize()
        v = float(self.buf[self.pending])
        self.pending = None
        return v


class EvalMetrics:
    """Device-side accumulators of the reference's eval loop (pert_gnn.py:254-294): sum |pred - y|, sum |pred - y| / y
    and sum of the per-graph pinball terms, kept in doubles ON THE DEVICE (``pert_eval_metrics_q``) so that a whole
    epoch needs ONE D2H read (``result()``) instead of the reference's per-batch syncs.

    ``tau``: one level (None: 0.5) or a sequence of T quantile levels for predictions [B, T].  ``acc`` holds 4T + 1
    doubles: per level the three sums and the count of graphs with y <= pred (``coverage``), then the count of graphs
    whose levels cross (``crossing``)."""

    def __init__(self, device, tau=None):
        self.levels = (0.5,) if tau is None else _as_levels(tau)
        self.tau = self.levels[0] if len(self.levels) == 1 else self.levels
        self._taus = _c_levels(self.levels)
        self.acc = torch.zeros(4 * len(self.levels) + 1, dtype=torch.float64, device=device)
        self.count = 0

    @property
    def device(self):
        return self.acc.device

    def reset(self):
        self.acc.zero_()
        self.count = 0

    def update(self, y, yhat):
        """Adds the graphs of labels ``y`` [B] and predictions ``yhat`` [B, T] ([B] or [B, 1] at T = 1)."""
        self.add(y, yhat)
        self.count += int(y.numel())

    @_lib.on_device_of
    def add(self, y, yhat, live=None):
        """The sums of ``update`` without counting the graphs; ``live``: the {N, B} word of a padded batch, whose ghost
        graphs are left out of the sums."""
        y = y.contiguous()
        T = len(self.levels)
        if yhat.numel() != y.numel() * T:
            raise ValueError(f"predictions {tuple(yhat.shape)} for {y.numel()} labels and {T} levels")
        yhat = yhat.reshape(-1).contiguous().float()
        _lib.call("pert_eval_metrics_q", _lib.ptr(y), _lib.ptr(yhat), self._taus, T, y.numel(), _lib.ptr(self.acc),
                  _lib.ptr(live), _lib.stream())
        ops.LAUNCHES["n"] += 1

    def result(self):
        """-> (mae, mape, quantile loss), each divided by the number of graphs seen, like pert_gnn.py:290-294; with T > 1
        levels each is a T-tuple in level order."""
        a = self.acc.cpu()
        n = max(self.count, 1)
        T = len(self.levels)
        per = [tuple(float(a[4 * t + k]) / n for t in range(T)) for k in range(3)]
        return tuple(per) if T > 1 else tuple(p[0] for p in per)

    def coverage(self):
        """-> T floats: the fraction of the graphs seen whose label is at or below the prediction of each level."""
        a = self.acc.cpu()
        n = max(self.count, 1)
        return tuple(float(a[4 * t + 3]) / n for t in range(len(self.levels)))

    def crossing(self):
        """-> the fraction of the graphs seen whose predicted levels cross (a higher level below a lower one)."""
        return float(self.acc[4 * len(self.levels)].item()) / max(self.count, 1)


@torch.no_grad()
def eval_step(model, data, tau=None, metrics: EvalMetrics | None = None, calibration=None, monotone=False):
    """Loop body of reference pert_gnn.py:260-289 on a device-resident Batch: engine forward (eval mode: BatchNorm
    running statistics), then the sums on the device.  With ``metrics`` the sums are accumulated there and nothing is
    returned to the host; without, returns the device tensor ``EvalMetrics.acc`` (at T = 1: mae, mape, quantile loss
    * B, coverage count, crossing count).  ``calibration`` / ``monotone``: as in ``predict``, applied to the predictions
    before the sums."""
    levels = _calibrated_levels(model, tau, calibration)
    _calibration_on(calibration, data.entry_id.device)
    global_pred, _ = model(*model_inputs(data))
    if calibration is not None or monotone:
        global_pred = global_pred.contiguous()
        _calib_apply(global_pred, data.entry_id, calibration.offsets if calibration is not None else None, monotone)
    m = metrics if metrics is not None else EvalMetrics(global_pred.device, levels)
    m.update(data.y, global_pred)
    return m.acc if metrics is None else None


@torch.no_grad()
def evaluate(model, loader, device, tau=None):
    """reference ``test(loader)`` (pert_gnn.py:254-294): model.eval(), every batch through eval_step, one read-back.
    A model with T > 1 quantile levels gets (mae, mape, qloss) as T-tuples in level order."""
    levels = resolve_tau(model, tau)
    was_training = model.training
    model.eval()
    m = EvalMetrics(device, levels)
    for data in loader:
        eval_step(model, data.to(device), levels, m)
    model.train(was_training)
    return m.result()


def _padded_forward(model, eng, buf):
    """Index build + eval-mode engine forward of a ``PaddedBatch`` -> (global_pred, local_pred, index)."""
    from .index import build_index

    x, cat_X, edge_index, edge_attr, pnn, probs, entry_id, batch = model_inputs(buf)
    index = build_index(edge_index, x.size(0), edge_attr, model.interface_embeds.num_embeddings,
                        model.rpctype_embeds.num_embeddings, check=False)
    gpred, lpred = eng.forward(x, cat_X, entry_id, probs, pnn, batch, index, False, live=buf.live)
    return gpred, lpred, index


@torch.no_grad()
def evaluate_bucketed(model, loader, device, tau=None, max_graphs=32, calibration=None, monotone=False):
    """``evaluate`` (same return) with every batch padded into its capacity bucket and the engine forward + metric sums
    replayed from one CUDA graph per bucket (eager on the first visit, captured on the second; graphs persist across
    calls on the same model, and a graph captured over an engine or workspace that has since been replaced is captured
    again).  Buckets beyond ``max_graphs`` and failed captures run the padded forward eagerly; a batch
    ``PaddedBatch`` cannot pad (per-pattern probabilities only) runs through ``eval_step``.

    ``calibration`` / ``monotone``: as in ``predict``, applied inside the graph before the metric sums.  The graph reads
    a persistent copy of the offset table, one per table shape, refreshed before the loop: calibrations of one shape
    share the graphs and a replay never reads stale offsets.  The table shape and ``monotone`` are part of the key;
    the calls without them keep their own state and graphs."""
    levels = _calibrated_levels(model, tau, calibration)
    calibrated = calibration is not None or monotone
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:      # "cuda" -> "cuda:<current>": the state is kept per device
        device = torch.device("cuda", torch.cuda.current_device())
    _calibration_on(calibration, device)
    was_training = model.training
    model.eval()
    name = "_bucketed_eval_calibrated" if calibrated else "_bucketed_eval"
    st = model.__dict__.get(name)
    if st is None or st.metrics.acc.device != device or st.metrics.levels != levels:
        # the graphs add into these metric sums (and hold the levels by value): new sums, new graphs
        st = model.__dict__[name] = _GraphCache()
        st.metrics = EvalMetrics(device, levels)
        st.tables = {}                                       # offset-table shape -> the table the graphs read
    st.max_graphs = max_graphs
    m = st.metrics
    m.reset()
    eng = model.engine()
    table, shape = None, None
    if calibration is not None:
        shape = tuple(calibration.offsets.shape)
        table = st.tables.get(shape)
        if table is None:
            table = st.tables[shape] = torch.empty(shape, dtype=torch.float32, device=device)
        table.copy_(calibration.offsets)

    def run(buf):
        out = _padded_forward(model, eng, buf)
        if calibrated:
            _calib_apply(out[0], buf.entry_id, table, monotone, live=buf.live)
        m.add(buf.y, out[0], live=buf.live)
        return out

    with torch.cuda.device(device):
        for data in loader:
            data = data.to(device)
            if not PaddedBatch.accepts(data):
                eval_step(model, data, levels, m, calibration, monotone)
                continue
            m.count += int(data.num_graphs)
            bucket, buf = st.pad(data)
            key = bucket + ((shape, bool(monotone)) if calibrated else ())
            st.cache(key, eng, buf.caps, lambda: run(buf), pin=buf)
    model.train(was_training)
    return m.result()


def _predict_cache(model, dev, max_graphs):
    """The graph cache of ``predict`` and ``calibrate``: one graph of the padded eval forward per capacity bucket."""
    st = model.__dict__.get("_bucketed_predict")
    if st is None or st.zero_y.device != dev:
        st = model.__dict__["_bucketed_predict"] = _GraphCache()
        st.zero_y = torch.zeros(0, dtype=torch.int64, device=dev)
    st.max_graphs = max_graphs
    return st


@torch.no_grad()
def predict(model, store, entry_ids, timestamps, batch_size=1024, asof=False, local=False, max_graphs=32, mixes=None,
            overrides=None, scenario_ids=None, calibration=None, monotone=False):
    """Predicted latency of every request (entry ``entry_ids[q]`` at time ``timestamps[q]``, ms) of a pattern store's
    entries: float32 device tensor [Q], in request order (duplicates and any order allowed).  With ``local``, also the
    local (per-node) predictions [sum of the requests' node counts] and ``node_ptr`` [Q+1] (int64), request q owning
    rows node_ptr[q] .. node_ptr[q+1]-1.

    The requests are assembled on the device in slices of ``batch_size`` (``PatternStore.assemble_requests``: the
    exact resource join, or with ``asof`` the newest row at or before the request's time bucket -- with the exact join a
    missing row sets the store's status word, see ``PatternStore.check``), and every slice runs the eval-mode forward
    padded into its capacity bucket, replayed from one CUDA graph per bucket as in ``evaluate_bucketed``.  A model with
    T > 1 quantile levels predicts [Q, T], column t the level-t quantile.  The workspace
    is sized once, on the host, for the largest slice.  Runs in eval mode under ``no_grad`` and restores the training
    flag; BatchNorm statistics, the dropout counter, parameters and optimizer state are left as they were.  A bad entry id
    raises ``PertGnnError`` before any launch.

    What-if prediction: ``mixes``, ``overrides`` and ``scenario_ids`` as in ``PatternStore.assemble_requests`` (per-
    request pattern mixes, resource override rows and each request's scenario, -1 for none), checked on the host and
    uploaded once per call (the override table sorted once); every slice assembles from slices of them.  The slices
    are sized, and ``node_ptr`` set, from the mixes' node counts.  A what-if slice pads into the same capacity buckets
    as a plain one, so it replays the graphs plain calls captured.

    ``calibration`` (a ``Calibration`` of the model's levels, else ``ValueError``) adds each request's entry offsets
    to its levels; ``monotone`` then replaces each row by its running max over the levels, so they never cross.  Either
    runs one ``pert_calib_apply`` launch over the whole result after the slices; without them nothing more is
    launched."""
    _calibrated_levels(model, None, calibration)
    what_if = mixes is not None or overrides is not None or scenario_ids is not None
    bs = int(batch_size)
    if what_if:
        w = store._what_if_arrays(entry_ids, timestamps, mixes, overrides, scenario_ids)
        ent, nodes, edges = w.ent, w.nodes, w.edges
    else:
        ent = store.check_entries(entry_ids)
        ts = np.asarray(timestamps, dtype=np.int64).reshape(-1)
        if ts.shape != ent.shape:
            raise _lib.PertGnnError(f"{ent.shape[0]} entry ids but {ts.shape[0]} timestamps")
        nodes, edges = store._h_ent_nodes[ent], store._h_ent_edges[ent]
    if bs < 1:
        raise _lib.PertGnnError("batch_size must be >= 1")
    Q = int(ent.shape[0])
    dev = store.device
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    _calibration_on(calibration, dev)
    node_ptr = np.zeros(Q + 1, dtype=np.int64)
    np.cumsum(nodes, out=node_ptr[1:])
    was_training = model.training
    model.eval()
    try:
        with torch.cuda.device(dev):
            st = _predict_cache(model, dev, max_graphs)
            if st.zero_y.numel() < min(bs, Q):
                # requests have no label: the pad kernel, which runs eagerly in front of every replay, is the only
                # reader of this zero column, so one buffer serves every bucket
                st.zero_y = torch.zeros(min(bs, Q), dtype=torch.int64, device=dev)
            eng = model.engine()
            T = eng.n_out
            gpred = torch.empty((Q, T) if T > 1 else (Q,), dtype=torch.float32, device=dev)
            lpred = torch.empty(int(node_ptr[-1]), dtype=torch.float32, device=dev) if local else None
            if Q:
                starts = np.arange(0, Q, bs)          # the slices' sizes, exactly: host-only, no device sync
                eng.reserve(*bucket_bound(int(np.add.reduceat(nodes, starts).max()),
                                          int(np.add.reduceat(edges, starts).max()), min(bs, Q)))
                if not what_if:
                    ent_d = torch.from_numpy(ent).to(dev, non_blocking=True)
                    ts_d = torch.from_numpy(ts).to(dev, non_blocking=True)
            for i in range(0, Q, bs):
                j = min(i + bs, Q)
                arrays = w.slice(i, j) if what_if else (ent_d[i:j], ts_d[i:j])
                data = store.assemble_requests(ent[i:j], None, asof=asof, device_arrays=arrays)
                data.y = st.zero_y[:j - i]
                bucket, buf = st.pad(data)
                g, loc, _ = st.cache(bucket, eng, buf.caps, lambda: _padded_forward(model, eng, buf), pin=buf)
                gpred[i:j].copy_(g[:j - i] if T > 1 else g[:j - i, 0])
                if local:
                    lpred[node_ptr[i]:node_ptr[j]].copy_(loc[:node_ptr[j] - node_ptr[i], 0])
            if Q and (calibration is not None or monotone):
                _calib_apply(gpred, w.ent_d if what_if else ent_d,
                             calibration.offsets if calibration is not None else None, monotone)
    finally:
        model.train(was_training)
    if not local:
        return gpred
    return gpred, lpred, torch.from_numpy(node_ptr).to(dev)


# ------------------------------------------------------------------------------------------ conformal calibration
CALIBRATION_GROUPINGS = ("entry", "global")


def _calibrated_levels(model, tau, calibration):
    """``resolve_tau(model, tau)``; with a calibration, ``tau`` None means the calibration's levels, and the levels
    must equal them (``ValueError``)."""
    if calibration is None:
        return resolve_tau(model, tau)
    if not isinstance(calibration, Calibration):
        raise TypeError(f"calibration must be a Calibration, got {type(calibration).__name__}")
    levels = resolve_tau(model, calibration.levels if tau is None else tau)
    if levels != calibration.levels:
        raise ValueError(f"the calibration's levels {calibration.levels} differ from the levels {levels}")
    if not calibration.offsets.is_cuda:
        raise _lib.PertGnnError("the calibration's tensors are on the host (no CPU fallback for the apply): move them "
                                "with Calibration.to(device)")
    return levels


def _calibration_on(calibration, device):
    """``PertGnnError`` unless ``calibration`` (or None) is on ``device``, where the predictions are."""
    if calibration is not None and calibration.device != torch.device(device):
        raise _lib.PertGnnError(f"the calibration is on {calibration.device}, the predictions on {device}: move it "
                                "with Calibration.to(device)")


def _calib_apply(yhat, group, off, monotone, live=None):
    """``pert_calib_apply`` in place on the contiguous predictions ``yhat`` [Q, T] ([Q] at T = 1): + the offset row of
    each group id ``group`` [Q] (ids outside the table read its last, global row), then the running max.  Every tensor
    must be on yhat's CUDA device (``PertGnnError`` before the launch)."""
    T = yhat.size(1) if yhat.dim() == 2 else 1
    if off is not None and off.size(1) != T:
        raise ValueError(f"an offset table of {off.size(1)} levels for predictions of {T}")
    if not yhat.is_cuda or any(t is not None and t.device != yhat.device for t in (group, off, live)):
        raise _lib.PertGnnError("pert_calib_apply: the predictions, entry ids, offsets and live word must be on one "
                                "CUDA device")
    _lib.call("pert_calib_apply", _lib.ptr(yhat), _lib.ptr(group), yhat.size(0), T, _lib.ptr(off),
              off.size(0) if off is not None else 0, int(bool(monotone)), _lib.ptr(live), _lib.stream())
    ops.LAUNCHES["n"] += 1


def min_calibration_size(tau):
    """The fewest graphs a split-conformal offset at level ``tau`` needs: the least n with ceil((n + 1) tau) <= n
    (None for tau = 1, which no finite set reaches)."""
    tau = float(tau)
    if tau >= 1.0:
        return None
    n = max(1, int(tau / (1.0 - tau)) - 1)
    while max(1, math.ceil((n + 1) * tau)) > n:
        n += 1
    return n


class Calibration:
    """Split-conformal offsets of a quantile model (conformalized quantile regression): ``offsets`` [G + 1, T] fp32,
    ``counts`` [G + 1] int32 and ``own`` [G + 1, T] int8 on the device, row g of entry id g and the last row the global
    group of every calibration graph.  For level tau and a group of n_g graphs, the offset is the k-th smallest score
    y - yhat of the group, k = max(1, ceil((n_g + 1) tau)), when k <= n_g and n_g >= ``min_count`` (``own`` = 1), else
    the global row's.  Then P(y <= yhat + offset) >= tau for a new request exchangeable with the calibration set, per
    entry for the entries with their own offset.

    Built by ``fit`` (or ``calibrate``), or from the three tensors, so that ``torch.save`` of them and of ``levels`` is
    all a caller needs to keep one.  ``predict``, ``eval_step`` and ``evaluate_bucketed`` take it as ``calibration=``."""

    def __init__(self, levels, offsets, counts, own, by="entry", min_count=1):
        self.levels = _as_levels(levels)
        if by not in CALIBRATION_GROUPINGS:
            raise ValueError(f"by must be one of {CALIBRATION_GROUPINGS}, got {by!r}")
        T = len(self.levels)
        if offsets.dim() != 2 or offsets.size(1) != T or offsets.size(0) < 1 or offsets.dtype != torch.float32:
            raise ValueError(f"offsets must be float32 [G + 1, {T}], got {offsets.dtype} {tuple(offsets.shape)}")
        if tuple(counts.shape) != (offsets.size(0),) or tuple(own.shape) != tuple(offsets.shape):
            raise ValueError(f"counts {tuple(counts.shape)} and own {tuple(own.shape)} do not match offsets "
                             f"{tuple(offsets.shape)}")
        if counts.device != offsets.device or own.device != offsets.device:
            raise ValueError("offsets, counts and own must be on one device")
        self.offsets, self.counts, self.own = offsets.contiguous(), counts, own
        self.by, self.min_count = by, int(min_count)

    def to(self, device):
        """This calibration with its tensors on ``device`` (e.g. after ``torch.load(..., map_location="cpu")``)."""
        return Calibration(self.levels, self.offsets.to(device), self.counts.to(device), self.own.to(device), self.by,
                           self.min_count)

    @property
    def n_groups(self):
        return self.offsets.size(0) - 1

    @property
    def device(self):
        return self.offsets.device

    @classmethod
    @_lib.on_device_of
    def fit(cls, y, yhat, entry_ids, levels, n_groups, by="entry", min_count=1):
        """Offsets from labels ``y`` [n] (int64), predictions ``yhat`` [n, T] ([n] at T = 1) and the graphs' entry ids
        ``entry_ids`` [n] (int64; ignored with ``by="global"``, which fits the global row only), all on one CUDA device,
        for ``n_groups`` entry ids.  Checked on the host, one ``pert_calib_offsets`` launch sequence, then one read of
        the status word.  ``ValueError`` for bad levels, shapes or ``by``, and for a set too small for a level (naming
        the least n); ``PertGnnError`` for a NaN or infinite prediction or an entry id outside [0, n_groups)."""
        levels = _as_levels(levels)
        T = len(levels)
        if by not in CALIBRATION_GROUPINGS:
            raise ValueError(f"by must be one of {CALIBRATION_GROUPINGS}, got {by!r}")
        if not 1 <= T <= _lib.MAX_QUANTILES:
            raise ValueError(f"1 to {_lib.MAX_QUANTILES} levels, got {T}")
        if any(not 0.0 <= t <= 1.0 for t in levels) or any(b <= a for a, b in zip(levels, levels[1:])):
            raise ValueError(f"levels must be strictly increasing in [0, 1], got {levels}")
        if operator.index(min_count) < 1:
            raise ValueError(f"min_count must be >= 1, got {min_count}")
        G = operator.index(n_groups) if by == "entry" else 0
        if G < 0:
            raise ValueError(f"n_groups must be >= 0, got {n_groups}")
        n = int(y.numel())
        if n < 1:
            raise ValueError("no calibration graphs")
        if yhat.numel() != n * T or (yhat.dim() == 2 and yhat.size(1) != T):
            raise ValueError(f"predictions {tuple(yhat.shape)} for {n} labels and {T} levels")
        for tau in levels:
            need = min_calibration_size(tau)
            if need is None or n < need:
                raise ValueError(f"{n} calibration graphs cannot give a conformal offset at level {tau}: it needs "
                                 + ("a finite set below 1" if need is None else f"at least n = {need}"))
        if by == "entry" and (entry_ids is None or entry_ids.numel() != n):
            raise ValueError(f"by='entry' needs one entry id per graph ({n})")
        if not (y.is_cuda and yhat.is_cuda) or y.device != yhat.device:
            raise _lib.PertGnnError("Calibration.fit needs the labels and predictions on one CUDA device")
        dev = y.device
        y = y.to(torch.int64).contiguous()
        yhat = yhat.reshape(n, T).to(torch.float32).contiguous()
        group = None
        if by == "entry":
            group = entry_ids.to(dev, torch.int64).contiguous()
        ws_bytes = _lib.lib().pert_calib_workspace_bytes(n, T, G)
        if ws_bytes < 0:
            raise ValueError(f"{n} graphs, {T} levels and {G} groups exceed the fit's sizes (n T < 2^31)")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        off = torch.empty(G + 1, T, dtype=torch.float32, device=dev)
        counts = torch.empty(G + 1, dtype=torch.int32, device=dev)
        own = torch.empty(G + 1, T, dtype=torch.int8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.call("pert_calib_offsets", _lib.ptr(y), _lib.ptr(yhat), _lib.ptr(group), n, T,
                  (C.c_double * T)(*levels), G, int(min_count), _lib.ptr(off), _lib.ptr(counts), _lib.ptr(own),
                  _lib.ptr(ws), ws_bytes, _lib.ptr(status), _lib.stream())
        ops.LAUNCHES["n"] += 1
        if int(status.item()) != 0:
            # the error path only: name the cause
            if not bool(torch.isfinite(y.float().reshape(n, 1) - yhat).all()):
                raise _lib.PertGnnError("Calibration.fit: a NaN or infinite score y - yhat (a NaN or infinite "
                                        "prediction)")
            raise _lib.PertGnnError(f"Calibration.fit: an entry id outside [0, {G})")
        return cls(levels, off, counts, own, by, min_count)


def _replayed_predictions(model, loader, device, max_graphs, caller):
    """-> the labels [n] (int64), predictions [n, T] and entry ids [n] (int64) of every batch of ``loader``, in loader
    order, on ``device``.  Every batch runs the padded, graph-replayed eval forward of ``predict`` (the same graph
    cache); a batch ``PaddedBatch`` cannot pad runs the eval forward eagerly.  Runs in eval mode under ``no_grad`` and
    restores the training flag.  ``ValueError`` naming ``caller`` when the loader yields nothing."""
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    ys, preds, ents = [], [], []
    was_training = model.training
    model.eval()
    try:
        with torch.cuda.device(device):
            st = _predict_cache(model, device, max_graphs)
            eng = model.engine()
            for data in loader:
                data = data.to(device)
                B = int(data.num_graphs)
                if PaddedBatch.accepts(data):
                    bucket, buf = st.pad(data)
                    g, _, _ = st.cache(bucket, eng, buf.caps, lambda: _padded_forward(model, eng, buf), pin=buf)
                else:
                    g, _ = model(*model_inputs(data))
                preds.append(g[:B].clone())         # a replay rewrites the graph's output
                ys.append(data.y.reshape(-1).to(torch.int64))
                ents.append(data.entry_id.reshape(-1).to(torch.int64))
    finally:
        model.train(was_training)
    if not ys:
        raise ValueError(f"{caller}: the loader yielded no batches")
    return torch.cat(ys), torch.cat(preds), torch.cat(ents)


@torch.no_grad()
def calibrate(model, loader, device, tau=None, by="entry", min_count=1, max_graphs=32):
    """Fits a ``Calibration`` of ``model`` on the labelled held-out batches of ``loader`` (e.g. a ``StoreLoader`` over
    held-out trace ids): every batch runs the padded, graph-replayed eval forward of ``predict`` (the same graph
    cache), its real rows' labels, predictions and entry ids are copied out on the device, and ``Calibration.fit``
    runs once over all of them with ``n_groups = model.entry_embeds.num_embeddings``.  The levels are
    ``resolve_tau(model, tau)``: a model trained at one level is calibrated at the ``tau`` it was trained with.  Runs
    in eval mode under ``no_grad`` and restores the training flag; BatchNorm statistics, the dropout counter, parameters
    and optimizer state are left as they were.  A batch ``PaddedBatch`` cannot pad runs the eval forward eagerly."""
    levels = resolve_tau(model, tau)
    y, yhat, ents = _replayed_predictions(model, loader, device, max_graphs, "calibrate")
    if yhat.size(1) != len(levels):
        raise ValueError(f"{len(levels)} levels for a head of {yhat.size(1)} outputs")
    return Calibration.fit(y, yhat, ents, levels, model.entry_embeds.num_embeddings, by=by, min_count=min_count)


# ------------------------------------------------------------------------------ conformal predictive distribution
class ScoreDistribution:
    """The split-conformal predictive distribution of a model's predictions around one base column (level ``level``):
    the held-out scores s = (float)y - yhat in fp32 (-0 -> +0), sorted per entry.  ``scores`` [ptr[-1]] fp32 and
    ``ptr`` [G + 2] int64 on the device: row g (0 <= g < G) holds entry g's scores at scores[ptr[g] .. ptr[g+1]), row
    G all n of them.  A query of entry g reads row g iff it has at least ``min_count`` (>= 1) scores, else row G; an id
    outside [0, G) -- an entry added after the fit -- reads row G.

    For a request with prediction yhat, in the row of m scores read:
    * ``tail``: with c = fl(x - yhat), lo = #{s > c} / (m + 1) and hi = (#{s >= c} + 1) / (m + 1) bracket
      P(latency > x); hi is the conservative SLO-violation probability.
    * ``pvalues``: hi at the observed latency y, the conformal p-value: for a trace exchangeable with the held-out set,
      P(p <= alpha) <= alpha (per entry for the entries on their own row).
    * ``quantile``: at any level tau, fl(yhat + s_(k)), k = max(1, ceil((m + 1) tau)), with the own-row rule of
      ``Calibration`` (k <= n_g and n_g >= min_count, else row G); +inf where k exceeds even row G's n.  At a level
      ``Calibration.fit`` accepts this equals its offset added by ``predict(calibration=...)``, bit for bit.

    Built by ``fit`` (or ``fit_distribution``), or from the two tensors, so that ``torch.save`` of them, ``level``,
    ``by``, ``min_count`` and ``column`` is all a caller needs to keep one.  ``column`` is the base column of a [Q, T]
    prediction (the index of ``level`` among a quantile model's levels).

    A sliding window: fitted with ``ts=`` (the graphs' store buckets, ``store.t["trace_ts"][ids]``), a distribution
    keeps a log of its graphs in insertion order, ``log = (y int64, yhat float32 (the base column), entry int64, ts
    int64)``, each [n] on the table's device (``log_y`` .. ``log_ts``; None without a log; pass ``log=`` to the
    constructor to keep one across ``torch.save``).  ``insert`` adds labelled graphs, ``evict(before)`` drops the logged
    graphs with ts < before (the cut of ``PatternStore.evict_traces``) and ``add_traces`` scores store traces, returns
    their p-values and inserts them.  Each update is one fit of the change and one merge on the GPU, and after any
    sequence of them ``scores`` and ``ptr`` equal, bit for bit, ``fit(log_y, log_yhat, log_entry, n_groups, ...)``.  The
    window is valid for one set of model parameters: after fine-tuning, fit again."""

    def __init__(self, level, scores, ptr, by="entry", min_count=1, column=0, *, log=None):
        self.level = float(level)
        if not 0.0 <= self.level <= 1.0:
            raise ValueError(f"level must be in [0, 1], got {level}")
        if by not in CALIBRATION_GROUPINGS:
            raise ValueError(f"by must be one of {CALIBRATION_GROUPINGS}, got {by!r}")
        if operator.index(min_count) < 1:
            raise ValueError(f"min_count must be >= 1, got {min_count}")
        if operator.index(column) < 0:
            raise ValueError(f"column must be >= 0, got {column}")
        if scores.dim() != 1 or scores.dtype != torch.float32 or scores.numel() < 1:
            raise ValueError(f"scores must be float32 [n], got {scores.dtype} {tuple(scores.shape)}")
        if ptr.dim() != 1 or ptr.dtype != torch.int64 or ptr.numel() < 2:
            raise ValueError(f"ptr must be int64 [G + 2], got {ptr.dtype} {tuple(ptr.shape)}")
        if ptr.device != scores.device:
            raise ValueError("scores and ptr must be on one device")
        self.scores, self.ptr = scores.contiguous(), ptr.contiguous()
        self.by, self.min_count, self.column = by, int(min_count), int(column)
        self.log = None
        if log is not None:
            if not isinstance(log, (tuple, list)) or len(log) != 4 or not all(torch.is_tensor(t) for t in log):
                raise ValueError("log must be four tensors (y, yhat, entry, ts)")
            n = log[0].numel()
            want = (torch.int64, torch.float32, torch.int64, torch.int64)
            if any(t.dim() != 1 or t.numel() != n or t.dtype != d for t, d in zip(log, want)):
                raise ValueError("log must be y int64, yhat float32, entry int64 and ts int64, each [n], got "
                                 + ", ".join(f"{t.dtype} {tuple(t.shape)}" for t in log))
            if n * (2 if by == "entry" else 1) != self.scores.numel():
                raise ValueError(f"a log of {n} graphs for a table of {self.scores.numel()} scores")
            if any(t.device != self.scores.device for t in log):
                raise ValueError("the log must be on the table's device")
            self.log = tuple(t.contiguous() for t in log)

    def to(self, device):
        """This distribution with its tensors on ``device`` (e.g. after ``torch.load(..., map_location="cpu")``)."""
        return ScoreDistribution(self.level, self.scores.to(device), self.ptr.to(device), self.by, self.min_count,
                                 self.column, log=None if self.log is None else tuple(t.to(device) for t in self.log))

    log_y = property(lambda self: None if self.log is None else self.log[0])
    log_yhat = property(lambda self: None if self.log is None else self.log[1])
    log_entry = property(lambda self: None if self.log is None else self.log[2])
    log_ts = property(lambda self: None if self.log is None else self.log[3])

    @property
    def n_groups(self):
        return self.ptr.numel() - 2

    @property
    def device(self):
        return self.scores.device

    @property
    def counts(self):
        """int64 [G + 1]: the scores of each entry's row, then of the global row."""
        return self.ptr[1:] - self.ptr[:-1]

    @classmethod
    @_lib.on_device_of
    def fit(cls, y, yhat, entry_ids, n_groups, level, by="entry", min_count=1, column=None, ts=None):
        """The distribution of labels ``y`` [n] (int64) around predictions ``yhat`` [n], or column ``column`` of
        ``yhat`` [n, T] (``column`` may be left out at T = 1), with the graphs' entry ids ``entry_ids`` [n] (int64;
        ignored with ``by="global"``, which keeps the global row only), all on one CUDA device, for ``n_groups`` entry
        ids.  ``level`` names the base column's level.  Checked on the host, one ``pert_cpd_fit`` launch sequence, then
        one read of the status word.  ``ValueError`` for bad shapes, ``level``, ``by``, ``min_count`` or ``column``;
        ``PertGnnError`` for host tensors, a NaN or infinite prediction or an entry id outside [0, n_groups).  With
        ``ts`` [n] (int64, the graphs' store buckets) the distribution keeps a log of its graphs, in this order, for
        ``insert`` / ``evict``."""
        level = float(level)
        if not 0.0 <= level <= 1.0:
            raise ValueError(f"level must be in [0, 1], got {level}")
        if by not in CALIBRATION_GROUPINGS:
            raise ValueError(f"by must be one of {CALIBRATION_GROUPINGS}, got {by!r}")
        if operator.index(min_count) < 1:
            raise ValueError(f"min_count must be >= 1, got {min_count}")
        G = operator.index(n_groups) if by == "entry" else 0
        if G < 0:
            raise ValueError(f"n_groups must be >= 0, got {n_groups}")
        n = int(y.numel())
        if n < 1:
            raise ValueError("no held-out graphs")
        if yhat.dim() not in (1, 2) or yhat.size(0) != n:
            raise ValueError(f"predictions {tuple(yhat.shape)} for {n} labels: [n] or [n, T]")
        T = yhat.size(1) if yhat.dim() == 2 else 1
        if column is None:
            if T > 1:
                raise ValueError(f"predictions of {T} levels: name the base column with column=")
            column = 0
        if not 0 <= operator.index(column) < T:
            raise ValueError(f"column {column} outside the {T} columns of the predictions")
        if by == "entry" and (entry_ids is None or entry_ids.numel() != n):
            raise ValueError(f"by='entry' needs one entry id per graph ({n})")
        _check_ts(ts, n)
        if not (y.is_cuda and yhat.is_cuda) or y.device != yhat.device:
            raise _lib.PertGnnError("ScoreDistribution.fit needs the labels and predictions on one CUDA device")
        dev = y.device
        if ts is not None and ts.device != dev:
            raise _lib.PertGnnError(f"the buckets ts must be on {dev}, with the labels")
        y = y.to(torch.int64).contiguous()
        yhat = yhat.reshape(n, T).to(torch.float32).contiguous()
        group = entry_ids.to(dev, torch.int64).contiguous() if by == "entry" else None
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        scores, ptr = _cpd_fit(y, yhat, T, int(column), group, n, G, status)
        ops.LAUNCHES["n"] += 1
        if int(status.item()) != 0:
            _raise_fit_error("fit", y, yhat[:, column], G)
        log = None
        if ts is not None:
            ent = (entry_ids.to(dev, torch.int64).reshape(-1) if entry_ids is not None and entry_ids.numel() == n
                   else torch.zeros(n, dtype=torch.int64, device=dev))
            log = (y, yhat[:, column].contiguous(), ent.contiguous(), ts.reshape(-1).contiguous())
        return cls(level, scores, ptr, by, min_count, column, log=log)

    # ---------------------------------------------------------------------------------------- sliding-window updates
    def _delta(self, y, yhat, entry_ids, ts, what):
        """-> (y int64, yhat [k] fp32 base column, entry int64, ts int64) of graphs to insert, checked on the host as
        ``fit`` checks them; ``PertGnnError`` for tensors on the host or on another device than the table."""
        if self.log is None:
            raise ValueError(f"ScoreDistribution.{what} needs a log: fit with ts=")
        if not torch.is_tensor(y) or not torch.is_tensor(yhat):
            raise ValueError("labels and predictions must be tensors")
        k = int(y.numel())
        if k < 1:
            raise ValueError("no graphs to insert")
        if yhat.dim() not in (1, 2) or yhat.size(0) != k:
            raise ValueError(f"predictions {tuple(yhat.shape)} for {k} labels: [k] or [k, T]")
        if yhat.dim() == 2 and yhat.size(1) > 1 and self.column >= yhat.size(1):
            raise ValueError(f"predictions of {yhat.size(1)} levels have no base column {self.column}")
        if self.by == "entry" and (entry_ids is None or entry_ids.numel() != k):
            raise ValueError(f"by='entry' needs one entry id per graph ({k})")
        _check_ts(ts, k, required=True)
        dev = self.device
        if not self.scores.is_cuda:
            raise _lib.PertGnnError("the distribution's tensors are on the host: move them with "
                                    "ScoreDistribution.to(device)")
        for name, t in (("labels", y), ("predictions", yhat), ("entry ids", entry_ids), ("buckets ts", ts)):
            if t is not None and t.device != dev:
                raise _lib.PertGnnError(f"the {name} must be on {dev}, where the distribution is")
        col = self.column if yhat.dim() == 2 and yhat.size(1) > 1 else 0
        yh = yhat.reshape(k, -1)[:, col].to(torch.float32).contiguous()
        ent = (entry_ids.reshape(-1).to(torch.int64).contiguous() if entry_ids is not None and entry_ids.numel() == k
               else torch.zeros(k, dtype=torch.int64, device=dev))
        return y.reshape(-1).to(torch.int64).contiguous(), yh, ent, ts.reshape(-1).contiguous()

    def _merged(self, y, yh, ent, G_new, sign, status):
        """The fit of the changed graphs (G_new groups) merged into (sign = +1) or out of (-1) the table: new
        (scores, ptr) tensors; the table is not touched.  Two launch sequences, no read of the status."""
        k = y.numel()
        group = ent if self.by == "entry" else None
        d_scores, d_ptr = _cpd_fit(y, yh, 1, 0, group, k, G_new, status)
        n_old, n_d = self.scores.numel(), d_scores.numel()
        ws_bytes = _lib.lib().pert_cpd_merge_workspace_bytes(self.n_groups, G_new, n_old, n_d)
        if ws_bytes < 0:
            raise ValueError(f"a table of {n_old} scores and {n_d} more exceed the fit's sizes (n < 2^30)")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        scores = torch.empty(n_old + sign * n_d, dtype=torch.float32, device=self.device)
        ptr = torch.empty(G_new + 2, dtype=torch.int64, device=self.device)
        _lib.call("pert_cpd_merge", _lib.ptr(self.scores), _lib.ptr(self.ptr), self.n_groups, n_old,
                  _lib.ptr(d_scores), _lib.ptr(d_ptr), G_new, n_d, sign, _lib.ptr(scores), _lib.ptr(ptr),
                  _lib.ptr(ws), ws_bytes, _lib.ptr(status), _lib.stream())
        ops.LAUNCHES["n"] += 2
        return scores, ptr

    def insert(self, y, yhat, entry_ids, ts, n_groups=None):
        """Adds labelled graphs to the window: labels ``y`` [k], predictions ``yhat`` [k] or [k, T] (the base column
        is taken, as in the queries), entry ids [k] (ignored with ``by="global"``) and buckets ``ts`` [k] (int64), on
        the table's device.  ``n_groups`` may grow the entry rows (ids from ``grow_embeddings``); it never shrinks them
        (``ValueError``).  One fit of the k graphs and one merge on the GPU, one status read; the new tensors replace
        the old ones only when it reads 0.  ``PertGnnError`` for a NaN or infinite score or an entry id outside [0,
        n_groups), and the distribution is left as it was."""
        G = self.n_groups
        G_new = G if n_groups is None or self.by == "global" else operator.index(n_groups)
        if G_new < G:
            raise ValueError(f"n_groups {G_new} would shrink the table's {G} entry rows")
        y, yh, ent, ts = self._delta(y, yhat, entry_ids, ts, "insert")
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            scores, ptr = self._merged(y, yh, ent, G_new, 1, status)
        if int(status.item()) != 0:
            _raise_fit_error("insert", y, yh, G_new)
        self.scores, self.ptr = scores, ptr
        self.log = tuple(torch.cat([a, b]) for a, b in zip(self.log, (y, yh, ent, ts)))

    def evict(self, before):
        """Drops every logged graph whose bucket is ``< before`` from the log and the table (the cut of
        ``PatternStore.evict_traces``), and returns how many.  The evicted log rows are fitted again (the same fp32
        scores) and removed in one merge on the GPU; the kept rows keep their order.  ``ValueError`` without a log or
        when nothing would be left; ``PertGnnError`` when the log's scores are not in the table (a log that does not
        belong to it).  A failed evict leaves the distribution as it was."""
        if self.log is None:
            raise ValueError("ScoreDistribution.evict needs a log: fit with ts=")
        y, yh, ent, ts = self.log
        drop = ts < int(before)
        k, n = int(drop.sum()), ts.numel()                # the one host read of the split
        if k == 0:
            return 0
        if k == n:
            raise ValueError(f"evicting all {n} logged graphs would leave the distribution without a score")
        if not self.scores.is_cuda:
            raise _lib.PertGnnError("the distribution's tensors are on the host: move them with "
                                    "ScoreDistribution.to(device)")
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            out, kept = torch.nonzero(drop).reshape(-1), torch.nonzero(~drop).reshape(-1)     # ascending: stable
            scores, ptr = self._merged(y[out], yh[out], ent[out], self.n_groups, -1, status)
        if int(status.item()) != 0:
            raise _lib.PertGnnError("ScoreDistribution.evict: the evicted scores are not all in the table (a log that "
                                    "does not belong to it)")
        self.scores, self.ptr = scores, ptr
        self.log = tuple(t[kept] for t in self.log)
        return k

    @torch.no_grad()
    def add_traces(self, model, store, ids, evict_before=None, max_graphs=32, batch_size=1024):
        """The online anomaly detector: runs the labelled store traces ``ids`` through the graph-replayed eval forward
        of ``fit_distribution`` (an unshuffled ``StoreLoader``), returns their conformal p-values (float64 [len(ids)])
        against the window as it stood before them, then inserts them with their buckets ``store.t["trace_ts"][ids]``
        and ``n_groups = max(n_groups, model.entry_embeds.num_embeddings)``, and last evicts ``evict_before`` if given.
        One forward, one ``pert_cpd_tail`` launch and one update; if the update fails the distribution is left as it
        was.  The window is valid for one set of model parameters: after fine-tuning, fit again."""
        from .store import StoreLoader

        if self.log is None:
            raise ValueError("ScoreDistribution.add_traces needs a log: fit with ts=")
        if not self.scores.is_cuda:
            raise _lib.PertGnnError("the distribution's tensors are on the host: move them with "
                                    "ScoreDistribution.to(device)")
        ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        y, yhat, ents = _replayed_predictions(model, StoreLoader(store, ids, batch_size), self.device, max_graphs,
                                              "add_traces")
        p = self.pvalues(yhat, ents, y)
        ts = store.t["trace_ts"][torch.from_numpy(ids).to(store.t["trace_ts"].device)].to(self.device)
        old = (self.scores, self.ptr, self.log)
        try:
            self.insert(y, yhat, ents, ts, n_groups=max(self.n_groups, model.entry_embeds.num_embeddings))
            if evict_before is not None:
                self.evict(evict_before)
        except BaseException:
            self.scores, self.ptr, self.log = old
            raise
        return p

    def _operands(self, yhat, entry_ids):
        """-> (yhat, ld, col, group, Q) for a query, or ``PertGnnError`` / ``ValueError`` before any launch."""
        if not self.scores.is_cuda:
            raise _lib.PertGnnError("the distribution's tensors are on the host (no CPU fallback for the queries): "
                                    "move them with ScoreDistribution.to(device)")
        if not torch.is_tensor(yhat) or yhat.device != self.device:
            raise _lib.PertGnnError(f"the predictions must be a tensor on {self.device}, where the distribution is")
        if entry_ids is not None and (not torch.is_tensor(entry_ids) or entry_ids.device != self.device):
            raise _lib.PertGnnError(f"the entry ids must be a tensor on {self.device}, where the distribution is")
        if yhat.dim() not in (1, 2):
            raise ValueError(f"predictions {tuple(yhat.shape)}: [Q] or [Q, T]")
        Q = yhat.size(0)
        yhat = yhat.to(torch.float32)
        if yhat.dim() == 2:
            if self.column >= yhat.size(1):
                raise ValueError(f"predictions of {yhat.size(1)} levels have no base column {self.column}")
            if yhat.stride(1) != 1 or yhat.stride(0) < yhat.size(1):
                yhat = yhat.contiguous()
            ld, col = max(yhat.stride(0), 1), self.column
        else:
            if yhat.stride(0) < 1:
                yhat = yhat.contiguous()
            ld, col = max(yhat.stride(0), 1), 0
        group = None
        if entry_ids is not None:
            if entry_ids.numel() != Q:
                raise ValueError(f"{entry_ids.numel()} entry ids for {Q} predictions")
            group = entry_ids.reshape(-1).to(torch.int64).contiguous()
        return yhat, ld, col, group, Q

    def _check(self, status, what):
        if int(status.item()) != 0:
            raise _lib.PertGnnError(f"ScoreDistribution.{what}: a NaN threshold, label or prediction")

    def _tail_counts(self, yhat, entry_ids, x=None, y=None):
        """-> (ge, gt [Q, S] int32, row [Q] int32, shape of the result) from one pert_cpd_tail launch and one status
        read; ``x`` as in ``tail``, or the labels ``y`` [Q]."""
        yhat, ld, col, group, Q = self._operands(yhat, entry_ids)
        dev = self.device
        if x is not None:
            if not torch.is_tensor(x):
                x = torch.tensor(float(x), dtype=torch.float32, device=dev)
            elif x.device != dev:
                raise _lib.PertGnnError(f"the thresholds must be on {dev}, where the distribution is")
            if x.dim() > 2 or (x.dim() and x.size(0) != Q):
                raise ValueError(f"thresholds {tuple(x.shape)} for {Q} predictions: a number, [Q] or [Q, S]")
            shape = (Q,) if x.dim() < 2 else (Q, x.size(1))
            x = (x.reshape(Q, -1) if x.dim() else x.reshape(1, 1).expand(Q, 1)).to(torch.float32).contiguous()
            S = x.size(1)
        else:
            if not torch.is_tensor(y) or y.device != dev:
                raise _lib.PertGnnError(f"the labels must be a tensor on {dev}, where the distribution is")
            if y.numel() != Q:
                raise ValueError(f"{y.numel()} labels for {Q} predictions")
            y = y.reshape(-1).to(torch.int64).contiguous()
            shape, S = (Q,), 1
        ge = torch.empty(Q, S, dtype=torch.int32, device=dev)
        gt = torch.empty(Q, S, dtype=torch.int32, device=dev)
        row = torch.empty(Q, dtype=torch.int32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.call("pert_cpd_tail", _lib.ptr(self.scores), _lib.ptr(self.ptr), self.n_groups, self.min_count,
                      _lib.ptr(yhat), ld, col, _lib.ptr(group), Q, _lib.ptr(x), S, _lib.ptr(y), _lib.ptr(ge),
                      _lib.ptr(gt), _lib.ptr(row), _lib.ptr(status), _lib.stream())
        ops.LAUNCHES["n"] += 1
        self._check(status, "tail" if y is None else "pvalues")
        return ge, gt, row, shape

    def tail(self, yhat, entry_ids, x):
        """-> (lo, hi) float64 bracketing P(latency > x) for every request: predictions ``yhat`` [Q] or [Q, T] (what
        ``predict`` returns, plain or what-if; the base column is taken from [Q, T]), entry ids [Q] (None: every request
        reads the global row) and thresholds ``x`` (ms): a number or 0-d tensor for all, [Q] per request (-> [Q]) or
        [Q, S] per request and tier (-> [Q, S]).  Tensors must be on the distribution's device (``PertGnnError``)."""
        ge, gt, row, shape = self._tail_counts(yhat, entry_ids, x=x)
        m1 = (self.counts[row.long()] + 1).double().reshape(-1, 1)
        return (gt.double() / m1).reshape(shape), ((ge.double() + 1) / m1).reshape(shape)

    def pvalues(self, yhat, entry_ids, y):
        """-> float64 [Q]: the conformal p-value (#{s >= fl(y - yhat)} + 1) / (m + 1) of every observed latency ``y``
        [Q] (int64 ms) given its prediction and entry, as in ``tail``.  Small p flags an abnormally slow trace: flag at
        p <= alpha for a false-alarm rate of at most alpha."""
        ge, _, row, _ = self._tail_counts(yhat, entry_ids, y=y)
        return (ge[:, 0].double() + 1) / (self.counts[row.long()] + 1).double()

    def quantile(self, yhat, entry_ids, levels):
        """-> float32 [Q, L]: the conformal quantile of every request at each of ``levels`` (1 to 8, strictly
        increasing in [0, 1]), chosen at query time; +inf where no finite conformal bound exists."""
        levels = _as_levels(levels)
        if not 1 <= len(levels) <= _lib.MAX_QUANTILES:
            raise ValueError(f"1 to {_lib.MAX_QUANTILES} levels, got {len(levels)}")
        if any(not 0.0 <= t <= 1.0 for t in levels) or any(b <= a for a, b in zip(levels, levels[1:])):
            raise ValueError(f"levels must be strictly increasing in [0, 1], got {levels}")
        yhat, ld, col, group, Q = self._operands(yhat, entry_ids)
        L = len(levels)
        out = torch.empty(Q, L, dtype=torch.float32, device=self.device)
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("pert_cpd_quantile", _lib.ptr(self.scores), _lib.ptr(self.ptr), self.n_groups, self.min_count,
                      _lib.ptr(yhat), ld, col, _lib.ptr(group), Q, (C.c_double * L)(*levels), L, _lib.ptr(out),
                      _lib.ptr(status), _lib.stream())
        ops.LAUNCHES["n"] += 1
        self._check(status, "quantile")
        return out


def _check_ts(ts, n, required=False):
    """``ValueError`` unless ``ts`` is an int64 tensor of ``n`` buckets (or None when not ``required``)."""
    if ts is None and not required:
        return
    if not torch.is_tensor(ts) or ts.dtype != torch.int64 or ts.numel() != n:
        got = f"{ts.dtype} {tuple(ts.shape)}" if torch.is_tensor(ts) else type(ts).__name__
        raise ValueError(f"ts must be int64 [{n}] (one store bucket per graph), got {got}")


def _cpd_fit(y, yhat, ld, col, group, n, G, status):
    """-> (scores, ptr): one ``pert_cpd_fit`` launch sequence into new tensors; the caller reads ``status``."""
    dev = y.device
    ws_bytes = _lib.lib().pert_cpd_workspace_bytes(n, G)
    if ws_bytes < 0:
        raise ValueError(f"{n} graphs and {G} groups exceed the fit's sizes (n < 2^30)")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    scores = torch.empty(2 * n if group is not None else n, dtype=torch.float32, device=dev)
    ptr = torch.empty(G + 2, dtype=torch.int64, device=dev)
    _lib.call("pert_cpd_fit", _lib.ptr(y), _lib.ptr(yhat), ld, col, _lib.ptr(group), n, G, _lib.ptr(scores),
              _lib.ptr(ptr), _lib.ptr(ws), ws_bytes, _lib.ptr(status), _lib.stream())
    return scores, ptr


def _raise_fit_error(what, y, yhat_col, G):
    """The error path of a fit whose status is set: name the cause."""
    if not bool(torch.isfinite(y.float() - yhat_col).all()):
        raise _lib.PertGnnError(f"ScoreDistribution.{what}: a NaN or infinite score y - yhat (a NaN or infinite "
                                "prediction)")
    raise _lib.PertGnnError(f"ScoreDistribution.{what}: an entry id outside [0, {G})")


def _base_level(model, level):
    """-> (level, column) of a distribution of ``model``'s predictions: ``level`` None is the model's only level; on a
    model of T > 1 levels ``level`` must be one of them (``ValueError``)."""
    q = getattr(model, "quantiles", None)
    if q is not None and len(q) > 1:
        if level is None or float(level) not in q:
            raise ValueError(f"a model of levels {q} needs level= one of them, got {level}")
        return float(level), q.index(float(level))
    return resolve_tau(model, level)[0], 0


@torch.no_grad()
def fit_distribution(model, loader, device, level=None, by="entry", min_count=1, max_graphs=32, ts=None):
    """Fits a ``ScoreDistribution`` of ``model`` on the labelled held-out batches of ``loader``, through the same
    padded, graph-replayed eval forward as ``calibrate``, with ``n_groups = model.entry_embeds.num_embeddings``.  The
    base column is the model's only level (``level`` None; a one-level model may name the level it was trained at), or
    on a quantile model of T > 1 levels the one ``level`` names (``ValueError`` otherwise).  ``ts`` [n], the buckets of
    the graphs in loader order (an unshuffled ``StoreLoader`` over ``ids`` and ``store.t["trace_ts"][ids]``), keeps a
    log for ``insert`` / ``evict`` / ``add_traces``."""
    level, column = _base_level(model, level)
    y, yhat, ents = _replayed_predictions(model, loader, device, max_graphs, "fit_distribution")
    return ScoreDistribution.fit(y, yhat, ents, model.entry_embeds.num_embeddings, level, by=by, min_count=min_count,
                                 column=column, ts=ts)


@torch.no_grad()
def score_traces(model, loader, device, dist, max_graphs=32):
    """-> float64 [n]: the conformal p-value (``ScoreDistribution.pvalues``) of every labelled trace ``loader`` yields,
    in loader order, from the same graph-replayed eval forward as ``fit_distribution``.  Flag the traces with
    p <= alpha as anomalously slow for a false-alarm rate of at most alpha.  A distribution on the host or on another
    device than ``device`` raises ``PertGnnError`` before the forward."""
    if not isinstance(dist, ScoreDistribution):
        raise TypeError(f"dist must be a ScoreDistribution, got {type(dist).__name__}")
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    if not dist.scores.is_cuda or dist.device != device:
        raise _lib.PertGnnError(f"the distribution is on {dist.device}, the predictions on {device}: move it with "
                                "ScoreDistribution.to(device)")
    y, yhat, ents = _replayed_predictions(model, loader, device, max_graphs, "score_traces")
    return dist.pvalues(yhat, ents, y)
