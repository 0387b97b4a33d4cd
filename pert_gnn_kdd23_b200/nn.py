"""Operator-level surface: the torch_geometric.nn pieces the reference model is built from
(reference model.py:2-7): ``TransformerConv``, ``Linear``, ``global_add_pool`` -- same constructor
arguments, parameter names and math (PyG 2.4.0), computed by the libpertgnn CUDA kernels.
"""
from __future__ import annotations

import math

import torch

from . import ops
from .index import GraphIndex, build_index, cached_index


class Linear(torch.nn.Module):
    """torch_geometric.nn.Linear(in_channels, out_channels, bias=True): y = x W^T + b.

    Lazy ``in_channels=-1`` (the reference's unused ``edge_linear``, model.py:68): PyG 2.4.0 keeps the weight an
    UninitializedParameter (optimisers skip it; not created here) but registers a real ``bias`` [out] -- kept, zero
    filled (PyG leaves it uninitialised), so ``state_dict`` / ``parameters()`` carry ``edge_linear.bias`` like the
    reference; it never receives a gradient."""

    def __init__(self, in_channels, out_channels, bias=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        if in_channels > 0:
            self.weight = torch.nn.Parameter(torch.empty(out_channels, in_channels))
            self.bias = torch.nn.Parameter(torch.empty(out_channels)) if bias else None
            self.reset_parameters()
        else:
            self.weight = None
            self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None

    def reset_parameters(self):
        if self.weight is None:
            return
        torch.nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.in_channels) if self.in_channels > 0 else 0
            torch.nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x):
        if self.weight is None:
            raise RuntimeError("lazy Linear(-1, ...) was never initialised (unused in the reference forward)")
        shp = x.shape
        y = ops.linear(x.reshape(-1, shp[-1]), self.weight, self.bias)
        return y.reshape(*shp[:-1], self.out_channels)


class BatchNorm1d(torch.nn.BatchNorm1d):
    """torch.nn.BatchNorm1d (reference model.py:33,43) over [N, C] input, with an optional fused ReLU epilogue.

    ``affine=False`` normalises with unit scale and zero shift.  Not implemented, and refused before anything runs:
    the [N, C, L] input form and ``momentum=None`` (the cumulative moving average) when the running statistics are
    updated.  A training batch of one row raises torch's ValueError."""

    def forward(self, x, relu=False):
        if x.dim() != 2:
            if x.dim() == 3:
                raise NotImplementedError("BatchNorm1d: only [N, C] input is implemented, not [N, C, L]")
            raise ValueError(f"expected 2D or 3D input (got {x.dim()}D input)")
        training = self.training or (self.running_mean is None)
        updates = self.training and self.running_mean is not None
        if updates and self.momentum is None:
            raise NotImplementedError("BatchNorm1d(momentum=None): the cumulative moving average is not implemented")
        if training and x.size(0) == 1:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size {x.size()}")
        weight, bias = self.weight, self.bias
        if not self.affine:
            weight = torch.ones(self.num_features, device=x.device, dtype=torch.float32)
            bias = torch.zeros(self.num_features, device=x.device, dtype=torch.float32)
        mom = 0.0 if self.momentum is None else self.momentum
        return ops.batch_norm(x, weight, bias, self.running_mean, self.running_var,
                              self.num_batches_tracked if updates else None, training, self.eps, mom, relu)


class TransformerConv(torch.nn.Module):
    """torch_geometric.nn.TransformerConv(in, out, heads=1, edge_dim=..., root_weight=True, bias=True).

    Only what the reference instantiates (model.py:26-51): heads=1, concat=True, beta=False, attention
    dropout 0.  ``forward(x, edge_index, edge_attr)`` keeps PyG's signature ([E,edge_dim] float edge features);
    ``forward_tables`` is the fast path used by SAGEDeterministic where the edge feature is
    cat(if_emb[a], rpc_emb[b]) and ``lin_edge`` (no bias) is folded into two small tables.
    """

    def __init__(self, in_channels, out_channels, heads=1, concat=True, beta=False, dropout=0.0, edge_dim=None,
                 bias=True, root_weight=True):
        super().__init__()
        if heads != 1 or beta or dropout != 0.0 or not concat or not bias:
            raise NotImplementedError("only the configuration used by the reference (heads=1, beta=False, "
                                      "dropout=0, concat=True, bias=True) is implemented")
        self.in_channels, self.out_channels, self.heads, self.edge_dim = in_channels, out_channels, heads, edge_dim
        self.root_weight = root_weight
        self.lin_key = Linear(in_channels, out_channels)
        self.lin_query = Linear(in_channels, out_channels)
        self.lin_value = Linear(in_channels, out_channels)
        self.lin_edge = Linear(edge_dim, out_channels, bias=False) if edge_dim is not None else None
        self.lin_skip = Linear(in_channels, out_channels) if root_weight else None

    def reset_parameters(self):
        for lin in (self.lin_key, self.lin_query, self.lin_value, self.lin_edge, self.lin_skip):
            if lin is not None:
                lin.reset_parameters()

    # -- node projections: ONE GEMM writing the q|k|v|skip planes ------------------------------------
    def _planes(self, x, col_perm=None, pad=0):
        lins = [self.lin_query, self.lin_key, self.lin_value] + ([self.lin_skip] if self.root_weight else [])
        W = torch.cat([l.weight for l in lins], dim=0)
        b = torch.cat([l.bias for l in lins], dim=0)
        if col_perm is not None:
            W = W[:, col_perm]
        if pad:
            W = torch.nn.functional.pad(W, (0, pad))
        return ops.linear(x, W, b, out_blocks=len(lins))

    def forward_tables(self, x, index: GraphIndex, if_table, rpc_table, col_perm=None, pad=0):
        """x [N,Din(+pad)]; if_table [n_if,H], rpc_table [n_rpc,H] embedding weights (edge feature halves)."""
        H = self.out_channels
        planes = self._planes(x, col_perm, pad)
        t_if = t_rpc = None
        if self.lin_edge is not None:
            We = self.lin_edge.weight
            t_if = ops.linear(if_table, We[:, :if_table.size(1)])
            t_rpc = ops.linear(rpc_table, We[:, if_table.size(1):])
        return ops.tconv(planes, t_if, t_rpc, index)

    def forward(self, x, edge_index, edge_attr=None):
        N = x.size(0)
        planes = self._planes(x)
        if self.lin_edge is None:
            index = cached_index(edge_index, N, None, 0, 0)
            return ops.tconv(planes, None, None, index)
        assert edge_attr is not None
        e = ops.linear(edge_attr, self.lin_edge.weight)                  # [E,H], as PyG materialises it
        index = _edge_row_index(edge_index, N)
        zero = torch.zeros(1, self.out_channels, device=x.device)
        return ops.tconv(planes, e, zero, index)


def _edge_row_index(edge_index, N):
    """Index whose 'interface id' of CSR slot p is the edge's own row (perm[p]) and whose 'rpc id' is 0, so a
    per-edge feature matrix [E,H] can be used as the interface table."""
    gi = cached_index(edge_index, N, None, 0, 0)
    if not gi.has_attr:
        gi.csr_if = gi.perm
        gi.csr_rpc = torch.zeros_like(gi.perm)
        gi.has_attr = True
        gi.n_if, gi.n_rpc = gi.E, 1
    return gi


def global_add_pool(x, batch, size=None):
    """torch_geometric.nn.global_add_pool (reference model.py:107).  ``size`` avoids PyG's batch.max() sync;
    ``batch=None`` sums all rows into one [1, H] graph, as PyG does."""
    if batch is None:
        batch, size = torch.zeros(x.size(0), device=x.device, dtype=torch.int64), 1
    elif size is None:
        size = int(batch.max()) + 1 if batch.numel() else 0
    ones = torch.ones(x.size(0), device=x.device)
    pool, _ = ops.pool_local(x, ones, ones, batch, None, None, size)
    return pool
