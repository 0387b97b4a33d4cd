"""Minimal PyG-compatible ``Data`` / ``Batch`` / ``DataLoader``.

The reference builds one ``torch_geometric.data.Data`` per trace
(reference pert_gnn.py:163-173) and batches them with
``torch_geometric.loader.DataLoader`` (pert_gnn.py:201-209); its train loop then
uses ``data.to(device)``, ``data.x`` ..., ``data.batch``, ``data.num_graphs`` and
``len(loader.dataset)`` (pert_gnn.py:219-251).  torch_geometric is not available
on the target boxes, so this module provides exactly that surface with the same
collation rules (SURVEY.md section 8b):

* every attribute is concatenated along dim 0, except attributes whose name
  contains ``index`` which are concatenated along the last dim and incremented
  by the cumulative node count (``x.size(0)``);
* 0-dim tensors are stacked into a 1-D tensor;
* ``batch`` [N] int64 and ``ptr`` [B+1] int64 are added.

Additions (not in PyG): ``Batch.pin_memory()`` stages the whole batch in ONE
pinned host slab and ``Batch.to(device, non_blocking=True)`` moves it with ONE
H2D copy (the reference does one copy per attribute plus B tiny ones per step,
pert_gnn.py:220-231); the per-attribute tensors on the device are views into
the slab.
"""
from __future__ import annotations

import torch
from torch.utils.data import DataLoader as _TorchDataLoader

_ALIGN = 256  # byte alignment of every attribute inside the slab (keeps float4 / TMA alignment)


class Data:
    """Attribute container (subset of torch_geometric.data.Data)."""

    def __init__(self, x=None, edge_index=None, edge_attr=None, y=None, **kwargs):
        self._store = {}
        for k, v in (("x", x), ("edge_index", edge_index), ("edge_attr", edge_attr), ("y", y)):
            if v is not None:
                self._store[k] = v
        self._store.update(kwargs)

    # -- attribute access ---------------------------------------------------
    def __getattr__(self, key):
        if key.startswith("_"):
            raise AttributeError(key)
        try:
            return self._store[key]
        except KeyError:
            raise AttributeError(f"'{type(self).__name__}' object has no attribute '{key}'") from None

    def __setattr__(self, key, value):
        if key.startswith("_"):
            object.__setattr__(self, key, value)
        else:
            self._store[key] = value

    def __getitem__(self, key):
        return self._store[key]

    def __setitem__(self, key, value):
        self._store[key] = value

    def __contains__(self, key):
        return key in self._store

    def keys(self):
        return list(self._store.keys())

    def items(self):
        return self._store.items()

    def to_dict(self):
        return dict(self._store)

    @property
    def num_nodes(self):
        if "x" in self._store:
            return self._store["x"].size(0)
        if "edge_index" in self._store and self._store["edge_index"].numel() > 0:
            return int(self._store["edge_index"].max()) + 1
        return 0

    @property
    def num_edges(self):
        return self._store["edge_index"].size(1) if "edge_index" in self._store else 0

    def _apply(self, fn):
        out = object.__new__(type(self))
        object.__setattr__(out, "_store", {k: (fn(v) if torch.is_tensor(v) else v)
                                            for k, v in self._store.items()})
        for k, v in self.__dict__.items():
            if k != "_store":
                object.__setattr__(out, k, v)
        return out

    def to(self, device, non_blocking=False):
        return self._apply(lambda t: t.to(device, non_blocking=non_blocking))

    def cpu(self):
        return self.to("cpu")

    def cuda(self, device=None, non_blocking=False):
        return self.to("cuda" if device is None else device, non_blocking=non_blocking)

    def pin_memory(self):
        return self._apply(lambda t: t.pin_memory())

    def __repr__(self):
        body = ", ".join(f"{k}={list(v.shape) if torch.is_tensor(v) else v}" for k, v in self._store.items())
        return f"{type(self).__name__}({body})"


class Batch(Data):
    """Disjoint union of graphs (subset of torch_geometric.data.Batch)."""

    @classmethod
    def from_data_list(cls, data_list):
        assert len(data_list) > 0
        keys = data_list[0].keys()
        n_nodes = [d.num_nodes for d in data_list]
        offs = [0]
        for n in n_nodes:
            offs.append(offs[-1] + n)
        store = {}
        for k in keys:
            vals = [d[k] for d in data_list]
            v0 = vals[0]
            if not torch.is_tensor(v0):
                store[k] = torch.tensor(vals) if isinstance(v0, (int, float)) else vals
            elif v0.dim() == 0:
                store[k] = torch.stack(vals)
            elif "index" in k:
                store[k] = torch.cat([v + offs[i] for i, v in enumerate(vals)], dim=-1)
            else:
                store[k] = torch.cat(vals, dim=0)
        store["batch"] = torch.repeat_interleave(
            torch.arange(len(data_list), dtype=torch.long), torch.tensor(n_nodes, dtype=torch.long))
        store["ptr"] = torch.tensor(offs, dtype=torch.long)
        out = cls()
        out._store.update(store)
        object.__setattr__(out, "_num_graphs", len(data_list))
        return out

    @property
    def num_graphs(self):
        ng = self.__dict__.get("_num_graphs")
        if ng is not None:
            return ng
        if "ptr" in self._store:
            return self._store["ptr"].numel() - 1
        return int(self._store["batch"].max()) + 1

    # -- single-slab staging --------------------------------------------------
    def _slab_layout(self):
        layout, off = [], 0
        for k, v in self._store.items():
            if torch.is_tensor(v):
                nbytes = v.numel() * v.element_size()
                layout.append((k, off, nbytes, v.dtype, tuple(v.shape)))
                off += (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        return layout, max(off, _ALIGN)

    def pin_memory(self):
        """Pack every tensor attribute into one pinned uint8 slab (one H2D later)."""
        layout, total = self._slab_layout()
        slab = torch.empty(total, dtype=torch.uint8).pin_memory() if torch.cuda.is_available() \
            else torch.empty(total, dtype=torch.uint8)
        out = self._apply(lambda t: t)
        for k, off, nbytes, dtype, shape in layout:
            view = slab[off:off + nbytes].view(dtype).view(shape)
            view.copy_(self._store[k])
            out._store[k] = view
        object.__setattr__(out, "_slab", slab)
        object.__setattr__(out, "_layout", layout)
        return out

    def to(self, device, non_blocking=False):
        slab = self.__dict__.get("_slab")
        dev = torch.device(device)
        if slab is None or dev.type != "cuda":
            return super().to(device, non_blocking=non_blocking)
        dslab = slab.to(dev, non_blocking=non_blocking)          # ONE H2D copy
        out = self._apply(lambda t: t)
        for k, off, nbytes, dtype, shape in self.__dict__["_layout"]:
            out._store[k] = dslab[off:off + nbytes].view(dtype).view(shape)
        object.__setattr__(out, "_slab", dslab)
        return out

    @property
    def h2d_bytes(self):
        """Bytes one ``.to(cuda)`` of this batch moves (for bench accounting)."""
        slab = self.__dict__.get("_slab")
        if slab is not None:
            return slab.numel()
        return sum(v.numel() * v.element_size() for v in self._store.values() if torch.is_tensor(v))


def _collate(data_list):
    return Batch.from_data_list(data_list)


def shard_by_edges(data_list, world):
    """Data-parallel partition of a list of graphs over ``world`` ranks, balanced by edge count rather than by graph
    count (SURVEY.md 8e: the conv kernels' work is per edge, and call-graph sizes are power-law distributed).
    Greedy longest-processing-time: graphs in descending edge order, each to the currently lightest rank (ties: fewer
    graphs, then lower rank).  Deterministic; returns ``world`` lists of indices into ``data_list`` (each sorted
    ascending so a rank keeps the dataset order).  The reference is single-GPU and has no counterpart."""
    assert world >= 1
    sizes = [(int(d.num_edges) + 1, i) for i, d in enumerate(data_list)]      # +1: isolated graphs still cost a row
    order = sorted(sizes, key=lambda t: (-t[0], t[1]))
    load = [0] * world
    parts = [[] for _ in range(world)]
    for sz, i in order:
        r = min(range(world), key=lambda k: (load[k], len(parts[k]), k))
        parts[r].append(i)
        load[r] += sz
    return [sorted(p) for p in parts]


class DevicePrefetcher:
    """Iterates an iterable of host ``Batch`` objects and yields device batches, issuing the (single-slab) H2D copy
    of batch i+1 on a side stream while batch i is being trained on -- the step no longer waits for PCIe.
    The reference moves each batch synchronously inside the loop (pert_gnn.py:231)."""

    def __init__(self, batches, device):
        self.batches = batches
        self.device = torch.device(device)
        # the ring outlives one pass over ``batches`` (epochs re-use the same device buffers, so a CUDA-graph
        # replayed step -- train.GraphedTrainStep keys its graphs by buffer address -- keeps hitting)
        self._side = None
        self._ring = [None, None, None]    # device slabs reused round-robin: no allocator traffic in the loop
        self._done = [None, None, None]    # event: the training step that consumed ring[k] has been issued + finished
        self._k = 0

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        if self._side is None:
            self._side = torch.cuda.Stream(self.device)
        side, ring, done = self._side, self._ring, self._done
        state = {"k": self._k}

        def load(b):
            if b.__dict__.get("_slab") is None:
                b = b.pin_memory()
            host = b.__dict__["_slab"]
            k = state["k"]
            state["k"] = (k + 1) % len(ring)
            if done[k] is not None:
                side.wait_event(done[k])   # the step that read this slab must be over before it is overwritten
            with torch.cuda.stream(side):
                if ring[k] is None or ring[k].numel() < host.numel():
                    # allocated ON the side stream: the caching allocator then only hands out a block whose previous
                    # users are ordered before this stream's work (a block freed on the main stream could still be
                    # read there); the consumer's use is ordered by the event below + record_stream
                    ring[k] = torch.empty(host.numel(), dtype=torch.uint8, device=self.device)
                    ring[k].record_stream(torch.cuda.current_stream(self.device))
                dslab = ring[k][:host.numel()]
                dslab.copy_(host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
            out = b._apply(lambda t: t)
            for key, off, nbytes, dtype, shape in b.__dict__["_layout"]:
                out._store[key] = dslab[off:off + nbytes].view(dtype).view(shape)
            object.__setattr__(out, "_slab", dslab)
            return out, ev, k

        it = iter(self.batches)
        try:
            nxt = load(next(it))
        except StopIteration:
            return
        try:
            while nxt is not None:
                cur, ev, k = nxt
                try:
                    nxt = load(next(it))
                except StopIteration:
                    nxt = None
                main = torch.cuda.current_stream(self.device)
                main.wait_event(ev)
                yield cur
                d = torch.cuda.Event()
                d.record(main)             # everything the consumer launched on this batch
                done[k] = d
        finally:
            self._k = state["k"]


class DataLoader(_TorchDataLoader):
    """torch_geometric.loader.DataLoader(dataset, batch_size, shuffle) look-alike."""

    def __init__(self, dataset, batch_size=1, shuffle=False, **kwargs):
        kwargs.pop("collate_fn", None)
        super().__init__(dataset, batch_size=batch_size, shuffle=shuffle, collate_fn=_collate, **kwargs)
