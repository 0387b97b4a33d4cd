"""CPU tests of embedding growth (train.grow_embeddings, FlatParams.grow, pert_flat_grow): the new flat layout against a
numpy restatement, the C-ABI's rejection of bad segment tables before any CUDA call, and the host-side refusals."""
import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from pert_gnn_kdd23_b200.model import SAGEDeterministic
from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, PeerAdam, grow_embeddings

BAD = -1


def _model(H=32, layers=2, n_cat=(24,), ent=6, n_if=31, rpc=5):
    torch.manual_seed(0)
    return SAGEDeterministic(9, list(n_cat), ent, n_if, rpc, H, layers, 0.0)


def _np_layout(shapes):
    """Restatement: every parameter starts on a 64-float boundary, in order; the length is the last end rounded up."""
    sizes = np.array([int(np.prod(s)) for s in shapes], dtype=np.int64)
    slots = (sizes + 63) // 64 * 64
    offs = np.concatenate([[0], np.cumsum(slots)[:-1]]).astype(np.int64)
    return offs, int(slots.sum()), sizes


def _grown_shapes(model, fp, rows):
    """The shapes with the tables of ``rows`` ({module: new row count}) grown."""
    by_id = {id(m.weight): n for m, n in rows.items()}
    return [(by_id[id(p)],) + tuple(p.shape[1:]) if id(p) in by_id else tuple(p.shape) for p in fp.params]


@pytest.mark.parametrize("H,layers,n_cat", [(32, 2, (24,)), (64, 3, (24, 7)), (100, 2, (5,)), (128, 8, (3, 4, 5, 6))])
def test_layout_restatement(H, layers, n_cat):
    m = _model(H, layers, n_cat)
    fp = FlatParams(m)
    offs, n, _ = _np_layout([tuple(p.shape) for p in fp.params])
    assert [o for o, _, _ in fp._layout] == offs.tolist() and fp.numel == n
    assert all(o % _lib.FLAT_ALIGN == 0 for o in offs)
    assert len(fp.params) <= _lib.FLAT_MAX_SEGS
    tabs = [m.cat_embedding[0], m.entry_embeds, m.interface_embeds, m.rpctype_embeds]
    for grow in ([{t: t.num_embeddings + 1} for t in tabs] + [{t: t.num_embeddings + 1000 + i for i, t in
                                                                enumerate(tabs)}, {m.interface_embeds: 1 << 20}]):
        new = _grown_shapes(m, fp, grow)
        shapes, got_offs, got_n, segs = fp.grow_plan(new)
        want_offs, want_n, want_sizes = _np_layout(new)
        old_sizes = np.array([p.numel() for p in fp.params], dtype=np.int64)
        assert shapes == new and got_offs == want_offs.tolist() and got_n == want_n
        assert np.array_equal(segs, np.stack([offs, want_offs, old_sizes, want_sizes], 1))
        # the parameters up to the first grown one stay; the ones after it never move down
        first = min(i for i, p in enumerate(fp.params) if tuple(p.shape) != new[i])
        assert np.array_equal(segs[:first + 1, 0], segs[:first + 1, 1])
        assert (segs[first + 1:, 1] >= segs[first + 1:, 0]).all()


def test_plan_refuses_shapes():
    m = _model()
    fp = FlatParams(m)
    shapes = [tuple(p.shape) for p in fp.params]
    i = next(k for k, p in enumerate(fp.params) if p is m.interface_embeds.weight)
    for bad, msg in (((shapes[i][0] - 1, shapes[i][1]), "cannot become"),           # shrinking
                     ((shapes[i][0], shapes[i][1] + 1), "cannot become"),           # a column more
                     ((shapes[i][0],), "cannot become")):                            # another rank
        with pytest.raises(_lib.PertGnnError, match=msg):
            fp.grow_plan(shapes[:i] + [bad] + shapes[i + 1:])
    with pytest.raises(_lib.PertGnnError, match="shapes for"):
        fp.grow_plan(shapes[:-1])


# ---- the C-ABI rejects every bad table before any CUDA call: the pointers below are never dereferenced ----------------
def _call(L, segs, n_old, n_new, ptrs=None, n_seg=None):
    a = np.ascontiguousarray(np.asarray(segs, dtype=np.int64).reshape(-1, 4))
    base = 1 << 40
    p = dict(p_old=base, p_new=base + (1 << 30), m_old=base + (2 << 30), m_new=base + (3 << 30), v_old=base + (4 << 30),
             v_new=base + (5 << 30), g_new=base + (6 << 30))
    p.update(ptrs or {})
    return L.pert_flat_grow(a.ctypes.data if a.size else None, a.shape[0] if n_seg is None else n_seg, n_old, n_new,
                            p["p_old"], p["p_new"], p["m_old"], p["m_new"], p["v_old"], p["v_new"], p["g_new"], None)


def test_abi_rejects_bad_segment_tables():
    L = _lib.lib()
    ok = [(0, 0, 100, 100), (128, 128, 10, 70), (192, 256, 64, 64)]     # a valid table: 256 -> 320 floats
    n_old, n_new = 256, 320
    cases = {
        "out of order": [(128, 128, 10, 70), (0, 0, 100, 100)],
        "overlap in the old layout": [(0, 0, 100, 100), (64, 128, 10, 70)],
        "overlap in the new layout": [(0, 0, 100, 100), (128, 64, 10, 70)],
        "shrinking": [(0, 0, 100, 99)],
        "negative length": [(0, 0, -1, 0)],
        "old offset unaligned": [(0, 0, 100, 100), (132, 128, 10, 70)],
        "new offset unaligned": [(0, 0, 100, 100), (128, 130, 10, 70)],
        "past n_old": ok[:2] + [(192, 256, 65, 65)],
        "past n_new": ok[:2] + [(192, 256, 64, 65)],
    }
    for what, segs in cases.items():
        assert _call(L, segs, n_old, n_new) == BAD, what
    assert _call(L, ok, n_old, 250) == BAD                               # n_new not aligned
    assert _call(L, ok, 250, n_new) == BAD                               # n_old not aligned
    assert _call(L, ok, n_old, 192) == BAD                               # n_new < n_old
    assert _call(L, ok, -64, n_new) == BAD
    assert _call(L, ok, n_old, n_new, n_seg=-1) == BAD
    assert _call(L, [(0, 0, 1, 1)] * 1, n_old, n_new, n_seg=_lib.FLAT_MAX_SEGS + 1) == BAD
    assert L.pert_flat_grow(None, 2, n_old, n_new, 1 << 40, 2 << 40, None, None, None, None, 3 << 40, None) == BAD
    # buffers: NULL, one half of a pair, misaligned, aliasing
    for bad in ({"p_old": None}, {"p_new": None}, {"g_new": None}, {"m_old": None}, {"v_new": None},
                {"g_new": (1 << 40) + 4}, {"p_new": 1 << 40}, {"g_new": (1 << 40) + (3 << 30) + 256},
                {"m_new": (1 << 40) + (2 << 30) + 1024 - 512}):
        assert _call(L, ok, n_old, n_new, bad) == BAD, bad


# ---- host refusals of grow_embeddings ----------------------------------------------------------------------------------
def test_grow_embeddings_refusals(monkeypatch):
    m = _model()
    before = [p.data_ptr() for p in m.parameters()]
    with pytest.raises(_lib.PertGnnError, match="never shrink"):
        grow_embeddings(m, interface=m.interface_embeds.num_embeddings - 1)
    with pytest.raises(TypeError):
        grow_embeddings(m, entry=7.5)
    with pytest.raises(_lib.PertGnnError, match="unsupported optimizer"):
        grow_embeddings(m, object(), entry=100)
    peer = PeerAdam.__new__(PeerAdam)
    peer.world = 2
    with pytest.raises(_lib.PertGnnError, match="PeerAdam"):
        grow_embeddings(m, peer, entry=100)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(_lib.PertGnnError, match="capture"):
        grow_embeddings(m, entry=100)
    monkeypatch.undo()
    # nothing to grow: nothing is touched, not even a FlatParams made
    rows = grow_embeddings(m, entry=m.entry_embeds.num_embeddings, cat=24)
    assert rows == {"cat": 24, "entry": 7, "interface": 32, "rpctype": 6}
    assert [p.data_ptr() for p in m.parameters()] == before and "_flat_params" not in m.__dict__


def test_fused_adam_over_another_model_is_refused():
    a, b = _model(), _model()
    opt = FusedAdam(FlatParams(a))
    with pytest.raises(_lib.PertGnnError, match="does not hold"):
        grow_embeddings(b, opt, entry=100)


def test_cpu_model_is_refused_before_anything_changes():
    m = _model()
    before = [p.data_ptr() for p in m.parameters()]
    with pytest.raises(_lib.PertGnnError, match="CUDA"):
        grow_embeddings(m, entry=100)
    assert [p.data_ptr() for p in m.parameters()] == before and m.entry_embeds.num_embeddings == 7
    fp = FlatParams(m)
    with pytest.raises(_lib.PertGnnError, match="CUDA"):
        fp.grow([tuple(p.shape) for p in fp.params])


def test_flat_params_know_their_optimizer():
    """FlatParams.grow relays the m and v of the FusedAdam over it, so a growth that does not name the optimizer cannot
    leave it with buffers of the old length; two live FusedAdams over one FlatParams are refused."""
    m = _model()
    fp = FlatParams(m)
    opt = FusedAdam(fp)
    assert fp._live_optimizers() == [opt]
    second = FusedAdam(fp)
    with pytest.raises(_lib.PertGnnError, match="2 FusedAdams"):
        fp.grow([tuple(p.shape) for p in fp.params])
    del second
    assert fp._live_optimizers() == [opt]


def test_adam_step_refuses_buffers_of_another_length():
    """The step runs over fp.numel floats of m and v: buffers of another length are refused on the host, before any
    launch, instead of being read and written past their end."""
    m = _model()
    opt = FusedAdam(FlatParams(m))
    opt.m = torch.zeros(opt.fp.numel - 64)
    with pytest.raises(_lib.PertGnnError, match="m / v hold"):
        opt.step()
    assert opt.t == 0
