"""-m gpu tests of hidden widths the attention kernels lack (include/pertgnn.h, pert_model_width): the model runs at the
kernel width Hp >= H with zero padding columns.  Every width 1..256 against the fp32 / fp64 oracles; representative
widths at cfg2 size with dropout, under graph replay and capacity buckets, on the operator path and through the
TransformerConv shim; 20 Adam steps in lockstep with the oracle, after which the padding slots of the packed
parameters must still be exactly 0; checkpoints interchangeable with the oracle's."""
import copy

import pytest
import torch

from oracle import model_oracle
from oracle.model_oracle import OracleSAGEDeterministic, OracleTransformerConv
from pert_gnn_kdd23_b200.synthetic import model_args
from tests.dropout_ref import dropout_masks, oracle_forward
from tests.engine_parts_ref import packed_pad_mask
from tests.helpers import (RTOL, assert_close, assert_close_ref, assert_grads_close_ref, forward_args,
                           is_structural_zero_grad, make_batch)

pytestmark = pytest.mark.gpu

REPRESENTATIVE = (10, 48, 100, 192, 200, 256)
SEED = 0x0A11_F1D7_4B1D_7E5


def _models(cfg, H, seed=0, prep=None):
    """-> (oracle, model on the GPU) with the same parameters; prep(oracle) edits them before they are copied."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    args = list(model_args(cfg))
    args[5] = H
    torch.manual_seed(seed)
    oracle = OracleSAGEDeterministic(*args)
    if prep is not None:
        prep(oracle)
    model = SAGEDeterministic(*args)
    model.load_state_dict(oracle.state_dict())
    return oracle, model.cuda()


def _loss(g, l, y):
    return model_oracle.torch_quantile_loss(y, g.flatten(), 0.5) + 1e-3 * l.square().mean()


def _parity(cfg, ng, H, p=0.0, tag="", prep=None):
    """One training forward + backward through the engine against the fp32 oracle with the fp64 arbiter, both run on
    the engine's active ReLUs (and dropout masks, restated at Hp and cut to H); then an eval forward against the
    oracle with its own ReLUs.  -> (model, batch) after the training step."""
    b = make_batch(cfg, ng)
    a32 = forward_args(b)
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    oracle, model = _models(cfg, H, prep=prep)
    assert list(model.state_dict()) == list(oracle.state_dict())
    assert all(v.shape == oracle.state_dict()[k].shape for k, v in model.state_dict().items())
    for m in (oracle, model):
        m.dropout = p
        m.train()
    model.seed_dropout(SEED)
    oracle64 = copy.deepcopy(oracle).double()
    bc = b.to("cuda")
    gc, lc = model(*forward_args(bc))
    eng = model._engine
    assert eng.Hp >= H and eng.Hp == model_width(H)
    relu = {k: v.cpu() for k, v in eng.active_relus().items()}
    drop = None
    if p > 0:
        N, Hp = b.x.size(0), eng.Hp
        drop = {k: v[:, :H] for k, v in dropout_masks(SEED, 0, N, Hp, p, len(model.bns)).items()}
        for k, keep in drop.items():   # every nonzero saved activation lies in the keep mask restated at Hp
            assert int((relu[k] & ~keep).sum()) == 0, f"{tag} {k}: kept outside the mask"
    loss_c = _loss(gc, lc, bc.y.float())
    loss_c.backward()
    go, lo = oracle_forward(oracle, *a32, relu_masks=relu, dropout_masks=drop)
    go64, lo64 = oracle_forward(oracle64, *a64, relu_masks=relu, dropout_masks=drop)
    loss_o, loss_64 = _loss(go, lo, b.y.float()), _loss(go64, lo64, b.y.double())
    loss_o.backward()
    loss_64.backward()
    assert_close_ref(gc, go, go64, what=f"{tag} global_predict")
    assert_close_ref(lc, lo, lo64, what=f"{tag} local_predict")
    assert_close_ref(loss_c, loss_o, loss_64, what=f"{tag} loss")
    assert_grads_close_ref(model.named_parameters(), oracle.named_parameters(), oracle64.named_parameters(), RTOL,
                           n_convs=len(model.convs))
    b32, b64 = dict(oracle.named_buffers()), dict(oracle64.named_buffers())
    for n, buf in model.named_buffers():
        assert_close_ref(buf.float(), b32[n].float(), b64[n].double(), what=f"{tag} {n}")
    # eval: BatchNorm on the running statistics just updated, no dropout
    model.eval()
    oracle.eval()
    with torch.no_grad():
        ge, le = model(*forward_args(bc))
        go_e, lo_e = oracle_forward(oracle, *a32)
    assert_close(ge, go_e, what=f"{tag} eval global_predict")
    assert_close(le, lo_e, what=f"{tag} eval local_predict")
    return model, b


def model_width(H):
    from pert_gnn_kdd23_b200 import _lib

    return _lib.lib().pert_model_width(H)


@pytest.mark.parametrize("H", range(1, 257))
def test_every_width_against_oracle(H):
    _parity(1, 8, H, tag=f"H={H}")


@pytest.mark.parametrize("H", REPRESENTATIVE)
def test_cfg2_with_dropout(H):
    """cfg2 size (N >= 4096): H = 48 takes the H = 64 fused node-linear kernels and the staged tile kernels."""
    model, b = _parity(2, None, H, p=0.1, tag=f"cfg2 H={H} p=0.1")
    assert b.x.size(0) >= 4096


def _flat_pair(H, p):
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam

    _, ma = _models(1, H)
    mb = copy.deepcopy(ma)
    for m in (ma, mb):
        m.dropout = p
        m.seed_dropout(1234)
    return (ma, FusedAdam(FlatParams(ma), lr=1e-3)), (mb, FusedAdam(FlatParams(mb), lr=1e-3))


@pytest.mark.parametrize("H", REPRESENTATIVE)
def test_graphed_and_bucketed_steps_match_eager(H):
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, GraphedTrainStep, fused_train_step

    d = make_batch(1, 24, seed=3).to("cuda")
    for Step in (GraphedTrainStep, BucketedTrainStep):
        (ma, oa), (mb, ob) = _flat_pair(H, 0.1)
        step = Step(mb, ob, 0.5)
        for n in range(3):                               # eager, capture + replay, replay
            la = fused_train_step(ma, oa, d, 0.5)
            lb = step(d)
            assert_close(lb, la, rtol=1e-4, what=f"{Step.__name__} H={H} loss step {n}")
        assert step.replays == 2 and step.capture_error is None, step.capture_error
        pa = dict(ma.named_parameters())
        for name, prm in mb.named_parameters():
            if is_structural_zero_grad(name, len(ma.convs)):
                continue
            logit = any(t in name for t in (".lin_query.", ".lin_key.", ".lin_edge."))   # as in _trajectory
            assert_close(prm, pa[name], rtol=2e-2 if logit else 2e-3, norm_only=logit,
                         what=f"{Step.__name__} H={H} {name}")
        assert_close(mb._engine.bn_running, ma._engine.bn_running, rtol=1e-4, what="BN running statistics")


@pytest.mark.parametrize("H", REPRESENTATIVE)
def test_evaluate_bucketed_matches_evaluate(H):
    from pert_gnn_kdd23_b200.train import evaluate, evaluate_bucketed, fused_train_step

    (ma, oa), _ = _flat_pair(H, 0.0)
    loader = [make_batch(1, n, seed=10 + n) for n in (16, 16, 7)]
    for d in loader:
        fused_train_step(ma, oa, d.to("cuda"), 0.5)
    want = evaluate(ma, loader, "cuda")
    for rep in range(3):
        got = evaluate_bucketed(ma, loader, "cuda")
        for g, w, what in zip(got, want, ("mae", "mape", "quantile")):
            assert abs(g - w) <= 1e-5 * abs(w), (H, rep, what, g, w)


@pytest.mark.parametrize("H", REPRESENTATIVE)
def test_operator_path_matches_engine(H):
    b = make_batch(1, 16).to("cuda")
    _, me = _models(1, H)
    mo = copy.deepcopy(me)
    mo.use_engine = False
    outs = []
    for m in (me, mo):
        m.train()
        g, l = m(*forward_args(b))
        _loss(g, l, b.y.float()).backward()
        outs.append((g, l))
    assert_close(outs[1][0], outs[0][0], what=f"H={H} global_predict")
    assert_close(outs[1][1], outs[0][1], what=f"H={H} local_predict")
    pe = dict(me.named_parameters())
    for name, prm in mo.named_parameters():
        if prm.grad is None or is_structural_zero_grad(name, len(me.convs)):
            continue
        norm = ".lin_key." in name or ".lin_query." in name     # cancellation-limited logit path (tests/helpers.py)
        assert_close(prm.grad, pe[name].grad, rtol=2e-2 if norm else 1e-3, norm_only=norm, what=f"H={H} grad {name}")
    for n, buf in mo.named_buffers():
        assert_close(buf.float(), dict(me.named_buffers())[n].float(), rtol=1e-4, what=f"H={H} {n}")


@pytest.mark.parametrize("H", [48, 100])
def test_transformer_conv_shim(H):
    from pert_gnn_kdd23_b200.nn import TransformerConv

    b = make_batch(1, 8)
    torch.manual_seed(1)
    Din, edge_dim = 20, 6
    ref = OracleTransformerConv(Din, H, edge_dim=edge_dim)
    conv = TransformerConv(Din, H, heads=1, edge_dim=edge_dim)
    conv.load_state_dict(ref.state_dict(), strict=False)
    conv = conv.cuda()
    N, E = b.x.size(0), b.edge_index.size(1)
    x = torch.randn(N, Din)
    ea = torch.randn(E, edge_dim)
    xc, eac = x.cuda().requires_grad_(), ea.cuda()
    out = conv(xc, b.edge_index.cuda(), eac)
    xr = x.clone().requires_grad_()
    want = ref(xr, b.edge_index, ea)
    assert out.shape == (N, H)
    assert_close(out, want, what=f"shim H={H} out")
    gout = torch.randn(N, H)
    out.backward(gout.cuda())
    want.backward(gout)
    assert_close(xc.grad, xr.grad, what=f"shim H={H} dx")
    pr = dict(ref.named_parameters())
    for n, prm in conv.named_parameters():
        if n in pr and prm.grad is not None and not n.endswith("lin_key.bias"):
            norm = n.startswith(("lin_key.", "lin_query."))
            assert_close(prm.grad, pr[n].grad, rtol=2e-2 if norm else 1e-3, norm_only=norm, what=f"shim H={H} {n}")


@pytest.mark.parametrize("H", [48, 200])
def test_padding_never_leaks(H, tmp_path):
    """20 FusedAdam steps in lockstep with the oracle trained by torch.optim.Adam; the padding slots of the packed
    parameters are exactly 0 afterwards; a checkpoint goes both ways."""
    import ctypes

    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    oracle, model = _models(1, H)
    model.train()
    oracle.train()
    opt = FusedAdam(FlatParams(model), lr=1e-3)
    opt_o = torch.optim.Adam(oracle.parameters(), lr=1e-3)
    b = make_batch(1, 8)
    bc = b.to("cuda")
    for n in range(20):
        loss_c = fused_train_step(model, opt, bc, 0.5)
        opt_o.zero_grad()
        go, _ = oracle(*forward_args(b))
        loss_o = model_oracle.torch_quantile_loss(b.y.float(), go.flatten(), 0.5)
        loss_o.backward()
        opt_o.step()
        assert_close(loss_c, loss_o, rtol=1e-3, what=f"H={H} loss step {n}")
    torch.cuda.synchronize()
    # parameters after 20 steps, norm-wise 5e-2: Adam moves every element by about lr per step whatever the size of its
    # gradient, so an element whose gradient is rounding noise on both sides (a weight direction a BatchNorm removes,
    # as for the biases of is_structural_zero_grad) drifts by up to 2 * 20 * lr between the two runs.  The predictions
    # below, which those directions do not reach, are held to 2e-3 element-wise.
    po = dict(oracle.named_parameters())
    for name, prm in model.named_parameters():
        if not is_structural_zero_grad(name, len(model.convs)):
            assert_close(prm, po[name], rtol=5e-2, norm_only=True, what=f"H={H} {name}")
    model.eval()
    oracle.eval()
    with torch.no_grad():
        gc, lc = model(*forward_args(bc))
        go, lo = oracle(*forward_args(b))
    assert_close(gc, go, rtol=2e-3, what=f"H={H} global_predict after 20 steps")
    assert_close(lc, lo, rtol=2e-3, what=f"H={H} local_predict after 20 steps")
    # the packed region (refreshed by that forward) is zero exactly where it holds padding
    eng = model._engine
    n_packed = eng.lib.pert_model_packed_bytes(ctypes.byref(eng.desc)) // 4
    pad = packed_pad_mask(eng.desc, eng.Hp, eng.n_convs, eng.fp.flat.numel())
    assert pad.numel() == n_packed
    packed = eng.ws[:n_packed].cpu()
    assert int((packed[pad] != 0).sum()) == 0, f"H={H}: padding slots of the packed parameters are not 0"
    assert int((packed[~pad] != 0).sum()) > 0.9 * int((~pad).sum())
    # checkpoints: same keys and shapes as the oracle's; the engine model's loads into a fresh oracle
    sd = model.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in oracle.state_dict().items()}
    path = tmp_path / "ckpt.pt"
    torch.save({k: v.cpu() for k, v in sd.items()}, path)
    fresh, _ = _models(1, H, seed=99)
    fresh.load_state_dict(torch.load(path))
    fresh.eval()
    with torch.no_grad():
        gf, lf = fresh(*forward_args(b))
    assert_close(gc, gf, what=f"H={H} checkpoint -> oracle global_predict")
    assert_close(lc, lf, what=f"H={H} checkpoint -> oracle local_predict")
