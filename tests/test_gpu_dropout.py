"""-m gpu tests of the dropout inside the step engine (BatchNorm apply + Philox mask, include/pertgnn.h):
the mask bit for bit against the restatement in tests/dropout_ref.py, full-model parity with dropout against the fp32
and fp64 oracles, the deterministic ends (p = 0, p = 1, eval), the device counter under CUDA-graph replay, the drop-in
autograd path, and reproducibility by seed."""
import copy
import ctypes

import pytest
import torch

from tests.dropout_ref import dropout_masks, oracle_forward, scale_of
from tests.helpers import (RTOL, assert_close, assert_close_ref, assert_grads_close, assert_grads_close_ref,
                           forward_args, is_structural_zero_grad, make_batch, make_models)

pytestmark = pytest.mark.gpu

SEED = 0x0123_4567_89ab_cdef


def _saved_acts(model, N, E, B):
    """{l: [N,H] view of x[l]} -- the post-BatchNorm-ReLU-dropout inputs of convs 1.. in the engine workspace."""
    eng = model._engine
    H = eng.desc.H
    out = {}
    for l in range(1, eng.n_convs):
        off = eng.lib.pert_model_workspace_offset(ctypes.byref(eng.desc), N, E, B, 0, l)
        assert off >= 0
        out[l] = eng.ws[off:off + N * H].view(N, H)
    return out


def _sizes(b):
    return b.x.size(0), b.edge_index.size(1), b.num_graphs


def _state(model):
    return [int(v) for v in model.dropout_state().cpu()]


@pytest.mark.parametrize("cfg, ng", [(1, None), (2, None)])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mask_bit_exact(cfg, ng, p):
    """Every nonzero of x[l+1] lies in the restated keep mask of layer l at the counter read before the forward, and
    x[l+1] equals the oracle's relu(bn(out)) * scale * mask (the oracle run with the same masks)."""
    b = make_batch(cfg, ng)
    oracle, model = make_models(cfg)
    oracle.train()
    model.train()
    oracle.dropout = model.dropout = p
    model.seed_dropout(SEED)
    torch.cuda.synchronize()
    seed, step = _state(model)
    assert step == 0
    with torch.no_grad():
        model(*forward_args(b.to("cuda")))
    torch.cuda.synchronize()
    assert _state(model) == [seed, 1]
    N, E, B = _sizes(b)
    H = model.hidden_channels
    masks = dropout_masks(seed, step, N, H, p, len(model.bns))
    pre = {}
    with torch.no_grad():
        oracle_forward(oracle, *forward_args(b), dropout_masks=masks, capture=pre)
    acts = _saved_acts(model, N, E, B)
    for l in range(len(model.bns)):
        got = acts[l + 1].cpu()
        keep = masks[f"bn{l}"]
        assert int(((got != 0) & ~keep).sum()) == 0, f"layer {l}: nonzero outside the keep mask"
        want = pre[f"bn{l}"] * keep * scale_of(p)
        assert_close(got, want, rtol=1e-5, what=f"cfg{cfg} p={p} x[{l + 1}]")
        # the mask is not vacuous: kept positions with a clearly positive pre-dropout value are nonzero
        live = keep & (pre[f"bn{l}"] > 1e-3)
        assert int(live.sum()) > 0 and bool((got[live] != 0).all())


def _parity_with_dropout(cfg, ng, tag, p=0.1):
    """_full_parity (tests/test_gpu_fullsize.py) with dropout: the engine's ReLU pattern (active and kept) and the
    restated dropout masks go into the fp32 and fp64 oracles."""
    from oracle import model_oracle

    b = make_batch(cfg, ng)
    a32 = forward_args(b)
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    oracle, model = make_models(cfg)
    for m in (oracle, model):
        m.dropout = p
        m.train()
    oracle64 = copy.deepcopy(oracle).double()
    oracle_free = copy.deepcopy(oracle)
    model.seed_dropout(SEED + cfg)
    bc = b.to("cuda")

    def loss_of(g, l, y):
        return model_oracle.torch_quantile_loss(y, g.flatten(), 0.5) + 1e-3 * l.square().mean()

    gc, lc = model(*forward_args(bc))
    assert model._engine._saved[-1] == p
    relu = {k: v.cpu() for k, v in model._engine.active_relus().items()}
    N = b.x.size(0)
    drop = dropout_masks(SEED + cfg, 0, N, model.hidden_channels, p, len(model.bns))
    loss_c = loss_of(gc, lc, bc.y.float())
    loss_c.backward()
    go, lo = oracle_forward(oracle, *a32, relu_masks=relu, dropout_masks=drop)
    go64, lo64 = oracle_forward(oracle64, *a64, relu_masks=relu, dropout_masks=drop)
    loss_o, loss_64 = loss_of(go, lo, b.y.float()), loss_of(go64, lo64, b.y.double())
    loss_o.backward()
    loss_64.backward()
    assert_close_ref(gc, go, go64, what=f"{tag} global_predict")
    assert_close_ref(lc, lo, lo64, what=f"{tag} local_predict")
    assert_close_ref(loss_c, loss_o, loss_64, what=f"{tag} loss")
    assert_grads_close_ref(model.named_parameters(), oracle.named_parameters(), oracle64.named_parameters(), RTOL,
                           n_convs=len(model.convs))
    b64 = dict(oracle64.named_buffers())
    b32 = dict(oracle.named_buffers())
    for n, bbuf in model.named_buffers():
        assert_close_ref(bbuf.float(), b32[n].float(), b64[n].double(), what=f"{tag} {n}")
    with torch.no_grad():
        gfree, lfree = oracle_forward(oracle_free, *a32, dropout_masks=drop)
    assert_close(gc, gfree, what=f"{tag} global_predict (oracle with its own ReLUs)")
    assert_close(lc, lfree, what=f"{tag} local_predict (oracle with its own ReLUs)")


def test_parity_with_dropout_cfg2():
    _parity_with_dropout(2, None, "cfg2[256] p=0.1")


def test_parity_with_dropout_cfg4_shard():
    _parity_with_dropout(4, 512, "cfg4[512 of 4096] p=0.1")


def _fwd_bwd(model, bc):
    for p in model.parameters():
        p.grad = None
    g, l = model(*forward_args(bc))
    (g.square().mean() + 1e-3 * l.square().mean()).backward()
    return g.detach(), l.detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


def test_p0_matches_unseeded_and_counter_still():
    """p = 0 never reads the dropout state: a seeded model and one whose state was never created agree, and the
    counter does not move.  The step is not bit-reproducible between two runs (atomic accumulations in the forward and
    backward), so values are compared at run-to-run bars: 1e-6 for the forward, the parity bars for the gradients."""
    _, m0 = make_models(2)
    m1 = copy.deepcopy(m0)
    m0.train()
    m1.train()
    m1.seed_dropout(SEED)
    bc = make_batch(2, 64).to("cuda")
    g0, l0, _ = _fwd_bwd(m0, bc)
    a0 = {k: v.clone() for k, v in _saved_acts(m0, *_sizes(bc)).items()}
    g1, l1, _ = _fwd_bwd(m1, bc)
    a1 = _saved_acts(m1, *_sizes(bc))
    assert "_dropout_state" not in m0.__dict__
    assert m0._engine._saved[-1] == 0.0 and m1._engine._saved[-1] == 0.0
    assert _state(m1) == [SEED, 0]
    assert_close(l1, l0, rtol=1e-6, what="local_predict p=0")
    assert_close(g1, g0, rtol=1e-6, what="global_predict p=0")
    for k in a0:
        assert_close(a1[k], a0[k], rtol=1e-6, what=f"x[{k}] p=0")
    assert_grads_close(m1.named_parameters(), m0.named_parameters(), RTOL, n_convs=len(m0.convs))


def test_p1_matches_torch_dropout():
    """p = 1 drops every BatchNorm output: every gradient matches the oracle with F.dropout(p=1)."""
    b = make_batch(2, 32)
    oracle, model = make_models(2)
    oracle.train()
    model.train()
    oracle.dropout = model.dropout = 1.0
    model.seed_dropout(SEED)
    bc = b.to("cuda")
    gc, lc, _ = _fwd_bwd(model, bc)
    for l, act in _saved_acts(model, *_sizes(bc)).items():
        assert int((act != 0).sum()) == 0, l
    go, lo = oracle(*forward_args(b))
    (go.square().mean() + 1e-3 * lo.square().mean()).backward()
    assert_close(gc, go, what="global_predict p=1")
    assert_close(lc, lo, what="local_predict p=1")
    assert_grads_close(model.named_parameters(), oracle.named_parameters(), RTOL, n_convs=len(model.convs))
    assert _state(model) == [SEED, 1]


def test_eval_ignores_dropout():
    """Eval mode passes p = 0 to the engine whatever model.dropout is (same kernels; compared at the run-to-run bar of
    test_p0_matches_unseeded_and_counter_still) and leaves the counter alone."""
    _, model = make_models(2)
    model.eval()
    model.seed_dropout(SEED)
    bc = make_batch(2, 64).to("cuda")
    with torch.no_grad():
        g0, l0 = model(*forward_args(bc))
        model.dropout = 0.5
        g1, l1 = model(*forward_args(bc))
    assert model._engine._saved[-1] == 0.0
    assert_close(l1, l0, rtol=1e-6, what="eval local_predict")
    assert_close(g1, g0, rtol=1e-6, what="eval global_predict")
    assert _state(model) == [SEED, 0]


def test_counter_under_graph_replay_and_a_new_rate():
    """GraphedTrainStep (eager, capture + replay, replays on two keys) against fused_train_step on a copy seeded alike:
    same losses, both counters at 8, and a replay draws the mask of ITS step, not the captured one.  Changing the rate
    is a new key: eager once, then exactly one capture."""
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep, fused_train_step

    _, model_a = make_models(2)
    model_a.dropout = 0.1
    model_a.train()
    model_b = copy.deepcopy(model_a)
    opt_a = FusedAdam(FlatParams(model_a), lr=1e-3)
    opt_b = FusedAdam(FlatParams(model_b), lr=1e-3)
    model_a.seed_dropout(SEED)
    model_b.seed_dropout(SEED)
    batches = [make_batch(2, 32, seed=s).to("cuda") for s in range(2)]
    step_b = GraphedTrainStep(model_b, opt_b, 0.5)
    for it in range(8):
        b = batches[it % 2]
        la = fused_train_step(model_a, opt_a, b, 0.5)
        lb = step_b(b)
        assert_close(lb, la, rtol=1e-4, what=f"loss step {it}")
    assert step_b.capture_error is None, step_b.capture_error
    assert step_b.replays == 6
    torch.cuda.synchronize()
    assert _state(model_a) == [SEED, 8] and _state(model_b) == [SEED, 8]
    # the last replay (batch 1, step counter 7) -- its key was captured at counter 3
    N, E, B = _sizes(batches[1])
    x1 = _saved_acts(model_b, N, E, B)[1].cpu()
    H = model_b.hidden_channels
    now = dropout_masks(SEED, 7, N, H, 0.1, 1)["bn0"]
    captured = dropout_masks(SEED, 3, N, H, 0.1, 1)["bn0"]
    assert int(((x1 != 0) & ~now).sum()) == 0
    assert int(((x1 != 0) & ~captured).sum()) > 0
    # a new rate is a new key: eager once, then captured and replayed with the new rate
    c0 = step_b.captures
    model_a.dropout = model_b.dropout = 0.3
    for it in range(2):
        la = fused_train_step(model_a, opt_a, batches[0], 0.5)
        lb = step_b(batches[0])
        assert_close(lb, la, rtol=1e-4, what=f"loss step {it} at p=0.3")
    assert step_b.captures == c0 + 1 and step_b.replays == 7
    torch.cuda.synchronize()
    assert _state(model_b) == [SEED, 10]
    x1 = _saved_acts(model_b, N, E, B)[1].cpu()
    assert int(((x1 != 0) & ~dropout_masks(SEED, 9, N, H, 0.3, 1)["bn0"]).sum()) == 0


def test_dropin_path_runs_engine():
    """model(*inputs) in training with dropout runs on the engine; its autograd gradients equal Engine.backward of the
    same forward (same counter)."""
    _, model = make_models(2)
    model.train()
    model.dropout = 0.2
    bc = make_batch(2, 64).to("cuda")
    model.seed_dropout(SEED)
    model.engine()._saved = None
    for p in model.parameters():
        p.grad = None
    g, _ = model(*forward_args(bc))
    assert model._engine._saved is not None and model._engine._saved[-1] == 0.2
    g.sum().backward()
    auto = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    model.seed_dropout(SEED)
    eng = model.engine()
    from pert_gnn_kdd23_b200.index import cached_index
    from pert_gnn_kdd23_b200.train import model_inputs

    x, cat_X, edge_index, edge_attr, pnn, probs, entry_id, batch = model_inputs(bc)
    index = cached_index(edge_index, x.size(0), edge_attr, model.interface_embeds.num_embeddings,
                         model.rpctype_embeds.num_embeddings)
    index.num_graphs = entry_id.numel()
    with torch.no_grad():
        g2, _ = eng.forward(x, cat_X, entry_id, probs, pnn, batch, index, True)
        gbuf = torch.zeros_like(eng.fp.flat)
        eng.backward(torch.ones_like(g2).reshape(-1), None, grads=gbuf)
    assert_close(g2, g.detach(), rtol=1e-6, what="engine forward vs drop-in forward")
    views = dict(zip([n for n, p in model.named_parameters() if p.requires_grad], eng.fp.views_of(gbuf)))
    scale = max(float(v.abs().max()) for v in auto.values())
    for n, v in auto.items():
        if is_structural_zero_grad(n, len(model.convs)):     # rounding noise only (tests/helpers.py)
            assert float(views[n].abs().max()) <= 1e-5 * scale and float(v.abs().max()) <= 1e-5 * scale, n
        else:
            assert_close(v, views[n], rtol=RTOL, what=f"grad {n}")


def test_operator_path_keeps_torch_dropout():
    """use_engine = False: torch's F.dropout, the same masks it draws under the same torch.manual_seed."""
    b = make_batch(2, 16)
    oracle, model = make_models(2)
    oracle.train()
    model.train()
    model.use_engine = False
    oracle.dropout = model.dropout = 0.25
    bc = b.to("cuda")
    N, H = b.x.size(0), model.hidden_channels
    torch.manual_seed(21)
    with torch.no_grad():
        g, l = model(*forward_args(bc))
    assert model._engine is None                      # the engine never ran
    torch.manual_seed(21)
    masks = {f"bn{i}": (torch.nn.functional.dropout(torch.ones(N, H, device="cuda"), 0.25, True) != 0).cpu()
             for i in range(len(model.bns))}
    with torch.no_grad():
        go, lo = oracle_forward(oracle, *forward_args(b), dropout_masks=masks)
    assert_close(g, go, what="operator path global_predict")
    assert_close(l, lo, what="operator path local_predict")


def test_same_seed_same_masks():
    """Two models with the same seed_dropout draw the same masks over three training steps; another seed does not.
    Compared on the zero patterns of x[1] (parameters already differ in the last bits through float atomics)."""
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    _, m0 = make_models(2)
    m0.dropout = 0.3
    m0.train()
    models = [m0, copy.deepcopy(m0), copy.deepcopy(m0)]
    opts = [FusedAdam(FlatParams(m), lr=1e-3) for m in models]
    for m, s in zip(models, (SEED, SEED, SEED + 1)):
        m.seed_dropout(s)
    bc = make_batch(2, 32).to("cuda")
    n = bc.x.size(0) * m0.hidden_channels
    for step in range(3):
        zs = []
        for m, o in zip(models, opts):
            fused_train_step(m, o, bc, 0.5)
            zs.append((_saved_acts(m, *_sizes(bc))[1] == 0).cpu())
        same = int((zs[0] != zs[1]).sum())
        other = int((zs[0] != zs[2]).sum())
        assert same <= 1e-5 * n, (step, same)          # a ReLU argument within rounding of 0 may flip
        assert other >= 0.05 * n, (step, other)
