"""-m gpu: padded batches and per-bucket graph replay (train.BucketedTrainStep, train.evaluate_bucketed).

A batch padded into its capacity bucket (pert_batch_pad: ghost graphs in the tail, the real {N, B} in a device word)
must compute, for the real graphs, what the eager unpadded step computes: loss, every gradient, the BatchNorm batch
and running statistics, num_batches_tracked, the dropout masks; the bucketed step and eval must follow the eager ones
over shuffled, variable-size batches."""
import copy

import numpy as np
import pytest
import torch

from tests.helpers import assert_close, assert_grads_close, is_structural_zero_grad, make_batch, make_models

pytestmark = pytest.mark.gpu


def _engine_step(model, opt, data, live=None):
    """One step up to the gradients (no Adam): -> loss; gradients in opt.fp.grad, BN state in the model."""
    from pert_gnn_kdd23_b200.train import _fused_fwd_bwd

    loss, _ = _fused_fwd_bwd(model, opt, data, 0.5, None, None, use_index_cache=False, live=live)
    torch.cuda.synchronize()
    return loss.clone()


def _bn_state(model):
    eng = model._engine
    return eng.bn_running.clone(), eng.bn_nbt.clone()


def _pair(cfg=1, p=0.0):
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam

    _, ma = make_models(cfg)
    mb = copy.deepcopy(ma)
    for m in (ma, mb):
        m.dropout = p
        m.seed_dropout(1234)
    return (ma, FusedAdam(FlatParams(ma), lr=1e-3)), (mb, FusedAdam(FlatParams(mb), lr=1e-3))


# ------------------------------------------------------------------------------------------------------ 1. pad kernel
@pytest.mark.parametrize("attr_cols,patterns", [(2, 1), (4, 3)])
def test_pad_kernel_layout(attr_cols, patterns):
    from pert_gnn_kdd23_b200.train import PaddedBatch, bucket_caps

    d = make_batch(1, 21, seed=5, patterns=patterns, edge_attr_cols=attr_cols).to("cuda")
    N, E, B = d.x.size(0), d.edge_index.size(1), d.num_graphs
    caps = bucket_caps(N, E, B)
    Nc, Ec, Bc = caps
    buf = PaddedBatch(caps, d)
    # every capacity buffer sits inside a larger allocation filled with a sentinel: nothing past it may change
    guards = {}
    for k in ("x", "cat_X", "edge_index", "edge_attr", "batch", "entry_id", "y", "rt_probs", "pattern_num_nodes",
              "live"):
        t = getattr(buf, k)
        big = torch.full((t.numel() + 4096,), 77, dtype=t.dtype, device=t.device)
        setattr(buf, k, big[:t.numel()].view(t.shape))
        guards[k] = big
    buf.fill(d)
    torch.cuda.synchronize()
    for k, big in guards.items():
        n = getattr(buf, k).numel()
        assert bool((big[n:] == 77).all()), f"{k}: written past the capacity buffer"
    eq = lambda a, b: bool(torch.equal(a, b))
    assert eq(buf.x[:N], d.x) and eq(buf.cat_X[:N], d.cat_X) and eq(buf.batch[:N], d.batch)
    assert eq(buf.edge_index[:, :E], d.edge_index) and eq(buf.edge_attr[:E], d.edge_attr)
    assert eq(buf.rt_probs[:N], d.rt_probs.reshape(N, 1)) and eq(buf.pattern_num_nodes[:N], d.pattern_num_nodes)
    assert eq(buf.entry_id[:B], d.entry_id) and eq(buf.y[:B], d.y)
    assert buf.live.tolist() == [N, B]
    ng, bg = Nc - N, Bc - B
    j = torch.arange(ng, device="cuda")
    assert eq(buf.batch[N:], B + torch.clamp(j, max=bg - 1))
    k = torch.arange(Ec - E, device="cuda")
    assert eq(buf.edge_index[0, E:], N + k % ng) and eq(buf.edge_index[1, E:], N + k % ng)
    assert bool((buf.x[N:] == 0).all()) and bool((buf.cat_X[N:] == 0).all()) and bool((buf.edge_attr[E:] == 0).all())
    assert bool((buf.rt_probs[N:] == 0).all()) and bool((buf.pattern_num_nodes[N:] == 1).all())
    assert bool((buf.entry_id[B:] == 0).all()) and bool((buf.y[B:] == 1).all())
    assert bool((torch.diff(buf.batch) >= 0).all())


# ------------------------------------------------------------------------------- 2. one step, padded vs unpadded
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("attr_cols,patterns", [(2, 1), (4, 3)])
def test_padded_step_matches_unpadded(p, attr_cols, patterns):
    from pert_gnn_kdd23_b200.train import PaddedBatch, bucket_caps

    (ma, oa), (mb, ob) = _pair(1, p)
    d = make_batch(1, 32, seed=7, patterns=patterns, edge_attr_cols=attr_cols).to("cuda")
    la = _engine_step(ma, oa, d)
    buf = PaddedBatch(bucket_caps(d.x.size(0), d.edge_index.size(1), d.num_graphs), d).fill(d)
    lb = _engine_step(mb, ob, buf, live=buf.live)
    assert_close(lb, la, rtol=1e-4, what="loss")
    assert_grads_close(list(mb.named_parameters()), list(ma.named_parameters()), 1e-4, n_convs=len(ma.convs))
    (ra, na), (rb, nb) = _bn_state(ma), _bn_state(mb)
    assert_close(rb, ra, rtol=1e-4, what="BN running statistics")
    assert torch.equal(na, nb) and int(na[0]) == 1
    if p > 0:                                 # the dropout masks of the real rows did not move
        act_a, act_b = ma._engine.active_relus(), mb._engine.active_relus()
        N = d.x.size(0)
        for k in act_a:
            if k.startswith("bn"):
                assert torch.equal(act_a[k], act_b[k][:N]), k


# ------------------------------------------------------------- 2b. one padded step against the fp32 / fp64 oracles
SEED = 0x5EED_0BAD_CAFE


def _padded_oracle_parity(b, cfg, p, tag):
    """One padded training step (``_fused_fwd_bwd`` on a ``PaddedBatch``, the path BucketedTrainStep runs) against the
    fp32 (reference path) and fp64 (arbiter) oracles on the UNPADDED batch, differentiated on the padded run's active
    ReLUs restricted to the real rows and graphs, with the dropout masks restated for the real rows (the mask depends on
    row and column only, so padding does not move it).  Global predictions, loss, every gradient, the BatchNorm running
    statistics and num_batches_tracked (tests/test_gpu_fullsize.py, _full_parity)."""
    from oracle import model_oracle
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, PaddedBatch, _fused_fwd_bwd, bucket_caps
    from tests.dropout_ref import dropout_masks, oracle_forward
    from tests.helpers import RTOL, assert_close_ref, assert_grads_close_ref, forward_args

    a32 = forward_args(b)
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    oracle, model = make_models(cfg)
    for m in (oracle, model):
        m.dropout = p
        m.train()
    oracle64 = copy.deepcopy(oracle).double()
    model.seed_dropout(SEED)
    opt = FusedAdam(FlatParams(model), lr=1e-3)
    bc = b.to("cuda")
    N, E, B = bc.x.size(0), bc.edge_index.size(1), bc.num_graphs
    caps = bucket_caps(N, E, B)
    buf = PaddedBatch(caps, bc).fill(bc)
    seed, step = [int(v) for v in model.dropout_state().cpu()]
    eng = model.engine(opt.fp)
    rec = {}
    fwd = eng.forward

    def recording_forward(*args, **kw):                # keep the predictions of the padded forward
        out = fwd(*args, **kw)
        rec["g"] = out[0]
        return out

    eng.forward = recording_forward
    try:
        loss_c, _ = _fused_fwd_bwd(model, opt, buf, 0.5, None, None, use_index_cache=False, live=buf.live)
    finally:
        del eng.forward
    torch.cuda.synchronize()
    assert eng._saved[8:11] == caps                   # the engine really ran at the capacity sizes
    gc = rec["g"][:B]
    act = model._engine.active_relus()
    relu = {k: (v[:B] if k == "head" else v[:N]).cpu() for k, v in act.items()}
    drop = dropout_masks(seed, step, N, model.hidden_channels, p, len(model.bns)) if p > 0 else None
    go, _ = oracle_forward(oracle, *a32, relu_masks=relu, dropout_masks=drop)
    go64, _ = oracle_forward(oracle64, *a64, relu_masks=relu, dropout_masks=drop)
    loss_o = model_oracle.torch_quantile_loss(b.y.float(), go.flatten(), 0.5)
    loss_64 = model_oracle.torch_quantile_loss(b.y.double(), go64.flatten(), 0.5)
    loss_o.backward()
    loss_64.backward()
    assert_close_ref(gc, go, go64, what=f"{tag} global_predict")
    assert_close_ref(loss_c.reshape(()), loss_o, loss_64, what=f"{tag} loss")
    assert_grads_close_ref(model.named_parameters(), oracle.named_parameters(), oracle64.named_parameters(), RTOL,
                           n_convs=len(model.convs))
    b32, b64 = dict(oracle.named_buffers()), dict(oracle64.named_buffers())
    for n, bbuf in model.named_buffers():
        assert_close_ref(bbuf.float(), b32[n].float(), b64[n].double(), what=f"{tag} {n}")


@pytest.fixture(scope="module")
def trace_store_batch():
    """A PERT-store batch: 4 edge-attribute columns, entries with 1-3 patterns each, assembled on the device."""
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    store = PatternStore.from_artifacts(make_trace_artifacts(seed=7, n_traces=400), "cuda")
    d = store.assemble(list(range(0, 400, 2))[:190])
    store.check()
    assert d.edge_attr.size(1) == 4 and d.x.size(0) >= 4096
    return d.to("cpu")


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("case", ["cfg2_jitter", "cfg3", "pert_store"])
def test_padded_step_matches_oracles(case, p, trace_store_batch):
    """cfg2 with jittered graph sizes (H = 64, two BatchNorms, the node-linear kernel that applies BatchNorm at
    N >= 4096), a cfg3 batch (H = 128, power-law graph sizes) and a PERT-store batch."""
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.synthetic import make_data_list

    if case == "cfg2_jitter":
        b, cfg = Batch.from_data_list(make_data_list(2, num_graphs=96, jitter=0.2)), 2
    elif case == "cfg3":
        b, cfg = make_batch(3, 128), 3
    else:
        b, cfg = trace_store_batch, 2
    _padded_oracle_parity(b, cfg, p, f"{case} p={p}")


# ---------------------------------------------------------------------------------- 3. ghosts are inert, and visibly so
def _ghost_run(base_models, d, caps, scramble=False, count_ghosts=False):
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, PaddedBatch

    m = copy.deepcopy(base_models)
    opt = FusedAdam(FlatParams(m), lr=1e-3)
    buf = PaddedBatch(caps, d).fill(d)
    N, E, B = d.x.size(0), d.edge_index.size(1), d.num_graphs
    if scramble:                              # random finite in-range ghost content (structure kept ghost-only)
        g = torch.Generator(device="cuda").manual_seed(11)
        buf.x[N:] = torch.randn(buf.x[N:].shape, generator=g, device="cuda")
        buf.cat_X[N:] = torch.randint(0, m.cat_embedding[0].num_embeddings, buf.cat_X[N:].shape, generator=g,
                                      device="cuda")
        buf.edge_attr[E:, 0] = torch.randint(0, m.interface_embeds.num_embeddings, (buf.edge_attr.size(0) - E,),
                                             generator=g, device="cuda")
        buf.edge_attr[E:, 1] = torch.randint(0, m.rpctype_embeds.num_embeddings, (buf.edge_attr.size(0) - E,),
                                             generator=g, device="cuda")
        buf.entry_id[B:] = torch.randint(0, m.entry_embeds.num_embeddings, buf.entry_id[B:].shape, generator=g,
                                         device="cuda")
        buf.rt_probs[N:] = torch.rand(buf.rt_probs[N:].shape, generator=g, device="cuda")
        buf.pattern_num_nodes[N:] = 1 + 5 * torch.rand(buf.pattern_num_nodes[N:].shape, generator=g, device="cuda")
        buf.y[B:] = torch.randint(1, 1000, buf.y[B:].shape, generator=g, device="cuda")
    if count_ghosts:
        buf.live.copy_(torch.tensor([caps[0], caps[2]], device="cuda"))
    loss = _engine_step(m, opt, buf, live=buf.live)
    return m, loss


def test_ghosts_are_inert_and_a_leak_is_detected():
    from pert_gnn_kdd23_b200.train import bucket_caps

    _, base = make_models(1)
    base.dropout = 0.0
    d = make_batch(1, 32, seed=9).to("cuda")
    caps = bucket_caps(d.x.size(0), d.edge_index.size(1), d.num_graphs)
    ref, lref = _ghost_run(base, d, caps)
    big = tuple(2 * c for c in caps)
    variants = {"2x capacity": (big, False), "scrambled ghosts": (caps, True), "2x + scrambled": (big, True)}
    for what, (cp, scr) in variants.items():
        m, loss = _ghost_run(base, d, cp, scramble=scr)
        assert_close(loss, lref, rtol=1e-5, what=f"{what}: loss")
        assert_grads_close(list(m.named_parameters()), list(ref.named_parameters()), 1e-5, n_convs=len(ref.convs))
        assert_close(m._engine.bn_running, ref._engine.bn_running, rtol=1e-5, what=f"{what}: BN running stats")
    # control: the ghosts counted as real (live = capacity) must break the same bars
    m, loss = _ghost_run(base, d, caps, scramble=True, count_ghosts=True)
    with pytest.raises(AssertionError):
        assert_close(m._engine.bn_running[:, 0], ref._engine.bn_running[:, 0], rtol=1e-5, what="control: BN mean")
    with pytest.raises(AssertionError):
        assert_grads_close(list(m.named_parameters()), list(ref.named_parameters()), 1e-5, n_convs=len(ref.convs))


# --------------------------------------------------------------------------------- 4. trajectory over shuffled batches
@pytest.fixture(scope="module")
def pert_store():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts

    art, _ = make_pert_artifacts(seed=3, n_patterns=64, n_entries=24, n_traces=400, device="cuda")
    return PatternStore.from_artifacts(art, "cuda")


def _store_pair(p):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam

    torch.manual_seed(0)
    ma = SAGEDeterministic(*model_args(2)).cuda()
    mb = copy.deepcopy(ma)
    for m in (ma, mb):
        m.dropout = p
        m.seed_dropout(99)
    return (ma, FusedAdam(FlatParams(ma), lr=1e-3)), (mb, FusedAdam(FlatParams(mb), lr=1e-3))


def _sync(dst, src):
    """(model, optimizer) dst := src in place -- parameters, Adam moments and step, BatchNorm running statistics and
    dropout counter -- so the graphs captured over dst's buffers stay valid."""
    (mb, ob), (ma, oa) = dst, src
    ob.fp.flat.copy_(oa.fp.flat)
    ob.m.copy_(oa.m)
    ob.v.copy_(oa.v)
    ob.t = oa.t
    mb._engine.bn_running.copy_(ma._engine.bn_running)
    mb._engine.bn_nbt.copy_(ma._engine.bn_nbt)
    mb.dropout_state().copy_(ma.dropout_state())


def _trajectory(store, batches, reserve, free_steps=8):
    """BucketedTrainStep against eager fused_train_step from identical weights, p = 0.1.  The first ``free_steps``
    steps run freely and the parameters are compared after them; from then on the bucketed side is reset to the eager
    side before every step, and each step's loss, every gradient and the BatchNorm running statistics are compared
    directly (no Adam between the two sides to normalise a difference away) -- replayed steps included."""
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, bucket_caps, fused_train_step

    a, b = _store_pair(0.1)
    (ma, oa), (mb, ob) = a, b
    step = BucketedTrainStep(mb, ob, 0.5)
    if reserve is not None:
        step.reserve(*reserve)
    visits, n = {}, 0
    for d in batches:
        if n >= free_steps:
            _sync(b, a)
        la = fused_train_step(ma, oa, d, 0.5)
        r0 = step.replays
        lb = step(d)
        assert_close(lb, la, rtol=1e-4, what=f"loss step {n}")
        key = bucket_caps(d.x.size(0), d.edge_index.size(1), d.num_graphs)
        visits[key] = visits.get(key, 0) + 1
        assert step.replays - r0 == (visits[key] > 1), f"step {n}: first visit eager, every later visit replayed"
        n += 1
        if n == free_steps:
            # parameters after free_steps steps, 2e-3 element-wise, skipping the zero-gradient parameters.  The
            # attention-logit weights carry cancellation-limited gradients whose rounding follows the tile geometry,
            # i.e. the padded sizes (tests/helpers.py, _check_one_grad); Adam turns that into +-lr on their smallest
            # elements, so they are held to the norm-wise 2e-2 of that rule.  The per-step comparisons below check
            # their gradients directly.
            pa = dict(ma.named_parameters())
            for name, prm in mb.named_parameters():
                if is_structural_zero_grad(name, len(ma.convs)):
                    continue
                logit = any(t in name for t in (".lin_query.", ".lin_key.", ".lin_edge."))
                assert_close(prm, pa[name], rtol=2e-2 if logit else 2e-3, norm_only=logit,
                             what=f"param {name} after {n} steps")
            assert torch.equal(ma._engine.bn_nbt, mb._engine.bn_nbt)
            assert_close(mb._engine.bn_running, ma._engine.bn_running, rtol=2e-3, what="BN running statistics")
        elif n > free_steps:
            # 1e-3: the two sides run different tile geometries over ~10^6 BatchNorm ReLU arguments, so a few of them
            # can land on the other side of zero (see _full_parity in tests/test_gpu_fullsize.py); the exact
            # same-linear-piece comparison is test_padded_step_matches_oracles
            assert_grads_close(list(mb.named_parameters()), list(ma.named_parameters()), 1e-3,
                               n_convs=len(ma.convs))
            assert_close(mb._engine.bn_running, ma._engine.bn_running, rtol=1e-4, what=f"BN running stats step {n}")
            assert torch.equal(ma._engine.bn_nbt, mb._engine.bn_nbt)
    assert n > free_steps + 4
    assert step.capture_error is None, step.capture_error
    assert step.replays == n - len(visits)            # exactly: every visit but the first of each bucket replays
    assert step.captures == sum(v > 1 for v in visits.values()) + step.invalidations
    assert 1.0 < step.pad_ratio < 1.25
    return step, visits


def test_bucketed_trajectory_matches_eager(pert_store):
    from pert_gnn_kdd23_b200.store import StoreLoader

    ids = list(range(len(pert_store)))[:300]          # 300 = 9 x 32 + 12: a partial last batch
    loader = StoreLoader(pert_store, ids, 32, shuffle=True, generator=torch.Generator().manual_seed(5))
    step, visits = _trajectory(pert_store, (d for _ in range(2) for d in loader), loader.max_sizes())
    assert step.invalidations == 0
    assert step.replays >= len(visits)                # buckets really repeat over the two shuffled epochs


def test_bucketed_growing_buckets_invalidate_and_still_match(pert_store):
    ids = np.arange(len(pert_store))
    sizes = np.array([pert_store.sizes([i])[0] for i in ids])
    order = ids[np.argsort(sizes, kind="stable")]
    groups = [order[i:i + 48] for i in range(0, 240, 48)]     # batches of increasing size
    # each batch three times in a row (eager, capture + replay, replay), then the next, bigger one; at the end the
    # first one again, whose graph points into a workspace the bigger buckets have replaced
    seq = [g for g in groups for _ in range(3)] + [groups[0]] * 2
    step, visits = _trajectory(pert_store, (pert_store.assemble(g) for g in seq), None)
    assert step.invalidations >= 1


# ---------------------------------------------------------------------------------------------------------------- 5. eval
def test_evaluate_bucketed_matches_evaluate(pert_store):
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import evaluate, evaluate_bucketed

    (ma, oa), _ = _store_pair(0.0)
    loader = StoreLoader(pert_store, list(range(len(pert_store)))[:350], 64)   # 5 x 64 + 30
    from pert_gnn_kdd23_b200.train import fused_train_step

    for d in loader:                                # trained a little: running statistics are not the initial ones
        fused_train_step(ma, oa, d, 0.5)
    want = evaluate(ma, loader, "cuda")
    for rep in range(3):                            # eager, capture + replay, replay
        got = evaluate_bucketed(ma, loader, "cuda")
        for g, w, what in zip(got, want, ("mae", "mape", "quantile")):
            assert abs(g - w) <= 1e-5 * abs(w), (rep, what, g, w)
    st = ma.__dict__["_bucketed_eval"]
    assert st.metrics.count == 350
    assert all(e["state"] == "graph" for e in st.buckets.values())      # the graphs persist across calls


def test_evaluate_bucketed_after_the_engine_is_recreated(pert_store):
    """Re-flattening the parameters re-creates the engine (new flat buffer, new workspace, its generation counter
    starting over): graphs captured over the old engine must not be replayed."""
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import FlatParams, evaluate, evaluate_bucketed, fused_train_step

    (ma, oa), _ = _store_pair(0.0)
    loader = StoreLoader(pert_store, list(range(len(pert_store)))[:200], 64)
    for d in loader:
        fused_train_step(ma, oa, d, 0.5)
    for _ in range(2):
        evaluate_bucketed(ma, loader, "cuda")         # graphs captured over the first engine
    old = ma._engine
    FlatParams(ma)                                    # parameters move into a new flat buffer
    with torch.no_grad():
        for prm in ma.parameters():
            prm.mul_(0.5)                             # ... and change: a stale graph would read the old values
    want = evaluate(ma, loader, "cuda")
    assert ma._engine is not old
    for rep in range(2):
        got = evaluate_bucketed(ma, loader, "cuda")
        for g, w, what in zip(got, want, ("mae", "mape", "quantile")):
            assert abs(g - w) <= 1e-5 * abs(w), (rep, what, g, w)
    st = ma.__dict__["_bucketed_eval"]
    assert all(e["state"] == "graph" and e["engine"] is ma._engine for e in st.buckets.values())
