"""-m gpu tests of the multi-quantile global head (tests/quantile_ref.py derives every bar):

* the head kernels at T in {1, 2, 3, 4, 8} outputs on their own inputs, at every kernel and padded width, from one graph
  to 131,075, with hot, uniform and last-row entry ids; the intermediates come from pert_model_workspace_offset_q;
* pert_pinball_loss_q and pert_eval_metrics_q against fp64 (B up to 10^6, levels at 0 and 1, ties, live ghosts), and at
  T = 1 against the plain calls;
* a T = 4 model at the cfg2 sizes against the fp32 / fp64 oracle whose global_linear2 is a PygLinear(H, 4);
* a one-level model against the reference model over graph replays, the padding of the packed [T, Hp] head after Adam
  steps, the four training paths against each other, predict and evaluate_bucketed."""
import copy
import ctypes
import math

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from tests import engine_parts_ref as R
from tests import quantile_ref as Q
from tests.helpers import assert_close, assert_grads_close, forward_args, make_batch

pytestmark = pytest.mark.gpu

KERNEL_WIDTHS = (4, 8, 16, 32, 64, 96, 128, 192, 256)
PADDED_WIDTHS = (5, 48, 100, 200)
CAT_ROWS = 6
N_ENTRY = 37
LEVELS = {1: (0.5,), 2: (0.5, 0.9), 3: (0.1, 0.5, 0.9), 4: (0.5, 0.9, 0.95, 0.99),
          8: (0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 0.99, 1.0)}
LOSS_LEVELS = {2: (0.0, 1.0), 3: (0.0, 0.5, 1.0), 4: (0.05, 0.5, 0.95, 1.0), 8: LEVELS[8]}
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest error as a fraction of its bar:")
        for k in sorted(WORST):
            print(f"  {k:28s} {WORST[k]:.3g}")


def _check(what, got, ref, bar, tag):
    w = R.worst(got, ref, bar)
    WORST[what] = max(WORST.get(what, 0.0), w)
    assert w <= 1.0, f"{tag} {what}: {w:.3g} of its bar"


def _note(what, r):
    WORST[what] = max(WORST.get(what, 0.0), float(r))


def _c_levels(t):
    return (ctypes.c_float * len(t))(*t)


# ------------------------------------------------------------------------------------------------------ head kernels
def _head_model(H, T, seed=0):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    torch.manual_seed(seed)
    m = SAGEDeterministic(4, [CAT_ROWS], N_ENTRY - 1, 7, 3, H, 2, 0.0, quantiles=LEVELS[T]).cuda()
    return m, m.engine()


def _ws(eng, b, which, shape):
    off = eng.lib.pert_model_workspace_offset_q(ctypes.byref(eng.desc), eng.n_out, b.N, b.E, b.B, which, 0)
    assert off >= 0, (which, off)
    return eng.ws[off:off + math.prod(shape)].view(shape).cpu()


def _head_case(model, eng, B, ent_mode, seed):
    from tests.test_gpu_engine_parts import _Batch, _entry_ids

    d, H, Hp, T = eng.desc, eng.desc.H, eng.Hp, eng.n_out
    tag = f"H={H} T={T} B={B} {ent_mode}"
    g = torch.Generator().manual_seed(seed)
    ids = _entry_ids(ent_mode, B, g)
    b = _Batch(model, B, torch.arange(B), ids, seed=seed)
    flat = eng.fp.flat.detach().cpu()
    model.train()
    with torch.no_grad():
        gp, _ = eng.forward(b.x, b.cat_X, b.entry_id, b.probs, b.pnn, b.batch, b.index, True)
    torch.cuda.synchronize()
    assert gp.shape == (B, T)
    W1, b1, W2, b2, ent = Q.head_params_q(d, Hp, flat, T)
    z = _ws(eng, b, 2, (B, 2 * Hp))
    h1 = _ws(eng, b, 1, (B, Hp))
    assert torch.equal(z[:, Hp:], ent[ids]), tag
    pre, pre_bar, _, _ = R.head_fwd_ref(z, W1, b1, W2[0], b2[:1], h1)
    _check("head h1", h1, torch.relu(pre), pre_bar, tag)
    pred, bar = Q.head_fwd_ref_q(h1, W2, b2)
    _check("head global_pred", gp.cpu(), pred, bar, tag)
    dg = torch.randn(B, T, generator=g)
    dg[torch.rand(B, T, generator=g) < 0.25] = 0.0
    grads = torch.zeros_like(eng.fp.flat)
    with torch.no_grad():
        eng.backward(dg.cuda(), None, grads=grads)
    torch.cuda.synchronize()
    gc = grads.cpu()
    ref = Q.head_bwd_ref_q(dg, z, h1, W1, W2, ids, d.n_entry)
    _check("head dpool", _ws(eng, b, 3, (B, Hp)), *ref["dpool"], tag)
    got = {"entry": R._mat(gc, d.off_entry, d.n_entry, H), "W1": R._mat(gc, d.off_g1_w, H, 2 * H),
           "b1": gc[d.off_g1_b:d.off_g1_b + H], "W2": R._mat(gc, d.off_g2_w, T, H),
           "b2": gc[d.off_g2_b:d.off_g2_b + T]}
    cut = {"entry": lambda t: t[:, :H], "W1": lambda t: torch.cat([t[:H, :H], t[:H, Hp:Hp + H]], 1),
           "b1": lambda t: t[:H], "W2": lambda t: t[:, :H], "b2": lambda t: t}
    for k, v in got.items():
        rv, rb = ref[k]
        _check(f"head d{k}", v, cut[k](rv), cut[k](rb), tag)


@pytest.mark.parametrize("T", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("H", KERNEL_WIDTHS + PADDED_WIDTHS)
def test_head_q(H, T):
    model, eng = _head_model(H, T)
    assert eng.n_out == T
    for i, (B, em) in enumerate(((1, "uniform"), (8, "hot"), (9, "last"), (4097, "uniform"))):
        _head_case(model, eng, B, em, seed=1000 * T + i)


@pytest.mark.parametrize("H,T", [(64, 4), (256, 8), (200, 3)])
def test_head_q_large_batch(H, T):
    model, eng = _head_model(H, T)
    _head_case(model, eng, 131075, "hot", seed=T)


# ------------------------------------------------------------------------------------------------------ loss
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pinball_q(y, yhat, taus, gs, live=None):
    B, T = yhat.shape
    lo = torch.full((1,), float("nan"), device="cuda")
    d = torch.full((B, T), float("nan"), device="cuda")
    p = _lib.ptr
    rc = _lib.lib().pert_pinball_loss_q(p(y), p(yhat), _c_levels(taus), T, B, Q.f32(gs), p(lo), p(d), p(live),
                                        _lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    return float(lo.item()), d.cpu().numpy()


@pytest.mark.parametrize("B", [1, 255, 257, 4097, 10 ** 6])
@pytest.mark.parametrize("T", [2, 3, 4, 8])
def test_pinball_q_matches_fp64(B, T):
    taus = LOSS_LEVELS[T]
    y, yhat = Q.quantile_data(B, T, seed=B + T)
    yd, yhd = _dev(y), _dev(yhat)
    for gs in (1.0, 0.125):
        loss, d = _pinball_q(yd, yhd, taus, gs)
        rl, rd = Q.pinball_q_worst(loss, d, *Q.pinball_q_ref(y, yhat, taus, gs), B * T)
        _note("pinball_q loss", rl)
        _note("pinball_q dyhat", rd)
        assert rl <= 1 and rd <= 1, (gs, rl, rd)


@pytest.mark.parametrize("live", [1, 255, 3000, 5000])
def test_pinball_q_live_ghosts(live):
    B, T = 4096, 4
    taus = LOSS_LEVELS[T]
    y, yhat = Q.quantile_data(B, T, seed=live)
    bl = min(B, live)
    y[bl:] = 1
    yhat[bl:] = np.resize(np.array([np.nan, np.inf, -np.inf], np.float32), (B - bl, T))
    word = torch.tensor([12345, live], dtype=torch.int64, device="cuda")
    loss, d = _pinball_q(_dev(y), _dev(yhat), taus, 0.5, word)
    assert math.isfinite(loss) and not d[bl:].any() and np.isfinite(d).all()
    rl, rd = Q.pinball_q_worst(loss, d, *Q.pinball_q_ref(y, yhat, taus, 0.5, live), bl * T)
    assert rl <= 1 and rd <= 1


@pytest.mark.parametrize("B", [1, 256, 257, 16385, 10 ** 6])
def test_one_level_equals_the_plain_calls(B):
    """T = 1: the loss is the plain kernel's, bit for bit; the metric sums follow the plain kernel's arithmetic, bit for
    bit within one block (B <= 256), and within the fp64 bar where blocks add in a run-dependent order."""
    from tests.loss_adam_ref import loss_data

    L, p = _lib.lib(), _lib.ptr
    y, yhat = loss_data(B, seed=B)
    yd, yhd = _dev(y), _dev(yhat)
    for tau in (0.0, 0.5, 0.95, 1.0):
        lq, dq = _pinball_q(yd, yhd.view(B, 1), (tau,), 0.125)
        lo = torch.empty(1, device="cuda")
        dp = torch.empty(B, device="cuda")
        assert L.pert_pinball_loss(p(yd), p(yhd), Q.f32(tau), B, Q.f32(0.125), p(lo), p(dp), _lib.stream()) == 0
        assert np.float32(lq).tobytes() == np.float32(lo.item()).tobytes(), tau
        assert np.array_equal(dq.reshape(-1).view(np.int32), dp.cpu().numpy().view(np.int32)), tau
        aq = torch.zeros(5, dtype=torch.float64, device="cuda")
        ap = torch.zeros(3, dtype=torch.float64, device="cuda")
        assert L.pert_eval_metrics_q(p(yd), p(yhd), _c_levels((tau,)), 1, B, p(aq), None, _lib.stream()) == 0
        assert L.pert_eval_metrics(p(yd), p(yhd), Q.f32(tau), B, p(ap), _lib.stream()) == 0
        got, want = aq.cpu().numpy(), ap.cpu().numpy()
        if B <= 256:
            assert np.array_equal(got[:3].view(np.int64), want.view(np.int64)), tau
        else:
            for g, w in zip(got[:3], want):
                assert abs(g - w) <= Q.metrics_q_bar(2 * B) * abs(w), (tau, g, w)
        ref = Q.metrics_q_ref(y, yhat[:, None], (tau,))
        assert got[3] == ref[3] and got[4] == 0.0


def _metrics_check(got, ref, T, n, tag):
    for t in range(T):
        for k, name in enumerate(("mae", "mape", "qloss")):
            g, r = got[4 * t + k], ref[4 * t + k]
            ratio = (0.0 if g == 0 else math.inf) if r == 0 else abs(g - r) / (Q.metrics_q_bar(n) * abs(r))
            _note(f"metrics_q {name}", ratio)
            assert ratio <= 1, (tag, t, name, g, r)
        assert got[4 * t + 3] == ref[4 * t + 3], (tag, t, "coverage")
    assert got[4 * T] == ref[4 * T], (tag, "crossing")


@pytest.mark.parametrize("B", [1, 256, 257, 16385, 10 ** 6])
@pytest.mark.parametrize("T", [2, 4, 8])
def test_eval_metrics_q_matches_fp64(B, T):
    taus = LOSS_LEVELS[T]
    y, yhat = Q.quantile_data(B, T, seed=7 * B + T)
    acc = torch.zeros(4 * T + 1, dtype=torch.float64, device="cuda")
    L, p = _lib.lib(), _lib.ptr
    assert L.pert_eval_metrics_q(p(_dev(y)), p(_dev(yhat)), _c_levels(taus), T, B, p(acc), None, _lib.stream()) == 0
    _metrics_check(acc.cpu().numpy(), Q.metrics_q_ref(y, yhat, taus), T, B, f"B={B} T={T}")


@pytest.mark.parametrize("live", [12345, 16385, 30000])
def test_eval_metrics_q_live_ghosts(live):
    B, T = 20000, 4
    taus = LEVELS[T]
    y, yhat = Q.quantile_data(B, T, seed=live)
    bl = min(B, live)
    y[bl:] = 1
    yhat[bl:] = np.float32(5.0)
    yhat[bl::2, 0] = np.float32(9.0)              # ghosts that would count as covered and as crossing
    acc = torch.zeros(4 * T + 1, dtype=torch.float64, device="cuda")
    word = torch.tensor([7, live], dtype=torch.int64, device="cuda")
    L, p = _lib.lib(), _lib.ptr
    assert L.pert_eval_metrics_q(p(_dev(y)), p(_dev(yhat)), _c_levels(taus), T, B, p(acc), p(word),
                                 _lib.stream()) == 0
    _metrics_check(acc.cpu().numpy(), Q.metrics_q_ref(y[:bl], yhat[:bl], taus), T, bl, f"live={live}")


# ------------------------------------------------------------------------------------------------------ whole model
def _cfg_pair(cfg, T):
    """(oracle with a PygLinear(H, T) global head on the CPU, quantile model on the GPU) with the same weights."""
    from oracle.model_oracle import OracleSAGEDeterministic, PygLinear
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args

    torch.manual_seed(0)
    oracle = OracleSAGEDeterministic(*model_args(cfg))
    oracle.global_linear2 = PygLinear(oracle.global_linear1.out_features, T)
    model = SAGEDeterministic(*model_args(cfg), quantiles=LEVELS[T])
    model.load_state_dict(oracle.state_dict())
    return oracle, model.cuda()


def test_cfg2_four_levels_against_the_oracle():
    """Forward [B, 4] and every parameter gradient of the mean pinball loss over the four levels, on the engine's linear
    piece of the network (tests/test_gpu_fullsize.py _full_parity), with that test's bars."""
    from pert_gnn_kdd23_b200.train import torch_quantile_loss
    from tests.helpers import assert_close_ref, assert_grads_close_ref

    oracle, model = _cfg_pair(2, 4)
    b = make_batch(2)
    a32 = forward_args(b)
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    oracle64 = copy.deepcopy(oracle).double()
    for m in (oracle, oracle64, model):
        m.train()
    taus = LEVELS[4]

    def loss_of(g, l, y):
        return torch_quantile_loss(y, g, taus) + 1e-3 * l.square().mean()

    bc = b.to("cuda")
    gc, lc = model(*forward_args(bc))
    assert gc.shape == (b.num_graphs, 4)
    masks = {k: v.cpu() for k, v in model._engine.active_relus().items()}
    loss_c = loss_of(gc, lc, bc.y.float())
    loss_c.backward()
    go, lo = oracle(*a32, relu_masks=masks)
    go64, lo64 = oracle64(*a64, relu_masks=masks)
    loss_o, loss_64 = loss_of(go, lo, b.y.float()), loss_of(go64, lo64, b.y.double())
    loss_o.backward()
    loss_64.backward()
    assert_close_ref(gc, go, go64, what="T=4 global_predict")
    assert_close_ref(lc, lo, lo64, what="T=4 local_predict")
    assert_close_ref(loss_c, loss_o, loss_64, what="T=4 loss")
    assert_grads_close_ref(model.named_parameters(), oracle.named_parameters(), oracle64.named_parameters(), 1e-4,
                           n_convs=len(model.convs))


def test_one_level_model_trains_like_the_reference_model():
    """quantiles=(0.5,) launches what the reference model launches (the plain entry points, the same counts).  Over 5
    graph replays (6 steps) the losses and parameters agree bit for bit where the step is deterministic; the engine adds some
    float sums with atomics, whose order may differ between two runs, so a difference must stay at that level."""
    from pert_gnn_kdd23_b200 import ops
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    b = make_batch(2, seed=5).to("cuda")
    runs = []
    for q in (None, (0.5,), None):            # the reference model twice: its own run-to-run difference
        torch.manual_seed(0)
        m = SAGEDeterministic(*model_args(2), quantiles=q).cuda()
        opt = FusedAdam(FlatParams(m), lr=1e-3)
        step = GraphedTrainStep(m, opt)
        losses, launches = [], []
        for _ in range(6):
            l0 = ops.LAUNCHES["n"]
            losses.append(float(step(b).item()))
            launches.append(ops.LAUNCHES["n"] - l0)
        assert step.replays == 5 and step.capture_error is None
        torch.cuda.synchronize()
        runs.append((losses, launches, opt.fp.flat.detach().cpu().clone()))
    (la, na, pa), (lb, nb, pb), (lc, nc, pc) = runs
    assert na == nb == nc
    same = la == lb and torch.equal(pa, pb)
    again = la == lc and torch.equal(pa, pc)
    print(f"one-level model vs reference model over 5 replays: {'bitwise equal' if same else 'not bitwise equal'}; "
          f"reference model vs itself: {'bitwise equal' if again else 'not bitwise equal'}")
    if not same:
        for x, y in zip(la, lb):
            assert abs(x - y) <= 1e-5 * abs(y), (la, lb)
        assert_close(pb, pa, rtol=1e-3, norm_only=True, what="parameters after 6 steps")


def test_padded_head_stays_zero_after_adam_steps():
    """H = 48 runs at Hp = 64: the packed [4, Hp] copy of global_linear2 holds the weights in columns [0, 48) and exact
    zeros in [48, 64) and in the slot's alignment tail after 20 Adam steps; every other padding slot of the packed
    region stays 0 too."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    args = list(model_args(1))
    args[5] = 48
    torch.manual_seed(0)
    m = SAGEDeterministic(*args, quantiles=LEVELS[4]).cuda()
    opt = FusedAdam(FlatParams(m), lr=1e-2)
    b = make_batch(1, 64, seed=3).to("cuda")
    for _ in range(20):
        fused_train_step(m, opt, b)
    m.eval()                                      # a forward packs the parameters Adam left
    with torch.no_grad():
        m(*forward_args(b))
    m.train()
    torch.cuda.synchronize()
    eng = m._engine
    d, H, Hp, T = eng.desc, 48, eng.Hp, 4
    assert Hp == 64
    nq = eng.lib.pert_model_packed_bytes_q(ctypes.byref(d), T) // 4
    n1 = eng.lib.pert_model_packed_bytes(ctypes.byref(d)) // 4
    packed = eng.ws[:nq].cpu()
    slot = packed[nq - R.al64(T * Hp):]
    w2 = slot[:T * Hp].view(T, Hp)
    flat = eng.fp.flat.detach().cpu()
    assert torch.equal(w2[:, :H], R._mat(flat, d.off_g2_w, T, H))
    assert int((w2[:, H:] != 0).sum()) == 0 and int((slot[T * Hp:] != 0).sum()) == 0
    mask = R.packed_pad_mask(d, Hp, len(m.convs), flat.numel())[:n1 - R.al64(Hp)]
    assert int((packed[:n1 - R.al64(Hp)][mask] != 0).sum()) == 0


@pytest.fixture(scope="module")
def pert_store():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts

    art, _ = make_pert_artifacts(seed=3, n_patterns=64, n_entries=24, n_traces=400, device="cuda")
    return art, PatternStore.from_artifacts(art, "cuda")


def _copy_state(dst, src):
    (mb, ob), (ma, oa) = dst, src
    ob.fp.flat.copy_(oa.fp.flat)
    ob.m.copy_(oa.m)
    ob.v.copy_(oa.v)
    ob.t = oa.t
    mb._engine.bn_running.copy_(ma._engine.bn_running)
    mb._engine.bn_nbt.copy_(ma._engine.bn_nbt)


def test_training_paths_agree_on_four_levels(pert_store):
    """GraphedTrainStep (replayed), BucketedTrainStep (replayed, on a shuffled, padded store batch), fused_train_step
    and the drop-in operator path (use_engine = False, autograd) from the same state: the loss and every gradient."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, FlatParams, FusedAdam, GraphedTrainStep,
                                           fused_train_step, train_step)

    _, store = pert_store
    loader = StoreLoader(store, list(range(len(store)))[:300], 40, shuffle=True,
                         generator=torch.Generator().manual_seed(2))
    batches = list(loader)
    torch.manual_seed(0)
    base = SAGEDeterministic(*model_args(2), quantiles=LEVELS[4]).cuda()
    pairs = []
    for _ in range(4):
        m = copy.deepcopy(base)
        opt = FusedAdam(FlatParams(m), lr=1e-3)
        m.engine(opt.fp)
        pairs.append((m, opt))
    ref, gr, bu, op = pairs
    for d in batches[:2]:                         # running statistics off their initial values
        fused_train_step(*ref, d)
    graphed, bucketed = GraphedTrainStep(*gr), BucketedTrainStep(*bu)
    bucketed.reserve(*loader.max_sizes())
    op[0].use_engine = False
    d = batches[2]
    snap = [t.clone() for t in (ref[1].fp.flat, ref[1].m, ref[1].v)]
    for call in range(3):                         # eager, capture + replay, replay
        for p in pairs:
            p[1].fp.flat.copy_(snap[0])
            p[1].m.copy_(snap[1])
            p[1].v.copy_(snap[2])
            p[1].t = ref[1].t
        for p in (gr, bu, op):
            _copy_state(p, ref)
        lr_ = float(fused_train_step(*ref, d).item())
        lg = float(graphed(d).item())
        lb = float(bucketed(d).item())
        lo = float(train_step(*op, d).item())
        for got, what in ((lg, "graphed"), (lb, "bucketed"), (lo, "operator path")):
            assert abs(got - lr_) <= 1e-4 * abs(lr_), (call, what, got, lr_)
        for p, what in ((gr, "graphed"), (bu, "bucketed"), (op, "operator path")):
            named = [(n, t) for n, t in p[0].named_parameters()]
            assert_grads_close(named, list(ref[0].named_parameters()), 1e-3, n_convs=len(base.convs))
    assert graphed.replays >= 1 and bucketed.replays >= 1
    assert graphed.capture_error is None and bucketed.capture_error is None


def _trace_requests(art, store):
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    return store._h_trace_entry.astype(np.int64), ts


def test_predict_and_evaluate_four_levels(pert_store):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import (EvalMetrics, FlatParams, FusedAdam, evaluate, evaluate_bucketed,
                                           fused_train_step, model_inputs, predict)

    art, store = pert_store
    torch.manual_seed(0)
    m = SAGEDeterministic(*model_args(2), quantiles=LEVELS[4]).cuda()
    opt = FusedAdam(FlatParams(m), lr=1e-3)
    loader = StoreLoader(store, list(range(len(store))), 64)
    for i, d in enumerate(loader):
        if i >= 4:
            break
        fused_train_step(m, opt, d)
    ent, ts = _trace_requests(art, store)
    got = predict(m, store, ent, ts, batch_size=96, asof=True)
    assert got.shape == (len(ent), 4) and got.dtype == torch.float32
    m.eval()
    with torch.no_grad():
        want = torch.cat([m(*model_inputs(store.assemble_requests(ent[i:i + 96], ts[i:i + 96], asof=True)))[0]
                          for i in range(0, len(ent), 96)])
    m.train()
    assert want.shape == got.shape
    assert_close(got, want, what="predict [Q, 4] vs eval forward")
    wi = predict(m, store, ent[:50], ts[:50], batch_size=32, asof=True, scenario_ids=np.full(50, -1))
    assert wi.shape == (50, 4)
    assert_close(wi, got[:50], what="what-if predict without a scenario")
    g, loc, ptr = predict(m, store, ent[:50], ts[:50], batch_size=32, asof=True, local=True)
    assert g.shape == (50, 4) and loc.dim() == 1 and ptr.shape == (51,)
    one = predict(m, store, ent[:5], ts[:5], asof=True)
    assert one.shape == (5, 4)

    eval_loader = StoreLoader(store, list(range(len(store)))[:350], 64)
    want_e = evaluate(m, eval_loader, "cuda")
    assert all(len(x) == 4 for x in want_e)
    for rep in range(3):
        got_e = evaluate_bucketed(m, eval_loader, "cuda")
        for gv, wv in zip(got_e, want_e):
            for a, b in zip(gv, wv):
                assert abs(a - b) <= 1e-5 * abs(b), (rep, gv, wv)
    st = m.__dict__["_bucketed_eval"]
    cov, cross = st.metrics.coverage(), st.metrics.crossing()
    assert len(cov) == 4 and all(0.0 <= c <= 1.0 for c in cov) and 0.0 <= cross <= 1.0
    ref = EvalMetrics("cuda", LEVELS[4])
    m.eval()
    with torch.no_grad():
        for d in eval_loader:
            ref.update(d.y, m(*model_inputs(d))[0])
    m.train()
    for a, b in zip(cov, ref.coverage()):
        assert abs(a - b) <= 0.01, (cov, ref.coverage())
    with pytest.raises(ValueError):
        evaluate(m, eval_loader, "cuda", tau=0.5)
