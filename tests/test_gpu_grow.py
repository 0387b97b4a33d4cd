"""Embedding growth on the GPU (train.grow_embeddings, FlatParams.grow, csrc/flat.cu).

1. The relayout is exact: old parameters and Adam state bit-identical, new slots 0, new rows the seeded N(0, 1) draws.
2. A grown model trains as a model built with the large tables from the start (whose extra rows never get a gradient
   before the new ids arrive), under GraphedTrainStep, BucketedTrainStep and the drop-in loop with torch.optim.Adam;
   every graph cache re-captures instead of replaying over freed memory.
3. A live store: append traces with new entries and interfaces, grow, train on the new range, predict the new entries
   against the fp32 / fp64 oracles.
4. A grown state_dict round-trips into a model built at the grown sizes; a second growth to the same store is a no-op.
"""
import copy

import numpy as np
import pytest
import torch

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_trace_table, model_args
from tests.helpers import (assert_close, assert_close_ref, elem_err, forward_args, is_structural_zero_grad,
                           make_batch)

pytestmark = pytest.mark.gpu

TABLES = ("cat", "entry", "interface", "rpctype")
GOLD_SEED = int(np.load(__file__.rsplit("/", 1)[0] + "/golden/ref_preprocess.npz")["seed"])


def _tables(m):
    return dict(zip(TABLES, (m.cat_embedding[0], m.entry_embeds, m.interface_embeds, m.rpctype_embeds)))


def _model(H, layers=2, rows=None, seed=0):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    a = list(model_args(1))
    a[5], a[6] = H, layers
    if rows is not None:
        a[1], a[2], a[3], a[4] = [rows["cat"]], rows["entry"] - 1, rows["interface"] - 1, rows["rpctype"] - 1
    torch.manual_seed(seed)
    return SAGEDeterministic(*a).cuda()


def _rows(m):
    return {k: e.num_embeddings for k, e in _tables(m).items()}


def _draws(rows, want, H, seed):
    """The rows grow_embeddings draws: table by table in TABLES order from one seeded generator."""
    g = torch.Generator("cuda")
    g.manual_seed(seed)
    return {k: torch.randn(want[k] - rows[k], H, generator=g, device="cuda") for k in TABLES if want[k] > rows[k]}


# ---- 1. the relayout is exact -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [32, 64, 100, 128])
@pytest.mark.parametrize("which", TABLES + ("all",))
def test_relayout_is_exact(H, which):
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, grow_embeddings

    model = _model(H)
    opt = FusedAdam(FlatParams(model))
    fp = opt.fp
    eng = model.engine(fp)
    opt.m.copy_(torch.randn_like(opt.m))
    opt.v.copy_(torch.rand_like(opt.v))
    fp.grad.copy_(torch.randn_like(fp.grad))
    opt.t = 7
    rows = _rows(model)
    add = {"cat": 5, "entry": 67, "interface": 1000, "rpctype": 3}
    want = {k: rows[k] + (add[k] if which in (k, "all") else 0) for k in TABLES}
    old = {n: p.detach().clone() for n, p in model.named_parameters()}
    old_m = {n: v.clone() for n, v in zip([n for n, _ in model.named_parameters()], fp.views_of(opt.m))}
    old_v = {n: v.clone() for n, v in zip([n for n, _ in model.named_parameters()], fp.views_of(opt.v))}
    bn = [eng.bn_running.clone(), eng.bn_nbt.clone()]
    got = grow_embeddings(model, opt, **{k: want[k] for k in TABLES if which in (k, "all")}, seed=11)
    assert got == want == _rows(model)
    draws = _draws(rows, want, H, 11)
    torch.cuda.synchronize()
    assert model._engine is None and opt.fp is fp and opt.t == 7
    tab = {id(e.weight): k for k, e in _tables(model).items()}
    expect_p = torch.zeros_like(fp.flat)
    expect_m, expect_v = torch.zeros_like(fp.flat), torch.zeros_like(fp.flat)
    for (n, p), (off, shape, _) in zip(model.named_parameters(), fp._layout):
        k = tab.get(id(p))
        r = old[n].shape[0] if old[n].dim() else 0
        assert p.data_ptr() == fp.flat.data_ptr() + off * 4 and tuple(p.shape) == shape
        full = torch.cat([old[n], draws[k]]) if k in draws else old[n]
        assert torch.equal(p.detach(), full), n
        expect_p[off:off + p.numel()] = full.reshape(-1)
        expect_m[off:off + old[n].numel()] = old_m[n].reshape(-1)
        expect_v[off:off + old[n].numel()] = old_v[n].reshape(-1)
        assert p.grad is not None and p.grad.data_ptr() == fp.grad.data_ptr() + off * 4, n
        if k in draws:
            assert r == rows[k] and tuple(p.shape) == (want[k], H)
    # whole buffers, bit for bit: padding and new slots 0, the gradient buffer 0
    for got_b, exp_b in ((fp.flat, expect_p), (opt.m, expect_m), (opt.v, expect_v)):
        assert torch.equal(got_b.view(torch.int32), exp_b.view(torch.int32))
    assert not fp.grad.any()
    new = model.engine(fp)
    assert new is not eng and new.desc.n_if == want["interface"] and new.desc.cat_rows[0] == want["cat"]
    assert torch.equal(new.bn_running, bn[0]) and torch.equal(new.bn_nbt, bn[1])


# ---- 2. equivalence with a model built large --------------------------------------------------------------------------
def _new_id_batch(b, shift):
    """``b`` with some ids moved up by ``shift`` (grown rows - old rows) into the rows only the grown tables have."""
    b = b._apply(torch.clone)
    b.entry_id[::2] += shift["entry"]
    b.edge_attr[::3, 0] += shift["interface"]
    b.edge_attr[::5, 1] += shift["rpctype"]
    b.cat_X[::4, 0] += shift["cat"]
    return b


def _pair(H, seed=3):
    """(A small, B large with A's initial rows and A's future grown rows, the grown row counts)."""
    # rpctype grows 4 -> 8 only: the conv kernels keep a shared-memory table path for n_rpc <= 8, so A and B run the same
    # conv kernels before and after the growth
    small = {"cat": 4096, "entry": 64, "interface": 1024, "rpctype": 4}
    big = {"cat": 8192, "entry": 128, "interface": 2048, "rpctype": 8}
    a = _model(H, rows=small, seed=seed)
    b = _model(H, rows=big, seed=seed + 1)
    draws = _draws(small, big, H, 5)
    sd = a.state_dict()
    for k, e in _tables(a).items():
        name = next(n for n, p in a.named_parameters() if p is e.weight)
        sd[name] = torch.cat([sd[name], draws[k]])
    b.load_state_dict(sd)
    return a, b, big


# named: grow_embeddings is handed the optimizer; without it the FlatParams relays the m and v of its FusedAdam itself.
# drop: between-layer dropout, masks from the engine's dropout counter, which must carry over into the new engine
@pytest.mark.parametrize("mode,named,drop", [("graphed", True, 0.0), ("bucketed", False, 0.0), ("torch_adam", True, 0.0),
                                          ("graphed", False, 0.2), ("torch_adam", True, 0.2)])
def test_grown_equals_built_large(mode, named, drop):
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, FlatParams, FusedAdam, GraphedTrainStep,
                                           grow_embeddings, train_step)

    H = 64
    a, b, big = _pair(H)
    small = _rows(a)
    old = [make_batch(1, num_graphs=24, seed=s).to("cuda") for s in (1, 2)]
    for x in old:
        x.edge_attr[:, 1] %= small["rpctype"]
    new = [_new_id_batch(x, {k: big[k] - small[k] for k in TABLES}) for x in old]
    steps, opts = [], []
    # eps = 1e-4: lin_key.bias and the lin_skip.bias of a conv feeding BatchNorm have a gradient that is 0 in exact
    # arithmetic, and with eps = 1e-8 Adam turns its rounding noise into full lr-sized steps that differ between A and B
    # (which round differently: the table GEMMs' dispatch depends on the row count) and reach the BatchNorm running
    # means.  eps = 1e-4 keeps those steps negligible and leaves the real updates (gradients >> 1e-4) as they are
    for m in (a, b):
        m.dropout = drop
        m.seed_dropout(7)
        if mode == "torch_adam":
            o = torch.optim.Adam(m.parameters(), lr=1e-3, eps=1e-4)
            steps.append(lambda d, m=m, o=o: train_step(m, o, d))
        else:
            o = FusedAdam(FlatParams(m), lr=1e-3, eps=1e-4)
            steps.append((GraphedTrainStep if mode == "graphed" else BucketedTrainStep)(m, o))
        opts.append(o)
    losses = [[], []]
    for i in range(4):                                   # eager, capture, replays
        for j in range(2):
            losses[j].append(steps[j](old[i % 2]).detach().clone().reshape(()))
    drop_state = a.dropout_state()
    assert grow_embeddings(a, opts[0] if named else None, entry=big["entry"], interface=big["interface"],
                           rpctype=big["rpctype"], cat=big["cat"], seed=5) == big
    assert a.dropout_state() is drop_state
    if mode != "torch_adam":
        assert opts[0].m.numel() == opts[0].v.numel() == opts[0].fp.numel
    for i in range(6):                                   # old buffers: invalidated graphs; new ids: new keys
        d = (old, new)[i % 2][i // 2 % 2]
        for j in range(2):
            losses[j].append(steps[j](d).detach().clone().reshape(()))
    torch.cuda.synchronize()
    if mode != "torch_adam":
        assert steps[0].invalidations >= 1 and steps[1].invalidations == 0
        assert steps[0].capture_error is None and steps[1].capture_error is None
    la, lb = torch.stack(losses[0]), torch.stack(losses[1])
    report = {"loss": torch.equal(la, lb)}
    assert_close(la, lb, what="losses")
    pb = dict(b.named_parameters())
    n_convs = len(a.convs)
    # the tensors whose gradient is 0 in exact arithmetic hold rounding noise only: not compared (they do not reach
    # the losses or the training-mode outputs, which are compared)
    noise = [n for n, _ in a.named_parameters() if is_structural_zero_grad(n, n_convs)]

    def close(x, y, n, what):
        if n in noise:
            return
        report[f"{n} {what}"] = torch.equal(x, y)
        if what in ("m", "v", "exp_avg", "exp_avg_sq") and (".lin_key." in n or ".lin_query." in n):
            # attention-logit gradients are cancellation-limited (tests/helpers.py _check_one_grad): norm-wise bar
            assert_close(x, y, rtol=2e-2, norm_only=True, what=f"{mode}: {n} {what}")
        else:
            assert_close(x, y, what=f"{mode}: {n} {what}")

    for n, p in a.named_parameters():
        close(p, pb[n], n, "param")
    if mode == "torch_adam":
        sa, sb = opts[0].state, opts[1].state
        for (n, p) in a.named_parameters():
            for key in ("exp_avg", "exp_avg_sq"):
                close(sa[p][key], sb[pb[n]][key], n, key)
            assert float(sa[p]["step"]) == float(sb[pb[n]]["step"])
    else:
        for buf in ("m", "v"):
            for (n, _), x, y in zip(a.named_parameters(), opts[0].fp.views_of(getattr(opts[0], buf)),
                                    opts[1].fp.views_of(getattr(opts[1], buf))):
                close(x, y, n, buf)
        assert opts[0].t == opts[1].t == 10
    for bn_a, bn_b in zip(a.bns, b.bns):
        for k in ("running_mean", "running_var"):
            assert_close(getattr(bn_a, k), getattr(bn_b, k), what=k)
        assert int(bn_a.num_batches_tracked) == int(bn_b.num_batches_tracked) == 10
    # the counter went on across the growth: the same {seed, step} as B's after 10 training forwards with dropout
    assert torch.equal(a.dropout_state(), b.dropout_state())
    assert int(a.dropout_state()[1]) == (10 if drop > 0 else 0)
    a.eval(), b.eval()
    with torch.no_grad():
        for d in new:
            ga, gb = a(*forward_args(d))[0], b(*forward_args(d))[0]
            report["predict"] = report.get("predict", True) and torch.equal(ga, gb)
            assert_close(ga, gb, what="predictions")
    print(f"{mode} (optimizer named: {named}, dropout {drop}): {sum(report.values())} of {len(report)} tensors bitwise equal; within the bar only: "
          f"{sorted(k for k, v in report.items() if not v)}; not compared (gradient 0 in exact arithmetic): {noise}; "
          f"largest loss difference {elem_err(la, lb):.2e}")


# ---- 3. a live store, end to end --------------------------------------------------------------------------------------
def _live_store():
    """Store of chunk 1 of the fixture table; chunk 2 brings entry 6 (new) and more traces of entry 4, and the new
    entry's calls use interface ids above every id of chunk 1."""
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.tracegroup import group_traces

    d = make_trace_table(GOLD_SEED)
    cols, res, n_ms = d["columns"], (d["resource_index"], d["resource_values"]), d["n_ms"]
    r = O.group_traces(cols)
    tid, ent = r["trace_id"], r["entry"]
    late = tid[(ent == 6) | ((ent == 4) & (tid % 2 == 0))]
    in_late = np.isin(cols["traceid"], late)
    c1 = {k: v[~in_late] for k, v in cols.items()}
    c2 = {k: v[in_late].copy() for k, v in cols.items()}
    c2["interface"][c2["entryid"] == 6] += int(cols["interface"].max()) + 1
    s = PatternStore.from_trace_groups(group_traces(c1, "cuda").check(), "span", *res, "cuda", n_ms=n_ms)
    return s, c2


def test_live_store_end_to_end():
    from pert_gnn_kdd23_b200.index import build_index
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, FlatParams, FusedAdam, evaluate_bucketed,
                                           grow_embeddings, model_inputs, predict)
    from oracle.model_oracle import OracleSAGEDeterministic

    s, c2 = _live_store()
    b0 = s.id_bounds()
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [b0["cat"]], b0["entry"] - 1, b0["interface"] - 1, b0["rpctype"] - 1, 32, 2,
                              0.0).cuda()
    opt = FusedAdam(FlatParams(model), lr=1e-3)
    step = BucketedTrainStep(model, opt)
    for _ in range(2):
        for batch in StoreLoader(s, range(len(s)), 16):
            step(batch)
    q_old = np.array([0, 1, 2, 2, 1, 0] * 6)
    ts_old = np.arange(q_old.shape[0]) * 7919 + 1000
    for _ in range(2):                                   # eager, then captured
        p_old = predict(model, s, q_old, ts_old, batch_size=16, asof=True)
        evaluate_bucketed(model, StoreLoader(s, range(len(s)), 16), "cuda")
    new = s.append_traces(c2)
    b1 = s.id_bounds()
    assert b1["entry"] > b0["entry"] and b1["interface"] > b0["interface"]
    rows = grow_embeddings(model, opt, s, seed=2)
    assert rows == {k: max(b0[k], b1[k]) for k in rows}
    # the growth alone leaves the predictions of untouched entries as they were
    assert_close(predict(model, s, q_old, ts_old, batch_size=16, asof=True), p_old, what="untouched entries")
    evaluate_bucketed(model, StoreLoader(s, range(len(s)), 16), "cuda")
    assert model.__dict__["_bucketed_predict"].invalidations >= 1
    assert model.__dict__["_bucketed_eval"].invalidations >= 1
    for _ in range(2):
        for batch in StoreLoader(s, list(new), 16):
            assert torch.isfinite(step(batch)).all()
    assert step.capture_error is None
    q_new = np.array([6, 4, 6, 4, 6] * 4)
    ts_new = np.arange(q_new.shape[0]) * 6151 + 2000
    got = predict(model, s, q_new, ts_new, batch_size=16, asof=True)
    b = s.assemble_requests(q_new, ts_new, asof=True)
    gi = build_index(b.edge_index, b.x.size(0), b.edge_attr, rows["interface"], rows["rpctype"], check=False)
    assert int(gi.status.item()) == 0                    # every id inside the grown tables
    assert int(b.cat_X.max()) < rows["cat"] and int(b.entry_id.max()) < rows["entry"]
    s.check()
    oracle = OracleSAGEDeterministic(9, [rows["cat"]], rows["entry"] - 1, rows["interface"] - 1, rows["rpctype"] - 1,
                                     32, 2, 0.0)
    oracle.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()})
    oracle.eval()
    oracle64 = copy.deepcopy(oracle).double()
    a32 = forward_args(b.to("cpu"))
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    with torch.no_grad():
        go, go64 = oracle(*a32)[0], oracle64(*a64)[0]
    assert_close_ref(got, go.reshape(-1), go64.reshape(-1), what="predict of the new entries vs oracles")
    model.eval()
    with torch.no_grad():
        assert_close(got, model(*model_inputs(b))[0].reshape(-1), what="predict vs forward")


# ---- 4. round trip and no-op ------------------------------------------------------------------------------------------
def test_round_trip_and_no_op():
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, grow_embeddings, model_inputs, predict

    s, c2 = _live_store()
    b0 = s.id_bounds()
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [b0["cat"]], b0["entry"] - 1, b0["interface"] - 1, b0["rpctype"] - 1, 32, 2,
                              0.0).cuda()
    opt = FusedAdam(FlatParams(model), lr=1e-3)
    s.append_traces(c2)
    rows = grow_embeddings(model, opt, s, seed=4)
    q = np.array([6, 4, 0, 1, 2] * 5)
    ts = np.arange(q.shape[0]) * 7001 + 500
    for _ in range(2):
        got = predict(model, s, q, ts, batch_size=8, asof=True)
    eng, st = model._engine, model.__dict__["_bucketed_predict"]
    caps, inv = st.captures, st.invalidations
    assert grow_embeddings(model, opt, s, seed=4) == rows
    again = predict(model, s, q, ts, batch_size=8, asof=True)
    assert model._engine is eng and st.captures == caps and st.invalidations == inv
    # a replay repeats the eval forward to within fp32 accumulation order (atomic sums), as in test_gpu_predict
    assert_close(again, got, what="predict after a no-op growth")
    fresh = SAGEDeterministic(9, [rows["cat"]], rows["entry"] - 1, rows["interface"] - 1, rows["rpctype"] - 1, 32, 2,
                              0.0).cuda()
    fresh.load_state_dict(model.state_dict())
    assert_close(predict(fresh, s, q, ts, batch_size=8, asof=True), got, what="grown state_dict in a fresh model")
    # the operator path reads the grown module weights directly
    b = s.assemble_requests(q, ts, asof=True)
    model.eval()
    model.use_engine = False
    with torch.no_grad():
        assert_close(model(*model_inputs(b))[0].reshape(-1), got, what="operator path after growth")
