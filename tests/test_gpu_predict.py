"""-m gpu: request assembly (PatternStore.assemble_requests) and batched prediction (train.predict).

Exact request assembly must reproduce trace assembly bit for bit (and with it the reference's own Data objects,
tests/golden/ref_loop.npz); the as-of join must equal the numpy restatement (oracle/asof_oracle.py) bit for bit; predict
must agree with the eval-mode forward of the same batches, with the fp32 / fp64 oracles and with evaluate_bucketed, and
leave the model's state untouched."""
import copy

import numpy as np
import pytest
import torch

from oracle import asof_oracle as A
from tests.helpers import assert_close, elem_err

pytestmark = pytest.mark.gpu

OUT_KEYS = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs", "entry_id",
            "rt_probs", "batch", "ptr")


def _trace_requests(art, store):
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    return store._h_trace_entry.astype(np.int64), ts


def _labels(art, store):
    return np.array([int(art["tr2data"][k]["y"]) for k in store.trace_keys], dtype=np.float64)


# ----------------------------------------------------------------------------------- 1. exact == trace assembly
def test_exact_requests_equal_trace_assembly():
    import os

    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    g = np.load(os.path.join(root, "tests", "golden", "ref_loop.npz"))
    art = make_trace_artifacts(int(g["hyper"][0]))
    store = PatternStore.from_artifacts(art, "cuda")
    ent, ts = _trace_requests(art, store)
    assert (ts % 30000 == 0).all()
    ids = np.arange(len(store))
    want = store.assemble(ids)
    for r in (0, 1, 29999):
        got = store.assemble_requests(ent, ts + r)
        assert "y" not in got and got.num_graphs == len(ids)
        for k in OUT_KEYS:
            assert torch.equal(got[k], want[k]), (r, k)
    # and per trace, so every trace is also its own reference Data object
    for i in ids[::7]:
        got = store.assemble_requests(ent[i:i + 1], ts[i:i + 1] + 29999, asof=True)
        for k in ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs"):
            assert np.array_equal(got[k].cpu().numpy(), g[f"d{i}_{k}"]), (i, k)
    store.check()


# ------------------------------------------------------------------------------------- 2. as-of join vs the oracle
def _sparse_art(seed=11):
    """Trace artefacts whose resource table covers buckets -60000 .. 180000 with ~30 % of the rows dropped (whole
    buckets included) and a few duplicate keys carrying other values."""
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(seed, n_entries=10, n_traces=40)
    rng = np.random.default_rng(seed)
    res_ms = sorted({m for _, m in art["resource_index"]})
    buckets = [30000 * k for k in range(-2, 7)]
    index = [(b, m) for b in buckets if b not in (0, 120000) for m in res_ms]      # two whole buckets missing
    keep = rng.random(len(index)) < 0.85
    index = [ix for ix, k in zip(index, keep) if k]
    dup = rng.choice(len(index), 6, replace=False)
    index = index + [index[i] for i in dup]
    index = [index[i] for i in rng.permutation(len(index))]
    art["resource_index"] = index
    art["resource_values"] = rng.random((len(index), 8))
    return art


def _expected_x(store, art, ent, ts, asof):
    """x of the requests from the store's host-side pattern tables and the numpy join."""
    h = {k: store.t[k].cpu().numpy() for k in ("ent_ptr", "ent_pat", "pat_nptr", "pat_ms", "pat_last", "ms_has_res")}
    g = np.concatenate([np.arange(h["pat_nptr"][p], h["pat_nptr"][p + 1])
                        for e in ent for p in h["ent_pat"][h["ent_ptr"][e]:h["ent_ptr"][e + 1]]])
    owner = np.repeat(np.arange(len(ent)), store._h_ent_nodes[ent])
    ms = h["pat_ms"][g]
    need = (h["pat_last"][g] == 1) & (h["ms_has_res"][ms] == 1)
    res_ts = np.array([t for t, _ in art["resource_index"]], dtype=np.int64)
    res_ms = np.array([m for _, m in art["resource_index"]], dtype=np.int64)
    join = A.asof_rows if asof else A.exact_rows
    rows = np.full(g.shape[0], -1, dtype=np.int64)
    rows[need] = join(res_ts, res_ms, A.time_bucket(ts)[owner[need]], ms[need])
    return A.features(rows, art["resource_values"]), need, rows


def test_asof_join_matches_the_oracle():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    store = PatternStore.from_artifacts(art, "cuda")
    rng = np.random.default_rng(2)
    ent = rng.integers(0, 10, 400)
    ts = rng.integers(-4 * 30000, 9 * 30000, 400)
    ts[:8] = [-10 ** 9, -60001, -30001, -1, 0, 29999, 30000, 10 ** 12]          # the bucket floor, both ends
    want_a, need, rows_a = _expected_x(store, art, ent, ts, True)
    want_e, _, rows_e = _expected_x(store, art, ent, ts, False)
    assert (need & (rows_a < 0)).any() and (need & (rows_e < 0) & (rows_a >= 0)).any() and (rows_e >= 0).any()
    store.status.zero_()
    got_a = store.assemble_requests(ent, ts, asof=True)
    assert np.array_equal(got_a.x.cpu().numpy(), want_a)
    store.check()                                       # as-of never flags a missing row
    got_e = store.assemble_requests(ent, ts)
    assert np.array_equal(got_e.x.cpu().numpy(), want_e)
    hit = rows_e >= 0
    assert np.array_equal(got_a.x.cpu().numpy()[hit], got_e.x.cpu().numpy()[hit])
    assert int(store.status.item()) == -3
    with pytest.raises(_lib.PertGnnError):
        store.check()
    store.status.zero_()
    # the other tensors do not depend on the join
    for k in OUT_KEYS[1:]:
        assert torch.equal(got_a[k], got_e[k]), k


# ------------------------------------------------------------------------------------------------------- 3. errors
def _store_with_an_empty_entry():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(7)
    n0 = len(art["entry2runtimes"])
    art["entry2runtimes"][n0 + 1] = dict(art["entry2runtimes"][1])     # entry n0 has no patterns
    return PatternStore.from_artifacts(art, "cuda"), n0


def test_bad_requests():
    import ctypes as C

    from pert_gnn_kdd23_b200 import _lib, ops
    from pert_gnn_kdd23_b200.store import _PertBatchOut

    store, empty = _store_with_an_empty_entry()
    n_ent = empty + 2
    l0 = ops.LAUNCHES["n"]
    for bad in (-1, n_ent, empty):
        with pytest.raises(_lib.PertGnnError, match=f"request 2: entry {bad} "):
            store.assemble_requests([0, 1, bad, 3], [0, 0, 0, 0])
    assert ops.LAUNCHES["n"] == l0
    torch.cuda.synchronize()
    assert int(store.status.item()) == 0
    # the device check: a direct call, outputs sized for the batch the kernels assemble (a bad entry reads entry 0)
    ent = np.array([1, -1, n_ent, empty], dtype=np.int64)
    ts = np.array([60000, 60000, 90000, 120000], dtype=np.int64)
    like = store.assemble_requests([1, 0, 0, 0], ts, asof=True)
    out = {k: torch.full_like(like[k], 7) for k in OUT_KEYS}
    o = _PertBatchOut()
    for k, v in out.items():
        setattr(o, k, v.data_ptr())
    offsets = torch.empty(3 * 5, dtype=torch.int32, device="cuda")
    ent_d, ts_d = torch.from_numpy(ent).cuda(), torch.from_numpy(ts).cuda()
    rc = _lib.lib().pert_store_assemble_requests(C.byref(store.desc), C.byref(store.asof_desc), ent_d.data_ptr(),
                                                 ts_d.data_ptr(), 4, like.x.size(0), like.edge_index.size(1),
                                                 offsets.data_ptr(), C.byref(o), store.status.data_ptr(),
                                                 _lib.stream())
    assert rc == 0
    assert int(store.status.item()) == -3
    for k in OUT_KEYS:
        assert torch.equal(out[k], like[k]), k
    store.status.zero_()
    # no requests: empty outputs, nothing launched
    b = store.assemble_requests([], [])
    assert b.num_graphs == 0 and b.x.shape == (0, 9) and b.edge_index.shape == (2, 0) and b.ptr.tolist() == [0]
    assert "y" not in b


# ----------------------------------------------------------------------------------------------- 4.-9. predict
@pytest.fixture(scope="module")
def pert_store():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts

    art, _ = make_pert_artifacts(seed=3, n_patterns=64, n_entries=24, n_traces=400, device="cuda")
    return art, PatternStore.from_artifacts(art, "cuda")


def _trained_model(store, hidden=64, p=0.0, steps=4):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    torch.manual_seed(0)
    args = list(model_args(2))
    args[5] = hidden
    m = SAGEDeterministic(*args).cuda()
    m.dropout = p
    m.seed_dropout(77)
    opt = FusedAdam(FlatParams(m), lr=1e-3)
    for i, d in enumerate(StoreLoader(store, list(range(len(store))), 64)):   # running statistics move off their init
        if i >= steps:
            break
        fused_train_step(m, opt, d, 0.5)
    return m, opt


def _requests(store, Q, seed, wide=False):
    """Q requests of entries with patterns: inside the buckets that have resource rows (60000 .. 300000, every 60000),
    or with ``wide`` anywhere from before the first to after the last one."""
    rng = np.random.default_rng(seed)
    ok = np.flatnonzero(store._h_ent_pats > 0)
    if wide:
        return rng.choice(ok, Q), rng.integers(-60000, 8 * 60000, Q)
    return rng.choice(ok, Q), 60000 * rng.integers(1, 6, Q) + rng.integers(0, 30000, Q)


def _eager(model, store, ent, ts, bs, asof):
    """(global [Q], local [sum N], ptr per batch) of the eval-mode forward on the unpadded batches of predict."""
    from pert_gnn_kdd23_b200.train import model_inputs

    was = model.training
    model.eval()
    gs, ls, ptrs = [], [], []
    with torch.no_grad():
        for i in range(0, len(ent), bs):
            d = store.assemble_requests(ent[i:i + bs], ts[i:i + bs], asof=asof)
            g, loc = model(*model_inputs(d))
            gs.append(g.reshape(-1))
            ls.append(loc.reshape(-1))
            ptrs.append(d.ptr)
    model.train(was)
    return torch.cat(gs), torch.cat(ls), ptrs


@pytest.mark.parametrize("asof", [False, True])
def test_predict_matches_the_forward(pert_store, asof):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, _ = _trained_model(store)
    ent, ts = _requests(store, 700, 1, wide=asof)
    got = predict(model, store, ent, ts, batch_size=96, asof=asof)
    want, _, _ = _eager(model, store, ent, ts, 96, asof)
    assert got.dtype == torch.float32 and got.shape == (700,) and got.is_cuda
    e = elem_err(got, want)
    print(f"predict vs eval-mode forward: largest element-wise difference {e:.3e}")
    assert_close(got, want, what="predict vs forward")
    store.check()


def test_predict_matches_the_oracles(pert_store):
    from pert_gnn_kdd23_b200.train import predict
    from tests.helpers import assert_close_ref, forward_args, make_models

    art, store = pert_store
    oracle, model = make_models(2)
    oracle.eval()
    ent, ts = _requests(store, 80, 2, wide=True)
    got = predict(model, store, ent, ts, batch_size=80, asof=True)
    oracle64 = copy.deepcopy(oracle).double()
    b = store.assemble_requests(ent, ts, asof=True).to("cpu")
    a32 = forward_args(b)
    a64 = [t.double() if t.is_floating_point() else t for t in a32]
    with torch.no_grad():
        go, _ = oracle(*a32)
        go64, _ = oracle64(*a64)
    assert_close_ref(got, go.reshape(-1), go64.reshape(-1), what="predict vs oracles")


def test_predict_mae_equals_evaluate_bucketed(pert_store):
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import evaluate_bucketed, predict

    art, store = pert_store
    model, _ = _trained_model(store)
    ent, ts = _trace_requests(art, store)
    y = _labels(art, store)
    for _ in range(2):
        pred = predict(model, store, ent, ts, batch_size=64)
        mae = float(np.abs(pred.double().cpu().numpy() - y).mean())
        want = evaluate_bucketed(model, StoreLoader(store, list(range(len(store))), 64), "cuda")[0]
        assert abs(mae - want) <= 1e-6 * abs(want), (mae, want)


def test_predict_order_duplicates_and_local(pert_store):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, _ = _trained_model(store)
    ent, ts = _requests(store, 300, 3, wide=True)
    base = predict(model, store, ent, ts, batch_size=128, asof=True)
    idx = np.random.default_rng(4).integers(0, 300, 500)          # shuffled, with duplicates
    again = predict(model, store, ent[idx], ts[idx], batch_size=128, asof=True)
    assert_close(again, base[torch.from_numpy(idx).cuda()], what="permuted requests")
    g, loc, node_ptr = predict(model, store, ent, ts, batch_size=128, asof=True, local=True)
    assert_close(g, base, what="global with local=True")
    wg, wl, ptrs = _eager(model, store, ent, ts, 128, True)
    assert loc.shape == wl.shape and node_ptr.shape == (301,) and node_ptr.dtype == torch.int64
    assert_close(loc, wl, what="local predictions")
    for k, p in enumerate(ptrs):
        i = 128 * k
        assert torch.equal(node_ptr[i:i + p.numel()] - node_ptr[i], p)


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_predict_has_no_side_effects(pert_store, p):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, opt = _trained_model(store, p=p)
    ent, ts = _requests(store, 200, 5)
    for training in (True, False):
        model.train(training)
        eng = model.engine()
        before = [opt.fp.flat.clone(), eng.bn_running.clone(), eng.bn_nbt.clone(), model.dropout_state().clone(),
                  opt.m.clone(), opt.v.clone(), opt.fp.grad.clone()]
        for _ in range(3):                                       # eager, captured and replayed buckets
            predict(model, store, ent, ts, batch_size=64)
        torch.cuda.synchronize()
        after = [opt.fp.flat, eng.bn_running, eng.bn_nbt, model.dropout_state(), opt.m, opt.v, opt.fp.grad]
        for k, (b, a) in enumerate(zip(before, after)):
            assert torch.equal(b, a), k
        assert model.training is training and model._engine is eng


def test_predict_replays_and_survives_a_new_engine(pert_store):
    from pert_gnn_kdd23_b200.train import FlatParams, predict

    art, store = pert_store
    model, _ = _trained_model(store)
    ent, ts = _requests(store, 640, 6)
    first = predict(model, store, ent, ts, batch_size=64)
    second = predict(model, store, ent, ts, batch_size=64)
    st = model.__dict__["_bucketed_predict"]
    c0, r0 = st.captures, st.replays
    third = predict(model, store, ent, ts, batch_size=64)
    assert st.capture_error is None, st.capture_error
    assert st.captures == c0 and st.replays - r0 == 10          # every batch replayed, nothing captured again
    assert st.captures >= 1
    for x in (second, third):
        assert_close(x, first, what="repeated predict")
    old = model._engine
    FlatParams(model)                                            # a new flat buffer: the engine is re-created
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(0.5)
    got = predict(model, store, ent, ts, batch_size=64)
    assert model._engine is not old
    want, _, _ = _eager(model, store, ent, ts, 64, False)
    assert_close(got, want, what="after the engine was re-created")
    assert all(e["state"] != "graph" or e["engine"] is model._engine for e in st.buckets.values())


@pytest.mark.parametrize("hidden", [48, 128])
def test_predict_other_widths(pert_store, hidden):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, _ = _trained_model(store, hidden=hidden)
    ent, ts = _requests(store, 300, 7, wide=True)
    for _ in range(2):
        got = predict(model, store, ent, ts, batch_size=100, asof=True)
    want, _, _ = _eager(model, store, ent, ts, 100, True)
    assert_close(got, want, what=f"H={hidden}")


def test_predict_at_scale():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts
    from pert_gnn_kdd23_b200.train import predict

    art, _ = make_pert_artifacts(seed=3, device="cuda")
    store = PatternStore.from_artifacts(art, "cuda")
    model, _ = _trained_model(store)
    ent, ts = _requests(store, 100000, 8, wide=True)
    got = predict(model, store, ent, ts, batch_size=1024, asof=True)
    want, _, _ = _eager(model, store, ent, ts, 1024, True)
    e = elem_err(got, want)
    print(f"predict at 1e5 requests vs eval-mode forward: largest element-wise difference {e:.3e}")
    assert_close(got, want, what="1e5 requests")
    store.check()
