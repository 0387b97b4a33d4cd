"""CPU tests of the capacity buckets behind train.BucketedTrainStep: the ladder and the capacity invariants the ghost
layout of pert_batch_pad relies on, host-side argument checks of the padded-batch C entry points (no CUDA call is
made for a rejected call), and StoreLoader.max_sizes as a bound over shuffled batches."""
import numpy as np
import pytest

from pert_gnn_kdd23_b200.train import bucket_bound, bucket_caps, ladder

SIZES = sorted({0, 1, 2, 3, 15, 16, 17, 18, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 170, 171, 255, 256, 257, 1000,
                1023, 1024, 1025, 4095, 4096, 4097, 12288, 12289, 50000, 131071, 131072, 131073, 999999})


def test_ladder_values_and_waste():
    assert [ladder(x) for x in range(17)] == list(range(17))
    assert ladder(17) == 18 and ladder(170) == 176 and ladder(171) == 176 and ladder(256) == 256
    prev = 0
    for x in range(0, 70000):
        v = ladder(x)
        assert v >= x and v >= prev                       # covers x, monotone
        if x > 16:
            assert v - x < x / 8                          # 4 significant bits: less than 1/8 wasted
            k = v.bit_length() - 4
            assert v % (1 << k) == 0 and 8 <= v >> k <= 15
        assert ladder(v) == v                             # ladder values are fixed points
        prev = v


@pytest.mark.parametrize("B", [1, 2, 15, 16, 17, 31, 170, 171, 256, 4096])
def test_capacity_invariants(B):
    for N in SIZES:
        if N < B:
            continue
        for E in SIZES:
            Nc, Ec, Bc = bucket_caps(N, E, B)
            assert Nc >= N and Ec >= E and Bc > B
            ghost_nodes, ghost_graphs, ghost_edges = Nc - N, Bc - B, Ec - E
            assert ghost_nodes >= max(1, ghost_graphs)    # every ghost graph owns a ghost node
            assert ghost_edges <= 4 * ghost_nodes         # ghost in-degree <= 4
            if E == 0:
                assert Ec == 0
            for v, x in ((Ec, E), (Bc, B + 1)):
                assert v == ladder(x)
            # padding stays small: the ghost nodes the ghost graphs / edges need, plus the ladder's 1/8 of the total
            need = max(Bc - B, -(-ghost_edges // 4))
            assert Nc - N <= need + (N + need) / 8
            # the reserve bound covers every smaller batch
            bN, bE, bB = bucket_bound(N, E, B)
            assert Nc <= bN and Ec <= bE and Bc <= bB


def test_bucket_bound_covers_every_smaller_batch():
    rng = np.random.default_rng(0)
    for _ in range(200):
        N, E, B = int(rng.integers(1, 200000)), int(rng.integers(0, 400000)), int(rng.integers(1, 300))
        bN, bE, bB = bucket_bound(N, E, B)
        for _ in range(50):
            b = int(rng.integers(1, B + 1))
            n = int(rng.integers(b, max(b, N) + 1))
            e = int(rng.integers(0, E + 1))
            Nc, Ec, Bc = bucket_caps(n, e, b)
            assert Nc <= bN and Ec <= bE and Bc <= bB, (n, e, b, N, E, B)


def test_on_ladder_sizes_still_get_a_ghost():
    # B + 1 on the ladder, E on the ladder (no ghost edges), N on the ladder
    Nc, Ec, Bc = bucket_caps(128, 256, 15)
    assert (Ec, Bc) == (256, 16) and Nc >= 129
    Nc, Ec, Bc = bucket_caps(16, 0, 1)
    assert (Nc, Ec, Bc) == (18, 0, 2)         # 17 is not on the ladder


def _pad_args(**over):
    """Arguments of pert_batch_pad for a valid small case with non-NULL dummy pointers (never dereferenced on the host:
    every case below is rejected before any CUDA call)."""
    a = dict(x=1, cat_X=1, edge_index=1, edge_attr=1, batch=1, entry_id=1, y=1, rt_probs=1, pnn=1, N=10, E=20, B=2,
             F=9, n_cat=1, attr_cols=2, x_cap=1, cat_X_cap=1, edge_index_cap=1, edge_attr_cap=1, batch_cap=1,
             entry_id_cap=1, y_cap=1, rt_probs_cap=1, pnn_cap=1, N_cap=12, E_cap=24, B_cap=3, live=1, stream=None)
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over", [
    {"x_cap": None}, {"live": None}, {"y": None}, {"entry_id": None}, {"x": None}, {"edge_index": None},
    {"pnn_cap": None}, {"N": -1}, {"E": -1}, {"B": -1}, {"B": 0}, {"F": 0}, {"n_cat": 0}, {"attr_cols": 0},
    {"N_cap": 9}, {"E_cap": 19}, {"B_cap": 1},
    {"B_cap": 2},                       # no ghost graph
    {"B_cap": 5},                       # 3 ghost graphs, 2 ghost nodes
    {"E_cap": 29},                      # 9 ghost edges on 2 ghost nodes: in-degree > 4
    {"N_cap": 1 << 31, "E_cap": 24},    # capacity beyond int32 node ids
])
def test_batch_pad_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_batch_pad(*_pad_args(**over)) == -1


def test_live_entries_reject_bad_arguments():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_pinball_loss_live(None, None, 0.5, 4, 1.0, None, None, None, None) == -1
    assert L.pert_pinball_loss_live(1, 1, 0.5, 0, 1.0, None, None, 1, None) == -1
    assert L.pert_eval_metrics_live(None, None, 0.5, 4, None, None, None) == -1
    assert L.pert_eval_metrics_live(1, 1, 0.5, -1, 1, 1, None) == -1
    # NULL model descriptor
    assert L.pert_model_forward_live(*([None] * 10 + [4, 4, 1] + [None] * 5 + [0, 1, 0.0] + [None] * 8)) == -1
    assert L.pert_model_backward_live(*([None] * 8 + [4, 4, 1] + [None] * 8 + [0, 1, 0.0] + [None] * 5)) == -1


def test_store_loader_max_sizes_bounds_every_shuffled_batch():
    """max_sizes and PatternStore.sizes read only the store's host tables, so a store with synthetic tables (no device
    arrays) exercises them exactly."""
    import torch

    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader

    rng = np.random.default_rng(3)
    store = PatternStore.__new__(PatternStore)
    n_ent, n_traces = 40, 500
    store._h_ent_nodes = rng.integers(3, 400, n_ent).astype(np.int64)
    store._h_ent_edges = rng.integers(0, 900, n_ent).astype(np.int64)
    store._h_ent_pats = rng.integers(1, 4, n_ent).astype(np.int64)
    store._h_trace_entry = rng.integers(0, n_ent, n_traces).astype(np.int64)
    ids = rng.choice(n_traces, 300, replace=False).tolist()
    for bs in (1, 7, 170, 256, 400):
        loader = StoreLoader(store, ids, bs, shuffle=True)
        mN, mE, mB = loader.max_sizes()
        assert mB == min(bs, len(ids))
        for seed in range(5):
            perm = torch.randperm(len(ids), generator=torch.Generator().manual_seed(seed)).numpy()
            order = np.asarray(ids)[perm]
            for i in range(0, len(order), bs):
                chunk = order[i:i + bs]
                n, e, _ = store.sizes(chunk)
                assert n <= mN and e <= mE and len(chunk) <= mB
        if bs >= len(ids):                                # the whole set is one batch: the bound is exact
            assert (mN, mE) == store.sizes(ids)[:2]
