"""-m gpu: replacing and deleting resource rows of a live store (PatternStore.append_resources(replace=True),
delete_resources), alone and mixed with plain appends and evictions.

The store's rows are a list L in arrival order; a replace removes every row of the batch's keys and appends the batch's
last row of each key, a delete removes every row of its keys (tests/resource_rows_ref.py).  After every update the
resource state must equal, bit for bit, the constructor's store of L with the same n_ms, and every assembly the same
call on that rebuilt store."""
import numpy as np
import pytest
import torch

from tests.helpers import assert_close
from tests.resource_rows_ref import ResourceRows
from tests.test_gpu_resource_update import (OUT_KEYS, B, _assert_same_assembly, _assert_same_state, _formats,
                                            _requests, _sparse_art, _state, _trained_model)

pytestmark = pytest.mark.gpu


def _index_format(rng, ts, ms):
    """The keys of a delete as constructor-style pairs, an int64 array, a CUDA tensor or an int32 CUDA tensor."""
    f = int(rng.integers(0, 4))
    a = np.stack([ts, ms], 1).astype(np.int64)
    return (list(zip(ts.tolist(), ms.tolist())), a, torch.from_numpy(a).cuda(), torch.from_numpy(a).cuda().int())[f]


# The operations of one seeded sequence.  The first 16 in a seeded order; then the table is emptied and refilled.
KINDS = ["republish", "late_fix", "dup_then_replace", "replace_absent", "replace_repeated", "delete_repeated",
         "delete_absent", "delete_last_of_ms", "delete_bucket", "replace_evict", "delete_evict", "append_next",
         "republish", "late_fix", "replace_empty", "delete_empty",
         "delete_all", "append_into_empty", "append_next", "republish", "late_fix", "replace_evict", "delete_bucket",
         "replace_repeated", "delete_evict"]


def _op(kind, rng, m, res_ms, newest):
    """The calls of one operation on the mirror's current rows: [(call, ts, ms, cut)], call in append / replace /
    delete."""
    have = np.unique(m.keys())
    hts, hms = have // m.n_ms, have % m.n_ms
    lo_t = int(hts.min()) if hts.size else newest
    hi_t = int(hts.max()) if hts.size else newest
    ts, ms, cut, call = np.zeros(0, np.int64), np.zeros(0, np.int64), None, "replace"
    if kind == "republish":                                      # the newest bucket again, with final values
        ms = np.array([x for x in res_ms if rng.random() < 0.9], dtype=np.int64)
        ts = np.full(ms.shape, hi_t, dtype=np.int64)
    elif kind == "late_fix" and have.size:                      # corrections of older buckets' rows
        pick = rng.choice(have.size, min(12, have.size), replace=False)
        ts, ms = hts[pick], hms[pick]
    elif kind == "dup_then_replace" and have.size:              # keys holding several rows from plain appends
        pick = rng.choice(have.size, min(5, have.size), replace=False)
        ts, ms = hts[pick], hms[pick]
        return [("append", np.repeat(ts, 2), np.repeat(ms, 2), None), ("replace", ts, ms, None)]
    elif kind == "replace_absent":                              # between buckets: no such key
        ms = rng.choice(res_ms, 8)
        ts = B * rng.integers(lo_t // B, hi_t // B + 1, 8) + rng.integers(1, B, 8)
    elif kind == "replace_repeated":                            # the last row of each key wins
        ms = rng.choice(res_ms, 6)
        ts = B * rng.integers(lo_t // B, hi_t // B + 2, 6)
        ms, ts = np.concatenate([ms, ms[:4], ms[:2]]), np.concatenate([ts, ts[:4], ts[:2]])
    elif kind == "delete_repeated" and have.size:
        pick = rng.choice(have.size, min(6, have.size), replace=False)
        ts, ms, call = np.concatenate([hts[pick], hts[pick][:3]]), np.concatenate([hms[pick], hms[pick][:3]]), "delete"
    elif kind == "delete_absent":
        ms = rng.choice(res_ms, 6)
        ts = B * rng.integers(lo_t // B, hi_t // B + 1, 6) + 7
        if have.size:                                            # one present key among them
            ts, ms = np.append(ts, hts[0]), np.append(ms, hms[0])
        call = "delete"
    elif kind == "delete_last_of_ms" and have.size:              # every row of one microservice: it loses ms_has_res
        x = int(rng.choice(np.unique(hms)))
        ts, ms, call = hts[hms == x], hms[hms == x], "delete"
    elif kind == "delete_bucket" and have.size:
        b = int(rng.choice(np.unique(hts)))
        ts, ms, call = hts[hts == b], hms[hts == b], "delete"
    elif kind == "replace_evict":                                # a replaced key below the cut is evicted too
        ms = np.array(res_ms, dtype=np.int64)
        ts = np.concatenate([np.full(len(res_ms) - 2, hi_t), [lo_t, lo_t + B]]).astype(np.int64)
        cut = lo_t + B
    elif kind == "delete_evict" and have.size:
        pick = rng.choice(have.size, min(8, have.size), replace=False)
        ts, ms, call, cut = hts[pick], hms[pick], "delete", lo_t + int(rng.integers(1, B))
    elif kind == "append_next":
        ms = np.array(res_ms, dtype=np.int64)
        ts, call = np.full(ms.shape, hi_t + B, dtype=np.int64), "append"
    elif kind == "delete_empty":
        call = "delete"
    elif kind == "delete_all":
        ts, ms, call = hts, hms, "delete"
    elif kind == "append_into_empty":
        ms = np.array(res_ms[:5], dtype=np.int64)
        ts, call = np.full(5, newest + B, dtype=np.int64), "append"
    return [(call, ts.astype(np.int64), ms.astype(np.int64), cut)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_replace_and_delete_equal_a_rebuilt_store(seed):
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art(21 + seed)
    store = PatternStore.from_artifacts(art, "cuda")
    mirror = ResourceRows(art)
    rng = np.random.default_rng(100 + seed)
    ent, ts_q = _requests(store, rng)
    res_ms = sorted(set(mirror.ms.tolist()))
    newest = int(mirror.ts.max())
    kinds = [KINDS[i] for i in rng.permutation(16)] + KINDS[16:]
    seen = set()
    for i, kind in enumerate(kinds):
        for call, ts, ms, cut in _op(kind, rng, mirror, res_ms, newest):
            vals = rng.random((ts.shape[0], 8))
            if call == "delete":
                got = store.delete_resources(_index_format(rng, ts, ms), evict_before=cut)
                assert got == mirror.delete(ts, ms, cut), (i, kind)
            else:
                idx, v, kept = _formats(rng, ts, ms, vals)
                store.append_resources(idx, v, evict_before=cut, replace=call == "replace")
                (mirror.replace if call == "replace" else mirror.append)(ts, ms, kept, cut)
            seen.add((kind, ts.size > 0))
            if mirror.ts.size:
                newest = max(newest, int(mirror.ts.max()))
            want = mirror.rebuild()
            _assert_same_state(store, want, (i, kind, call))
            _assert_same_assembly(store, want, ent, ts_q, (i, kind, call))
        if kind == "delete_all":
            assert store.desc.n_res == 0 and int(store.t["ms_has_res"].sum()) == 0
        if kind == "delete_last_of_ms":
            gone = np.setdiff1d(res_ms, mirror.ms)
            assert gone.size and not bool(store.t["ms_has_res"][torch.from_numpy(gone).cuda()].any())
    assert {(k, True) for k in set(KINDS) - {"replace_empty", "delete_empty"}} <= seen


# ------------------------------------------------------------------------------------------------- join semantics
def test_joins_after_delete_and_replace():
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    store = PatternStore.from_artifacts(art, "cuda")
    has = store.t["ms_has_res"].cpu().numpy()
    h = {k: store.t[k].cpu().numpy() for k in ("ent_ptr", "ent_pat", "pat_nptr", "pat_ms", "pat_last")}
    for e in np.flatnonzero(store._h_ent_pats > 0):               # an entry and the resourced ms it joins on
        g = np.concatenate([np.arange(h["pat_nptr"][p], h["pat_nptr"][p + 1])
                            for p in h["ent_pat"][h["ent_ptr"][e]:h["ent_ptr"][e + 1]]])
        need = np.unique(h["pat_ms"][g][(h["pat_last"][g] == 1) & (has[h["pat_ms"][g]] == 1)])
        if need.size:
            break
    b, m = 3 * B, int(need[0])
    rng = np.random.default_rng(5)
    # every joined ms gets a row at b (replace inserts the absent ones), m one at b - B
    rows = np.array([(b, x) for x in need] + [(b - B, m)], dtype=np.int64)
    vals = rng.random((rows.shape[0], 8))
    store.append_resources(rows, vals, replace=True)

    def flagged():
        store.status.zero_()
        store.assemble_requests([e], [b + 5])
        code = int(store.status.item())
        store.status.zero_()
        return code == -3

    want_new = torch.from_numpy(vals).float().cuda()
    for asof in (False, True):                                    # the replaced values under both joins
        got, found = store.lookup_resources(rows[:, 0] + 5, rows[:, 1], asof=asof)
        assert bool(found.all()) and torch.equal(got, want_new), asof
    assert not flagged()
    assert store.delete_resources([(b, m)]) == 1
    assert flagged()                                              # the exact join misses (b, m) while m has rows
    assert int(store.t["ms_has_res"][m]) == 1
    got, found = store.lookup_resources([b + 5], [m])
    assert not bool(found.any())
    got, found = store.lookup_resources([b + 5], [m], asof=True)  # the as-of join reads (b - B, m)
    assert bool(found.all()) and torch.equal(got[0], want_new[-1])


# ---------------------------------------------------------------------------------------------- serving loop
def test_serving_loop_replaces_the_provisional_bucket():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts
    from pert_gnn_kdd23_b200.train import predict

    art, _ = make_pert_artifacts(seed=4, n_patterns=64, n_entries=24, n_traces=400, device="cuda")
    store = PatternStore.from_artifacts(art, "cuda")
    model = _trained_model(store)
    mirror = ResourceRows(dict(art, n_ms=store.n_ms))
    now = int(store.t["res_keys"][-1].item()) // store.n_ms + B   # the bucket being filled
    res_ms = np.unique(store.t["res_keys"].cpu().numpy() % store.n_ms)
    rows = np.stack([np.full(res_ms.shape, now), res_ms], 1)
    rng = np.random.default_rng(0)
    provisional = rng.random((rows.shape[0], 8))
    store.append_resources(rows, provisional)                     # published while the bucket is still open
    mirror.append(rows[:, 0], rows[:, 1], provisional)
    Q = 600
    ent = rng.choice(np.flatnonzero(store._h_ent_pats > 0), Q)
    ts = np.where(np.arange(Q) % 2 == 0, now + rng.integers(0, B, Q), rng.integers(-B, now, Q))
    predict(model, store, ent, ts, batch_size=96, asof=True)      # every bucket seen twice: all captured
    before = predict(model, store, ent, ts, batch_size=96, asof=True)
    x_before = store.assemble_requests(ent, ts, asof=True)
    st = model.__dict__["_bucketed_predict"]
    graphs = {k: v.get("graph") for k, v in st.buckets.items()}
    captures = st.captures
    final = rng.random((rows.shape[0], 8))
    store.append_resources(torch.from_numpy(rows).cuda(), torch.from_numpy(final).cuda(), replace=True)
    mirror.replace(rows[:, 0], rows[:, 1], final)
    after = predict(model, store, ent, ts, batch_size=96, asof=True)
    assert st.captures == captures and {k: v.get("graph") for k, v in st.buckets.items()} == graphs
    rebuilt = mirror.rebuild()
    _assert_same_state(store, rebuilt)
    assert_close(after, predict(model, rebuilt, ent, ts, batch_size=96, asof=True), what="after the replace")
    x_after = store.assemble_requests(ent, ts, asof=True)
    node_changed = (x_after.x != x_before.x).any(1).to(torch.int32)
    changed = torch.zeros(Q, dtype=torch.int32, device="cuda").index_add_(0, x_after.batch, node_changed) > 0
    in_now = torch.from_numpy(ts >= now).cuda()
    assert float(changed[in_now].float().mean()) > 0.9 and not bool(changed[~in_now].any())
    assert_close(after[~changed], before[~changed], what="requests whose rows did not change")
    assert bool((after[changed] != before[changed]).all())


# ------------------------------------------------------------------------------------------------------- scale
def _table(n_ms, n_b, g):
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(7)
    art.update(resource_index=[], resource_values=np.zeros((0, 8)), n_ms=n_ms)
    store = PatternStore.from_artifacts(art, "cuda")
    order = torch.randperm(n_ms * n_b, device="cuda", generator=g)
    store.append_resources(torch.stack([(order // n_ms) * B, order % n_ms], 1),
                           torch.rand(n_ms * n_b, 8, device="cuda", generator=g))
    return store


def _assert_rebuilt(store, keys, vals, n_ms):
    """The device rebuild of L = (keys, vals) in arrival order against the store."""
    from pert_gnn_kdd23_b200.store import asof_index

    sk, perm = torch.sort(keys, stable=True)
    assert store.desc.n_res == sk.numel()
    assert torch.equal(store.t["res_keys"], sk)
    assert torch.equal(store.t["res_vals"], vals[perm])
    assert torch.equal(store.t["ms_has_res"], (torch.bincount(sk % n_ms, minlength=n_ms) > 0).to(torch.uint8))
    for (name, got), want in zip(store.asof_t.items(), asof_index(sk, n_ms)):
        assert torch.equal(got, want), name


def test_scale_ten_million_rows():
    n_ms, n_b, k = 30000, 334, 30000                              # 1.002e7 rows
    g = torch.Generator(device="cuda").manual_seed(0)
    store = _table(n_ms, n_b, g)
    keys0, vals0 = store.t["res_keys"].clone(), store.t["res_vals"].clone()
    # replace: the newest bucket, 10 % of the rows in older buckets (some twice), while evicting the oldest bucket
    late = torch.rand(k, device="cuda", generator=g) < 0.1
    ts1 = torch.where(late, torch.randint(0, n_b, (k,), device="cuda", generator=g) * B,
                      torch.full((k,), (n_b - 1) * B, device="cuda"))
    ms1 = torch.randint(0, n_ms, (k,), device="cuda", generator=g)
    v1 = torch.rand(k, 8, device="cuda", generator=g)
    store.append_resources(torch.stack([ts1, ms1], 1), v1, evict_before=B, replace=True)
    k1 = ts1 * n_ms + ms1
    sk1, p1 = torch.sort(k1, stable=True)
    last = torch.ones(k, dtype=torch.bool, device="cuda")
    last[:-1] = sk1[1:] != sk1[:-1]                               # keep-last dedupe of the batch
    pick = torch.sort(p1[last])[0]                                # in input order
    keys = torch.cat([keys0[~torch.isin(keys0, k1)], k1[pick]])
    vals = torch.cat([vals0[~torch.isin(keys0, k1)], v1[pick]])
    keep = keys >= B * n_ms
    keys, vals = keys[keep], vals[keep]
    _assert_rebuilt(store, keys, vals, n_ms)
    # delete: 3e4 keys, some absent, some repeated
    dts = torch.randint(0, n_b + 1, (k,), device="cuda", generator=g) * B
    dms = torch.randint(0, n_ms, (k,), device="cuda", generator=g)
    dk = dts * n_ms + dms
    gone = torch.isin(keys, dk)
    assert store.delete_resources(torch.stack([dts, dms], 1)) == int(gone.sum())
    _assert_rebuilt(store, keys[~gone], vals[~gone], n_ms)


# --------------------------------------------------------------------------------------- rejected calls
def test_rejected_calls_leave_the_store_unchanged():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import PatternStore

    store = PatternStore.from_artifacts(_sparse_art(), "cuda")
    before = {k: v.clone() for k, v in _state(store).items()}
    ptrs = bytes(store.desc), bytes(store.asof_desc)
    top = (2 ** 63 - 1) // store.n_ms
    dev = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")     # noqa: E731
    bad = [
        ([(0, 1), (B, store.n_ms)], "resource row 1: microservice"),
        (dev([[0, 1], [B, -1], [0, 99]]), "resource row 1: microservice -1"),
        (dev([[0, 1], [B, 2], [top, store.n_ms - 1]]), "resource row 2: timestamp"),
        (torch.zeros(2, 2, device="cuda"), "integer \\(timestamp, ms\\) pairs"),
        (np.zeros((2, 3), dtype=np.int64), "resource_index: \\[k, 2\\]"),
    ]
    for idx, msg in bad:
        k = int(idx.shape[0]) if hasattr(idx, "shape") else len(idx)
        for call in (lambda: store.delete_resources(idx), lambda: store.delete_resources(idx, evict_before=B),
                     lambda: store.append_resources(idx, torch.zeros(k, 8, device="cuda"), replace=True),
                     lambda: store.append_resources(idx, np.zeros((k, 8)), replace=True, evict_before=B)):
            with pytest.raises(PertGnnError, match=msg):
                call()
            now = _state(store)
            for name in before:
                assert torch.equal(now[name].cpu(), before[name].cpu()), (msg, name)
            assert (bytes(store.desc), bytes(store.asof_desc)) == ptrs
    with pytest.raises(PertGnnError, match="resource_values: shape"):
        store.append_resources(dev([[0, 1]]), torch.zeros(2, 8, device="cuda"), replace=True)
    with pytest.raises(PertGnnError, match="evict_before"):
        store.delete_resources([(0, 1)], evict_before=1 << 63)
    assert (bytes(store.desc), bytes(store.asof_desc)) == ptrs


def test_replace_values_from_an_unaligned_view():
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    store = PatternStore.from_artifacts(art, "cuda")
    mirror = ResourceRows(art)
    res_ms = sorted(set(mirror.ms.tolist()))
    rows = np.array([[6 * B, m] for m in res_ms] + [[B, m] for m in res_ms[:5]], dtype=np.int64)
    k = rows.shape[0]
    flat = torch.rand(8 * k + 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    vals = flat[1:1 + 8 * k].view(k, 8)
    assert vals.is_contiguous() and vals.data_ptr() % 16 == 4
    store.append_resources(torch.from_numpy(rows).cuda(), vals, evict_before=-B, replace=True)
    mirror.replace(rows[:, 0], rows[:, 1], vals.cpu().double().numpy(), -B)
    _assert_same_state(store, mirror.rebuild())


def test_replace_and_delete_on_a_second_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    store = PatternStore.from_artifacts(art, "cuda:1")
    mirror = ResourceRows(art)
    rows = np.array([[3 * B, m] for m in range(0, store.n_ms, 3)], dtype=np.int64)
    vals = np.random.default_rng(0).random((rows.shape[0], 8))
    with torch.cuda.device(0):
        store.append_resources(torch.from_numpy(rows).to("cuda:1"), vals, evict_before=-B, replace=True)
        n = store.delete_resources(rows[::2])
    mirror.replace(rows[:, 0], rows[:, 1], vals, -B)
    assert n == mirror.delete(rows[::2, 0], rows[::2, 1])
    want = mirror.rebuild()
    for k, v in _state(store).items():
        assert v.device.index in (None, 1) or k == "n_res"
        assert torch.equal(v.cpu(), _state(want)[k].cpu()), k
