"""Raw chunks of a stream on the GPU (rawtable.RawStream, csrc/rawtable.cu pert_raw_stream_*): a fresh stream's first
chunk against process_raw bit for bit (and so the reference's get_df() golden), seeded multi-chunk runs against the
numpy restatement (tests/raw_stream_ref.py), the time-ordered whole-table equality, the status word, determinism, a
second device, and a serving loop raw rows -> store -> window -> model -> predict."""
import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from pert_gnn_kdd23_b200.rawtable import RawStream, RawTables, process_raw, read_raw
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables
from pert_gnn_kdd23_b200.tracegroup import COLUMNS
from tests.raw_stream_ref import RefStream, chunk_of, time_chunks
from tests.test_raw_tables import FIXTURES, GOLD, assert_equals_golden, write_fixture

pytestmark = pytest.mark.gpu

NAMES = ("ms_names", "traceid_names", "interface_names", "rpcid_values", "rpctype_names", "entry_names")


def _bits(t):
    return t.view(torch.int64) if t.is_floating_point() else t


def _assert_same_result(a, b):
    """Two ProcessedTables bit for bit: columns, rows, resource rows, n_ms and the name lists."""
    for k in COLUMNS:
        assert torch.equal(a.columns[k], b.columns[k]), k
    assert torch.equal(a.row, b.row)
    assert torch.equal(a.resource_index, b.resource_index)
    assert torch.equal(_bits(a.resource_values), _bits(b.resource_values))
    assert a.n_ms == b.n_ms
    for k in NAMES:
        assert getattr(a, k) == getattr(b, k), k


def _assert_equals_ref(p, r):
    for k in COLUMNS:
        assert np.array_equal(p.columns[k].cpu().numpy(), r["columns"][k]), k
    assert np.array_equal(p.row.cpu().numpy(), r["row"])
    assert np.array_equal(p.resource_index.cpu().numpy(), r["resource_index"])
    v = p.resource_values.cpu().numpy()
    assert np.array_equal(np.isnan(v), np.isnan(r["resource_values"]))
    assert np.array_equal(v[~np.isnan(v)], r["resource_values"][~np.isnan(v)])
    assert np.array_equal(p.resource_ms.cpu().numpy(), r["resource_ms"])
    assert p.n_ms == r["n_ms"]
    for k in NAMES:
        assert getattr(p, k) == r["names"][k], k


# ---- a fresh stream's first chunk is process_raw ------------------------------------------------------------------
@pytest.mark.parametrize("fx", FIXTURES)
def test_first_chunk_equals_process_raw_on_fixtures(fx, tmp_path):
    gold = np.load(GOLD)
    calls, res = write_fixture(str(tmp_path), gold, fx)
    raw = read_raw(calls, res)
    p = RawStream("cuda").process(raw).check()
    _assert_same_result(p, process_raw(raw, "cuda").check())
    assert_equals_golden(gold, fx, {k: v.cpu().numpy() for k, v in p.columns.items()}, p.row.cpu().numpy(),
                         p.resource_index.cpu().numpy(), p.resource_values.cpu().numpy())


def test_first_chunk_equals_process_raw_at_scale():
    raw = make_random_raw_tables(3, 200_000)
    assert len(raw) > 5_000_000
    s = RawStream("cuda", min_occurence=100)
    p = s.process(raw).check()
    _assert_same_result(p, process_raw(raw, "cuda", min_occurence=100).check())
    assert s.n_ms == p.n_ms and s.ms_names == p.ms_names and s.entry_names == p.entry_names


def test_first_chunk_equals_process_raw_with_hash_collisions():
    raw = make_random_raw_tables(5, 1500, dup=0.2)
    p = RawStream("cuda", min_occurence=3, hash_bits=3).process(raw).check()
    _assert_same_result(p, process_raw(raw, "cuda", min_occurence=3).check())


# ---- several chunks against the restatement -----------------------------------------------------------------------
def _chunks(seed):
    """Whole-trace chunks exercising every rule: the 1-trace and empty chunks, values that come back, names new in a
    later chunk that sort before old ones, entries admitted later, coverage growing as resources arrive, traces without
    an entry, duplicate rows (make_random_raw_tables repeats 5 % of the rows)."""
    raw = make_random_raw_tables(seed, 900, n_entries=12, n_ms=200, n_if=40)
    tr, ms = raw.calls["traceid"], raw.resources["msname"]
    ends = (tr == tr.min()) | (tr == tr.max())
    first = chunk_of(raw, np.flatnonzero(tr == tr.min()), np.flatnonzero(ms % 7 == 0))
    middle = chunk_of(raw, np.flatnonzero(~ends), np.flatnonzero(ms % 7 != 0))
    empty = chunk_of(raw, np.zeros(0, np.int64), np.zeros(0, np.int64))
    last = chunk_of(raw, np.flatnonzero(tr == tr.max()), np.zeros(0, np.int64))
    return [first] + time_chunks(middle, 5, res_first="by_ms", seed=seed) + [empty, last]


@pytest.mark.parametrize("seed,min_occ", [(11, 10), (12, 0), (13, 30)])
def test_chunks_equal_restatement(seed, min_occ):
    chunks = _chunks(seed)
    s, ref = RawStream("cuda", min_occurence=min_occ), RefStream(min_occ)
    for c in chunks:
        _assert_equals_ref(s.process(c).check(), ref.process(c))
    assert s.n_ms == len(ref.names["ms_names"])


def test_time_ordered_chunks_equal_whole_table():
    """Chunks in time order, resources in chunk 1, min_occurence = 0: the concatenated outputs are process_raw of the
    whole table, every id compared through its value, rows in (chunk, timestamp) order."""
    raw = make_random_raw_tables(21, 3000)
    whole = process_raw(raw, "cuda", min_occurence=0).check()
    s = RawStream("cuda", min_occurence=0)
    parts = [s.process(c).check() for c in time_chunks(raw, 4, res_first=True, seed=5)]
    names = {"traceid": s.traceid_names, "interface": s.interface_names, "rpcid": s.rpcid_values,
             "rpctype": s.rpctype_names, "um": s.ms_names, "dm": s.ms_names}
    wnames = {"traceid": whole.traceid_names, "interface": whole.interface_names, "rpcid": whole.rpcid_values,
              "rpctype": whole.rpctype_names, "um": whole.ms_names, "dm": whole.ms_names}

    def rows(cols, v):
        c = {k: x.cpu().numpy() for k, x in cols.items()}
        return sorted(zip(*(([v[k][i] for i in c[k]] if k in v else c[k].tolist()) for k in COLUMNS
                            if k != "entryid")))

    cat = {k: torch.cat([p.columns[k] for p in parts]) for k in COLUMNS}
    assert rows(cat, names) == rows(whole.columns, wnames)
    for p in parts:
        assert bool((p.columns["timestamp"].diff() >= 0).all())


def test_out_of_range_codes_set_the_status_word():
    raw = make_random_raw_tables(7, 300)
    s = RawStream("cuda", min_occurence=2)
    s.process(chunk_of(raw, np.flatnonzero(raw.calls["traceid"] < 100), np.arange(10))).check()
    c = chunk_of(raw, np.flatnonzero(raw.calls["traceid"] >= 100), np.arange(10, len(raw.resources["msname"])))
    c.calls["interface"][3] = len(c.dicts["interface"])
    c.resources["msname"][0] = -1
    p = s.process(c)
    with pytest.raises(_lib.PertGnnError, match="out of range"):
        p.check()
    assert int(p.resource_ms[0]) == -1 and bool((p.resource_ms[1:] >= 0).all())


def test_two_streams_are_bit_identical():
    chunks = _chunks(14)
    a, b = RawStream("cuda", min_occurence=5), RawStream("cuda", min_occurence=5)
    for c in chunks:
        pa, pb = a.process(c).check(), b.process(c).check()
        _assert_same_result(pa, pb)
        assert torch.equal(pa.resource_ms, pb.resource_ms)


def test_second_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("one visible GPU")
    chunks = _chunks(15)
    s, ref = RawStream("cuda:1", min_occurence=5), RefStream(5)
    for c in chunks:
        p = s.process(c).check()
        assert p.columns["traceid"].device == torch.device("cuda:1")
        _assert_equals_ref(p, ref.process(c))


# ---- the serving loop -----------------------------------------------------------------------------------------------
def _fixture_chunks(tmp_path, n_chunks):
    """The golden CSV fixture cut into chunks of whole traces in time order; chunk 0 holds the fixture's resource rows,
    chunk j > 0 the same rows j hours later (new buckets for the sample window)."""
    gold = np.load(GOLD)
    raw = read_raw(*write_fixture(str(tmp_path), gold, "numeric"))
    K = len(raw.resources["timestamp"])
    res = {k: np.concatenate([v] * n_chunks) for k, v in raw.resources.items()}
    res["timestamp"] = res["timestamp"] + np.repeat(np.arange(n_chunks), K) * 3_600_000
    big = RawTables(raw.calls, res, raw.dicts)
    chunks = time_chunks(big, n_chunks, res_first=True, seed=3)
    part = np.repeat(np.arange(n_chunks), K)
    return [chunk_of(big, np.flatnonzero(np.isin(big.calls["traceid"], np.unique(
        [big.dicts["traceid"].index(c.dicts["traceid"][i]) for i in c.calls["traceid"]]))), np.flatnonzero(part == j))
        for j, c in enumerate(chunks)]


def test_serving_loop_end_to_end(tmp_path):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.tracegroup import group_traces
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep, grow_embeddings, predict
    from tests.test_gpu_trace_append import _assert_same, _rebuilt

    chunks = _fixture_chunks(tmp_path, 4)
    N_MS = 512
    stream = RawStream("cuda", min_occurence=5, max_ms=N_MS)
    hist = stream.process(chunks[0]).check()
    idx, vals = hist.resource_index, torch.nan_to_num(hist.resource_values)
    groups = group_traces({k: v for k, v in hist.columns.items()}, "cuda").check()
    store = PatternStore.from_trace_groups(groups, "span", idx, vals, n_ms=N_MS)
    only_traces = PatternStore.from_trace_groups(groups, "span", idx, vals, n_ms=N_MS)
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [N_MS], 8, 32, 8, 32, 2, 0.0).cuda()
    opt = FusedAdam(FlatParams(model), lr=1e-3)
    grow_embeddings(model, opt, store, seed=0)
    step = GraphedTrainStep(model, opt, 0.5)
    for i, batch in enumerate(StoreLoader(store, list(range(len(store))), 64)):
        assert torch.isfinite(step(batch)).all()
        if i == 2:
            break
    win = ResourceSampleWindow(store.n_ms)
    outs = [hist]
    for c in chunks[1:]:
        chunk = stream.process(c).check()
        outs.append(chunk)
        if len(chunk):
            new = store.append_traces(chunk.columns)
            only_traces.append_traces(chunk.columns)
            assert len(new) == int(torch.unique(chunk.columns["traceid"]).numel())
        ok = chunk.resource_ms >= 0
        r = c.resources
        ts = torch.from_numpy(r["timestamp"]).cuda()[ok]
        rows = win.add(ts, chunk.resource_ms[ok], torch.from_numpy(r["instance_cpu_usage"]).cuda()[ok],
                       torch.from_numpy(r["instance_memory_usage"]).cuda()[ok])
        if rows.index.shape[0]:
            store.append_resources(rows.index, torch.nan_to_num(rows.values), replace=True)
        grow_embeddings(model, opt, store, seed=1)
        ent = store._h_trace_entry.astype(np.int64)
        pred = predict(model, store, ent[-64:], store.t["trace_ts"].cpu().numpy()[-64:], batch_size=64, asof=True)
        assert torch.isfinite(pred).all()
        store.check()
    assert stream.n_ms <= N_MS
    # the trace side of the store: the constructor fed the chunk-ordered grouping of the concatenated outputs
    cat = {k: np.concatenate([o.columns[k].cpu().numpy() for o in outs]) for k in COLUMNS}
    chunk_of_row = np.concatenate([np.full(len(o), j) for j, o in enumerate(outs)])
    _assert_same(only_traces, _rebuilt(cat, chunk_of_row, "span", (idx.cpu().numpy(), vals.cpu().numpy()), N_MS))
