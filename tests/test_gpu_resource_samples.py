"""-m gpu: raw resource samples aggregated into open-bucket statistics on the GPU (rawtable.ResourceSampleWindow).

After every ``add`` the rows it returns (the keys it touched) and ``rows()`` (every open key) must equal, NaN-aware and
bit for bit, ``process_raw`` over a RawTables holding every accepted sample so far (and no call rows), restricted to
those keys; the host mirror (tests/resource_samples_ref.py, statistics from the numpy oracle) must agree too.  The
store loop feeds the rows to ``append_resources(replace=True)`` and must end bit for bit at the store built from
``process_raw`` over all samples."""
import numpy as np
import pytest
import torch

from tests.helpers import assert_close
from tests.resource_samples_ref import SampleWindowRef

pytestmark = pytest.mark.gpu

B = 30000
I64_MAX = (1 << 63) - 1


def _raw(n_ms, ts, ms, cpu, mem):
    """RawTables of the samples and one call row: a one-span trace whose um and dm are the first sample's microservice
    (process_raw leaves no output empty then; the row adds no microservice, so the ids are those of the samples)."""
    from pert_gnn_kdd23_b200.rawtable import CALL_COLUMNS, RawTables

    ms = np.asarray(ms, np.int64)
    call = {k: np.zeros(1, np.int64) for k in CALL_COLUMNS}
    call["um"][0] = call["dm"][0] = ms[0]
    call["rt"][0] = 1
    res = {"timestamp": np.asarray(ts, np.int64), "msname": ms,
           "instance_cpu_usage": np.asarray(cpu, np.float64), "instance_memory_usage": np.asarray(mem, np.float64)}
    dicts = {"traceid": ["t"], "interface": ["i"], "rpcid": ["0"], "rpctype": ["http"],
             "ms": [f"ms{i:06d}" for i in range(n_ms)]}
    return RawTables(call, res, dicts)


def _processed(n_ms, ts, ms, cpu, mem):
    """process_raw's resource rows of the samples: (keys ts * n_ms + ms ascending, values [G, 8]), ms mapped back from
    process_raw's ids (the microservices with samples) to the window's through ``ms_names``."""
    from pert_gnn_kdd23_b200.rawtable import process_raw

    p = process_raw(_raw(n_ms, ts, ms, cpu, mem), "cuda", min_occurence=0).check()
    ids = np.array([int(n[2:]) for n in p.ms_names], dtype=np.int64)
    idx = p.resource_index.cpu().numpy()
    key = idx[:, 0] * n_ms + ids[idx[:, 1]]
    assert np.all(np.diff(key) > 0)
    return key, p.resource_values.cpu().numpy()


def _same_bits(got, want, what=""):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(got)
    assert np.array_equal(nan, np.isnan(want)), what
    assert np.array_equal(got[~nan].view(np.int64), want[~nan].view(np.int64)), what


class _Stream:
    """The window, its host mirror and every accepted sample in arrival order."""

    def __init__(self, n_ms):
        from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

        self.n_ms = n_ms
        self.win = ResourceSampleWindow(n_ms, "cuda")
        self.ref = SampleWindowRef(n_ms)
        self.cols = [[] for _ in range(4)]

    def add(self, ts, ms, cpu, mem, fmt=0):
        ins = [np.asarray(c) for c in (ts, ms, cpu, mem)]
        if fmt == 1:
            ins = [c.tolist() for c in ins]
        elif fmt == 2:
            ins = [torch.from_numpy(ins[0]).cuda(), torch.from_numpy(ins[1]).cuda().int(),
                   torch.from_numpy(ins[2]).cuda(), torch.from_numpy(ins[3]).cuda()]
        rows = self.win.add(*ins)
        touched, late = self.ref.add(ts, ms, cpu, mem)
        ok = np.asarray(ts, np.int64) >= self.ref.sealed
        for a, c in zip(self.cols, (ts, ms, cpu, mem)):
            a.append(np.asarray(c)[ok])
        return rows, touched, late

    def check(self, rows, touched, late, what=""):
        n_ms = self.n_ms
        assert rows.late == late, what
        assert rows.index.dtype == torch.int64 and rows.values.dtype == torch.float64 and rows.index.is_cuda
        full = self.win.rows()
        cat = [np.concatenate(c) if c else np.zeros(0) for c in self.cols]
        have = cat[0].size > 0
        key, vals = _processed(n_ms, *cat) if have else (np.zeros(0, np.int64), np.zeros((0, 8)))
        for r, want_keys, name in ((rows, touched, "rows"), (full, self.ref.keys(), "rows()")):
            idx = r.index.cpu().numpy().reshape(-1, 2)
            got_keys = idx[:, 0] * n_ms + idx[:, 1]
            assert got_keys.tolist() == list(want_keys), (what, name)
            assert np.all((idx[:, 1] >= 0) & (idx[:, 1] < n_ms))
            got = r.values.cpu().numpy().reshape(-1, 8)
            pos = np.searchsorted(key, got_keys)
            assert np.array_equal(key[pos], got_keys), (what, name)
            _same_bits(got, vals[pos], (what, name, "process_raw"))
            if len(want_keys):
                _, oracle = self.ref.stats(want_keys)
                _same_bits(got, oracle, (what, name, "oracle"))
        assert self.win.n_keys == len(self.ref.keys()) and self.win.n_samples == sum(
            len(v) for v in self.ref.samples.values()), what


def _values(rng, n, all_nan=False):
    """Usages with equal values, +-0.0, NaN and +-inf among ordinary numbers."""
    v = rng.random(n) * 100
    kind = rng.random(n)
    v[kind < 0.25] = rng.integers(-2, 3, int((kind < 0.25).sum())) * 0.5          # equal values, +0.0
    v[(kind >= 0.25) & (kind < 0.33)] = -0.0
    v[(kind >= 0.33) & (kind < 0.40)] = np.nan
    v[(kind >= 0.40) & (kind < 0.42)] = np.inf
    v[(kind >= 0.42) & (kind < 0.44)] = -np.inf
    if all_nan:
        v[:] = np.nan
    return v


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_stream_equals_process_raw(seed):
    rng = np.random.default_rng(seed)
    n_ms = 40
    s = _Stream(n_ms)
    active, now = 10, 4
    seen = set()
    for step in range(25):
        if step % 5 == 4:
            active = min(n_ms, active + 4)                  # new microservices
        if step % 7 == 6:
            now += 1
        if step % 8 == 7:
            s.win.seal(B * (now - 1))
            s.ref.seal(B * (now - 1))
            if step % 16 == 15:
                s.win.seal(B * (now - 3))                   # a lower seal: no-op
        if step in (2, 17) or rng.random() < 0.08:
            ts = ms = np.zeros(0, np.int64)
            cpu = mem = np.zeros(0)
            seen.add("empty")
        else:
            nk = int(rng.integers(1, 30))
            kts = B * rng.integers(now - 2, now + 1, nk) + np.where(rng.random(nk) < 0.2, 7, 0)
            kms = rng.integers(0, active, nk)
            cnt = rng.integers(1, 9, nk)
            if step == 5 or rng.random() < 0.3:
                cnt[0] = int(rng.integers(100, 400))          # a hot key
                seen.add("hot")
            ts, ms = np.repeat(kts, cnt), np.repeat(kms, cnt)
            order = rng.permutation(ts.size)
            ts, ms = ts[order], ms[order]
            cpu, mem = _values(rng, ts.size), _values(rng, ts.size)
            cpu[(ms % 7 == 3)] = np.nan                       # all-NaN keys
            mem[(ts // B) % 5 == 2] = 1.25                    # all-equal keys
        fmt = int(rng.integers(0, 3))
        rows, touched, late = s.add(ts.astype(np.int64), ms.astype(np.int64), cpu, mem, fmt)
        if late:
            seen.add("late")
        s.check(rows, touched, late, (seed, step))
    assert {"empty", "hot", "late"} <= seen


def test_seal():
    n_ms = 8
    rng = np.random.default_rng(7)
    s = _Stream(n_ms)
    for b in range(4):
        ts = np.repeat(B * b + np.arange(n_ms) % 2, 3)
        ms = np.repeat(np.arange(n_ms), 3)
        rows, touched, late = s.add(ts, ms, _values(rng, ts.size), _values(rng, ts.size))
        s.check(rows, touched, late, b)
    before = s.win.rows()
    s.win.seal(2 * B)
    s.ref.seal(2 * B)
    after = s.win.rows()
    keep = (before.index[:, 0] >= 2 * B).cpu()
    assert torch.equal(after.index.cpu(), before.index.cpu()[keep])
    assert torch.equal(after.values.cpu().view(torch.int64), before.values.cpu()[keep].view(torch.int64))
    snap = {k: v.clone() for k, v in s.win.t.items()}

    def unchanged():
        for k, v in snap.items():
            a, b = s.win.t[k], v
            if a.dtype == torch.float64:
                a, b = a.view(torch.int64), b.view(torch.int64)
            assert torch.equal(a, b), k

    # late samples: counted, nothing changes
    rows, touched, late = s.add(np.array([0, B, 2 * B - 1]), np.array([1, 2, 3]), np.ones(3), np.ones(3))
    assert late == 3 and rows.index.shape == (0, 2) and rows.values.shape == (0, 8)
    s.check(rows, touched, late, "late")
    unchanged()
    s.win.seal(B)                                             # lower: a no-op
    assert s.win.sealed == 2 * B
    unchanged()
    # late and open samples in one call
    rows, touched, late = s.add(np.array([B, 3 * B, 0, 3 * B]), np.array([1, 5, 2, 5]), np.array([1.0, 2, 3, 4]),
                                np.array([-0.0, 0.0, 1, 2]), fmt=2)
    assert late == 2 and touched == [3 * B * n_ms + 5]
    s.check(rows, touched, late, "mixed")
    # seal everything, then add again
    s.win.seal(10 * B)
    s.ref.seal(10 * B)
    assert s.win.n_keys == 0 and s.win.n_samples == 0 and s.win.rows().index.shape == (0, 2)
    rows, touched, late = s.add(np.array([10 * B, 11 * B, 10 * B]), np.array([0, 7, 0]), np.array([3.0, 1, 2]),
                                np.array([np.nan, 1, 2]))
    assert late == 0 and len(touched) == 2
    s.check(rows, touched, late, "after sealing everything")
    s.win.seal(I64_MAX)                                        # cut * n_ms beyond int64: every key sealed
    assert s.win.n_keys == 0
    rows = s.win.add([11 * B], [7], [1.0], [1.0])
    assert rows.late == 1 and s.win.n_keys == 0


def test_rejected_calls_leave_the_window_unchanged():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

    n_ms = 16
    w = ResourceSampleWindow(n_ms, "cuda")
    rng = np.random.default_rng(3)
    w.add(rng.integers(0, 3, 50) * B, rng.integers(0, n_ms, 50), rng.random(50), rng.random(50))
    snap = {k: v.clone() for k, v in w.t.items()}
    n_keys, n_samples = w.n_keys, w.n_samples
    cu = lambda a, d=torch.int64: torch.tensor(a, dtype=d, device="cuda")      # noqa: E731
    bad = [
        (([0, B], [1, n_ms], [1.0, 1], [1.0, 1]), "resource row 1: microservice 16"),
        ((cu([0, B]), cu([-1, 2]), cu([1.0, 1], torch.float64), cu([1.0, 1], torch.float64)),
         "resource row 0: microservice -1"),
        ((cu([0, I64_MAX // 4]), cu([1, 2]), cu([1.0, 1], torch.float64), cu([1.0, 1], torch.float64)),
         "resource row 1: timestamp"),
        ((cu([0.0, 1.0], torch.float64), cu([1, 2]), cu([1.0, 1], torch.float64), cu([1.0, 1], torch.float64)),
         "timestamps: integers expected"),
        (([0, B], [1, 2], [1.0, "x"], [1.0, 1]), "sample 1: instance_cpu_usage 'x'"),
        (([0, B], [1, 2], [1.0, 1], [1.0]), "different lengths"),
        ((cu([0, B]), cu([1, 2]), cu([True, False], torch.bool), cu([1.0, 1], torch.float64)), "numbers expected"),
    ]
    for args, msg in bad:
        with pytest.raises(PertGnnError, match=msg):
            w.add(*args)
    assert w.n_keys == n_keys and w.n_samples == n_samples
    for k, v in snap.items():
        a, b = w.t[k], v
        if a.dtype == torch.float64:
            a, b = a.view(torch.int64), b.view(torch.int64)
        assert torch.equal(a, b), k


def test_scale_a_million_open_samples():
    n_ms, n_b = 30000, 4
    rng = np.random.default_rng(11)
    s = _Stream(n_ms)
    kts = np.repeat(np.arange(n_b) * B, n_ms)
    kms = np.tile(np.arange(n_ms), n_b)
    cnt = rng.integers(1, 18, kts.size)                         # 9 per key on average
    ts, ms = np.repeat(kts, cnt), np.repeat(kms, cnt)
    order = rng.permutation(ts.size)
    ts, ms = ts[order], ms[order]
    cpu, mem = _values(rng, ts.size), _values(rng, ts.size)
    assert ts.size > 10 ** 6
    parts = np.array_split(np.arange(ts.size), 4)
    for p in parts:
        rows = s.win.add(torch.from_numpy(ts[p]).cuda(), torch.from_numpy(ms[p]).cuda(), torch.from_numpy(cpu[p]).cuda(),
                         torch.from_numpy(mem[p]).cuda())
        assert rows.late == 0
    for a, c in zip(s.cols, (ts, ms, cpu, mem)):
        a.append(c)
    # one 3e5-sample add: a new bucket and more samples of the open ones
    k = 300000
    ts2 = np.where(rng.random(k) < 0.5, n_b * B, rng.integers(0, n_b, k) * B)
    ms2 = rng.integers(0, n_ms, k)
    c2, m2 = _values(rng, k), _values(rng, k)
    rows = s.win.add(ts2, ms2, c2, m2)
    for a, c in zip(s.cols, (ts2, ms2, c2, m2)):
        a.append(c)
    key, vals = _processed(n_ms, *[np.concatenate(c) for c in s.cols])
    touched = np.unique(ts2 * n_ms + ms2)
    for r, want in ((rows, touched), (s.win.rows(), key)):
        idx = r.index.cpu().numpy()
        got_keys = idx[:, 0] * n_ms + idx[:, 1]
        assert np.array_equal(got_keys, want)
        _same_bits(r.values.cpu().numpy(), vals[np.searchsorted(key, got_keys)])
    assert s.win.n_samples == ts.size + k


def test_store_loop_equals_the_store_of_all_samples():
    """History -> process_raw -> store; the rest of the samples streamed through the window into
    append_resources(replace=True), one call also evicting; the store, its joins and predict equal those of the store
    built from process_raw over every sample."""
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts
    from pert_gnn_kdd23_b200.train import predict
    from tests.test_gpu_resource_update import _assert_same_assembly, _assert_same_state, _trained_model

    rng = np.random.default_rng(5)
    art = make_trace_artifacts(7)
    n_ms, n_b = art["n_ms"], 12
    # every microservice has samples in every bucket, so process_raw's ids are the window's ids
    kts = np.repeat(np.arange(n_b) * B, n_ms)
    kms = np.tile(np.arange(n_ms), n_b)
    cnt = rng.integers(1, 9, kts.size)
    ts, ms = np.repeat(kts, cnt), np.repeat(kms, cnt)
    order = np.argsort(ts + rng.integers(0, 2 * B, ts.size), kind="stable")   # roughly in time, buckets overlapping
    ts, ms = ts[order], ms[order]
    cpu = rng.integers(0, 40, ts.size) * 0.25                                 # finite: the store feeds a model
    mem = np.where(rng.random(ts.size) < 0.1, -0.0, rng.random(ts.size))
    h = int(np.searchsorted(np.sort(ts), 7 * B))                              # the history: arrivals before ...
    hist = np.arange(ts.size) < h
    open_from = int(ts[:h].max()) - B                                         # ... and its last two buckets open

    def store_of(sel, cut=None):
        from pert_gnn_kdd23_b200.rawtable import process_raw

        p = process_raw(_raw(n_ms, ts[sel], ms[sel], cpu[sel], mem[sel]), "cuda", min_occurence=0).check()
        assert p.n_ms == n_ms and p.ms_names == [f"ms{i:06d}" for i in range(n_ms)]
        idx, vals = p.resource_index.cpu().numpy(), p.resource_values.cpu().numpy()
        keep = idx[:, 0] >= cut if cut is not None else np.ones(idx.shape[0], bool)
        return PatternStore.from_artifacts(dict(art, resource_index=[tuple(r) for r in idx[keep].tolist()],
                                                resource_values=vals[keep]), "cuda")

    store = store_of(hist)
    model = _trained_model(store)
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

    win = ResourceSampleWindow(n_ms, "cuda")
    win.seal(open_from)
    seed = hist & (ts >= open_from)
    win.add(ts[seed], ms[seed], cpu[seed], mem[seed])
    Q = 400
    ent = rng.choice(np.flatnonzero(store._h_ent_pats > 0), Q)
    q_ts = rng.integers(0, n_b * B, Q)
    predict(model, store, ent, q_ts, batch_size=96, asof=True)                # every bucket seen twice: all captured
    predict(model, store, ent, q_ts, batch_size=96, asof=True)
    st = model.__dict__["_bucketed_predict"]
    graphs = {k: v.get("graph") for k, v in st.buckets.items()}
    captures = st.captures
    rest = np.flatnonzero(~hist)
    cut = 2 * B
    for i, part in enumerate(np.array_split(rest, 8)):
        cur = int(ts[part].min()) - B
        if cur > win.sealed:
            win.seal(cur)                                                     # older buckets are final
        rows = win.add(torch.from_numpy(ts[part]).cuda(), torch.from_numpy(ms[part]).cuda(),
                       torch.from_numpy(cpu[part]).cuda(), torch.from_numpy(mem[part]).cuda())
        assert rows.late == 0
        store.append_resources(rows.index, rows.values, replace=True, evict_before=cut if i == 3 else None)
    want = store_of(np.ones(ts.size, bool), cut)
    _assert_same_state(store, want)
    _assert_same_assembly(store, want, ent, q_ts)
    got = predict(model, store, ent, q_ts, batch_size=96, asof=True)
    assert st.captures == captures and {k: v.get("graph") for k, v in st.buckets.items()} == graphs
    assert_close(got, predict(model, want, ent, q_ts, batch_size=96, asof=True), what="predict on the rebuilt store")
