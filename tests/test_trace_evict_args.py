"""PatternStore.evict_traces without a GPU: the window restatement (tests/trace_window_ref.py) against the chunk-ordered
grouping for append-only sequences and against a brute-force recount after evictions, the host argument checks, and
the C-ABI argument checks of the eviction calls in csrc/ingest.cu."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table
from tests import trace_chunk_ref as R
from tests.trace_window_ref import KEY_COLS, REP_COLS, TraceWindow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_preprocess.npz")


def _fixture_cols():
    return make_trace_table(int(np.load(GOLD)["seed"]))["columns"]


def _split(cols, chunk_of_trace):
    """Rows of every chunk, in chunk order, and the per-row chunk column."""
    u, inv = np.unique(cols["traceid"], return_inverse=True)
    row_chunk = chunk_of_trace(u)[inv]
    return [{k: v[row_chunk == c] for k, v in cols.items()} for c in np.unique(row_chunk)], row_chunk


@pytest.mark.parametrize("table", ["fixture", "random"])
def test_append_only_equals_the_chunk_ordered_grouping(table):
    cols = _fixture_cols() if table == "fixture" else make_random_trace_table(3, 3000, rows=(1, 10), n_patterns=300,
                                                                               n_entries=9, n_ms=64, n_if=16)
    rng = np.random.default_rng(4)
    parts, row_chunk = _split(cols, lambda u: rng.integers(0, 4, u.shape[0]))
    w = TraceWindow()
    for c, part in enumerate(parts):
        w.append(part)
        upto = row_chunk <= c
        sub = {k: v[upto] for k, v in cols.items()}
        r = R.group_traces(sub, row_chunk[upto])
        assert list(w.patterns) == [int(x) for x in r["ins_runtime"]] and w.next_rt == len(r["ins_runtime"])
        rp, perm = r["row_ptr"], r["perm"]
        for g, t in zip(r["ins_runtime"], r["rep_trace"]):
            rows = w.patterns[int(g)][1]
            for k in REP_COLS:
                assert np.array_equal(rows[k], sub[k][perm[rp[t]:rp[t + 1]]]), (g, k)
        e2r = w.entry2runtimes()
        assert len(e2r) == max(r["entry2runtimes"]) + 1
        for e, mix in e2r.items():
            assert list(mix.items()) == list(r["entry2runtimes"].get(e, {}).items()), e
        want = O.tr2data(r)
        got = w.tr2data()
        assert list(got) == list(want)
        for tid, v in want.items():
            assert (got[tid]["entry_id"], got[tid]["runtime_id"], got[tid]["timestamp"], got[tid]["y"]) == \
                (v["entry_id"], v["runtime_id"], v["timestamp"], int(v["y"]))


def _recount(w):
    """The store's content recomputed from the surviving traces alone."""
    counts, first = {}, {}
    for e, g, _, _ in w.traces.values():
        counts.setdefault(e, {}).setdefault(g, 0)
        counts[e][g] += 1
    return counts


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_evictions_agree_with_a_brute_force_recount(seed):
    cols = make_random_trace_table(10 + seed, 2500, rows=(1, 8), n_patterns=250, n_entries=8, n_ms=64, n_if=8,
                                   span=240000)
    rng = np.random.default_rng(seed)
    parts, _ = _split(cols, lambda u: rng.integers(0, 6, u.shape[0]))
    w = TraceWindow()
    seen = set()
    for step, part in enumerate(parts):
        w.append(part)
        seen |= set(part["traceid"].tolist())
        cut = [0, 30000, 95000, 95000, 210000, 240000][step]
        before_keys = {e: list(m) for e, m in w.entries.items()}
        old = list(w.traces)
        remap = w.evict(cut)
        # remap: survivors keep their order, -1 for the evicted
        assert [old[i] for i in np.flatnonzero(remap >= 0)] == list(w.traces)
        assert np.array_equal(remap[remap >= 0], np.arange(len(w.traces)))
        assert all(b >= cut for _, _, b, _ in w.traces.values())
        # counts equal a recount; each entry's keys are its old keys in order, minus the emptied ones
        rc = _recount(w)
        for e in range(w.n_ent):
            assert w.entries.get(e, {}) == rc.get(e, {}), e
            assert list(w.entries.get(e, {})) == [g for g in before_keys.get(e, []) if g in rc.get(e, {})]
        # a pattern lives while a trace has its runtime; ids are never reused
        assert set(w.patterns) == {g for _, g, _, _ in w.traces.values()}
        assert all(g < w.next_rt for g in w.patterns)
        assert set(w.by_key.values()) == set(w.patterns)
        # the sizing views agree with the dicts
        cnt, tot = w.pair_counts()
        assert cnt.sum() == tot.sum() == len(w.traces) and (cnt > 0).all()
        rows, ptr = w.key_rows()
        assert rows.shape == (len(KEY_COLS), ptr[-1]) and ptr.shape[0] == len(w.patterns) + 1


def test_a_returning_runtime_is_new():
    cols = _fixture_cols()
    r = O.group_traces(cols)
    bucket = r["bucket"]
    rt = r["runtime"]
    lone = [x for x in np.unique(rt) if len(set(bucket[rt == x])) == 1 and bucket[rt == x][0] == 0]
    g = lone[0]
    t = int(np.flatnonzero(rt == g)[0])
    w = TraceWindow()
    w.append(cols)
    n = w.next_rt
    key = w.patterns[g][0]
    w.evict(1)
    assert g not in w.patterns and key not in w.by_key
    again = {k: v[cols["traceid"] == r["trace_id"][t]].copy() for k, v in cols.items()}
    again["traceid"][:] = cols["traceid"].max() + 1
    w.append(again)
    assert w.by_key[key] == n and w.next_rt == n + 1 and list(w.patterns)[-1] == n


# ---- host checks -----------------------------------------------------------------------------------------------------
def test_before_outside_int64_is_refused():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import PatternStore

    s = PatternStore.__new__(PatternStore)
    for v in (1 << 63, -(1 << 63) - 1, 1 << 80):
        with pytest.raises(PertGnnError, match="outside int64"):
            s.evict_traces(v)


def test_stores_without_runtime_keys_refuse():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import PatternStore

    s = PatternStore.__new__(PatternStore)
    with pytest.raises(PertGnnError, match="from_trace_groups to evict traces"):
        s.evict_traces(30000)


# ---- C-ABI argument checks --------------------------------------------------------------------------------------------
def _store(T=4, n_pat=2, n_ent=3):
    from pert_gnn_kdd23_b200._lib import PertStore

    s = PertStore()
    s.n_traces, s.n_pat, s.n_ent, s.attr_cols = T, n_pat, n_ent, 2
    for f, _ in PertStore._fields_:
        if f not in ("n_pat", "n_ent", "n_res", "n_ms", "attr_cols", "n_traces"):
            setattr(s, f, 1)
    return s


def _state(n_pat=2, pairs=5, ptr=1, trace_pat=1, cnt=1, tot=1, tid=1, key_rows=6):
    from pert_gnn_kdd23_b200._lib import PertIngestState, PertRuntimeKeys

    return PertIngestState(PertRuntimeKeys(n_pat, 8, ptr, 1), trace_pat, tid, cnt, tot, pairs, 10, 12, key_rows)


WS = 1 << 20


@pytest.mark.parametrize("over", [dict(store=None), dict(ing=None), dict(ws=None), dict(sizes=None),
                                  dict(ws_bytes=64), dict(store=_store(T=-1)), dict(store=_store(n_pat=3)),
                                  dict(ing=_state(pairs=-1)), dict(ing=_state(ptr=None)),
                                  dict(ing=_state(trace_pat=None)), dict(ing=_state(cnt=None)),
                                  dict(ing=_state(tot=None)), dict(ing=_state(key_rows=9)),
                                  dict(store=_store(T=1 << 31))])
def test_evict_count_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    a = dict(store=_store(), ing=_state(), ws=1, ws_bytes=WS, sizes=1)
    a.update(over)
    ref = lambda x: C.byref(x) if x is not None else None                # noqa: E731
    assert _lib.lib().pert_ingest_evict_count(ref(a["store"]), ref(a["ing"]), 0, a["ws"], a["ws_bytes"], a["sizes"],
                                              None) == -1


def test_evict_workspace_bytes_rejects_bad_sizes():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    for args in ((-1, 0, 0, 0), (0, -1, 0, 0), (0, 0, -1, 0), (0, 0, 0, -1), (1 << 31, 0, 0, 0)):
        assert L.pert_ingest_evict_workspace_bytes(*args) == -1
    assert L.pert_ingest_evict_workspace_bytes(4, 5, 2, 3) > 0


def _out(**null):
    from pert_gnn_kdd23_b200._lib import EVICT_ARRAYS, PertEvictOut, PertMixOut

    mix = PertMixOut(*[0 if null.get(k) else 1 for k, _ in PertMixOut._fields_])
    return PertEvictOut(mix, *[0 if null.get(k) else 1 for k in EVICT_ARRAYS], null.get("key_ld", 8))


@pytest.mark.parametrize("over", [dict(store=None), dict(ing=None), dict(ws=None), dict(out=None), dict(sizes=None),
                                  dict(ws_bytes=64), dict(sizes=[5, 1, 1, 1, 1, 1]), dict(sizes=[1, 6, 1, 1, 1, 1]),
                                  dict(sizes=[1, 1, 3, 1, 1, 1]), dict(sizes=[1, 1, 1, 11, 1, 1]),
                                  dict(sizes=[1, 1, 1, 1, 13, 1]), dict(sizes=[1, 1, 1, 1, 1, 7]),
                                  dict(sizes=[-1, 1, 1, 1, 1, 1]), dict(out=_out(key_ld=0)),
                                  dict(out=_out(remap=1)), dict(out=_out(trace_tid=1)), dict(out=_out(ent_ptr=1)),
                                  dict(out=_out(cnt=1)), dict(out=_out(pat_new=1)), dict(out=_out(pat_attr=1)),
                                  dict(out=_out(key_rows=1)), dict(out=_out(pat_last=1)), dict(ing=_state(tid=None))])
def test_evict_apply_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    a = dict(store=_store(), ing=_state(), ws=1, ws_bytes=WS, out=_out(), sizes=[2, 3, 1, 5, 6, 3])
    a.update(over)
    ref = lambda x: C.byref(x) if x is not None else None                # noqa: E731
    sizes = (C.c_longlong * 6)(*a["sizes"]) if a["sizes"] is not None else None
    assert _lib.lib().pert_ingest_evict_apply(ref(a["store"]), ref(a["ing"]), sizes, a["ws"], a["ws_bytes"],
                                              ref(a["out"]), None) == -1
