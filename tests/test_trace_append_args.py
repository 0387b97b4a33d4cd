"""PatternStore.append_traces without a GPU: the chunk-ordered grouping (tests/trace_chunk_ref.py) against the oracle
and against a brute-force statement of its ordering rules, the host argument checks, and the C-ABI argument checks of
csrc/ingest.cu."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table
from tests import trace_chunk_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_preprocess.npz")


def _fixture_cols():
    return make_trace_table(int(np.load(GOLD)["seed"]))["columns"]


def _same(a, b):
    for k in ("trace_id", "entry", "runtime", "bucket", "y", "order", "occurrences", "ins_runtime", "rep_trace",
              "row_ptr", "perm"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    assert list(a["entry2runtimes"]) == list(b["entry2runtimes"])
    for e, v in b["entry2runtimes"].items():
        assert list(a["entry2runtimes"][e].items()) == list(v.items()), e


@pytest.mark.parametrize("cols", [_fixture_cols(), make_random_trace_table(3, 3000, rows=(1, 12), n_patterns=300)])
def test_one_chunk_is_the_oracle(cols):
    want = O.group_traces(cols)
    _same(R.group_traces(cols), want)
    _same(R.group_traces(cols, np.full(len(cols["traceid"]), 7)), want)


def _chunk_of_rows(cols, n_chunks, seed):
    """A random chunk per trace, broadcast to its rows."""
    tid = cols["traceid"]
    u, inv = np.unique(tid, return_inverse=True)
    return np.random.default_rng(seed).integers(0, n_chunks, u.shape[0])[inv]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_chunk_order_rules_by_brute_force(seed):
    """Groupings of the prefixes chunks 0..c: what the store holds after c + 1 appends.  Each must extend the one
    before by the rules of append_traces."""
    cols = _fixture_cols()
    ch = _chunk_of_rows(cols, 4, seed)
    prev = None
    for c in range(4):
        rows = ch <= c
        sub = {k: v[rows] for k, v in cols.items()}
        res = R.group_traces(sub, ch[rows])
        T, tid = len(res["trace_id"]), res["trace_id"]
        # traces by (chunk, traceid); the iteration order is (chunk, entry, traceid)
        key = list(zip(res["trace_chunk"], tid))
        assert key == sorted(key)
        it = [(res["trace_chunk"][t], res["entry"][t], tid[t]) for t in res["order"]]
        assert it == sorted(it)
        # runtimes: equal key rows <=> equal id; ids numbered by first (chunk, traceid)
        rp, perm = res["row_ptr"], res["perm"]
        rows_of = [tuple(map(tuple, np.stack([sub[k][perm[rp[t]:rp[t + 1]]] for k in ("um", "dm", "interface")], 1)))
                   for t in range(T)]
        first = {}
        for t in range(T):
            first.setdefault(rows_of[t], len(first))
            assert res["runtime"][t] == first[rows_of[t]]
        if prev is not None:
            pres, ptid = prev
            n_old = len(pres["ins_runtime"])
            T_old = len(ptid)
            assert np.array_equal(tid[:T_old], ptid) and np.array_equal(res["runtime"][:T_old], pres["runtime"])
            # old traces keep their iteration positions; the new ones follow
            assert np.array_equal(res["order"][:T_old], pres["order"])
            # old runtimes keep representative and insertion index; new ones follow in the chunk's iteration order
            assert np.array_equal(res["ins_runtime"][:n_old], pres["ins_runtime"])
            assert np.array_equal(tid[res["rep_trace"][:n_old]], ptid[pres["rep_trace"]])
            new_rt = res["ins_runtime"][n_old:]
            assert sorted(new_rt) == list(range(n_old, len(res["ins_runtime"])))
            pos = {t: p for p, t in enumerate(res["order"])}
            assert all(res["trace_chunk"][t] == c for t in res["rep_trace"][n_old:])
            assert [pos[t] for t in res["rep_trace"][n_old:]] == sorted(pos[t] for t in res["rep_trace"][n_old:])
            # entry mixes: old keys in order, then the new ones; probability = (old + chunk count) / (old + chunk total)
            for e, mix in res["entry2runtimes"].items():
                old = list(pres["entry2runtimes"].get(e, {}))
                assert list(mix)[:len(old)] == old
                ts = [t for t in range(T) if res["entry"][t] == e]
                for r, p in mix.items():
                    assert p == sum(res["runtime"][t] == r for t in ts) / len(ts)
        prev = (res, tid)


def test_a_traceid_in_two_chunks_is_refused():
    cols = _fixture_cols()
    ch = np.zeros(len(cols["traceid"]), dtype=np.int64)
    ch[np.flatnonzero(cols["traceid"] == cols["traceid"][0])[-1]] = 1
    with pytest.raises(ValueError, match="two chunks"):
        R.group_traces(cols, ch)


def test_microservice_ids_are_checked_and_the_first_bad_row_named():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import _check_span_ms

    cols = _fixture_cols()
    _check_span_ms(cols, 24)
    for col, row, v in (("um", 9, 24), ("dm", 4, -1), ("um", 0, 1 << 40)):
        bad = {k: a.copy() for k, a in cols.items()}
        bad[col][row] = v
        bad["dm"][row + 3] = 99                                          # a later bad row is not the one named
        with pytest.raises(PertGnnError, match=f"span row {row}: {col} = {v} is outside"):
            _check_span_ms(bad, 24)


def test_stores_without_runtime_keys_refuse():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import PatternStore

    s = PatternStore.__new__(PatternStore)
    with pytest.raises(PertGnnError, match="from_trace_groups"):
        s.append_traces(_fixture_cols())


def _keys(n=2, ld=4, ptr=1, rows=1):
    from pert_gnn_kdd23_b200._lib import PertRuntimeKeys

    return PertRuntimeKeys(n, ld, ptr, rows)


def _table(S=64, bits=64, slot=1, h=1):
    from pert_gnn_kdd23_b200._lib import PertRuntimeTable

    return PertRuntimeTable(S, bits, slot, h, h)


@pytest.mark.parametrize("over", [dict(keys=None), dict(first=-1), dict(first=3), dict(table=_table(S=48)),
                                  dict(table=_table(S=32)), dict(table=_table(bits=0)), dict(table=_table(bits=65)),
                                  dict(table=_table(slot=None)), dict(table=_table(h=None)),
                                  dict(keys=_keys(n=40)), dict(keys=_keys(ptr=None)), dict(keys=_keys(n=-1))])
def test_table_insert_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    a = dict(keys=_keys(), first=0, table=_table())
    a.update(over)
    k, t = a["keys"], a["table"]
    assert _lib.lib().pert_ingest_table_insert(C.byref(k) if k else None, a["first"], C.byref(t), None) == -1


@pytest.mark.parametrize("over", [dict(chunk=None), dict(table=None), dict(n_new=None), dict(ws=None),
                                  dict(ws_bytes=8), dict(pat_of=None), dict(rin=None), dict(chunk=_keys(n=-2)),
                                  dict(keys=_keys(n=33))])
def test_match_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    a = dict(keys=_keys(), table=_table(), chunk=_keys(n=3), rin=1, pat_of=1, n_new=1, ws=1, ws_bytes=1 << 20)
    a.update(over)
    ref = lambda s: C.byref(s) if s is not None else None                # noqa: E731
    assert L.pert_ingest_match(ref(a["keys"]), ref(a["table"]), ref(a["chunk"]), a["rin"], a["pat_of"], 1, 1,
                               a["n_new"], a["ws"], a["ws_bytes"], None) == -1
    assert L.pert_ingest_match_workspace_bytes(-1) == -1


def _mix(n_ent=3, n_pairs=4, ptr=1):
    from pert_gnn_kdd23_b200._lib import PertChunkMix

    return PertChunkMix(n_ent, n_pairs, ptr, 1, 1, 1, 1, 1)


@pytest.mark.parametrize("over", [dict(store=None), dict(chunk=None), dict(out=None), dict(ws=None),
                                  dict(ws_bytes=16), dict(n_pairs=-1), dict(n_ent_out=1), dict(chunk=_mix(n_ent=9)),
                                  dict(chunk=_mix(ptr=None)), dict(chunk=_mix(n_pairs=-1)), dict(cnt=None),
                                  dict(tot=None), dict(nptr=None), dict(n_pairs=1 << 31)])
def test_merge_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertMixOut, PertStore

    s = PertStore()
    s.n_ent = 2
    for f in ("ent_ptr", "ent_pat", "ent_nodes", "ent_edges"):
        setattr(s, f, 1)
    a = dict(store=s, cnt=1, tot=1, n_pairs=5, chunk=_mix(), nptr=1, n_ent_out=3, out=PertMixOut(*([1] * 7)), ws=1,
             ws_bytes=1 << 20)
    a.update(over)
    ref = lambda x: C.byref(x) if x is not None else None                # noqa: E731
    assert _lib.lib().pert_ingest_merge(ref(a["store"]), a["cnt"], a["tot"], a["n_pairs"], ref(a["chunk"]),
                                        a["nptr"], 1, a["n_ent_out"], ref(a["out"]), a["ws"], a["ws_bytes"],
                                        None) == -1
    assert _lib.lib().pert_ingest_merge_workspace_bytes(-1, 0, 0) == -1
