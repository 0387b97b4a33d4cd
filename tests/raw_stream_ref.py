"""Numpy restatement of rawtable.RawStream (DESIGN.md §8p): oracle/raw_table_oracle.py's process_raw, run over one
chunk at a time and continued from the stream's state.  ``defects`` switches on one deliberate error each, so the
tests can show that the GPU comparisons would catch it:
  "rank_by_value"  new interface / rpcid / rpctype / entry ids ranked by stream code instead of first position;
  "chunk_counts"   the occurrence filter counts this chunk's traces only;
  "chunk_has_res"  coverage reads this chunk's resource rows only;
  "number_dropped" microservices of dropped rows get ids too."""
import numpy as np

from oracle import raw_table_oracle as O
from pert_gnn_kdd23_b200.rawtable import CALL_COLUMNS, USAGE

CODED = ("ms", "interface", "rpcid", "rpctype")
DEFECTS = ("rank_by_value", "chunk_counts", "chunk_has_res", "number_dropped")


def _grow(a, n, fill):
    return np.concatenate([a, np.full(n - len(a), fill, a.dtype)]) if n > len(a) else a


class RefStream:
    def __init__(self, min_occurence=100, defects=()):
        assert set(defects) <= set(DEFECTS)
        self.min_occurence, self.defects = min_occurence, set(defects)
        self.codes = {k: {} for k in CODED}                       # value -> stream code
        self.ids = {k: np.zeros(0, np.int64) for k in CODED}      # stream code -> id, -1 none
        self.has_res = np.zeros(0, bool)                          # per ms stream code
        self.entries, self.ent_cnt = {}, np.zeros(0, np.int64)    # (dm, interface) stream codes -> id; counts
        self.n_tr = 0
        self.names = {k: [] for k in ("ms_names", "traceid_names", "interface_names", "rpcid_values",
                                      "rpctype_names", "entry_names")}

    def _continue(self, col, sc):
        """Ids of the stream codes ``sc`` (positions in sorted order): the old id, or next + rank among the new ones
        (by first position, or by stream code under rank_by_value); returns them and the new codes in id order."""
        ids = self.ids[col]
        out = ids[sc].copy()
        new = out < 0
        nxt = int(ids.max(initial=-1)) + 1
        if "rank_by_value" in self.defects:
            uniq, rank = np.unique(sc[new], return_inverse=True)
        else:
            rank, uniq = O._first_codes(sc[new])
        out[new] = nxt + rank.reshape(-1)
        ids[uniq] = nxt + np.arange(len(uniq))
        return out, uniq

    def process(self, raw):
        d = raw.dicts
        maps = {}
        for col in CODED:
            known = self.codes[col]
            maps[col] = np.array([known.setdefault(v, len(known)) for v in d[col]], np.int64)
            self.ids[col] = _grow(self.ids[col], len(known), -1)
        self.has_res = _grow(self.has_res, len(self.codes["ms"]), False)
        inv = {col: {c: v for v, c in self.codes[col].items()} for col in CODED}
        c = {k: raw.calls[k] for k in CALL_COLUMNS}
        n_ms = len(d["ms"])
        # 9. resources, as the oracle
        r = raw.resources
        perm = np.lexsort((r["msname"], r["timestamp"]))
        ts, ms = r["timestamp"][perm], r["msname"][perm]
        start = np.ones(len(perm), bool)
        start[1:] = (ts[1:] != ts[:-1]) | (ms[1:] != ms[:-1])
        gid = np.cumsum(start) - 1
        G = int(start.sum())
        vals = np.concatenate([O._group_stats(r[u][perm], gid, G) for u in USAGE], axis=1)
        own_res = np.zeros(n_ms, bool)
        own_res[ms[(ms >= 0) & (ms < n_ms)]] = True
        has_res = own_res.copy()
        if "chunk_has_res" not in self.defects:
            has_res |= self.has_res[maps["ms"]]
        # 1. + 2.
        rows = np.stack([c[k] for k in CALL_COLUMNS], axis=1)
        _, first = np.unique(rows, axis=0, return_index=True)
        kept = np.sort(first)
        order = kept[np.argsort(c["timestamp"][kept], kind="stable")]
        s = {k: v[order] for k, v in c.items()}
        tr = s["traceid"]
        # 3. traceid ids continue the counter; interface ids over every row
        tr_rank, tr_code = O._first_codes(tr)
        tr_new = self.n_tr + tr_rank
        if_new, if_codes = self._continue("interface", maps["interface"][s["interface"]])
        # 4. entries (as the oracle), keyed by stream codes
        n_tr = len(d["traceid"])
        tmin = np.full(n_tr, np.iinfo(np.int64).max)
        np.minimum.at(tmin, tr, s["timestamp"])
        art = np.abs(s["rt"])
        amax = np.zeros(n_tr, np.int64)
        np.maximum.at(amax, tr, art)
        http = d["rpctype"].index("http") if "http" in d["rpctype"] else -1
        unk = d["ms"].index("(?)") if "(?)" in d["ms"] else -1
        cand = (s["rpctype"] == http) & (s["timestamp"] == tmin[tr]) & (art == amax[tr])
        q = cand & (s["um"] == unk)
        P = np.arange(len(tr))
        ncand, nq = np.bincount(tr[cand], minlength=n_tr), np.bincount(tr[q], minlength=n_tr)
        cpos, qpos = np.full(n_tr, -1), np.full(n_tr, -1)
        for arr, m in ((cpos, cand), (qpos, q)):
            u, f = np.unique(tr[m], return_index=True)
            arr[u] = P[m][f]
        epos = np.where(ncand == 1, cpos, np.where((ncand > 1) & (nq == 1), qpos, -1))
        he = epos[tr] >= 0
        ekey = maps["ms"][s["dm"][epos[tr]]] * (1 << 32) + maps["interface"][s["interface"][epos[tr]]]
        ent_new = np.full(len(tr), -1)
        known = np.array([self.entries.get(int(k), -1) for k in ekey[he]], np.int64)
        nxt = len(self.entries)
        fresh = known < 0
        if "rank_by_value" in self.defects:
            ukeys, rank = np.unique(ekey[he][fresh], return_inverse=True)
        else:
            rank, ukeys = O._first_codes(ekey[he][fresh])
        known[fresh] = nxt + rank.reshape(-1)
        ent_new[he] = known
        for i, k in enumerate(ukeys):
            self.entries[int(k)] = nxt + i
        new_ent_keys = ukeys
        rpc_new, rty_new = np.full(len(tr), -1), np.full(len(tr), -1)
        rpc_new[he], rpc_codes = self._continue("rpcid", maps["rpcid"][s["rpcid"][he]])
        rty_new[he], rty_codes = self._continue("rpctype", maps["rpctype"][s["rpctype"][he]])
        # 5. coverage
        pairs = np.unique(np.concatenate([tr[he] * n_ms + s["um"][he], tr[he] * n_ms + s["dm"][he]]))
        ndist = np.bincount(pairs // n_ms, minlength=n_tr) if n_ms else np.zeros(n_tr, np.int64)
        nres = (np.bincount(pairs // n_ms, weights=has_res[pairs % n_ms], minlength=n_tr).astype(np.int64)
                if n_ms else np.zeros(n_tr, np.int64))
        with np.errstate(invalid="ignore", divide="ignore"):
            covered = (epos >= 0) & (nres.astype(np.float64) / ndist.astype(np.float64) >= 0.6)
        # 6. occurrences: the stream's counts so far plus this chunk's
        t_ent = np.full(n_tr, -1)
        t_ent[tr[he]] = ent_new[he]
        self.ent_cnt = _grow(self.ent_cnt, len(self.entries), 0)
        chunk = np.bincount(t_ent[covered], minlength=len(self.entries))
        total = chunk if "chunk_counts" in self.defects else self.ent_cnt + chunk
        keep_t = covered & (total[np.maximum(t_ent, 0)] > self.min_occurence)
        self.ent_cnt = self.ent_cnt + chunk
        keep = keep_t[tr]
        # 7. microservice ids: names of this chunk's resource rows and surviving um / dm without an id, name order
        rows_ms = keep if "number_dropped" not in self.defects else np.ones(len(tr), bool)
        used = own_res | has_res
        used[s["um"][rows_ms]] = True
        used[s["dm"][rows_ms]] = True
        ms_ids = self.ids["ms"]
        cid = ms_ids[maps["ms"]]
        new_ms = used & (cid < 0)
        nxt = int(ms_ids.max(initial=-1)) + 1
        chunk_id = np.where(cid >= 0, cid, nxt + np.cumsum(new_ms) - 1)
        ms_ids[maps["ms"][new_ms]] = chunk_id[new_ms]
        self.has_res[maps["ms"][own_res]] = True
        # 8. the processed columns
        out = {"traceid": tr_new, "timestamp": s["timestamp"], "rpcid": rpc_new, "um": chunk_id[s["um"]],
               "dm": chunk_id[s["dm"]], "interface": if_new, "rpctype": rty_new, "rt": s["rt"], "entryid": ent_new}
        out = {k: v[keep].astype(np.int64) for k, v in out.items()}
        res_ms = np.full(len(r["msname"]), -1, np.int64)
        ok = (r["msname"] >= 0) & (r["msname"] < n_ms)
        res_ms[ok] = chunk_id[r["msname"][ok]]
        # name lists
        nm = self.names
        self.n_tr += len(tr_code)
        nm["traceid_names"] += [d["traceid"][i] for i in tr_code]
        nm["ms_names"] += [d["ms"][i] for i in np.flatnonzero(new_ms)]
        nm["interface_names"] += [inv["interface"][i] for i in if_codes]
        nm["rpcid_values"] += [inv["rpcid"][i] for i in rpc_codes]
        nm["rpctype_names"] += [inv["rpctype"][i] for i in rty_codes]
        if_ids = self.ids["interface"]
        nm["entry_names"] += [f"{inv['ms'][int(k) >> 32]}_{if_ids[int(k) & 0xffffffff]}" for k in new_ent_keys]
        return {"columns": out, "row": order[keep], "resource_index": np.stack([ts[start], chunk_id[ms[start]]], 1),
                "resource_values": vals, "resource_ms": res_ms, "n_ms": int((ms_ids >= 0).sum()),
                "names": {k: list(v) for k, v in nm.items()}}


def chunk_of(raw, call_rows, res_rows):
    """The RawTables of the given call-graph and resource rows of ``raw`` with chunk-local dictionaries (values in
    first-appearance order, microservices recoded to name order by RawTables), as read_raw gives for that chunk."""
    from pert_gnn_kdd23_b200.rawtable import RawTables

    calls = {k: v[call_rows] for k, v in raw.calls.items()}
    res = {k: v[res_rows] for k, v in raw.resources.items()}
    dicts = {}
    for col in ("traceid", "interface", "rpcid", "rpctype"):
        u, inv = np.unique(calls[col], return_inverse=True)
        rank, _ = O._first_codes(calls[col])
        firsts = np.zeros(len(u), np.int64)
        firsts[inv.reshape(-1)] = rank
        order = np.argsort(firsts)
        dicts[col] = [raw.dicts[col][i] for i in u[order]]
        calls[col] = rank
    allms = np.concatenate([calls["um"], calls["dm"], res["msname"]])
    u, inv = np.unique(allms, return_inverse=True)
    dicts["ms"] = [raw.dicts["ms"][i] for i in u]
    inv = inv.reshape(-1)
    R = len(calls["um"])
    calls["um"], calls["dm"], res["msname"] = inv[:R], inv[R:2 * R], inv[2 * R:]
    return RawTables(calls, res, dicts)


def time_chunks(raw, n_chunks, res_first=True, seed=0):
    """``raw`` cut into ``n_chunks`` chunks of whole traces in time order (a trace's time: its first timestamp), at
    random cut points; every resource row in chunk 1 (``res_first``), spread evenly over the chunks, or all rows of
    microservice code m (``"by_ms"``) / of the i-th distinct timestamp (``"by_ts"``) in chunk m (i) mod n_chunks."""
    rng = np.random.default_rng(seed)
    tr = raw.calls["traceid"]
    tmin = np.full(int(tr.max()) + 1, np.iinfo(np.int64).max)
    np.minimum.at(tmin, tr, raw.calls["timestamp"])
    ranks = np.argsort(np.argsort(tmin[np.unique(tr)], kind="stable"), kind="stable")
    traces = np.unique(tr)
    cuts = np.sort(rng.choice(np.arange(1, len(traces)), n_chunks - 1, replace=False))
    part = np.searchsorted(cuts, ranks, side="right")               # chunk of every trace
    t_part = np.zeros(int(tr.max()) + 1, np.int64)
    t_part[traces] = part
    K = len(raw.resources["timestamp"])
    if res_first == "by_ms":                                        # each microservice's rows in one chunk
        r_part = raw.resources["msname"] % n_chunks
    elif res_first == "by_ts":                                      # each timestamp's rows in one chunk
        r_part = np.unique(raw.resources["timestamp"], return_inverse=True)[1].reshape(-1) % n_chunks
    else:
        r_part = np.zeros(K, np.int64) if res_first else np.arange(K) * n_chunks // max(K, 1)
    return [chunk_of(raw, np.flatnonzero(t_part[tr] == k), np.flatnonzero(r_part == k)) for k in range(n_chunks)]
