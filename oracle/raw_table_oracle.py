"""Numpy restatement of the reference's get_df() raw-data branch (preprocess.py:201-261) on dictionary-encoded rows
(rawtable.RawTables), with the stable tie rule of rawtable.process_raw: rows with equal timestamps keep concatenation
order, and microservice ids follow the dictionary's (lexicographic) order.  Vectorised, so it also checks the device at
millions of rows.  Returns the arrays ProcessedTables holds."""
import numpy as np

from pert_gnn_kdd23_b200.rawtable import CALL_COLUMNS, USAGE


def _first_codes(v):
    """Series.factorize: code of every value by first appearance."""
    if len(v) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    uniq, first, inv = np.unique(v, return_index=True, return_inverse=True)
    rank = np.empty(len(uniq), np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(uniq))
    return rank[inv.reshape(-1)], v[np.sort(first)]


def _group_stats(vals, gid, G):
    """pandas group max / min / Kahan mean / median of one float64 column (rows in group order), NaN skipped."""
    out = np.full((G, 4), np.nan)
    ok = ~np.isnan(vals)
    nobs = np.bincount(gid[ok], minlength=G)
    mx, mn = np.full(G, -np.inf), np.full(G, np.inf)
    s, c = np.zeros(G), np.zeros(G)
    start = np.searchsorted(gid, np.arange(G))
    pos = np.arange(len(gid)) - start[gid]
    for j in range(int(pos.max(initial=-1)) + 1):     # the j-th row of every group, in row order
        sel = (pos == j) & ok
        g, v = gid[sel], vals[sel]
        mx[g] = np.where(v > mx[g], v, mx[g])
        mn[g] = np.where(v < mn[g], v, mn[g])
        y = v - c[g]
        t = s[g] + y
        cg = (t - s[g]) - y
        c[g] = np.where(np.isnan(cg), 0.0, cg)
        s[g] = t
    has = nobs > 0
    out[has, 0], out[has, 1], out[has, 2] = mx[has], mn[has], s[has] / nobs[has]
    order = np.lexsort((vals, gid))                    # NaN last inside every group
    sv = vals[order]
    h = nobs // 2
    odd = has & (nobs % 2 == 1)
    even = has & (nobs % 2 == 0)
    out[odd, 3] = sv[start[odd] + h[odd]]
    out[even, 3] = (sv[start[even] + h[even]] + sv[start[even] + h[even] - 1]) / 2
    return out


def process_raw(raw, min_occurence=100):
    c = {k: raw.calls[k] for k in CALL_COLUMNS}
    n_ms = len(raw.dicts["ms"])
    # 9. resources: stable sort by (timestamp, ms), groups, statistics
    r = raw.resources
    perm = np.lexsort((r["msname"], r["timestamp"]))
    ts, ms = r["timestamp"][perm], r["msname"][perm]
    start = np.ones(len(perm), bool)
    start[1:] = (ts[1:] != ts[:-1]) | (ms[1:] != ms[:-1])
    gid = np.cumsum(start) - 1
    G = int(start.sum())
    vals = np.concatenate([_group_stats(r[u][perm], gid, G) for u in USAGE], axis=1)
    g_ts, g_ms = ts[start], ms[start]
    has_res = np.zeros(n_ms, bool)
    has_res[ms] = True
    # 1. drop_duplicates, keeping the first row;  2. stable sort by timestamp
    rows = np.stack([c[k] for k in CALL_COLUMNS], axis=1)
    _, first = np.unique(rows, axis=0, return_index=True)
    kept = np.sort(first)
    order = kept[np.argsort(c["timestamp"][kept], kind="stable")]
    s = {k: v[order] for k, v in c.items()}
    # 3. traceid and interface codes over the sorted table
    tr_new, tr_code = _first_codes(s["traceid"])
    if_new, if_code = _first_codes(s["interface"])
    # 4. entries
    tr = s["traceid"]
    n_tr = len(raw.dicts["traceid"])
    tmin = np.full(n_tr, np.iinfo(np.int64).max)
    np.minimum.at(tmin, tr, s["timestamp"])
    art = np.abs(s["rt"])
    amax = np.zeros(n_tr, np.int64)
    np.maximum.at(amax, tr, art)
    http = raw.dicts["rpctype"].index("http") if "http" in raw.dicts["rpctype"] else -1
    unk = raw.dicts["ms"].index("(?)") if "(?)" in raw.dicts["ms"] else -1
    cand = (s["rpctype"] == http) & (s["timestamp"] == tmin[tr]) & (art == amax[tr])
    q = cand & (s["um"] == unk)
    P = np.arange(len(tr))
    ncand, nq = np.bincount(tr[cand], minlength=n_tr), np.bincount(tr[q], minlength=n_tr)
    cpos, qpos = np.full(n_tr, -1), np.full(n_tr, -1)
    for arr, m in ((cpos, cand), (qpos, q)):
        u, f = np.unique(tr[m], return_index=True)
        arr[u] = P[m][f]
    epos = np.where(ncand == 1, cpos, np.where((ncand > 1) & (nq == 1), qpos, -1))
    has_entry = epos[tr] >= 0
    ekey = s["dm"][epos[tr]] * len(raw.dicts["interface"]) + s["interface"][epos[tr]]
    ent_new = np.full(len(tr), -1)
    rpc_new, rty_new = np.full(len(tr), -1), np.full(len(tr), -1)
    ent_new[has_entry], ent_key = _first_codes(ekey[has_entry])
    rpc_new[has_entry], rpc_code = _first_codes(s["rpcid"][has_entry])
    rty_new[has_entry], rty_code = _first_codes(s["rpctype"][has_entry])
    # 5. coverage: distinct {um, dm} per trace, the share with resource rows (IEEE double quotient)
    pairs = np.unique(np.concatenate([tr[has_entry] * n_ms + s["um"][has_entry],
                                      tr[has_entry] * n_ms + s["dm"][has_entry]]))
    ndist = np.bincount(pairs // n_ms, minlength=n_tr)
    nres = np.bincount(pairs // n_ms, weights=has_res[pairs % n_ms], minlength=n_tr).astype(np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        covered = (epos >= 0) & (nres.astype(np.float64) / ndist.astype(np.float64) >= 0.6)
    # 6. occurrences per entry (traces surviving 5)
    t_ent = np.full(n_tr, -1)
    t_ent[tr[has_entry]] = ent_new[has_entry]
    cnt = np.bincount(t_ent[covered], minlength=len(ent_key))
    keep_t = covered & (cnt[np.maximum(t_ent, 0)] > min_occurence)
    keep = keep_t[tr]
    # 7. microservice ids: every resource ms and the surviving um / dm, in dictionary order
    used = has_res.copy()
    used[s["um"][keep]] = True
    used[s["dm"][keep]] = True
    ms_id = np.cumsum(used) - 1
    # 8. the processed columns
    out = {"traceid": tr_new, "timestamp": s["timestamp"], "rpcid": rpc_new, "um": ms_id[s["um"]],
           "dm": ms_id[s["dm"]], "interface": if_new, "rpctype": rty_new, "rt": s["rt"], "entryid": ent_new}
    out = {k: v[keep].astype(np.int64) for k, v in out.items()}
    n_if = len(raw.dicts["interface"])
    if_id = np.full(n_if, -1)
    if_id[if_code] = np.arange(len(if_code))
    return {"columns": out, "row": order[keep], "resource_index": np.stack([g_ts, ms_id[g_ms]], axis=1),
            "resource_values": vals, "ms_code": np.flatnonzero(used), "tr_code": tr_code, "if_code": if_code,
            "rpc_code": rpc_code, "rty_code": rty_code, "ent_dm": ent_key // n_if, "ent_if": if_id[ent_key % n_if]}
