"""Plain numpy restatement of the resource join of request assembly (PatternStore.assemble_requests): which row of
``resource_df`` (the reference's (timestamp, msname) table, pert_gnn.py:40-67) a request at time ``t`` reads for a
microservice.

  (1) the request's time bucket is t // 30000 * 30000, floor division (get_tr2ts_map, preprocess.py:39);
  (2) exact join: the row keyed (bucket, ms), the first of several equal keys (resource_df.loc; the store's lower bound
      over its stably sorted keys); none -> the reference's KeyError;
  (3) as-of join: the row of ms with the largest timestamp <= bucket (resource_df.index.get_indexer([ts],
      method="pad"), the lookup misc.py:373-376 keeps commented out), the first of several rows with that timestamp, so
      an exact hit picks the row of (2); none -> the missing indicator [0 x 8, 1].
"""
import numpy as np

BUCKET = 30000


def time_bucket(ts):
    return np.asarray(ts, dtype=np.int64) // BUCKET * BUCKET


def exact_rows(res_ts, res_ms, q_bucket, q_ms):
    """Row index (into the input rows) of the exact match of every query (bucket, ms), -1 where there is none."""
    return _lookup(res_ts, res_ms, q_bucket, q_ms, asof=False)


def asof_rows(res_ts, res_ms, q_bucket, q_ms):
    """Row index (into the input rows) of the as-of match of every query (bucket, ms), -1 where there is none."""
    return _lookup(res_ts, res_ms, q_bucket, q_ms, asof=True)


def _lookup(res_ts, res_ms, q_bucket, q_ms, asof):
    res_ts, res_ms = np.asarray(res_ts, dtype=np.int64), np.asarray(res_ms, dtype=np.int64)
    q_bucket, q_ms = np.asarray(q_bucket, dtype=np.int64), np.asarray(q_ms, dtype=np.int64)
    n = res_ts.shape[0]
    if n == 0:
        return np.full(q_ms.shape[0], -1, dtype=np.int64)
    order =np.lexsort((np.arange(n), res_ts, res_ms))              # ms, then timestamp, then input order
    # timestamps -> ranks over rows and queries, so (ms, rank) is one int64 key ordered like (ms, timestamp)
    times = np.unique(np.concatenate([res_ts, q_bucket]))
    R = times.shape[0]
    key = res_ms[order] * R + np.searchsorted(times, res_ts[order])
    q_key = q_ms * R + np.searchsorted(times, q_bucket)
    if asof:
        last = np.searchsorted(key, q_key, side="right") - 1         # last row with (ms, ts) <= (q_ms, bucket)
        ok = last >= 0
        ok[ok] = res_ms[order[last[ok]]] == q_ms[ok]
        hit = np.where(ok, key[np.maximum(last, 0)], -1)
    else:
        hit = q_key
    first = np.searchsorted(key, hit, side="left")                  # first row of that key
    found = first < n
    found[found] = key[first[found]] == hit[found]
    if asof:
        found &= ok
    return np.where(found, order[np.minimum(first, n - 1)], -1)


def features(rows, resource_values):
    """x rows [Q, 9] float32 of the joined rows: the 8 statistics and 0, or [0 x 8, 1] where ``rows`` is -1."""
    rows = np.asarray(rows, dtype=np.int64)
    vals = np.asarray(resource_values, dtype=np.float64).astype(np.float32)
    x = np.zeros((rows.shape[0], 9), dtype=np.float32)
    hit = rows >= 0
    x[hit, :8] = vals[rows[hit]]
    x[~hit, 8] = 1.0
    return x
