"""Times rawtable.RawStream.process on chunks of a stream that holds a long history, against process_raw on the same
chunk alone and on history + chunk.

  python tools/time_raw_stream.py                              # 10^6-trace history, chunks of 2e4 and 1e5 traces

Arms, alternated within every repetition after one warm-up call each (a chunk's traceids are relabelled for every
call before the timed windows, since a stream refuses a traceid it has seen):
  stream       RawStream.process on a stream whose history is --history traces (about 30 rows each);
  fresh        RawStream.process on a stream that has seen one chunk only: the same call without the history;
  chunk        process_raw of the chunk alone;
  whole        process_raw of a table of history + chunk traces (what re-running process_raw over the window costs).
Each is one pair of CUDA events around the whole call, host-to-device copies and host synchronisations included, CSV
parsing excluded (the tables are generated already encoded), as tools/time_raw_tables.py times process_raw.  The host
part of a stream call that maps the chunk's dictionaries to stream codes (RawStream._map) is timed on its own with a
host clock and reported separately; it is included in ``stream``.
"""
import argparse
import json
import time

import numpy as np
import torch

from measure import card, timed
from pert_gnn_kdd23_b200.rawtable import RawStream, RawTables, process_raw
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables


def relabel(raw, tag):
    """The chunk with traceids no other chunk has."""
    d = dict(raw.dicts, traceid=[f"{tag}/{v}" for v in raw.dicts["traceid"]])
    return RawTables(raw.calls, raw.resources, d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--history", type=int, default=1_000_000)
    ap.add_argument("--chunks", type=int, nargs="+", default=[20_000, 100_000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = card(split=True)
    out = {"gpu": name, "power_limit": power, "history_traces": a.history, "sizes": {}}
    hist = make_random_raw_tables(1, a.history)
    out["history_rows"] = len(hist)
    big = RawStream("cuda", min_occurence=100)
    big.process(hist).check()
    del hist
    calls = iter(range(1 << 30))                                 # a fresh traceid prefix for every stream call
    for n in a.chunks:
        chunk = make_random_raw_tables(2, n)
        whole = make_random_raw_tables(3, a.history + n)
        fresh = RawStream("cuda", min_occurence=100)
        fresh.process(relabel(chunk, "seed")).check()
        pre = {k: iter([relabel(chunk, f"{k}{next(calls)}") for _ in range(a.reps + 1)]) for k in ("b", "f")}
        arms = {"stream": lambda: big.process(next(pre["b"])),        # relabelled before the timed window
                "fresh": lambda: fresh.process(next(pre["f"])),
                "chunk": lambda: process_raw(chunk, "cuda"),
                "whole": lambda: process_raw(whole, "cuda")}
        ms = {k: [] for k in arms}
        for k, f in arms.items():                                # warm-up
            f().check()
        map_ms = []
        for _ in range(a.reps):
            for k, f in arms.items():
                p, t = timed(f)
                p.check()
                ms[k].append(t)
            c = relabel(chunk, f"m{next(calls)}")
            t0 = time.perf_counter()
            big._map(c)
            map_ms.append((time.perf_counter() - t0) * 1e3)
        med = {k: float(np.median(v)) for k, v in ms.items()}
        out["sizes"][n] = {"rows": len(chunk), "ms": {k: sorted(v) for k, v in ms.items()}, "map_ms": sorted(map_ms),
                           "stream_over_chunk": med["stream"] / med["chunk"],
                           "stream_over_fresh": med["stream"] / med["fresh"]}
        del whole
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
