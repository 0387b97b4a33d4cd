"""What keeping the conformal score table current costs (ScoreDistribution.insert / evict, pert_cpd_merge).

Arms, on synthetic windows of n in {1e5, 1e6, 1e7} graphs whose buckets hold delta graphs each, for delta in {1e3,
1e4, 1e5} and three entry mixes (64 uniform entries, 1e4 entries, a Zipf mix where one entry holds 90 %):
  * update: the steady state of a sliding window, insert delta new graphs (a bucket of their own) then evict the
    oldest bucket (delta graphs), each with its fit of the change, its merge and its status read (the evict also with
    its split of the log); ms of the pair, each call timed on its own with the new graphs made beforehand.
  * refit: the baseline, ScoreDistribution.fit (pert_cpd_fit) of the whole updated log; ms.
  The two are alternated, --runs times each; median [min, max].
  * merge+ / merge-: pert_cpd_merge alone, inserting and removing the delta table, CUDA events around --reps calls;
    its algorithmic bytes (the old table and the delta table read once, the new table written once) over its time,
    and their share of the 3.35 TB/s data-sheet HBM bandwidth.
Prints the card name, power limit and clocks, one JSON line per measurement and a summary.

    python tools/time_score_window.py [--runs 3] [--reps 20] [--sizes 100000,1000000,10000000]
"""
import argparse
import json
import statistics

import torch

from measure import HBM_BYTES_PER_S, card, timed


def make_set(n, mix, dev, seed):
    g = torch.Generator(dev).manual_seed(seed)
    if mix == "uniform64":
        G, e = 64, torch.randint(0, 64, (n,), device=dev, generator=g)
    elif mix == "entries1e4":
        G, e = 10 ** 4, torch.randint(0, 10 ** 4, (n,), device=dev, generator=g)
    else:
        G = 10 ** 4
        e = torch.where(torch.rand(n, device=dev, generator=g) < 0.9, torch.full((n,), G // 2, device=dev),
                        torch.randint(0, G, (n,), device=dev, generator=g))
    y = torch.randint(0, 2000, (n,), device=dev, generator=g)
    yhat = y.float() + 100 * torch.randn(n, device=dev, generator=g)
    return y, yhat, e.to(torch.int64), G


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="100000,1000000,10000000")
    ap.add_argument("--deltas", default="1000,10000,100000")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.train import ScoreDistribution, _cpd_fit

    print(json.dumps({"card": card(sm_clock=True)}), flush=True)
    dev = "cuda"
    results = {}

    def record(key, value, **extra):
        results.setdefault(key, []).append(value)
        print(json.dumps(dict(arm=key[0], case=key[1], ms=value, **extra)), flush=True)

    for n in [int(x) for x in a.sizes.split(",")]:
        for delta in [int(x) for x in a.deltas.split(",")]:
            if delta >= n:
                continue
            for mix in ("uniform64", "entries1e4", "zipf90"):
                case = f"n={n} delta={delta} {mix}"
                y, yhat, e, G = make_set(n, mix, dev, 0)
                ts = torch.arange(n, device=dev) // delta
                d = ScoreDistribution.fit(y, yhat, e, G, 0.5, ts=ts)
                oldest = [0]

                def batch(i):
                    yb, yhb, eb, _ = make_set(delta, mix, dev, i)
                    return yb, yhb, eb, torch.full((delta,), n // delta + i, device=dev, dtype=torch.int64)

                def update(b):
                    _, ms_in = timed(lambda: d.insert(*b))
                    oldest[0] += 1
                    _, ms_out = timed(lambda: d.evict(oldest[0]))
                    return ms_in, ms_out

                def refit():
                    return ScoreDistribution.fit(d.log_y, d.log_yhat, d.log_entry, d.n_groups, 0.5)

                update(batch(0))
                refit()
                for r in range(a.runs):
                    ms_in, ms_out = update(batch(r + 1))
                    record(("update", case), ms_in + ms_out, insert_ms=ms_in, evict_ms=ms_out)
                    _, ms = timed(refit)
                    record(("refit", case), ms)
                ref = refit()
                print(json.dumps({"case": case, "window": d.log_y.numel(), "update_equal_to_refit":
                                  bool(torch.equal(ref.ptr, d.ptr) and torch.equal(ref.scores.view(torch.int32),
                                                                                   d.scores.view(torch.int32)))}),
                      flush=True)

                # pert_cpd_merge alone, on a fixed old table and delta table
                yb, yhb, eb, _ = make_set(delta, mix, dev, 99)
                st = torch.zeros(1, dtype=torch.int32, device=dev)
                dsc, dptr = _cpd_fit(yb, yhb, 1, 0, eb, delta, G, st)
                bigger = ScoreDistribution.fit(torch.cat([d.log_y, yb]), torch.cat([d.log_yhat, yhb]),
                                               torch.cat([d.log_entry, eb]), G, 0.5)
                for sign, old in ((1, d), (-1, bigger)):
                    n_old, n_d = old.scores.numel(), dsc.numel()
                    ws_bytes = _lib.lib().pert_cpd_merge_workspace_bytes(G, G, n_old, n_d)
                    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                    out = torch.empty(n_old + sign * n_d, device=dev)
                    optr = torch.empty(G + 2, dtype=torch.int64, device=dev)

                    def merge():
                        _lib.call("pert_cpd_merge", _lib.ptr(old.scores), _lib.ptr(old.ptr), G, n_old, _lib.ptr(dsc),
                                  _lib.ptr(dptr), G, n_d, sign, _lib.ptr(out), _lib.ptr(optr), _lib.ptr(ws), ws_bytes,
                                  _lib.ptr(st), _lib.stream())

                    merge()
                    nbytes = 4 * (n_old + n_d + out.numel()) + 8 * 3 * (G + 2)
                    for _ in range(a.runs):
                        _, ms = timed(merge, reps=a.reps)
                        record(("merge+" if sign > 0 else "merge-", case), ms, bytes=nbytes,
                               tb_per_s=nbytes / (ms * 1e-3) / 1e12, hbm_share=nbytes / (ms * 1e-3) / HBM_BYTES_PER_S)
                    assert int(st.item()) == 0
                del d, y, yhat, e, ts, bigger, ref
                torch.cuda.empty_cache()

    print("summary (median [min, max] over runs, ms):")
    for (arm, case), v in results.items():
        print(f"  {arm:7s} {case:38s}: {statistics.median(v):.4g}  [{min(v):.4g}, {max(v):.4g}]")


if __name__ == "__main__":
    main()
