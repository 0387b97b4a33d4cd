"""What the conformal predictive distribution costs.

Arms:
  * fit: ScoreDistribution.fit (pert_cpd_fit) on synthetic (y, yhat, entry id) sets of n in {1e5, 1e6, 1e7} graphs
    and three entry mixes (64 uniform entries, 1e4 entries, a Zipf mix where one entry holds 90 %), against a torch
    baseline that builds the same table with stable torch.sort calls (by score, then by entry, and the global row by
    score); the two alternated, ms per fit, median and range over --runs.  The algorithmic bytes (fit_bytes: the
    labels, predictions and ids read once, the 2n-float table written once) and their share of the 3.35 TB/s
    data-sheet HBM bandwidth are printed beside the fit's time.
  * queries: ScoreDistribution.tail at Q in {1e6, 1e7} requests and S in {1, 4} thresholds each, and
    ScoreDistribution.quantile at L in {1, 4} levels, on the 1e6-graph Zipf table; requests per s.  Each call includes
    its one status read.
  * predict: train.predict of --requests as-of requests on the PERT-exact store (synthetic.make_pert_artifacts(seed=3),
    4096 traces over 64 entries), alone and followed by tail at two SLO tiers, alternated; requests per s.
Every timed window is bracketed by a device synchronise and CUDA events (tools/measure.py) after a warm-up.  Prints the
card name, power limit and clocks, one JSON line per measurement and a summary.

    python tools/time_distribution.py [--runs 5] [--requests 1000000]
"""
import argparse
import json
import statistics

import numpy as np
import torch

from measure import HBM_BYTES_PER_S, card, timed


def make_set(n, mix, dev, seed=0):
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


def torch_table(y, yhat, e):
    """The same table with torch: a stable sort by score, then a stable sort of that order by entry; row G a sort."""
    s = y.float() - yhat
    s = torch.where(s == 0, torch.zeros_like(s), s)
    by_score = torch.sort(s, stable=True)
    by_entry = torch.sort(e[by_score.indices], stable=True).indices
    return torch.cat([by_score.values[by_entry], by_score.values])


def fit_bytes(n):
    return n * (8 + 4 + 8) + 2 * n * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--requests", type=int, default=10 ** 6)
    ap.add_argument("--predict-batch", type=int, default=4096)
    ap.add_argument("--sizes", default="100000,1000000,10000000")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import ScoreDistribution, fit_distribution, predict

    print(json.dumps({"card": card(sm_clock=True)}), flush=True)
    dev = "cuda"
    results = {}

    def record(key, value, **extra):
        results.setdefault(key, []).append(value)
        print(json.dumps(dict(arm=key[0], case=key[1], ms=value, **extra)), flush=True)

    # ---- fit against the torch baseline
    zipf6 = None
    for n in [int(x) for x in a.sizes.split(",")]:
        for mix in ("uniform64", "entries1e4", "zipf90"):
            y, yhat, e, G = make_set(n, mix, dev)
            ours = ScoreDistribution.fit(y, yhat, e, G, 0.5)
            case = f"n={n} {mix}"
            print(json.dumps({"case": case, "equal_to_torch_baseline":
                              bool(torch.equal(ours.scores.view(torch.int32),
                                               torch_table(y, yhat, e).view(torch.int32)))}), flush=True)
            for _ in range(a.runs):
                _, ms = timed(lambda: ScoreDistribution.fit(y, yhat, e, G, 0.5))
                record(("fit", case), ms, hbm_share=fit_bytes(n) / (ms * 1e-3) / HBM_BYTES_PER_S)
                _, ms = timed(lambda: torch_table(y, yhat, e))
                record(("torch", case), ms)
            if n == 10 ** 6 and mix == "zipf90":
                zipf6 = (ours, G)
            del y, yhat, e, ours
            torch.cuda.empty_cache()

    # ---- queries on the 1e6-graph Zipf table
    if zipf6 is not None:
        d, G = zipf6
        for Q in (10 ** 6, 10 ** 7):
            g = torch.Generator(dev).manual_seed(1)
            yq = 1000 + 100 * torch.randn(Q, device=dev, generator=g)
            eq = torch.randint(-1, G + 1, (Q,), device=dev, generator=g)
            for S in (1, 4):
                x = (yq[:, None] + 50 * torch.randn(Q, S, device=dev, generator=g)).squeeze(1).contiguous()
                d.tail(yq, eq, x)
                for _ in range(a.runs):
                    _, ms = timed(lambda: d.tail(yq, eq, x))
                    record(("tail", f"Q={Q} S={S}"), ms, requests_per_s=Q / (ms / 1e3))
            for lv in ((0.99,), (0.5, 0.9, 0.99, 0.999)):
                d.quantile(yq, eq, lv)
                for _ in range(a.runs):
                    _, ms = timed(lambda: d.quantile(yq, eq, lv))
                    record(("quantile", f"Q={Q} L={len(lv)}"), ms, requests_per_s=Q / (ms / 1e3))
            del yq, eq, x

    # ---- predict alone and predict + tail
    art, _ = make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, device=dev)
    store = PatternStore.from_artifacts(art, dev)
    torch.manual_seed(0)
    m = SAGEDeterministic(*model_args(2)).to(dev)
    d = fit_distribution(m, StoreLoader(store, list(range(len(store))), 256), dev, level=0.5)
    rng = np.random.default_rng(0)
    ok = np.flatnonzero(store._h_ent_pats > 0)
    ts_all = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    ent, ts = rng.choice(ok, a.requests), rng.choice(ts_all, a.requests)
    ent_d = torch.from_numpy(ent).to(dev)
    slo = torch.tensor([[300.0, 600.0]], device=dev).expand(a.requests, 2).contiguous()

    arms = {"predict": lambda: predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True),
            "predict+tail": lambda: d.tail(predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True), ent_d,
                                           slo)}
    for fn in arms.values():
        fn()
    for _ in range(a.runs):
        for arm, fn in arms.items():
            _, ms = timed(fn)
            record(("serve", arm), ms, requests_per_s=a.requests / (ms / 1e3))

    print("summary (median over runs, ms):")
    for (arm, case), v in results.items():
        print(f"  {arm:9s} {case:28s}: {statistics.median(v):.4g}  (min {min(v):.4g}, max {max(v):.4g})")


if __name__ == "__main__":
    main()
