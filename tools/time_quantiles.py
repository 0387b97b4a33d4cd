"""What a multi-quantile global head costs, and what it predicts: the reference model (one output) against a model with
quantiles = (0.5, 0.9, 0.95, 0.99) (T = 4), arms alternated within one process.

Arms:
  * graphed: GraphedTrainStep at cfg2 (256 graphs of ~200 nodes) on one resident batch, ms per step;
  * bucketed: BucketedTrainStep over a shuffled StoreLoader of PERT-exact artefacts (synthetic.make_pert_artifacts(
    seed=3, n_patterns=256, n_entries=64, n_traces=4096), batches of 256 traces), ms per step over whole epochs;
  * predict: train.predict of --requests requests (as-of join, --predict-batch per slice), requests per second;
  * quality (reported, not asserted): the T = 4 model trained for --epochs epochs on 60 % of the traces, then its
    per-level coverage (share of held-out traces with y <= the level's prediction) and the share of traces whose levels
    cross, from evaluate_bucketed on the other 40 %.
Each timed window is bracketed by a device synchronise and CUDA events (tools/measure.py) after a warm-up that captured
the graphs.  Prints the card name and power limit and one JSON line per run, then a summary.

    python tools/time_quantiles.py [--runs 5] [--steps 200] [--requests 1000000] [--epochs 30]
"""
import argparse
import json
import statistics

import numpy as np
import torch

from measure import card, timed

LEVELS = (0.5, 0.9, 0.95, 0.99)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--requests", type=int, default=10 ** 6)
    ap.add_argument("--predict-batch", type=int, default=4096)
    ap.add_argument("--epochs", type=int, default=30)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_data_list, make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, FlatParams, FusedAdam, GraphedTrainStep,
                                           evaluate_bucketed, predict)

    print(f"card: {card()}", flush=True)
    dev = "cuda"

    def new_model(q):
        torch.manual_seed(0)
        m = SAGEDeterministic(*model_args(2), quantiles=q).to(dev).train()
        return m, FusedAdam(FlatParams(m), lr=3e-4)

    arms = {"T=1": None, "T=4": LEVELS}
    results = {}

    def record(kind, name, value, unit):
        results.setdefault((kind, name), []).append(value)
        print(json.dumps({"arm": kind, "model": name, unit: value}), flush=True)

    # ---- graphed step at cfg2
    batch = Batch.from_data_list(make_data_list(2)).to(dev)
    graphed = {}
    for name, q in arms.items():
        m, opt = new_model(q)
        step = GraphedTrainStep(m, opt)
        for _ in range(10):
            step(batch)
        graphed[name] = step
    for _ in range(a.runs):
        for name, step in graphed.items():
            _, ms = timed(lambda: step(batch), reps=a.steps)
            record("graphed", name, ms, "ms_per_step")

    # ---- bucketed step over a shuffled store
    art, _ = make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, device=dev)
    store = PatternStore.from_artifacts(art, dev)
    ids = list(range(len(store)))
    loader = StoreLoader(store, ids, 256, shuffle=True, generator=torch.Generator().manual_seed(1))
    bucketed = {}
    for name, q in arms.items():
        m, opt = new_model(q)
        step = BucketedTrainStep(m, opt)
        step.reserve(*loader.max_sizes())
        for _ in range(3):
            for d in loader:
                step(d)
        bucketed[name] = step

    def epoch(step):
        n = 0
        for d in loader:
            step(d)
            n += 1
        return n

    for _ in range(a.runs):
        for name, step in bucketed.items():
            n, ms = timed(lambda: epoch(step))
            record("bucketed", name, ms / n, "ms_per_step")

    # ---- predict throughput
    rng = np.random.default_rng(0)
    ok = np.flatnonzero(store._h_ent_pats > 0)
    ts_all = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    ent = rng.choice(ok, a.requests)
    ts = rng.choice(ts_all, a.requests)
    models = {name: bucketed[name].model for name in arms}
    for m in models.values():
        predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True)       # captures every bucket
    for _ in range(a.runs):
        for name, m in models.items():
            out, ms = timed(lambda: predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True))
            record("predict", name, a.requests / (ms / 1e3), "requests_per_s")
    print(json.dumps({"predict_shape": {n: list(predict(m, store, ent[:8], ts[:8], asof=True).shape)
                                        for n, m in models.items()}}), flush=True)

    # ---- quality of the T = 4 model on held-out traces
    cut = int(0.6 * len(ids))
    perm = np.random.default_rng(7).permutation(len(ids))
    train_ids, test_ids = perm[:cut].tolist(), perm[cut:].tolist()
    m, opt = new_model(LEVELS)
    step = BucketedTrainStep(m, opt)
    tl = StoreLoader(store, train_ids, 256, shuffle=True, generator=torch.Generator().manual_seed(3))
    step.reserve(*tl.max_sizes())
    for _ in range(a.epochs):
        for d in tl:
            step(d)
    ev = StoreLoader(store, test_ids, 256)
    mae, mape, qloss = evaluate_bucketed(m, ev, dev)
    met = m.__dict__["_bucketed_eval"].metrics
    print(json.dumps({"quality": {"levels": LEVELS, "epochs": a.epochs, "train_traces": len(train_ids),
                                  "test_traces": len(test_ids), "coverage": met.coverage(), "crossing": met.crossing(),
                                  "mae": mae, "qloss": qloss}}), flush=True)

    print("summary (median over runs):")
    for (kind, name), v in results.items():
        print(f"  {kind:9s} {name}: {statistics.median(v):.4g}  (min {min(v):.4g}, max {max(v):.4g})")


if __name__ == "__main__":
    main()
