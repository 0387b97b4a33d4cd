"""Cost of the between-layer dropout at cfg2 (256 graphs x 200 nodes, H = 64, 3 convs).

Two comparisons, each as alternating runs of the two arms (--runs each), every run timed with CUDA events around
--steps training steps on two resident batches after a warm-up that captured every graph:
  * the fused step replayed from CUDA graphs (train.GraphedTrainStep, what bench.py times) at p = 0 and at p = 0.1;
  * the drop-in loop body (train.train_step with torch.optim.Adam, reference pert_gnn.py:231-247) at p = 0.1 with
    use_engine True (dropout inside the engine) against False (one autograd Function per operator + torch F.dropout).
Prints the card name and power limit, then one JSON line per run and a summary line.

    python tools/time_dropout.py [--steps 50] [--warmup 8] [--runs 3]
"""
import argparse
import json

import torch

from measure import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import make_data_list, model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep, train_step

    print(f"card: {card()}", flush=True)
    batches = [Batch.from_data_list(make_data_list(2, seed=s)).to("cuda") for s in range(2)]
    B = batches[0].num_graphs

    def model_with(p):
        torch.manual_seed(0)
        m = SAGEDeterministic(*model_args(2)).cuda().train()
        m.dropout = p
        m.seed_dropout(1)
        return m

    def graphed(p):
        m = model_with(p)
        opt = FusedAdam(FlatParams(m), lr=3e-4)
        g = GraphedTrainStep(m, opt, 0.5)
        return lambda d: g(d)

    def dropin(use_engine):
        m = model_with(0.1)
        m.use_engine = use_engine
        opt = torch.optim.Adam(m.parameters(), lr=3e-4)
        return lambda d: train_step(m, opt, d, 0.5)

    for title, arms in (("GraphedTrainStep", {"p=0": graphed(0.0), "p=0.1": graphed(0.1)}),
                        ("drop-in train_step p=0.1", {"engine": dropin(True), "operators": dropin(False)})):
        for step in arms.values():
            timed(step, max(a.warmup, 4), rotate=batches)   # every key: eager, capture + replay, replays
        res = {k: [] for k in arms}
        for r in range(a.runs):
            for k, step in arms.items():
                _, ms = timed(step, a.steps, rotate=batches)
                res[k].append(ms)
                print(json.dumps({"what": title, "arm": k, "run": r, "ms_per_step": round(ms, 4),
                                  "dags_per_s": round(B / ms * 1e3, 1)}), flush=True)
        summ = {k: {"ms_min": round(min(v), 4), "ms_max": round(max(v), 4),
                    "dags_per_s_best": round(B / min(v) * 1e3, 1)} for k, v in res.items()}
        print(json.dumps({"summary": title, **summ}), flush=True)


if __name__ == "__main__":
    main()
