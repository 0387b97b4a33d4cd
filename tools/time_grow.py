"""Cost of growing a trained model's embedding tables (train.grow_embeddings) and what it does to the train step.

Model: the cfg2 model (SAGEDeterministic(*model_args(2)), H = 64, 3 convs) with FusedAdam, trained by
train.GraphedTrainStep on two resident cfg2 batches (256 graphs each), alternated.  Per repetition, on a fresh model:
  * steady before: --steps graph-replayed steps after --warmup, CUDA events around the window, per step;
  * grow: grow_embeddings doubling the entry, interface and rpctype tables and the microservice table, host clock
    around the call and a device synchronise (new rows drawn, one pert_flat_grow launch over params, m and v);
  * first step after growth: the step whose graph was captured over the old engine: the new engine is built, the
    graph captured again and replayed (host clock to a synchronise); then the second key's first step the same way;
  * steady after: as before, on the grown model;
  * steady built at the grown sizes: as before, on a fresh model constructed with the grown tables (the step a grown
    model should match: the row counts select kernel paths, e.g. the conv kernels' shared-memory rpctype table for
    n_rpc <= 8, and the doubled rpctype table here leaves it).
A second arm grows a cfg2 model whose interface table has 2^20 rows (256 MB of parameters, 768 MB with m and v) by
64 entry rows, so that the whole large table moves: the time of grow_embeddings only.
Prints the card name and power limit, then one JSON line: median and [min, max] over the repetitions, in ms.

    python tools/time_grow.py [--reps 5] [--steps 50] [--warmup 10]
"""
import argparse
import json
import statistics
import sys

import torch

from measure import card, host_ms, timed


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_grow.py needs a GPU")
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import make_data_list, model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep, grow_embeddings

    print("card:", card(), flush=True)
    batches = [Batch.from_data_list(make_data_list(2, seed=s)).to("cuda") for s in (11, 12)]
    out = {k: [] for k in ("steady_before", "grow", "first_step_after", "second_key_first_step", "steady_after",
                           "steady_built_at_grown_sizes", "grow_1M_interface")}
    for rep in range(args.reps):
        torch.manual_seed(rep)
        model = SAGEDeterministic(*model_args(2)).cuda()
        opt = FusedAdam(FlatParams(model), lr=1e-3)
        step = GraphedTrainStep(model, opt)
        timed(step, args.warmup, rotate=batches)
        out["steady_before"].append(timed(step, args.steps, rotate=batches)[1])
        rows = {"cat": 2 * model.cat_embedding[0].num_embeddings, "entry": 2 * model.entry_embeds.num_embeddings,
                "interface": 2 * model.interface_embeds.num_embeddings,
                "rpctype": 2 * model.rpctype_embeds.num_embeddings}
        _, ms = host_ms(lambda: grow_embeddings(model, opt, seed=rep, **rows))
        out["grow"].append(ms)
        inv = step.invalidations
        out["first_step_after"].append(host_ms(lambda: step(batches[0]))[1])
        out["second_key_first_step"].append(host_ms(lambda: step(batches[1]))[1])
        assert step.invalidations == inv + 2 and step.capture_error is None
        timed(step, args.warmup, rotate=batches)
        out["steady_after"].append(timed(step, args.steps, rotate=batches)[1])
        del step, opt, model
        a = list(model_args(2))
        a[1], a[2], a[3], a[4] = [rows["cat"]], rows["entry"] - 1, rows["interface"] - 1, rows["rpctype"] - 1
        torch.manual_seed(rep)
        built = SAGEDeterministic(*a).cuda()
        step = GraphedTrainStep(built, FusedAdam(FlatParams(built), lr=1e-3))
        timed(step, args.warmup, rotate=batches)
        out["steady_built_at_grown_sizes"].append(timed(step, args.steps, rotate=batches)[1])
        del step, built

        a = list(model_args(2))
        a[3] = (1 << 20) - 1
        torch.manual_seed(rep)
        big = SAGEDeterministic(*a).cuda()
        bopt = FusedAdam(FlatParams(big), lr=1e-3)
        bstep = GraphedTrainStep(big, bopt)
        timed(bstep, 3, rotate=batches)
        n = big.entry_embeds.num_embeddings + 64
        out["grow_1M_interface"].append(host_ms(lambda: grow_embeddings(big, bopt, entry=n, seed=rep))[1])
        del bstep, bopt, big
        torch.cuda.empty_cache()
    res = {k: stats(v) for k, v in out.items()}
    res.update(card=card(), reps=args.reps, steps=args.steps, unit="ms")
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
