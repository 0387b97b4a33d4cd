"""Where the graph-replayed cfg2 train step spends its GPU time between kernels.

Replays train.GraphedTrainStep on bench.py's cfg2 shape (256 DAGs x 200 nodes, H = 64, 3 convs, resident batches)
under torch.profiler (CUDA activity only, in a run of its own), writes the trace, and prints for one step (the one with
the median sum of gaps): every GPU activity in issue order with its duration and the idle gap before it, then the sum
of the gaps and the step's span from its first to its last activity.  A gap is time in which no kernel, memset or copy
of the step runs on the device; the host-side gap between one step's Adam and the next replay is not part of a step.
Prints the card name and power limit first.

    python tools/time_step_gaps.py [--steps 16] [--trace PATH]   (default: step_gaps.pt.trace.json in the temp dir)
"""
import argparse
import json
import os
import statistics
import tempfile

import torch

from measure import card

N_ROT = 8   # distinct resident batches, as bench.py


def make_batches(cfg, count, dev):
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.synthetic import make_data_list

    out = []
    for r in range(count):
        dl = make_data_list(cfg, seed=1000 + cfg + 131 * r)
        for d in dl:
            d._store.pop("level", None)
            d._store.pop("min_depth", None)
        out.append(Batch.from_data_list(dl).to(dev))
    return out


def gpu_activities(trace):
    """Kernels, memsets and copies of the trace, (start us, end us, name), sorted by start."""
    ev = []
    for e in trace.get("traceEvents", []):
        if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy"):
            ev.append((float(e["ts"]), float(e["ts"]) + float(e.get("dur", 0.0)), e["name"]))
    return sorted(ev)


def split_steps(ev):
    """One list per step: the activities up to and including each Adam kernel (k_adam ends every step)."""
    steps, cur = [], []
    for a in ev:
        cur.append(a)
        if a[2].startswith("k_adam") or "k_adam(" in a[2]:
            steps.append(cur)
            cur = []
    return steps


def step_gaps(step):
    """Per activity: (name, duration, idle gap before it); the first activity has no predecessor in the step."""
    rows, end = [], None
    for s, e, n in step:
        gap = 0.0 if end is None else max(0.0, s - end)
        rows.append((n, e - s, gap))
        end = e if end is None else max(end, e)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--trace", default=os.path.join(tempfile.gettempdir(), "step_gaps.pt.trace.json"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from torch.profiler import ProfilerActivity, profile

    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    print(f"card: {card()}", flush=True)
    dev = torch.device("cuda", 0)
    batches = make_batches(2, N_ROT, dev)
    torch.manual_seed(0)
    model = SAGEDeterministic(*model_args(2)).to(dev)
    step = GraphedTrainStep(model, FusedAdam(FlatParams(model), lr=3e-4), 0.5)
    for i in range(3 * N_ROT):                       # every batch captured (second visit) and replayed
        step(batches[i % N_ROT])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            step(batches[i % N_ROT])
        torch.cuda.synchronize()
    os.makedirs(os.path.dirname(a.trace) or ".", exist_ok=True)
    prof.export_chrome_trace(a.trace)
    with open(a.trace) as f:
        steps = split_steps(gpu_activities(json.load(f)))
    steps = [s for s in steps if len(s) > 1][1:]     # the first may start inside the profiler's warm-up
    assert steps, "no complete step in the trace"
    tables = [step_gaps(s) for s in steps]
    sums = [sum(g for _, _, g in t) for t in tables]
    spans = [s[-1][1] - s[0][0] for s in steps]
    med = sorted(range(len(tables)), key=lambda i: sums[i])[len(tables) // 2]
    print(f"{'dur_us':>8} {'gap_us':>8}  activity (step {med} of {len(tables)}, median sum of gaps)")
    for n, d, g in tables[med]:
        print(f"{d:8.2f} {g:8.2f}  {n[:110]}")
    busy = [sum(d for _, d, _ in t) for t in tables]
    print(json.dumps({"card": card(), "steps": len(tables), "activities_per_step": len(tables[med]),
                      "gap_us_per_step_median": statistics.median(sums), "gap_us_per_step_min": min(sums),
                      "gap_us_per_step_max": max(sums), "span_us_median": statistics.median(spans),
                      "busy_us_median": statistics.median(busy), "trace": a.trace}))


if __name__ == "__main__":
    main()
