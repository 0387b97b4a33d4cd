"""What a hidden width costs: train.GraphedTrainStep on one resident cfg2 batch (256 graphs of 200 nodes / 600 edges,
3 convs, as bench.py's flagship) at each --widths value.  A width the attention kernels lack runs at the next kernel
width Hp (include/pertgnn.h, pert_model_width) and is expected to cost about what Hp costs.

The widths run alternately, --runs rounds; each run is a window of at least --min-seconds of replayed steps bracketed
by a device synchronise and CUDA events, after a warm-up that captured the graph.  Prints the card name and power
limit, one JSON line per run and a summary line per width (median ms per step and DAGs/s).

    python tools/time_widths.py [--widths 32 48 64 100 128 200 256] [--runs 3] [--min-seconds 1.0]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + " (power limit not readable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", type=int, nargs="+", default=[32, 48, 64, 100, 128, 200, 256])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import make_data_list, model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    print(f"card: {card()}", flush=True)
    data = Batch.from_data_list(make_data_list(2)).to("cuda")
    B = data.num_graphs
    arms = {}
    for H in a.widths:
        args = list(model_args(2))
        args[5] = H
        torch.manual_seed(0)
        model = SAGEDeterministic(*args).cuda()
        model.train()
        step = GraphedTrainStep(model, FusedAdam(FlatParams(model), lr=1e-4), 0.5)
        for _ in range(5):                                # eager, capture, replays
            step(data)
        torch.cuda.synchronize()
        assert step.replays >= 3 and step.capture_error is None, step.capture_error
        arms[H] = (step, [])

    def window(step):
        n, ms = 0, 0.0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        while ms < 1e3 * a.min_seconds:
            torch.cuda.synchronize()
            e0.record()
            for _ in range(20):
                step(data)
            e1.record()
            torch.cuda.synchronize()
            ms += e0.elapsed_time(e1)
            n += 20
        return ms / n

    for r in range(a.runs):
        for H, (step, res) in arms.items():
            ms = window(step)
            res.append(ms)
            print(json.dumps({"H": H, "Hp": _lib.lib().pert_model_width(H), "run": r, "ms_per_step": round(ms, 4),
                              "dags_per_s": round(B / ms * 1e3, 1)}), flush=True)
    for H, (step, res) in arms.items():
        ms = statistics.median(res)
        print(json.dumps({"summary": True, "H": H, "Hp": _lib.lib().pert_model_width(H),
                          "median_ms_per_step": round(ms, 4), "dags_per_s": round(B / ms * 1e3, 1),
                          "spread_ms": round(max(res) - min(res), 4)}), flush=True)


if __name__ == "__main__":
    main()
