"""Per-bucket CUDA-graph replay on real, variable-size batches: the train step and the eval loop over a shuffled
pattern store, eager against bucketed.

Input: PERT-exact artefacts (synthetic.make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096), the
data of bench.py's `pert_pipeline`) in a resident PatternStore, batches assembled on the device by a shuffled
StoreLoader -- every batch has its own (N, E, B) and its own buffers, so train.GraphedTrainStep never replays there.
Arms, at each --batch-sizes value (170 = the reference default, 256 = bench.py's):
  * train: eager fused_train_step against BucketedTrainStep (padded to capacity buckets, one graph per bucket);
  * eval:  evaluate against evaluate_bucketed over 40 % of the traces (the reference's test split).
The two arms of a pair run alternately, --runs times each; every run is a window of whole epochs of at least
--min-seconds, bracketed by a device synchronise and CUDA events, after a warm-up that visited (and captured) the
buckets.  Prints the card name and power limit, one JSON line per run and a summary per pair (ms per step, DAGs/s,
pad_ratio, captures and replays).

    python tools/time_bucketed_step.py [--batch-sizes 170 256] [--runs 3] [--min-seconds 0.6] [--warmup-epochs 4]
"""
import argparse
import json
import os
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
    ap.add_argument("--batch-sizes", type=int, nargs="+", default=[170, 256])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=0.6)
    ap.add_argument("--warmup-epochs", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, FlatParams, FusedAdam, evaluate, evaluate_bucketed,
                                           fused_train_step)

    print(f"card: {card()}", flush=True)
    dev = "cuda"
    art, _ = make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, device=dev)
    store = PatternStore.from_artifacts(art, dev)
    ids = list(range(len(store)))
    eval_ids = ids[:int(0.4 * len(ids))]

    def new_model():
        torch.manual_seed(0)
        m = SAGEDeterministic(*model_args(2)).to(dev).train()
        return m, FusedAdam(FlatParams(m), lr=3e-4)

    for bs in a.batch_sizes:
        gen = torch.Generator().manual_seed(bs)
        loader = StoreLoader(store, ids, bs, shuffle=True, generator=gen)
        eval_loader = StoreLoader(store, eval_ids, bs)
        m_e, o_e = new_model()
        m_b, o_b = new_model()
        bucketed = BucketedTrainStep(m_b, o_b, 0.5)
        bucketed.reserve(*loader.max_sizes())

        def train_eager(epochs):
            n = g = 0
            for _ in range(epochs):
                for d in loader:
                    fused_train_step(m_e, o_e, d, 0.5)
                    n, g = n + 1, g + d.num_graphs
            return n, g

        def train_bucketed(epochs):
            n = g = 0
            for _ in range(epochs):
                for d in loader:
                    bucketed(d)
                    n, g = n + 1, g + d.num_graphs
            return n, g

        def eval_eager(epochs):
            for _ in range(epochs):
                evaluate(m_e, eval_loader, dev)
            return epochs * len(eval_loader), epochs * len(eval_ids)

        def eval_bucketed(epochs):
            for _ in range(epochs):
                evaluate_bucketed(m_b, eval_loader, dev)
            return epochs * len(eval_loader), epochs * len(eval_ids)

        def window(fn, epochs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            steps, dags = fn(epochs)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / 1e3, steps, dags

        for title, arms in (("train", {"eager": train_eager, "bucketed": train_bucketed}),
                            ("eval", {"eager": eval_eager, "bucketed": eval_bucketed})):
            epochs = {}
            for k, fn in arms.items():                        # warm-up: every bucket eager, captured, replayed
                fn(a.warmup_epochs)
                secs, _, _ = window(fn, 1)                    # epochs per window: at least --min-seconds
                epochs[k] = max(1, int(a.min_seconds / max(secs, 1e-6)) + 1)
            c0, r0 = bucketed.captures, bucketed.replays
            res = {k: [] for k in arms}
            for r in range(a.runs):
                for k, fn in arms.items():
                    secs, steps, dags = window(fn, epochs[k])
                    ms = secs * 1e3 / steps
                    res[k].append((ms, dags / secs))
                    print(json.dumps({"batch_size": bs, "what": title, "arm": k, "run": r, "seconds": round(secs, 3),
                                      "steps": steps, "ms_per_step": round(ms, 4),
                                      "dags_per_s": round(dags / secs, 1)}), flush=True)
            summ = {k: {"ms_per_step_min": round(min(x[0] for x in v), 4),
                        "ms_per_step_max": round(max(x[0] for x in v), 4),
                        "dags_per_s_best": round(max(x[1] for x in v), 1)} for k, v in res.items()}
            extra = {}
            if title == "train":
                extra = {"pad_ratio": round(bucketed.pad_ratio, 4), "captures_total": bucketed.captures,
                         "captures_in_timed_runs": bucketed.captures - c0,
                         "replays_in_timed_runs": bucketed.replays - r0, "invalidations": bucketed.invalidations,
                         "capture_error": bucketed.capture_error}
            else:
                st = m_b.__dict__["_bucketed_eval"]
                extra = {"eval_buckets": len(st.buckets),
                         "eval_graphs": sum(e["state"] == "graph" for e in st.buckets.values()),
                         "eval_capture_error": st.capture_error}
            print(json.dumps({"summary": title, "batch_size": bs, **summ, **extra}), flush=True)


if __name__ == "__main__":
    main()
