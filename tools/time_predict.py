"""Serving throughput: requests/s of train.predict against the eager loop over the same request list.

Input: PERT-exact artefacts (synthetic.make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096), the
data of bench.py's `pert_pipeline`) in a resident PatternStore; --requests requests (default 10^6) of random entries at
random times from before the first resource bucket to after the last one; an H = 64, 3-conv model (model_args(2)),
trained a few steps so that its BatchNorm running statistics are not the initial ones.
Arms, at each --batch-sizes value and with the exact and the as-of resource join:
  * eager:   PatternStore.assemble_requests + model(*model_inputs(batch)) per slice of the list, eval mode;
  * predict: train.predict (the same slices padded to capacity buckets, one CUDA graph per bucket, one copy each).
The two arms run alternately, --runs times each; every run covers the whole request list, bracketed by a device
synchronise and CUDA events, after one warm-up pass per arm that visited (and, for predict, captured) the buckets.
Prints the card name and power limit, one JSON line per run, and a summary per (batch size, join) with the largest
element-wise difference between the two arms' predictions.

    python tools/time_predict.py [--requests 1000000] [--batch-sizes 1024 4096] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
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
    ap.add_argument("--requests", type=int, default=1_000_000)
    ap.add_argument("--batch-sizes", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step, model_inputs, predict

    print(f"card: {card()}", flush=True)
    dev = "cuda"
    art, _ = make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, device=dev)
    store = PatternStore.from_artifacts(art, dev)
    torch.manual_seed(0)
    model = SAGEDeterministic(*model_args(2)).to(dev)
    opt = FusedAdam(FlatParams(model), lr=3e-4)
    for i, d in enumerate(StoreLoader(store, list(range(len(store))), 256)):
        if i >= 8:
            break
        fused_train_step(model, opt, d, 0.5)
    model.eval()
    rng = np.random.default_rng(0)
    ent = rng.choice(np.flatnonzero(store._h_ent_pats > 0), a.requests)
    ts = rng.integers(-60000, 8 * 60000, a.requests)          # resource rows: 60000 .. 300000
    Q = a.requests

    for bs in a.batch_sizes:
        for asof in (False, True):
            out = {}

            def eager():
                ent_d, ts_d = torch.from_numpy(ent).to(dev), torch.from_numpy(ts).to(dev)
                res = torch.empty(Q, dtype=torch.float32, device=dev)
                with torch.no_grad():
                    for i in range(0, Q, bs):
                        d = store.assemble_requests(ent[i:i + bs], None, asof=asof,
                                                    device_arrays=(ent_d[i:i + bs], ts_d[i:i + bs]))
                        g, _ = model(*model_inputs(d))
                        res[i:i + bs].copy_(g.reshape(-1))
                return res

            def graphed():
                return predict(model, store, ent, ts, batch_size=bs, asof=asof)

            arms = {"eager": eager, "predict": graphed}
            for k, fn in arms.items():                    # warm-up: every bucket visited, captured and replayed
                out[k] = fn()
                if k == "predict":
                    fn()
            torch.cuda.synchronize()
            res = {k: [] for k in arms}
            for r in range(a.runs):
                for k, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    out[k] = fn()
                    e1.record()
                    torch.cuda.synchronize()
                    secs = e0.elapsed_time(e1) / 1e3
                    res[k].append(Q / secs)
                    print(json.dumps({"batch_size": bs, "join": "asof" if asof else "exact", "arm": k, "run": r,
                                      "seconds": round(secs, 3), "requests_per_s": round(Q / secs, 1)}), flush=True)
            g, e = out["predict"].double(), out["eager"].double()
            rms = e.pow(2).mean().sqrt()
            st = model.__dict__["_bucketed_predict"]
            print(json.dumps({"summary": True, "batch_size": bs, "join": "asof" if asof else "exact",
                              **{f"{k}_requests_per_s_best": round(max(v), 1) for k, v in res.items()},
                              **{f"{k}_requests_per_s_min": round(min(v), 1) for k, v in res.items()},
                              "speedup_best": round(max(res["predict"]) / max(res["eager"]), 3),
                              "max_elem_diff": float(((g - e).abs() / (e.abs() + rms)).max()),
                              "buckets": len(st.buckets), "captures": st.captures,
                              "capture_error": st.capture_error}), flush=True)


if __name__ == "__main__":
    main()
