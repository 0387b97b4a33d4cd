"""What the conformal calibration costs and what it does to coverage.

Arms:
  * fit: Calibration.fit (pert_calib_offsets) on synthetic (y, yhat, entry id) sets of n in {1e5, 1e6, 1e7} graphs,
    T in {1, 4, 8} levels and three entry mixes (64 uniform entries, 1e4 entries, a Zipf mix where one entry holds
    90 %), against a torch baseline that computes the same offsets by a stable sort of the composite (entry, score)
    key per level and a gather; the two alternated, ms per fit, median and range over --runs.  The algorithmic bytes
    per tier (fit_bytes) and their share of the 3.35 TB/s data-sheet HBM bandwidth are printed beside the fit's time.
  * predict: train.predict of --requests as-of requests with and without calibration=, alternated, requests per s.
  * quality (reported, not asserted): a T = 4 model trained for --epochs epochs on half the traces of the PERT-exact
    store (synthetic.make_pert_artifacts(seed=3), 4096 traces over 64 entries), calibrated on a quarter and evaluated
    on the last quarter: per-level coverage and crossing, raw, calibrated and calibrated with monotone=True.
Every timed window is bracketed by a device synchronise and CUDA events (tools/measure.py) after a warm-up.  Prints the
card name and power limit, one JSON line per measurement and a summary.

    python tools/time_calibration.py [--runs 5] [--requests 1000000] [--epochs 30]
"""
import argparse
import json
import statistics

import numpy as np
import torch

from measure import HBM_BYTES_PER_S, card, timed

LEVELS = {1: (0.95,), 4: (0.5, 0.9, 0.95, 0.99), 8: (0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99, 0.999)}


def make_set(n, T, mix, dev, seed=0):
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
    yhat = y[:, None].float() + 100 * torch.randn(n, T, device=dev, generator=g)
    return y, yhat, e.to(torch.int64), G


def torch_offsets(y, yhat, e, G, levels):
    """The same offsets with torch: per level a stable sort of the (entry, order-preserving score key) composite,
    then a gather of the k-th score of each entry and of the whole set."""
    n, T = yhat.shape
    s = y.float()[:, None] - yhat
    s = torch.where(s == 0, torch.zeros_like(s), s)
    cnt = torch.bincount(e, minlength=G)
    ptr = torch.cumsum(cnt, 0) - cnt
    u = s.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    key = torch.where(u >= 2 ** 31, u ^ 0xFFFFFFFF, u | 2 ** 31)
    out = torch.empty(G + 1, T, device=y.device)
    for t, tau in enumerate(levels):
        order = torch.sort((e << 32) | key[:, t], stable=True).indices
        ss = s[order, t]
        k = torch.ceil((cnt.double() + 1) * tau).clamp(min=1).long()
        kg = max(1, int(np.ceil((n + 1) * tau)))
        glob = torch.kthvalue(s[:, t], kg).values
        mine = (k <= cnt) & (cnt > 0)
        idx = (ptr + torch.minimum(k, cnt.clamp(min=1)) - 1).clamp(0, n - 1)
        out[:G, t] = torch.where(mine, ss[idx], glob)
        out[G, t] = glob
    return out


SMALL = 4096                          # CB_SMALL of csrc/calib.cu: larger segments run the 4-pass tiled select


def fit_bytes(n, T, counts):
    """Bytes the fit must move, per tier: y and yhat read once, the ids twice (count, scatter), the keys written once;
    then each segment's keys (every entry and the global row of all n) read once when it has at most SMALL graphs
    (staged in shared memory) and once per radix pass (4) when it is larger.  Entry counts and outputs are negligible."""
    def reads(m):
        return m * T * 4 * (1 if m <= SMALL else 4)
    return n * 8 + n * T * 4 + 2 * n * 8 + n * T * 4 + reads(n) + sum(reads(int(m)) for m in counts if m > 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--requests", type=int, default=10 ** 6)
    ap.add_argument("--predict-batch", type=int, default=4096)
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--sizes", default="100000,1000000,10000000")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import (BucketedTrainStep, Calibration, FlatParams, FusedAdam, calibrate,
                                           evaluate_bucketed, predict)

    name, power = card(split=True)
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    dev = "cuda"
    results = {}

    def record(key, value, **extra):
        results.setdefault(key, []).append(value)
        print(json.dumps(dict(arm=key[0], case=key[1], ms=value, **extra)), flush=True)

    # ---- fit against the torch baseline
    for n in [int(x) for x in a.sizes.split(",")]:
        for T in (1, 4, 8):
            for mix in ("uniform64", "entries1e4", "zipf90"):
                y, yhat, e, G = make_set(n, T, mix, dev)
                lv = LEVELS[T]
                ours = Calibration.fit(y, yhat, e, lv, G)
                ref = torch_offsets(y, yhat, e, G, lv)
                case = f"n={n} T={T} {mix}"
                b = fit_bytes(n, T, torch.bincount(e, minlength=G).tolist())
                print(json.dumps({"case": case, "equal_to_torch_baseline": bool(torch.equal(ours.offsets, ref))}),
                      flush=True)
                for _ in range(a.runs):
                    _, ms = timed(lambda: Calibration.fit(y, yhat, e, lv, G))
                    record(("fit", case), ms, hbm_share=b / (ms * 1e-3) / HBM_BYTES_PER_S)
                    _, ms = timed(lambda: torch_offsets(y, yhat, e, G, lv))
                    record(("torch", case), ms)
                del y, yhat, e, ours, ref
                torch.cuda.empty_cache()

    # ---- predict with and without the calibration
    art, _ = make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, device=dev)
    store = PatternStore.from_artifacts(art, dev)
    ids = np.random.default_rng(7).permutation(len(store))

    def new_model():
        torch.manual_seed(0)
        m = SAGEDeterministic(*model_args(2), quantiles=LEVELS[4]).to(dev).train()
        return m, FusedAdam(FlatParams(m), lr=3e-4)

    m, opt = new_model()
    step = BucketedTrainStep(m, opt)
    tl = StoreLoader(store, ids[:len(ids) // 2].tolist(), 256, shuffle=True,
                     generator=torch.Generator().manual_seed(3))
    step.reserve(*tl.max_sizes())
    for _ in range(a.epochs):
        for d in tl:
            step(d)
    q = len(ids) // 4
    cal = calibrate(m, StoreLoader(store, ids[len(ids) // 2:len(ids) // 2 + q].tolist(), 256), dev)
    rng = np.random.default_rng(0)
    ok = np.flatnonzero(store._h_ent_pats > 0)
    ts_all = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    ent, ts = rng.choice(ok, a.requests), rng.choice(ts_all, a.requests)
    arms = {"plain": {}, "calibrated": {"calibration": cal}}
    for kw in arms.values():
        predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True, **kw)
    for _ in range(a.runs):
        for arm, kw in arms.items():
            _, ms = timed(lambda: predict(m, store, ent, ts, batch_size=a.predict_batch, asof=True, **kw))
            record(("predict", arm), ms, requests_per_s=a.requests / (ms / 1e3))

    # ---- quality on the last quarter
    ev = StoreLoader(store, ids[len(ids) // 2 + q:].tolist(), 256)
    out = {"levels": LEVELS[4], "epochs": a.epochs, "train_traces": len(ids) // 2, "calibration_traces": q,
           "test_traces": len(ev.dataset), "own_per_level": cal.own[:-1].sum(0).tolist()}
    for arm, kw in (("raw", {}), ("calibrated", {"calibration": cal}),
                    ("calibrated_monotone", {"calibration": cal, "monotone": True})):
        mae, _, _ = evaluate_bucketed(m, ev, dev, **kw)
        met = m.__dict__["_bucketed_eval_calibrated" if kw else "_bucketed_eval"].metrics
        out[arm] = {"coverage": met.coverage(), "crossing": met.crossing(), "mae": mae}
    print(json.dumps({"quality": out}), flush=True)

    print("summary (median over runs, ms):")
    for (arm, case), v in results.items():
        print(f"  {arm:9s} {case:28s}: {statistics.median(v):.4g}  (min {min(v):.4g}, max {max(v):.4g})")


if __name__ == "__main__":
    main()
