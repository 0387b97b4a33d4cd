"""What-if serving throughput: requests/s of train.predict with per-request mixes and resource scenarios against
plain predict, and the time of the assembly alone.

Input: the make_pert_artifacts store of tools/time_predict.py (seed 3, 256 patterns, 64 entries, 4096 traces), an
H = 64 model trained a few steps, --requests requests (default 10^6) of random entries at random times, batch
--batch-size (default 1024), the as-of join.  Arms, run alternately --runs times each after a warm-up pass that
captures every bucket:
  * plain:    predict(ent, ts);
  * own:      predict with every request's own stored mix given as a what-if mix;
  * mixes:    predict with random 2-4-pattern mixes;
  * scenario: predict with 16 scenarios, each overriding 10 % of the microservices, one random scenario per request.
Before timing, the own arm must equal the plain arm (assembly bitwise, predictions bitwise or within the test
tolerance) and the first batch of the mixes and scenario arms must equal the numpy restatement of tests/test_gpu_whatif.
Then the assembly alone: CUDA events around the loop of assemble_requests calls over the whole request list, plain vs
each what-if form with its inputs already checked and uploaded, and apart from it the per-call host preparation (checks,
runtime resolution, uploads, the override sort).  Prints the card name and power limit, one JSON line per run and a
summary with the mean node count per request of every arm.

    python tools/time_what_if.py [--requests 1000000] [--batch-size 1024] [--runs 5]
"""
import argparse
import json

import numpy as np
import torch

from measure import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=1_000_000)
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts, model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step, predict
    from tests.helpers import assert_close
    from tests.test_gpu_whatif import _restate

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
    Q, bs = a.requests, a.batch_size
    ent = rng.choice(np.flatnonzero(store._h_ent_pats > 0), Q)
    ts = rng.integers(-60000, 8 * 60000, Q)
    # own mixes
    e_ptr, e_pat, e_prob = (store.t[k].cpu().numpy() for k in ("ent_ptr", "ent_pat", "ent_prob"))
    lens = e_ptr[ent + 1] - e_ptr[ent]
    sl = np.repeat(e_ptr[ent] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(lens.sum())
    rt_ids = np.asarray(store.rt_ids, dtype=np.int64)
    own = (np.concatenate([[0], np.cumsum(lens)]), rt_ids[e_pat[sl]], e_prob[sl].astype(np.float64))
    # random 2-4-pattern mixes (distinct runtimes per mix)
    k = rng.integers(2, 5, Q)
    n_pat = len(rt_ids)
    first = rng.integers(0, n_pat, Q)
    step = rng.integers(1, n_pat // 4, Q)
    pats = (first[:, None] + step[:, None] * np.arange(4)[None, :]) % n_pat
    keep = np.arange(4)[None, :] < k[:, None]
    mixes = (np.concatenate([[0], np.cumsum(k)]), rt_ids[pats[keep]], rng.random(int(k.sum())))
    # 16 scenarios over 10 % of the microservices each
    n_ov = max(1, store.n_ms // 10)
    ov_s = np.repeat(np.arange(16), n_ov)
    ov_m = np.concatenate([rng.choice(store.n_ms, n_ov, replace=False) for _ in range(16)])
    ov = (ov_s, ov_m, rng.random((ov_s.size, 8)))
    scen = rng.integers(0, 16, Q)
    arms = {"plain": {}, "own": {"mixes": own}, "mixes": {"mixes": mixes},
            "scenario": {"overrides": ov, "scenario_ids": scen}}
    res = (art["resource_index"], art["resource_values"])

    # ---- correctness first
    b_plain = store.assemble_requests(ent[:bs], ts[:bs], asof=True)
    b_own = store.assemble_requests(ent[:bs], ts[:bs], asof=True, mixes=(own[0][:bs + 1], own[1][:own[0][bs]],
                                                                         own[2][:own[0][bs]]))
    keys = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs", "entry_id",
            "rt_probs", "batch", "ptr")
    assert all(torch.equal(b_plain[k2], b_own[k2]) for k2 in keys)
    mix_list = [(mixes[1][mixes[0][q]:mixes[0][q + 1]], mixes[2][mixes[0][q]:mixes[0][q + 1]]) for q in range(bs)]
    own_list = [(own[1][own[0][q]:own[0][q + 1]], own[2][own[0][q]:own[0][q + 1]]) for q in range(bs)]
    for name, kw, ml in (("mixes", arms["mixes"], mix_list), ("scenario", arms["scenario"], own_list)):
        sub = {"mixes": (kw["mixes"][0][:bs + 1], kw["mixes"][1][:kw["mixes"][0][bs]],
                         kw["mixes"][2][:kw["mixes"][0][bs]])} if "mixes" in kw else \
            {"overrides": ov, "scenario_ids": scen[:bs]}
        got = store.assemble_requests(ent[:bs], ts[:bs], asof=True, **sub)
        want, _ = _restate(store, ent[:bs], ts[:bs], ml, True, res, overrides=sub.get("overrides"),
                           scen=sub.get("scenario_ids"))
        for k2 in keys:
            assert np.array_equal(got[k2].cpu().numpy(), want[k2]), (name, k2)
    out = {}
    for name, kw in arms.items():                       # warm-up: every bucket visited, captured and replayed
        for _ in range(2):
            out[name] = predict(model, store, ent, ts, batch_size=bs, asof=True, **kw)
    bitwise = torch.equal(out["own"], out["plain"])
    if not bitwise:
        assert_close(out["own"], out["plain"], what="own mixes vs plain")
    print(json.dumps({"check": "own-mix predict vs plain predict", "bitwise": bitwise}), flush=True)
    st = model.__dict__["_bucketed_predict"]
    c0 = st.captures

    # ---- predict throughput
    rate = {n: [] for n in arms}
    for r in range(a.runs):
        for name, kw in arms.items():
            secs = timed(lambda: predict(model, store, ent, ts, batch_size=bs, asof=True, **kw))[1] / 1e3
            rate[name].append(Q / secs)
            print(json.dumps({"arm": name, "run": r, "seconds": round(secs, 3), "requests_per_s": round(Q / secs, 1)}),
                  flush=True)

    # ---- assembly alone: the loop of assemble_requests calls over the whole list
    def plain_loop():
        ent_d, ts_d = torch.from_numpy(ent).to(dev), torch.from_numpy(ts).to(dev)
        for i in range(0, Q, bs):
            store.assemble_requests(ent[i:i + bs], None, asof=True, device_arrays=(ent_d[i:i + bs], ts_d[i:i + bs]))

    def what_if_loop(w):
        def run():
            for i in range(0, Q, bs):
                store.assemble_requests(None, None, asof=True, device_arrays=w.slice(i, i + bs))
        return run

    # the per-call host checks, runtime resolution and uploads (once per predict call) are timed apart from the loop
    prep = {n: [] for n in arms if n != "plain"}
    prepared = {}
    for r in range(a.runs):
        for n in prep:
            prepared[n], ms = timed(lambda: store._what_if_arrays(ent, ts, **arms[n]))
            prep[n].append(ms / 1e3)
    loops = {"plain": plain_loop, **{n: what_if_loop(w) for n, w in prepared.items()}}
    asm = {n: [] for n in loops}
    for fn in loops.values():
        fn()
    for r in range(a.runs):
        for name, fn in loops.items():
            secs = timed(fn)[1] / 1e3
            asm[name].append(secs)
            print(json.dumps({"assembly": name, "run": r, "seconds": round(secs, 4)}), flush=True)
    nodes = {"plain": float(store._h_ent_nodes[ent].mean()), "own": float(prepared["own"].nodes.mean()),
             "mixes": float(prepared["mixes"].nodes.mean()), "scenario": float(prepared["scenario"].nodes.mean())}
    med = {n: float(np.median(v)) for n, v in rate.items()}
    amed = {n: float(np.median(v)) for n, v in asm.items()}
    print(json.dumps({"summary": True, "requests": Q, "batch_size": bs, "join": "asof",
                      **{f"{n}_requests_per_s_median": round(v, 1) for n, v in med.items()},
                      **{f"{n}_requests_per_s_range": [round(min(v), 1), round(max(v), 1)] for n, v in rate.items()},
                      **{f"{n}_vs_plain": round(med[n] / med["plain"], 3) for n in arms},
                      **{f"assembly_{n}_ms_median": round(1e3 * v, 2) for n, v in amed.items()},
                      **{f"assembly_{n}_vs_plain": round(amed[n] / amed["plain"], 3) for n in loops},
                      **{f"host_prep_{n}_ms_median": round(1e3 * float(np.median(v)), 1) for n, v in prep.items()},
                      **{f"nodes_per_request_{n}": round(v, 1) for n, v in nodes.items()},
                      "own_bitwise": bitwise, "captures_after_warmup": st.captures - c0,
                      "capture_error": st.capture_error}), flush=True)


if __name__ == "__main__":
    main()
