"""How much of each conv-chain handoff L2 serves: every consumer of the cfg2 chain timed hot, cold and at an L2-sized
batch, next to its time inside the graph-replayed train step.

The chain (H = 64) hands its outputs from kernel to kernel: node-linear forward -> conv forward -> next node-linear
forward; node-linear backward -> conv backward (target + source pass) -> node-linear backward of the conv before.  Each
consumer is driven through its C-ABI entry point (pert_bn_linear_fwd_planes in BatchNorm mode, pert_tconv_fwd_stats,
pert_tconv_bwd_bn, pert_linear_bwd_planes_ex) with the arguments the engine passes, on the cfg2 batch's graph index
and operand buffers of the trained shapes, in three states:
  hot   right after its real producer ran on the same buffers, as in the step;
  cold  after a 512 MB read that flushes L2;
  fits  hot at a quarter-size batch (64 graphs: each handoff fits L2 several times over), scaled by the byte ratio to
        cfg2.  An upper bound on what L2 residency can buy.
CUDA events around each consumer call, median of --reps.  Called on their own the kernels run without the chain's L2
policy (csrc/sm90.cuh: the engine sets it on its chain only), so these three columns measure the kernels under the
default policy.  The `step` column is the consumer's median time inside GraphedTrainStep (a torch.profiler run of its
own; the conv backward is its target plus its source pass), where the chain's policy applies.  Prints the card name and
power limit first, the step's ms and DAGs/s, and one JSON line last.

    python tools/time_l2_handoff.py [--reps 30] [--prof-steps 16]
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import tempfile

import torch

from measure import HBM_BYTES_PER_S, card, timed
from time_step_gaps import N_ROT, gpu_activities, make_batches, split_steps

H = 64
FLUSH_BYTES = 512 << 20


def consumers(n_graphs):
    """[(name, producer, consumer, algorithmic bytes of the consumer)] at one batch size, with its buffers."""
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.index import build_index
    from pert_gnn_kdd23_b200.synthetic import N_IF, N_RPC
    from tests.helpers import make_batch

    L, p = _lib.lib(), _lib.ptr
    st = torch.cuda.current_stream().cuda_stream
    b = make_batch(2, n_graphs)
    N, B = b.x.size(0), b.num_graphs
    gi = build_index(b.edge_index.cuda(), N, b.edge_attr.cuda(), N_IF, N_RPC).check()
    E = gi.E
    g = torch.Generator(device="cuda").manual_seed(n_graphs)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)   # noqa: E731
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device="cuda", dtype=dt)   # noqa: E731
    W4 = rnd(4 * H, H) / math.sqrt(H)
    W4t, b4 = W4.t().contiguous(), rnd(4 * H) * 0.1
    t_if, t_rpc = rnd(N_IF, H) * 0.1, rnd(N_RPC, H) * 0.1
    gamma, beta, rm, rv, nbt = rnd(H).abs() + 0.5, rnd(H) * 0.1, z(H), z(H) + 1, z(1, dt=torch.int64)
    mean, rstd = z(H), z(H)                          # written by the node-linear forward (training)
    bn_ws_bytes = L.pert_bn_workspace_bytes(N, H)
    bn_acc = z(bn_ws_bytes // 8, dt=torch.float64)
    planes, out, xl = rnd(4, N, H) * 0.5, rnd(N, H), torch.relu(rnd(N, H))
    dplanes, dx, alpha, dsp, rpc_ws = rnd(4, N, H), rnd(N, H), z(E), z(E), z(16 * N)
    dW4, db4, dt_if, dt_rpc, dgam, dbet = z(4 * H, H), z(4 * H), z(N_IF, H), z(N_RPC, H), z(H), z(H)
    sums = z(2 * H, dt=torch.float64)
    fused = ctypes.c_int(0)
    bn = _lib.PertBnBwd(p(dx), p(xl), p(out), p(mean), p(rstd), p(gamma), p(sums), p(dgam), p(dbet), None, 1.0)

    def lin_fwd():                                   # A = out[l-1] -> x[l], the four planes (BatchNorm mode)
        return L.pert_bn_linear_fwd_planes(p(out), H, 1, p(gamma), p(beta), p(rm), p(rv), p(nbt), 1e-5, 0.1, 1,
                                           p(mean), p(rstd), p(xl), H, p(bn_acc), bn_ws_bytes, 1, 0.0, None, 0,
                                           p(W4), H, p(b4), p(planes), N * H, N, H, H, st)

    def conv_fwd():                                  # planes -> out[l], alpha, BatchNorm sums (+=)
        return L.pert_tconv_fwd_stats(p(planes[0]), p(planes[1]), p(planes[2]), p(planes[3]), H, p(gi.rowptr),
                                      p(gi.csr_src), p(gi.csr_if), p(gi.csr_rpc), p(t_if), p(t_rpc), p(out), H,
                                      p(alpha), N_RPC, N, E, B, H, H, p(bn_acc), None, ctypes.byref(fused), st)

    def conv_bwd():                                  # dx, y = x[l], x = out[l-1], q k v -> g, dq, dk, dv
        return L.pert_tconv_bwd_bn(p(dplanes[3]), H, p(planes[0]), p(planes[1]), p(planes[2]), H, p(gi.rowptr),
                                   p(gi.csr_src), p(gi.csr_if), p(gi.csr_rpc), p(gi.colptr), p(gi.csc_pos),
                                   p(gi.csc_dst), p(t_if), p(t_rpc), p(alpha), p(dplanes[0]), p(dplanes[1]),
                                   p(dplanes[2]), H, p(dsp), p(rpc_ws), p(dt_if), p(dt_rpc), N_RPC, N, E, B, H, H,
                                   ctypes.byref(bn), st)

    def lin_bwd():                                   # dY = dplanes, X = x[l], bn_x = out[l-1] -> dx, sums (+=)
        return L.pert_linear_bwd_planes_ex(p(dplanes), N * H, p(xl), H, p(W4t), 4 * H, p(dW4), H, p(db4), p(dx), H,
                                           N, H, H, H, p(out), p(mean), p(rstd), 1.0, None, p(sums), st)

    def reset():                                     # the accumulated sums, before each producer (not timed)
        bn_acc.zero_()
        sums.zero_()

    reset()
    for f in (conv_fwd, lin_fwd, lin_bwd, conv_bwd):   # valid statistics and sums first
        _lib.check(f(), f.__name__)
    assert fused.value == 1, "the tile kernel did not take the shape"
    row = 4 * N * H
    idx_csr, idx_csc = 4 * (N + 1) + 12 * E, 4 * (N + 1) + 8 * E + 8 * E
    return N, reset, [
        ("node-linear fwd", "k_bn_linear_fwd_planes", conv_fwd, lin_fwd, row + row + 4 * row),
        ("conv fwd", "k_tile_fwd", lin_fwd, conv_fwd, 4 * row + row + 4 * E + idx_csr),
        # target: dx, y, x, k, v, g, dq, alpha, ds; source: g, q, dk, dv, alpha, ds
        ("conv bwd", "k_tile_bwd", lin_bwd, conv_bwd, 7 * row + 8 * E + idx_csr + 4 * row + 8 * E + idx_csc),
        ("node-linear bwd", "k_linear_bwd_planes", conv_bwd, lin_bwd, 4 * row + row + 2 * row + row),
    ]


def states(reset, cases, reps, flush):
    """{name: (hot ms, cold ms)}: the consumer's median over reps, right after its producer / after its producer and
    an L2 flush."""
    out = {}
    for name, _, prod, cons, _ in cases:
        res = []
        for cold in (False, True):
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
            for e0, e1 in ev:
                reset()
                prod()                               # the consumer's inputs are the producer's, as in the step
                if cold:
                    flush.sum()
                e0.record()
                cons()
                e1.record()
            torch.cuda.synchronize()
            res.append(statistics.median(e0.elapsed_time(e1) for e0, e1 in ev))
        out[name] = tuple(res)
    return out


def in_step(prof_steps):
    """(ms per replayed cfg2 step, DAGs/s, {kernel family: [median us per occurrence in the step]})."""
    from torch.profiler import ProfilerActivity, profile

    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    dev = torch.device("cuda", 0)
    batches = make_batches(2, N_ROT, dev)
    torch.manual_seed(0)
    model = SAGEDeterministic(*model_args(2)).to(dev)
    step = GraphedTrainStep(model, FusedAdam(FlatParams(model), lr=3e-4), 0.5)
    for i in range(3 * N_ROT):                       # every batch captured (second visit) and replayed
        step(batches[i % N_ROT])
    _, ms = timed(lambda b: step(b), 200, rotate=batches)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(prof_steps):
            step(batches[i % N_ROT])
        torch.cuda.synchronize()
    trace = os.path.join(tempfile.gettempdir(), "l2_handoff.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        steps = [s for s in split_steps(gpu_activities(json.load(f))) if len(s) > 1][1:]
    os.remove(trace)
    assert steps, "no complete step in the trace"
    fams = ("k_bn_linear_fwd_planes", "k_tile_fwd", "k_tile_bwd_dst", "k_tile_bwd_src", "k_linear_bwd_planes")
    per = {}
    for s in steps:
        seen = {}
        for t0, t1, name in s:
            fam = next((c for c in fams if c in name), None)
            if fam:
                k = seen.get(fam, 0)
                seen[fam] = k + 1
                per.setdefault(fam, {}).setdefault(k, []).append(t1 - t0)
    med = {f: [statistics.median(v[k]) for k in sorted(v)] for f, v in per.items()}
    med["k_tile_bwd"] = [a + b for a, b in zip(med["k_tile_bwd_dst"], med["k_tile_bwd_src"])]
    return ms, batches[0].num_graphs / ms * 1e3, med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--prof-steps", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(f"card: {card()}", flush=True)
    flush = torch.ones(FLUSH_BYTES // 4, device="cuda")
    N, reset, full = consumers(256)
    hc = states(reset, full, a.reps, flush)
    n_small, reset_s, small = consumers(64)
    fit = states(reset_s, small, a.reps, flush)
    ms, dags, med = in_step(a.prof_steps)
    print(f"step: {ms:.4f} ms  {dags:,.0f} DAGs/s   (cfg2: N = {N}; fits: N = {n_small}, scaled by bytes)")
    print(f"{'consumer':<16} {'MB':>6} {'step us':>16} {'hot us':>8} {'cold us':>8} {'fits us':>8} {'hot TB/s':>9}")
    rows = []
    for (name, fam, _, _, by), (_, _, _, _, by_s) in zip(full, small):
        hot, cold = (t * 1e3 for t in hc[name])
        fits = fit[name][0] * 1e3 * by / by_s
        st = med.get(fam, [])
        # the middle layer: the one whose producer and consumer both sit inside the chain on either side
        mid = st[1] if len(st) == 3 else (st[0] if st else float("nan"))
        rows.append({"consumer": name, "mb": round(by / 1e6, 1), "step_us": [round(x, 1) for x in st],
                     "hot_us": round(hot, 1), "cold_us": round(cold, 1), "fits_us": round(fits, 1)})
        print(f"{name:<16} {by / 1e6:6.1f} {'/'.join(f'{x:.1f}' for x in st):>16} {hot:8.1f} {cold:8.1f} "
              f"{fits:8.1f} {by / (hot * 1e-6) / 1e12:9.2f}   (middle layer in step {mid:.1f}; "
              f"{by / (hot * 1e-6) / HBM_BYTES_PER_S:.0%} of HBM hot)")
    print(json.dumps({"card": card(), "step_ms": round(ms, 4), "dags_per_s": round(dags), "consumers": rows}))


if __name__ == "__main__":
    main()
