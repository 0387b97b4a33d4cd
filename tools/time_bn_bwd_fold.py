"""Kernel-level timing of the BatchNorm backward between two convs at the engine's cfg2 shape (N = 51,200, H = 64, the
cfg2 batch's graphs): the separate pass pert_bn_bwd (reduce + apply over dx, y, x), and the two kernels it is folded
into -- the fused node-linear backward (pert_linear_bwd_planes against pert_linear_bwd_planes_ex with the column sums)
and the conv backward (pert_tconv_bwd_c against pert_tconv_bwd_bn, whose target pass forms g) -- alone and as the
sequence the engine runs for one BatchNorm layer: linear, BatchNorm, conv against linear_ex, conv_bn.

Protocol: trains of back-to-back launches with CUDA events around each train, over two operand sets so that
consecutive launches do not find each other's planes in L2; the median train gives us per launch.

    python tools/time_bn_bwd_fold.py [--trains 9] [--per-train 10]
"""
import argparse
import ctypes
import math

import torch

from measure import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trains", type=int, default=9)
    ap.add_argument("--per-train", type=int, default=10)
    a = ap.parse_args()
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.index import build_index
    from pert_gnn_kdd23_b200.synthetic import N_IF, N_RPC
    from tests.helpers import make_batch

    L, ptr = _lib.lib(), _lib.ptr
    st = torch.cuda.current_stream().cuda_stream
    b = make_batch(2)
    N, B, H = b.x.size(0), b.num_graphs, 64
    gi = build_index(b.edge_index.cuda(), N, b.edge_attr.cuda(), N_IF, N_RPC).check()
    E = gi.E
    print(f"card: {card()}")
    print(f"N={N} E={E} H={H}; one [N, H] fp32 plane = {N * H * 4 / 1e6:.1f} MB")
    rnd = lambda *s: torch.randn(*s, device="cuda")   # noqa: E731
    W4t = (rnd(4 * H, H) / math.sqrt(H)).t().contiguous()
    t_if, t_rpc = rnd(N_IF, H) * 0.1, rnd(N_RPC, H) * 0.1
    mean, rstd, gamma = rnd(H) * 0.1, rnd(H).abs() + 0.5, rnd(H)
    dW4, db4, dgam, dbet = (torch.zeros(4 * H, H, device="cuda"), torch.zeros(4 * H, device="cuda"),
                            torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda"))
    sums32 = torch.zeros(2 * H, device="cuda")
    sets = []
    for _ in range(2):
        o = dict(dY=rnd(4, N, H), y=torch.relu(rnd(N, H)), x=rnd(N, H), dx=torch.empty(N, H, device="cuda"),
                 q=rnd(N, H) * 0.5, k=rnd(N, H) * 0.5, v=rnd(N, H) * 0.5, d=torch.empty(3, N, H, device="cuda"),
                 alpha=torch.empty(E, device="cuda"), dsp=torch.empty(E, device="cuda"),
                 rpc_ws=torch.empty(16 * N, device="cuda"), dt_if=torch.zeros_like(t_if),
                 dt_rpc=torch.zeros_like(t_rpc), sums=torch.zeros(2 * H, dtype=torch.float64, device="cuda"))
        out = torch.empty(N, H, device="cuda")
        _lib.check(L.pert_tconv_fwd(ptr(o["q"]), ptr(o["k"]), ptr(o["v"]), None, H, ptr(gi.rowptr), ptr(gi.csr_src),
                                    ptr(gi.csr_if), ptr(gi.csr_rpc), ptr(t_if), ptr(t_rpc), ptr(out), H,
                                    ptr(o["alpha"]), N_RPC, N, E, B, H, st), "pert_tconv_fwd")
        o["bn"] = _lib.PertBnBwd(ptr(o["dx"]), ptr(o["y"]), ptr(o["x"]), ptr(mean), ptr(rstd), ptr(gamma),
                                 ptr(o["sums"]), ptr(dgam), ptr(dbet), None, 1.0)
        sets.append(o)

    def linear(o):
        return L.pert_linear_bwd_planes(ptr(o["dY"]), N * H, ptr(o["y"]), H, ptr(W4t), 4 * H, ptr(dW4), H, ptr(db4),
                                        ptr(o["dx"]), H, N, H, H, H, st)

    def linear_ex(o):
        return L.pert_linear_bwd_planes_ex(ptr(o["dY"]), N * H, ptr(o["y"]), H, ptr(W4t), 4 * H, ptr(dW4), H,
                                           ptr(db4), ptr(o["dx"]), H, N, H, H, H, ptr(o["x"]), ptr(mean), ptr(rstd),
                                           1.0, None, ptr(o["sums"]), st)

    def bn(o):   # g into the skip plane of dY, as the engine does
        return L.pert_bn_bwd(ptr(o["dx"]), H, ptr(o["y"]), H, ptr(o["x"]), H, ptr(mean), ptr(rstd), ptr(gamma), 1, 1,
                             ptr(o["dY"][3]), H, ptr(dgam), ptr(dbet), ptr(sums32), N, H, st)

    def conv_args(o):
        return (ptr(o["dY"][3]), H, ptr(o["q"]), ptr(o["k"]), ptr(o["v"]), H, ptr(gi.rowptr), ptr(gi.csr_src),
                ptr(gi.csr_if), ptr(gi.csr_rpc), ptr(gi.colptr), ptr(gi.csc_pos), ptr(gi.csc_dst), ptr(t_if),
                ptr(t_rpc), ptr(o["alpha"]), ptr(o["d"][0]), ptr(o["d"][1]), ptr(o["d"][2]), H, ptr(o["dsp"]),
                ptr(o["rpc_ws"]), ptr(o["dt_if"]), ptr(o["dt_rpc"]), N_RPC, N, E, B, H, H)

    def conv(o):
        return L.pert_tconv_bwd_c(*conv_args(o), st)

    def conv_bn(o):
        return L.pert_tconv_bwd_bn(*conv_args(o), ctypes.byref(o["bn"]), st)

    def seq(*fns):
        def run(o):
            for f in fns:
                rc = f(o)
                if rc:
                    return rc
            return 0
        return run

    cases = (("pert_bn_bwd (reduce + apply)", bn), ("node-linear backward", linear),
             ("node-linear backward + BatchNorm sums", linear_ex), ("conv backward", conv),
             ("conv backward + BatchNorm apply", conv_bn), ("unfolded: linear, BatchNorm, conv", seq(linear, bn, conv)),
             ("folded: linear + sums, conv + apply", seq(linear_ex, conv_bn)))
    res = {}
    for label, fn in cases:
        for o in sets:
            _lib.check(fn(o), label)
        times = sorted(timed(fn, a.per_train, rotate=sets)[1] * 1e3 for _ in range(a.trains))
        res[label] = times[len(times) // 2]
        print(f"{label:42s} {res[label]:8.1f} us per launch (median of {a.trains} trains; range "
              f"{times[0]:.1f} .. {times[-1]:.1f})")
    print(f"fold saves {res['unfolded: linear, BatchNorm, conv'] - res['folded: linear + sums, conv + apply']:.1f} us "
          f"per BatchNorm layer; the pass it removes costs {res['pert_bn_bwd (reduce + apply)']:.1f} us alone")


if __name__ == "__main__":
    main()
