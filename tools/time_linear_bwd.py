"""Kernel-level timing of the node-linear backward at the engine's cfg2 shapes (N = 51,200, H = 64):
the fused pert_linear_bwd_planes against the two-kernel path (pert_gemm_tn with the bias column sums, then
pert_gemm_nt for dX).

Protocol: trains of back-to-back launches over operand sets rotated so that the bytes touched exceed L2, with CUDA
events around each train; the median train gives us per launch.  Bytes and FLOPs are the algorithm's, computed from
the shapes: read dY (4 N H), read X (N K), write dX (N Kd), all fp32; 2 N 4H (K + Kd) multiply-adds, x3 for 3xTF32.

    python tools/time_linear_bwd.py [--trains 9] [--per-train 12]
"""
import argparse

import torch

from measure import HBM_BYTES_PER_S, TF32_FLOP_PER_S, card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=51200)
    ap.add_argument("--trains", type=int, default=9)
    ap.add_argument("--per-train", type=int, default=12)
    a = ap.parse_args()
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    N, H = a.N, 64
    st = torch.cuda.current_stream().cuda_stream
    print(f"card: {card()}")
    for name, K, Kd in (("layer 0", 80, 64), ("layer 1", 64, 64)):
        per_set = (4 * N * H + N * K + N * Kd) * 4
        nsets = max(2, -(-3 * 50 * 2 ** 20 // per_set))
        sets = []
        for s in range(nsets):
            sets.append(dict(dY=torch.randn(4, N, H, device="cuda"), X=torch.randn(N, K, device="cuda"),
                             dX=torch.empty(N, K, device="cuda")))
        W4t = torch.randn(K, 4 * H, device="cuda") / K ** 0.5
        dW4 = torch.zeros(4 * H, K, device="cuda")
        db4 = torch.zeros(4 * H, device="cuda")

        def fused(o):
            return L.pert_linear_bwd_planes(o["dY"].data_ptr(), N * H, o["X"].data_ptr(), K, W4t.data_ptr(), 4 * H,
                                            dW4.data_ptr(), K, db4.data_ptr(), o["dX"].data_ptr(), K, N, H, K, Kd, st)

        def pair(o):
            rc = L.pert_gemm_tn(o["dY"].data_ptr(), H, H, N * H, o["X"].data_ptr(), K, 0, 0, dW4.data_ptr(), K,
                                db4.data_ptr(), N, 4 * H, K, st)
            return rc or L.pert_gemm_nt(o["dY"].data_ptr(), H, H, N * H, W4t.data_ptr(), 4 * H, None,
                                        o["dX"].data_ptr(), K, 0, 0, N, Kd, 4 * H, 0, 0, st)

        byts = (4 * N * H + N * K + N * Kd) * 4
        flops = 3 * 2 * N * 4 * H * (K + Kd)
        floor = max(byts / HBM_BYTES_PER_S, flops / TF32_FLOP_PER_S)
        bound = "HBM" if byts / HBM_BYTES_PER_S >= flops / TF32_FLOP_PER_S else "TF32"
        print(f"{name}: N={N} H={H} K={K} Kd={Kd}  bytes {byts / 1e6:.1f} MB  3xTF32 work {flops / 1e9:.2f} GFLOP  "
              f"floor {floor * 1e6:.1f} us ({bound}-bound at the data-sheet peaks)")
        for label, fn in (("fused", fused), ("pair", pair)):
            for o in sets:                      # warm-up: module load, attribute set-up
                _lib.check(fn(o), label)
            times = sorted(timed(fn, a.per_train, rotate=sets)[1] * 1e3 for _ in range(a.trains))
            us = times[len(times) // 2]
            print(f"  {label:5s}: {us:7.1f} us/launch (trains: min {times[0]:.1f}, max {times[-1]:.1f})  "
                  f"{byts / us / 1e3:7.1f} GB/s  {100 * byts / us / 1e-6 / HBM_BYTES_PER_S:5.1f} % of HBM peak  "
                  f"{100 * flops / us / 1e-6 / TF32_FLOP_PER_S:5.1f} % of TF32 peak  "
                  f"({100 * floor / (us * 1e-6):.1f} % of the {bound} floor)")


if __name__ == "__main__":
    main()
