"""Kernel-level timing of the node-linear forward at the engine's cfg2 shapes (N = 51,200, H = 64): the fused
pert_bn_linear_fwd_planes against the two-launch path (pert_bn_fwd for x[l], then pert_gemm_nt for the planes).

  BN mode, K = 64 (convs >= 1): A = relu(bn(out[l-1])) is computed while A is loaded and also written to x[l].  Both arms
    use the running statistics (eval mode): the ABI's pert_bn_fwd has no entry for the conv epilogue's ready-made batch
    sums, and in eval both arms do the same per-element work, after one tiny k_bn_eval_stats launch each.
  plain mode, K = 80 (conv 0): A = x[0] as it is; the pair is pert_gemm_nt alone.

Protocol: trains of back-to-back launches over operand sets rotated so that the bytes touched exceed L2, with CUDA
events around each train; the median train gives us per launch.  Bytes are the algorithm's, computed from the shapes
(all fp32): BN mode reads 4NH and writes 4NH (x[l]) + 16NH (planes) = 78.6 MB; plain mode reads 4NK and writes 16NH =
68.8 MB.

    python tools/time_linear_fwd.py [--trains 9] [--per-train 12]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12        # H100 SXM data sheet, B/s


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + " (power limit not readable)"


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
    gamma, beta = 1 + 0.1 * torch.randn(H, device="cuda"), 0.1 * torch.randn(H, device="cuda")
    rm, rv = 0.1 * torch.randn(H, device="cuda"), 1 + torch.rand(H, device="cuda")
    mean, rstd = torch.empty(H, device="cuda"), torch.empty(H, device="cuda")
    for name, K, bn in (("BN mode (conv l >= 1)", 64, True), ("plain mode (conv 0)", 80, False)):
        byts = (N * H + N * H + 4 * N * H) * 4 if bn else (N * K + 4 * N * H) * 4
        nsets = max(2, -(-3 * 50 * 2 ** 20 // byts))
        sets = [dict(A=torch.randn(N, K, device="cuda"), x=torch.empty(N, H, device="cuda"),
                     P=torch.empty(4, N, H, device="cuda")) for _ in range(nsets)]
        W4 = torch.randn(4 * H, K, device="cuda") / K ** 0.5
        b4 = torch.randn(4 * H, device="cuda")

        def fused(o):
            if bn:
                return L.pert_bn_linear_fwd_planes(
                    o["A"].data_ptr(), K, 1, gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), None,
                    1e-5, 0.1, 0, mean.data_ptr(), rstd.data_ptr(), o["x"].data_ptr(), H, None, 0, 0, 0.0, None, 0,
                    W4.data_ptr(), K, b4.data_ptr(), o["P"].data_ptr(), N * H, N, H, K, st)
            return L.pert_bn_linear_fwd_planes(o["A"].data_ptr(), K, 0, None, None, None, None, None, 0.0, 0.0, 0,
                                               None, None, None, 0, None, 0, 0, 0.0, None, 0, W4.data_ptr(), K,
                                               b4.data_ptr(), o["P"].data_ptr(), N * H, N, H, K, st)

        def pair(o):
            src = o["A"]
            if bn:
                rc = L.pert_bn_fwd(o["A"].data_ptr(), H, gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(),
                                   rv.data_ptr(), None, 1e-5, 0.1, 0, 1, mean.data_ptr(), rstd.data_ptr(),
                                   o["x"].data_ptr(), H, N, H, None, 0, st)
                if rc:
                    return rc
                src = o["x"]
            return L.pert_gemm_nt(src.data_ptr(), K, 0, 0, W4.data_ptr(), K, b4.data_ptr(), o["P"].data_ptr(), H, H,
                                  N * H, N, 4 * H, K, 0, 0, st)

        print(f"{name}: N={N} H={H} K={K}  algorithmic bytes {byts / 1e6:.1f} MB  "
              f"HBM floor {byts / HBM_PEAK * 1e6:.1f} us at the data-sheet {HBM_PEAK / 1e12:.2f} TB/s")
        for label, fn in (("fused", fused), ("pair", pair)):
            for o in sets:                      # warm-up: module load, attribute set-up
                _lib.check(fn(o), label)
            torch.cuda.synchronize()
            times = []
            for _ in range(a.trains):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(a.per_train):
                    fn(sets[i % nsets])
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / a.per_train)
            times.sort()
            us = times[len(times) // 2]
            print(f"  {label:5s}: {us:7.1f} us/launch (trains: min {times[0]:.1f}, max {times[-1]:.1f})  "
                  f"{byts / us / 1e6:6.2f} TB/s  {100 * byts / us / 1e-6 / HBM_PEAK:5.1f} % of the data-sheet HBM "
                  f"bandwidth")


if __name__ == "__main__":
    main()
