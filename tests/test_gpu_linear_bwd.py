"""-m gpu tests of the fused node-linear backward (pert_linear_bwd_planes, csrc/linear_bwd.cu) against float64:
dX = dY . W4[:, :Kd] (written, columns >= Kd untouched), dW4 += dY^T . X, db4 += colsum(dY), with the bars of
test_gpu_fullsize._planes_case; dX bit-identical across runs; and one cfg2 engine step against the two-kernel path."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from tests.helpers import assert_close, is_structural_zero_grad

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 64
SENTINEL = 12345.0


def _run(dY, X, W4, dW4, db4, dX, Kd):
    from pert_gnn_kdd23_b200 import _lib

    N, K = X.shape
    W4t = W4.t().contiguous()
    _lib.call("pert_linear_bwd_planes", dY.data_ptr(), N * H, X.data_ptr(), K, W4t.data_ptr(), 4 * H, dW4.data_ptr(),
              K, db4.data_ptr(), dX.data_ptr(), K, N, H, K, Kd, torch.cuda.current_stream().cuda_stream)


def _case(N, K, Kd, seed, stress=False):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_linear_bwd_planes_supported(N, H, K, Kd) == 1
    g = torch.Generator().manual_seed(seed)
    dY = torch.randn(4, N, H, generator=g)
    X = torch.randn(N, K, generator=g)
    W4 = torch.randn(4 * H, K, generator=g) / math.sqrt(K)
    if stress:
        dY[1, :, 5] *= 1e4                       # one dominant column
        r = torch.randn(N, generator=g)
        dY[3, :, 10], dY[3, :, 11] = 1e3 * r, -1e3 * r   # a pair whose dX contributions cancel exactly
        W4[3 * H + 11] = W4[3 * H + 10]
    dW0 = torch.randn(4 * H, K, generator=g)     # += into non-zero gradients
    db0 = torch.randn(4 * H, generator=g)
    dYc, Xc, Wc = dY.cuda(), X.cuda(), W4.cuda()
    dW4, db4 = dW0.cuda(), db0.cuda()
    dX = torch.full((N, K), SENTINEL, device="cuda")
    _run(dYc, Xc, Wc, dW4, db4, dX, Kd)
    dX2 = torch.full((N, K), SENTINEL, device="cuda")
    _run(dYc, Xc, Wc, torch.zeros_like(dW4), torch.zeros_like(db4), dX2, Kd)
    torch.cuda.synchronize()

    Yd = dY.double().permute(1, 0, 2).reshape(N, 4 * H)
    rX = Yd @ W4.double()[:, :Kd]
    rW = Yd.t() @ X.double()
    rb = Yd.sum(0)
    tag = f"N={N} K={K} Kd={Kd}{' stress' if stress else ''}"
    for got, want, what, tol in ((dX[:, :Kd], rX, "dX", 4e-6), (dW4.cpu().double() - dW0.double(), rW, "dW4", 3e-5),
                                 (db4.cpu().double() - db0.double(), rb, "db4", 2e-5)):
        assert_close(got, want, rtol=tol, what=f"{what} {tag}", norm_only=True)
        assert_close(got, want, rtol=5 * tol, what=f"{what} {tag} (element-wise)")
    if Kd < K:
        assert bool((dX[:, Kd:] == SENTINEL).all()), f"dX columns >= Kd overwritten ({tag})"
    assert torch.equal(dX, dX2), f"dX differs between two runs ({tag})"


@pytest.mark.parametrize("N,K,Kd", [(4096, 64, 64), (4096 + 13, 80, 64), (4096 + 13, 80, 80), (51200, 64, 64),
                                    (51200, 80, 64), (51277, 80, 80), (51277, 64, 64), (102400, 64, 64),
                                    (102400, 80, 64)])
def test_linear_bwd_planes_vs_fp64(N, K, Kd):
    """Full and partial last tiles; N = 4096 leaves fewer tiles than twice the clusters of an H100."""
    _case(N, K, Kd, seed=N + K + Kd)


@pytest.mark.parametrize("K,Kd", [(64, 64), (80, 64)])
def test_linear_bwd_planes_large_and_cancelling_columns(K, Kd):
    _case(51277, K, Kd, seed=K, stress=True)


_STEP = r"""
import json, sys, torch
sys.path.insert(0, {root!r})
from tests.helpers import forward_args, make_batch, make_models
from oracle.model_oracle import torch_quantile_loss
_, model = make_models(2, seed=0)
b = make_batch(2).to("cuda:0")
g, l = model(*forward_args(b))
torch_quantile_loss(b.y.float(), g.flatten(), 0.5).backward()
torch.cuda.synchronize()
torch.save({{n: p.grad.cpu() for n, p in model.named_parameters() if p.grad is not None}}, {out!r})
"""


def test_engine_step_fused_matches_two_kernel_path(tmp_path):
    """One cfg2 training step: every gradient of the fused path against PERT_LINEAR_BWD_FUSED=0 (child processes:
    the switch is read once per process)."""
    grads = {}
    for flag in ("1", "0"):
        out = str(tmp_path / f"grads{flag}.pt")
        env = dict(os.environ, PERT_LINEAR_BWD_FUSED=flag)
        subprocess.run([sys.executable, "-c", _STEP.format(root=ROOT, out=out)], env=env, cwd=ROOT, check=True)
        grads[flag] = torch.load(out)
    assert grads["1"].keys() == grads["0"].keys() and len(grads["1"]) > 10
    n_convs = 1 + max(int(n.split(".")[1]) for n in grads["1"] if n.startswith("convs."))
    bad = {}
    for n, a in grads["1"].items():
        b = grads["0"][n].double()
        e = float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))
        if e > 1e-5 and not is_structural_zero_grad(n, n_convs):
            bad[n] = e
    assert not bad, json.dumps(bad)
