"""-m gpu tests of the node-linear forward with the BatchNorm apply folded in (pert_bn_linear_fwd_planes,
csrc/linear_fwd.cu), called through the C entry:
  * BN mode: x[l] = dropout(relu(bn(A))) bit-identical to pert_bn_fwd on the same inputs (the dropout mask from the
    restatement of tests/dropout_ref.py), and so are mean / rstd, the running statistics and num_batches_tracked;
  * the planes against fp64 of the same A under DESIGN section 3's NT 3xTF32 element-wise bar
    tau * (|A| . |W|^T + |b|);
  * plain mode (conv 0, K = 80): the planes against fp64 under the same bar;
  * rows past N and the memory just after x[l] and the planes untouched; two runs give bit-identical planes."""
import math

import numpy as np
import pytest
import torch

from tests.dropout_ref import dropout_mask, scale_of

pytestmark = pytest.mark.gpu

H = 64
U = 2.0 ** -24
SENTINEL = 12345.0
EPS, MOMENTUM = 1e-5, 0.1
SEED, STEP, LAYER = 0x1234_5678_9ABC, 7, 1


def _tau_nt(K):
    """DESIGN section 3, NT 3xTF32 with one plane: product error + one truncated ulp per wgmma + the bias."""
    return 3 * 2.0 ** -21 + 3 * math.ceil(K / 8) * 2 * U + 2 * U


def _lib():
    from pert_gnn_kdd23_b200 import _lib as L

    return L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bn_state(g):
    return dict(gamma=(1 + 0.3 * torch.randn(H, generator=g)).cuda(), beta=(0.2 * torch.randn(H, generator=g)).cuda(),
                rm=(0.1 * torch.randn(H, generator=g)).cuda(), rv=(1 + torch.rand(H, generator=g)).cuda(),
                nbt=torch.tensor([3], dtype=torch.int64).cuda())


def _copy_state(s):
    return {k: v.clone() for k, v in s.items()}


def _fused(A, W4, b4, N, K, bn=None, training=1, p=0.0, ctr=None):
    """One call; returns (x_buf, planes_buf, pz, stats) with sentinel-filled padding around every output."""
    L = _lib()
    pz = (N + 64) * H                                        # 64 spare rows after every plane
    planes = torch.full((4 * pz + 256,), SENTINEL, device="cuda")
    x_buf = torch.full((N * H + 256,), SENTINEL, device="cuda")
    mean = torch.full((H,), SENTINEL, device="cuda")
    rstd = torch.full((H,), SENTINEL, device="cuda")
    ws_bytes = L.lib().pert_bn_workspace_bytes(N, H)
    ws = torch.zeros(ws_bytes // 8 + 8, dtype=torch.float64, device="cuda")
    if bn is None:
        args = (A.data_ptr(), K, 0, None, None, None, None, None, 0.0, 0.0, 0, None, None, None, 0, None, 0, 0, 0.0,
                None, 0)
    else:
        args = (A.data_ptr(), K, 1, bn["gamma"].data_ptr(), bn["beta"].data_ptr(), bn["rm"].data_ptr(),
                bn["rv"].data_ptr(), bn["nbt"].data_ptr(), EPS, MOMENTUM, training, mean.data_ptr(), rstd.data_ptr(),
                x_buf.data_ptr(), H, ws.data_ptr(), ws_bytes, 0, p, ctr.data_ptr() if ctr is not None else None, LAYER)
    L.call("pert_bn_linear_fwd_planes", *args, W4.data_ptr(), K, b4.data_ptr(), planes.data_ptr(), pz, N, H, K,
           _stream())
    return x_buf, planes, pz, (mean, rstd)


def _reference_bn(A, bn, N, training):
    """pert_bn_fwd (k_bn_partial / k_bn_eval_stats + k_bn_apply) on the same inputs: y, mean, rstd; updates bn."""
    L = _lib()
    y = torch.empty(N, H, device="cuda")
    mean, rstd = torch.empty(H, device="cuda"), torch.empty(H, device="cuda")
    ws_bytes = L.lib().pert_bn_workspace_bytes(N, H)
    ws = torch.zeros(ws_bytes // 8 + 8, dtype=torch.float64, device="cuda")
    L.call("pert_bn_fwd", A.data_ptr(), H, bn["gamma"].data_ptr(), bn["beta"].data_ptr(), bn["rm"].data_ptr(),
           bn["rv"].data_ptr(), bn["nbt"].data_ptr(), EPS, MOMENTUM, training, 1, mean.data_ptr(), rstd.data_ptr(),
           y.data_ptr(), H, N, H, ws.data_ptr(), ws_bytes, _stream())
    return y, mean, rstd


def _check_planes(planes, pz, N, A, W4, b4, tag):
    """fp64 of the same A under the element-wise bar; spare rows and the tail untouched."""
    A64, W64, b64 = A.double(), W4.double(), b4.double()
    ref = A64 @ W64.t() + b64
    mag = A64.abs() @ W64.abs().t() + b64.abs()
    got = torch.stack([planes[z * pz: z * pz + N * H].view(N, H) for z in range(4)], 1).reshape(N, 4 * H)
    err = (got.double() - ref).abs()
    ratio = float((err / (_tau_nt(A.size(1)) * mag)).max())
    assert ratio <= 1.0, f"planes {tag}: element-wise error {ratio:.3g} x the bar"
    for z in range(4):
        assert bool((planes[z * pz + N * H: (z + 1) * pz] == SENTINEL).all()), f"rows past N of plane {z} ({tag})"
    assert bool((planes[4 * pz:] == SENTINEL).all()), f"memory after the planes ({tag})"


def _operands(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = (2.0 * torch.randn(N, K, generator=g) + 0.5).cuda()   # shifted: the normalisation has work to do
    W4 = (torch.randn(4 * H, K, generator=g) / math.sqrt(K)).cuda()
    b4 = (0.1 * torch.randn(4 * H, generator=g)).cuda()
    return g, A, W4, b4


@pytest.mark.parametrize("N", [4096, 4159, 51200])
@pytest.mark.parametrize("mode", ["train", "train_dropout", "eval"])
def test_bn_linear_fwd_planes_bn_mode(N, mode):
    L = _lib()
    assert L.lib().pert_bn_linear_fwd_planes_supported(N, H, H) == 1
    g, A, W4, b4 = _operands(N, H, seed=N + len(mode))
    training = 0 if mode == "eval" else 1
    p = 0.1 if mode == "train_dropout" else 0.0
    ctr = torch.tensor([SEED, STEP], dtype=torch.int64, device="cuda")
    s0 = _bn_state(g)
    s_ref, s_fused, s_again = _copy_state(s0), _copy_state(s0), _copy_state(s0)
    y_ref, mean_ref, rstd_ref = _reference_bn(A, s_ref, N, training)
    if p > 0:
        keep = torch.from_numpy(dropout_mask(SEED, STEP, LAYER, N, H, p)).cuda()
        y_ref = torch.where(keep, y_ref * scale_of(p), torch.zeros_like(y_ref))
    x_buf, planes, pz, (mean, rstd) = _fused(A, W4, b4, N, H, s_fused, training, p, ctr)
    _, planes2, _, _ = _fused(A, W4, b4, N, H, s_again, training, p, ctr)
    torch.cuda.synchronize()
    tag = f"N={N} {mode}"
    x = x_buf[:N * H].view(N, H)
    if not torch.equal(x, y_ref):
        bad = (x != y_ref).nonzero()
        rows = bad[:, 0].unique()
        raise AssertionError(
            f"x[l] differs from pert_bn_fwd ({tag}): {bad.size(0)} elements in {rows.numel()} rows (tiles "
            f"{sorted(set((rows // 64).tolist()))[:16]}), first {[(int(r), int(c), float(x[r, c]), float(y_ref[r, c])) for r, c in bad[:6].tolist()]}; "
            f"mean equal {torch.equal(mean, mean_ref)}, rstd equal {torch.equal(rstd, rstd_ref)}, "
            f"max |d mean| {float((mean - mean_ref).abs().max())}, max |d rstd| {float((rstd - rstd_ref).abs().max())}")
    assert bool((x_buf[N * H:] == SENTINEL).all()), f"memory after x[l] ({tag})"
    assert torch.equal(mean, mean_ref) and torch.equal(rstd, rstd_ref), f"mean / rstd ({tag})"
    for k in ("rm", "rv", "nbt"):
        assert torch.equal(s_fused[k], s_ref[k]), f"{k} ({tag})"
    if training:
        assert int(s_fused["nbt"]) == 4 and not torch.equal(s_fused["rm"], s0["rm"])
    else:
        assert all(torch.equal(s_fused[k], s0[k]) for k in ("rm", "rv", "nbt")), f"eval changed the state ({tag})"
    if p > 0:
        kept = float(keep.float().mean())
        assert 0.85 < kept < 0.95, kept
    _check_planes(planes, pz, N, y_ref, W4, b4, tag)
    assert torch.equal(planes, planes2), f"planes differ between two runs ({tag})"


@pytest.mark.parametrize("N", [4096, 4159, 51200])
def test_bn_linear_fwd_planes_plain_mode(N):
    """Conv 0: K = 80, A used as it is."""
    K = 80
    L = _lib()
    assert L.lib().pert_bn_linear_fwd_planes_supported(N, H, K) == 1
    _, A, W4, b4 = _operands(N, K, seed=N)
    _, planes, pz, _ = _fused(A, W4, b4, N, K)
    _, planes2, _, _ = _fused(A, W4, b4, N, K)
    torch.cuda.synchronize()
    _check_planes(planes, pz, N, A, W4, b4, f"N={N} plain K=80")
    assert torch.equal(planes, planes2), f"planes differ between two runs (N={N} plain)"


def test_bn_linear_fwd_planes_large_and_cancelling_columns():
    """A dominant column and a pair of columns whose contributions cancel: each output is held to the size of its own
    terms, not to the tensor's rms."""
    N, K = 4159, 80
    g, A, W4, b4 = _operands(N, K, seed=5)
    A[:, 7] *= 1e4
    r = torch.randn(N, generator=g).cuda()
    A[:, 20], A[:, 21] = 1e3 * r, 1e3 * r
    W4[:, 21] = -W4[:, 20]
    _, planes, pz, _ = _fused(A, W4, b4, N, K)
    torch.cuda.synchronize()
    _check_planes(planes, pz, N, A, W4, b4, "stress")
    assert np.isfinite(planes.cpu().numpy()).all()
