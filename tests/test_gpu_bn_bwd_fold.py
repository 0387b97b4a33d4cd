"""-m gpu tests of the BatchNorm backward folded into the node-linear backward (pert_linear_bwd_planes_ex: column sums)
and the conv backward target pass (pert_tconv_bwd_bn: g = BN backward of dx), against the separate passes
pert_linear_bwd_planes + pert_bn_bwd + pert_tconv_bwd_c on the same inputs, at the cfg2 graph shape and at a jittered
batch whose graphs are cut by tile boundaries: dX bit for bit, g / dgamma / dbeta / every conv gradient within the
element-wise 1e-4 bar, the fp64 column sums against an fp64 restatement, ghost rows of a padded batch g = 0 exactly.
Then whole engine steps (training with dropout, eval) against the unfolded path."""
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from tests.helpers import assert_close, elem_err, is_structural_zero_grad, make_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 64


def _graph(jittered):
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.index import build_index
    from pert_gnn_kdd23_b200.synthetic import N_IF, N_RPC, make_data_list

    b = Batch.from_data_list(make_data_list(2, num_graphs=96, jitter=0.2)) if jittered else make_batch(2)
    N = b.x.size(0)
    gi = build_index(b.edge_index.cuda(), N, b.edge_attr.cuda(), N_IF, N_RPC).check()
    return gi, N, b.num_graphs, N_IF, N_RPC


def _case(jittered, p_drop=0.0, n_live=None, seed=0):
    from pert_gnn_kdd23_b200 import _lib

    call, ptr, st = _lib.call, _lib.ptr, _lib.stream()
    gi, N, B, n_if, n_rpc = _graph(jittered)
    E = gi.E
    assert _lib.lib().pert_linear_bwd_planes_supported(N, H, H, H) == 1
    assert _lib.lib().pert_tconv_bwd_bn_supported(H, n_rpc) == 1
    nl = N if n_live is None else n_live
    gen = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=gen)   # noqa: E731
    # BatchNorm of the previous conv: input x, batch statistics over the live rows, y = relu(bn(x)) [* keep / (1 - p)]
    x = rnd(N, H) * 1.7 + 0.4
    xd = x[:nl].double()
    mean = xd.mean(0).float()
    rstd = (1.0 / torch.sqrt(xd.var(0, unbiased=False) + 1e-5)).float()
    gamma, beta = rnd(H) * 0.5 + 1.0, rnd(H) * 0.5
    y = torch.relu((x - mean) * rstd * gamma + beta)
    scale = 1.0
    if p_drop > 0:
        scale = float(torch.tensor(1.0 / (1.0 - p_drop), dtype=torch.float64).float())
        y = y * (torch.rand(N, H, generator=gen) >= p_drop).float() * scale
    dY = rnd(4, N, H)
    W4t = (rnd(4 * H, H) / math.sqrt(H)).t().contiguous()
    q, k, v, s = (rnd(N, H) * 0.5 for _ in range(4))
    t_if, t_rpc = rnd(n_if, H) * 0.1, rnd(n_rpc, H) * 0.1
    cu = lambda t: t.cuda().contiguous()              # noqa: E731
    x, mean, rstd, gamma, y, dY, W4t, q, k, v, s, t_if, t_rpc = map(cu, (x, mean, rstd, gamma, y, dY, W4t, q, k, v, s,
                                                                         t_if, t_rpc))
    live = torch.tensor([nl, B], dtype=torch.int64, device="cuda") if n_live is not None else None
    # the forward of the conv: alpha
    out = torch.empty(N, H, device="cuda")
    alpha = torch.empty(max(E, 1), device="cuda")
    call("pert_tconv_fwd", ptr(q), ptr(k), ptr(v), ptr(s), H, ptr(gi.rowptr), ptr(gi.csr_src), ptr(gi.csr_if),
         ptr(gi.csr_rpc), ptr(t_if), ptr(t_rpc), ptr(out), H, ptr(alpha), n_rpc, N, E, B, H, st)

    def conv_bwd(name, g, *extra):
        d = torch.full((3, N, H), float("nan"), device="cuda")
        r = {"dsp": torch.empty(max(E, 1), device="cuda"), "dt_if": torch.zeros_like(t_if),
             "dt_rpc": torch.zeros_like(t_rpc)}
        rpc_ws = torch.empty(16 * N, device="cuda")
        call(name, ptr(g), H, ptr(q), ptr(k), ptr(v), H, ptr(gi.rowptr), ptr(gi.csr_src), ptr(gi.csr_if),
             ptr(gi.csr_rpc), ptr(gi.colptr), ptr(gi.csc_pos), ptr(gi.csc_dst), ptr(t_if), ptr(t_rpc), ptr(alpha),
             ptr(d[0]), ptr(d[1]), ptr(d[2]), H, ptr(r["dsp"]), ptr(rpc_ws), ptr(r["dt_if"]), ptr(r["dt_rpc"]), n_rpc,
             N, E, B, H, H, *extra, st)
        r.update(dq=d[0], dk=d[1], dv=d[2])
        return r

    # separate passes
    dW_r, db_r = torch.zeros(4 * H, H, device="cuda"), torch.zeros(4 * H, device="cuda")
    dX_r = torch.empty(N, H, device="cuda")
    call("pert_linear_bwd_planes", ptr(dY), N * H, ptr(y), H, ptr(W4t), 4 * H, ptr(dW_r), H, ptr(db_r), ptr(dX_r), H,
         N, H, H, H, st)
    g_r = torch.zeros(N, H, device="cuda")
    dgam_r, dbet_r = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    sums32 = torch.empty(2 * H, device="cuda")
    dz_in = (dX_r * scale).contiguous()                # pert_bn_bwd has no relu_scale: dx * scale rounds as __fmul_rn
    call("pert_bn_bwd", ptr(dz_in), H, ptr(y), H, ptr(x), H, ptr(mean), ptr(rstd), ptr(gamma), 1, 1, ptr(g_r), H,
         ptr(dgam_r), ptr(dbet_r), ptr(sums32), nl, H, st)   # the live rows are a prefix: ghost rows keep g = 0
    ref = conv_bwd("pert_tconv_bwd_c", g_r)

    # folded
    dW_f, db_f = torch.zeros_like(dW_r), torch.zeros_like(db_r)
    dX_f = torch.empty(N, H, device="cuda")
    sums = torch.zeros(2 * H, dtype=torch.float64, device="cuda")
    call("pert_linear_bwd_planes_ex", ptr(dY), N * H, ptr(y), H, ptr(W4t), 4 * H, ptr(dW_f), H, ptr(db_f), ptr(dX_f),
         H, N, H, H, H, ptr(x), ptr(mean), ptr(rstd), scale, ptr(live), ptr(sums), st)
    g_f = torch.full((N, H), float("nan"), device="cuda")
    dgam_f, dbet_f = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    bn = _lib.PertBnBwd(ptr(dX_f), ptr(y), ptr(x), ptr(mean), ptr(rstd), ptr(gamma), ptr(sums), ptr(dgam_f),
                        ptr(dbet_f), ptr(live), scale)
    got = conv_bwd("pert_tconv_bwd_bn", g_f, ctypes.byref(bn))
    torch.cuda.synchronize()

    tag = f"{'jittered' if jittered else 'cfg2'} p={p_drop} live={n_live}"
    assert torch.equal(dX_f, dX_r), f"dX differs from pert_linear_bwd_planes ({tag})"
    assert_close(dW_f, dW_r, what=f"dW4 {tag}")
    assert_close(db_f, db_r, what=f"db4 {tag}")
    # the fp64 sums against an fp64 restatement over the live rows
    dz = (dX_f[:nl].double() * scale) * (y[:nl] > 0).double()
    xh = (x[:nl].double() - mean.double()) * rstd.double()
    want = torch.cat([dz.sum(0), (dz * xh).sum(0)])
    assert elem_err(sums, want) <= 1e-5, f"BatchNorm sums ({tag}): {elem_err(sums, want):.3e}"
    assert_close(dbet_f, dbet_r, what=f"dbeta {tag}")
    assert_close(dgam_f, dgam_r, what=f"dgamma {tag}")
    assert_close(g_f[:nl], g_r[:nl], what=f"g {tag}")
    if nl < N:
        assert bool((g_f[nl:] == 0).all()) and not bool(torch.signbit(g_f[nl:]).any()), f"ghost rows of g ({tag})"
    for key in ("dq", "dk", "dv", "dt_if", "dt_rpc"):
        assert_close(got[key], ref[key], what=f"{key} {tag}")
    assert_close(got["dsp"][:E], ref["dsp"][:E], what=f"ds {tag}")


@pytest.mark.parametrize("jittered", [False, True])
def test_fold_matches_separate_passes(jittered):
    _case(jittered)


@pytest.mark.parametrize("jittered", [False, True])
def test_fold_with_dropout(jittered):
    _case(jittered, p_drop=0.1, seed=1)


def test_fold_padded_batch_ghost_rows():
    """A padded batch: the statistics, the sums and the mean terms count the rows below live[0]; the rest get g = 0."""
    _case(False, n_live=51200 - 1234, seed=2)


def test_fold_rejects_bad_arguments():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_tconv_bwd_bn_supported(128, 8) == 0 and L.pert_tconv_bwd_bn_supported(64, 8) == 1
    assert L.pert_tconv_bwd_bn_supported(64, 65) == 0
    buf = torch.zeros(1024, device="cuda")
    p = buf.data_ptr()
    args = [p, 64] + [p] * 3 + [64] + [p] * 13 + [64] + [p] * 4 + [8, 100, 100, 1, 64, 64]
    assert L.pert_tconv_bwd_bn(*args, None, None) == -1                     # no argument block
    bn = _lib.PertBnBwd(p, p, p, p, p, p, None, p, p, None, 1.0)            # no sums
    assert L.pert_tconv_bwd_bn(*args, ctypes.byref(bn), None) == -1
    lin = [p, 100 * 64, p, 64, p, 256, p, 64, p, p, 64, 100, 64, 64, 64]
    assert L.pert_linear_bwd_planes_ex(*lin, None, p, p, 1.0, None, p, None) == -1     # sums without bn_x
    lin80 = [p, 100 * 64, p, 80, p, 256, p, 80, p, p, 80, 100, 64, 80, 80]
    assert L.pert_linear_bwd_planes_ex(*lin80, p, p, p, 1.0, None, p, None) == -1      # K != H


_STEP = r"""
import json, sys, torch
sys.path.insert(0, {root!r})
from tests.helpers import forward_args, make_batch, make_models
from oracle.model_oracle import torch_quantile_loss
_, model = make_models(2, seed=0)
model.dropout = {p}
model.seed_dropout(7)
if not {training}:
    model.eval()
b = make_batch(2).to("cuda:0")
g, l = model(*forward_args(b))
torch_quantile_loss(b.y.float(), g.flatten(), 0.5).backward()
torch.cuda.synchronize()
torch.save({{n: p.grad.cpu() for n, p in model.named_parameters() if p.grad is not None}}, {out!r})
"""


@pytest.mark.parametrize("training,p", [(True, 0.0), (True, 0.1), (False, 0.0)])
def test_engine_step_matches_unfolded_path(tmp_path, training, p):
    """One cfg2 step (the fold runs in training) against the same step with PERT_LINEAR_BWD_FUSED=0, which takes the
    two GEMMs and the separate BatchNorm passes (child processes: the switch is read once per process).  The bar is
    test_gpu_linear_bwd's for that comparison."""
    grads = {}
    for flag in ("1", "0"):
        out = str(tmp_path / f"grads{flag}.pt")
        env = dict(os.environ, PERT_LINEAR_BWD_FUSED=flag)
        subprocess.run([sys.executable, "-c", _STEP.format(root=ROOT, out=out, p=p, training=training)], env=env,
                       cwd=ROOT, check=True)
        grads[flag] = torch.load(out)
    assert grads["1"].keys() == grads["0"].keys() and len(grads["1"]) > 10
    bad = {}
    for n, a in grads["1"].items():
        b = grads["0"][n].double()
        e = float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))
        if e > 1e-5 and not is_structural_zero_grad(n, 3):
            bad[n] = e
    assert not bad, json.dumps(bad)
