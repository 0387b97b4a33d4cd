"""CPU tests of the node kernels' host-side checks (csrc/nodeops.cu) and of the nn shims' refusals: every bad argument
is rejected before anything is launched, so none of these needs a device."""
import pytest
import torch

BADARG, UNSUPPORTED = -1, -2
FAKE = 1 << 20   # never dereferenced: validation runs first


def _lib():
    from pert_gnn_kdd23_b200 import _lib as L

    return L.lib()


def _bn_fwd(**kw):
    a = dict(x=FAKE, ld_x=64, gamma=FAKE, beta=FAKE, rm=FAKE, rv=FAKE, nbt=FAKE, eps=1e-5, momentum=0.1, training=1,
             relu=1, mean=FAKE, rstd=FAKE, y=FAKE, ld_y=64, N=129, H=64, ws=FAKE, ws_bytes=1 << 16, stream=None)
    a.update(kw)
    return _lib().pert_bn_fwd(*a.values())


def _bn_bwd(**kw):
    a = dict(dy=FAKE, ld_dy=64, y=FAKE, ld_y=64, x=FAKE, ld_x=64, mean=FAKE, rstd=FAKE, gamma=FAKE, relu=1, training=1,
             dx=FAKE, ld_dx=64, dgamma=FAKE, dbeta=FAKE, sums=FAKE, N=129, H=64, stream=None)
    a.update(kw)
    return _lib().pert_bn_bwd(*a.values())


@pytest.mark.parametrize("bad", [
    dict(H=1028, ld_x=1028, ld_y=1028), dict(H=62, ld_x=64, ld_y=64), dict(H=0), dict(N=-1), dict(ld_x=66),
    dict(ld_y=66), dict(x=None), dict(y=None), dict(gamma=None), dict(mean=None), dict(x=FAKE + 4),
])
def test_bn_fwd_badarg(bad):
    assert _bn_fwd(**bad) == BADARG


@pytest.mark.parametrize("bad", [
    dict(H=1028, ld_dy=1028, ld_y=1028, ld_x=1028, ld_dx=1028), dict(H=62), dict(N=-1), dict(ld_dy=66),
    dict(ld_x=66), dict(ld_dx=66), dict(ld_y=66), dict(relu=1, y=None), dict(dx=None), dict(sums=None),
    dict(dy=FAKE + 4),
])
def test_bn_bwd_badarg(bad):
    assert _bn_bwd(**bad) == BADARG


def test_bn_bwd_ld_y_unused_without_relu():
    """Without ReLU the saved output is not read, so its pointer and stride are not checked (N = 0: nothing runs)."""
    assert _bn_bwd(relu=0, y=None, ld_y=3, N=0) == 0


def test_embedding_badarg():
    L = _lib()
    fwd = lambda **kw: L.pert_embedding_fwd(*dict(dict(table=FAKE, n_rows=10, ids=FAKE, id_stride=1, out=FAKE,  # noqa
                                                       ld_out=64, N=100, H=64, acc=0, status=None, stream=None),
                                                  **kw).values())
    bwd = lambda **kw: L.pert_embedding_bwd(*dict(dict(dy=FAKE, ld_dy=64, ids=FAKE, id_stride=1, dt=FAKE,  # noqa
                                                       n_rows=10, N=100, H=64, stream=None), **kw).values())
    for bad in (dict(H=62), dict(H=0), dict(ld_out=66), dict(N=-1), dict(n_rows=0), dict(table=None), dict(out=None),
                dict(out=FAKE + 4)):
        assert fwd(**bad) == BADARG, bad
    for bad in (dict(H=62), dict(H=0), dict(ld_dy=66), dict(N=-1), dict(dy=None), dict(dt=None), dict(dt=FAKE + 8)):
        assert bwd(**bad) == BADARG, bad
    assert fwd(N=0) == 0 and bwd(N=0) == 0


def test_pool_badarg_and_widths():
    L = _lib()
    fwd = lambda **kw: L.pert_pool_fwd(*dict(dict(x=FAKE, ld=64, probs=FAKE, pnn=FAKE, batch=FAKE, w=None, b=None,  # noqa
                                                  local=None, pool=FAKE, N=100, B=4, H=64, status=None, stream=None),
                                             **kw).values())
    bwd = lambda **kw: L.pert_pool_bwd(*dict(dict(dpool=FAKE, dlocal=None, x=FAKE, ld=64, probs=FAKE, pnn=FAKE,  # noqa
                                                  batch=FAKE, w=None, dx=FAKE, ld_dx=64, dw=None, db=None, N=100, B=4,
                                                  H=64, stream=None), **kw).values())
    for bad in (dict(N=-1), dict(B=-1), dict(x=None), dict(batch=None), dict(pool=None), dict(ld=66),
                dict(x=FAKE + 4)):
        assert fwd(**bad) == BADARG, bad
    for bad in (dict(N=-1), dict(B=-1), dict(dx=None), dict(probs=None), dict(ld_dx=66), dict(dlocal=FAKE)):
        assert bwd(**bad) == BADARG, bad
    for H in (1, 5, 12, 48, 100, 200, 260, 512):       # widths the pool kernel lacks: refused before the zero-fill
        assert fwd(H=H, ld=(H + 3) // 4 * 4) == UNSUPPORTED, H
    # empty batches and pools may pass NULL (empty tensors); nothing is launched
    assert fwd(N=0, B=0, x=None, probs=None, pnn=None, batch=None, pool=None) == 0
    assert bwd(N=0, B=0, dpool=None, x=None, probs=None, pnn=None, batch=None, dx=None) == 0


# ---------------------------------------------------------------------------------- nn shims, CPU tensors
def _bn(C=8, **kw):
    from pert_gnn_kdd23_b200.nn import BatchNorm1d

    return BatchNorm1d(C, **kw)


@pytest.mark.parametrize("shape", [(4, 8, 3), (4, 8, 3, 2)])
def test_batchnorm_refuses_non_2d_input(shape):
    """torch's BatchNorm1d takes [N, C, L] as well; the shim normalises [N, C] only and says so."""
    bn = _bn()
    with pytest.raises(NotImplementedError if len(shape) == 3 else ValueError):
        bn(torch.randn(*shape))
    with pytest.raises(ValueError):
        bn(torch.randn(8))


def test_batchnorm_refuses_cumulative_momentum():
    bn = _bn(momentum=None)
    with pytest.raises(NotImplementedError, match="momentum=None"):
        bn(torch.randn(4, 8))
    assert int(bn.num_batches_tracked) == 0 and torch.equal(bn.running_var, torch.ones(8))


def test_batchnorm_training_one_row_raises_like_torch():
    x = torch.randn(1, 8)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        torch.nn.BatchNorm1d(8)(x)
    bn = _bn()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        bn(x)
    bn_nostats = _bn(track_running_stats=False).eval()    # no running statistics: eval normalises by the batch
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        bn_nostats(x)
    assert int(bn.num_batches_tracked) == 0 and torch.equal(bn.running_mean, torch.zeros(8))


def test_batchnorm_cpu_input_has_no_fallback():
    """Valid input that passes the shim's checks reaches the CUDA path, which refuses CPU tensors."""
    from pert_gnn_kdd23_b200._lib import PertGnnError

    for bn in (_bn(), _bn(affine=False), _bn(momentum=None).eval()):
        with pytest.raises(PertGnnError, match="CUDA"):
            bn(torch.randn(4, 8))
