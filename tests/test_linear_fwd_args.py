"""CPU tests of pert_bn_linear_fwd_planes' argument checks: every bad argument is rejected with PERT_ERR_BADARG before
the device is touched, shapes and layouts outside the kernel get PERT_ERR_UNSUPPORTED with nothing launched, and the
shape predicate refuses what the kernel does not take."""
import pytest

BADARG, UNSUPPORTED = -1, -2
FAKE = 1 << 20   # never dereferenced: validation runs first


def _args(**kw):
    N = kw.get("N", 4096)
    a = dict(A=FAKE, lda=64, bn=1, gamma=FAKE, beta=FAKE, rm=FAKE, rv=FAKE, nbt=FAKE, eps=1e-5, momentum=0.1,
             training=1, mean=FAKE, rstd=FAKE, x_out=FAKE, ld_x_out=64, ws=FAKE, ws_bytes=1 << 12, stats_ready=0,
             dropout=0.1, drop_ctr=FAKE, drop_layer=0, W4=FAKE, ldw=64, b4=FAKE, planes=FAKE, pz=N * 64, N=N, H=64,
             K=64, stream=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("bad", [
    dict(A=None), dict(W4=None), dict(b4=None), dict(planes=None), dict(N=-1), dict(H=0), dict(K=0), dict(lda=63),
    dict(ldw=63), dict(pz=4096 * 64 - 1),
    # BatchNorm mode: the checks of pert_bn_fwd_ex
    dict(gamma=None), dict(beta=None), dict(mean=None), dict(rstd=None), dict(x_out=None), dict(ld_x_out=63),
    dict(gamma=FAKE + 4), dict(dropout=-0.1), dict(dropout=1.5), dict(dropout=float("nan")), dict(drop_ctr=None),
    dict(ws=None), dict(ws_bytes=8), dict(ws=FAKE + 4), dict(training=0, rm=None), dict(training=0, rv=None),
    dict(N=(1 << 32) // 16, pz=(1 << 32) * 4),   # N * H / 4 = 2^32 float4 groups overflow the mask counter
])
def test_bn_linear_fwd_planes_badarg(bad):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_bn_linear_fwd_planes(*_args(**bad)) == BADARG


@pytest.mark.parametrize("odd", [
    dict(N=4095, pz=4095 * 64), dict(H=128, K=128, lda=128, ldw=128, ld_x_out=128, pz=4096 * 128),
    dict(K=96, lda=96, ldw=96, ld_x_out=96),
    dict(K=80, lda=80, ldw=80, ld_x_out=80),      # BatchNorm mode needs K = H
    dict(lda=68), dict(ld_x_out=68), dict(pz=4096 * 64 + 2), dict(A=FAKE + 4), dict(planes=FAKE + 8),
    dict(x_out=FAKE + 4),
    dict(bn=0, K=72, lda=72, ldw=72),
])
def test_bn_linear_fwd_planes_unsupported_layouts(odd):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_bn_linear_fwd_planes(*_args(**odd)) == UNSUPPORTED


def test_bn_linear_fwd_planes_plain_mode_ignores_bn_arguments():
    """bn = 0 does not look at the BatchNorm arguments (all NULL here); the shape is still checked first."""
    from pert_gnn_kdd23_b200 import _lib

    nulls = dict(bn=0, gamma=None, beta=None, rm=None, rv=None, nbt=None, mean=None, rstd=None, x_out=None, ws=None,
                 drop_ctr=None, dropout=float("nan"), K=80, lda=80, ldw=80)
    assert _lib.lib().pert_bn_linear_fwd_planes(*_args(**nulls, N=4095, pz=4095 * 64)) == UNSUPPORTED
    assert _lib.lib().pert_bn_linear_fwd_planes(*_args(**nulls, A=None)) == BADARG


def test_bn_linear_fwd_planes_unsupported_shapes():
    """Shapes outside the kernel are refused whatever the device (the supported ones are checked on the GPU, where the
    predicate also asks whether the kernel fits)."""
    from pert_gnn_kdd23_b200 import _lib

    ok = _lib.lib().pert_bn_linear_fwd_planes_supported
    assert ok(4095, 64, 64) == 0 and ok(4095, 64, 80) == 0    # small batches: pert_bn_fwd_ex + pert_gemm_nt
    assert ok(51200, 128, 128) == 0 and ok(51200, 64, 96) == 0 and ok(51200, 64, 72) == 0 and ok(51200, 32, 64) == 0
    assert ok(1 << 31, 64, 64) == 0
