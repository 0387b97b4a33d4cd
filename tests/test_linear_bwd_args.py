"""CPU tests of pert_linear_bwd_planes' argument checks: every bad argument is rejected with PERT_ERR_BADARG before the
device is touched, and the shape predicate refuses what the fused kernel does not take."""
import pytest

BADARG = -1
FAKE = 1 << 20   # never dereferenced: validation runs first


def _args(**kw):
    a = dict(dY=FAKE, pz=4096 * 64, X=FAKE, ldx=80, W4t=FAKE, ldw=256, dW4=FAKE, ldw4=80, db4=FAKE, dX=FAKE,
             ldx_out=80, N=4096, H=64, K=80, Kd=64, stream=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("bad", [dict(dY=None), dict(X=None), dict(W4t=None), dict(dW4=None), dict(db4=None),
                                 dict(dX=None), dict(N=-1), dict(H=0), dict(K=0), dict(Kd=0), dict(Kd=96),
                                 dict(ldx=79), dict(ldw=255), dict(ldw4=79), dict(ldx_out=63),
                                 dict(pz=4096 * 64 - 1)])
def test_linear_bwd_planes_badarg(bad):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_linear_bwd_planes(*_args(**bad)) == BADARG


def test_linear_bwd_planes_unsupported_shapes():
    """Shapes outside the fused kernel are refused whatever the device (the supported ones are checked on the GPU,
    where the predicate also asks whether a cluster of the kernel's CTAs fits)."""
    from pert_gnn_kdd23_b200 import _lib

    ok = _lib.lib().pert_linear_bwd_planes_supported
    assert ok(4095, 64, 64, 64) == 0                        # small batches: the GEMM pair
    assert ok(51200, 128, 128, 128) == 0 and ok(51200, 64, 96, 64) == 0 and ok(51200, 64, 80, 72) == 0
