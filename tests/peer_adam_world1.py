"""pert_allreduce_adam at world = 1 in the form PERT_PEER_MODE selects (ag: k_allreduce_adam, rs:
k_reduce_scatter_adam), against pert_adam_step on the same inputs and the fp64 reference of tests/loss_adam_ref.py.
The form is read once per process, so tests/test_gpu_loss_adam.py runs this script once per form:
    PERT_PEER_MODE=ag python tests/peer_adam_world1.py
Sizes: the scalar tail (n % 4 = 1, 2, 3), a sub-block size, and both sides of one grid-stride pass (SM count x 256
threads x 4 floats, read at run time).  Each size gets a fresh zeroed exchange buffer and 20 steps 1, 2, 3, ... in
order (the kernel's arrival counters and flags are monotonic in the step), which covers both halves of the all-gather
form's double buffer.  Prints PEER_WORLD1_OK and the worst errors as fractions of their bars."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from pert_gnn_kdd23_b200 import _lib
from tests.loss_adam_ref import adam_grad, adam_hyper, adam_state, adam_worst

STEPS = 20


def bits(t):
    return t.view(torch.int32)


def main():
    mode = os.environ.get("PERT_PEER_MODE", "")
    assert mode in ("ag", "rs"), mode
    L = _lib.lib()
    torch.cuda.init()
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    one_pass = sms * 256 * 4
    sizes = [1, 2, 3, 4, 5, 1023, one_pass - 1, one_pass, one_pass + 3, one_pass + 4, 2 * one_pass + 7]
    configs = [adam_hyper(lr=1e-3, betas=(0.9, 0.999), weight_decay=1e-2, grad_scale=0.125),
               adam_hyper(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, grad_scale=1.0)]
    worst = [0.0, 0.0, 0.0]
    st = _lib.stream()
    for k, n in enumerate(sizes):
        hp = configs[k % 2]
        # one rank maps no peer, so a plain device allocation serves as the exchange buffer
        xbuf = torch.zeros(L.pert_peer_exchange_bytes(n), dtype=torch.uint8, device="cuda")
        xbufs = (ctypes.c_void_p * 1)(xbuf.data_ptr())
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        timing = torch.zeros(5, dtype=torch.int64, device="cuda")
        rng = np.random.default_rng(k)
        p, g = adam_state(n, seed=k)
        pa = torch.from_numpy(p).cuda()
        ma, va = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        pb, mb, vb = pa.clone(), ma.clone(), va.clone()
        P = _lib.ptr
        for t in range(1, STEPS + 1):
            gd = torch.from_numpy(g).cuda()
            before = [x.cpu().numpy() for x in (pa, ma, va)]
            _lib.check(L.pert_adam_step(P(pa), P(gd), P(ma), P(va), n, hp["lr"], hp["b1"], hp["b2"], hp["eps"],
                                        hp["wd"], t, hp["gs"], st), "pert_adam_step")
            _lib.check(L.pert_allreduce_adam(P(pb), P(gd), P(mb), P(vb), n, hp["lr"], hp["b1"], hp["b2"],
                                             hp["eps"], hp["wd"], t, hp["gs"], xbufs, 0, 1, P(status), P(timing),
                                             st), "pert_allreduce_adam")
            for a, b, what in ((pa, pb, "p"), (ma, mb, "m"), (va, vb, "v")):
                assert torch.equal(bits(a), bits(b)), (mode, n, t, what)
            out = [x.cpu().numpy() for x in (pb, mb, vb)]
            w = adam_worst(before[0], g, before[1], before[2], t, hp, out)
            assert max(w) <= 1, (mode, n, t, w)
            worst = [max(a, b) for a, b in zip(worst, w)]
            g = adam_grad(n, rng)
        torch.cuda.synchronize()
        assert int(status.item()) == 0, (mode, n, int(status.item()))
        assert int(timing[4].item()) == STEPS, (mode, n, timing.tolist())
    print(f"PEER_WORLD1_OK mode={mode} sms={sms} sizes={len(sizes)} worst_m={worst[0]:.4g} worst_v={worst[1]:.4g} "
          f"worst_delta={worst[2]:.4g}")


if __name__ == "__main__":
    main()
