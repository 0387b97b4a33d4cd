"""Dead scratch that the step engine's H = 64 conv chain drops from L2 without a write-back (discard_l2, csrc/sm90.cuh):
the skip plane after the conv forward, the backward planes after the node-linear backward, and dx after the target
pass.  Their contents are undefined after a step, so nothing may read them again: a second backward from the same
forward must give the same gradients, and a second forward from the same parameters the same predictions.  Both are
also checked against the operator path, which runs none of the chain's hints or discards: a discard that hit a line
the backward reads would make both engine backwards agree with each other, but not with it."""
import copy

import pytest
import torch

from tests.helpers import assert_close, forward_args, make_batch, make_models

pytestmark = pytest.mark.gpu

# run-to-run spread of the engine's fp32 atomics (DESIGN section 7): gradients 2e-5 .. 9e-5 relative norm
GRAD_SPREAD = 1e-4
# engine against the operator path (other kernels, other summation orders), relative norm of the whole gradient
PATHS = 1e-3


def test_discarded_scratch_is_not_read_again():
    from pert_gnn_kdd23_b200.index import cached_index
    from pert_gnn_kdd23_b200.train import model_inputs

    _, model = make_models(2)
    model.train()
    model.dropout = 0.0                                   # the second forward draws no new mask
    op = copy.deepcopy(model)
    op.use_engine = False
    b = make_batch(2, 256, seed=1000).to("cuda")
    eng = model.engine()
    x, cat_X, edge_index, edge_attr, pnn, probs, entry_id, batch = model_inputs(b)
    index = cached_index(edge_index, x.size(0), edge_attr, model.interface_embeds.num_embeddings,
                         model.rpctype_embeds.num_embeddings)
    index.num_graphs = entry_id.numel()
    N, H = x.size(0), eng.Hp
    # the shape runs the chain that discards (the fused node linears at H = 64)
    assert H == 64 and eng.lib.pert_bn_linear_fwd_planes_supported(N, H, H) == 1
    assert eng.lib.pert_linear_bwd_planes_supported(N, H, H, H) == 1
    gen = torch.Generator(device="cuda").manual_seed(7)
    with torch.no_grad():
        g1, l1 = eng.forward(x, cat_X, entry_id, probs, pnn, batch, index, True)
        d_global = torch.randn(g1.shape, device="cuda", generator=gen)
        grads = []
        for _ in range(2):
            gbuf = torch.zeros_like(eng.fp.flat)          # the backward accumulates (+=)
            eng.backward(d_global.reshape(-1), None, grads=gbuf)
            grads.append(gbuf)
        g2, l2 = eng.forward(x, cat_X, entry_id, probs, pnn, batch, index, True)
    torch.cuda.synchronize()
    assert float(grads[0].abs().max()) > 0
    assert_close(grads[1], grads[0], rtol=GRAD_SPREAD, what="second backward from one forward", norm_only=True)
    assert_close(g2, g1, rtol=1e-5, what="global predictions of a second forward", norm_only=True)
    assert_close(l2, l1, rtol=1e-5, what="local predictions of a second forward", norm_only=True)

    go, lo = op(*forward_args(b))
    (go * d_global).sum().backward()
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    ref = dict(op.named_parameters())
    flat = lambda views: torch.cat([v.reshape(-1) for v in views])   # noqa: E731
    want = flat([ref[n].grad if ref[n].grad is not None else torch.zeros_like(ref[n]) for n in names])
    assert_close(g1, go.detach(), rtol=PATHS, what="engine forward against the operator path", norm_only=True)
    assert_close(flat(eng.fp.views_of(grads[0])), want, rtol=PATHS, what="engine backward against the operator path",
                 norm_only=True)
