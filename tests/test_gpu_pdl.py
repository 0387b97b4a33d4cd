"""Programmatic dependent launch in the step engine (csrc/common.cuh): the conv chain's kernels start their set-up
while their predecessor drains.  Graph replay and eager issue must train the same model, and a captured step must
really hold the programmatic edges (a memset or an event between two chain kernels would cut them)."""
import copy
import ctypes

import pytest
import torch

from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

STEPS = 30


def _batch(jitter, seed):
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.synthetic import make_data_list

    dl = make_data_list(2, num_graphs=256, seed=seed, jitter=jitter)
    for d in dl:
        d._store.pop("level", None)
        d._store.pop("min_depth", None)
    return Batch.from_data_list(dl).to("cuda")


def _models():
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam

    torch.manual_seed(0)
    ma = SAGEDeterministic(*model_args(2)).cuda()
    mb = copy.deepcopy(ma)
    return (ma, FusedAdam(FlatParams(ma), lr=3e-4)), (mb, FusedAdam(FlatParams(mb), lr=3e-4))


@pytest.mark.parametrize("arm", ["graph", "jittered", "bucketed"])
def test_replayed_steps_match_eager_steps(arm):
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, GraphedTrainStep, fused_train_step

    (ma, oa), (mb, ob) = _models()
    batches = [_batch(0.2 if arm == "jittered" else 0.0, 1000 + 131 * r) for r in range(3)]
    if arm == "bucketed":
        step = BucketedTrainStep(mb, ob, 0.5)
        step.reserve(*(max(v) for v in zip(*[(b.x.size(0), b.edge_index.size(1), b.num_graphs) for b in batches])))
    else:
        step = GraphedTrainStep(mb, ob, 0.5)
    for it in range(STEPS):
        d = batches[it % len(batches)]
        la = fused_train_step(ma, oa, d, 0.5)
        lb = step(d)
        assert_close(torch.as_tensor(lb).reshape(1).float(), torch.as_tensor(la).reshape(1).float(), rtol=1e-4,
                     what=f"{arm} loss step {it}", norm_only=True)
    torch.cuda.synchronize()
    assert step.capture_error is None and step.replays >= STEPS - 2 * len(batches)
    assert_close(ob.fp.flat, oa.fp.flat, rtol=2e-3, what=f"{arm} parameters", norm_only=True)
    assert_close(ob.fp.grad, oa.fp.grad, rtol=2e-3, what=f"{arm} gradients", norm_only=True)
    ea, eb = ma._engine, mb._engine
    assert_close(eb.bn_running, ea.bn_running, rtol=2e-3, what=f"{arm} BatchNorm running statistics", norm_only=True)
    assert torch.equal(eb.bn_nbt, ea.bn_nbt)


# ---------------------------------------------------------------------------------------- edges of a captured step
class _KernelNodeParams(ctypes.Structure):
    _fields_ = [("func", ctypes.c_void_p), ("grid", ctypes.c_uint * 3), ("block", ctypes.c_uint * 3),
                ("shared", ctypes.c_uint), ("params", ctypes.c_void_p), ("extra", ctypes.c_void_p)]


class _EdgeData(ctypes.Structure):
    _fields_ = [("from_port", ctypes.c_ubyte), ("to_port", ctypes.c_ubyte), ("type", ctypes.c_ubyte),
                ("reserved", ctypes.c_ubyte * 5)]


def _cudart():
    """The CUDA runtime torch itself loaded."""
    with open("/proc/self/maps") as f:
        paths = {ln.split()[-1] for ln in f if "libcudart.so" in ln}
    assert paths, "torch has not loaded libcudart"
    return ctypes.CDLL(sorted(paths)[0])


def _kernel_name(rt, node):
    kind = ctypes.c_int()
    assert rt.cudaGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(kind)) == 0
    if kind.value != 0:                                  # cudaGraphNodeTypeKernel
        return None
    p, name = _KernelNodeParams(), ctypes.c_char_p()
    if rt.cudaGraphKernelNodeGetParams(ctypes.c_void_p(node), ctypes.byref(p)) != 0 or \
            rt.cudaFuncGetName(ctypes.byref(name), ctypes.c_void_p(p.func)) != 0:
        return None                                      # not a runtime-API kernel of this library
    return name.value.decode()


def test_captured_conv_chain_has_programmatic_edges():
    from pert_gnn_kdd23_b200.train import _fused_fwd_bwd, fused_train_step

    (m, o), _ = _models()
    d = _batch(0.0, 1000)
    fused_train_step(m, o, d, 0.5)                       # workspace, auxiliary stream and module loads
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        _fused_fwd_bwd(m, o, d, 0.5, None, None, use_index_cache=False)
    rt = _cudart()
    graph = ctypes.c_void_p(g.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert rt.cudaGraphGetEdges_v2(graph, None, None, None, ctypes.byref(n)) == 0
    src, dst = (ctypes.c_void_p * n.value)(), (ctypes.c_void_p * n.value)()
    data = (_EdgeData * n.value)()
    assert rt.cudaGraphGetEdges_v2(graph, src, dst, data, ctypes.byref(n)) == 0
    chain = ("k_bn_linear_fwd_planes", "k_tile_fwd", "k_tile_bwd_dst", "k_tile_bwd_src", "k_linear_bwd_planes")

    def fam(node):
        name = _kernel_name(rt, node)
        return next((c for c in chain if name and c in name), None)

    prog, plain = [], []
    for i in range(n.value):
        a, b = fam(src[i]), fam(dst[i])
        if a and b:
            (prog if data[i].type == 1 else plain).append((a, b))   # cudaGraphDependencyTypeProgrammatic
    # 3 convs: forward linear -> conv -> linear -> conv -> linear -> conv (5 edges), backward dst -> src -> linear
    # -> dst ... (8 edges)
    assert not plain, f"chain kernels joined by full edges: {plain}"
    assert len(prog) == 13, prog
    assert ("k_tile_fwd", "k_bn_linear_fwd_planes") in prog and ("k_linear_bwd_planes", "k_tile_bwd_dst") in prog
    del g
