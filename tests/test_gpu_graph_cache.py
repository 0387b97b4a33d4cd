"""-m gpu: train._GraphCache, the capture-and-replay bookkeeping of every graph-replayed step in train.py.

The cache is driven directly with a tiny engine and a step of one kernel (``pert_eval_metrics``, which adds |0 - 1| per
label into a device sum, so the sum counts how often the kernel really ran): eager first visit, capture + replay,
replays, the stale-graph rules, the ``max_graphs`` cap, a failed capture and the ``ops.LAUNCHES`` bookkeeping.  Then
``GraphedTrainStep`` across a workspace re-allocation."""
import copy

import pytest
import torch

from tests.helpers import assert_close, make_batch, make_models

pytestmark = pytest.mark.gpu

B = 8
SMALL = (64, 128, 4)
BIG = (4096, 8192, 64)


def _step():
    """-> (model, engine, fn, runs): ``fn`` launches one kernel and returns the device sum; ``runs()`` is how many
    times the kernel has run (synchronising)."""
    from pert_gnn_kdd23_b200.train import EvalMetrics

    _, model = make_models(1)
    eng = model.engine()
    m = EvalMetrics("cuda")
    y = torch.ones(B, dtype=torch.int64, device="cuda")
    yhat = torch.zeros(B, dtype=torch.float32, device="cuda")

    def fn():
        m.update(y, yhat)
        return m.acc

    def runs():
        torch.cuda.synchronize()
        return int(m.acc[0].item()) // B

    return model, eng, fn, runs


def _counters(c):
    return c.captures, c.replays, c.invalidations


def test_eager_then_capture_then_replay():
    from pert_gnn_kdd23_b200 import ops
    from pert_gnn_kdd23_b200.train import _GraphCache

    _, eng, fn, runs = _step()
    c = _GraphCache()
    l0 = ops.LAUNCHES["n"]
    first = c.cache("k", eng, SMALL, fn)                 # eager
    assert runs() == 1 and _counters(c) == (0, 0, 0) and ops.LAUNCHES["n"] - l0 == 1
    assert eng.ws is not None and eng.ws_key == SMALL    # the workspace was sized before the step
    second = c.cache("k", eng, SMALL, fn)                # captured, then replayed
    assert runs() == 2 and _counters(c) == (1, 1, 0) and ops.LAUNCHES["n"] - l0 == 2
    third = c.cache("k", eng, SMALL, fn)                 # replayed
    assert runs() == 3 and _counters(c) == (1, 2, 0) and ops.LAUNCHES["n"] - l0 == 3
    assert third is second and first is second          # the tensor the capture wrote into
    ent = c.buckets["k"]
    assert ent["engine"] is eng and ent["ws"] is eng.ws and ent["ws_gen"] == eng.ws_generation
    assert c.capture_error is None


def test_workspace_reallocation_recaptures_the_visited_key_only():
    from pert_gnn_kdd23_b200.train import _GraphCache

    _, eng, fn, runs = _step()
    c = _GraphCache()
    for k in ("a", "a", "b", "b"):
        c.cache(k, eng, SMALL, fn)
    assert _counters(c) == (2, 2, 0)
    gen, graph_b = eng.ws_generation, c.buckets["b"]["graph"]
    c.cache("big", eng, BIG, fn)                         # eager, and the workspace grows
    assert eng.ws_generation == gen + 1
    c.cache("a", eng, SMALL, fn)                         # stale: captured again and replayed on this visit
    assert _counters(c) == (3, 3, 1)
    assert c.buckets["a"]["ws_gen"] == eng.ws_generation
    assert c.buckets["b"]["graph"] is graph_b and c.buckets["b"]["ws_gen"] == gen      # not touched yet
    c.cache("a", eng, SMALL, fn)
    assert _counters(c) == (3, 4, 1)
    c.cache("b", eng, SMALL, fn)
    assert _counters(c) == (4, 5, 2) and c.buckets["b"]["graph"] is not graph_b
    assert runs() == 8 and c.capture_error is None


def test_a_recreated_engine_invalidates_its_graph():
    from pert_gnn_kdd23_b200.train import FlatParams, _GraphCache

    model, eng, fn, runs = _step()
    c = _GraphCache()
    for _ in range(2):
        c.cache("k", eng, SMALL, fn)
    FlatParams(model)                                    # parameters move: the next engine() is a new one
    eng2 = model.engine()
    assert eng2 is not eng and eng2.ws is None
    c.cache("k", eng2, SMALL, fn)
    assert _counters(c) == (2, 2, 1)
    ent = c.buckets["k"]
    assert ent["engine"] is eng2 and ent["ws"] is eng2.ws and eng2.ws_key == SMALL
    c.cache("k", eng2, SMALL, fn)
    assert _counters(c) == (2, 3, 1) and runs() == 4


def test_a_key_beyond_max_graphs_stays_eager():
    from pert_gnn_kdd23_b200 import ops
    from pert_gnn_kdd23_b200.train import _GraphCache

    _, eng, fn, runs = _step()
    c = _GraphCache(max_graphs=1)
    for _ in range(2):
        c.cache("a", eng, SMALL, fn)
    l0 = ops.LAUNCHES["n"]
    for _ in range(4):
        c.cache("b", eng, SMALL, fn)
    assert _counters(c) == (1, 1, 0) and c.buckets["b"]["state"] == "eager"
    assert runs() == 6 and ops.LAUNCHES["n"] - l0 == 4
    c.cache("a", eng, SMALL, fn)
    assert _counters(c) == (1, 2, 0) and runs() == 7


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")     # the refused capture recorded nothing
def test_a_failed_capture_stays_eager():
    from pert_gnn_kdd23_b200 import ops
    from pert_gnn_kdd23_b200.train import _GraphCache

    _, eng, fn, runs = _step()

    def refuses_capture():
        if torch.cuda.is_current_stream_capturing():     # raised before anything is launched
            raise RuntimeError("not capturable")
        return fn()

    c = _GraphCache()
    l0 = ops.LAUNCHES["n"]
    for _ in range(4):
        c.cache("k", eng, SMALL, refuses_capture)
    assert "not capturable" in c.capture_error
    assert _counters(c) == (0, 0, 0) and c.buckets["k"]["state"] == "eager"
    assert runs() == 4 and ops.LAUNCHES["n"] - l0 == 4  # every visit ran eagerly, the failed capture counted nothing


def test_graphed_step_recaptures_on_the_visit_after_workspace_growth():
    """small (eager), small (capture + replay), big (eager: the workspace grows), small: its graph points into the old
    workspace, so this visit captures it again and replays it; every loss equals eager fused_train_step's."""
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep, fused_train_step

    _, model_a = make_models(1)
    model_b = copy.deepcopy(model_a)
    opt_a = FusedAdam(FlatParams(model_a), lr=1e-3)
    opt_b = FusedAdam(FlatParams(model_b), lr=1e-3)
    small = make_batch(1, 16, seed=1).to("cuda")
    big = make_batch(1, 64, seed=2).to("cuda")
    gs = GraphedTrainStep(model_b, opt_b, 0.5)
    want = [(0, 0, 0), (1, 1, 0), (1, 1, 0), (2, 2, 1), (2, 3, 1)]
    for it, data in enumerate([small, small, big, small, small]):
        gen = model_b._engine.ws_generation if model_b._engine is not None else None
        la = fused_train_step(model_a, opt_a, data, 0.5)
        lb = gs(data)
        assert_close(lb, la, what=f"loss step {it}")
        assert _counters(gs) == want[it], (it, _counters(gs))
        if it == 2:
            assert model_b._engine.ws_generation == gen + 1
    key = gs._key(small) + (True, float(model_b.dropout))
    ent = gs.buckets[key]
    assert ent["ws_gen"] == model_b._engine.ws_generation and ent["pin"] is small
    assert gs.capture_error is None
