"""Gradient accumulation with ``DistributedDataParallel.no_sync()`` on one H100 (backend "b200", world size 1): ResNet-18
and the tutorial's Net with every flat optimizer on its kernel path, bit for bit against the optimizer applied once to the
accumulated sum, without host synchronisation, and captured k = 4 cycles against eager ones.  Workers in
tests/accumulation_workers.py."""
import pytest
import torch

import accumulation_workers as W
import capturable_workers as CW
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def test_accumulated_cycles_equal_the_reference():
    b2.launch(W.w_gpu_against_reference, size=1, backend="b200", join_timeout_s=800)


@pytest.mark.parametrize("name,make", CW.optimizers(), ids=[n for n, _ in CW.optimizers()])
def test_captured_cycle_replays_equal_eager_cycles(name, make):
    dev = torch.device("cuda", 0)
    eager, _, n_eager = W.graph_cycles(make, 5, False, dev)
    graph, opt, n_graph = W.graph_cycles(make, 5, True, dev)
    assert CW.same(eager, graph), name
    assert n_eager == n_graph == 5 and opt.steps == W.GRAPH_WARMUP + 5
