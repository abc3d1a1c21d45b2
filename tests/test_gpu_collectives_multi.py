"""The collectives comm.py routes to the peer-memory kernels on ``backend="b200"``: PRODUCT / MAX / MIN all-reduce, reduce,
broadcast and all-gather, through the public API.  World 1 on one GPU; on several GPUs against NCCL at the available world
sizes, an odd world and a sub-group."""
import pytest
import torch

import collectives_workers as W
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def go(fn, size):
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


def test_world_one_collectives_equal_torch():
    go(W.w_collectives_world1, 1)


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_routed_collectives_match_nccl(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    go(W.w_collectives_vs_nccl, world)


@pytest.mark.multigpu
def test_routed_collectives_on_a_subgroup_match_nccl():
    n = torch.cuda.device_count()
    go(W.w_collectives_subgroup_vs_nccl, min(n, 4))
