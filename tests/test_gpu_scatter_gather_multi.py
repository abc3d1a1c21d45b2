"""``comm.scatter`` and ``comm.gather`` on ``backend="b200"``: the peer-memory kernels through the public API, never NCCL.
World 1 on one GPU; on several GPUs against NCCL at the available world sizes, an odd world and a sub-group."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import scatter_gather_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def go(fn, size):
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


def test_world_one_scatter_and_gather_equal_torch():
    go(W.w_scatter_gather_world1, 1)


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_scatter_and_gather_match_nccl(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    go(W.w_scatter_gather_vs_nccl, world)


@pytest.mark.multigpu
def test_scatter_and_gather_on_a_subgroup_match_nccl():
    n = torch.cuda.device_count()
    go(W.w_scatter_gather_subgroup_vs_nccl, min(n, 4))
