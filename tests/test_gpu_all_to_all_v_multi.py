"""``comm.all_to_all_single`` with split sizes and ``comm.all_to_all`` on ``backend="b200"``: the variable-segment kernel
through the public API, never NCCL.  World 1 on one GPU; on several GPUs against NCCL at the available world sizes and on a
sub-group, with random splits that change from call to call."""
import pytest
import torch

import all_to_all_v_workers as W
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def go(fn, size):
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


def test_world_one_calls_equal_torch():
    go(W.w_world1, 1)


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_all_to_all_with_splits_and_lists_match_nccl(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    go(W.w_vs_nccl, world)


@pytest.mark.multigpu
def test_all_to_all_with_splits_and_lists_on_a_subgroup_match_nccl():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    go(W.w_subgroup_vs_nccl, min(n, 4))
