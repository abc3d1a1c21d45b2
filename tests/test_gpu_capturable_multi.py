"""Captured DDP steps with ``capturable=True`` on ``backend="b200"`` with real GPUs: graph replays equal eager steps bit for
bit, unsharded and sharded, and the replicas are identical.  Skipped below two GPUs."""
import pytest
import torch

import capturable_workers as WK
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 8])
def test_graph_equals_eager_across_ranks(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(WK.w_graph_equals_eager, size=world, backend="b200", join_timeout_s=600)
