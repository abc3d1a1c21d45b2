"""``FlatEMA`` with a sharded kernel-mode ``FlatSGD`` on ``backend="b200"`` with real GPUs: the EMA of the owned slices and
``average_parameters()`` against the unsharded run.  Skipped below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import ema_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 8])
def test_sharded_ema_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_gpu_multi, size=world, backend="b200", join_timeout_s=800)
