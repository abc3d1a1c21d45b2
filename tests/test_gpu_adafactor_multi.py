"""``DistributedDataParallel`` + ``FlatAdafactor`` on ``backend="b200"`` with real GPUs: replicas bit-identical, and the
result bit for bit one FlatAdafactor fed the averaged gradients.  Skipped below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import adafactor_gpu_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_adafactor_ddp_replicas_and_averaged_gradient(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_ddp, size=world, backend="b200", join_timeout_s=600)
