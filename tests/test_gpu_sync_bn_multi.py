"""``SyncBatchNorm`` across real GPUs on ``backend="b200"`` (the peer-memory exchange): against ``torch.nn.SyncBatchNorm`` on
NCCL within tolerance, replica buffers bit-identical.  Skips below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import sync_bn_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 8])
def test_against_torch_sync_batch_norm(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_against_torch_on_gpus, size=world, backend="b200", join_timeout_s=600)
