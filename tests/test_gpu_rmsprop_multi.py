"""``DistributedDataParallel`` + ``FlatRMSprop`` on ``backend="b200"`` with real GPUs: the RMSprop instances of the sharded
kernel across NVLink through the public API, with and without overlap, fp32 and bf16 buckets, with momentum and centered;
fp32 parameters and state bit-identical to ``sharded=False`` on the two-shot all-reduce, identical replicas, and a checkpoint
round trip through ``named_state`` across sharded and unsharded runs.  Skipped below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import rmsprop_gpu_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_rmsprop_ddp_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_sharded_ddp, size=world, backend="b200", join_timeout_s=600)
