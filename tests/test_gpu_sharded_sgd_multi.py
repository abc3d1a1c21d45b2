"""``DistributedDataParallel`` + ``FlatSGD(sharded=True)`` on ``backend="b200"`` with real GPUs: the sharded_sgd kernel across
NVLink through the public API, with and without overlap, fp32 and bf16 buckets, 10 steps; fp32 parameters bit-identical to
``sharded=False`` on the two-shot all-reduce, identical replicas, checkpoint round trip.  World 1 on one GPU."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import sharded_sgd_gpu_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def go(fn, size):
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


def test_world_one_is_the_unsharded_path():
    go(W.w_world1, 1)


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_ddp_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    go(W.w_sharded_ddp, world)
