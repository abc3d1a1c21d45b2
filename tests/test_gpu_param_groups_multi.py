"""``DistributedDataParallel`` + grouped ``FlatSGD`` / ``FlatAdamW`` with ``sharded=True`` on ``backend="b200"`` with real
GPUs: the grouped instances of the sharded kernel across NVLink equal the grouped unsharded kernels bit for bit, with
identical replicas.  Skipped below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import param_groups_gpu_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 8])
def test_sharded_grouped_equals_unsharded_grouped(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_sharded_groups_ddp, size=world, backend="b200", join_timeout_s=600)
