"""``DistributedDataParallel`` + sharded ``FlatLAMB`` / ``FlatLARS`` on ``backend="b200"`` with real GPUs: sharded against
unsharded, replicas and trust ratios identical on every rank, no host synchronisation, ``no_sync()`` with ``FlatEMA`` and a
checkpoint into an unsharded optimizer.  Skipped below two GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import sharded_layerwise_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_lamb_and_lars_ddp(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_multi, size=world, backend="b200", join_timeout_s=600)
