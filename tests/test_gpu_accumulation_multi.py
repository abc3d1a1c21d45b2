"""Gradient accumulation with ``no_sync()`` on ``backend="b200"`` with real GPUs and overlap on: sharded and unsharded
optimizers against the reference and across ranks, and the exchange kernels once per bucket per optimizer step (a
torch.profiler count).  Skipped below two GPUs."""
import pytest
import torch

import accumulation_workers as W
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_accumulation_across_ranks(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    b2.launch(W.w_gpu_multi, size=world, backend="b200", join_timeout_s=800)
