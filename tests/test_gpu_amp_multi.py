"""fp16 loss scaling on two or more GPUs (backend b200): an overflow on one rank makes every rank skip, and the replicas stay
bit-identical, eager and captured.  Worker in tests/amp_workers.py."""
import pytest
import torch

import amp_workers as W
import dist_tuto.pth_b200 as b2

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                                                  reason="needs two or more GPUs")]


def test_overflow_on_one_rank_skips_every_rank():
    b2.launch(W.w_gpu_multi, size=min(torch.cuda.device_count(), 4), backend="b200", join_timeout_s=800)
