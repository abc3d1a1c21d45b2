"""``comm.batch_isend_irecv`` on ``backend="b200"`` across GPUs: rings and all-pairs exchanges through the peer-memory batch
kernel equal NCCL's own ``batch_isend_irecv`` bit for bit and never reach NCCL's point-to-point; a batch on one side
matches single calls on the other.  Skipped below 2 GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import p2p_batch_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


def go(fn, size):
    if torch.cuda.device_count() < size:
        pytest.skip(f"needs {size} GPUs")
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ring_and_all_pairs_equal_nccl(world):
    go(W.w_ring_and_all_pairs_vs_nccl, world)


def test_a_batch_against_single_calls():
    go(W.w_batch_against_single_calls, 2)
