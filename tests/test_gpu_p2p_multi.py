"""``comm.send`` / ``recv`` / ``isend`` / ``irecv`` on ``backend="b200"`` across GPUs: the peer-memory kernels through the
public API, never NCCL.  Skipped below 2 GPUs."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import p2p_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


def go(fn, size):
    if torch.cuda.device_count() < size:
        pytest.skip(f"needs {size} GPUs")
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


def test_pingpong_at_every_benchmark_size():
    go(W.w_pingpong, 2)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ring_and_all_pairs_exchange(world):
    go(W.w_ring_and_all_pairs, world)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_ring_allreduce_equals_nccl(world):
    go(W.w_ring_allreduce_vs_nccl, world)
