"""``FlatSGD(sharded=True)`` on gloo CPU ranks: the plumbing of the sharded optimizer (hooks, the ``step()`` contract, memory
layout, checkpoints) with torch ops in place of the peer-memory kernel.  Workers in tests/sharded_optim_workers.py."""
import pytest

import dist_tuto.pth_b200 as b2
import sharded_optim_workers as W

pytestmark = pytest.mark.timeout(240)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=200)


@pytest.mark.parametrize("size", [2, 3])
def test_sharded_is_bit_identical_to_unsharded_and_checkpoints_cross(size):
    go(W.w_sharded_equals_unsharded, size)


@pytest.mark.parametrize("size", [2, 3])
def test_step_contract_and_refusals(size):
    go(W.w_contract, size)


def test_named_momentum_crosses_world_sizes_2_to_3(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_SHARDED_CKPT", str(tmp_path / "sharded.pt"))
    go(W.w_save_named, 2)
    go(W.w_load_named, 3)


def test_world_size_1_is_the_unsharded_path():
    W.w_world1(0, 1)
