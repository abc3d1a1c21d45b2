"""``FlatAdamW`` on gloo CPU ranks (worlds 2 and 3): bit for bit ``torch.optim.AdamW(foreach=False)`` unsharded, the sharded
plumbing with torch ops in place of the peer-memory kernel, checkpoints across modes and world sizes, and
examples/train_ddp.py with ``--optimizer adamw``.  Workers in tests/adamw_optim_workers.py."""
import os
import re
import subprocess
import sys

import pytest

import dist_tuto.pth_b200 as b2
import adamw_optim_workers as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=240)


@pytest.mark.parametrize("size", [2, 3])
def test_unsharded_is_bit_for_bit_torch_adamw(size):
    go(W.w_bit_equal_to_torch, size)


def test_named_state_loads_into_torch_adamw_and_back():
    go(W.w_named_state_round_trip, 2)


@pytest.mark.parametrize("size", [2, 3])
def test_sharded_agrees_with_unsharded_and_checkpoints_cross_modes(size):
    go(W.w_sharded, size)


@pytest.mark.parametrize("size", [2, 3])
def test_step_contract_and_refusals(size):
    go(W.w_contract, size)


def test_checkpoint_crosses_world_sizes_2_to_3(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_ADAMW_CKPT", str(tmp_path / "adamw.pt"))
    go(W.w_save, 2)
    go(W.w_load, 3)


def test_world_size_1_is_the_unsharded_path():
    W.w_world1(0, 1)


@pytest.mark.parametrize("sharded", [False, True])
def test_example_train_ddp_with_adamw(sharded):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "6", "--optimizer", "adamw"] + (["--sharded-optimizer"] if sharded else [])
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 6: loss ([0-9.]+) \(mean over ranks [0-9.]+\), AdamW moment elements on this rank (\d+)", p.stdout)
    assert sorted(r for r, *_ in lines) == ["0", "1"], p.stdout
    assert all(0.5 < float(loss) < 5.0 for _, loss, _ in lines)
