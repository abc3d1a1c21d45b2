"""``FlatLAMB`` and ``FlatLARS`` on gloo CPU ranks (worlds 2 and 3): bit for bit the per-parameter torch-op reference,
replicas bit-identical, checkpoints across FlatAdamW / FlatSGD, the refusals, and examples/train_ddp.py with
``--optimizer lamb`` / ``lars``.  Workers in tests/layerwise_workers.py."""
import os
import re
import subprocess
import sys

import pytest

import dist_tuto.pth_b200 as b2
import layerwise_workers as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=240)


@pytest.mark.parametrize("size", [2, 3])
def test_bit_equal_to_the_torch_op_reference(size):
    go(W.w_bit_equal, size)


def test_checkpoints_round_trip_and_cross_to_adamw_and_sgd(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_LW_CKPT_DIR", str(tmp_path))
    go(W.w_checkpoints, 2)


@pytest.mark.parametrize("size", [2, 3])
def test_refusals(size):
    go(W.w_refusals, size)


@pytest.mark.parametrize("optimizer", ["lamb", "lars"])
def test_example_train_ddp(optimizer):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_ddp.py"), "--size", "2", "--steps", "6",
                        "--optimizer", optimizer], capture_output=True, text=True, timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 6: loss ([0-9.]+) \(mean over ranks [0-9.]+\), ", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"], p.stdout
    assert all(0.5 < float(loss) < 5.0 for _, loss in lines)
