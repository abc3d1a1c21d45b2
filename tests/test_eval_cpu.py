"""Evaluation on the CPU tier: evaluation shards, evaluate(Net on CPU) and train(eval_dataset=...) over gloo, and the
example's --eval flag."""
import os
import re
import subprocess
import sys

import pytest

import dist_tuto.pth_b200 as b2
import eval_workers as W
from dist_tuto.pth_b200.data import partition_eval_dataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


@pytest.mark.parametrize("n", [0, 3, 10000, 10007])
def test_eval_shards_are_contiguous_and_cover_every_sample_once(n):
    data = list(range(n))
    for world in range(1, 9):
        parts = [partition_eval_dataset(data, rank=r, world_size=world) for r in range(world)]
        idx = [list(p.index) for p in parts]
        assert [j for i in idx for j in i] == list(range(n))     # contiguous, disjoint, in rank order, every index once
        sizes = [len(p) for p in parts]
        assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
        assert all(parts[r][k] == idx[r][k] for r in range(world) for k in range(len(idx[r])))


@pytest.mark.parametrize("world", [2, 3])
def test_evaluate_cpu_net_over_ranks_equals_one_process(world):
    b2.launch(W.w_evaluate_cpu_net, size=world, backend="gloo", join_timeout_s=250)


def test_train_torch_engine_with_evaluation_world2():
    b2.launch(W.w_train_torch_with_eval, size=2, backend="gloo", join_timeout_s=250)


def test_train_config_rejects_unknown_eval_settings():
    with pytest.raises(ValueError):
        b2.TrainConfig(eval_dataset="test")
    with pytest.raises(ValueError):
        b2.TrainConfig(eval_dataset="default", eval_every=0)


def test_train_mnist_example_eval_flag():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--size", "2", "--max-steps", "20",
                        "--eval"], capture_output=True, text=True, timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    acc = re.findall(r"Rank\s+(\d)\s*, epoch\s+0\s*: test loss\s+([0-9.]+)\s*, accuracy\s+([0-9.]+)", p.stdout)
    assert sorted(r for r, _, _ in acc) == ["0", "1"], p.stdout
    assert len({(l, a) for _, l, a in acc}) == 1 and 0.0 <= float(acc[0][2]) <= 1.0
