"""Gradient accumulation with ``DistributedDataParallel.no_sync()`` on gloo CPU ranks (worlds 2 and 3): every flat optimizer
and mode against a reference without DDP, the exchange counts, the refusals, and ``examples/train_ddp.py
--accumulation-steps``.  Workers in tests/accumulation_workers.py."""
import os
import re
import subprocess
import sys

import pytest

import accumulation_workers as W
import dist_tuto.pth_b200 as b2

pytestmark = pytest.mark.timeout(600)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=540)


@pytest.mark.parametrize("size", [2, 3])
def test_accumulated_cycles_equal_the_reference(size):
    go(W.w_against_reference, size)


@pytest.mark.parametrize("size", [2, 3])
def test_refusals_exchange_nothing(size):
    go(W.w_errors, size)


def test_no_sync_at_world_one_and_its_flag():
    """One process, no process group needed: the flag nests and restores, and the guards hold at world size 1."""
    net = W.Net()
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=600)
    opt = b2.FlatSGD(ddp, lr=0.1, momentum=0.9)
    assert ddp.require_backward_grad_sync
    with ddp.no_sync():
        with ddp.no_sync():
            W._loss(ddp, 0, 0, 0, 2).backward()
        assert not ddp.require_backward_grad_sync
        with pytest.raises(RuntimeError, match="inside no_sync"):
            b2.average_gradients(net)
    assert ddp.require_backward_grad_sync
    with pytest.raises(RuntimeError, match="never exchanged"):
        opt.step()
    assert opt.steps == 0
    W._loss(ddp, 0, 0, 1, 2).backward()
    b2.average_gradients(ddp)
    opt.step()
    assert opt.steps == 1
    ddp.zero_grad()                       # zeroing the buckets also forgets an unexchanged accumulation
    with ddp.no_sync():
        W._loss(ddp, 0, 1, 0, 2).backward()
    ddp.zero_grad()
    opt.step()
    with ddp.no_sync():                   # an exception inside the context restores the flag
        with pytest.raises(ValueError):
            raise ValueError
    assert ddp.require_backward_grad_sync
    ddp.remove_hooks()


@pytest.mark.parametrize("optimizer,sharded", [("sgd", False), ("adamw", False), ("lamb", False), ("lars", False),
                                               ("sgd", True), ("adamw", True)])
def test_example_train_ddp_accumulates(optimizer, sharded):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "4", "--optimizer", optimizer, "--accumulation-steps", "2"]
    if sharded:
        args.append("--sharded-optimizer")
    p = subprocess.run([sys.executable, os.path.join(root, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=root)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 4: loss ([0-9.]+)", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"] and all(0.1 < float(x) < 5.0 for _, x in lines), p.stdout
