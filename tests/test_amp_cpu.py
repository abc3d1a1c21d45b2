"""fp16 loss scaling with ``torch.amp.GradScaler("cpu")`` on gloo CPU ranks (worlds 1 to 3): FlatSGD and FlatAdamW bit for
bit against torch's optimizers with their own scaler through overflows on one rank, FlatLAMB / FlatLARS against themselves
fed the unscaled gradient, the sharded refusal, and ``examples/train_ddp.py --amp``.  Workers in tests/amp_workers.py."""
import os
import re
import subprocess
import sys

import pytest
import torch

import amp_workers as W
from accumulation_workers import Net
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatLAMB, FlatLARS, FlatSGD

pytestmark = pytest.mark.timeout(900)


@pytest.mark.parametrize("size", [1, 2, 3])
def test_scaled_steps_equal_torch_with_its_scaler(size):
    b2.launch(W.w_all, size=size, backend="gloo", join_timeout_s=840)


@pytest.mark.parametrize("cls", [FlatSGD, FlatAdamW, FlatLAMB, FlatLARS])
def test_gradscaler_contract(cls):
    """The flag GradScaler looks for, one parameter group per torch's layout, and attributes deleted after the step."""
    net = Net()
    opt = cls(net, lr=0.01)
    assert opt._step_supports_amp_scaling
    assert sum(len(g["params"]) for g in opt.param_groups) == len(list(net.parameters()))
    assert all({"params", "lr", "weight_decay"} <= set(g) for g in opt.param_groups)
    scaler = torch.amp.GradScaler("cpu", init_scale=1000.0)
    scaler.scale(W._loss(net, 0, 0, 0, 1) * float("inf")).backward()
    scaler.step(opt)
    scaler.update()
    assert opt.steps == 0 and scaler.get_scale() == 500.0
    assert not hasattr(opt, "grad_scale") and not hasattr(opt, "found_inf")
    scaler.scale(W._loss(net, 0, 0, 0, 1)).backward()
    scaler.step(opt)
    assert opt.steps == 1


def test_layerwise_param_groups_follow_lr():
    net = Net()
    opt = FlatLAMB(net, lr=0.01, weight_decay=0.1)
    opt.param_groups[0]["lr"] = 0.5
    assert opt.lr == 0.5 and opt.scalars()[6] == 0.5
    opt.weight_decay = 0.2
    assert opt.param_groups[0]["weight_decay"] == 0.2


@pytest.mark.parametrize("optimizer", ["sgd", "adamw", "lamb", "lars"])
def test_example_train_ddp_amp(optimizer):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "4", "--optimizer", optimizer, "--amp", "--accumulation-steps", "2", "--ema-decay", "0.9"]
    p = subprocess.run([sys.executable, os.path.join(root, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=root)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 4: loss ([0-9.]+)", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"] and all(0.1 < float(x) < 5.0 for _, x in lines), p.stdout
    scales = re.findall(r"Rank (\d), loss scale ([0-9.e+]+), updates applied (\d+) of 4", p.stdout)
    assert len(scales) == 2 and len({(s, a) for _, s, a in scales}) == 1, p.stdout


def test_example_refuses_amp_with_sharded_optimizer():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "examples", "train_ddp.py"), "--amp", "--sharded-optimizer"],
                       capture_output=True, text=True, timeout=120, cwd=root)
    assert p.returncode == 2 and "--amp needs an unsharded optimizer" in p.stderr, p.stderr
