"""``FlatAdafactor`` on gloo CPU ranks (worlds 1-3): bit for bit ``torch.optim.Adafactor(foreach=False)``, parameters and
state, on a model with every shape class (0-D, 1-D, R == 1, C == 1, 3-D, a channels_last conv weight), with parameter
groups, the lr schedule, clipping, ``no_sync()`` accumulation and ``torch.amp.GradScaler("cpu")`` with inf and NaN overflows on
one rank; ``FlatEMA``; checkpoints from world 2 to 3 and into and out of ``torch.optim.Adafactor``; the argument checks and
refusals; and examples/train_ddp.py with ``--optimizer adafactor``.  Workers in tests/adafactor_workers.py."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import adafactor_workers as W
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200 import FlatAdafactor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=240)


@pytest.mark.parametrize("size", [1, 2, 3])
def test_bit_for_bit_torch_adafactor(size):
    go(W.w_all_cases, size)


@pytest.mark.parametrize("size", [1, 2])
def test_ema_over_adafactor(size):
    go(W.w_ema, size)


def test_checkpoint_crosses_world_sizes_2_to_3(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_ADAFACTOR_CKPT", str(tmp_path / "adafactor.pt"))
    go(W.w_save, 2)
    go(W.w_load, 3)


def test_named_state_into_torch_adafactor_and_back():
    go(W.w_torch_round_trip, 2)


def _net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Linear(5, 4), nn.Tanh(), nn.Linear(4, 3))


@pytest.mark.parametrize("kw, msg", [
    (dict(lr=-1.0), "Learning rate should be >= 0 but is: -1.0"),
    (dict(beta2_decay=0.5), "beta2_decay should be <= 0 but is: 0.5"),
    (dict(eps=(-1.0, 1e-3)), "epsilon1 should be >= 0 but is: -1.0"),
    (dict(eps=(None, -1.0)), "epsilon2 should be >= 0 but is: -1.0"),
    (dict(d=0.5), "Clipping threshold d should be >= 1 but is: 0.5"),
    (dict(weight_decay=-0.1), "weight_decay should be >= 0 but is: -0.1"),
    (dict(sharded=True), "cannot be sharded"),
    (dict(max_grad_norm=0.0), "max_grad_norm"),
])
def test_argument_checks_are_torchs(kw, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        FlatAdafactor(_net(), **kw)
    if "sharded" not in kw and "max_grad_norm" not in kw:
        with pytest.raises(ValueError, match=re.escape(msg)):
            torch.optim.Adafactor(_net().parameters(), **kw)


@pytest.mark.parametrize("extra", ["maximize", "foreach", "capturable", "differentiable"])
def test_torch_extras_are_not_taken(extra):
    with pytest.raises(TypeError):
        FlatAdafactor(_net(), **{extra: False})


def test_group_checks():
    net = _net()
    with pytest.raises(ValueError, match="weight_decay should be >= 0"):
        FlatAdafactor(net, param_groups=[{"params": [net[0].weight], "weight_decay": -1.0}])
    with pytest.raises(ValueError, match="has the key 'd'"):
        FlatAdafactor(_net(), param_groups=[{"params": [net[0].weight], "d": 2.0}])


def test_state_layout_and_checkpoint_forms():
    """The state flat holds R + C floats per slice of a factored tensor and numel for the others; state_dict round-trips;
    load_named_state refuses an entry of another number of dimensions."""
    net = _net()
    opt = FlatAdafactor(net, lr=1e-2)
    assert sum(f.numel() for f in opt.state_flats) == (4 + 5) + 4 + (3 + 4) + 3
    x = torch.randn(2, 5)
    net(x).sum().backward()
    opt.step()
    sd = opt.state_dict()
    other = FlatAdafactor(_net(), lr=0.5)
    other.load_state_dict(sd)
    assert other.lr == 1e-2 and other.steps == 1 and all(torch.equal(a, b) for a, b in zip(other.state_flats, opt.state_flats))
    named = opt.named_state(net)
    assert set(named["0.weight"]) == {"step", "row_var", "col_var"} and named["0.weight"]["row_var"].shape == (4, 1)
    assert named["0.weight"]["col_var"].shape == (1, 5) and set(named["0.bias"]) == {"step", "variance"}
    bad = dict(named, **{"0.weight": {"step": named["0.weight"]["step"], "variance": torch.zeros(4, 5)}})
    fresh = _net()
    with pytest.raises(ValueError, match="row_var"):
        FlatAdafactor(fresh).load_named_state(fresh, bad)


def _example(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_ddp.py"), "--size", "2", "--steps", "3",
                           *args], capture_output=True, text=True, timeout=240, cwd=ROOT)


def test_example_trains_with_adafactor():
    r = _example("--optimizer", "adafactor", "--amp", "--accumulation-steps", "2", "--ema-decay", "0.9",
                 "--no-decay-bias-norm")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "Adafactor state elements on this rank" in r.stdout and "EMA model" in r.stdout and "loss scale" in r.stdout


@pytest.mark.parametrize("flag, msg", [("--sharded-optimizer", "cannot be sharded"), ("--cuda-graph", "no capturable form")])
def test_example_refuses_sharded_and_cuda_graph(flag, msg):
    r = _example("--optimizer", "adafactor", flag)
    assert r.returncode == 2 and msg in r.stderr, r.stderr[-2000:]
