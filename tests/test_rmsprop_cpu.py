"""``FlatRMSprop`` on gloo CPU ranks (worlds 1-3): bit for bit ``torch.optim.RMSprop(foreach=False)`` over every option
combination, parameter groups, the lr schedule, clipping, ``no_sync()`` accumulation and ``torch.amp.GradScaler("cpu")`` with
inf and NaN overflows on one rank; the sharded torch-op path; ``FlatEMA``; checkpoints across modes and from world 2 to 3;
the per-name state through ``torch.optim.RMSprop``; the argument checks; and examples/train_ddp.py with
``--optimizer rmsprop``.  Workers in tests/rmsprop_workers.py."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
import rmsprop_workers as W
from dist_tuto.pth_b200 import FlatRMSprop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=240)


@pytest.mark.parametrize("size", [1, 2, 3])
def test_bit_for_bit_torch_rmsprop(size):
    """Every case of rmsprop_workers.CASES at this world size."""
    go(W.w_all_cases, size)


@pytest.mark.parametrize("size", [2, 3])
def test_ema_over_rmsprop(size):
    go(W.w_ema, size)


@pytest.mark.parametrize("size", [2, 3])
def test_checkpoints_across_sharded_and_unsharded(size):
    go(W.w_checkpoints, size)


def test_named_state_loads_into_torch_rmsprop_and_back():
    go(W.w_named_state_round_trip, 2)


def test_checkpoint_crosses_world_sizes_2_to_3(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_RMSPROP_CKPT", str(tmp_path / "rmsprop.pt"))
    go(W.w_save, 2)
    go(W.w_load, 3)


@pytest.mark.parametrize("size", [2, 3])
def test_sharded_refusals(size):
    go(W.w_contract, size)


def _net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Linear(5, 4), nn.Tanh(), nn.Linear(4, 3))


@pytest.mark.parametrize("kw,msg", [(dict(lr=-1.0), "Invalid learning rate: -1.0"), (dict(eps=-1e-8), "Invalid epsilon value"),
                                    (dict(momentum=-0.1), "Invalid momentum value: -0.1"),
                                    (dict(weight_decay=-0.1), "Invalid weight_decay value: -0.1"),
                                    (dict(alpha=-0.5), "Invalid alpha value: -0.5")])
def test_argument_checks_are_torch_s(kw, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        FlatRMSprop(_net(), **kw)
    with pytest.raises(ValueError, match=re.escape(msg)):           # torch's own message, word for word
        torch.optim.RMSprop(_net().parameters(), **kw)


@pytest.mark.parametrize("kw", [dict(maximize=True), dict(differentiable=True), dict(foreach=True)])
def test_options_that_are_not_taken(kw):
    with pytest.raises(TypeError):
        FlatRMSprop(_net(), **kw)


def test_group_and_mode_refusals():
    net = _net()
    with pytest.raises(ValueError, match="sets only 'lr' and 'weight_decay'"):
        FlatRMSprop(net, param_groups=[{"params": [net[0].weight], "momentum": 0.5}])
    net = _net()
    with pytest.raises(ValueError, match="Invalid weight_decay value"):
        FlatRMSprop(net, param_groups=[{"params": [net[0].weight], "weight_decay": -1.0}])
    with pytest.raises(ValueError, match="CUDA parameters"):
        FlatRMSprop(_net(), capturable=True)


def test_state_flats_follow_the_options():
    for mu, centered in ((0.0, False), (0.9, False), (0.0, True), (0.9, True)):
        opt = FlatRMSprop(_net(), momentum=mu, centered=centered)
        assert len(opt.square_avg_flats) == 1
        assert len(opt.momentum_buffer_flats) == (1 if mu > 0 else 0) and len(opt.grad_avg_flats) == (1 if centered else 0)
        assert set(opt.state_dict()) >= {"square_avg", "momentum_buffer", "grad_avg", "alpha", "centered", "momentum"}


def _example(*extra):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "6", "--optimizer", "rmsprop", *extra]
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 6: loss ([0-9.]+) \(mean over ranks ([0-9.]+)\), RMSprop state elements on this rank "
                       r"(\d+)", p.stdout)
    assert sorted(r for r, *_ in lines) == ["0", "1"], p.stdout
    return {int(r): (loss, mean, int(n)) for r, loss, mean, n in lines}, p.stdout


def test_example_train_ddp_with_rmsprop_sharded_prints_the_same_losses():
    plain, _ = _example()
    sharded, _ = _example("--sharded-optimizer")
    for r in (0, 1):
        assert plain[r][:2] == sharded[r][:2]                        # the printed losses, digit for digit
        assert 0.5 < float(plain[r][0]) < 5.0
        assert plain[r][2] // 2 <= sharded[r][2] <= plain[r][2] // 2 + 128   # half the state (+ padding) per rank


def test_example_train_ddp_with_rmsprop_and_the_other_options():
    _, out = _example("--no-decay-bias-norm", "--accumulation-steps", "2", "--ema-decay", "0.9", "--amp")
    assert re.search(r"Rank 0, EMA model: held-out loss [0-9.]+", out) and re.search(r"Rank 0, loss scale", out), out
