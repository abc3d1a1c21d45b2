"""LRSchedule on the CPU tier: the closed form against torch.optim.lr_scheduler, validation, epoch units, FlatSGD with a
schedule, train(engine="torch") resumed mid-warmup over gloo, and the example's schedule flags."""
import os
import re
import subprocess
import sys
import warnings

import pytest
import torch
from torch.optim.lr_scheduler import ConstantLR, CosineAnnealingLR, LinearLR, MultiStepLR, SequentialLR

import dist_tuto.pth_b200 as b2
import lr_workers as W
from dist_tuto.pth_b200 import LRSchedule
from dist_tuto.pth_b200.ops.optim import FlatSGD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def _torch_lrs(schedule, base, n, params=None):
    """lr of updates 0..n-1 from SequentialLR(LinearLR, <decay>) -- torch counts the decay from the end of the warmup."""
    p = params if params is not None else [torch.nn.Parameter(torch.zeros(1))]
    opt = torch.optim.SGD(p, lr=base)
    W_ = int(schedule.warmup_steps)
    if schedule.decay == "multistep":
        decay = MultiStepLR(opt, [int(m) - W_ for m in schedule.milestones], gamma=schedule.gamma)
    elif schedule.decay == "cosine":
        decay = CosineAnnealingLR(opt, int(schedule.total_steps) - W_, eta_min=base * schedule.min_factor)
    else:
        decay = ConstantLR(opt, factor=1.0, total_iters=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sched = SequentialLR(opt, [LinearLR(opt, schedule.warmup_start, 1.0, W_), decay], [W_]) if W_ else decay
        out = []
        for _ in range(n):
            out.append(opt.param_groups[0]["lr"])
            opt.step()
            sched.step()
    return opt, sched, out


CONFIGS = [
    dict(warmup_steps=10),
    dict(warmup_steps=25, warmup_start=0.1),
    dict(warmup_steps=10, decay="multistep", milestones=[40, 120, 200], gamma=0.3),
    dict(warmup_steps=0, decay="multistep", milestones=[1, 2, 150], gamma=0.5),
    dict(warmup_steps=10, decay="cosine", total_steps=310, min_factor=0.05),
    dict(warmup_steps=30, warmup_start=0.5, decay="cosine", total_steps=400),
    dict(warmup_steps=0, decay="cosine", total_steps=300, min_factor=0.2),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_schedule_matches_torch_lr_schedulers(cfg):
    s = LRSchedule(**cfg)
    base = 0.32
    _, _, want = _torch_lrs(s, base, 300)
    for k, w in enumerate(want):
        got = s.lr_at(base, k)
        assert abs(got - w) <= 1e-6 * w, (k, got, w)


def test_cosine_stays_at_min_factor_after_total_steps():
    s = LRSchedule(warmup_steps=5, decay="cosine", total_steps=50, min_factor=0.1)
    assert s.factor(50) == s.factor(51) == s.factor(10 ** 6)
    assert abs(s.factor(50) - 0.1) < 1e-15 and s.factor(5) == 1.0


def test_lr_is_one_fp32_rounding_of_an_fp64_product():
    s = LRSchedule(warmup_steps=3, warmup_start=0.25)
    import struct
    f32 = lambda x: struct.unpack("f", struct.pack("f", x))[0]   # noqa: E731
    for k in range(5):
        assert s.lr_at(0.01, k) == f32(f32(0.01) * s.factor(k))
    assert LRSchedule().lr_at(0.01, 7) == f32(0.01)               # constant: the fp32 base lr


@pytest.mark.parametrize("kw", [
    dict(warmup_steps=-1), dict(warmup_steps=2.5), dict(warmup_start=0.0), dict(warmup_start=1.5),
    dict(decay="linear"), dict(unit="batch"),
    dict(decay="multistep", milestones=[5, 3]), dict(decay="multistep", milestones=list(range(9))),
    dict(decay="multistep", milestones=[-1]), dict(decay="multistep", milestones=[3], gamma=0.0),
    dict(decay="multistep", milestones=[3], gamma=1.5), dict(milestones=[3]),
    dict(decay="cosine"), dict(warmup_steps=10, decay="cosine", total_steps=10),
    dict(decay="cosine", total_steps=10, min_factor=-0.1), dict(decay="cosine", total_steps=10, min_factor=1.5),
])
def test_invalid_schedules_are_rejected(kw):
    with pytest.raises(ValueError):
        LRSchedule(**kw)


def test_epoch_units_resolve_to_steps():
    s = LRSchedule(warmup_steps=0.5, decay="multistep", milestones=[2, 3.5], gamma=0.5, unit="epoch")
    r = s.resolve(10)
    assert (r.unit, r.warmup_steps, r.milestones) == ("step", 5, (20, 35))
    assert LRSchedule(warmup_steps=1, decay="cosine", total_steps=3, unit="epoch").resolve(7).total_steps == 21
    assert r.resolve(3) is r
    with pytest.raises(ValueError):
        s.lr_at(0.1, 0)                                            # epoch units must be resolved first
    with pytest.raises(ValueError):
        s.resolve(0)
    with pytest.raises(ValueError):
        FlatSGD(torch.nn.Linear(4, 4), lr_schedule=s)               # optimizers and trainers take step units
    with pytest.raises(ValueError):
        b2.TrainConfig(lr_schedule="cosine")


def test_schedule_round_trips_through_dict_and_tuple():
    s = LRSchedule(warmup_steps=4, warmup_start=0.2, decay="multistep", milestones=[10, 20], gamma=0.5)
    assert LRSchedule.from_dict(s.to_dict()) == s
    assert s.as_tuple() == (2, 4, 0, 0.2, 0.5, 0.0, [10, 20])
    c = LRSchedule(warmup_steps=2, decay="cosine", total_steps=9, min_factor=0.1)
    assert c.as_tuple() == (3, 2, 9, 1.0 / 3.0, 0.1, 0.1, [])
    assert LRSchedule().as_tuple()[0] == 1


@pytest.mark.parametrize("cfg", [CONFIGS[2], CONFIGS[5]], ids=["multistep", "cosine"])
def test_flat_sgd_with_schedule_equals_torch_sgd_with_scheduler(cfg):
    cfg = dict(cfg, **({"milestones": [12, 30]} if "milestones" in cfg else {"warmup_steps": 8, "total_steps": 60}))
    s = LRSchedule(**cfg)
    torch.manual_seed(0)
    ref = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))
    mine = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))
    mine.load_state_dict(ref.state_dict())
    opt_ref, sched_ref, _ = _torch_lrs(s, 0.2, 0, list(ref.parameters()))
    for g in opt_ref.param_groups:
        g["momentum"] = 0.5
    opt = FlatSGD(mine, lr=0.2, momentum=0.5, lr_schedule=s)
    x, y = torch.randn(50, 8, 6), torch.randn(50, 8, 3)
    for k in range(50):
        for m, o in ((ref, opt_ref), (mine, opt)):
            loss = ((m(x[k]) - y[k]) ** 2).mean()
            loss.backward()
            o.step()
            o.zero_grad()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sched_ref.step()
        for a, b in zip(ref.parameters(), mine.parameters()):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), k
    assert opt.steps == 50 and opt.state_dict()["steps"] == 50
    fresh = FlatSGD(torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3)), lr=0.2,
                    momentum=0.5, lr_schedule=s)
    fresh.load_state_dict(opt.state_dict())
    assert fresh.steps == 50 and fresh.lr_at() == opt.lr_at() == s.lr_at(0.2, 50)


def test_train_torch_engine_schedule_resumed_mid_warmup_is_bit_equal(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_LR_TEST_DIR", str(tmp_path))
    b2.launch(W.w_torch_engine_schedule_resume, size=2, backend="gloo", join_timeout_s=250)


def test_train_without_schedule_reports_the_constant_lr():
    from dist_tuto.pth_b200.data import SyntheticMNIST
    out = b2.train(0, 1, b2.TrainConfig(epochs=2, max_steps=3, dataset=SyntheticMNIST(n=256, seed=1), engine="torch",
                                        device="cpu", lr=0.02, log=lambda *a: None))
    assert out["lr"] == [0.02, 0.02]


@pytest.mark.parametrize("flags", [
    ["--warmup-epochs", "0.5", "--lr-decay", "cosine", "--lr-min-factor", "0.1"],
    ["--warmup-epochs", "0.25", "--warmup-start", "0.5", "--lr-decay", "multistep", "--lr-milestones", "0.5", "--lr-gamma", "0.5"],
])
def test_train_mnist_example_schedule_flags(flags):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--size", "2", "--epochs", "1",
                        "--max-steps", "6"] + flags, capture_output=True, text=True, timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank\s+(\d)\s*, epoch\s+0\s*:\s+([0-9.]+)", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"] and all(0.5 < float(v) < 5.0 for _, v in lines)
