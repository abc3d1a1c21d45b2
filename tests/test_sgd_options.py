"""CPU tier: weight decay and Nesterov momentum -- FlatSGD against torch.optim.SGD bit for bit, the validation every
engine shares, a resumed train() run, the example's flags, and the exact fp32 fma of the kernels' model."""
import os
import random
import re
import struct
import subprocess
import sys
from fractions import Fraction

import pytest
import torch

import dist_tuto.pth_b200 as b2
import sgd_options_model as SM
from dist_tuto.pth_b200 import LRSchedule
from dist_tuto.pth_b200.ops.optim import FlatSGD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f32(x):
    return struct.unpack("f", struct.pack("f", x))[0]


def _net():
    return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))


@pytest.mark.parametrize("nesterov", [False, True], ids=["momentum", "nesterov"])
@pytest.mark.parametrize("wd", [0.0, 1e-2], ids=["wd0", "wd1e-2"])
@pytest.mark.parametrize("sched", [None, LRSchedule(warmup_steps=5, decay="multistep", milestones=[12], gamma=0.5)],
                         ids=["const", "schedule"])
def test_flat_sgd_equals_torch_sgd_bit_for_bit(wd, nesterov, sched):
    torch.manual_seed(0)
    ref, mine = _net(), _net()
    mine.load_state_dict(ref.state_dict())
    opt_ref = torch.optim.SGD(ref.parameters(), lr=0.2, momentum=0.5, weight_decay=wd, nesterov=nesterov, foreach=False)
    opt = FlatSGD(mine, lr=0.2, momentum=0.5, weight_decay=wd, nesterov=nesterov, lr_schedule=sched)
    x, y = torch.randn(20, 8, 6), torch.randn(20, 8, 3)
    for k in range(20):
        for grp in opt_ref.param_groups:
            grp["lr"] = 0.2 if sched is None else sched.lr_at(0.2, k)
        for m, o in ((ref, opt_ref), (mine, opt)):
            ((m(x[k]) - y[k]) ** 2).mean().backward()
            o.step()
            o.zero_grad()
        for (n, a), b in zip(ref.named_parameters(), mine.parameters()):
            assert torch.equal(a.detach(), b.detach()), (k, n)
    sd = opt.state_dict()
    assert sd["nesterov"] is nesterov and sd["weight_decay"] == wd


def test_flat_sgd_loads_checkpoints_written_without_nesterov():
    opt = FlatSGD(_net(), lr=0.1, momentum=0.5, nesterov=True)
    sd = opt.state_dict()
    del sd["nesterov"]
    opt.load_state_dict(sd)
    assert opt.nesterov is False
    sd["nesterov"] = True
    opt.load_state_dict(sd)
    assert opt.nesterov is True


def test_negative_weight_decay_and_nesterov_without_momentum_are_refused():
    with pytest.raises(ValueError, match="weight_decay"):
        b2.TrainConfig(weight_decay=-1e-4)
    with pytest.raises(ValueError, match="nesterov"):
        b2.TrainConfig(momentum=0.0, nesterov=True)
    with pytest.raises(ValueError, match="weight_decay"):
        FlatSGD(_net(), weight_decay=-0.5)
    with pytest.raises(ValueError, match="nesterov"):
        FlatSGD(_net(), momentum=0.0, nesterov=True)
    # the trainers check before they touch the extension or a device
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    for cls in (FusedTrainer, BatchedTrainer):
        with pytest.raises(ValueError, match="weight_decay"):
            cls(128, weight_decay=-1e-3)
        with pytest.raises(ValueError, match="nesterov"):
            cls(128, momentum=0.0, nesterov=True)
    cfg = b2.TrainConfig(weight_decay=5e-4, nesterov=True)
    assert (cfg.weight_decay, cfg.nesterov) == (5e-4, True)
    assert (b2.TrainConfig().weight_decay, b2.TrainConfig().nesterov) == (0.0, False)


class _Stop(Exception):
    pass


def test_train_torch_engine_resumed_with_both_options_is_bit_equal(tmp_path, monkeypatch):
    """train(engine="torch") with weight decay and Nesterov: a run stopped after its first in-progress checkpoint and
    resumed from it ends with the parameters of the uninterrupted run.  Dropout is off (the torch engine does not
    checkpoint the host RNG of its masks) and each epoch's shuffle is seeded by the epoch index, as the native loader does."""
    from dist_tuto.pth_b200.data import BatchLoader, SyntheticMNIST
    it = BatchLoader.__iter__

    def epoch_seeded_iter(self):
        self._gen.manual_seed(1000 + self._epoch)
        self._epoch += 1
        return it(self)
    monkeypatch.setattr(BatchLoader, "_epoch", 0, raising=False)
    monkeypatch.setattr(BatchLoader, "__iter__", epoch_seeded_iter)
    ds = SyntheticMNIST(n=512, seed=5)

    def cfg(**kw):
        return b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0, weight_decay=1e-2,
                              nesterov=True, log=kw.pop("log", lambda *a: None), **kw)
    whole = b2.train(0, 1, cfg())
    assert whole["steps"] == 12
    plain = b2.train(0, 1, b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0,
                                          log=lambda *a: None))
    assert any(not torch.equal(a, b) for a, b in zip(whole["model"].parameters(), plain["model"].parameters()))
    ck = str(tmp_path / "run.pt")

    def stop_in_epoch_1(*a):
        if a[:4] == ("Rank ", 0, ", epoch ", 1):
            raise _Stop()
    with pytest.raises(_Stop):
        b2.train(0, 1, cfg(checkpoint=ck, checkpoint_every=1, log=stop_in_epoch_1))
    blob = torch.load(ck, map_location="cpu")
    assert blob["in_progress"] and blob["epoch"] == 1 and blob["steps"] == 4
    assert blob["optim"]["nesterov"] is True and blob["optim"]["weight_decay"] == 1e-2
    resumed = b2.train(0, 1, cfg(resume=ck))
    assert resumed["steps"] == 8
    for (n, a), (_, b) in zip(whole["model"].named_parameters(), resumed["model"].named_parameters()):
        assert torch.equal(a.detach(), b.detach()), n


def test_train_mnist_example_passes_weight_decay_and_nesterov_through(tmp_path):
    """The flags reach TrainConfig: the run records them in its FlatSGD checkpoint."""
    ck = str(tmp_path / "ex.pt")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--size", "1", "--epochs", "1",
                        "--max-steps", "4", "--weight-decay", "1e-3", "--nesterov", "--checkpoint", ck],
                       capture_output=True, text=True, timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    assert re.search(r"Rank\s+0\s*, epoch\s+0\s*:", p.stdout), p.stdout
    optim = torch.load(ck, map_location="cpu")["optim"]
    assert optim["weight_decay"] == 1e-3 and optim["nesterov"] is True and optim["steps"] == 4
    q = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--help"], capture_output=True,
                       text=True, timeout=120, env=env, cwd=ROOT)
    assert "--weight-decay" in q.stdout and "--nesterov" in q.stdout


# ------------------------------------------------------------------------------------------------ the kernels' model
def test_fma32_is_the_correctly_rounded_fp32_fma():
    rnd = random.Random(7)
    a, b, c = [], [], []
    for _ in range(3000):
        a.append(_f32(rnd.uniform(-2, 2) * 2.0 ** rnd.randint(-12, 12)))
        b.append(_f32(rnd.uniform(-2, 2) * 2.0 ** rnd.randint(-12, 12)))
        c.append(_f32(rnd.uniform(-2, 2) * 2.0 ** rnd.randint(-30, 12)))
    # a sum just above the halfway point between two fp32 values: fp64 rounding lands on the midpoint, and rounding that
    # again to fp32 goes to the even neighbour -- the wrong one
    a.append(-(2.0 ** -24) * (1 - 2.0 ** -18)); b.append(1 + 2.0 ** -18); c.append(1 + 2.0 ** -23)
    got = SM.fma32(torch.tensor(a), torch.tensor(b), torch.tensor(c)).tolist()
    for x, y, z, g in zip(a, b, c, got):
        want = SM.round_f32(Fraction(x) * Fraction(y) + Fraction(z))
        assert g == want, (x, y, z, g, want)
    naive = float((torch.tensor(a[-1:]).double() * torch.tensor(b[-1:]).double() + torch.tensor(c[-1:]).double()).float())
    assert naive != got[-1] == 1 + 2.0 ** -23


def test_sgd_update_model_matches_torch_sgd_in_fp64_closely():
    g = torch.Generator().manual_seed(3)
    p = torch.randn(4096, generator=g)
    m = torch.zeros_like(p)
    grads = [torch.randn(4096, generator=g) for _ in range(6)]
    for wd in (0.0, 1e-2):
        for nest in (False, True):
            pp, mm = p.clone(), m.clone()
            for gr in grads:
                pp, mm = SM.sgd_update(gr, pp, mm, 0.5, 0.05, wd, nest)
            ref = SM.torch_sgd_fp64(p, grads, [0.05] * 6, 0.5, wd, nest)
            assert torch.allclose(pp.double(), ref, rtol=1e-5, atol=1e-6), (wd, nest)
