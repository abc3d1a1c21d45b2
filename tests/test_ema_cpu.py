"""``FlatEMA`` on gloo CPU ranks (worlds 2 and 3): every flat optimizer and mode against ``AveragedModel`` bit for bit,
``average_parameters()``, checkpoints (also from world 2 to world 3), the refusals, and ``examples/train_ddp.py
--ema-decay``.  Workers in tests/ema_workers.py."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch

import dist_tuto.pth_b200 as b2
import ema_workers as W

pytestmark = pytest.mark.timeout(900)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=840)


@pytest.mark.parametrize("size", [2, 3])
def test_ema_equals_averaged_model(size):
    go(W.w_against_reference, size)


@pytest.mark.parametrize("size", [2, 3])
def test_checkpoints_round_trip(size):
    go(W.w_checkpoints, size)


@pytest.mark.parametrize("size", [2, 3])
def test_sharded_exchange_inside_average_parameters_is_refused(size):
    go(W.w_sharded_exchange_refused, size)


def test_model_must_own_the_optimizer_parameters():
    """A plain-module optimizer needs model=; a DDP wrapper is unwrapped once; a module that does not hold the optimizer's
    parameters is refused; an inner attribute called ``module`` is not unwrapped."""
    net = W.Net()
    opt = b2.FlatSGD(net, lr=0.05)
    with pytest.raises(ValueError, match="model="):
        b2.FlatEMA(opt)
    with pytest.raises(ValueError, match="lacks"):
        b2.FlatEMA(opt, model=W.Net())
    ema = b2.FlatEMA(opt, model=net)
    assert ema._buf_names == ["bn.running_mean", "bn.running_var"]

    class Wrapper(torch.nn.Module):                  # a user model with a submodule called "module"
        def __init__(self):
            super().__init__()
            self.module = W.Net()
            self.head_bn = torch.nn.BatchNorm1d(5)

        def forward(self, x):
            return self.head_bn(self.module(x))
    wrapped = Wrapper()
    ddp = b2.DistributedDataParallel(wrapped, bucket_cap_bytes=600)
    ema = b2.FlatEMA(b2.FlatSGD(ddp, lr=0.05))
    assert ema._buf_names == ["module.bn.running_mean", "module.bn.running_var", "head_bn.running_mean",
                              "head_bn.running_var"]
    assert b2.FlatEMA(b2.FlatSGD(ddp, lr=0.05), model=ddp)._buf_names == ema._buf_names
    ddp.remove_hooks()


def test_sharded_ema_moves_from_world_2_to_world_3(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_EMA_CKPT", str(tmp_path / "ema.pt"))
    go(W.w_save_named, 2)
    go(W.w_load_named, 3)


def test_world_one_matches_the_reference_and_sharded_is_unsharded():
    """One process, no process group: sharded=True at world size 1 is the unsharded path."""
    for sharded in (False, True):
        net, ddp, opt, ema = W.build("sgd", dict(lr=0.05, momentum=0.9, sharded=sharded), decay=0.6, every=2, warmup_steps=2)
        ref = W.Net()
        ref.load_state_dict(net.state_dict())
        avg = W.AveragedModel(ref, multi_avg_fn=W.get_ema_multi_avg_fn(0.6), use_buffers=True)
        for it in range(8):
            W.train_step(ddp, opt, 0, it)
            ema.update()
            ref.load_state_dict(net.state_dict())
            if (it + 1) % 2 == 0:
                avg.update_parameters(ref)
                if it + 1 <= 2:
                    avg.n_averaged.fill_(0)
            W.check_against(ema.named_ema(ddp), avg, f"world 1, sharded={sharded}, step {it + 1}")
        assert [e.numel() for e in ema.ema_flats] == [p.numel() for p in opt.param_flats]
        W.check_average_parameters(net, ddp, opt, ema, avg, "world 1", W.batch(0, 999, 0)[0])
        ddp.remove_hooks()


@pytest.mark.parametrize("kw,match", [(dict(decay=-0.1), "decay"), (dict(decay=1.5), "decay"), (dict(decay=math.nan), "decay"),
                                      (dict(decay=math.inf), "decay"), (dict(decay=True), "decay"), (dict(decay="0.9"), "decay"),
                                      (dict(every=0), "every"), (dict(every=1.5), "every"), (dict(every=True), "every"),
                                      (dict(warmup_steps=-1), "warmup_steps"), (dict(warmup_steps=0.5), "warmup_steps")])
def test_bad_settings_are_refused(kw, match):
    net, ddp, opt, _ = W.build("sgd", dict(lr=0.05))
    with pytest.raises(ValueError, match=match):
        b2.FlatEMA(opt, **kw)
    ddp.remove_hooks()


def test_other_optimizers_are_refused():
    net = W.Net()
    with pytest.raises(ValueError, match="flat optimizer"):
        b2.FlatEMA(torch.optim.SGD(net.parameters(), lr=0.1))


def test_settings_are_read_only_and_decay_edges_work():
    net, ddp, opt, ema = W.build("sgd", dict(lr=0.05), decay=1.0, every=2, warmup_steps=3)
    assert (ema.decay, ema.every, ema.warmup_steps) == (1.0, 2, 3)
    for attr in ("decay", "every", "warmup_steps"):
        with pytest.raises(AttributeError):
            setattr(ema, attr, 1)
    ddp.remove_hooks()
    net, ddp, opt, ema = W.build("sgd", dict(lr=0.05), decay=0.0)     # w = 1: the EMA is the live model
    for it in range(3):
        W.train_step(ddp, opt, 0, it)
        ema.update()
    live = dict(net.named_parameters())
    assert all(W.same_bits(t, live[n]) for n, t in ema.named_ema(ddp).items() if n in live)
    ddp.remove_hooks()


def test_refusals_change_nothing():
    net, ddp, opt, ema = W.build("sgd", dict(lr=0.05, momentum=0.9), decay=0.8)
    W.train_step(ddp, opt, 0, 0)
    ema.update()
    sd = ema.state_dict()
    snap = [e.clone() for e in ema.ema_flats + ema.ema_buffers]
    with pytest.raises(ValueError, match="written with"):
        ema.load_state_dict(dict(sd, every=2))
    with pytest.raises(ValueError, match="buffers"):
        ema.load_state_dict(dict(sd, buffers={}))
    with ema.average_parameters():
        with pytest.raises(RuntimeError, match="inside average_parameters"):
            ema.load_state_dict(sd)
        with pytest.raises(RuntimeError, match="inside average_parameters"):
            ema.load_named_ema(ddp, {})
    assert all(W.same_bits(a, b) for a, b in zip(ema.ema_flats + ema.ema_buffers, snap))
    assert opt.steps == 1
    W.train_step(ddp, opt, 0, 1)         # the optimizer steps again after the block
    assert opt.steps == 2
    ddp.remove_hooks()


@pytest.mark.parametrize("optimizer,sharded", [("sgd", False), ("adamw", False), ("lamb", False), ("lars", False),
                                               ("sgd", True), ("adamw", True)])
def test_example_train_ddp_with_ema(optimizer, sharded):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "6", "--optimizer", optimizer, "--ema-decay", "0.9", "--ema-every", "2",
            "--ema-warmup-steps", "2"]
    if sharded:
        args += ["--sharded-optimizer", "--accumulation-steps", "2"]
    p = subprocess.run([sys.executable, os.path.join(root, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=root)
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(re.findall(r"Rank (\d), step 6: loss", p.stdout)) == ["0", "1"], p.stdout
    lines = re.findall(r"Rank (\d), EMA model: held-out loss ([0-9.]+)", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"] and all(0.1 < float(x) < 10.0 for _, x in lines), p.stdout
