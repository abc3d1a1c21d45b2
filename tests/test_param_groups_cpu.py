"""``param_groups`` of ``FlatSGD`` / ``FlatAdamW`` on gloo CPU ranks (worlds 2 and 3): bit for bit torch's optimizers with
the same groups, an LRSchedule and a mid-run lr change; the no-decay group; checkpoints; the refusals.  Workers in
tests/param_groups_workers.py."""
import pytest
import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
import param_groups_workers as W
from dist_tuto.pth_b200.ops.optim import MAX_PARAM_GROUPS, FlatAdamW, FlatSGD
from dist_tuto.pth_b200.parallel.ddp import GradBucket

pytestmark = pytest.mark.timeout(600)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=540)


@pytest.mark.parametrize("size", [2, 3])
def test_groups_are_bit_for_bit_torch(size):
    go(W.w_bit_equal_to_torch, size)


def test_no_decay_group_gets_no_decay():
    go(W.w_no_decay_group, 2)


@pytest.mark.parametrize("size", [2, 3])
def test_checkpoints_carry_the_groups(size):
    go(W.w_checkpoint, size)


def test_grouped_sharded_continues_unsharded():
    go(W.w_world_change, 3)


def test_param_groups_none_and_default_group():
    net = W._mlp()
    opt = FlatSGD(net, lr=0.1, weight_decay=0.01)
    assert not opt._grouped and len(opt.param_groups) == 1
    assert opt.param_groups[0]["lr"] == 0.1 and len(opt.param_groups[0]["params"]) == len(list(net.parameters()))
    opt.param_groups[0]["lr"] = 0.2                  # the default group is the optimizer's lr
    assert opt.lr == 0.2
    opt.weight_decay = 0.5
    assert opt.param_groups[0]["weight_decay"] == 0.5
    net = W._mlp()
    every = [{"params": [p]} for p in net.parameters()]
    opt = FlatAdamW(net, param_groups=every)         # every parameter named: no default group
    assert len(opt.param_groups) == len(every)


@pytest.mark.parametrize("Flat", [FlatSGD, FlatAdamW])
def test_refusals_leave_the_model_untouched(Flat):
    net = W._mlp()
    other = nn.Linear(2, 2)
    ptrs = [p.data_ptr() for p in net.parameters()]
    w0 = net[0].weight
    bad = [([{"params": [other.weight]}], "no gradient bucket"),
           ([{"params": [w0]}, {"params": [w0]}], "twice"),
           ([{"params": [w0, w0]}], "twice"),
           ([{"params": []}], "empty"),
           ([{"params": [w0], "betas": (0.9, 0.9)}], "'betas'"),
           ([{"params": [w0], "momentum": 0.5}], "'momentum'"),
           ([{"params": [w0], "nesterov": True}], "'nesterov'"),
           ([{"params": [w0], "eps": 1e-3}], "'eps'"),
           ([{"params": [w0], "weight_decay": -1.0}], "weight_decay"),
           ([{"lr": 0.1}], "no 'params'"),
           ({"params": [w0]}, "list of dicts")]
    if Flat is FlatAdamW:
        bad.append(([{"params": [w0], "lr": -0.1}], "learning rate"))
    for groups, msg in bad:
        with pytest.raises(ValueError, match=msg):
            Flat(net, param_groups=groups)
        assert not hasattr(net, "_grad_bucket") and [p.data_ptr() for p in net.parameters()] == ptrs
    # more than 64 groups, the default group included
    many = nn.Sequential(*[nn.Linear(1, 1, bias=False) for _ in range(MAX_PARAM_GROUPS + 1)])
    with pytest.raises(ValueError, match="at most 64"):
        Flat(many, param_groups=[{"params": [m.weight]} for m in many])
    with pytest.raises(ValueError, match="at most 64"):
        Flat(many, param_groups=[{"params": [m.weight]} for m in list(many)[:MAX_PARAM_GROUPS]])
    Flat(many, param_groups=[{"params": [m.weight]} for m in list(many)[:MAX_PARAM_GROUPS - 1]])


def test_misaligned_cuda_bucket_is_refused():
    if not torch.cuda.is_available():
        pytest.skip("the alignment rule concerns CUDA buckets")
    net = W._mlp().cuda()
    object.__setattr__(net, "_grad_bucket", GradBucket(list(net.parameters()), align=1, symmetric=False))
    with pytest.raises(ValueError, match="multiple of 4"):
        FlatSGD(net, param_groups=[{"params": [net[0].bias], "weight_decay": 0.0}])


def test_kernel_and_binding_agree_on_the_group_limit():
    pytest.importorskip("dist_tuto.pth_b200._C")
    from dist_tuto.pth_b200.ops import _ext

    assert _ext.C().max_param_groups() == MAX_PARAM_GROUPS


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_example_train_ddp_with_no_decay_groups(optimizer):
    import os
    import re
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    args = ["--size", "2", "--steps", "6", "--optimizer", optimizer, "--sharded-optimizer", "--no-decay-bias-norm"]
    p = subprocess.run([sys.executable, os.path.join(root, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=root)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 6: loss ([0-9.]+)", p.stdout)
    assert sorted(r for r, _ in lines) == ["0", "1"] and all(0.5 < float(x) < 5.0 for _, x in lines), p.stdout
