"""CPU tier: gradient-norm clipping (``max_grad_norm``) -- the kernels' fp32 coefficient against torch's, FlatSGD against
``clip_grad_norm_`` + ``torch.optim.SGD`` bit for bit, the validation every engine shares, a two-rank gloo run resumed
from a checkpoint, and the example's flag."""
import math
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

import dist_tuto.pth_b200 as b2
import grad_clip_model as GM
import grad_clip_workers as GW
from dist_tuto.pth_b200 import LRSchedule
from dist_tuto.pth_b200.ops.optim import FlatSGD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def _net():
    return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))


def _torch_coef(n, c):
    """What clip_grad_norm_ computes from a total norm n (fp32 tensor) and max_norm c."""
    return (c / (torch.tensor(n, dtype=torch.float32) + 1e-6)).clamp(max=1.0)


def test_coefficient_model_equals_torch():
    rnd = random.Random(11)
    ns = [0.0, float("inf"), float("nan"), 1e-6, 1e-7, 3e-38]
    ns += [rnd.uniform(0.5, 2) * 10.0 ** rnd.randint(-8, 30) for _ in range(4000)]
    for n in ns:
        n32 = float(np.float32(n))
        for c in (n32 * 0.5, n32 * 2.0, 1.0, 0.1, 1e3, rnd.uniform(0.5, 2) * 10.0 ** rnd.randint(-6, 6)):
            if not (math.isfinite(c) and c > 0) or float(np.float32(c)) == 0.0:
                continue
            want = _torch_coef(n32, c)
            got = GM.coef32(n32, c)
            if math.isnan(float(want)):
                assert np.isnan(got), (n, c)
            else:
                assert float(got) == float(want), (n, c, float(got), float(want))
    # a plain fp32 division differs from torch's reciprocal-then-multiply in many cases: the model is the latter
    diff = sum(float(np.float32(c) / (np.float32(n) + np.float32(1e-6))) != float(GM.coef32(n, c))
               for n, c in ((rnd.uniform(1, 100), rnd.uniform(0.1, 1)) for _ in range(2000)))
    assert diff > 50


@pytest.mark.parametrize("c", [0.3, 1e6], ids=["clipping", "never"])
def test_flat_sgd_equals_clip_grad_norm_and_torch_sgd_bit_for_bit(c):
    sched = LRSchedule(warmup_steps=3, decay="multistep", milestones=[8], gamma=0.5)
    torch.manual_seed(0)
    ref, mine = _net(), _net()
    mine.load_state_dict(ref.state_dict())
    opt_ref = torch.optim.SGD(ref.parameters(), lr=0.2, momentum=0.5, weight_decay=1e-2, nesterov=True, foreach=False)
    opt = FlatSGD(mine, lr=0.2, momentum=0.5, weight_decay=1e-2, nesterov=True, lr_schedule=sched, max_grad_norm=c)
    assert opt.grad_norm() is None
    x, y = torch.randn(12, 8, 6), torch.randn(12, 8, 3)
    clipped = 0
    for k in range(12):
        for grp in opt_ref.param_groups:
            grp["lr"] = sched.lr_at(0.2, k)
        ((ref(x[k]) - y[k]) ** 2).mean().backward()
        norm = torch.nn.utils.clip_grad_norm_(ref.parameters(), c, foreach=False)
        opt_ref.step()
        opt_ref.zero_grad()
        ((mine(x[k]) - y[k]) ** 2).mean().backward()
        opt.step()
        opt.zero_grad()
        assert opt.grad_norm() == float(norm)
        clipped += float(norm) > c
        for (n, a), b in zip(ref.named_parameters(), mine.parameters()):
            assert torch.equal(a.detach(), b.detach()), (k, n)
    assert clipped == (12 if c < 1 else 0)
    sd = opt.state_dict()
    assert sd["max_grad_norm"] == c
    del sd["max_grad_norm"]                   # a checkpoint written before the option: no clipping
    opt.load_state_dict(sd)
    assert opt.max_grad_norm is None


@pytest.mark.parametrize("bad", [0, 0.0, -1.0, float("inf"), float("nan"), 1e-50, 1e40, "1.0", True])
def test_bad_max_grad_norm_is_refused(bad):
    with pytest.raises(ValueError, match="max_grad_norm"):
        b2.TrainConfig(max_grad_norm=bad)
    with pytest.raises(ValueError, match="max_grad_norm"):
        FlatSGD(_net(), max_grad_norm=bad)
    # the trainers check before they touch the extension or a device
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    for cls in (FusedTrainer, BatchedTrainer):
        with pytest.raises(ValueError, match="max_grad_norm"):
            cls(128, max_grad_norm=bad)


def test_good_values_are_kept():
    assert b2.TrainConfig().max_grad_norm is None
    assert b2.TrainConfig(max_grad_norm=1).max_grad_norm == 1.0
    assert FlatSGD(_net(), max_grad_norm=2.5).max_grad_norm == 2.5


def test_train_torch_engine_world2_clip_keeps_replicas_equal_and_resumes_bit_equal(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_CLIP_TEST_DIR", str(tmp_path))
    b2.launch(GW.w_torch_engine_clip_resume, size=2, backend="gloo", join_timeout_s=250)


def test_train_mnist_example_passes_max_grad_norm_through(tmp_path):
    """The flag reaches TrainConfig: the run records it in its FlatSGD checkpoint."""
    ck = str(tmp_path / "ex.pt")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--size", "1", "--epochs", "1",
                        "--max-steps", "4", "--max-grad-norm", "0.5", "--checkpoint", ck],
                       capture_output=True, text=True, timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    optim = torch.load(ck, map_location="cpu")["optim"]
    assert optim["max_grad_norm"] == 0.5 and optim["steps"] == 4
    q = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_mnist.py"), "--help"], capture_output=True,
                       text=True, timeout=120, env=env, cwd=ROOT)
    assert "--max-grad-norm" in q.stdout
