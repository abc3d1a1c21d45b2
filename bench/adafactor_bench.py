#!/usr/bin/env python
"""FlatAdafactor against torch.optim.Adafactor, and the optimizer-state bytes of each against FlatAdamW.

    python bench/adafactor_bench.py [--iters 20] [--reps 5] [--out result.json]

Two models on one GPU, DistributedDataParallel buckets of ``--bucket-mb``:
  * ResNet-18 (11.7 M fp32 parameters, 62 tensors, conv weights factored over their kernel dimensions);
  * a transformer-style stack of Linear layers: 4 blocks of 4096x1024, 1024x4096, 3072x1024 and 1024x1024 weights with biases.
Per model, the device time of one ``step()`` (CUDA events around ``--iters`` calls after a warm-up, medians of ``--reps``
rounds, the arms alternating inside every round):
    FlatAdafactor                  three launches per bucket (zero_grad=False, so every call sees the same gradients)
    torch Adafactor foreach=True   torch.optim.Adafactor(foreach=True) on the same shapes
    torch Adafactor foreach=False  torch.optim.Adafactor(foreach=False)
and the optimizer state of each (FlatAdafactor's state flats, torch's per-parameter state, FlatAdamW's two moments), in
bytes.  torch's Adafactor synchronises the host twice per tensor, so its times include those waits.  Needs a GPU: without one
it fails.  Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
HP = dict(lr=1e-2, weight_decay=1e-4)


def transformer_stack():
    layers = []
    for _ in range(4):
        layers += [nn.Linear(1024, 4096), nn.Linear(4096, 1024), nn.Linear(1024, 3072), nn.Linear(3072, 1024),
                   nn.Linear(1024, 1024)]
    return nn.Sequential(*layers)


def _state_bytes(tensors):
    return int(sum(t.numel() * t.element_size() for t in tensors))


def arms_for(make, dev):
    """The three step() arms on copies of one model with the same gradients, and the state bytes of each optimizer."""
    torch.manual_seed(1234)
    model = make().to(dev).to(memory_format=torch.channels_last) if make is ResNet18 else make().to(dev)
    ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
    opt = b2.FlatAdafactor(ddp, zero_grad=False, **HP)
    for gb in opt.buckets:
        gb.flat.normal_(std=1e-3)
    arms = {"FlatAdafactor": opt.step}
    state = {"FlatAdafactor": _state_bytes(opt.state_flats)}
    for foreach in (True, False):
        torch.manual_seed(1234)
        net = make().to(dev)
        if make is ResNet18:
            net = net.to(memory_format=torch.channels_last)
        for p in net.parameters():
            p.grad = torch.randn_like(p) * 1e-3
        topt = torch.optim.Adafactor(net.parameters(), foreach=foreach, **HP)
        topt.step()                                               # creates the state
        arms[f"torch Adafactor foreach={foreach}"] = topt.step
        state[f"torch Adafactor foreach={foreach}"] = _state_bytes(
            [v for s in topt.state.values() for k, v in s.items() if k != "step"])
    n = sum(gb.numel for gb in opt.buckets)
    state["FlatAdamW (exp_avg + exp_avg_sq)"] = 8 * n
    ddp.remove_hooks()
    return arms, {"parameters": n, "tensors": sum(len(gb.params) for gb in opt.buckets), "buckets": len(opt.buckets),
                  "launches_per_step": 3 * len(opt.buckets), "state_bytes": state}


def _rounds(arms, iters, dev):
    runs = {k: [] for k in arms}
    for fn in arms.values():
        _timed(fn, 3, dev)                                        # warm-up
    for _ in range(ARGS.reps):
        for k, fn in arms.items():
            runs[k].append(_timed(fn, iters, dev))
    return {k: {"median": statistics.median(v), "runs": [round(t, 5) for t in v]} for k, v in runs.items()}


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    res = dict(gpu_info(), iters=ARGS.iters, reps=ARGS.reps, bucket_mb=ARGS.bucket_mb, hyper_parameters=HP)
    for name, make in (("resnet18", ResNet18), ("linear_stack", transformer_stack)):
        arms, info = arms_for(make, dev)
        res[name] = dict(info, step_ms=_rounds(arms, ARGS.iters, dev))
    line = json.dumps(res)
    print(line, flush=True)
    if ARGS.out:
        os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
        with open(ARGS.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bucket-mb", type=int, default=25)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adafactor_bench.py measures on a GPU; none is visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=1, backend="b200", join_timeout_s=1500)
