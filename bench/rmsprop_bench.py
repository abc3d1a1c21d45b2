#!/usr/bin/env python
"""FlatRMSprop against torch.optim.RMSprop, and the sharded RMSprop kernel against the path it replaces.

    python bench/rmsprop_bench.py --gpus 1 [--iters 100] [--reps 5] [--out result.json]

* ``step()`` on the parameters and gradients of a ResNet-18 (11.7 M fp32 parameters, DistributedDataParallel buckets of
  ``--bucket-mb``) with torchvision's RMSprop settings (alpha 0.9, eps 0.0316, momentum 0.9, weight decay 1e-5), device
  time per call (CUDA events around ``--iters`` calls after a warm-up, medians of ``--reps`` rounds, the arms alternating
  inside every round):
    FlatRMSprop                 one rmsprop_flat launch per bucket (zero_grad=False, so every call sees the same gradients)
    torch RMSprop foreach=True  torch.optim.RMSprop(foreach=True) on the same shapes (torch 2.11 has no fused RMSprop: its
                                constructor takes no ``fused`` argument)
* per fp32 bucket size (1, 8, 25, 64 MB) and per momentum 0 / 0.9 x centered off / on, device time per call, max over ranks:
    allreduce+rmsprop_flat      the bucket's all-reduce with the 1/W scale, then rmsprop_flat on the whole flat with
                                re-zeroing -- what FlatRMSprop(sharded=False) runs per bucket
    sharded_rmsprop             ONE launch: reduce-scatter, RMSprop on the owned slice, parameter all-gather, re-zeroing

With --gpus 1 the all-reduce is a no-op and sharded_rmsprop runs with one rank (no peer traffic): that run times the kernels'
single-GPU cost only.  The bucket arms at two or more ranks need --gpus >= 2.  Needs GPUs: without one it fails.  Prints one
JSON line with the card's name and power limit read in the same run.
"""
import argparse
import inspect
import json
import os
import statistics
import sys
import types

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.ops.optim import rmsprop_scalars  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
HP = dict(lr=1e-3, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-5)


def step_arms(dev):
    """The two step() arms on a ResNet-18's parameters, each with its own copy and the same gradients."""
    assert "fused" not in inspect.signature(torch.optim.RMSprop.__init__).parameters, "torch now has a fused RMSprop: time it"
    arms = {}
    torch.manual_seed(1234)
    model = ResNet18(num_classes=1000).to(dev)
    ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
    opt = b2.FlatRMSprop(ddp, zero_grad=False, **HP)
    for gb in opt.buckets:
        gb.flat.normal_(std=1e-3)
    arms["FlatRMSprop"] = opt.step
    torch.manual_seed(1234)
    net = ResNet18(num_classes=1000).to(dev)
    for p in net.parameters():
        p.grad = torch.randn_like(p) * 1e-3
    arms["torch RMSprop foreach=True"] = torch.optim.RMSprop(net.parameters(), foreach=True, **HP).step
    n = sum(gb.numel for gb in opt.buckets)
    return arms, {"parameters": n, "buckets": len(opt.buckets), "bucket_mb": ARGS.bucket_mb, "hyper_parameters": HP}


def bucket_arms(w, mb, dev, momentum, centered):
    W = w.world
    n_vec = ((mb << 20) // 16 + W - 1) // W * W
    n = n_vec * 4
    gh, ph = w.alloc(n, torch.float32), w.alloc_bytes(n * 4, ll=False)
    g = gh.local[:n]
    g.normal_()
    whole = [torch.zeros(n, device=dev) for _ in range(4)]          # p, square_avg, grad_avg, momentum_buffer
    shard = [torch.zeros(n // W, device=dev) for _ in range(3)]     # square_avg, grad_avg, momentum_buffer
    sc = rmsprop_scalars(HP["lr"], HP["alpha"], HP["eps"], HP["weight_decay"], momentum)
    ga, buf = (whole[2] if centered else None), (whole[3] if momentum > 0 else None)
    sga, sbuf = (shard[1] if centered else None), (shard[2] if momentum > 0 else None)

    def unsharded():
        w.all_reduce_(g, scale=1.0 / W, handle=gh)
        w.C.rmsprop_flat(whole[0], whole[1], ga, buf, g, sc, centered, True)

    def sharded():
        w.C.sharded_rmsprop(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, shard[0], sga, sbuf, n_vec, sc, centered, 1.0 / W, True, w.rank,
                            W, w.max_blocks)

    return {"allreduce+rmsprop_flat": unsharded, "sharded_rmsprop": sharded}


def _rounds(arms, iters, dev):
    runs = {k: [] for k in arms}
    for fn in arms.values():
        _timed(fn, 10, dev)                                       # warm-up
    for _ in range(ARGS.reps):
        for k, fn in arms.items():
            runs[k].append(_timed(fn, iters, dev))
    return {k: {"median": statistics.median(v), "runs": [round(t, 5) for t in v]} for k, v in runs.items()}


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    w = symm.lookup_world(None)
    res = dict(gpu_info(), n_gpus=size, iters=ARGS.iters, reps=ARGS.reps)
    arms, info = step_arms(dev)
    res["resnet18_step_ms"] = _rounds(arms, ARGS.iters, dev)
    res["resnet18"] = info
    res["buckets_ms"] = {f"{mb}MB momentum {mu} centered {int(c)}": _rounds(bucket_arms(w, mb, dev, mu, c), ARGS.iters, dev)
                         for mb in (1, 8, 25, 64) for mu in (0.0, 0.9) for c in (False, True)}
    if size == 1:
        res["note"] = "one GPU: no peer traffic in the bucket arms; multi-GPU times are not measured by this run"
    if rank == 0:
        line = json.dumps(res)
        print(line, flush=True)
        if ARGS.out:
            os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
            with open(ARGS.out, "w") as f:
                f.write(line + "\n")
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bucket-mb", type=int, default=25)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < ARGS.gpus:
        raise SystemExit(f"rmsprop_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
