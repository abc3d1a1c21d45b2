#!/usr/bin/env python
"""FlatAdamW against torch.optim.AdamW, and the sharded AdamW kernel against the path it replaces.

    python bench/adamw_bench.py --gpus 1 [--iters 100] [--reps 5] [--out result.json]

* ``step()`` on the parameters and gradients of a ResNet-18 (11.7 M fp32 parameters, DistributedDataParallel buckets of
  ``--bucket-mb``), device time per call (CUDA events around ``--iters`` calls after a warm-up, medians of ``--reps`` rounds,
  the arms alternating inside every round):
    FlatAdamW                 one adamw_flat launch per bucket (zero_grad=False, so every call sees the same gradients)
    torch AdamW fused=True    torch.optim.AdamW(fused=True) on the same shapes
    torch AdamW foreach=True  torch.optim.AdamW(foreach=True)
* per bucket size (1, 8, 25, 64 MB of fp32 gradients), device time per call, max over ranks:
    allreduce+adamw_flat      the bucket's all-reduce with the 1/W scale, then adamw_flat on the whole flat with re-zeroing --
                              what FlatAdamW(sharded=False) runs per bucket
    sharded_adamw             ONE launch: reduce-scatter, AdamW on the owned slice, parameter all-gather, re-zeroing

With --gpus 1 the all-reduce is a no-op and sharded_adamw runs with one rank (no peer traffic): that run times the kernels'
single-GPU cost only.  The bucket arms at two or more ranks need --gpus >= 2.  Needs GPUs: without one it fails.  Prints one
JSON line with the card's name and power limit read in the same run.
"""
import argparse
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
from dist_tuto.pth_b200.ops.optim import adamw_scalars  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
HP = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)


def step_arms(dev):
    """The three step() arms on a ResNet-18's parameters, each with its own copy and the same gradients."""
    arms = {}
    torch.manual_seed(1234)
    model = ResNet18(num_classes=1000).to(dev)
    ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
    opt = b2.FlatAdamW(ddp, zero_grad=False, **HP)
    for gb in opt.buckets:
        gb.flat.normal_(std=1e-3)
    arms["FlatAdamW"] = opt.step
    for kind in ("fused", "foreach"):
        torch.manual_seed(1234)
        net = ResNet18(num_classes=1000).to(dev)
        for p in net.parameters():
            p.grad = torch.randn_like(p) * 1e-3
        topt = torch.optim.AdamW(net.parameters(), **HP, **{kind: True})
        arms[f"torch AdamW {kind}=True"] = topt.step
    n = sum(gb.numel for gb in opt.buckets)
    return arms, {"parameters": n, "buckets": len(opt.buckets), "bucket_mb": ARGS.bucket_mb}


def bucket_arms(w, mb, dev):
    W = w.world
    n_vec = ((mb << 20) // 16 + W - 1) // W * W
    n = n_vec * 4
    gh, ph = w.alloc(n, torch.float32), w.alloc_bytes(n * 4, ll=False)
    g = gh.local[:n]
    p_flat, m_flat, v_flat = (torch.zeros(n, device=dev) for _ in range(3))
    m_shard, v_shard = torch.zeros(n // W, device=dev), torch.zeros(n // W, device=dev)
    g.normal_()
    sc = adamw_scalars(HP["lr"], HP["betas"], HP["eps"], HP["weight_decay"], 10)

    def unsharded():
        w.all_reduce_(g, scale=1.0 / W, handle=gh)
        w.C.adamw_flat(p_flat, m_flat, v_flat, g, sc, True)

    def sharded():
        w.C.sharded_adamw(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, v_shard, n_vec, sc, 1.0 / W, True, w.rank, W,
                          w.max_blocks)

    return {"allreduce+adamw_flat": unsharded, "sharded_adamw": sharded}


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
    res["buckets_ms"] = {f"{mb}MB": _rounds(bucket_arms(w, mb, dev), ARGS.iters, dev) for mb in (1, 8, 25, 64)}
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
        raise SystemExit(f"adamw_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
