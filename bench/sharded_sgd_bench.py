#!/usr/bin/env python
"""The sharded optimizer step against the path it replaces: all-reduce + sgd_flat versus sharded_sgd, per bucket and in
the ResNet-18 step.

    python bench/sharded_sgd_bench.py --gpus 8 [--iters 200] [--reps 5] [--steps 30] [--out result.json]

Per bucket size (1, 8, 25, 64 MB of fp32 gradients), device time per call (CUDA events around `--iters` calls after a warm-up,
medians of `--reps` rounds, the two arms alternating inside every round, max over ranks):
  allreduce+sgd_flat   the bucket's fused all-reduce with the 1/W scale (variant by size, as DistributedDataParallel launches
                       it), then sgd_flat on the whole flat with re-zeroing -- what FlatSGD(sharded=False) runs per bucket
  sharded_sgd          ONE launch: reduce-scatter, update of the owned slice, parameter all-gather, re-zeroing
Then the ResNet-18 bf16-autocast step of bench/resnet_bench.py (DistributedDataParallel + FlatSGD, fp32 buckets) with
sharded=False and sharded=True, alternating, device-timed.

With --gpus 1 the all-reduce is a no-op, sharded_sgd runs with one rank (no peer traffic) and FlatSGD(sharded=True) is the
unsharded path: that run times the kernels' single-GPU cost only and says nothing about NVLink.  Needs GPUs: without one it
fails.  Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
LR, MU, WD = 0.01, 0.9, 5e-4


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(power)}


def _timed(fn, iters, dev):
    """ms per call of fn over `iters` calls, device-timed, max over ranks."""
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def bucket_arms(w, mb, dev):
    """The two per-bucket arms on symmetric buffers of `mb` MB of fp32 gradients."""
    W = w.world
    n_vec = ((mb << 20) // 16 + W - 1) // W * W
    n = n_vec * 4
    gh, ph = w.alloc(n, torch.float32), w.alloc_bytes(n * 4, ll=False)
    g = gh.local[:n]
    p_flat, m_flat = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    m_shard = torch.zeros(n // W, device=dev)
    g.normal_()

    def unsharded():
        w.all_reduce_(g, scale=1.0 / W, handle=gh)
        w.C.sgd_flat(p_flat, m_flat, g, LR, MU, WD, True, False)

    def sharded():
        w.C.sharded_sgd(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, n_vec, LR, MU, WD, False, 1.0 / W, True, w.rank, W,
                        w.max_blocks)

    return {"allreduce+sgd_flat": unsharded, "sharded_sgd": sharded}


def resnet_arm(sharded, dev):
    torch.manual_seed(1234)
    model = ResNet18(num_classes=1000).to(dev).to(memory_format=torch.channels_last)
    ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
    opt = b2.FlatSGD(ddp, lr=0.01, momentum=0.5, sharded=sharded)
    x = torch.randn(ARGS.batch, 3, ARGS.res, ARGS.res, device=dev).to(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (ARGS.batch,), device=dev)

    def step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(ddp(x), y)
        loss.backward()
        b2.average_gradients(ddp)
        opt.step()

    return step


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    w = symm.lookup_world(None)
    res = dict(gpu_info(), n_gpus=size, iters=ARGS.iters, reps=ARGS.reps, buckets_ms={}, resnet18_ms={})
    for mb in (1, 8, 25, 64):
        arms = bucket_arms(w, mb, dev)
        runs = {k: [] for k in arms}
        for fn in arms.values():
            _timed(fn, 10, dev)                                   # warm-up
        for _ in range(ARGS.reps):
            for k, fn in arms.items():
                runs[k].append(_timed(fn, ARGS.iters, dev))
        res["buckets_ms"][f"{mb}MB"] = {k: {"median": statistics.median(v), "runs": [round(t, 5) for t in v]}
                                        for k, v in runs.items()}
    torch.backends.cudnn.benchmark = True
    steps = {"sharded=False": resnet_arm(False, dev), "sharded=True": resnet_arm(True, dev)}
    runs = {k: [] for k in steps}
    for fn in steps.values():
        _timed(fn, ARGS.warmup, dev)
    for _ in range(ARGS.reps):
        for k, fn in steps.items():
            runs[k].append(_timed(fn, ARGS.steps, dev))
    res["resnet18_ms"] = {k: {"median": statistics.median(v), "runs": [round(t, 4) for t in v]} for k, v in runs.items()}
    res["resnet18"] = {"per_gpu_batch": ARGS.batch, "res": ARGS.res, "bucket_mb": ARGS.bucket_mb, "steps": ARGS.steps}
    if size == 1:
        res["note"] = ("one GPU: no peer traffic, and FlatSGD(sharded=True) is the unsharded path; multi-GPU times are not "
                       "measured by this run")
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
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--bucket-mb", type=int, default=8)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < ARGS.gpus:
        raise SystemExit(f"sharded_sgd_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
