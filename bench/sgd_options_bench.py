#!/usr/bin/env python
"""What weight decay and Nesterov momentum cost in the optimizer kernels, on one GPU.

    python bench/sgd_options_bench.py [--steps 2000] [--reps 5] [--out result.json]

Device time per step (CUDA events around `--steps` steps, after a warm-up, medians of `--reps` alternated rounds) for
four arms -- default, weight_decay=5e-4, nesterov, both -- on three paths:
  fused-graph   FusedTrainer at batch 128 (the slot path: convnet_step + reduce_sgd), steps replayed as CUDA graphs
  fused-native  the same trainer driven by the C++ step executor (run_native over a NativeBatchLoader)
  batched       BatchedTrainer at batch 4096 (wgmma engine + allreduce_sgd), graph replays
The arms of a path run one after another inside each round, so drift between rounds hits every arm alike.

Prints one JSON line with the table and the device name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dist_tuto.pth_b200 import data as D  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer  # noqa: E402

ARMS = {"default": {}, "wd": {"weight_decay": 5e-4}, "nesterov": {"nesterov": True},
        "both": {"weight_decay": 5e-4, "nesterov": True}}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(power)}


def _pinned_batches(n, bsz, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 256, (bsz, 1, 28, 28), generator=g, dtype=torch.uint8).pin_memory(),
             torch.randint(0, 10, (bsz,), generator=g).pin_memory()) for _ in range(n)]


def time_graph(tr, batches, steps):
    """us per step over `steps` graph replays (the trainer's own stream)."""
    for x, y in batches:                         # capture / warm every slot
        tr.step(x, y)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(tr.stream)
    for k in range(steps):
        tr.step(*batches[k % len(batches)])
    if hasattr(tr, "sync_lag"):
        tr.sync_lag(0)
    t1.record(tr.stream)
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / steps


def time_native(tr, loader, steps):
    tr.run_native(loader, max_steps=50)          # builds the executor and warms it
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    done, _ = tr.run_native(loader, max_steps=steps)
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / max(done, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sgd_options_bench.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    small, large = _pinned_batches(4, 128, 1), _pinned_batches(2, 4096, 2)
    n_native = (a.steps + 60) * 128
    part = D.Partition(D.SyntheticMNIST(n=n_native, seed=3), list(range(n_native)))
    fused = {k: FusedTrainer(128, device=dev, raw_uint8=True, **kw) for k, kw in ARMS.items()}
    batched = {k: BatchedTrainer(4096, device=dev, raw_uint8=True, **kw) for k, kw in ARMS.items()}
    times = {p: {k: [] for k in ARMS} for p in ("fused-graph", "fused-native", "batched")}
    # one loader per arm for the whole run: each run_native call starts a new epoch of it on the arm's executor
    loaders = {k: D.NativeBatchLoader(part, 128, seed=9, raw_uint8=True, pin_memory=True, num_buffers=6) for k in ARMS}
    for _ in range(a.reps):
        for k in ARMS:
            times["fused-graph"][k].append(time_graph(fused[k], small, a.steps))
        for k in ARMS:
            times["fused-native"][k].append(time_native(fused[k], loaders[k], a.steps))
        for k in ARMS:
            times["batched"][k].append(time_graph(batched[k], large, max(50, a.steps // 10)))
    for ld in loaders.values():
        ld._l.stop()
    table = {p: {k: {"median_us": statistics.median(v), "runs_us": [round(x, 3) for x in v]} for k, v in arms.items()}
             for p, arms in times.items()}
    res = dict(info, steps=a.steps, reps=a.reps, us_per_step=table)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
