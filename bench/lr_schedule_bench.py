#!/usr/bin/env python
"""Learning-rate schedules on one GPU: what warmup + decay buys at large batch, and what computing the lr in the
optimizer kernels costs.

    python bench/lr_schedule_bench.py [--epochs 5] [--batches 4096 8192] [--steps 2000] [--reps 5]

Convergence: train(engine="batched") on the default training set of partition_dataset() (MNIST when it is on disk, the
synthetic set otherwise) for `--epochs` epochs at each per-GPU batch B, with the test loss / accuracy of evaluate() after
every epoch, in three arms:
  (a) const      lr 0.01, constant (the tutorial's setting, chosen for batch 128)
  (b) scaled     lr 0.01 * B / 128, constant (linear scaling, no warmup)
  (c) warm+cos   lr 0.01 * B / 128, one epoch of linear warmup from 1/3, then cosine decay to 0 at the last epoch
An arm diverged when its training loss is not finite or ends above its first epoch's value.

Cost: FusedTrainer at batch 128 (the slot path: convnet_step + reduce_sgd, replayed as graphs) with a cosine schedule and
without one, timed with CUDA events over `--steps` steps, alternating `--reps` times in this process (medians reported).

Prints one JSON line with both tables and the device name and power limit read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200 import LRSchedule  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"device": name, "power_limit_w": float(power)}


def convergence(batch, epochs):
    scaled = 0.01 * batch / 128
    arms = {"const": (0.01, None), "scaled": (scaled, None),
            "warm+cos": (scaled, LRSchedule(warmup_steps=1, decay="cosine", total_steps=epochs, unit="epoch"))}
    out = {}
    for name, (lr, sched) in arms.items():
        r = b2.train(0, 1, b2.TrainConfig(epochs=epochs, global_batch=batch, engine="batched", lr=lr, device="cuda:0",
                                          lr_schedule=sched, eval_dataset="default", eval_every=1, log=lambda *a: None))
        acc = [round(e["accuracy"], 4) for e in r["eval"]]
        out[name] = {"lr": lr, "test_accuracy": acc, "test_loss": [round(e["loss"], 4) for e in r["eval"]],
                     "train_loss": [round(v, 4) for v in r["loss"]], "lr_last_update": r["lr"],
                     "diverged": (not all(math.isfinite(v) for v in r["loss"])) or r["loss"][-1] > r["loss"][0]}
    return out


def step_cost(steps, reps):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(3)
    batches = [(torch.randint(0, 256, (128, 1, 28, 28), generator=g, dtype=torch.uint8).pin_memory(),
                torch.randint(0, 10, (128,), generator=g).pin_memory()) for _ in range(4)]
    cos = LRSchedule(warmup_steps=100, decay="cosine", total_steps=10 ** 6, min_factor=0.01)
    trainers = {"none": FusedTrainer(128, device=dev, raw_uint8=True),
                "cosine": FusedTrainer(128, device=dev, raw_uint8=True, lr_schedule=cos)}
    times = {k: [] for k in trainers}
    for tr in trainers.values():                       # capture every slot's graph and warm up
        for i in range(200):
            tr.step(*batches[i % 4])
        tr.sync_lag(0)
    torch.cuda.synchronize()
    for _ in range(reps):
        for name, tr in trainers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with tr.active():
                e0.record()
                for i in range(steps):
                    tr.step(*batches[i % 4])
                e1.record()
            tr.sync_lag(0)
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps * 1e3)
    return {k: {"us_per_step_median": round(statistics.median(v), 3), "us_per_step": [round(t, 3) for t in v]}
            for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[4096, 8192])
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lr_schedule_bench needs a GPU")
    torch.cuda.set_device(0)
    res = {"bench": "lr_schedule", **gpu_info(), "epochs": a.epochs,
           "train_set": type(b2.data.default_dataset()).__name__}
    res["convergence"] = {str(b): convergence(b, a.epochs) for b in a.batches}
    res["step_cost_batch128"] = step_cost(a.steps, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
