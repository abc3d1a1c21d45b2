#!/usr/bin/env python
"""What gradient-norm clipping (max_grad_norm) costs, on one GPU.

    python bench/grad_clip_bench.py [--steps 2000] [--reps 3] [--out result.json]

Device time per step (CUDA events around `--steps` steps after a warm-up; `--reps` rounds that alternate clipping off and
on) with max_grad_norm = 1e-3, so that a coefficient below 1 is in force at every update (checked), on four paths:
  slot       FusedTrainer at batch 128 (convnet_step + reduce_sgd), graph replays
  cluster    FusedTrainer at batch 16 (cluster step kernel + allreduce_sgd), graph replays
  batched    BatchedTrainer at batch 4096 (wgmma engine + allreduce_sgd), graph replays
  flat-sgd   FlatSGD.step() alone over ResNet-18's parameters in 8 MB gradient buckets (grad_sqnorm per bucket, then
             sgd_flat per bucket), eager launches
Anything that needs more than one GPU (the push exchange) is not measured here.

Prints one JSON line with the table and the device name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

from sgd_options_bench import _pinned_batches, gpu_info, time_graph  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer  # noqa: E402

C_CLIP = 1e-3
ARMS = {"off": {}, "on": {"max_grad_norm": C_CLIP}}


class _Buckets:
    """The DistributedDataParallel surface FlatSGD reads: ResNet-18's parameters in reverse order, 8 MB per bucket."""

    def __init__(self, model, cap_bytes=8 << 20):
        from dist_tuto.pth_b200.parallel.ddp import GradBucket
        self.buckets, cur, size = [], [], 0
        for p in reversed(list(model.parameters())):
            cur.append(p)
            size += p.numel() * 4
            if size >= cap_bytes:
                self.buckets.append(GradBucket(cur))
                cur, size = [], 0
        if cur:
            self.buckets.append(GradBucket(cur))

    def _reset(self):
        pass

    def zero_grad(self):
        pass


def flat_sgd_setup(dev, clip):
    from dist_tuto.pth_b200.models.resnet import ResNet18
    from dist_tuto.pth_b200.ops.optim import FlatSGD
    torch.manual_seed(0)
    model = ResNet18().to(dev)
    eng = _Buckets(model)
    object.__setattr__(model, "_ddp_engine", eng)
    g = torch.Generator(device=dev).manual_seed(1)
    for gb in eng.buckets:
        gb.flat.copy_(torch.randn(gb.flat.numel(), generator=g, device=dev) * 1e-2)
    # zero_grad=False: the buckets keep their gradients, so every timed step clips the same norm
    return FlatSGD(model, lr=0.01, momentum=0.9, zero_grad=False, **({"max_grad_norm": C_CLIP} if clip else {}))


def time_flat(opt, steps):
    for _ in range(5):
        opt.step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        opt.step()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_clip_bench.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    b128, b16, b4096 = _pinned_batches(4, 128, 1), _pinned_batches(4, 16, 4), _pinned_batches(2, 4096, 2)
    slot = {k: FusedTrainer(128, device=dev, raw_uint8=True, **kw) for k, kw in ARMS.items()}
    cluster = {k: FusedTrainer(16, device=dev, raw_uint8=True, **kw) for k, kw in ARMS.items()}
    assert all(tr.cluster > 1 for tr in cluster.values())
    batched = {k: BatchedTrainer(4096, device=dev, raw_uint8=True, **kw) for k, kw in ARMS.items()}
    flat = {k: flat_sgd_setup(dev, k == "on") for k in ARMS}
    times = {p: {k: [] for k in ARMS} for p in ("slot", "cluster", "batched", "flat-sgd")}
    for _ in range(a.reps):
        for k in ARMS:
            times["slot"][k].append(time_graph(slot[k], b128, a.steps))
        for k in ARMS:
            times["cluster"][k].append(time_graph(cluster[k], b16, a.steps))
        for k in ARMS:
            times["batched"][k].append(time_graph(batched[k], b4096, max(50, a.steps // 10)))
        for k in ARMS:
            times["flat-sgd"][k].append(time_flat(flat[k], max(50, a.steps // 10)))
    norms = {"slot": slot["on"].grad_norm(), "cluster": cluster["on"].grad_norm(), "batched": batched["on"].grad_norm(),
             "flat-sgd": flat["on"].grad_norm()}
    assert all(n > C_CLIP for n in norms.values()), norms          # the coefficient was below 1
    table = {p: {k: {"median_us": statistics.median(v), "runs_us": [round(x, 3) for x in v]} for k, v in arms.items()}
             for p, arms in times.items()}
    for p in table:
        table[p]["on_minus_off_us"] = round(table[p]["on"]["median_us"] - table[p]["off"]["median_us"], 3)
    res = dict(info, steps=a.steps, reps=a.reps, max_grad_norm=C_CLIP, last_norms=norms, us_per_step=table,
               flat_sgd_buckets=len(flat["on"].buckets), multi_gpu="not measured")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
