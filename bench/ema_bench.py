#!/usr/bin/env python
"""What an exponential moving average of the weights costs: ``FlatEMA.update()`` against ``torch._foreach_lerp_`` over the
same tensors (``AveragedModel``'s path), and a captured ResNet-18 step with and without the update.

    python bench/ema_bench.py --gpus 1 [--iters 100] [--reps 5] [--out result.json]

Workloads (world size 1, FlatSGD, decay 0.9999, every update a lerp):
    ResNet-18    its parameters and BatchNorm running statistics (11.7 M fp32), default buckets
    100M         24 Linear(2048, 2048) layers (100.7 M fp32) in 25 MB buckets
Arms: ``flat`` is ``FlatEMA.update()`` (one ``ema_update`` launch); ``torch`` is ``torch._foreach_lerp_(ema, live, 1 - decay)``
over per-tensor EMA copies of the parameters and fp32 buffers.  Both move 12 bytes per element (read EMA and live, write
EMA).  Device time per call: CUDA events around ``--iters`` calls after a warm-up, medians of ``--reps`` rounds with the
arms alternating inside every round.  The step part times replays of one captured ResNet-18 step (batch 32, 3 x 32 x 32,
bf16 autocast, capturable FlatSGD) with and without ``update()`` at every = 1.  Needs a GPU; prints one JSON line with
the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from sharded_sgd_bench import gpu_info  # noqa: E402

DECAY = 0.9999


def timed(fn, iters):
    """Device ms per call of ``fn`` over ``iters`` calls."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def alternate(arms, iters, reps):
    """{arm: median ms per call}, the arms alternating inside every round."""
    for fn in arms.values():          # warm-up
        timed(fn, 5)
    got = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            got[k].append(timed(fn, iters))
    return {k: statistics.median(v) for k, v in got.items()}


def big_model():
    return nn.Sequential(*[nn.Linear(2048, 2048, bias=False) for _ in range(24)])


def update_arms(name, model, bucket_cap_bytes, dev, a):
    ddp = b2.DistributedDataParallel(model, bucket_cap_bytes=bucket_cap_bytes)
    opt = b2.FlatSGD(ddp, lr=0.05, momentum=0.9)
    ema = b2.FlatEMA(opt, decay=DECAY)
    opt.steps = 10                     # every update lerps
    live = [p.detach() for p in model.parameters()] + [b for b in model.buffers() if b.dtype == torch.float32]
    shadow = [t.clone() for t in live]
    n = sum(t.numel() for t in live)
    assert n == sum(e.numel() for e in ema.ema_flats + ema.ema_buffers)
    ms = alternate({"flat": ema.update, "torch": lambda: torch._foreach_lerp_(shadow, live, 1 - DECAY)}, a.iters, a.reps)
    ddp.remove_hooks()
    out = {"workload": name, "elements": n, "tensors": len(live), "buckets": len(opt.buckets)}
    for k, v in ms.items():
        out[f"{k}_us"] = round(v * 1e3, 2)
        out[f"{k}_GBps"] = round(12 * n / (v * 1e-3) / 1e9, 1)
    out["flat_over_torch"] = round(ms["flat"] / ms["torch"], 3)
    return out


def step_arms(dev, a):
    """Replays of one captured ResNet-18 step, without and with ``update()``."""
    graphs = {}
    for arm in ("step", "step+update"):
        torch.manual_seed(0)
        m = ResNet18().to(dev).to(memory_format=torch.channels_last)
        ddp = b2.DistributedDataParallel(m)
        opt = b2.FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=5e-4, capturable=True)
        ema = b2.FlatEMA(opt, decay=DECAY) if arm == "step+update" else None
        g = torch.Generator(device=dev).manual_seed(1)
        x = torch.randn(32, 3, 32, 32, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (32,), generator=g, device=dev)

        def step():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(ddp(x), y)
            loss.backward()
            b2.average_gradients(ddp)
            opt.step()
            if ema is not None:
                ema.update()

        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for _ in range(3):
                step()
        torch.cuda.current_stream(dev).wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graphs[arm] = (graph, ddp, m, opt, ema, x, y)   # everything the graph reads stays alive while it replays
    ms = alternate({k: v[0].replay for k, v in graphs.items()}, a.iters, a.reps)
    torch.cuda.synchronize()
    for v in graphs.values():
        v[1].remove_hooks()
    return {"workload": "ResNet-18 captured step, batch 32", **{f"{k}_ms": round(v, 4) for k, v in ms.items()},
            "update_share": round((ms["step+update"] - ms["step"]) / ms["step"], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.gpus != 1:
        ap.error("the EMA update does no communication: it is measured at --gpus 1")
    if not torch.cuda.is_available():
        sys.exit("ema_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    torch.manual_seed(0)
    rows = [update_arms("ResNet-18", ResNet18().to(dev), 8 << 20, dev, a),
            update_arms("100M", big_model().to(dev), 25 << 20, dev, a),
            step_arms(dev, a)]
    res = {"bench": "ema", **info, "iters": a.iters, "reps": a.reps, "results": rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
