#!/usr/bin/env python
"""What fp16 loss scaling costs in a training step: ResNet-18 (batch 32, 3 x 32 x 32 as in graph_step_bench.py and
ema_bench.py, channels_last, world size 1, 1000 classes) with

    flat_fp16     fp16 autocast, torch.amp.GradScaler, FlatAdamW (the scaled update kernels; eager: one found_inf read)
    torch_fused   fp16 autocast, torch.amp.GradScaler, torch.optim.AdamW(fused=True) on the plain module
    flat_bf16     bf16 autocast, no scaler, FlatAdamW (the path without loss scaling)

each eager and as replays of one captured step (``capturable=True``; torch's arm fused and capturable).  One step is
forward, backward, ``average_gradients`` (the flat arms), the optimizer step and, with a scaler, ``scaler.update()``.

    python bench/amp_bench.py --gpus 1 [--iters 50] [--reps 5] [--out result.json]

Device time per step: CUDA events around ``--iters`` steps after a warm-up, the median of ``--reps`` rounds with the arms
alternating inside every round.  Every arm is built, warmed up (three eager steps on a side stream, as torch requires
before a capture) and synchronised on its own, and the script says which arm it is on before each phase, so an error is
attributed to its arm.  Autocast runs with ``cache_enabled=False``, as a captured step needs.  Needs a GPU; prints one
JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from sharded_sgd_bench import gpu_info  # noqa: E402

ARMS = ("flat_fp16", "torch_fused", "flat_bf16")


def say(*a):
    print(*a, file=sys.stderr, flush=True)


def arm(kind, graph, dev):
    """The step function of arm ``kind``: an eager step, or one replay of a captured step."""
    torch.manual_seed(0)
    m = ResNet18().to(dev).to(memory_format=torch.channels_last)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(32, 3, 32, 32, generator=gen).to(dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (32,), generator=gen).to(dev)
    dtype = torch.bfloat16 if kind == "flat_bf16" else torch.float16
    scaler = None if kind == "flat_bf16" else torch.amp.GradScaler("cuda")
    if kind == "torch_fused":
        model, opt = m, torch.optim.AdamW(m.parameters(), lr=1e-3, fused=True, capturable=graph)
    else:
        model = b2.DistributedDataParallel(m)
        opt = b2.FlatAdamW(model, lr=1e-3, capturable=graph)

    def step():
        with torch.autocast("cuda", dtype=dtype, cache_enabled=False):
            loss = F.cross_entropy(model(x), y)
        if scaler is None:
            loss.backward()
        else:
            scaler.scale(loss).backward()
        if kind != "torch_fused":
            b2.average_gradients(model)
        if scaler is None:
            opt.step()
        else:
            scaler.step(opt)
            scaler.update()
        if kind == "torch_fused":
            opt.zero_grad(set_to_none=False)

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
            s.synchronize()
    torch.cuda.current_stream(dev).wait_stream(s)
    if not graph:
        return step
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    torch.cuda.synchronize(dev)

    def replay():
        g.replay()
    # the graph reads and writes the model, optimizer, scaler and input tensors, which only the step closure holds: keep
    # them alive as long as the replay function, or their memory is freed and reused under the graph
    replay.step = step
    return replay


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.gpus != 1 or not torch.cuda.is_available():
        sys.exit("amp_bench.py measures on one GPU: --gpus 1 on a machine with CUDA")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(gpu_info(), workload="ResNet-18, batch 32, 3x32x32, channels_last, 1000 classes, world 1",
               unit="ms per step (device time)")
    for mode in ("eager", "captured"):
        arms = {}
        for k in ARMS:
            say(f"[amp_bench] {mode} {k}: build and warm up")
            arms[k] = arm(k, mode == "captured", dev)
            say(f"[amp_bench] {mode} {k}: first timed calls")
            timed(arms[k], 3)
        got = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, fn in arms.items():
                got[k].append(timed(fn, a.iters))
        res[mode] = {k: round(statistics.median(v), 4) for k, v in got.items()}
        say(f"[amp_bench] {mode}: {res[mode]}")
        del arms
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
