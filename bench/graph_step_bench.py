#!/usr/bin/env python
"""What a CUDA graph saves a DistributedDataParallel training step: eager steps against replays of one captured step.

    python bench/graph_step_bench.py --gpus 1 [--iters 50] [--reps 7] [--out result.json]

Workloads (backend "b200", DistributedDataParallel at world size ``--gpus``):
    Net          the tutorial's Net, global batch 128 (strong scaling: 128 / W per GPU)
    ResNet-18    batch 32 per GPU, 3 x 32 x 32, bf16 autocast, channels_last
each with FlatSGD (momentum 0.9, weight decay 5e-4) and FlatAdamW.  One step is forward, backward (the bucket exchanges
run in the DDP hooks), ``average_gradients`` and ``step()``.  Arms:
    eager        the default optimizer (capturable=False), every launch issued from Python
    graph        capturable=True, warm-up steps on a side stream, one step captured, ``replay()`` per step
With more than one GPU both arms run ``sharded=True``.  Device time per step: CUDA events around ``--iters`` steps after a
warm-up, medians of ``--reps`` rounds with the arms alternating inside every round.  Needs a GPU; prints one JSON line with
the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import types

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.convnet import Net  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
OPTS = {"FlatSGD": (b2.FlatSGD, dict(lr=0.05, momentum=0.9, weight_decay=5e-4)),
        "FlatAdamW": (b2.FlatAdamW, dict(lr=1e-3, weight_decay=1e-2))}


def _arm(workload, opt_name, graph, dev, size):
    torch.manual_seed(1234)
    if workload == "Net":
        model, x = Net().to(dev), torch.randn(128 // size, 1, 28, 28, device=dev)
        y = torch.randint(0, 10, (x.shape[0],), device=dev)
        autocast = False
    else:
        model = ResNet18().to(dev).to(memory_format=torch.channels_last)
        x = torch.randn(32, 3, 32, 32, device=dev).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (32,), device=dev)
        autocast = True
    ddp = b2.DistributedDataParallel(model)
    Flat, hp = OPTS[opt_name]
    opt = Flat(ddp, sharded=size > 1, **({"capturable": True} if graph else {}), **hp)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast, cache_enabled=False):
            loss = F.cross_entropy(ddp(x), y)
        loss.backward()
        b2.average_gradients(ddp)
        opt.step()

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream(dev).wait_stream(s)
    if not graph:
        return step
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return lambda: (g.replay(), step)[0]       # `step` keeps the static inputs, the model and the optimizer alive


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    res = dict(gpu_info(), n_gpus=size, iters=ARGS.iters, reps=ARGS.reps, sharded=size > 1)
    for workload in ("Net", "ResNet-18"):
        for opt_name in OPTS:
            arms = {a: _arm(workload, opt_name, a == "graph", dev, size) for a in ("eager", "graph")}
            runs = {a: [] for a in arms}
            for fn in arms.values():
                _timed(fn, 10, dev)
            for _ in range(ARGS.reps):
                for a, fn in arms.items():
                    runs[a].append(_timed(fn, ARGS.iters, dev) * 1e3)       # us per step
            med = {a: statistics.median(v) for a, v in runs.items()}
            res[f"{workload} {opt_name}"] = {"eager_us": round(med["eager"], 1), "graph_us": round(med["graph"], 1),
                                             "speedup": round(med["eager"] / med["graph"], 3),
                                             "runs_us": {a: [round(t, 1) for t in v] for a, v in runs.items()}}
    if size == 1:
        res["note"] = "one GPU: DDP at world size 1 (no exchange); the sharded multi-GPU form is not measured by this run"
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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < ARGS.gpus:
        raise SystemExit(f"graph_step_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
