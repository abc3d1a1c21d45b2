#!/usr/bin/env python
"""Gradient accumulation with ``DistributedDataParallel.no_sync()``: what k micro-batches per optimizer step cost and save.

    python bench/accumulation_bench.py --gpus 1 [--iters 20] [--reps 5] [--out result.json]

Workloads (backend "b200", DistributedDataParallel at world size ``--gpus``, FlatSGD momentum 0.9, weight decay 5e-4):
    Net          the tutorial's Net, micro-batch 128 per GPU
    ResNet-18    micro-batch 32 per GPU, 3 x 32 x 32, bf16 autocast, channels_last
at k = 1, 2, 4, 8 micro-batches per optimizer step.  One cycle is k - 1 forward / backward passes under ``no_sync()``, the
last one, ``average_gradients`` and ``step()``.  Reported per (workload, k):
    counted      bucket exchange launches per optimizer step (the DDP engine's launches, counted in the run; at world size 1
                 a launch exchanges nothing) and the NVLink bytes one GPU would send per optimizer step at world sizes 2
                 and 8 (two-shot all-reduce of every fp32 bucket, the model of bench/allreduce_sweep.py), from the bucket
                 sizes; per sample the bytes fall as 1 / k
    eager        device time per cycle, capturable=False, every launch issued from Python
    graph        device time per cycle, capturable=True, one replay of a captured cycle
CUDA events around ``--iters`` cycles after a warm-up, medians of ``--reps`` rounds with the arms alternating.  Needs a GPU;
prints one JSON line with the card's name and power limit read in the same run.
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
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
KS = (1, 2, 4, 8)
HP = dict(lr=0.05, momentum=0.9, weight_decay=5e-4)


def _arm(workload, k, graph, dev):
    torch.manual_seed(1234)
    if workload == "Net":
        model = Net().to(dev)
        xs = [torch.randn(128, 1, 28, 28, device=dev) for _ in range(k)]
        autocast = False
    else:
        model = ResNet18().to(dev).to(memory_format=torch.channels_last)
        xs = [torch.randn(32, 3, 32, 32, device=dev).contiguous(memory_format=torch.channels_last) for _ in range(k)]
        autocast = True
    ys = [torch.randint(0, 10, (x.shape[0],), device=dev) for x in xs]
    ddp = b2.DistributedDataParallel(model)
    opt = b2.FlatSGD(ddp, **({"capturable": True} if graph else {}), **HP)

    def fwd_bwd(x, y):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast, cache_enabled=False):
            loss = F.cross_entropy(ddp(x), y) / k
        loss.backward()

    def cycle():
        for x, y in zip(xs[:-1], ys[:-1]):
            with ddp.no_sync():
                fwd_bwd(x, y)
        fwd_bwd(xs[-1], ys[-1])
        b2.average_gradients(ddp)
        opt.step()

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(3):
            cycle()
    torch.cuda.current_stream(dev).wait_stream(s)
    if not graph:
        return cycle, ddp
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cycle()
    return (lambda: (g.replay(), cycle)[0]), ddp        # `cycle` keeps the static inputs, the model and the optimizer alive


def _counted(fn, ddp):
    """Bucket launches of one eager cycle, and the two-shot NVLink bytes per GPU per optimizer step at worlds 2 and 8."""
    launches = []
    orig = DistributedDataParallel._launch

    def counting(self, b):
        launches.append(b.gb.numel * b.gb.flat.element_size())
        return orig(self, b)
    DistributedDataParallel._launch = counting
    try:
        fn()
    finally:
        DistributedDataParallel._launch = orig
    torch.cuda.synchronize()
    return {"exchange_launches_per_step": len(launches), "buckets": len(ddp.buckets),
            "nvlink_bytes_per_step_w2": round(sum(2 * n * 1 / 2 for n in launches)),
            "nvlink_bytes_per_step_w8": round(sum(2 * n * 7 / 8 for n in launches))}


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    res = dict(gpu_info(), n_gpus=size, iters=ARGS.iters, reps=ARGS.reps, optimizer="FlatSGD")
    for workload in ("Net", "ResNet-18"):
        for k in KS:
            arms = {a: _arm(workload, k, a == "graph", dev) for a in ("eager", "graph")}
            row = _counted(*arms["eager"])
            runs = {a: [] for a in arms}
            for fn, _ in arms.values():
                _timed(fn, 3, dev)
            for _ in range(ARGS.reps):
                for a, (fn, _) in arms.items():
                    runs[a].append(_timed(fn, ARGS.iters, dev) * 1e3)       # us per cycle
            med = {a: statistics.median(v) for a, v in runs.items()}
            row.update(eager_us_per_cycle=round(med["eager"], 1), graph_us_per_cycle=round(med["graph"], 1),
                       runs_us={a: [round(t, 1) for t in v] for a, v in runs.items()})
            res[f"{workload} k={k}"] = row
            for _, d in arms.values():
                d.remove_hooks()
            del arms
    if size == 1:
        res["note"] = ("one GPU: DDP at world size 1, where a bucket launch exchanges nothing; the NVLink bytes are counted "
                       "from the bucket sizes, and multi-GPU times are not measured by this run")
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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < ARGS.gpus:
        raise SystemExit(f"accumulation_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
