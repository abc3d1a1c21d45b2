#!/usr/bin/env python
"""What parameter groups cost FlatSGD and FlatAdamW.

    python bench/param_groups_bench.py --gpus 1 [--iters 100] [--reps 5] [--out result.json]

* ``step()`` on the parameters and gradients of a ResNet-18 (DistributedDataParallel buckets of ``--bucket-mb``), device time
  per call (CUDA events around ``--iters`` calls after a warm-up, medians of ``--reps`` rounds, the arms alternating inside
  every round), for FlatSGD (momentum 0.9, weight decay 5e-4) and FlatAdamW, each:
    no groups         param_groups=None: sgd_flat / adamw_flat
    2 groups          no weight decay on the ndim <= 1 tensors (the grouped kernels)
    1 per tensor      one group per parameter tensor (62 groups)
* per bucket of 1, 8, 25 and 64 MB of fp32 gradients, the sharded kernel at world size 1, ungrouped against grouped with 64
  groups in runs of 1..4096 vectors: sharded_sgd / sharded_sgd_grouped and sharded_adamw / sharded_adamw_grouped.

Needs a GPU.  Prints one JSON line with the card's name and power limit read in the same run.
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
SGD_HP = dict(lr=0.1, momentum=0.9, weight_decay=5e-4)
ADAMW_HP = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)


def step_arms(dev):
    arms = {}
    for name, Flat, hp in (("FlatSGD", b2.FlatSGD, SGD_HP), ("FlatAdamW", b2.FlatAdamW, ADAMW_HP)):
        for label in ("no groups", "2 groups", "1 per tensor"):
            torch.manual_seed(1234)
            model = ResNet18(num_classes=1000).to(dev)
            ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
            params = list(model.parameters())
            groups = {"no groups": None, "2 groups": [{"params": [p for p in params if p.ndim <= 1], "weight_decay": 0.0}],
                      "1 per tensor": [{"params": [p], "lr": hp["lr"] * (0.5 + i / len(params))} for i, p in enumerate(params)]}
            opt = Flat(ddp, zero_grad=False, param_groups=groups[label], **hp)
            for gb in opt.buckets:
                gb.flat.normal_(std=1e-3)
            arms[f"{name} {label}"] = opt.step
    return arms, {"tensors": len(params), "buckets": len(opt.buckets), "bucket_mb": ARGS.bucket_mb}


def bucket_arms(w, mb, dev):
    n_vec = (mb << 20) // 16
    n = n_vec * 4
    gh, ph = w.alloc(n, torch.float32), w.alloc_bytes(n * 4, ll=False)
    gh.local[:n].normal_()
    m_shard, v_shard = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    g = torch.Generator().manual_seed(mb)
    lens = torch.randint(1, 4097, (n_vec // 2048 + 64,), generator=g)
    ids = torch.arange(lens.numel()) % 64
    gmap = torch.repeat_interleave(ids, lens)[:n_vec].to(torch.uint8).to(dev)
    assert gmap.numel() == n_vec
    lrs, wds = [0.1 * (1 + i / 64) for i in range(64)], [5e-4 if i % 2 else 0.0 for i in range(64)]
    sc = adamw_scalars(1e-3, (0.9, 0.999), 1e-8, 1e-2, 10)
    per = [adamw_scalars(1e-3 * (1 + i / 64), (0.9, 0.999), 1e-8, wds[i], 10) for i in range(64)]
    decays, steps = [s[0] for s in per], [s[4] for s in per]
    C, r = w.C, w.rank
    return {
        "sharded_sgd": lambda: C.sharded_sgd(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, n_vec, 0.1, 0.9, 5e-4, False, 1.0,
                                             False, r, 1, w.max_blocks),
        "sharded_sgd_grouped": lambda: C.sharded_sgd_grouped(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, gmap, n_vec, lrs, wds,
                                                             0.9, False, 1.0, False, r, 1, w.max_blocks),
        "sharded_adamw": lambda: C.sharded_adamw(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, v_shard, n_vec, sc, 1.0, False,
                                                 r, 1, w.max_blocks),
        "sharded_adamw_grouped": lambda: C.sharded_adamw_grouped(False, gh.ptrs, ph.ptrs, gh.sig_ptrs, m_shard, v_shard, gmap,
                                                                 n_vec, sc, decays, steps, 1.0, False, r, 1, w.max_blocks)}


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
    res["sharded_w1_buckets_ms"] = {f"{mb}MB": _rounds(bucket_arms(w, mb, dev), ARGS.iters, dev) for mb in (1, 8, 25, 64)}
    res["note"] = "world size 1: no peer traffic in the bucket arms; multi-GPU times are not measured by this run"
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
        raise SystemExit(f"param_groups_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
