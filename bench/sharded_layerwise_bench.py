#!/usr/bin/env python
"""Sharded LAMB / LARS against the path it replaces: all-reduce + lamb_flat / lars_flat versus sharded_lamb / sharded_lars,
per bucket and in the ResNet-18 step.

    python bench/sharded_layerwise_bench.py --gpus 8 [--iters 100] [--reps 5] [--steps 20] [--out result.json]

Per fp32 bucket (1, 8, 25, 64 MB laid out as 3x3x256x256 conv weights each followed by two 512-element norm tensors, and
ResNet-18's parameters as one bucket), device time per call (CUDA events around `--iters` calls after a warm-up, medians of
`--reps` rounds, the arms alternating inside every round, max over ranks):
  allreduce+lamb_flat    the bucket's fused all-reduce with the 1/W scale, then lamb_flat (two launches) with re-zeroing --
                         what FlatLAMB(sharded=False) runs per bucket
  sharded_lamb           the two sharded launches: gradient exchange, LAMB on the owned slice, per-tensor sums across the
                         ranks, parameter all-gather, re-zeroing
  allreduce+lars_flat / sharded_lars   the same for LARS
Then the ResNet-18 bf16-autocast step (DistributedDataParallel + FlatLAMB, fp32 buckets) with sharded=False and sharded=True,
alternating, device-timed.

With --gpus 1 the all-reduce is a no-op, the sharded kernels run with one rank (no peer traffic) and FlatLAMB(sharded=True)
is the unsharded path: that run times the kernels' single-GPU cost only and says nothing about NVLink.  Needs GPUs: without
one it fails.  Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.ops.optim import lamb_scalars  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import _timed, gpu_info  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
LAMB = lamb_scalars(1e-3, (0.9, 0.999), 1e-6, 0.01, 10)
LARS = dict(lr=0.1, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-3, eps=1e-8, nesterov=False)


def conv_layout(n):
    """Tensor sizes filling `n` elements: 3x3x256x256 weights, each followed by two 512-element norm tensors."""
    out, left = [], n
    while left > 0:
        for k in (589824, 512, 512):
            if left > 0:
                out.append(min(k, left))
                left -= (out[-1] + 3) // 4 * 4
    return out


def resnet18_layout():
    return [p.numel() for p in ResNet18(num_classes=1000).parameters()]


def bucket_arms(w, numels, dev):
    """The four per-bucket arms on symmetric buffers holding tensors of `numels` elements (offsets at multiples of 4)."""
    W, C = w.world, w.C
    offsets, o = [], 0
    for k in numels:
        offsets.append(o)
        o += (k + 3) // 4 * 4
    n_vec = ((o + 3) // 4 + W - 1) // W * W
    n, T = n_vec * 4, len(numels)
    adapt = [k > 512 for k in numels]
    gh, ph, sh = w.alloc(n, torch.float32), w.alloc_bytes(n * 4, ll=False), w.alloc_bytes(16 * T, ll=False)
    g = gh.local[:n]
    g.normal_()
    p_flat = ph.view(torch.float32, n)
    p_flat.normal_()
    f = lambda k: torch.zeros(k, device=dev)  # noqa: E731
    ut, unc = C.layerwise_table(offsets, numels, adapt, n, dev)
    uws = (f(2 * unc), torch.zeros(T, dtype=torch.int32, device=dev), torch.zeros(2 * T, dtype=torch.float64, device=dev), f(T))
    st = C.sharded_layerwise_table(offsets, numels, adapt, n, w.rank, W, dev)
    sws = (f(2 * st.n_chunks), torch.zeros(T, dtype=torch.int32, device=dev), f(T))
    m, v, ms, vs, gs = f(n), f(n), f(n // W), f(n // W), f(n // W)
    head = (False, gh.ptrs, ph.ptrs, sh.ptrs, gh.sig_ptrs)

    def ar_lamb():
        w.all_reduce_(g, scale=1.0 / W, handle=gh)
        C.lamb_flat(p_flat, m, v, g, ut, unc, *uws, LAMB, True)

    def sh_lamb():
        C.sharded_lamb(*head, ms, vs, st, *sws, n_vec, LAMB, 1.0 / W, True, w.rank, W, w.max_blocks)

    lars = (LARS["lr"], LARS["momentum"], LARS["weight_decay"], LARS["trust_coefficient"], LARS["eps"], LARS["nesterov"])

    def ar_lars():
        w.all_reduce_(g, scale=1.0 / W, handle=gh)
        C.lars_flat(p_flat, m, g, ut, unc, *uws, *lars, True)

    def sh_lars():
        C.sharded_lars(*head, ms, gs, st, *sws, n_vec, *lars, 1.0 / W, True, w.rank, W, w.max_blocks)

    arms = {"allreduce+lamb_flat": ar_lamb, "sharded_lamb": sh_lamb, "allreduce+lars_flat": ar_lars, "sharded_lars": sh_lars}
    return arms, (gh, ph, sh), {"elements": n, "tensors": T, "chunks_unsharded": unc, "chunks_this_rank": st.n_chunks}


def resnet_arm(sharded, dev):
    torch.manual_seed(1234)
    model = ResNet18(num_classes=1000).to(dev).to(memory_format=torch.channels_last)
    ddp = DistributedDataParallel(model, bucket_cap_bytes=ARGS.bucket_mb << 20)
    opt = b2.FlatLAMB(ddp, lr=1e-3, sharded=sharded)
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
    res = dict(gpu_info(), n_gpus=size, iters=ARGS.iters, reps=ARGS.reps, buckets_ms={}, layouts={}, resnet18_step_ms={})
    layouts = {f"{mb}MB": conv_layout((mb << 20) // 4) for mb in (1, 8, 25, 64)}
    layouts["resnet18"] = resnet18_layout()
    for name, numels in layouts.items():
        arms, keep, info = bucket_arms(w, numels, dev)
        runs = {k: [] for k in arms}
        for fn in arms.values():
            _timed(fn, 5, dev)                                    # warm-up
        for _ in range(ARGS.reps):
            for k, fn in arms.items():
                runs[k].append(_timed(fn, ARGS.iters, dev))
        res["buckets_ms"][name] = {k: {"median": statistics.median(t), "runs": [round(x, 5) for x in t]} for k, t in runs.items()}
        res["layouts"][name] = info
        del arms, keep
    torch.backends.cudnn.benchmark = True
    steps = {"sharded=False": resnet_arm(False, dev), "sharded=True": resnet_arm(True, dev)}
    runs = {k: [] for k in steps}
    for fn in steps.values():
        _timed(fn, ARGS.warmup, dev)
    for _ in range(ARGS.reps):
        for k, fn in steps.items():
            runs[k].append(_timed(fn, ARGS.steps, dev))
    res["resnet18_step_ms"] = {k: {"median": statistics.median(t), "runs": [round(x, 4) for x in t]} for k, t in runs.items()}
    res["resnet18"] = {"per_gpu_batch": ARGS.batch, "res": ARGS.res, "bucket_mb": ARGS.bucket_mb, "steps": ARGS.steps}
    if size == 1:
        res["note"] = ("one GPU: no peer traffic, and FlatLAMB(sharded=True) is the unsharded path; multi-GPU times are not "
                       "measured by this run")
    if rank == 0:
        line = json.dumps(res)
        print(line, flush=True)
        if ARGS.out:
            os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
            with open(ARGS.out, "w") as fh:
                fh.write(line + "\n")
    import torch.distributed as dist
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--bucket-mb", type=int, default=25)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < ARGS.gpus:
        raise SystemExit(f"sharded_layerwise_bench.py measures on {ARGS.gpus} GPU(s); {torch.cuda.device_count()} visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
