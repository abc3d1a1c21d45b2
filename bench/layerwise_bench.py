#!/usr/bin/env python
"""FlatLAMB and FlatLARS against FlatAdamW, FlatSGD and torch ``_foreach`` implementations of LAMB and LARS.

    python bench/layerwise_bench.py [--iters 100] [--reps 5] [--bucket-mb 25] [--out result.json]

``step()`` on the parameters and gradients of a ResNet-18 (11.7 M fp32 parameters, DistributedDataParallel buckets of
``--bucket-mb``, as bench/adamw_bench.py), device time per call (CUDA events around ``--iters`` calls after a warm-up,
medians of ``--reps`` rounds, the arms alternating inside every round), ``zero_grad=False`` so every call sees the same
gradients:

    FlatLAMB / FlatLARS             two layerwise kernels per bucket (csrc/layerwise.cu)
    FlatAdamW / FlatSGD             one adamw_flat / sgd_flat launch per bucket: the same update without trust ratios
    foreach LAMB / foreach LARS     the same maths on the parameter list with torch._foreach_* ops and _foreach_norm

Achieved bytes/s count what the kernels must move per parameter element, not what they measured: LAMB 40 B (the norms
kernel reads p, g, m, v and writes m, v; the apply kernel reads p, m, v and writes p), LARS 28 B (reads p, g; then reads
p, g, m and writes p, m); with re-zeroed gradients each adds 4 B.  Needs a GPU; prints one JSON line with the card's
name and power limit read in the same run.
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
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel  # noqa: E402
from sharded_sgd_bench import gpu_info  # noqa: E402

LAMB = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=1e-2)
LARS = dict(lr=0.1, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-3, eps=1e-8)
BYTES = {"FlatLAMB": 40, "FlatLARS": 28, "FlatAdamW": 28, "FlatSGD": 20}


def _timed(fn, iters):
    """ms per call of fn over `iters` calls, device-timed."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def _flat_arm(cls, dev, mb, **hp):
    torch.manual_seed(1234)
    ddp = DistributedDataParallel(ResNet18(num_classes=1000).to(dev), bucket_cap_bytes=mb << 20)
    opt = cls(ddp, zero_grad=False, **hp)
    for gb in opt.buckets:
        gb.flat.normal_(std=1e-3)
    return opt.step, sum(gb.numel for gb in opt.buckets), len(opt.buckets)


def _foreach_arm(kind, dev):
    torch.manual_seed(1234)
    ps = [p.detach() for p in ResNet18(num_classes=1000).to(dev).parameters()]
    gs = [torch.randn_like(p) * 1e-3 for p in ps]
    ms, vs = [torch.zeros_like(p) for p in ps], [torch.zeros_like(p) for p in ps]
    adapt = [p.ndim > 1 for p in ps]
    wd = [LAMB["weight_decay"] if a else 0.0 for a in adapt] if kind == "lamb" else \
        [LARS["weight_decay"] if a else 0.0 for a in adapt]
    mask = torch.tensor(adapt, device=dev)
    t = [0]

    def ratios(a, b, num, den):
        w, q = torch.stack(torch._foreach_norm(a)), torch.stack(torch._foreach_norm(b))
        return torch.where(mask & (w > 0) & (q > 0), num(w) / den(w, q), torch.ones_like(w)).unbind()

    def lamb():
        t[0] += 1
        b1, b2_ = LAMB["betas"]
        torch._foreach_lerp_(ms, gs, 1 - b1)
        torch._foreach_mul_(vs, b2_)
        torch._foreach_addcmul_(vs, gs, gs, value=1 - b2_)
        den = torch._foreach_sqrt(vs)
        torch._foreach_div_(den, (1 - b2_ ** t[0]) ** 0.5)
        torch._foreach_add_(den, LAMB["eps"])
        u = torch._foreach_div(ms, den)
        torch._foreach_mul_(u, 1 / (1 - b1 ** t[0]))
        torch._foreach_add_(u, torch._foreach_mul(ps, wd))
        r = ratios(ps, u, lambda w: w, lambda w, q: q)
        torch._foreach_mul_(u, r)
        torch._foreach_add_(ps, u, alpha=-LAMB["lr"])

    def lars():
        r = ratios(ps, gs, lambda w: LARS["trust_coefficient"] * w,
                   lambda w, q: q + LARS["weight_decay"] * w + LARS["eps"])
        d = torch._foreach_add(gs, torch._foreach_mul(ps, wd))
        torch._foreach_mul_(d, r)
        torch._foreach_mul_(ms, LARS["momentum"])
        torch._foreach_add_(ms, d)
        torch._foreach_add_(ps, ms, alpha=-LARS["lr"])

    return lamb if kind == "lamb" else lars


def main(args):
    dev = torch.device("cuda", 0)
    res = dict(gpu_info(), iters=args.iters, reps=args.reps, bucket_mb=args.bucket_mb)
    arms = {}
    arms["FlatLAMB"], n, nb = _flat_arm(b2.FlatLAMB, dev, args.bucket_mb, **LAMB)
    arms["FlatAdamW"], *_ = _flat_arm(b2.FlatAdamW, dev, args.bucket_mb, **LAMB)
    arms["FlatLARS"], *_ = _flat_arm(b2.FlatLARS, dev, args.bucket_mb, **LARS)
    arms["FlatSGD"], *_ = _flat_arm(b2.FlatSGD, dev, args.bucket_mb, lr=0.1, momentum=0.9, weight_decay=1e-4)
    arms["foreach LAMB"] = _foreach_arm("lamb", dev)
    arms["foreach LARS"] = _foreach_arm("lars", dev)
    runs = {k: [] for k in arms}
    for fn in arms.values():
        _timed(fn, 10)
    for _ in range(args.reps):
        for k, fn in arms.items():
            runs[k].append(_timed(fn, args.iters))
    res["resnet18"] = {"parameters": n, "buckets": nb}
    res["step_ms"] = {k: {"median": statistics.median(v), "runs": [round(x, 5) for x in v]} for k, v in runs.items()}
    res["achieved_GBps"] = {k: round(BYTES[k] * n / (res["step_ms"][k]["median"] * 1e-3) / 1e9, 1) for k in BYTES}
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bucket-mb", type=int, default=25)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("layerwise_bench.py measures on a GPU; none is visible")
    main(a)
