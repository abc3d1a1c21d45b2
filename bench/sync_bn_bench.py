"""SyncBatchNorm (parallel/sync_bn.py, csrc/batchnorm.cu) on one GPU: every ResNet-18 BatchNorm shape at per-GPU batch 64,
224x224, bf16, channels_last.

* per layer: forward and forward+backward of ``b2.SyncBatchNorm`` against cuDNN ``BatchNorm2d`` (world size 1; the exchange
  is skipped there, the same kernels run);
* per kernel: time of each of the four kernels alone and its achieved HBM bytes/s, from the bytes the shape implies (stats:
  read x; apply: read x, write y; backward reduce: read x and dy; backward apply: read x and dy, write dx) over CUDA-event
  time;
* a whole ResNet-18 step (bf16 autocast, channels_last, SGD) with ``nn.BatchNorm2d`` and with the converted model.

Comparisons against ``torch.nn.SyncBatchNorm`` at world size >= 2 need several GPUs and are not part of this one-GPU run.
The card name and power limit are read in the same run.  One JSON line per row, then a summary line.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.models.resnet import ResNet18  # noqa: E402
from dist_tuto.pth_b200.ops import _ext  # noqa: E402
from dist_tuto.pth_b200.parallel.sync_bn import exchange_numel  # noqa: E402

SHAPES = [(64, 112), (64, 56), (128, 28), (256, 14), (512, 7)]   # (channels, spatial side) of ResNet-18's 20 BN layers
COUNT = {(64, 112): 1, (64, 56): 4, (128, 28): 5, (256, 14): 5, (512, 7): 5}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (power limit unread: {e!r})"


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps                            # us per call


def layer_rows(batch, reps):
    K = _ext.C()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for C, s in SHAPES:
        x = torch.randn(batch, C, s, s, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dy = torch.randn_like(x)
        ref = nn.BatchNorm2d(C).cuda()
        mine = b2.SyncBatchNorm(C).cuda()
        xr = x.detach().requires_grad_(True)

        def fwd(m):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return m(xr)

        def fb(m):
            fwd(m).backward(dy)

        row = {"C": C, "hw": s, "layers": COUNT[(C, s)],
               "cudnn_fwd_us": timed(lambda: fwd(ref), reps), "ours_fwd_us": timed(lambda: fwd(mine), reps),
               "cudnn_fwd_bwd_us": timed(lambda: fb(ref), reps), "ours_fwd_bwd_us": timed(lambda: fb(mine), reps)}
        # the four kernels alone
        w, bias = mine.weight.detach(), mine.bias.detach()
        rm, rv = mine.running_mean, mine.running_var
        tickets = torch.zeros(C, dtype=torch.int32, device="cuda")
        ex = torch.empty(exchange_numel(1 + 2 * C, 1), dtype=torch.float64, device="cuda")
        exb = torch.empty(exchange_numel(2 * C, 1), dtype=torch.float64, device="cuda")
        stats = torch.empty(2 * C + 1, dtype=torch.float64, device="cuda")
        y, dx = torch.empty_like(x), torch.empty_like(x)
        gw, gb = torch.empty_like(w), torch.empty_like(w)
        calls = {
            "bn_stats": (1, lambda: K.bn_launch(0, x, None, None, ex, stats, tickets, None, None, None, None, None, None, None,
                                                0.0, 0.0, sms)),
            "bn_apply": (2, lambda: K.bn_launch(1, x, None, y, ex, stats, None, w, bias, rm, rv, None, None, None, 0.1, 1e-5,
                                                sms)),
            "bn_backward_reduce": (2, lambda: K.bn_launch(2, x, dy, None, exb, stats, tickets, None, None, None, None, None,
                                                          gw, gb, 0.0, 0.0, sms)),
            "bn_backward_apply": (3, lambda: K.bn_launch(3, x, dy, dx, exb, stats, None, w, None, None, None, None, None, None,
                                                         0.0, 0.0, sms)),
        }
        nbytes = x.numel() * x.element_size()
        for name, (tensors, fn) in calls.items():
            us = timed(fn, reps)
            row[f"{name}_us"] = us
            row[f"{name}_TBps"] = tensors * nbytes / (us * 1e-6) / 1e12
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def resnet_step(batch, steps, sync):
    torch.manual_seed(0)
    net = ResNet18(num_classes=1000).cuda().to(memory_format=torch.channels_last)
    if sync:
        net = b2.SyncBatchNorm.convert_sync_batchnorm(net)
    opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9)
    x = torch.randn(batch, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (batch,), device="cuda")

    def step():
        opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(net(x), t)
        loss.backward()
        opt.step()

    return timed(step, steps, warm=5) / 1e3                          # ms per step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3, help="alternated rounds of the whole-step comparison")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sync_bn_bench needs a CUDA GPU")
    who = card()
    rows = layer_rows(a.batch, a.reps)
    bn, sy = [], []
    for _ in range(a.rounds):
        bn.append(resnet_step(a.batch, a.steps, False))
        sy.append(resnet_step(a.batch, a.steps, True))
    summary = {"card": who, "batch": a.batch, "resnet18_step_ms_batchnorm": sorted(bn)[len(bn) // 2],
               "resnet18_step_ms_syncbn": sorted(sy)[len(sy) // 2], "rounds_batchnorm": bn, "rounds_syncbn": sy,
               "bn_fwd_bwd_us_total_cudnn": sum(r["cudnn_fwd_bwd_us"] * r["layers"] for r in rows),
               "bn_fwd_bwd_us_total_ours": sum(r["ours_fwd_bwd_us"] * r["layers"] for r in rows),
               "world_ge_2": "not measured (one GPU)"}
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
