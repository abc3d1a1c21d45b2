#!/usr/bin/env python
"""Test-set evaluation on one GPU: the forward-only eval kernel against the other in-repo path and cuDNN.

    python bench/eval_bench.py [--sizes 10000 60000] [--calls 50] [--reps 5]

For each N, on N device-resident uint8 samples (synthetic test set) and seeded random parameters, three arms compute the
nll sum and #correct; each arm is warmed up, then timed with CUDA events over `--calls` back-to-back calls, and the arms
alternate `--reps` times in this one process (the median per-call time is reported):
  (a) eval     convnet_eval (csrc/convnet_eval.cu): one launch, sums on the device
  (b) forward  convnet_forward (the training step kernel with backward off, one CTA per sample) + torch nll_loss / argmax
  (c) cudnn    torch Net.eval() in fp32 (cuDNN, TF32 off) on the normalised images + nll_loss / argmax
Prints one JSON line: us per call and samples/s per arm; arm (a)'s achieved FP32 rate from the forward FLOPs of the
layer shapes and its share of the FP32 peak (data sheet, and SMs x 128 lanes x 2 x max SM clock); the device name,
power limit and max SM clock read in the same run; and two result checks at the timed sizes: (a) agrees with (c), and
two calls of (a) are bit-equal.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dist_tuto.pth_b200.data import SyntheticMNIST, EVAL_SEED  # noqa: E402
from dist_tuto.pth_b200.models.convnet import Net  # noqa: E402
from dist_tuto.pth_b200.ops import _ext  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_fused import convnet_forward, pack_params  # noqa: E402

FP32_PEAK_DATASHEET = 67e12        # H100 SXM, dense FP32, at up to 700 W


def forward_flops_per_sample() -> int:
    """Multiply-adds x 2 of the forward pass, from the layer shapes of Net."""
    conv1 = 10 * 24 * 24 * (1 * 5 * 5)         # 10 channels, 24x24 outputs, 25 taps
    conv2 = 20 * 8 * 8 * (10 * 5 * 5)          # 20 channels, 8x8 outputs, 250 taps
    fc1, fc2 = 50 * 320, 10 * 50
    return 2 * (conv1 + conv2 + fc1 + fc2)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"device": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def timed(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls * 1e3      # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10000, 60000])
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    if args.calls < 50:
        raise SystemExit("--calls must be >= 50")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    C = _ext.C()
    info = gpu_info()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    peak_clock = sms * 128 * 2 * info["max_sm_clock_mhz"] * 1e6
    torch.manual_seed(1234)
    net = Net().to(dev).eval()
    params = pack_params(net, dev)
    ds = SyntheticMNIST(n=max(args.sizes), seed=EVAL_SEED)
    mean, std = ds.mean, ds.std
    out = dict(info, sms=sms, calls=args.calls, reps=args.reps, flops_per_sample=forward_flops_per_sample(), runs=[])
    for n in args.sizes:
        x, y = ds.images[:n].to(dev), ds.labels[:n].to(dev)
        result = torch.zeros(3, dtype=torch.float64, device=dev)
        slots = torch.zeros(C.convnet_eval_slot_words(0), dtype=torch.int32, device=dev)
        res = {}

        def arm_eval():
            C.convnet_eval(params, x, y, result, slots, mean, std, None)
            res["a"] = result

        def arm_forward():
            lp = convnet_forward(params, x)
            res["b"] = (F.nll_loss(lp, y, reduction="sum"), (lp.argmax(1) == y).sum())

        def arm_cudnn():
            with torch.no_grad():
                lp = net(((x.float() / 255.0 - mean) / std).unsqueeze(1))
            res["c"] = (F.nll_loss(lp, y, reduction="sum"), (lp.argmax(1) == y).sum())

        arms = {"eval": arm_eval, "forward": arm_forward, "cudnn": arm_cudnn}
        for fn in arms.values():                  # warm-up: module load, cuDNN algorithm choice, allocator
            for _ in range(5):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(timed(fn, args.calls))
        run = {"n": n}
        for k, ts in times.items():
            us = statistics.median(ts)
            run[k] = {"us_per_call": round(us, 2), "samples_per_s": round(n / (us * 1e-6)), "us_all_reps": [round(t, 2) for t in ts]}
        flop_rate = n * out["flops_per_sample"] / (run["eval"]["us_per_call"] * 1e-6)
        run["eval"].update(tflops=round(flop_rate / 1e12, 3), share_fp32_peak_datasheet=round(flop_rate / FP32_PEAK_DATASHEET, 4),
                           share_fp32_peak_at_max_clock=round(flop_rate / peak_clock, 4))
        run["eval_speedup_vs_forward"] = round(run["forward"]["us_per_call"] / run["eval"]["us_per_call"], 3)
        run["eval_speedup_vs_cudnn"] = round(run["cudnn"]["us_per_call"] / run["eval"]["us_per_call"], 3)
        # result checks at this size
        arm_eval()
        first = result.clone()
        arm_eval()
        a = result.tolist()
        arm_cudnn()
        c_loss, c_correct = float(res["c"][0]), int(res["c"][1])
        arm_forward()
        b_loss, b_correct = float(res["b"][0]), int(res["b"][1])
        run["check"] = {"eval_bit_equal_twice": bool(torch.equal(first, result)),
                        "eval": {"nll_sum": a[0], "correct": int(a[1]), "n": int(a[2])},
                        "cudnn": {"nll_sum": c_loss, "correct": c_correct},
                        "forward": {"nll_sum": b_loss, "correct": b_correct},
                        "eval_vs_cudnn_loss_rel": abs(a[0] - c_loss) / abs(c_loss),
                        "eval_vs_cudnn_correct_diff": int(a[1]) - c_correct}
        run["check"]["eval_agrees_with_cudnn"] = (run["check"]["eval_vs_cudnn_loss_rel"] < 1e-5 and int(a[2]) == n
                                                  and abs(int(a[1]) - c_correct) <= max(1, n // 1000))
        out["runs"].append(run)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
