"""Bytes that really cross NVLink per all-reduce, from the GPU's own link counters (not from an algorithm formula).

    python bench/nvlink_bytes.py --gpus N [--out gpurun_out/nvlink_bytes_N.json]

Nsight Compute cannot profile these kernels (they spin on their peers, so a replayed or serialised launch deadlocks:
see DESIGN.md section 6), so the traffic is read from NVML's per-device NVLink data counters
(``NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX / _RX``, KiB, summed over the links; ``nvidia-smi nvlink -gt d`` as fallback)
before and after ``iters`` back-to-back all-reduces of one variant and size.  Reported per all-reduce and per GPU next to
the model used in bench/allreduce_sweep.py (`link_bytes()`), for every variant of csrc/allreduce.cu and for NCCL.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402

import types
ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None


class LinkCounters:
    """(tx_bytes, rx_bytes) of one GPU, summed over its NVLink links."""

    def __init__(self, dev):
        self.uuid = "GPU-" + str(torch.cuda.get_device_properties(dev).uuid)
        self.how = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByUUID(self.uuid)
            self.ids = (pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX, pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX)
            self.read_nvml()
            self.how = "nvml field values (KiB)"
        except Exception as e:  # noqa: BLE001
            self.nvml_error = repr(e)
            self.read_smi()
            self.how = "nvidia-smi nvlink -gt d"

    def read_nvml(self):
        vals = self.nv.nvmlDeviceGetFieldValues(self.h, [(i, 0xFFFFFFFF) for i in self.ids])     # scope: all links
        out = []
        for v in vals:
            if v.nvmlReturn != 0:
                raise RuntimeError(f"field {v.fieldId}: nvmlReturn {v.nvmlReturn}")
            out.append(int(v.value.ullVal) * 1024)
        return tuple(out)

    def read_smi(self):
        txt = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", self.uuid], capture_output=True, text=True, timeout=20).stdout
        tx = sum(int(m) for m in re.findall(r"Data Tx:\s*(\d+)\s*KiB", txt))
        rx = sum(int(m) for m in re.findall(r"Data Rx:\s*(\d+)\s*KiB", txt))
        if "Data Tx" not in txt:
            raise RuntimeError("no NVLink data counters in nvidia-smi output: " + txt[:200])
        return tx * 1024, rx * 1024

    def read(self):
        return self.read_nvml() if self.how and self.how.startswith("nvml") else self.read_smi()


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    w = symm.lookup_world(None)
    lc = LinkCounters(dev)
    max_bytes = ARGS.max_mb << 20
    hd = w.alloc(max_bytes // 4, torch.float32)
    plain = torch.ones(max_bytes // 4, device=dev)
    variants = [("ll", 3), ("oneshot", 0), ("twoshot", 1)] + ([("nvls", 2)] if w.multicast else []) + [("nccl", -1)]

    def model(name, nbytes):
        return {"ll": 2 * nbytes * (size - 1), "oneshot": nbytes * (size - 1), "twoshot": 2 * nbytes * (size - 1) / size,
                "nvls": 2 * nbytes / size, "nccl": 2 * nbytes * (size - 1) / size}[name]

    rows = []
    for nbytes in (64 << 10, 1 << 20, max_bytes):
        n = nbytes // 4
        t = hd.local[:n]
        iters = max(20, min(2000, (2 << 30) // nbytes))
        for name, v in variants:
            if v == 3 and nbytes > symm.LL_CAP_VEC * 16:
                continue
            if v == 0 and nbytes > (8 << 20):
                continue
            fn = (lambda: dist.all_reduce(plain[:n])) if v < 0 else (lambda v=v: w.all_reduce_(t, scale=1.0 / size, handle=hd, variant=v))
            t.fill_(1.0)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            dist.barrier()
            torch.cuda.synchronize()
            time.sleep(0.05)
            tx0, rx0 = lc.read()
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
            dist.barrier()          # every rank has finished its kernels: all traffic of the batch is counted
            torch.cuda.synchronize()
            time.sleep(0.05)
            tx1, rx1 = lc.read()
            # the two barriers are NCCL all-reduces of a few bytes: negligible next to iters x nbytes
            row = {"variant": name, "bytes": nbytes, "iters": iters, "tx_per_allreduce": (tx1 - tx0) / iters,
                   "rx_per_allreduce": (rx1 - rx0) / iters, "model_tx_per_allreduce": model(name, nbytes)}
            row["tx_over_payload"] = row["tx_per_allreduce"] / nbytes
            row["tx_over_model"] = row["tx_per_allreduce"] / row["model_tx_per_allreduce"]
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    if rank == 0:
        out = {"n_gpus": size, "counter_source": lc.how, "nvml_error": getattr(lc, "nvml_error", None), "gpu": lc.uuid,
               "symm": w.describe(), "rows": rows}
        os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
        json.dump(out, open(ARGS.out, "w"), indent=1)
        print("WROTE", ARGS.out, flush=True)
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--max-mb", type=int, default=64)
    ap.add_argument("--out", default=None)
    ARGS = ap.parse_args()
    ARGS.out = ARGS.out or f"gpurun_out/nvlink_bytes_{ARGS.gpus}.json"
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    if "RANK" in os.environ:
        b2.init_from_env(body, backend="b200")
    else:
        b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=900)
