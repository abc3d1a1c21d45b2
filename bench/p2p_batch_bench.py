"""Ring and all-pairs exchanges with ``batch_isend_irecv`` across GPUs over NVSwitch: one peer-memory batch vs separate
``isend`` / ``irecv`` vs NCCL's ``batch_isend_irecv``.

Runs with ``backend="b200"``, so the ``batch`` arm is ``comm.batch_isend_irecv`` (one launch of the batch kernel of
``csrc/p2p.cu`` per exchange), the ``single`` arm is one ``comm.isend`` / ``comm.irecv`` per op (one launch each, on the
same peer-memory kernels) and the ``nccl`` arm is ``torch.distributed.batch_isend_irecv`` on NCCL.  Every exchange lists
its sends before its receives.  Times are CUDA events on the current stream around ``--iters`` exchanges, after warm-up,
MAX over ranks.  It compares GPUs, so it refuses to run on fewer than two.  The JSON output records the card and its power
limit, read in the same run.

    python bench/p2p_batch_bench.py --gpus 8 --out p2p_batch_world8.json
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200 import comm  # noqa: E402

ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None
SIZES = [4, 1024, 16 << 10, 256 << 10, 1 << 20, 8 << 20]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"device": name, "power_limit_w": float(power)}


def peers(rank, size, pattern):
    """(destinations, sources) of one exchange."""
    if pattern == "ring":
        return [(rank + 1) % size], [(rank - 1) % size]
    others = [q for q in range(size) if q != rank]
    return others, others


def exchange(arm, x, outs, dsts, srcs):
    if arm == "batch":
        reqs = comm.batch_isend_irecv([comm.P2POp(comm.isend, x, q) for q in dsts] +
                                      [comm.P2POp(comm.irecv, outs[q], q) for q in srcs])
    elif arm == "single":
        reqs = [comm.isend(x, q) for q in dsts] + [comm.irecv(outs[q], q) for q in srcs]
    else:
        reqs = dist.batch_isend_irecv([dist.P2POp(dist.isend, x, q) for q in dsts] +
                                      [dist.P2POp(dist.irecv, outs[q], q) for q in srcs])
    for r in reqs:
        r.wait()


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    rows = []
    for pattern in ("ring", "all_pairs"):
        dsts, srcs = peers(rank, size, pattern)
        for nbytes in SIZES:
            x = torch.ones(nbytes, dtype=torch.uint8, device=dev)
            outs = {q: torch.zeros_like(x) for q in srcs}
            iters = ARGS.iters if nbytes <= (1 << 20) else max(5, ARGS.iters // 10)
            row = {"pattern": pattern, "bytes": nbytes, "world": size}
            for arm in ("batch", "single", "nccl"):
                for _ in range(5):
                    exchange(arm, x, outs, dsts, srcs)
                torch.cuda.synchronize()
                dist.barrier()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    exchange(arm, x, outs, dsts, srcs)
                e1.record()
                e1.synchronize()
                us = torch.tensor([e0.elapsed_time(e1) / iters * 1e3], device=dev)
                dist.all_reduce(us, op=dist.ReduceOp.MAX)
                row[arm + "_us"] = float(us.item())
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    if rank == 0 and ARGS.out:
        os.makedirs(os.path.dirname(os.path.abspath(ARGS.out)), exist_ok=True)
        json.dump({"rows": rows, "backend": "b200", "gpu": gpu_info()}, open(ARGS.out, "w"), indent=1)
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=0, help="world size (default: every visible GPU)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default="")
    ARGS = ap.parse_args()
    n = ARGS.gpus or torch.cuda.device_count()
    if n < 2 or torch.cuda.device_count() < n:
        sys.exit(f"p2p_batch_bench compares exchanges between GPUs: it needs at least 2, {torch.cuda.device_count()} "
                 "visible")
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=n, backend="b200", join_timeout_s=900)
