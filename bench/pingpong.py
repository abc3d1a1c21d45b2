"""send/recv ping-pong latency at 2 GPUs over NVSwitch (BASELINE.json config #5; ptp.py / tuto.md:82-91).

Runs with ``backend="b200"``, so the ``b2`` arm is our ``send``/``recv`` on the peer-memory point-to-point kernels
(``csrc/p2p.cu``) and the ``torch`` arm is raw ``torch.distributed`` on NCCL.  The JSON output records the card and its
power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402

import types
ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"device": name, "power_limit_w": float(power)}


def body(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device())
    rows = []
    for nbytes in [4, 64, 1024, 16 << 10, 256 << 10, 1 << 20, 16 << 20]:
        t = torch.zeros(max(1, nbytes // 4), device=dev)
        iters = 200 if nbytes <= (1 << 20) else 40

        def pp(send, recv):
            if rank == 0:
                send(t, 1)
                recv(t, 1)
            elif rank == 1:
                recv(t, 0)
                send(t, 0)

        res = {}
        for name, s_fn, r_fn in (("b2", lambda x, p: b2.send(x, dst=p), lambda x, p: b2.recv(x, src=p)),
                                 ("torch", lambda x, p: dist.send(x, dst=p), lambda x, p: dist.recv(x, src=p))):
            for _ in range(5):
                pp(s_fn, r_fn)
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                pp(s_fn, r_fn)
            e1.record()
            e1.synchronize()
            res[name + "_oneway_us"] = e0.elapsed_time(e1) / iters / 2 * 1e3
        res["bytes"] = nbytes
        res["b2_GBs"] = nbytes / (res["b2_oneway_us"] * 1e-6) / 1e9
        rows.append(res)
        if rank == 0:
            print(json.dumps(res), flush=True)
    if rank == 0:
        os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
        json.dump({"rows": rows, "backend": "b200", "gpu": gpu_info()}, open(ARGS.out, "w"), indent=1)
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/pingpong.json")
    ARGS = ap.parse_args()
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    b2.launch(body, size=2, backend="b200", join_timeout_s=600)
