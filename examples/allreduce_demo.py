#!/usr/bin/env python
"""The reference's ``gloo.py`` / ``allreduce.py`` scenario (gloo.py:37-47): a 2x2 tensor is all-reduced 4 times
(it grows by x world_size each round), once with the library collective and once with the hand-rolled ring
``allreduce(send, recv)`` (gloo.py:8-34, fixed -- see ring.py).

    python examples/allreduce_demo.py [--size 4] [--backend gloo|b200]     # fork-N launcher
    mpirun -n 4 python examples/allreduce_demo.py --backend mpi             # rank/size from the launcher
    torchrun --nproc-per-node 4 examples/allreduce_demo.py --backend mpi

On ``--backend b200`` the collective is the fused sm_90a peer-memory kernel (no NCCL on that call)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dist_tuto.pth_b200 as dist  # noqa: E402
from dist_tuto.pth_b200.utils import say  # noqa: E402  (print as one write: ranks share the terminal)


def run(rank, size):
    cuda = torch.cuda.is_available() and "nccl" in str(torch.distributed.get_backend())
    dev = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    torch.manual_seed(rank)
    t = torch.rand(2, 2, device=dev)
    r = t.clone()
    for _ in range(4):
        c = t.clone()
        dist.all_reduce(c, dist.reduce_op.SUM)
        t = c
        out = torch.empty_like(r)
        dist.allreduce(r, out)                    # ring on isend/recv
        r = out
    if cuda:
        torch.cuda.synchronize()
    say("Rank ", rank, "\n collective:", t.flatten().tolist(), "\n ring:      ", r.flatten().tolist())
    assert torch.allclose(t, r, rtol=1e-4)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4)
    ap.add_argument("--backend", default="gloo")
    a = ap.parse_args()
    if a.backend == "mpi":
        dist.init_processes(0, 0, run, backend="mpi")     # tuto.md:393-398 recipe
    else:
        dist.launch(run, size=a.size, backend=a.backend)
