#!/usr/bin/env python
"""Point-to-point messaging demos of the tutorial (tuto.md:77-120) on this framework.

    python examples/p2p_demo.py [--backend gloo|b200]

blocking:      rank 0 increments a tensor and ``send``s it, rank 1 ``recv``s it -> both print 1.0
non-blocking:  same with ``isend``/``irecv``; the data is only valid after ``req.wait()``.
On ``--backend b200`` the tensors live on the GPUs and the transfer runs on the library's peer-memory point-to-point
kernels (``csrc/p2p.cu``) over NVSwitch; on ``--backend nccl`` it is NCCL p2p."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dist_tuto.pth_b200 as dist  # noqa: E402
from dist_tuto.pth_b200.utils import say  # noqa: E402  (print as one write: ranks share the terminal)

CUDA = False


def run(rank, size):
    dev = torch.device("cuda", torch.cuda.current_device()) if CUDA else torch.device("cpu")
    tensor = torch.zeros(1, device=dev)
    if rank == 0:
        tensor += 1
        dist.send(tensor=tensor, dst=1)           # blocks until the buffer may be reused
    else:
        dist.recv(tensor=tensor, src=0)           # receiver pre-allocates
    say("[blocking]     Rank ", rank, " has data ", tensor[0].item())

    tensor = torch.zeros(1, device=dev)
    if rank == 0:
        tensor += 1
        req = dist.isend(tensor=tensor, dst=1)
        say("Rank 0 started sending")
    else:
        req = dist.irecv(tensor=tensor, src=0)
        say("Rank 1 started receiving")
    req.wait(sync=True)                           # do not touch `tensor` before this returns
    say("[non-blocking] Rank ", rank, " has data ", tensor[0].item())


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="gloo")
    a = ap.parse_args()
    CUDA = a.backend in ("b200", "nccl")
    dist.launch(run, size=2, backend=a.backend)
