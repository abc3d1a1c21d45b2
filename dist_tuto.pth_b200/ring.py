"""User-level ring all-reduce on point-to-point primitives (layer L3).

Parity: ``allreduce(send, recv)`` of gloo.py:8-34 == allreduce.py:8-34 ==
tuto.md:328-351 -- out-of-place, ``recv <- sum over ranks of send``.

The reference version is buggy as committed (SURVEY §2.6 D3: its staging
buffers start as zeros and are never filled, and it accumulates the function
arguments instead of the received data).  This module implements the semantics
the tutorial describes: at step 0 every rank sends its own tensor to its right
neighbour, at every later step it forwards what it just received, and it adds
each received tensor into the accumulator.  Two staging buffers alternate so a
buffer with an ``isend`` in flight is never overwritten.

``allreduce_chunked`` is the tutorial's "exercise" (tuto.md:354): the
bandwidth-optimal ring (reduce-scatter + all-gather over 1/N-sized chunks),
2(N-1)/N * M bytes per rank instead of (N-1) * M.

Both run on whatever p2p backend ``comm`` picks for the tensors: the
peer-memory kernels of ``csrc/p2p.cu`` for CUDA tensors on ``backend="b200"``,
NCCL send/recv otherwise, gloo for CPU tensors.  The *hot* gradient all-reduce
of the framework does not use this file -- see ``parallel/symm.py``.
"""
from __future__ import annotations

import torch

from . import comm

__all__ = ["allreduce", "allreduce_chunked"]


def _neighbours(group):
    ranks = comm.group_ranks(group)
    me = ranks.index(comm.get_rank())
    n = len(ranks)
    return n, me, ranks[(me - 1 + n) % n], ranks[(me + 1) % n]


def allreduce(send: torch.Tensor, recv: torch.Tensor, group=None) -> torch.Tensor:
    """Ring all-reduce: ``recv[:] = sum_r send_r`` (whole tensor per step)."""
    if send.shape != recv.shape:
        raise ValueError("send and recv must have the same shape")
    size, _, left, right = _neighbours(group)
    send_c = send.contiguous()
    accum = send_c.clone()
    if size > 1:
        bufs = (send_c.clone(), torch.empty_like(send_c))  # bufs[0] holds what we forward next
        for i in range(size - 1):
            out_buf, in_buf = bufs[i % 2], bufs[(i + 1) % 2]
            req = comm.isend(out_buf, right, group=group)
            comm.recv(in_buf, left, group=group)
            accum += in_buf
            req.wait()
    recv.copy_(accum.view_as(recv))
    return recv


def allreduce_chunked(send: torch.Tensor, recv: torch.Tensor, group=None) -> torch.Tensor:
    """Bandwidth-optimal ring: reduce-scatter then all-gather over N chunks."""
    if send.shape != recv.shape:
        raise ValueError("send and recv must have the same shape")
    size, me, left, right = _neighbours(group)
    flat = send.contiguous().view(-1).clone()
    n = flat.numel()
    if size == 1 or n == 0:
        recv.copy_(flat.view_as(recv))
        return recv
    chunk = (n + size - 1) // size
    pad = chunk * size - n
    if pad:
        flat = torch.cat([flat, flat.new_zeros(pad)])
    chunks = flat.view(size, chunk)
    tmp = torch.empty_like(chunks[0])
    # reduce-scatter: after step s rank r owns the partial sum of chunk (r - s) mod N
    for s in range(size - 1):
        si, ri = (me - s) % size, (me - s - 1) % size
        req = comm.isend(chunks[si].contiguous(), right, group=group)
        comm.recv(tmp, left, group=group)
        chunks[ri] += tmp
        req.wait()
    # all-gather: rank r starts with the fully reduced chunk (r + 1) mod N
    for s in range(size - 1):
        si, ri = (me + 1 - s) % size, (me - s) % size
        req = comm.isend(chunks[si].contiguous(), right, group=group)
        comm.recv(tmp, left, group=group)
        chunks[ri].copy_(tmp)
        req.wait()
    recv.copy_(flat[:n].view_as(recv))
    return recv
