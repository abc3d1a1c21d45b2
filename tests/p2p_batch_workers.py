"""Worker functions for ``comm.batch_isend_irecv``: a gloo ring on CPU tensors (tests/test_p2p_batch_routing.py), and on
``backend="b200"`` rings and all-pairs exchanges through the peer-memory batch kernel, compared with NCCL's own
``batch_isend_irecv`` (tests/test_gpu_p2p_batch_multi.py)."""
import contextlib

import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm


def w_gloo_ring(rank, size):
    """Every rank sends to its right and receives from its left in one batch, sends listed first; then again with torch's
    own P2POp mixed in and two messages to the same peer."""
    x = torch.arange(5, dtype=torch.float64) + 10 * rank
    y = torch.zeros(5, dtype=torch.float64)
    right, left = (rank + 1) % size, (rank - 1) % size
    reqs = comm.batch_isend_irecv([comm.P2POp(comm.isend, x, right), comm.P2POp(comm.irecv, y, left)])
    assert len(reqs) == 2
    for r in reqs:
        r.wait()
    assert torch.equal(y, torch.arange(5, dtype=torch.float64) + 10 * left), y
    a, b = torch.full((3,), rank, dtype=torch.int32), torch.full((7,), -rank, dtype=torch.int32)
    ga, gb = torch.zeros(3, dtype=torch.int32), torch.zeros(7, dtype=torch.int32)
    for r in comm.batch_isend_irecv([dist.P2POp(dist.isend, a, right), comm.P2POp(comm.isend, b, right),
                                     dist.P2POp(dist.irecv, ga, left), comm.P2POp(dist.irecv, gb, left)]):
        r.wait()
    assert torch.equal(ga, torch.full((3,), left, dtype=torch.int32))
    assert torch.equal(gb, torch.full((7,), -left, dtype=torch.int32))
    dist.barrier()


# ---------------------------------------------------------------------------------------------------------- b200
@contextlib.contextmanager
def _no_nccl_p2p():
    """Inside: torch.distributed's point-to-point calls raise, so a call that reaches them fails the test."""
    names = ("send", "recv", "isend", "irecv", "batch_isend_irecv")
    saved = [getattr(dist, n) for n in names]

    def refuse(*a, **k):
        raise AssertionError("point-to-point reached NCCL on a symmetric world")
    for n in names:
        setattr(dist, n, refuse)
    try:
        yield
    finally:
        for n, f in zip(names, saved):
            setattr(dist, n, f)


def _bytes(nbytes, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()


CASES = [(3 << 20, torch.float32), (17, torch.uint8), (100003, torch.int64), (1 << 20, torch.bfloat16), (0, torch.int32)]


def _exchange(rank, size, pattern, use_nccl):
    """ring: send right and receive left; all-pairs: send to and receive from every peer.  Sends are listed before
    receives.  Returns the received tensors by source."""
    out = {}
    for k, (n, dtype) in enumerate(CASES):
        mine = [_bytes(n * torch.empty((), dtype=dtype).element_size(), 100 * k + r).view(dtype) for r in range(size)]
        if pattern == "ring":
            dsts, srcs = [(rank + 1) % size], [(rank - 1) % size]
        else:
            dsts = srcs = [q for q in range(size) if q != rank]
        got = {q: torch.zeros_like(mine[rank]) for q in srcs}
        if use_nccl:
            ops = [dist.P2POp(dist.isend, mine[rank], q) for q in dsts] + [dist.P2POp(dist.irecv, got[q], q) for q in srcs]
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        else:
            with _no_nccl_p2p():
                ops = [comm.P2POp(comm.isend, mine[rank], q) for q in dsts] + \
                      [comm.P2POp(comm.irecv, got[q], q) for q in srcs]
                for r in comm.batch_isend_irecv(ops):
                    r.wait()
        for q in srcs:
            assert torch.equal(got[q].view(torch.uint8), mine[q].view(torch.uint8)), (pattern, n, dtype, q)
        out.update({(k, q): got[q] for q in srcs})
    return out


def w_ring_and_all_pairs_vs_nccl(rank, size):
    """The batch kernel's ring and all-pairs exchanges equal NCCL's batch_isend_irecv of the same lists, bit for bit, and
    never reach NCCL's point-to-point."""
    from dist_tuto.pth_b200.parallel import symm
    assert symm.lookup_world(None) is not None
    for pattern in ("ring", "all_pairs"):
        ours = _exchange(rank, size, pattern, use_nccl=False)
        ref = _exchange(rank, size, pattern, use_nccl=True)
        for key, t in ours.items():
            assert torch.equal(t.view(torch.uint8), ref[key].view(torch.uint8)), (pattern, key)
    torch.cuda.synchronize()
    dist.barrier()


def w_batch_against_single_calls(rank, size):
    """Ranks 0 and 1: one side batches, the other uses isend / irecv, then the roles swap, with messages larger than a
    pair's mailbox and sends issued before receives."""
    if rank < 2:
        peer = 1 - rank
        for k, n in enumerate([3 << 20, 17, 1 << 20]):
            x = _bytes(n, 10 * k + rank)
            want = _bytes(n, 10 * k + peer)
            y = torch.zeros_like(x)
            with _no_nccl_p2p():
                if rank == k % 2:
                    reqs = comm.batch_isend_irecv([comm.P2POp(comm.isend, x, peer), comm.P2POp(comm.irecv, y, peer)])
                else:
                    reqs = [comm.isend(x, peer), comm.irecv(y, peer)]
                for r in reqs:
                    r.wait()
            assert torch.equal(y, want), (k, n)
    torch.cuda.synchronize()
    dist.barrier()
