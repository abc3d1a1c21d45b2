"""Worker functions (run under ``launch(..., backend="b200")``) for tests/test_gpu_p2p_multi.py: ``comm.send`` / ``recv`` /
``isend`` / ``irecv`` on the peer-memory kernels, and the tutorial's ring all-reduce on top of them, against NCCL."""
import contextlib

import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm, ring
from dist_tuto.pth_b200.parallel import symm

PINGPONG_BYTES = [4, 64, 1024, 16 << 10, 256 << 10, 1 << 20, 16 << 20]     # the sizes of bench/pingpong.py


@contextlib.contextmanager
def _no_nccl_p2p():
    """Inside: torch.distributed's point-to-point calls raise, so a call that reaches them fails the test."""
    names = ("send", "recv", "isend", "irecv")
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


def w_pingpong(rank, size):
    """Ranks 0 and 1 bounce a message at every ping-pong size; the others idle.  Any dtype, bit for bit."""
    assert symm.lookup_world(None) is not None
    for k, n in enumerate(PINGPONG_BYTES):
        x = _bytes(n, k)
        y = torch.zeros_like(x)
        with _no_nccl_p2p():
            if rank == 0:
                comm.send(x, dst=1)
                assert comm.recv(y, src=1) == 1
                assert torch.equal(y, x.flip(0)), n
            elif rank == 1:
                comm.recv(y, src=0)
                assert torch.equal(y, x), n
                comm.send(y.flip(0).contiguous(), dst=0)
    torch.cuda.synchronize()
    dist.barrier()


def w_ring_and_all_pairs(rank, size):
    """A ring (isend right, recv left) and an all-pairs exchange (isend to every peer, irecv from every peer), at sizes
    that need acknowledgements inside one message and at ragged ones, in several dtypes."""
    for k, (n, dtype) in enumerate([(3 << 20, torch.float32), (17, torch.uint8), (100003, torch.int64),
                                    (1 << 20, torch.bfloat16)]):
        mine = [_bytes(n * torch.empty((), dtype=dtype).element_size(), 100 * k + r).view(dtype) for r in range(size)]
        right, left = (rank + 1) % size, (rank - 1) % size
        got = torch.zeros_like(mine[rank])
        with _no_nccl_p2p():
            req = comm.isend(mine[rank], right)
            comm.recv(got, left)
            req.wait()
        assert torch.equal(got.view(torch.uint8), mine[left].view(torch.uint8)), ("ring", n, dtype)
        outs = {q: torch.zeros_like(mine[rank]) for q in range(size) if q != rank}
        with _no_nccl_p2p():
            reqs = [comm.isend(mine[rank], q) for q in outs] + [comm.irecv(outs[q], q) for q in outs]
            for r in reqs:
                r.wait()
        for q, o in outs.items():
            assert torch.equal(o.view(torch.uint8), mine[q].view(torch.uint8)), ("all pairs", n, dtype, q)
    torch.cuda.synchronize()
    dist.barrier()


def w_ring_allreduce_vs_nccl(rank, size):
    """ring.allreduce and ring.allreduce_chunked (the tutorial's ring, tuto.md:328-354) on the peer-memory point-to-point
    path equal NCCL's all_reduce; integer-valued inputs make every summation order exact."""
    for n in (1, 1000, 262147, 2 << 20):
        g = torch.Generator().manual_seed(n + rank)
        x = torch.randint(-1000, 1000, (n,), generator=g).float().cuda()
        ref = x.clone()
        dist.all_reduce(ref)
        for fn in (ring.allreduce, ring.allreduce_chunked):
            out = torch.zeros_like(x)
            with _no_nccl_p2p():
                fn(x, out)
            assert torch.equal(out, ref), (fn.__name__, n)
    torch.cuda.synchronize()
    dist.barrier()
