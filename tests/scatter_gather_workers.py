"""Worker functions (run under ``launch(..., backend="b200")``) for tests/test_gpu_scatter_gather_multi.py: ``comm.scatter``
and ``comm.gather`` on the peer-memory kernels, compared with NCCL's own result on the same inputs."""
import contextlib

import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm
from dist_tuto.pth_b200.parallel import symm

SIZES = [5, 3000, 40000, 300001]          # LL, one-shot and two-shot, some ragged
DTYPES = (torch.int64, torch.bfloat16, torch.uint8)


@contextlib.contextmanager
def _no_nccl_scatter_gather():
    """Inside: torch.distributed.scatter / gather raise, so a call that reaches them fails the test."""
    saved = dist.scatter, dist.gather

    def refuse(*a, **k):
        raise AssertionError("scatter / gather reached NCCL on a symmetric world")
    dist.scatter = dist.gather = refuse
    try:
        yield
    finally:
        dist.scatter, dist.gather = saved


def _check_group(rank, ranks, group):
    world = len(ranks)
    w = symm.lookup_world(group)
    assert w is not None and w.world == world
    for k, n in enumerate(SIZES):
        for dtype in DTYPES:
            g = torch.Generator().manual_seed(11 * k + rank)
            x = torch.randint(-2 ** 62, 2 ** 62, (n,), generator=g, dtype=torch.int64).to(dtype).cuda()
            for j, root in enumerate(sorted({ranks[0], ranks[-1], ranks[world // 2]})):
                block = (k + j) % 2 == 0
                # scatter: the root's list (one block, or separate tensors); every other rank passes its own, ignored
                if block:
                    lst = list((x.repeat(world) + torch.arange(world, device="cuda").repeat_interleave(n).to(dtype))
                               .view(world, n).unbind(0))
                else:
                    lst = [(x + s).contiguous() for s in range(world)]
                ours, ref = torch.zeros_like(x), torch.zeros_like(x)
                with _no_nccl_scatter_gather():
                    comm.scatter(ours, src=root, scatter_list=lst, group=group)
                dist.scatter(ref, scatter_list=[t.clone() for t in lst] if rank == root else None, src=root, group=group)
                assert torch.equal(ours.view(torch.uint8), ref.view(torch.uint8)), ("scatter", dtype, n, root)
                # gather
                if block:
                    ours = list(torch.zeros(world * n, dtype=dtype, device="cuda").view(world, n).unbind(0))
                else:
                    ours = [torch.zeros_like(x) for _ in range(world)]
                ref = [torch.zeros_like(x) for _ in range(world)]
                with _no_nccl_scatter_gather():
                    comm.gather(x, dst=root, gather_list=ours, group=group)
                dist.gather(x, gather_list=ref if rank == root else None, dst=root, group=group)
                if rank == root:
                    for a, b in zip(ours, ref):
                        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), ("gather", dtype, n, root)
                else:
                    assert all(int(a.count_nonzero()) == 0 for a in ours), ("gather: a non-root's list was written", n)
            # the ptp.py helper, unchanged
            root = ranks[-1]
            lst = [torch.zeros_like(x) for _ in range(world)] if rank == root else None
            with _no_nccl_scatter_gather():
                comm.gather_to_root(x, rank, lst, root=root, group=group)
            if rank == root:
                ref = [torch.zeros_like(x) for _ in range(world)]
                dist.gather(x, gather_list=ref, dst=root, group=group)
                assert all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(lst, ref))
            else:
                dist.gather(x, gather_list=None, dst=root, group=group)
    torch.cuda.synchronize()


def w_scatter_gather_vs_nccl(rank, size):
    _check_group(rank, list(range(size)), None)


def w_scatter_gather_subgroup_vs_nccl(rank, size):
    ranks = list(range(1, size)) if size > 2 else [0, 1]
    g = comm.new_group(ranks)
    if rank in ranks:
        symm.init_world(g)
        _check_group(rank, ranks, g)
    comm.barrier()


def w_scatter_gather_world1(rank, size):
    """One rank through the public API: scatter and gather equal their torch value, any dtype, and never reach NCCL."""
    assert size == 1 and symm.lookup_world(None) is not None
    y = torch.arange(-3, 9, dtype=torch.int64, device="cuda") * (2 ** 40)
    t = torch.zeros_like(y)
    with _no_nccl_scatter_gather():
        comm.scatter(t, src=0, scatter_list=[y])
    assert torch.equal(t, y)
    z = torch.tensor([-0.0, float("nan"), 1e-40], device="cuda")
    outs = [torch.zeros_like(z)]
    with _no_nccl_scatter_gather():
        comm.gather(z, dst=0, gather_list=outs)
        comm.gather_to_root(y, 0, [t], root=0)
    assert torch.equal(outs[0].view(torch.int32), z.view(torch.int32))
    assert torch.equal(t, y)
