"""Worker functions (run under ``launch(..., backend="b200")``) for tests/test_gpu_collectives_multi.py: the collectives
``comm.py`` routes to the peer-memory kernels, compared with NCCL's own result on the same inputs."""
import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm
from dist_tuto.pth_b200.parallel import symm

SIZES = [5, 3000, 40000, 300001]          # LL, one-shot and two-shot, some ragged
OPS = [dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT, dist.ReduceOp.MAX, dist.ReduceOp.MIN]


def _inputs(rank, n, dtype, seed, op):
    g = torch.Generator().manual_seed(seed * 101 + rank)
    x = torch.randn(n, generator=g)
    if op == dist.ReduceOp.PRODUCT:                  # keep products of up to 8 terms away from overflow and subnormals
        x = (torch.rand(n, generator=g) + 0.5) * torch.where(x < 0, -1.0, 1.0)
    return x.to(dtype).cuda()


def _tol(dtype):
    return (1e-5, 1e-6) if dtype == torch.float32 else (2e-2, 1e-2)


def _check_group(rank, ranks, group):
    """Every routed collective over ``group`` (global ``ranks``) against NCCL."""
    world = len(ranks)
    w = symm.lookup_world(group)
    assert w is not None and w.world == world
    for k, n in enumerate(SIZES):
        for op in OPS:
            for dtype in (torch.float32, torch.bfloat16):
                x = _inputs(rank, n, dtype, k, op)
                ours, ref = x.clone(), x.clone()
                comm.all_reduce(ours, op=op, group=group)
                dist.all_reduce(ref, op=op, group=group)
                rtol, atol = _tol(dtype)
                if op in (dist.ReduceOp.MAX, dist.ReduceOp.MIN):
                    assert torch.equal(ours, ref), ("all_reduce", op, dtype, n)
                else:
                    torch.testing.assert_close(ours, ref, rtol=rtol * world, atol=atol)
                root = ranks[(k + 1) * len(ranks) // 3 % world]
                ours = x.clone()
                comm.reduce(ours, root, op=op, group=group)
                if rank == root:
                    if op in (dist.ReduceOp.MAX, dist.ReduceOp.MIN):
                        assert torch.equal(ours, ref), ("reduce", op, dtype, n)
                    else:
                        torch.testing.assert_close(ours, ref, rtol=rtol * world, atol=atol)
                else:
                    assert torch.equal(ours, x), ("reduce: a non-root's tensor changed", op, dtype, n)
        for dtype in (torch.int64, torch.bfloat16, torch.uint8):
            g = torch.Generator().manual_seed(7 * k + rank)
            x = torch.randint(-2 ** 62, 2 ** 62, (n,), generator=g, dtype=torch.int64).to(dtype).cuda()
            for root in sorted({ranks[0], ranks[-1], ranks[world // 2]}):
                ours, ref = x.clone(), x.clone()
                comm.broadcast(ours, root, group=group)
                dist.broadcast(ref, root, group=group)
                assert torch.equal(ours.view(torch.uint8), ref.view(torch.uint8)), ("broadcast", dtype, n, root)
            ours = [torch.zeros_like(x) for _ in range(world)]
            ref = [torch.zeros_like(x) for _ in range(world)]
            comm.all_gather(ours, x, group=group)
            dist.all_gather(ref, x, group=group)
            for a, b in zip(ours, ref):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), ("all_gather", dtype, n)
    torch.cuda.synchronize()


def w_collectives_vs_nccl(rank, size):
    _check_group(rank, list(range(size)), None)


def w_collectives_subgroup_vs_nccl(rank, size):
    ranks = list(range(1, size)) if size > 2 else [0, 1]
    g = comm.new_group(ranks)
    if rank in ranks:
        symm.init_world(g)
        _check_group(rank, ranks, g)
    comm.barrier()


def w_collectives_world1(rank, size):
    """One rank through the public API: each collective equals its torch value."""
    assert size == 1 and symm.lookup_world(None) is not None
    x = torch.tensor([1.5, -0.0, float("nan"), -3.0], device="cuda")
    t = x.clone()
    comm.all_reduce(t, op=comm.reduce_op.MAX)
    assert torch.equal(t.view(torch.int32), x.view(torch.int32))
    t = x.clone()
    comm.reduce(t, 0, op=comm.reduce_op.PRODUCT)
    assert torch.equal(t.view(torch.int32), x.view(torch.int32))
    y = torch.arange(-3, 9, dtype=torch.int64, device="cuda") * (2 ** 40)
    t = y.clone()
    comm.broadcast(t, 0)
    assert torch.equal(t, y)
    outs = [torch.zeros_like(y)]
    comm.all_gather(outs, y)
    assert torch.equal(outs[0], y)
