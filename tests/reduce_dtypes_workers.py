"""Worker functions (run under ``launch(..., backend="b200")``) for tests/test_gpu_reduce_dtypes_multi.py: ``comm.all_reduce``
and ``comm.reduce`` of fp16, fp64, int8, uint8, int32, int64 and bool on the peer-memory kernels, compared with NCCL's own
result on the same inputs."""
import contextlib

import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm
from dist_tuto.pth_b200.parallel import symm

SIZES = [5, 3000, 40000, 300001]          # LL, one-shot and two-shot, some ragged
DTYPES = (torch.float16, torch.float64, torch.int8, torch.uint8, torch.int32, torch.int64, torch.bool)
OPS = (dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT, dist.ReduceOp.MAX, dist.ReduceOp.MIN)


@contextlib.contextmanager
def _no_nccl_reductions():
    """Inside: torch.distributed.all_reduce / reduce raise, so a call that reaches them fails the test."""
    saved = dist.all_reduce, dist.reduce

    def refuse(*a, **k):
        raise AssertionError("all_reduce / reduce reached NCCL on a symmetric world")
    dist.all_reduce = dist.reduce = refuse
    try:
        yield
    finally:
        dist.all_reduce, dist.reduce = saved


def _inputs(dtype, op, n, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.bool:
        return (torch.rand(n, generator=g) < 0.5).cuda()
    if dtype.is_floating_point:
        x = torch.rand(n, generator=g, dtype=torch.float64) * 1.5 + 0.5 if op == dist.ReduceOp.PRODUCT else \
            torch.randn(n, generator=g, dtype=torch.float64)
        return x.to(dtype).cuda()
    info = torch.iinfo(dtype)
    return torch.randint(info.min, info.max, (n,), generator=g, dtype=torch.int64).to(dtype).cuda()


def _same(ours, ref, dtype, op):
    if dtype.is_floating_point and op in (dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT):
        tol = 4e-3 if dtype == torch.float16 else 1e-12            # NCCL rounds fp16 after every step; fp64 may reorder
        return torch.allclose(ours.double(), ref.double(), rtol=tol, atol=tol)
    return torch.equal(ours.view(-1).view(torch.uint8), ref.view(-1).view(torch.uint8))


def _check_group(rank, ranks, group):
    world = len(ranks)
    w = symm.lookup_world(group)
    assert w is not None and w.world == world
    for k, n in enumerate(SIZES):
        for dtype in DTYPES:
            for j, op in enumerate(OPS):
                x = _inputs(dtype, op, n, 1000 * k + 10 * j + rank)
                ours, ref = x.clone(), x.clone()
                with _no_nccl_reductions():
                    comm.all_reduce(ours, op=op, group=group)
                dist.all_reduce(ref, op=op, group=group)
                assert _same(ours, ref, dtype, op), ("all_reduce", dtype, op, n)
                root = ranks[(k + j) % world]
                ours, ref = x.clone(), x.clone()
                with _no_nccl_reductions():
                    comm.reduce(ours, root, op=op, group=group)
                dist.reduce(ref, dst=root, op=op, group=group)
                if rank == root:
                    assert _same(ours, ref, dtype, op), ("reduce", dtype, op, n, root)
                else:
                    assert torch.equal(ours.view(-1).view(torch.uint8), x.view(-1).view(torch.uint8)), ("reduce", n)
    torch.cuda.synchronize()


def w_reduce_dtypes_vs_nccl(rank, size):
    _check_group(rank, list(range(size)), None)


def w_reduce_dtypes_subgroup_vs_nccl(rank, size):
    ranks = list(range(1, size)) if size > 2 else [0, 1]
    g = comm.new_group(ranks)
    if rank in ranks:
        symm.init_world(g)
        _check_group(rank, ranks, g)
    comm.barrier()


def w_evaluate_takes_the_fp64_kernels(rank, size):
    """evaluate() of a CUDA net on backend="b200" sums its float64 [loss, correct, n] with comm.all_reduce, now on the fp64
    kernels: equal to a CPU float64 evaluation of the whole set, the same on every rank, and without NCCL."""
    import torch.nn.functional as F

    import dist_tuto.pth_b200 as b2
    from dist_tuto.pth_b200.data import SyntheticMNIST
    from dist_tuto.pth_b200.models.convnet import Net
    ds = SyntheticMNIST(n=1001, seed=21)
    torch.manual_seed(5)
    net = Net()
    with torch.no_grad():
        x = ((ds.images.double() / 255.0 - ds.mean) / ds.std).unsqueeze(1)
        out = net.double().eval()(x)
        loss = float(F.nll_loss(out, ds.labels, reduction="sum"))
        correct = int((out.argmax(1) == ds.labels).sum())
    net = net.float().cuda()
    with _no_nccl_reductions():
        got = b2.evaluate(net, ds)
    assert got["n"] == 1001 and got["correct"] == correct, (got, correct)
    assert abs(got["loss"] * 1001 - loss) <= 1e-4 * abs(loss), (got["loss"] * 1001, loss)
    gathered = [None] * size
    dist.all_gather_object(gathered, got)
    assert all(g == got for g in gathered)
