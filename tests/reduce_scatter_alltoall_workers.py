"""Worker functions for the reduce-scatter, all-to-all and all-gather-into-tensor calls of comm.py: on gloo (CPU tensors,
tests/test_reduce_scatter_alltoall_model.py) against a value every rank computes itself, and under
``launch(..., backend="b200")`` (tests/test_gpu_reduce_scatter_alltoall_multi.py) against NCCL on the same inputs, with the
NCCL entry points refused while our calls run."""
import contextlib

import torch
import torch.distributed as dist

from dist_tuto.pth_b200 import comm
from dist_tuto.pth_b200.parallel import symm

_NAMES = ("reduce_scatter", "reduce_scatter_tensor", "all_to_all_single", "all_gather_into_tensor", "all_gather",
          "all_reduce")


def _input(rank, n, dtype, seed):
    g = torch.Generator().manual_seed(seed + 1000 * rank)
    if dtype == torch.bool:
        return torch.rand(n, generator=g) < 0.5
    if dtype.is_floating_point:
        return (torch.randn(n, generator=g) * 4).to(dtype)
    info = torch.iinfo(dtype)
    return torch.randint(info.min, info.max, (n,), generator=g, dtype=torch.int64).to(dtype)


def w_gloo(rank, size):
    """The four calls on CPU tensors go to gloo and give torch's results."""
    seg = 6
    xs = [torch.arange(size * seg, dtype=torch.float32) * (r + 1) + 0.25 for r in range(size)]
    o = torch.empty(seg)
    comm.reduce_scatter_tensor(o, xs[rank])
    assert torch.equal(o, sum(x.view(size, seg)[rank] for x in xs)), o
    o = torch.empty(seg)
    comm.reduce_scatter(o, [t.clone() for t in xs[rank].view(size, seg).unbind(0)], op=comm.reduce_op.MAX)
    assert torch.equal(o, torch.stack([x.view(size, seg)[rank] for x in xs]).amax(0)), o
    ys = [torch.arange(size * 3, dtype=torch.int64) + 100 * r for r in range(size)]
    o = torch.empty_like(ys[rank])
    comm.all_to_all_single(o, ys[rank])
    assert torch.equal(o, torch.cat([y.view(size, 3)[rank] for y in ys])), o
    o = torch.empty(size * 5, dtype=torch.int32)
    comm.all_gather_into_tensor(o, torch.full((5,), rank, dtype=torch.int32))
    assert torch.equal(o, torch.arange(size, dtype=torch.int32).repeat_interleave(5)), o


@contextlib.contextmanager
def _no_nccl():
    """Inside: torch.distributed's collectives of these calls raise, so a call that reaches them fails the test."""
    saved = {n: getattr(dist, n) for n in _NAMES}

    def refuse(*a, **k):
        raise AssertionError("a reduce-scatter, all-to-all or all-gather reached NCCL on a symmetric world")
    for n in _NAMES:
        setattr(dist, n, refuse)
    try:
        yield
    finally:
        for n, f in saved.items():
            setattr(dist, n, f)


SEGMENTS = [5, 1024, 3001, 8192, 40000]                      # elements per rank's segment: LL, pull, some ragged
RS_DTYPES = (torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int8, torch.uint8, torch.int32, torch.int64,
             torch.bool)
OPS = (comm.reduce_op.SUM, comm.reduce_op.PRODUCT, comm.reduce_op.MAX, comm.reduce_op.MIN)


def _same(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# unit roundoff of each float dtype: a float sum of more than two terms is compared with NCCL within a bound
_EPS = {torch.float64: 2.0 ** -52, torch.float32: 2.0 ** -23, torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}


def _agrees(ours, ref, dtype, op, world):
    """Bit for bit, except a float SUM over more than two ranks: NCCL's ring starts each slice at another rank and rounds
    every step to the dtype (NVLS and PAT use other orders again), while ours folds in rank order through one accumulator
    and rounds once, and float addition is not associative.  For |x| ~ 4 * randn the two differ by a few units in the last
    place of partial sums up to ~ 4 x world, well inside rtol 4 x world x eps, atol 64 x world x eps; a wrong or missing term
    is off by O(1)."""
    if dtype.is_floating_point and op == comm.reduce_op.SUM and world > 2:
        e = _EPS[dtype]
        return torch.allclose(ours.double(), ref.double(), rtol=4 * world * e, atol=64 * world * e)
    return _same(ours, ref)


def _check_group(rank, ranks, group):
    world = len(ranks)
    w = symm.lookup_world(group)
    assert w is not None and w.world == world
    for k, n in enumerate(SEGMENTS):
        for d, dtype in enumerate(RS_DTYPES):
            op = OPS[(k + d) % 4]
            if op == comm.reduce_op.PRODUCT and dtype.is_floating_point:
                op = comm.reduce_op.MAX                     # NCCL's fp products fold in another order and may overflow
            x = _input(rank, world * n, dtype, 31 * k + d).cuda()
            ours, ref = torch.zeros(n, dtype=dtype, device="cuda"), torch.zeros(n, dtype=dtype, device="cuda")
            with _no_nccl():
                comm.reduce_scatter_tensor(ours, x, op=op, group=group)
            dist.reduce_scatter_tensor(ref, x, op=op, group=group)
            assert _agrees(ours, ref, dtype, op, world), ("reduce_scatter_tensor", dtype, n, op)
            lst = [t.clone() for t in x.view(world, n).unbind(0)]
            ours2 = torch.zeros_like(ours)
            with _no_nccl():
                comm.reduce_scatter(ours2, lst, op=op, group=group)
            assert _same(ours2, ours), ("reduce_scatter: not the bits of reduce_scatter_tensor", dtype, n, op)
        for dtype in (torch.int64, torch.bfloat16, torch.uint8):
            x = _input(rank, world * n, dtype, 7 * k).cuda()
            ours, ref = torch.zeros_like(x), torch.zeros_like(x)
            with _no_nccl():
                comm.all_to_all_single(ours, x, group=group)
            dist.all_to_all_single(ref, x, group=group)
            assert _same(ours, ref), ("all_to_all_single", dtype, n)
            y = x[:n]
            ours, ref = torch.zeros_like(x), torch.zeros_like(x)
            with _no_nccl():
                comm.all_gather_into_tensor(ours, y, group=group)
            dist.all_gather_into_tensor(ref, y, group=group)
            assert _same(ours, ref), ("all_gather_into_tensor", dtype, n)
    torch.cuda.synchronize()


def w_vs_nccl(rank, size):
    _check_group(rank, list(range(size)), None)


def w_subgroup_vs_nccl(rank, size):
    ranks = list(range(1, size)) if size > 2 else [0, 1]
    g = comm.new_group(ranks)
    if rank in ranks:
        symm.init_world(g)
        _check_group(rank, ranks, g)
    comm.barrier()


def w_world1(rank, size):
    """One rank through the public API: the four calls equal their torch value and never reach NCCL."""
    assert size == 1 and symm.lookup_world(None) is not None
    x = torch.tensor([-0.0, float("nan"), 1e-40, 3.5], device="cuda")
    for fn in (comm.reduce_scatter_tensor, comm.all_to_all_single, comm.all_gather_into_tensor):
        o = torch.zeros_like(x)
        with _no_nccl():
            fn(o, x)
        assert _same(o, x), fn.__name__
    o = torch.zeros(4, dtype=torch.int64, device="cuda")
    y = torch.arange(4, dtype=torch.int64, device="cuda") * 2 ** 40
    with _no_nccl():
        comm.reduce_scatter(o, [y], op=comm.reduce_op.MIN)
    assert torch.equal(o, y)
