"""Worker functions for ``comm.all_to_all_single`` with split sizes and ``comm.all_to_all``: on gloo (CPU tensors,
tests/test_all_to_all_v_model.py) against tests/all_to_all_v_model.py, and under ``launch(..., backend="b200")``
(tests/test_gpu_all_to_all_v_multi.py) against NCCL on the same inputs, with the NCCL entry points refused while our calls
run.  Every rank draws the same split matrix from a shared seed, so the splits of one call agree between ranks."""
import contextlib

import torch
import torch.distributed as dist

import all_to_all_v_model as AM
from dist_tuto.pth_b200 import comm
from dist_tuto.pth_b200.parallel import symm

_NAMES = ("all_to_all_single", "all_to_all")


def split_matrix(world: int, seed: int, hot: bool, most: int = 40) -> list:
    """``S[s][d]``: rows rank s sends to rank d.  ``hot``: one destination takes most rows (token dispatch to a popular
    expert), the rest are small random counts, zeros included."""
    g = torch.Generator().manual_seed(seed)
    S = torch.randint(0, most + 1, (world, world), generator=g)
    S[torch.rand(world, world, generator=g) < 0.2] = 0
    if hot:
        h = int(torch.randint(0, world, (1,), generator=g))
        S[:, h] += 10 * most
    return S.tolist()


def rows_of(S: list, rank: int, dtype, tail: tuple, seed: int) -> torch.Tensor:
    """Rank ``rank``'s input: sum(S[rank]) rows of shape ``tail``, seeded by rank."""
    g = torch.Generator().manual_seed(seed + 7919 * rank)
    n = sum(S[rank])
    shape = (n,) + tail
    if dtype == torch.bool:
        return torch.rand(shape, generator=g) < 0.5
    if dtype.is_floating_point or dtype.is_complex:
        return (torch.randn(shape, generator=g) * 4).to(dtype)
    info = torch.iinfo(dtype)
    return torch.randint(info.min, info.max, shape, generator=g, dtype=torch.int64).to(dtype)


def w_gloo(rank, size):
    """``comm.all_to_all_single`` with split sizes on CPU tensors goes to gloo and gives the model's bytes, for consistent
    splits of several dtypes and row shapes (gloo has no list form)."""
    for k, (dtype, tail) in enumerate([(torch.int64, (3,)), (torch.float32, ()), (torch.uint8, (2, 5)),
                                       (torch.bfloat16, (7,))]):
        S = split_matrix(size, 100 + k, hot=k % 2 == 1, most=6)
        xs = [rows_of(S, s, dtype, tail, 10 * k) for s in range(size)]
        outs = [torch.full((sum(S[p][r] for p in range(size)),) + tail, 0, dtype=dtype) for r in range(size)]
        want = AM.single_form(xs, S, outs, [[S[p][r] for p in range(size)] for r in range(size)])[rank]
        o = outs[rank].clone()
        comm.all_to_all_single(o, xs[rank], [S[p][rank] for p in range(size)], S[rank])
        assert torch.equal(o.reshape(-1).view(torch.uint8), want.reshape(-1).view(torch.uint8)), (dtype, S)
        assert torch.equal(o, AM.by_slicing(xs, S)[rank]), (dtype, S)


@contextlib.contextmanager
def _no_nccl():
    """Inside: torch.distributed's all-to-all calls raise, so a call that reaches them fails the test."""
    saved = {n: getattr(dist, n) for n in _NAMES}

    def refuse(*a, **k):
        raise AssertionError("an all-to-all with split sizes or the list form reached NCCL on a symmetric world")
    for n in _NAMES:
        setattr(dist, n, refuse)
    try:
        yield
    finally:
        for n, f in saved.items():
            setattr(dist, n, f)


def _same(a, b):
    return torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))


DTYPES = (torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int8, torch.uint8, torch.int32, torch.int64,
          torch.bool, torch.complex64)


def _check_group(rank, ranks, group, calls=6):
    world = len(ranks)
    me = ranks.index(rank)
    w = symm.lookup_world(group)
    assert w is not None and w.world == world
    for k in range(calls):                                   # splits change from call to call
        dtype = DTYPES[k % len(DTYPES)]
        tail = [(), (3,), (16,), (5, 2)][k % 4]
        most = [3, 40, 2000, 9000][k % 4]
        S = split_matrix(world, 1000 + 17 * k, hot=k % 2 == 0, most=most)
        x = rows_of(S, me, dtype, tail, 31 * k).cuda()
        out_splits = [S[p][me] for p in range(world)]
        ours = torch.zeros((sum(out_splits),) + tail, dtype=dtype, device="cuda")
        ref = torch.zeros_like(ours)
        with _no_nccl():
            comm.all_to_all_single(ours, x, out_splits, S[me], group=group)
        dist.all_to_all_single(ref, x, out_splits, S[me], group=group)
        assert _same(ours, ref), ("all_to_all_single", dtype, S)
        ins = [x[sum(S[me][:d]):sum(S[me][:d + 1])].clone() for d in range(world)]
        outs = [torch.zeros((out_splits[p],) + tail, dtype=dtype, device="cuda") for p in range(world)]
        refs = [torch.zeros_like(o) for o in outs]
        with _no_nccl():
            comm.all_to_all(outs, ins, group=group)
        dist.all_to_all(refs, ins, group=group)
        for p in range(world):
            assert _same(outs[p], refs[p]), ("all_to_all", dtype, S, p)
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
    """One rank through the public API: both calls equal their torch value and never reach NCCL."""
    assert size == 1 and symm.lookup_world(None) is not None
    x = torch.tensor([[-0.0, float("nan")], [1e-40, 3.5], [7.0, -2.0]], device="cuda")
    o = torch.zeros_like(x)
    with _no_nccl():
        comm.all_to_all_single(o, x, [3], [3])
    assert _same(o, x)
    o = torch.zeros_like(x)
    with _no_nccl():
        comm.all_to_all_single(o, x, output_split_sizes=[3])
    assert _same(o, x)
    y = torch.arange(5, dtype=torch.int64, device="cuda") * 2 ** 40
    outs = [torch.zeros(5, dtype=torch.int64, device="cuda")]
    with _no_nccl():
        comm.all_to_all(outs, [y])
    assert torch.equal(outs[0], y)
    with _no_nccl():
        comm.all_to_all_single(x, x, [3], [3])                # in place
    assert _same(x, torch.tensor([[-0.0, float("nan")], [1e-40, 3.5], [7.0, -2.0]], device="cuda"))
    torch.cuda.synchronize()
