"""Workers of tests/test_sync_bn_cpu.py (spawned processes, gloo @127.0.0.1): ``SyncBatchNorm`` on CPU ranks against fp64
``F.batch_norm`` on the concatenated global batch.  Local batch sizes differ between ranks, and one rank has none."""
import torch
import torch.distributed as tdist
import torch.nn as nn
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2

C = 5
SHAPES = {2: (), 3: (4,), 4: (3, 2), 5: (2, 2, 2)}


def _sizes(size):
    return [5, 0, 3, 2][:size]


def _global(dim, size, step, seed=0):
    g = torch.Generator().manual_seed(1000 * seed + 10 * dim + step)
    n = sum(_sizes(size))
    x = torch.randn((n, C) + SHAPES[dim], generator=g, dtype=torch.float64) * 1.5 + 0.7
    dy = torch.randn(x.shape, generator=g, dtype=torch.float64)
    return x, dy


def _mine(t, rank, size):
    s = _sizes(size)
    a = sum(s[:rank])
    return t[a:a + s[rank]]


def _gather(t):
    out = [torch.empty_like(t) for _ in range(tdist.get_world_size())]
    tdist.all_gather(out, t.contiguous())
    return out


def _close(a, b, what, tol=2e-6):
    a, b = a.double(), b.double()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = (a - b).abs().max().item() if a.numel() else 0.0
    assert err <= tol * (1 + b.abs().max().item() if b.numel() else 1), (what, err)


def _modules(momentum, affine, track):
    torch.manual_seed(7)
    ref = nn.BatchNorm1d(C, momentum=momentum, affine=affine, track_running_stats=track).double()
    if affine:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
    mine = b2.SyncBatchNorm(C, momentum=momentum, affine=affine, track_running_stats=track)
    mine.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    return ref, mine


def _ref_step(ref, x, training):
    """fp64 torch batch norm of the global batch (any rank); BatchNorm1d takes [N, C, L] so flatten the spatial dims."""
    ref.train(training)
    xr = x.reshape(x.shape[0], C, -1).detach().requires_grad_(True)
    return xr, ref(xr)


def w_matches_global_batch_norm(rank, size):
    for dim in (2, 3, 4, 5):
        for momentum, affine, track in ((0.1, True, True), (None, True, True), (0.3, False, True), (0.1, True, False)):
            ref, mine = _modules(momentum, affine, track)
            for step in range(3):
                training = step < 2                         # the last step runs in eval mode
                x, dy = _global(dim, size, step, seed=size)
                xr, yr = _ref_step(ref, x, training)
                yr.backward(dy.reshape(yr.shape))
                yr = yr.detach()
                if not training and not track:              # eval without running stats: local batch statistics, no sync
                    xl = _mine(x, rank, size)
                    yl = F.batch_norm(xl, None, None, ref.weight, ref.bias, True, 0.0, ref.eps) if xl.shape[0] > 1 else xl
                    yr = torch.cat([x[:sum(_sizes(size)[:rank])], yl, x[sum(_sizes(size)[:rank + 1]):]]).reshape(yr.shape)
                mine.train(training)
                xm = _mine(x, rank, size).float()
                if dim == 4 and step == 1:
                    xm = xm.contiguous(memory_format=torch.channels_last)
                xm.requires_grad_(True)
                for p in mine.parameters():
                    p.grad = None
                if not training and not track and xm.shape[0] == 1:
                    continue
                y = mine(xm)
                assert y.dtype == xm.dtype and y.shape == xm.shape
                _close(y.detach(), _mine(yr.reshape(x.shape), rank, size), ("y", dim, momentum, affine, track, step))
                y.backward(_mine(dy, rank, size).float())
                if training:
                    _close(xm.grad, _mine(xr.grad.reshape(x.shape), rank, size),
                           ("grad_input", dim, momentum, affine, track, step), tol=1e-5)
                    if affine:
                        for p, pr in ((mine.weight, ref.weight), (mine.bias, ref.bias)):
                            g = p.grad.clone() if p.grad is not None else torch.zeros_like(p)
                            tdist.all_reduce(g)
                            _close(g, pr.grad, ("sum of local grads", dim, step), tol=1e-5)
                            pr.grad = None
                if track:
                    _close(mine.running_mean, ref.running_mean, ("running_mean", dim, momentum, step))
                    _close(mine.running_var, ref.running_var, ("running_var", dim, momentum, step))
                    assert int(mine.num_batches_tracked) == int(ref.num_batches_tracked)
                    for t in (mine.running_mean, mine.running_var):
                        for o in _gather(t):
                            assert torch.equal(o, t), "running buffers differ between ranks"


def w_convert_and_state_dict(rank, size):
    torch.manual_seed(1)
    net = nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4), nn.Sequential(nn.BatchNorm1d(4)),
                        nn.SyncBatchNorm(4, momentum=None, affine=False))
    net[1].weight.requires_grad_(False)
    net.eval()
    before = {n: p for n, p in net.named_parameters()}
    bufs = {n: b for n, b in net.named_buffers()}
    keys = net.state_dict().keys()
    out = b2.SyncBatchNorm.convert_sync_batchnorm(net)
    assert out is net
    for i in (1, 3):
        assert type(out[i]) is b2.SyncBatchNorm and isinstance(out[i], nn.SyncBatchNorm)
    assert type(out[2][0]) is b2.SyncBatchNorm and out[3].momentum is None and not out[3].affine
    for n, p in out.named_parameters():
        assert p is before[n], n
    for n, b in out.named_buffers():
        assert b is bufs[n], n
    assert not out[1].weight.requires_grad and not out[1].training and out.state_dict().keys() == keys
    single = b2.SyncBatchNorm.convert_sync_batchnorm(nn.BatchNorm3d(6))
    assert type(single) is b2.SyncBatchNorm
    theirs = nn.SyncBatchNorm(4)
    with torch.no_grad():
        theirs.running_mean.uniform_()
        theirs.weight.uniform_()
    theirs.num_batches_tracked.fill_(9)
    mine = b2.SyncBatchNorm(4)
    mine.load_state_dict(theirs.state_dict())
    back = nn.SyncBatchNorm(4)
    back.load_state_dict(mine.state_dict())
    for k, v in theirs.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k


def w_subgroup(rank, size):
    """World 3, group {0, 2}: rank 1 runs alone (its own statistics)."""
    g02, g1 = tdist.new_group([0, 2]), tdist.new_group([1])
    torch.manual_seed(3)
    x = torch.randn(4 * 3, C, 6, dtype=torch.float64)
    mine = b2.SyncBatchNorm(C, process_group=g02 if rank in (0, 2) else g1)
    xs = x[4 * rank:4 * rank + 4]
    y = mine(xs.float())
    ref = torch.cat([x[0:4], x[8:12]]) if rank in (0, 2) else x[4:8]
    want = F.batch_norm(ref, None, None, training=True)
    part = want[:4] if rank == 0 else want[4:] if rank == 2 else want
    _close(y, part, ("subgroup", rank))


def w_against_torch_on_gpus(rank, size):
    """tests/test_gpu_sync_bn_multi.py: b200 backend against torch's SyncBatchNorm on NCCL."""
    torch.manual_seed(0)
    C = 64
    theirs = torch.nn.SyncBatchNorm(C).cuda()
    mine = b2.SyncBatchNorm(C).cuda()
    mine.load_state_dict(theirs.state_dict())
    for step in range(3):
        g = torch.Generator(device="cuda").manual_seed(10 * step + rank)
        x = torch.randn(4 + rank, C, 14, 14, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
        dy = torch.randn(x.shape, generator=g, device="cuda")
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        ya, yb = theirs(xa), mine(xb)
        ya.backward(dy)
        yb.backward(dy)
        torch.testing.assert_close(yb, ya, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(xb.grad, xa.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(mine.running_var, theirs.running_var, rtol=1e-5, atol=1e-6)
        for t in (mine.running_mean, mine.running_var):
            out = [torch.empty_like(t) for _ in range(size)]
            tdist.all_gather(out, t)
            assert all(torch.equal(o, t) for o in out), "replica buffers differ"
