"""SyncBatchNorm kernels (csrc/batchnorm.cu) on one H100.

* kernels at world size 1, driven one by one through the binding: fp32 / bf16 / fp16, plain and channels-last layouts,
  C in {1, 3, 64, 512, 2049}, N x L from 2 through the ResNet stem, odd sizes for every tail, a grid cap that makes CTAs
  stride over tiles; every output against fp64 within c 2^-24 (|x k1| + |k0|) plus the output's rounding, sentinels behind
  every output, two runs bit-identical;
* emulated ranks, worlds 1-8 on one GPU (tests/test_gpu_collectives_emulated.symm_worlds, one stream per rank): forward and
  backward through ``SyncBatchNormFunction`` with uneven and zero local batches; mean, invstd and running stats bit-identical
  on every rank and within the bound of the fp64 global reference;
* the module at world size 1: against cuDNN ``BatchNorm2d``, no host synchronisation (``momentum=None`` included), a
  captured CUDA graph replaying bit-equal to eager, and a converted ResNet-18 training under bf16 autocast.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
import test_gpu_collectives_emulated as CE
import test_gpu_comm_emulated as E
from dist_tuto.pth_b200.parallel.sync_bn import SyncBatchNormFunction, exchange_numel

pytestmark = E.pytestmark
C_BOUND = 3.0
OUT_EPS = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
OUT_SUB = {dt: torch.finfo(dt).tiny * torch.finfo(dt).eps for dt in OUT_EPS}   # subnormal spacing of the output
SENT = -12345.0


@pytest.fixture(scope="module")
def K():
    from dist_tuto.pth_b200.ops import _ext
    return _ext.C()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fmt(shape, cl):
    if not cl:
        return torch.contiguous_format
    return torch.channels_last if len(shape) == 4 else torch.channels_last_3d


def _backed(shape, dtype, fmt, fill=SENT):
    """A tensor of ``shape`` in ``fmt`` that is the front of a larger buffer (one more sample) filled with ``fill``: the
    samples behind it are the sentinels."""
    big = torch.full((shape[0] + 1,) + tuple(shape[1:]), fill, dtype=dtype, device="cuda").contiguous(memory_format=fmt)
    return big, big[:shape[0]]


def _flat_backed(n, dtype, fill=SENT):
    big = torch.full((n + 37,), fill, dtype=dtype, device="cuda")
    return big, big[:n]


def _sent_ok(big, n_front, what):
    tail = big[n_front:]
    assert bool((tail == SENT).all()), f"{what}: a kernel wrote behind its output"


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(-1).view(torch.uint8).cpu(),
                                              b.contiguous().view(-1).view(torch.uint8).cpu())


def _dims(x):
    return [0] + list(range(2, x.dim()))


def _b(x, v):
    return v.view([1, -1] + [1] * (x.dim() - 2))


CASES = [  # (shape, layouts)
    ((2, 1, 1, 1), (False,)),
    ((2, 2049), (False,)),
    ((5, 3, 7, 3), (False, True)),
    ((9, 64, 13, 11), (False, True)),
    ((33, 64, 17, 19), (False, True)),
    ((3, 512, 7, 7), (False, True)),
    ((4, 2049, 3, 5), (False, True)),
    ((6, 64, 33), (False,)),
    ((2, 8, 4, 4, 8), (False, True)),
    ((64, 64, 112, 112), (False, True)),
]


def _run_kernels(K, x, w, b, rm, rv, dy, mb, eps=1e-5, momentum=0.1):
    """stats -> apply -> backward reduce -> backward apply at world 1, every output in a sentinel-backed buffer."""
    C, fmt = x.shape[1], _fmt(x.shape, not x.is_contiguous())
    tickets = torch.zeros(C, dtype=torch.int32, device="cuda")
    n_ex = exchange_numel(1 + 2 * C, 1)
    ex_big, ex = _flat_backed(n_ex, torch.float64)
    st_big, stats = _flat_backed(2 * C + 1, torch.float64)
    y_big, y = _backed(x.shape, x.dtype, fmt)
    K.bn_launch(0, x, None, None, ex, stats, tickets, None, None, None, None, None, None, None, 0.0, 0.0, mb)
    K.bn_launch(1, x, None, y, ex, stats, None, w, b, rm, rv, None, None, None, momentum, eps, mb)
    exb_big, exb = _flat_backed(exchange_numel(2 * C, 1), torch.float64)
    gw_big, gw = _flat_backed(C, w.dtype)
    gb_big, gb = _flat_backed(C, w.dtype)
    K.bn_launch(2, x, dy, None, exb, stats, tickets, None, None, None, None, None, gw, gb, 0.0, 0.0, mb)
    dx_big, dx = _backed(x.shape, x.dtype, fmt)
    K.bn_launch(3, x, dy, dx, exb, stats, None, w, None, None, None, None, None, None, 0.0, 0.0, mb)
    torch.cuda.synchronize()
    for big, n, what in ((ex_big, n_ex, "ex"), (st_big, 2 * C + 1, "stats"), (exb_big, exb.numel(), "backward ex"),
                         (gw_big, C, "grad_weight"), (gb_big, C, "grad_bias")):
        _sent_ok(big, n, what)
    for big, what in ((y_big, "y"), (dx_big, "dx")):
        _sent_ok(big[x.shape[0]:].reshape(-1), 0, what)
    assert int(tickets.abs().sum()) == 0, "tickets not reset"
    return dict(ex=ex.clone(), stats=stats.clone(), y=y.clone(), exb=exb.clone(), gw=gw.clone(), gb=gb.clone(), dx=dx.clone())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("pdtype", ["fp32", "same"])
def test_kernels_world_one_against_fp64(K, sms, dtype, pdtype):
    g = torch.Generator(device="cuda").manual_seed(5)
    for shape, layouts in CASES:
        if pdtype == "same" and shape[1] == 64 and shape[0] == 64 and dtype == torch.float32:
            continue                                        # the stem once per dtype is enough for fp32 parameters
        for cl in layouts:
            C = shape[1]
            pd = torch.float32 if pdtype == "fp32" else dtype
            x = (torch.randn(shape, generator=g, device="cuda") * 2 + 0.5).to(dtype).contiguous(memory_format=_fmt(shape, cl))
            dy = torch.randn(shape, generator=g, device="cuda").to(dtype).contiguous(memory_format=_fmt(shape, cl))
            w = (torch.rand(C, generator=g, device="cuda") + 0.5).to(pd)
            b = (torch.rand(C, generator=g, device="cuda") - 0.5).to(pd)
            rm0 = torch.rand(C, generator=g, device="cuda").to(pd)
            rv0 = (torch.rand(C, generator=g, device="cuda") + 0.5).to(pd)
            for mb in (sms, 3):
                rm_big, rm = _flat_backed(C, pd)
                rv_big, rv = _flat_backed(C, pd)
                rm.copy_(rm0)
                rv.copy_(rv0)
                out = _run_kernels(K, x, w, b, rm, rv, dy, mb)
                _sent_ok(rm_big, C, "running_mean")
                _sent_ok(rv_big, C, "running_var")
                # fp64 reference
                xd, dyd, wd, bd = x.double(), dy.double(), w.double(), b.double()
                N = x.numel() // C
                mean = xd.mean(_dims(x))
                var = xd.var(_dims(x), unbiased=False)
                invstd = 1.0 / torch.sqrt(var + 1e-5)
                k1, k0 = wd * invstd, bd - mean * wd * invstd
                yref = xd * _b(x, k1) + _b(x, k0)
                bound = C_BOUND * 2.0 ** -24 * (xd.abs() * _b(x, k1.abs()) + _b(x, k0.abs())) + OUT_EPS[dtype] * yref.abs() + OUT_SUB[dtype]
                what = (str(dtype), pdtype, shape, cl, mb)
                assert bool(((out["y"].double() - yref).abs() <= bound).all()), ("y", what)
                assert torch.allclose(out["stats"][:C], mean, rtol=1e-12, atol=1e-12), ("mean", what)
                assert torch.allclose(out["stats"][C:2 * C], invstd, rtol=1e-9), ("invstd", what)
                pe = 2.0 ** -23 if pd == torch.float32 else OUT_EPS[pd] * 2
                rm_ref = 0.9 * rm0.double() + 0.1 * mean
                rv_ref = 0.9 * rv0.double() + 0.1 * var * N / (N - 1)
                assert torch.allclose(rm.double(), rm_ref, rtol=pe, atol=pe), ("running_mean", what)
                assert torch.allclose(rv.double(), rv_ref, rtol=pe, atol=pe), ("running_var", what)
                xmu = xd - _b(x, mean)
                sdy, sdx = dyd.sum(_dims(x)), (dyd * xmu).sum(_dims(x))
                scale = dyd.abs().sum(_dims(x)) * (1 + xmu.abs().amax(_dims(x)))
                assert bool(((out["gb"].double() - sdy).abs() <= pe * sdy.abs() + 1e-12 * scale).all()), ("grad_bias", what)
                gwr = sdx * invstd
                assert bool(((out["gw"].double() - gwr).abs() <= pe * gwr.abs() + 1e-12 * scale * invstd).all()), \
                    ("grad_weight", what)
                ka = wd * invstd
                kb = -ka * invstd * invstd * sdx / N
                kc = -ka * sdy / N - kb * mean
                dxr = dyd * _b(x, ka) + xd * _b(x, kb) + _b(x, kc)
                bound = C_BOUND * 2.0 ** -24 * (dyd.abs() * _b(x, ka.abs()) + xd.abs() * _b(x, kb.abs()) + _b(x, kc.abs())) \
                    + OUT_EPS[dtype] * dxr.abs() + OUT_SUB[dtype] + 2.0 ** -22 * (_b(x, (kb * mean).abs()))
                assert bool(((out["dx"].double() - dxr).abs() <= bound).all()), ("dx", what)
                rm.copy_(rm0)
                rv.copy_(rv0)
                again = _run_kernels(K, x, w, b, rm, rv, dy, mb)
                for k in out:
                    assert _bits(out[k], again[k]), ("not reproducible", k, what)


def _emulated_case(worlds, sizes, C, spatial, dtype, cl, momentum, seed):
    W = len(worlds)
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs, dys = [], []
    for n in sizes:
        shape = (n, C) + spatial
        fmt = _fmt(shape, cl)
        xs.append((torch.randn(shape, generator=g, device="cuda") * 1.5 - 0.3).to(dtype).contiguous(memory_format=fmt)
                  .requires_grad_(True))
        dys.append(torch.randn(shape, generator=g, device="cuda").to(dtype).contiguous(memory_format=fmt))
    w = (torch.rand(C, generator=g, device="cuda") + 0.5).requires_grad_(True)
    b = (torch.rand(C, generator=g, device="cuda") - 0.5).requires_grad_(True)
    rms = [torch.zeros(C, device="cuda") for _ in range(W)]
    rvs = [torch.ones(C, device="cuda") for _ in range(W)]
    nbts = [torch.full((), 3, dtype=torch.int64, device="cuda") for _ in range(W)]
    tickets = [torch.zeros(C, dtype=torch.int32, device="cuda") for _ in range(W)]
    ys, grads = [None] * W, [None] * W

    def fwd(r, world):
        ys[r] = SyncBatchNormFunction.apply(xs[r], w, b, rms[r], rvs[r], nbts[r] if momentum is None else None,
                                            0.0 if momentum is None else momentum, 1e-5, world, tickets[r])

    def bwd(r, world):
        grads[r] = torch.autograd.grad(ys[r], [xs[r], w, b], dys[r], retain_graph=True)

    CE.on_ranks(worlds, fwd)
    CE.on_ranks(worlds, bwd)
    stats = [y.grad_fn.saved_tensors[2] for y in ys]
    for r in range(1, W):
        for a, bb, what in ((stats[r], stats[0], "mean / invstd / N"), (rms[r], rms[0], "running_mean"),
                            (rvs[r], rvs[0], "running_var")):
            assert _bits(a, bb), (what, r, W)
    xg = torch.cat([x.detach().double() for x in xs])
    dyg = torch.cat([d.double() for d in dys])
    N = xg.numel() // C
    mean = xg.mean(_dims(xg))
    var = xg.var(_dims(xg), unbiased=False)
    assert int(stats[0][2 * C]) == N
    assert torch.allclose(stats[0][:C], mean, rtol=1e-12, atol=1e-12)
    assert torch.allclose(stats[0][C:2 * C], 1 / torch.sqrt(var + 1e-5), rtol=1e-9)
    m = 1.0 / 3 if momentum is None else momentum
    assert torch.allclose(rms[0].double(), m * mean, rtol=2e-7, atol=1e-7)
    assert torch.allclose(rvs[0].double(), (1 - m) + m * var * N / (N - 1), rtol=2e-7, atol=1e-7)
    xr = xg.clone().requires_grad_(True)
    wr, br = w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    yr = F.batch_norm(xr, None, None, wr, br, True, 0.0, 1e-5)
    gx, gw, gb = torch.autograd.grad(yr, [xr, wr, br], dyg)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    off = 0
    for r, n in enumerate(sizes):
        torch.testing.assert_close(ys[r].double(), yr[off:off + n].detach(), rtol=tol, atol=tol)
        torch.testing.assert_close(grads[r][0].double(), gx[off:off + n], rtol=tol, atol=tol)
        off += n
    torch.testing.assert_close(sum(gr[1].double() for gr in grads), gw, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(sum(gr[2].double() for gr in grads), gb, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("world", range(1, 9))
def test_emulated_ranks_share_bit_identical_statistics(sms, world):
    # every kernel instance runs once at world 1 first: a module loaded lazily while a peer's kernel spins may wait for it
    warm = CE.symm_worlds(1, sms, [0])
    cases = [(64, (5, 6), torch.bfloat16, True, 0.1), (3, (7,), torch.float32, False, None),
             (130, (), torch.float16, False, 0.2)]
    for k, (C, spatial, dtype, cl, mom) in enumerate(cases):
        _emulated_case(warm[0], [4], C, spatial, dtype, cl, mom, k)
    worlds, keep = CE.symm_worlds(world, sms, list(range(world)))
    for k, (C, spatial, dtype, cl, mom) in enumerate(cases):
        sizes = [(3 * r + k) % 5 for r in range(world)]
        sizes[0] = max(sizes[0], 2)                      # the global batch holds more than one value per channel
        _emulated_case(worlds, sizes, C, spatial, dtype, cl, mom, 100 * world + k)
    del keep, warm


def test_module_against_cudnn_batch_norm():
    torch.manual_seed(0)
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 3e-2)):
        ref = nn.BatchNorm2d(64).cuda()
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
        mine = b2.SyncBatchNorm.convert_sync_batchnorm(nn.Sequential(nn.BatchNorm2d(64))).cuda()[0]
        mine.load_state_dict(ref.state_dict())
        for step in range(3):
            x = (torch.randn(16, 64, 28, 28, device="cuda") * 2 + 1).to(dtype).contiguous(memory_format=torch.channels_last)
            xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
                ya, yb = ref(xa), mine(xb)
            assert yb.dtype == x.dtype and yb.is_contiguous(memory_format=torch.channels_last)
            torch.testing.assert_close(yb.float(), ya.float(), rtol=tol, atol=tol)
            dy = torch.randn_like(ya)
            ya.backward(dy)
            yb.backward(dy)
            torch.testing.assert_close(xb.grad.float(), xa.grad.float(), rtol=tol, atol=tol)
            torch.testing.assert_close(mine.weight.grad, ref.weight.grad, rtol=1e-3, atol=1e-3)
            torch.testing.assert_close(mine.bias.grad, ref.bias.grad, rtol=1e-3, atol=1e-3)
            torch.testing.assert_close(mine.running_mean, ref.running_mean, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(mine.running_var, ref.running_var, rtol=1e-5, atol=1e-6)
            assert int(mine.num_batches_tracked) == int(ref.num_batches_tracked)
        ref.eval()
        mine.eval()
        x = torch.randn(4, 64, 8, 8, device="cuda")
        torch.testing.assert_close(mine(x), ref(x), rtol=1e-5, atol=1e-5)


def test_no_host_synchronisation_and_graph_replay_bit_equal():
    torch.manual_seed(1)
    for momentum in (0.1, None):
        m = b2.SyncBatchNorm(32, momentum=momentum).cuda()
        x = torch.randn(8, 32, 10, 10, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_(True)
        dy = torch.randn_like(x)
        m(x).backward(dy)                                   # warm-up: lazy allocations and module loads
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = m(x)
            y.backward(dy)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
    # graph: forward + backward captured, replayed, against eager from the same state
    m = b2.SyncBatchNorm(32, momentum=None).cuda()
    x = torch.randn(8, 32, 10, 10, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_(True)
    dy = torch.randn_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            m(x).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    m.weight.grad = None
    m.bias.grad = None
    with torch.cuda.graph(graph):
        y = m(x)
        y.backward(dy)
    m.load_state_dict(state)
    graph.replay()
    torch.cuda.synchronize()
    got = (y.clone(), x.grad.clone(), m.weight.grad.clone(), {k: v.clone() for k, v in m.state_dict().items()})
    m.load_state_dict(state)
    x2 = x.detach().clone().requires_grad_(True)
    m.weight.grad = None
    m.bias.grad = None
    y2 = m(x2)
    y2.backward(dy)
    assert _bits(got[0], y2) and _bits(got[1], x2.grad) and _bits(got[2], m.weight.grad)
    for k, v in m.state_dict().items():
        assert _bits(got[3][k], v), k


def test_converted_resnet18_trains_like_batch_norm_under_bf16_autocast():
    from dist_tuto.pth_b200.models.resnet import ResNet18
    losses = {}
    for conv in (False, True):
        torch.manual_seed(0)
        net = ResNet18().cuda().to(memory_format=torch.channels_last)
        if conv:
            net = b2.SyncBatchNorm.convert_sync_batchnorm(net)
            assert sum(isinstance(mod, b2.SyncBatchNorm) for mod in net.modules()) == 20
        opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
        g = torch.Generator(device="cuda").manual_seed(3)
        out = []
        for _ in range(4):
            x = torch.randn(32, 3, 32, 32, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
            t = torch.randint(0, 10, (32,), generator=g, device="cuda")
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(net(x), t)
            opt.zero_grad()
            loss.backward()
            opt.step()
            out.append(float(loss))
        losses[conv] = out
    for a, b_ in zip(losses[False], losses[True]):
        assert abs(a - b_) <= 0.05 * abs(a), losses
