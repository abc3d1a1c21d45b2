"""SyncBatchNorm kernels (csrc/batchnorm.cu) in every configuration ``SyncBatchNorm`` hands them, on one H100, against the
fp64 reference and bounds of tests/sync_bn_checks.py.

* Kernels through ``bn_launch`` at world 1, every output in a sentinel-backed buffer (parameter-sized buffers are backed
  by twice their size, so a write in a wider dtype lands on sentinels), tickets zero afterwards, each case run twice and
  bit-identical, at ``max_blocks`` = SM count and 3:
  weight / bias / running stats each present or absent (``weight=None``, ``bias=None``, ``running_mean=None``); every
  (input, parameter, running-stat) dtype triple; ``momentum=None`` with a device ``num_batches_tracked`` of 5; the channel
  counts around a channels-last tile (fp32 C = 124 / 128 / 132, bf16 / fp16 C = 248 / 256 / 264) in both layouts; and
  16-byte-misaligned x, dy, y and dx (offset views of a flat buffer with C or L a multiple of 8), which take the scalar
  kernels.
* ``SyncBatchNorm`` against ``nn.BatchNorm{1,2,3}d`` in float64 on CPU from the same state, for three steps and then in
  eval: affine x track_running_stats x momentum in {0.1, None}; and every branch of ``SyncBatchNormFunction``: a contiguous
  ``dy`` for a channels-last ``x`` and the reverse, a channel slice, ``x`` without grad (``bn_backward_reduce`` only), frozen
  affine parameters, a zero weight, and a bias without a weight.
* Emulated ranks, worlds 1-8 (tests/emulated_ranks.symm_worlds): no affine, no running stats, mixed dtypes,
  misaligned local inputs and a zero-size local batch; y and dx within the world-1 bound of the global batch, the
  parameters' gradients within it of each rank's local sums, statistics and running stats bit-identical across ranks.
* A global count of one at world >= 2: the running var is NaN, as torch's ``batch_norm_gather_stats_with_counts`` makes it
  non-finite.
* A large-mean input records the error of the one-pass fp64 variance (printed, not asserted).
"""
import pytest
import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
import emulated_ranks as E
import sync_bn_checks as S
from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.parallel import sync_bn as SB
from dist_tuto.pth_b200.parallel.sync_bn import SyncBatchNormFunction, exchange_numel
from emulated_ranks import pytestmark, sms  # noqa: F401

SENT = -12345.0
DT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
# (input, parameter, running-stat) dtypes: each of the latter two fp32 or the input's
TRIPLES = ["fp32-fp32-fp32", "bf16-fp32-fp32", "bf16-bf16-fp32", "bf16-fp32-bf16", "bf16-bf16-bf16",
           "fp16-fp32-fp32", "fp16-fp16-fp32", "fp16-fp32-fp16", "fp16-fp16-fp16"]


@pytest.fixture(scope="module")
def K():
    return _ext.C()


def _fmt(ndim, cl):
    if not cl or ndim < 4:
        return torch.contiguous_format
    return torch.channels_last if ndim == 4 else torch.channels_last_3d


def _strides(shape, cl):
    return torch.empty(shape, device="meta").contiguous(memory_format=_fmt(len(shape), cl)).stride()


def _flat_view(shape, dtype, cl, off, fill=SENT):
    """A tensor of ``shape`` (plain or channels-last) at element ``off`` of a flat buffer filled with ``fill`` that holds 64
    more elements behind it: off = 1 makes it 16-byte misaligned."""
    n = 1
    for s in shape:
        n *= s
    big = torch.full((off + n + 64,), fill, dtype=dtype, device="cuda")
    return big, torch.as_strided(big, shape, _strides(shape, cl), off)


def _sent_ok(big, view, what):
    n = view.numel()
    off = view.storage_offset()
    assert bool((big[:off] == SENT).all()) and bool((big[off + n:] == SENT).all()), f"{what}: a kernel wrote outside"


def _pbacked(v, dtype=None):
    """A copy of the per-channel vector v in a buffer of twice its size plus 37, the rest sentinels."""
    if v is None:
        return None, None
    C = v.numel()
    big = torch.full((2 * C + 37,), SENT, dtype=dtype or v.dtype, device="cuda")
    big[:C].copy_(v)
    return big, big[:C]


def _bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.detach().contiguous().view(-1).view(torch.uint8).cpu(),
                                              b.detach().contiguous().view(-1).view(torch.uint8).cpu())


def _place(t, cl, off):
    """t copied into a sentinel-backed flat view (layout cl, element offset off)."""
    big, v = _flat_view(tuple(t.shape), t.dtype, cl, off)
    v.copy_(t)
    return big, v


def run_kernels(K, x, dy, w, b, rm0, rv0, momentum, nbt, mb, y_off=0, dx_off=0, eps=1e-5):
    """stats -> apply -> backward reduce -> backward apply at world 1, as SyncBatchNormFunction calls them; weight / bias /
    running stats may be None, and grad_weight / grad_bias are asked for with a weight / a bias."""
    C, cl = x.shape[1], not x.is_contiguous()
    tickets = torch.zeros(C, dtype=torch.int32, device="cuda")
    ex_big, ex = _flat_view((exchange_numel(1 + 2 * C, 1),), torch.float64, False, 0)
    st_big, stats = _flat_view((2 * C + 1,), torch.float64, False, 0)
    y_big, y = _flat_view(tuple(x.shape), x.dtype, cl, y_off)
    rm_big, rm = _pbacked(rm0)
    rv_big, rv = _pbacked(rv0)
    nbt_t = None if nbt is None else torch.full((), nbt, dtype=torch.int64, device="cuda")
    K.bn_launch(0, x, None, None, ex, stats, tickets, None, None, None, None, None, None, None, 0.0, 0.0, mb)
    K.bn_launch(1, x, None, y, ex, stats, None, w, b, rm, rv, nbt_t, None, None, momentum, eps, mb)
    exb_big, exb = _flat_view((exchange_numel(2 * C, 1),), torch.float64, False, 0)
    gw_big, gw = _pbacked(None if w is None else torch.zeros_like(w))
    gb_big, gb = _pbacked(None if b is None else torch.zeros_like(b))
    K.bn_launch(2, x, dy, None, exb, stats, tickets, None, None, None, None, None, gw, gb, 0.0, 0.0, mb)
    dx_big, dx = _flat_view(tuple(x.shape), x.dtype, cl, dx_off)
    K.bn_launch(3, x, dy, dx, exb, stats, None, w, None, None, None, None, None, None, 0.0, 0.0, mb)
    torch.cuda.synchronize()
    for big, v, what in ((ex_big, ex, "ex"), (st_big, stats, "stats"), (y_big, y, "y"), (exb_big, exb, "backward ex"),
                         (dx_big, dx, "dx"), (rm_big, rm, "running_mean"), (rv_big, rv, "running_var"),
                         (gw_big, gw, "grad_weight"), (gb_big, gb, "grad_bias")):
        if big is not None:
            _sent_ok(big, v, what)
    assert int(tickets.abs().sum()) == 0, "tickets not reset"
    assert int(stats[2 * C]) == x.numel() // C
    return dict(y=y.clone(), mean=stats[:C].clone(), invstd=stats[C:2 * C].clone(), stats=stats.clone(), ex=ex.clone(),
                exb=exb.clone(), dx=dx.clone(), rm=None if rm is None else rm.clone(),
                rv=None if rv is None else rv.clone(), gw=None if gw is None else gw.clone(),
                gb=None if gb is None else gb.clone())


def _inputs(shape, dtype, pdtype, rdtype, cl, seed, x_off=0, dy_off=0):
    """x with distinct channel means and std 1.5, dy with mean 0.3, weights in [0.5, 1.5) and biases of both signs."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = shape[1]
    off = torch.linspace(-1.0, 1.0, C, device="cuda").view([1, C] + [1] * (len(shape) - 2))
    x = (torch.randn(shape, generator=g, device="cuda") * 1.5 + off).to(dtype)
    dy = (torch.randn(shape, generator=g, device="cuda") + 0.3).to(dtype)
    x = _place(x, cl, x_off)[1]
    dy = _place(dy, cl, dy_off)[1]
    w = (torch.rand(C, generator=g, device="cuda") + 0.5).to(pdtype)
    b = (torch.rand(C, generator=g, device="cuda") - 0.5).to(pdtype)
    rm = torch.rand(C, generator=g, device="cuda").to(rdtype)
    rv = (torch.rand(C, generator=g, device="cuda") + 0.5).to(rdtype)
    return x, dy, w, b, rm, rv


def check_case(K, mbs, x, dy, w, b, rm0, rv0, momentum=0.1, nbt=None, y_off=0, dx_off=0, what=()):
    """Every output within the bounds, twice, bit-identical; returns the worst ratios."""
    pd = w.dtype if w is not None else (b.dtype if b is not None else torch.float32)
    rd = rm0.dtype if rm0 is not None else torch.float32
    fwd = S.forward_ref(x, w, b, rm0, rv0, momentum, nbt)
    bwd = S.backward_ref(x, dy, fwd, w)
    worst = {}
    for mb in mbs:
        out = run_kernels(K, x, dy, w, b, rm0, rv0, 0.0 if momentum is None else momentum, nbt, mb, y_off, dx_off)
        ratios = S.forward_checks(out, x, fwd, x.dtype, rd)
        ratios.update(S.backward_checks(out, x, dy, fwd, bwd, x.dtype, pd))
        assert not S.failures(ratios), (what, mb, ratios)
        again = run_kernels(K, x, dy, w, b, rm0, rv0, 0.0 if momentum is None else momentum, nbt, mb, y_off, dx_off)
        for k in out:
            assert _bits(out[k], again[k]), ("not reproducible", k, what, mb)
        for k, v in ratios.items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


# ------------------------------------------------------------------------------------------------ kernels at world 1
@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
def test_weight_bias_and_running_stats_present_or_absent(K, sms, dtype):
    dt = DT[dtype]
    for shape, cl in (((6, 24, 5, 7), True), ((6, 24, 5, 7), False), ((37, 24), True), ((4, 24, 16), False)):
        x, dy, w0, b0, rm0, rv0 = _inputs(shape, dt, torch.float32, torch.float32, cl, seed=shape[0])
        for w in (w0, None):                             # weight=None
            for b in (b0, None):                         # bias=None
                for rm, rv in ((rm0, rv0), (None, None)):    # running_mean=None, running_var=None
                    check_case(K, (sms, 3), x, dy, w, b, rm, rv,
                               what=(dtype, shape, cl, w is None, b is None, rm is None))


@pytest.mark.parametrize("triple", TRIPLES)
def test_input_parameter_and_running_stat_dtypes(K, sms, triple):
    dt, pd, rd = (DT[s] for s in triple.split("-"))
    for shape, cl in (((5, 64, 6, 6), True), ((5, 64, 6, 6), False), ((3, 40, 16), False), ((50, 16), True)):
        x, dy, w, b, rm, rv = _inputs(shape, dt, pd, rd, cl, seed=7)
        for momentum, nbt in ((0.1, None), (None, 5)):
            check_case(K, (sms, 3), x, dy, w, b, rm, rv, momentum, nbt, what=(triple, shape, cl, momentum))


def test_momentum_none_reads_num_batches_tracked_on_the_device(K, sms):
    """The module passes momentum 0.0 with the counter; the factor must be 1 / num_batches_tracked (1/5), not 0."""
    for cl in (True, False):
        x, dy, w, b, rm, rv = _inputs((4, 32, 5, 5), torch.float32, torch.float32, torch.float32, cl, seed=3)
        check_case(K, (sms, 3), x, dy, w, b, rm, rv, momentum=None, nbt=5, what=cl)
        out = run_kernels(K, x, dy, w, b, rm, rv, 0.0, 5, sms)
        fwd = S.forward_ref(x, w, b, rm, rv, None, 5)
        assert S.check_running(out["rm"], fwd["rm"], torch.float32) <= 1.0
        assert not torch.equal(out["rm"], rm), "momentum=None left the running mean unchanged"


@pytest.mark.parametrize("dtype,channels", [("fp32", (124, 128, 132)), ("bf16", (248, 256, 264)),
                                            ("fp16", (248, 256, 264))])
def test_channels_last_tile_edges(K, sms, dtype, channels):
    """A tile is cx lanes x V channels, at most 256: C just below, at and just above a tile, so the last tile holds a partial
    vector count; also channel-first at the same C (with L a multiple of 8, vectorised)."""
    dt = DT[dtype]
    for C in channels:
        for shape, cl in (((5, C, 3, 5), True), ((3, C, 4, 4), False), ((70, C), True)):
            x, dy, w, b, rm, rv = _inputs(shape, dt, torch.float32, dt, cl, seed=C)
            check_case(K, (sms, 3, 1), x, dy, w, b, rm, rv, what=(dtype, C, shape, cl))


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
def test_misaligned_views_take_the_scalar_kernels(K, sms, dtype):
    """Views at one element past a 16-byte boundary, with C (channels-last) or L (channel-first) a multiple of 8, so that
    only the pointer clears the vector path; one of x / dy / y / dx misaligned at a time, then all four.  Not compared bit for
    bit with the aligned run: the scalar kernels map lanes and splits differently, so the fp64 sums run in another order."""
    dt = DT[dtype]
    for shape, cl in (((4, 16, 3, 5), True), ((4, 5, 4, 4), False), ((33, 64), True), ((3, 24, 8), False)):
        for xo, dyo, yo, dxo in ((1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (1, 1, 1, 1)):
            x, dy, w, b, rm, rv = _inputs(shape, dt, dt, torch.float32, cl, seed=11, x_off=xo, dy_off=dyo)
            assert (x.data_ptr() % 16 != 0) == bool(xo) and (dy.data_ptr() % 16 != 0) == bool(dyo)
            check_case(K, (sms, 3), x, dy, w, b, rm, rv, y_off=yo, dx_off=dxo, what=(dtype, shape, cl, xo, dyo, yo, dxo))


def test_large_mean_records_the_one_pass_variance_error(K, sms):
    """var = max(S2/N - mean^2, 0) loses about (mean/std)^2 ulps of fp64 to cancellation; record how far from zero-mean
    inputs invstd stays within rtol 1e-9 (printed, not asserted)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    print()
    for ratio in (0.0, 10.0, 100.0, 300.0, 1e3, 3e3, 1e4):
        for cl in (True, False):
            x = (torch.randn(32, 16, 16, 16, generator=g, device="cuda") + ratio).contiguous(memory_format=_fmt(4, cl))
            dy = torch.randn_like(x)
            out = run_kernels(K, x, dy, None, None, None, None, 0.1, None, sms)
            fwd = S.forward_ref(x)
            rel = float(((out["invstd"] - fwd["invstd"].cuda()).abs() / fwd["invstd"].cuda()).max())
            merr = float(((out["mean"] - fwd["mean"].cuda()).abs() / (1 + fwd["mean"].cuda().abs())).max())
            print(f"mean/std {ratio:g} {'channels-last' if cl else 'channel-first'}: invstd rel error {rel:.3g}, "
                  f"mean error {merr:.3g}")
            assert rel == rel and merr == merr


# ------------------------------------------------------------------------------------------------------------ module
class _Spy:
    """Records the kernel kinds SyncBatchNormFunction launches and the exchanges it issues."""

    def __init__(self, monkeypatch):
        self.kinds, self.exchanges = [], 0
        real_C, real_ex = _ext.C, SB._exchange
        spy = self

        class Proxy:
            def __getattr__(self, name):
                return getattr(real_C(), name)

            def bn_launch(self, kind, *a):
                spy.kinds.append(kind)
                return real_C().bn_launch(kind, *a)

        def exchange(buf, comm_):
            if comm_ is not None:
                spy.exchanges += 1
            return real_ex(buf, comm_)

        proxy = Proxy()
        monkeypatch.setattr(_ext, "C", lambda: proxy)
        monkeypatch.setattr(SB, "_exchange", exchange)

    def reset(self):
        self.kinds, self.exchanges = [], 0


_BN = {3: nn.BatchNorm1d, 4: nn.BatchNorm2d, 5: nn.BatchNorm3d}
_SHAPES = {3: (6, 8, 10), 4: (4, 8, 5, 6), 5: (3, 8, 3, 4, 5)}


def _pair(ndim, affine, track, momentum, seed=0):
    torch.manual_seed(seed)
    ref = _BN[ndim](8, momentum=momentum, affine=affine, track_running_stats=track).double()
    if affine:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
    if track:
        with torch.no_grad():
            ref.running_mean.uniform_(-0.5, 0.5)
            ref.running_var.uniform_(0.5, 1.5)
    mine = b2.SyncBatchNorm(8, momentum=momentum, affine=affine, track_running_stats=track).cuda()
    mine.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    ref.load_state_dict({k: v.double().cpu() if v.is_floating_point() else v.cpu() for k, v in mine.state_dict().items()})
    return ref, mine


def _compare_step(ref, mine, x, dy, train, what):
    """One forward + backward of both modules from the same state; y and x.grad against the kernels' bounds around the
    fp64 module's values, the parameters' grads and the buffers likewise."""
    ref.train(train)
    mine.train(train)
    rm0 = None if mine.running_mean is None else mine.running_mean.clone()
    rv0 = None if mine.running_var is None else mine.running_var.clone()
    xr = x.detach().double().cpu().requires_grad_(True)
    xm = x.detach().requires_grad_(True)                 # x's own strides and offset, a channel slice included
    yr, ym = ref(xr), mine(xm)
    yr.backward(dy.double().cpu())
    ym.backward(dy)
    batch_stats = train or not mine.track_running_stats
    if batch_stats:
        mom = mine.momentum
        nbt = None if mine.num_batches_tracked is None else int(mine.num_batches_tracked)
        fwd = S.forward_ref(x, mine.weight, mine.bias, rm0 if train else None, rv0 if train else None, mom, nbt)
        torch.testing.assert_close(fwd["y"], yr.detach(), rtol=1e-12, atol=1e-12)   # the helper is torch's batch norm
        bwd = S.backward_ref(x, dy, fwd, mine.weight)
        torch.testing.assert_close(bwd["dx"], xr.grad, rtol=1e-10, atol=1e-12)
        ratios = S.forward_checks(dict(y=ym, rm=mine.running_mean if train else None,
                                       rv=mine.running_var if train else None), x, fwd, x.dtype)
        ratios.update(S.backward_checks(dict(dx=xm.grad, gw=None if mine.weight is None else mine.weight.grad,
                                             gb=None if mine.bias is None else mine.bias.grad), x, dy, fwd, bwd, x.dtype))
        assert not S.failures(ratios), (what, ratios)
    else:                                                # eval with running stats: torch's own batch_norm, no kernels
        torch.testing.assert_close(ym.double().cpu(), yr.detach(), rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(xm.grad.double().cpu(), xr.grad, rtol=1e-5, atol=1e-5)
    if mine.track_running_stats:
        for k in ("running_mean", "running_var"):
            torch.testing.assert_close(getattr(mine, k).double().cpu(), getattr(ref, k), rtol=1e-6, atol=1e-6)
        assert int(mine.num_batches_tracked) == int(ref.num_batches_tracked), what
    if mine.affine:
        for k in ("weight", "bias"):
            torch.testing.assert_close(getattr(mine, k).grad.double().cpu(), getattr(ref, k).grad, rtol=1e-5, atol=1e-5)
            getattr(mine, k).grad = None
            getattr(ref, k).grad = None
    return xm.grad


@pytest.mark.parametrize("ndim", [3, 4, 5])
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("track", [True, False])
@pytest.mark.parametrize("momentum", [0.1, None])
def test_module_against_fp64_batch_norm(ndim, affine, track, momentum):
    ref, mine = _pair(ndim, affine, track, momentum)
    g = torch.Generator(device="cuda").manual_seed(ndim)
    for step in range(4):
        train = step < 3                                   # three training steps, then eval (with or without running stats)
        cl = ndim > 3 and step % 2 == 1
        x = (torch.randn(_SHAPES[ndim], generator=g, device="cuda") * 2 + 0.5).contiguous(
            memory_format=_fmt(ndim, cl))
        dy = torch.randn(_SHAPES[ndim], generator=g, device="cuda") + 0.2
        _compare_step(ref, mine, x, dy, train, (ndim, affine, track, momentum, step))


def test_function_branches(monkeypatch):
    """Layout copies, non-contiguous inputs and which kernels run for each combination of gradients wanted."""
    spy = _Spy(monkeypatch)
    ref, mine = _pair(4, True, True, 0.1, seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    shape = (4, 8, 6, 5)
    x = torch.randn(shape, generator=g, device="cuda") * 2 + 0.5
    dy = torch.randn(shape, generator=g, device="cuda") + 0.2
    cl = torch.channels_last
    # channels-last x with a contiguous dy (copied into x's layout), and the reverse
    for xs, dys, what in ((x.contiguous(memory_format=cl), dy, "cl x, contiguous dy"),
                          (x, dy.contiguous(memory_format=cl), "contiguous x, cl dy")):
        spy.reset()
        gx = _compare_step(ref, mine, xs, dys, True, what)
        assert spy.kinds == [0, 1, 2, 3] and spy.exchanges == 0, (what, spy.kinds)
        assert gx.stride() == xs.stride(), what
    # a channel slice (non-contiguous in every layout): computed on a contiguous copy
    ref8, mine8 = _pair(4, True, True, 0.1, seed=2)
    wide = torch.randn(4, 12, 6, 5, generator=g, device="cuda") * 2 + 0.5
    xs = wide[:, 2:10]
    assert not xs.is_contiguous() and not xs.is_contiguous(memory_format=cl)
    _compare_step(ref8, mine8, xs, dy, True, "channel slice")
    # x without grad: bn_backward_reduce only, local grad_weight / grad_bias
    spy.reset()
    y = mine(x)
    y.backward(dy)
    assert spy.kinds == [0, 1, 2], spy.kinds
    fwd = S.forward_ref(x, mine.weight, mine.bias)
    sums = S.grad_sums(x, dy, fwd["mean"], fwd["invstd"])
    assert S.check_grad_weight(mine.weight.grad, sums, fwd["invstd"], torch.float32) <= 1.0
    assert S.check_grad_bias(mine.bias.grad, sums, torch.float32) <= 1.0
    mine.weight.grad = mine.bias.grad = None
    # frozen affine parameters, x requiring grad: no parameter gradients, stats + apply + reduce + apply
    mine.weight.requires_grad_(False)
    mine.bias.requires_grad_(False)
    spy.reset()
    xg = x.clone().requires_grad_(True)
    mine(xg).backward(dy)
    assert spy.kinds == [0, 1, 2, 3] and mine.weight.grad is None and mine.bias.grad is None
    fwd = S.forward_ref(x, mine.weight, mine.bias)
    bwd = S.backward_ref(x, dy, fwd, mine.weight)
    assert S.check_dx(xg.grad, x, dy, fwd, bwd, torch.float32) <= 1.0
    # nothing wanted: no backward kernel
    spy.reset()
    mine(x).sum()
    assert spy.kinds == [0, 1]


def test_zero_weight_and_bias_without_weight():
    """weight all zero (zero_init_residual): y = bias, dx = 0, grad_weight still the sums; the functional form with a bias
    but no weight gives the bias its gradient."""
    g = torch.Generator(device="cuda").manual_seed(4)
    x = (torch.randn(6, 16, 7, 7, generator=g, device="cuda") * 2 + 0.5).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(x.shape, generator=g, device="cuda") + 0.2
    m = b2.SyncBatchNorm(16).cuda()
    with torch.no_grad():
        m.weight.zero_()
        m.bias.uniform_(-0.5, 0.5)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    y.backward(dy)
    fwd = S.forward_ref(x, m.weight, m.bias)
    bwd = S.backward_ref(x, dy, fwd, m.weight)
    assert torch.equal(y, S.bview(y, m.bias.detach()).expand_as(y))
    assert not S.failures(S.backward_checks(dict(dx=xg.grad, gw=m.weight.grad, gb=m.bias.grad), x, dy, fwd, bwd,
                                            torch.float32))
    assert bool((xg.grad == 0).all()) and bool((m.weight.grad != 0).all())
    b = (torch.rand(16, generator=g, device="cuda") - 0.5).requires_grad_(True)
    xg = x.clone().requires_grad_(True)
    y = SB.sync_batch_norm(xg, None, b, None, None, None, 0.1, 1e-5)
    y.backward(dy)
    fwd = S.forward_ref(x, None, b)
    bwd = S.backward_ref(x, dy, fwd, None)
    assert b.grad is not None, "a bias without a weight got no gradient"
    assert not S.failures(S.backward_checks(dict(dx=xg.grad, gb=b.grad), x, dy, fwd, bwd, torch.float32))
    assert S.check_y(y, x, fwd, torch.float32) <= 1.0


# ---------------------------------------------------------------------------------------------------- emulated ranks
EMU_CASES = [  # (C, spatial, dtype, pdtype, rdtype, affine, track, cl, momentum, misaligned)
    (24, (5, 6), "bf16", "fp32", "bf16", False, True, True, 0.1, False),       # no affine, mixed dtypes
    (16, (7,), "fp16", "fp16", "fp32", True, False, False, 0.1, False),        # no running stats, fp16 parameters
    (32, (3, 4), "fp32", "fp32", "fp32", True, True, True, None, True),        # misaligned local x / dy, momentum=None
    (8, (16,), "bf16", "bf16", "bf16", True, True, False, 0.2, True),          # misaligned channel-first, L = 16
    (130, (), "fp16", "fp32", "fp16", True, True, False, None, False),
]


def emulated_case(worlds, sizes, case, seed, x_grad=True):
    C, spatial, dtype, pdtype, rdtype, affine, track, cl, momentum, mis = case
    dt, pd, rd = DT[dtype], DT[pdtype], DT[rdtype]
    W = len(worlds)
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs, dys = [], []
    for n in sizes:
        shape = (n, C) + spatial
        x = (torch.randn(shape, generator=g, device="cuda") * 1.5 - 0.3).to(dt)
        dy = (torch.randn(shape, generator=g, device="cuda") + 0.3).to(dt)
        xs.append(_place(x, cl and len(shape) >= 4, int(mis))[1].requires_grad_(x_grad))
        dys.append(_place(dy, cl and len(shape) >= 4, int(mis))[1])
    w = (torch.rand(C, generator=g, device="cuda") + 0.5).to(pd).requires_grad_(True) if affine else None
    b = (torch.rand(C, generator=g, device="cuda") - 0.5).to(pd).requires_grad_(True) if affine else None
    rm0 = torch.rand(C, generator=g, device="cuda").to(rd) if track else None
    rv0 = (torch.rand(C, generator=g, device="cuda") + 0.5).to(rd) if track else None
    rms = [None if rm0 is None else rm0.clone() for _ in range(W)]
    rvs = [None if rv0 is None else rv0.clone() for _ in range(W)]
    nbts = [torch.full((), 4, dtype=torch.int64, device="cuda") for _ in range(W)]
    tickets = [torch.zeros(C, dtype=torch.int32, device="cuda") for _ in range(W)]
    ys, grads = [None] * W, [None] * W
    wants = [t for t in (w, b) if t is not None]

    def fwd_(r, world):
        ys[r] = SyncBatchNormFunction.apply(xs[r], w, b, rms[r], rvs[r], nbts[r] if momentum is None and track else None,
                                            0.0 if momentum is None else momentum, 1e-5, world, tickets[r])

    def bwd_(r, world):
        grads[r] = torch.autograd.grad(ys[r], ([xs[r]] if x_grad else []) + wants, dys[r], retain_graph=True)

    E.on_ranks(worlds, fwd_)
    E.on_ranks(worlds, bwd_)
    stats = [y.grad_fn.saved_tensors[2] for y in ys]
    for r in range(1, W):
        for a, bb, what in ((stats[r], stats[0], "mean / invstd / N"), (rms[r], rms[0], "running_mean"),
                            (rvs[r], rvs[0], "running_var")):
            assert _bits(a, bb), (what, r, W, case)
    xg = torch.cat([x.detach() for x in xs])
    dyg = torch.cat(dys)
    fwd = S.forward_ref(xg, w, b, rm0, rv0, momentum, 4)
    bwd = S.backward_ref(xg, dyg, fwd, w)
    assert int(stats[0][2 * C]) == fwd["N"]
    ratios = S.forward_checks(dict(mean=stats[0][:C], invstd=stats[0][C:2 * C], rm=rms[0], rv=rvs[0]), xg, fwd, dt, rd)
    off = 0
    for r, n in enumerate(sizes):
        sl = slice(off, off + n)
        f_r = dict(fwd, y=fwd["y"][sl], k1=fwd["k1"], k0=fwd["k0"])
        ratios[f"y{r}"] = S.check_y(ys[r], xs[r], f_r, dt)
        local = S.grad_sums(xs[r], dys[r], fwd["mean"], fwd["invstd"])
        got = dict(gw=grads[r][int(x_grad)] if affine else None, gb=grads[r][int(x_grad) + 1] if affine else None)
        if x_grad:
            got["dx"] = grads[r][0]
        for k, v in S.backward_checks(got, xs[r], dys[r], fwd, dict(bwd, dx=bwd["dx"][sl]), dt, pd, local).items():
            ratios[f"{k}{r}"] = v
        off += n
    assert not S.failures(ratios), (W, sizes, case, ratios)


@pytest.mark.parametrize("world", range(1, 9))
def test_emulated_ranks_new_configurations(sms, world, monkeypatch):
    # every kernel instance runs once at world 1 first: a module loaded lazily while a peer's kernel spins may wait for it
    warm = E.symm_worlds(1, sms, [0])
    for k, case in enumerate(EMU_CASES):
        emulated_case(warm[0], [4], case, k)
        if case[5]:
            emulated_case(warm[0], [4], case, k, x_grad=False)
    worlds, keep = E.symm_worlds(world, sms, list(range(world)))
    for k, case in enumerate(EMU_CASES):
        sizes = [(2 * r + k + 1) % 4 for r in range(world)]
        sizes[0] = max(sizes[0], 2)                      # the global batch holds more than one value per channel
        if world > 1:
            sizes[-1] = 0                                # a zero-size local batch
        emulated_case(worlds, sizes, case, 100 * world + k)
    # x without grad: each rank's local grad_weight / grad_bias, no backward exchange
    spy = _Spy(monkeypatch)
    sizes = [3 + r % 2 for r in range(world)]
    emulated_case(worlds, sizes, EMU_CASES[2], 7, x_grad=False)
    assert spy.kinds == [0, 1] * world + [2] * world, spy.kinds
    assert spy.exchanges == world, spy.exchanges             # the forward's, one per rank; none in the backward
    del keep, warm


@pytest.mark.parametrize("world", [2, 3, 8])
def test_global_count_of_one(sms, world):
    """One rank holds one value per channel, the others none.  The kernels follow torch's formula: running_var takes
    var N / (N - 1) = 0 / 0, a NaN, where torch's batch_norm_gather_stats_with_counts divides by n - 1 = 0 as well and gets a
    non-finite value; mean, y (= bias) and dx (= 0) stay finite."""
    warm = E.symm_worlds(1, sms, [0])
    case = (12, (), "fp32", "fp32", "fp32", True, True, False, 0.1, False)
    emulated_case(warm[0], [4], case, 0)
    worlds, keep = E.symm_worlds(world, sms, list(range(world)))
    C = 12
    g = torch.Generator(device="cuda").manual_seed(world)
    xs = [torch.randn(1 if r == 0 else 0, C, generator=g, device="cuda").requires_grad_(True) for r in range(world)]
    dys = [torch.randn(x.shape, generator=g, device="cuda") for x in xs]
    w = (torch.rand(C, generator=g, device="cuda") + 0.5).requires_grad_(True)
    b = (torch.rand(C, generator=g, device="cuda") - 0.5).requires_grad_(True)
    rm0, rv0 = torch.rand(C, device="cuda"), torch.rand(C, device="cuda") + 0.5
    rms, rvs = [rm0.clone() for _ in range(world)], [rv0.clone() for _ in range(world)]
    tickets = [torch.zeros(C, dtype=torch.int32, device="cuda") for _ in range(world)]
    ys, grads = [None] * world, [None] * world

    def fwd_(r, wd):
        ys[r] = SyncBatchNormFunction.apply(xs[r], w, b, rms[r], rvs[r], None, 0.1, 1e-5, wd, tickets[r])

    def bwd_(r, wd):
        grads[r] = torch.autograd.grad(ys[r], [xs[r], w, b], dys[r], retain_graph=True)

    E.on_ranks(worlds, fwd_)
    E.on_ranks(worlds, bwd_)
    fwd = S.forward_ref(xs[0], w, b, rm0, rv0, 0.1)
    assert fwd["N"] == 1 and bool(torch.isnan(fwd["rv"]).all())
    for r in range(world):
        assert _bits(rms[r], rms[0]) and _bits(rvs[r], rvs[0])
        assert bool(torch.isnan(rvs[r]).all()), ("running_var", r, rvs[r])
        assert S.check_running(rms[r], fwd["rm"], torch.float32) <= 1.0
    assert S.check_y(ys[0], xs[0], fwd, torch.float32) <= 1.0
    bwd = S.backward_ref(xs[0], dys[0], fwd, w)
    assert not S.failures(S.backward_checks(dict(dx=grads[0][0], gw=grads[0][1], gb=grads[0][2]), xs[0], dys[0], fwd, bwd,
                                            torch.float32))
    assert bool(torch.isfinite(ys[0]).all()) and bool(torch.isfinite(grads[0][0]).all())
    # torch's formula on the same statistics (the rank without values is masked out, as torch.nn.SyncBatchNorm does)
    mean, invstd = torch.batch_norm_stats(xs[0].detach(), 1e-5)
    trm, trv = rm0.clone(), rv0.clone()
    tm, ti = torch.batch_norm_gather_stats_with_counts(xs[0].detach(), mean[None], invstd[None], trm, trv, 0.1, 1e-5,
                                                       torch.ones(1, device="cuda"))
    torch.testing.assert_close(tm, fwd["mean"].float().cuda())
    torch.testing.assert_close(trm, rms[0])
    assert not bool(torch.isfinite(trv).any()), ("torch's running_var", trv)
    del keep, warm
