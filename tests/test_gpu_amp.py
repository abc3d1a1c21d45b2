"""fp16 loss scaling on one H100: the scaled instances of the flat update kernels against their existing instances (with
sentinels around every buffer), the gated step counter, every flat optimizer on an fp16-autocast ResNet-18 driven by
``torch.amp.GradScaler`` against the same optimizer behind an explicit ``scaler.unscale_``, and a captured step with
``scaler.step`` / ``scaler.update`` and ``FlatEMA.update`` against eager steps, an overflowing replay included."""
import pytest
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.models.resnet import ResNet18
from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatEMA, FlatLAMB, FlatLARS, FlatSGD, adamw_scalars, lamb_scalars
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a GPU")]
DEV = torch.device("cuda", 0)
N = 4099                       # 1024 vectors and a 3-element tail
PAD = 64
SENT = -7.25


def guarded(src):
    """``src`` copied into the middle of a sentinel-filled buffer: (buffer, view)."""
    buf = torch.full((src.numel() + 2 * PAD,), SENT, dtype=src.dtype, device=DEV)
    view = buf[PAD:PAD + src.numel()]
    view.copy_(src)
    return buf, view


def sentinels_intact(buf):
    return bool((buf[:PAD] == SENT).all() and (buf[-PAD:] == SENT).all())


def scalar(x):
    return torch.tensor([x], dtype=torch.float32, device=DEV)


def unscaled(g, s):
    """torch's GradScaler.unscale_: g * fp32(1 / double(S)) on the device."""
    return g * scalar(s).double().reciprocal().float()


def state(seed):
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(N, generator=gen)
    m = torch.randn(N, generator=gen) * 0.1
    v = torch.rand(N, generator=gen) * 0.01
    g = torch.randn(N, generator=gen) * 3e-3
    g[::97] *= 1e-35                            # tiny values (~1e-38, a few of them subnormal)
    return p, m, v, g


C = None


def kern():
    global C
    if C is None:
        C = _ext.C()
    return C


def run(name, g_src, scale, found_inf=None, seed=1, zero_grad=True):
    """One launch of kernel ``name`` on fresh guarded state; returns every buffer (sentinels checked) and the aux outputs."""
    C = kern()
    p, m, v, _ = state(seed)
    bufs = [guarded(t.to(DEV)) for t in (p, m, v, g_src)]
    P, M, V, G = (b[1] for b in bufs)
    sq = torch.zeros(2, dtype=torch.float64, device=DEV)
    ws = torch.zeros(C.grad_sqnorm_workspace_numel(), dtype=torch.float32, device=DEV)
    gs = None if scale is None else scalar(scale)
    kw = {} if gs is None else {"grad_scale": gs}
    norm = torch.full((1,), SENT, device=DEV)
    clip = dict(max_grad_norm=0.01, sqnorms=sq, grad_norm_out=norm)
    gmap = torch.tensor([0, 1] * 512 + [1], dtype=torch.uint8, device=DEV)
    if name.endswith("clip") or name.startswith("cap"):
        C.grad_sqnorm(G, sq, 0, ws, **kw)
        C.grad_sqnorm(G[:17], sq, 1, ws, **kw)
    if name == "sgd":
        C.sgd_flat(P, M, G, 0.05, 0.9, 0.01, zero_grad, True, **kw)
    elif name == "sgd_clip":
        C.sgd_flat(P, M, G, 0.05, 0.9, 0.01, zero_grad, False, **clip, **kw)
    elif name == "sgd_grouped_clip":
        C.sgd_flat_grouped(P, M, G, gmap, [0.05, 0.1], [0.0, 0.01], 0.9, zero_grad, True, **clip, **kw)
    elif name == "adamw":
        C.adamw_flat(P, M, V, G, adamw_scalars(1e-3, (0.9, 0.999), 1e-8, 0.01, 3), zero_grad, **kw)
    elif name == "adamw_grouped_clip":
        sc = adamw_scalars(1e-3, (0.9, 0.999), 1e-8, 0.01, 3)
        C.adamw_flat_grouped(P, M, V, G, gmap, sc, [1.0, sc[0]], [sc[4], 2 * sc[4]], zero_grad, **clip, **kw)
    elif name in ("lamb", "lars_clip"):
        table, n_chunks = C.layerwise_table([0, 1500], [1500, N - 1500], [True, True], N, DEV)
        ws2 = (torch.zeros(2 * n_chunks, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV),
               torch.zeros(4, dtype=torch.float64, device=DEV))
        ratios = torch.full((2,), SENT, device=DEV)
        if name == "lamb":
            C.lamb_flat(P, M, V, G, table, n_chunks, *ws2, ratios, lamb_scalars(1e-3, (0.9, 0.999), 1e-6, 0.01, 3), zero_grad, **kw)
        else:
            C.lars_flat(P, M, G, table, n_chunks, *ws2, ratios, 0.1, 0.9, 1e-4, 1e-3, 1e-8, False, zero_grad, **clip, **kw)
        norm = torch.cat([norm, ratios])
    else:                                       # capturable: cap_sgd / cap_adamw, grouped and clipped
        lay = C.flat_scalars_layout()
        table = torch.zeros(lay["table_bytes"], dtype=torch.uint8, device=DEV)
        counter = torch.zeros(1, dtype=torch.int64, device=DEV)
        block = torch.zeros(lay["block_bytes"], dtype=torch.uint8, device=DEV)
        b1, b2_ = (0.9, 0.999) if name == "cap_adamw" else (0.0, 0.0)
        C.flat_scalars_sync(table, counter, block, [0.05, 0.1], [0.0, 0.01], b1, b2_, 1e-8 if b1 else 0.0, None, 2)
        amp = {} if found_inf is None else dict(grad_scale=gs, found_inf=scalar(found_inf))
        if name == "cap_sgd":
            C.sgd_flat_cap(P, M, G, gmap, block, 0.9, zero_grad, True, **clip, **amp)
        else:
            C.adamw_flat_cap(P, M, V, G, gmap, block, zero_grad, **clip, **amp)
    torch.cuda.synchronize()
    for b, _ in bufs:
        assert sentinels_intact(b), name
    return [t.clone() for t in (P, M, V, G, norm, sq)]


NAMES = ["sgd", "sgd_clip", "sgd_grouped_clip", "adamw", "adamw_grouped_clip", "lamb", "lars_clip", "cap_sgd", "cap_adamw"]


def _same(a, b):
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x, y.view(torch.int32) if y.dtype == torch.float32
                           else y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("scale", [2.0 ** 16, 1.0])
def test_scaled_instance_on_scaled_gradient_equals_existing(name, scale):
    g = state(1)[3].to(DEV)
    amp = {"found_inf": 0.0} if name.startswith("cap") else {}
    want = run(name, g, None, **({} if not amp else {"found_inf": None}))
    got = run(name, g * scale, scale, **amp)
    assert _same(want, got[:3] + [want[3]] + got[4:]), name         # the gradient buffers differ: scaled or zeroed
    assert torch.equal(got[3], torch.zeros_like(got[3]))


@pytest.mark.parametrize("name", NAMES)
def test_scaled_instance_equals_torch_unscale(name):
    """S = 1000 is not a power of two: the update must see exactly torch's g * fp32(1 / double(S)), subnormals included."""
    G = state(2)[3].to(DEV) * 1000.0
    amp = {"found_inf": 0.0} if name.startswith("cap") else {}
    want = run(name, unscaled(G, 1000.0), None, **({} if not amp else {"found_inf": None}))
    got = run(name, G, 1000.0, **amp)
    assert _same(want[:3] + want[4:], got[:3] + got[4:]), name


@pytest.mark.parametrize("name", ["cap_sgd", "cap_adamw"])
@pytest.mark.parametrize("zero_grad", [True, False])
def test_capturable_instance_skips_on_found_inf(name, zero_grad):
    p, m, v, g = (t.to(DEV) for t in state(3))
    got = run(name, g * 8.0, 8.0, found_inf=1.0, seed=3, zero_grad=zero_grad)
    assert torch.equal(got[0], p) and torch.equal(got[1], m) and torch.equal(got[2], v)
    assert torch.equal(got[3], torch.zeros_like(g) if zero_grad else g * 8.0)
    assert bool((got[4] == SENT).all()), "a skipped step wrote grad_norm_out"


def test_unscaling_keeps_subnormal_inputs():
    """A scale below 1 turns subnormal scaled gradients into normal ones: torch's unscale keeps the subnormal input, as
    the kernels' non-ftz ``mul.rn.f32`` does (the ``.ftz`` form would give 0).  With zero momentum, no weight decay and
    mu = 0.5, SGD stores ``m = g`` exactly, so the unscaled gradient is visible in every element."""
    C = kern()
    S = 2.0 ** -24
    G = state(4)[3].to(DEV) * 1e-36                          # every element subnormal or tiny
    G[::2] = torch.arange(1, G[::2].numel() + 1, device=DEV, dtype=torch.float32) * 1.4e-45     # exact subnormals
    want = unscaled(G, S)
    assert bool((G[::2].abs() < 1.1754944e-38).all()) and bool((want[::2].abs() >= 1.1754944e-38).all())
    for grouped in (False, True):
        p, m = torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)
        g = G.clone()
        if grouped:
            gmap = torch.zeros((N + 3) // 4, dtype=torch.uint8, device=DEV)
            C.sgd_flat_grouped(p, m, g, gmap, [0.0], [0.0], 0.5, False, False, grad_scale=scalar(S))
        else:
            C.sgd_flat(p, m, g, 0.0, 0.5, 0.0, False, False, grad_scale=scalar(S))
        torch.cuda.synchronize()
        nz = want != 0                                       # fmaf(0, 0, -0) is +0: zeros compare by value
        assert torch.equal(m[nz].view(torch.int32), want[nz].view(torch.int32)) and bool((m[~nz] == 0).all()), grouped


def test_gated_advance_leaves_counter_and_block():
    C = kern()
    lay = C.flat_scalars_layout()
    table = torch.zeros(lay["table_bytes"], dtype=torch.uint8, device=DEV)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    block = torch.zeros(lay["block_bytes"], dtype=torch.uint8, device=DEV)
    C.flat_scalars_sync(table, counter, block, [0.05], [0.01], 0.9, 0.999, 1e-8, None, 5)
    before = (counter.clone(), block.clone())
    C.flat_scalars_advance(table, counter, block, found_inf=scalar(float("nan")))
    C.flat_scalars_advance(table, counter, block, found_inf=scalar(1.0))
    assert torch.equal(counter, before[0]) and torch.equal(block, before[1])
    C.flat_scalars_advance(table, counter, block, found_inf=scalar(0.0))
    gated = (counter.clone(), block.clone())
    counter.copy_(before[0]); block.copy_(before[1])
    C.flat_scalars_advance(table, counter, block)
    assert int(counter) == 6 and torch.equal(counter, gated[0]) and torch.equal(block, gated[1])


def test_binding_refusals():
    C = kern()
    p = torch.zeros(8, device=DEV)
    for bad in (torch.ones(2, device=DEV), torch.ones(1, dtype=torch.float64, device=DEV), torch.ones(1)):
        with pytest.raises(RuntimeError, match="grad_scale"):
            C.sgd_flat(p, p.clone(), p.clone(), 0.1, 0.9, 0.0, True, grad_scale=bad)


# ---------------------------------------------------------------------------------------------------- ResNet-18 under DDP
OPTS = {"sgd": lambda d, **kw: FlatSGD(d, lr=0.05, momentum=0.9, weight_decay=1e-4, max_grad_norm=5.0, **kw),
        "adamw": lambda d, **kw: FlatAdamW(d, lr=1e-3, weight_decay=0.01, max_grad_norm=5.0, **kw),
        "sgd_noclip": lambda d, **kw: FlatSGD(d, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, **kw),
        "adamw_noclip": lambda d, **kw: FlatAdamW(d, lr=1e-3, weight_decay=0.01, **kw),
        "lamb": lambda d, **kw: FlatLAMB(d, lr=1e-3, weight_decay=0.01, **kw),
        "lars": lambda d, **kw: FlatLARS(d, lr=0.5, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-2, **kw)}


def data(n, seed=11):
    gen = torch.Generator().manual_seed(seed)
    return [(torch.randn(8, 3, 64, 64, generator=gen).to(DEV).contiguous(memory_format=torch.channels_last),
             torch.randint(0, 100, (8,), generator=gen).to(DEV)) for _ in range(n)]


def resnet_run(kind, explicit, steps=8):
    torch.manual_seed(5)
    m = ResNet18(num_classes=100).to(DEV).to(memory_format=torch.channels_last)
    ddp = DistributedDataParallel(m)
    opt = OPTS[kind](ddp)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 24, growth_interval=2)
    scales = []
    for x, y in data(steps):
        with torch.autocast("cuda", dtype=torch.float16):
            loss = F.cross_entropy(ddp(x), y)
        scaler.scale(loss).backward()
        b2.average_gradients(ddp)
        if explicit:
            scaler.unscale_(opt)
        scaler.step(opt)
        scaler.update()
        scales.append(scaler.get_scale())
    ddp.remove_hooks()
    return [t.detach().clone() for t in m.parameters()], opt.steps, scales


@pytest.mark.parametrize("kind", list(OPTS))
def test_resnet18_scaler_step_equals_explicit_unscale(kind):
    a, b = resnet_run(kind, False), resnet_run(kind, True)
    assert a[1] == b[1] and a[2] == b[2]
    assert a[1] < 8 and a[2][0] < 2.0 ** 24, "the early overflows of a large init_scale were not skipped"
    assert all(torch.equal(x, y) for x, y in zip(a[0], b[0])), kind


def graphed_amp(kind, graph, n=8, warmup=3, overflow_at=5):
    """Capturable optimizer + GradScaler + FlatEMA: warm-up steps on a side stream, then ``n`` eager steps or replays of
    one captured step; before step ``overflow_at`` the scale is set to 2^30 so that step overflows."""
    torch.manual_seed(5)
    m = ResNet18(num_classes=100).to(DEV).to(memory_format=torch.channels_last)
    ddp = DistributedDataParallel(m)
    opt = OPTS[kind](ddp, capturable=True)
    ema = FlatEMA(opt, decay=0.9)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    batches = data(warmup + n)
    x, y = batches[0][0].clone(), batches[0][1].clone()

    def step():
        with torch.autocast("cuda", dtype=torch.float16):
            loss = F.cross_entropy(ddp(x), y)
        scaler.scale(loss).backward()
        b2.average_gradients(ddp)
        scaler.step(opt)
        scaler.update()
        ema.update()

    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        for i in range(warmup):
            x.copy_(batches[i][0]); y.copy_(batches[i][1])
            step()
    torch.cuda.current_stream(DEV).wait_stream(s)
    g = None
    if graph:
        g = torch.cuda.CUDAGraph()
        torch.cuda.set_sync_debug_mode("error")
        try:
            with torch.cuda.graph(g):
                step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    trace = []
    for i in range(warmup, warmup + n):
        x.copy_(batches[i][0]); y.copy_(batches[i][1])
        if i == warmup + overflow_at:
            scaler._scale.fill_(2.0 ** 30)
            before = ([t.clone() for t in m.parameters()], int(opt._cap_counter))
        if graph:
            torch.cuda.set_sync_debug_mode("error")
            g.replay()
            torch.cuda.set_sync_debug_mode(0)
        else:
            step()
        if i == warmup + overflow_at:
            assert all(torch.equal(a, b) for a, b in zip(before[0], m.parameters())) and int(opt._cap_counter) == before[1]
            assert float(scaler._scale) == 2.0 ** 29
        trace.append((float(scaler._scale), int(opt._cap_counter)))
    torch.cuda.synchronize()
    ddp.remove_hooks()
    return [t.detach().clone() for t in m.state_dict().values()], [e.clone() for e in ema.ema_flats], trace


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_captured_scaled_step_replays_equal_eager_steps(kind):
    eager, graph = graphed_amp(kind, False), graphed_amp(kind, True)
    assert eager[2] == graph[2]
    for a, b in zip(eager[0] + eager[1], graph[0] + graph[1]):
        assert torch.equal(a, b), kind
