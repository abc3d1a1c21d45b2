"""``FlatEMA`` on one H100: the ``ema_update`` kernel alone against torch's CUDA ``_foreach_lerp_`` bit for bit (both
weight branches, subnormals, signed zeros, large values, short and unaligned entries, sentinels after every entry, copy mode,
the device-counter instance up to t >= 2^32), emulated sharded slices against the whole flat, ResNet-18 training against
``AveragedModel`` on CUDA, a captured step + update() against eager steps, no host synchronisation, and one launch per
update.  Workers in tests/ema_workers.py."""
import pytest
import torch

import capturable_workers as CW
import dist_tuto.pth_b200 as b2
import ema_workers as W
from dist_tuto.pth_b200.ops import _ext

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = torch.device("cuda", 0)
SENTINEL = 12345.678
DECAYS = (0.9999, 0.9, 0.5, 0.3, 1e-4, 0.0, 1.0)
TINY = 1.1754942e-38                        # the largest fp32 subnormal


def values(n, g):
    """fp32 values of five kinds: normal, subnormal, signed zero, large (positive, so that no difference overflows), one."""
    kind = torch.randint(0, 5, (n,), generator=g)
    normal = torch.randn(n, generator=g)
    sub = (torch.rand(n, generator=g) * 2 - 1) * TINY
    zero = torch.where(torch.rand(n, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))
    big = 1e37 + torch.rand(n, generator=g) * 3e38
    out = torch.where(kind == 0, normal, torch.where(kind == 1, sub, torch.where(kind == 2, zero,
                                                                                 torch.where(kind == 3, big, normal + 1))))
    return out.to(torch.float32)


def carve(lengths, seed, same_alignment):
    """Two sentinel-filled pools and the (ema, live) views of ``lengths`` in them, each followed by sentinels.  With
    ``same_alignment`` the two views of an entry start at the same element offset (the vector path with a head); otherwise
    at offsets that differ mod 4 for most entries (the scalar path)."""
    g = torch.Generator().manual_seed(seed)
    total = sum(lengths) + 12 * len(lengths) + 16
    pools = [torch.full((total,), SENTINEL, device=DEV) for _ in range(2)]
    views = []
    oe = int(torch.randint(0, 4, (1,), generator=g))
    op = oe if same_alignment else oe + 1 + int(torch.randint(0, 3, (1,), generator=g))
    for n in lengths:
        e, p = pools[0][oe:oe + n], pools[1][op:op + n]
        e.copy_(values(n, g))
        p.copy_(values(n, g))
        views.append((e, p))
        step = n + 5 + int(torch.randint(0, 4, (1,), generator=g))
        oe += step
        op += step if same_alignment else n + 5 + int(torch.randint(0, 4, (1,), generator=g))
    return pools, views


def bits(t):
    return t.view(torch.int32)


def run_kernel(views, **kw):
    C = _ext.C()
    table = C.ema_table([e for e, _ in views], [p for _, p in views])
    C.ema_update(*table, **kw)


LENGTHS = {"short": [n for n in range(1, 10) for _ in range(2)],
           "tails": [4 * k + r for k in (1, 7, 64, 1000) for r in range(4)] + [65537],
           "many": [int(x) for x in torch.randint(1, 200, (300,), generator=torch.Generator().manual_seed(3))],
           "one": [(1 << 20) + 3]}


@pytest.mark.parametrize("lengths", list(LENGTHS), ids=list(LENGTHS))
@pytest.mark.parametrize("same_alignment", [True, False], ids=["aligned-alike", "misaligned"])
def test_kernel_equals_torch_foreach_lerp(lengths, same_alignment):
    for i, decay in enumerate(DECAYS):
        (ep, pp), views = carve(LENGTHS[lengths], 17 + i, same_alignment)
        ref = ep.clone()
        ref_views = [ref[e.storage_offset():e.storage_offset() + e.numel()] for e, _ in views]
        torch._foreach_lerp_(ref_views, [p for _, p in views], 1 - decay)
        live = pp.clone()
        run_kernel(views, w=1 - decay)
        torch.cuda.synchronize()
        assert torch.equal(bits(ep), bits(ref)), (lengths, decay, int((bits(ep) != bits(ref)).sum()))
        assert torch.equal(bits(pp), bits(live)), "the live values changed"


def test_copy_mode_copies_every_bit():
    (ep, pp), views = carve(LENGTHS["tails"] + LENGTHS["short"], 5, False)
    ref = ep.clone()
    for e, p in views:
        ref[e.storage_offset():e.storage_offset() + e.numel()].copy_(p)
    run_kernel(views, w=0.1, copy=True)
    torch.cuda.synchronize()
    assert torch.equal(bits(ep), bits(ref))


def test_device_counter_instance_decides_skip_copy_lerp():
    every, warmup = 3, 4
    (ep0, pp), views = carve(LENGTHS["tails"], 9, True)
    C = _ext.C()
    ts = list(range(0, 16)) + [(1 << 32) + d for d in range(-4, 5)] + [(1 << 40) + d for d in range(3)]
    for t in ts:
        ep = ep0.clone()
        mine = [(ep[e.storage_offset():e.storage_offset() + e.numel()], p) for e, p in views]
        expect = ep0.clone()
        ev = [expect[e.storage_offset():e.storage_offset() + e.numel()] for e, _ in views]
        if t % every == 0:
            if t - every <= warmup:
                torch._foreach_copy_(ev, [p for _, p in views])
            else:
                torch._foreach_lerp_(ev, [p for _, p in views], 1 - 0.9)
        table = C.ema_table([e for e, _ in mine], [p for _, p in mine])
        counter = torch.tensor([t], dtype=torch.int64, device=DEV)
        C.ema_update(*table, w=1 - 0.9, counter=counter, every=every, warmup_steps=warmup)
        torch.cuda.synchronize()
        assert torch.equal(bits(ep), bits(expect)), t
        assert int(counter) == t


@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_slices_equal_the_whole_flat(world):
    """The owned slices of W emulated ranks (the padded flat cut as the sharded optimizer cuts it) with the buffers, one
    launch per rank, equal one launch over the whole flat."""
    g = torch.Generator().manual_seed(world)
    numel = 123457
    n_vec = ((numel * 4 + 15) // 16 + world - 1) // world * world
    n_pad, per = n_vec * 4, n_vec * 4 // world
    live = values(n_pad, g).to(DEV)
    ema0 = values(n_pad, g).to(DEV)
    bufs = [values(n, g).to(DEV) for n in (64, 3, 257)]
    ebufs = [values(b.numel(), g).to(DEV) for b in bufs]
    for decay in (0.999, 0.25):
        whole = ema0.clone()
        wb = [e.clone() for e in ebufs]
        run_kernel([(whole, live)] + list(zip(wb, bufs)), w=1 - decay)
        shards = []
        for r in range(world):
            shard = ema0[r * per:(r + 1) * per].clone()
            rb = [e.clone() for e in ebufs]
            run_kernel([(shard, live[r * per:(r + 1) * per])] + list(zip(rb, bufs)), w=1 - decay)
            shards.append(shard)
            assert all(torch.equal(bits(a), bits(b)) for a, b in zip(rb, wb))
        torch.cuda.synchronize()
        assert torch.equal(bits(torch.cat(shards)), bits(whole)), (world, decay)


def test_binding_refusals():
    C = _ext.C()
    a = torch.zeros(8, device=DEV)
    for emas, lives in [([], []), ([a], []), ([a.cpu()], [a.cpu()]), ([a.double()], [a.double()]), ([a], [a[:4]]),
                        ([a[:0]], [a[:0]])]:
        with pytest.raises(RuntimeError, match="ema_table"):
            C.ema_table(emas, lives)
    table = C.ema_table([a], [torch.ones(8, device=DEV)])
    with pytest.raises(RuntimeError, match="every"):
        C.ema_update(*table, w=0.1, counter=torch.zeros(1, dtype=torch.int64, device=DEV), every=0)
    with pytest.raises(RuntimeError, match="counter"):
        C.ema_update(*table, w=0.1, counter=torch.zeros(1, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="table"):
        C.ema_update(table[0].cpu(), table[1], w=0.1)
    torch.cuda.synchronize()
    assert torch.equal(a, torch.zeros(8, device=DEV)), "a refused call launched"


def test_cuda_buffers_must_be_fp32():
    m = torch.nn.Sequential(torch.nn.Linear(4, 4)).to(DEV)
    m.register_buffer("h16", torch.zeros(3, dtype=torch.float16, device=DEV))
    ddp = b2.DistributedDataParallel(m)
    opt = b2.FlatSGD(ddp, lr=0.1)
    with pytest.raises(ValueError, match="fp32"):
        b2.FlatEMA(opt)
    ddp.remove_hooks()


def test_resnet18_training_equals_averaged_model():
    b2.launch(W.w_gpu_training, size=1, backend="b200", join_timeout_s=800)


@pytest.mark.parametrize("name,make", CW.optimizers(), ids=[n for n, _ in CW.optimizers()])
def test_captured_step_and_update_replays_equal_eager_steps(name, make):
    eager = W.graphed_ema(make, 12, False, DEV)
    graph = W.graphed_ema(make, 12, True, DEV)
    assert eager[2] == graph[2] == 15
    for a, b in zip(eager[0] + eager[1], graph[0] + graph[1]):
        assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)), name


def _small(capturable):
    torch.manual_seed(7)
    m = CW.net().to(DEV).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(m)
    opt = b2.FlatSGD(ddp, lr=0.05, momentum=0.9, capturable=capturable)
    return m, ddp, opt


def _step(ddp, opt, i):
    g = torch.Generator(device=DEV).manual_seed(i)
    x = torch.randn(8, 3, 12, 12, generator=g, device=DEV).contiguous(memory_format=torch.channels_last)
    torch.nn.functional.cross_entropy(ddp(x), torch.randint(0, 10, (8,), generator=g, device=DEV)).backward()
    b2.average_gradients(ddp)
    opt.step()


@pytest.mark.parametrize("capturable", [False, True])
def test_update_does_not_synchronise(capturable):
    m, ddp, opt = _small(capturable)
    ema = b2.FlatEMA(opt, decay=0.99, every=2, warmup_steps=1)
    for i in range(1, 7):
        _step(ddp, opt, i)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ema.update()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    ddp.remove_hooks()


@pytest.mark.parametrize("capturable", [False, True])
def test_one_launch_per_update(capturable):
    """torch.profiler counts the EMA kernels of each update: one per update that is not skipped (every update with a
    capturable optimizer, whose kernel decides on the device).  A warm-up update loads the kernel and a throwaway profiler
    session starts the profiler before anything is counted."""
    from torch.profiler import ProfilerActivity, profile

    m, ddp, opt = _small(capturable)
    ema = b2.FlatEMA(opt, decay=0.99, every=2, warmup_steps=1)
    ema.update()                          # t = 0: a copy of the values just copied, so the kernel is loaded
    with profile(activities=[ProfilerActivity.CUDA]):
        torch.ones(1, device=DEV).add_(1)
        torch.cuda.synchronize()
    for i in range(1, 7):
        _step(ddp, opt, i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            # once another process has used the GPU, a session loses kernel records at its start, and the profiler keeps
            # only the device activity inside its window: ~10 ms sleep kernels keep the update well inside it
            torch.cuda._sleep(20_000_000)
            torch.cuda.synchronize()
            ema.update()
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)
            torch.cuda.synchronize()
        kernels = [(e.key, e.count) for e in prof.key_averages()]
        n = sum(c for k, c in kernels if "ema_kernel" in k)
        assert n == (1 if capturable or i % 2 == 0 else 0), (capturable, i, kernels)
    ddp.remove_hooks()


def test_update_in_a_capture_needs_a_capturable_optimizer():
    m, ddp, opt = _small(False)
    ema = b2.FlatEMA(opt)
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match="capturable"):
            with torch.cuda.graph(g, stream=s):
                ema.update()
    m2, ddp2, opt2 = _small(True)
    ema2 = b2.FlatEMA(opt2)
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="capture"):
        with torch.cuda.graph(g2):
            with ema2.average_parameters():
                pass
    torch.cuda.synchronize()
    ddp.remove_hooks()
    ddp2.remove_hooks()
