"""FlatLAMB's and FlatLARS's kernels (csrc/layerwise.cu) on one GPU: ``lamb_flat`` and ``lars_flat`` bit for bit against the
model of tests/layerwise_model.py over many layouts, with sentinels behind every flat, state and workspace; the tickets
zero after every call; two runs bit-identical; the error against fp64 within the model's bound; and a ResNet-18 trained
through ``DistributedDataParallel`` + ``FlatLAMB`` / ``FlatLARS`` under bf16 autocast."""
import math
import random

import pytest
import torch

import layerwise_cases as TM
import layerwise_model as L
from emulated_ranks import C, _bits, _untouched, _with_sentinel  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

LAMB_HP = dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1)
LARS_HP = dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4, nesterov=False)
C_ = L.CHUNK
random.seed(5)
LAYOUTS = {f"single_{k}": [k] for k in (1, 2, 3, 4, 5, 1023, C_ - 1, C_, C_ + 1, 2 * C_ - 1, 2 * C_ + 1, (1 << 20) + 3)}
LAYOUTS["chunk_multiples"] = [C_ - 1, C_ + 1, 2 * C_ - 1, 5, 2 * C_, 3 * C_ + 1, 7]
LAYOUTS["tiny_3000"] = [random.randint(1, 9) for _ in range(3000)]
LAYOUTS["mixed"] = [300, 1, 17, 70001, 64, 4097, 2, 130]
SENT64, SENT_I32 = 12345.678, 0x5EADBEEF


def _layout(numels):
    offsets, n = [], 0
    for k in numels:
        offsets.append(n)
        n += (k + 3) // 4 * 4
    return offsets, n


def _state(numels, seed, zero_p=None, zero_g=None):
    """Bucket flats with the tensors at their offsets and zeros in the alignment gaps, as FlatLAMB lays them out."""
    offsets, n = _layout(numels)
    gen = torch.Generator().manual_seed(seed)
    p, g, m, v = (torch.zeros(n) for _ in range(4))
    for i, (o, k) in enumerate(zip(offsets, numels)):
        s = slice(o, o + k)
        scale = 2.0 ** (i % 5 - 2)
        p[s] = torch.randn(k, generator=gen) * scale
        g[s] = torch.randn(k, generator=gen) * 0.1
        m[s] = torch.randn(k, generator=gen) * 0.01
        v[s] = torch.rand(k, generator=gen) * 1e-3
    if zero_p is not None:
        p[offsets[zero_p]:offsets[zero_p] + numels[zero_p]] = 0
    if zero_g is not None:
        g[offsets[zero_g]:offsets[zero_g] + numels[zero_g]] = 0
    return offsets, n, p, g, m, v


class Work:
    """The workspaces of one bucket, each followed by sentinels."""

    def __init__(self, C, offsets, numels, adapt, n):
        self.table, self.n_chunks = C.layerwise_table(offsets, numels, adapt, n, torch.device("cuda"))
        nt = len(numels)
        self.partials = _with_sentinel(torch.zeros(2 * self.n_chunks))
        self.tickets = torch.cat([torch.zeros(nt, dtype=torch.int32), torch.full((4,), SENT_I32, dtype=torch.int32)]).cuda()
        self.sums = torch.cat([torch.zeros(2 * nt, dtype=torch.float64), torch.full((4,), SENT64, dtype=torch.float64)]).cuda()
        self.ratios = _with_sentinel(torch.ones(nt))
        self.nc, self.nt = self.n_chunks, nt

    def args(self):
        return (self.table, self.nc, self.partials[:2 * self.nc], self.tickets[:self.nt], self.sums[:2 * self.nt],
                self.ratios[:self.nt])

    def check(self, what):
        assert not self.tickets[:self.nt].any(), f"{what}: a ticket was left nonzero"
        assert bool((self.tickets[self.nt:] == SENT_I32).all()) and bool((self.sums[2 * self.nt:] == SENT64).all()), \
            f"{what}: a sentinel behind the tickets or the sums changed"
        assert _untouched(self.partials[2 * self.nc:]) and _untouched(self.ratios[self.nt:]), \
            f"{what}: a sentinel behind the partials or the ratios changed"


def run_lamb(C, numels, adapt, seed, hp=LAMB_HP, steps=2, clip=None, zero_p=None, zero_g=None):
    offsets, n, p, g, m, v = _state(numels, seed, zero_p, zero_g)
    bufs = [_with_sentinel(x) for x in (p, g, m, v)]
    dp, dg, dm, dv = bufs
    w = Work(C, offsets, numels, adapt, n)
    want = (p, m, v)
    for t in range(1, steps + 1):
        kw, coef = {}, None
        if clip is not None:
            sq = torch.zeros(2, dtype=torch.float64, device="cuda")
            ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
            C.grad_sqnorm(dg[:n], sq, 0, ws)
            C.grad_sqnorm(torch.full((4096,), 0.05, device="cuda"), sq, 1, ws)
            coef = L.clip_coef(sq.cpu().tolist(), clip)
            assert coef < 1.0
            kw = dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=torch.zeros(1, device="cuda"))
        C.lamb_flat(dp[:n], dm[:n], dv[:n], dg[:n], *w.args(), TM_scalars(hp, t), t == steps, **kw)
        wp, wm, wv, wr = L.lamb_step(want[0], g, want[1], want[2], offsets, numels, adapt, hp, t, coef=coef)
        what = f"lamb {len(numels)} tensors t {t}"
        for name, got, x in zip("pmv", (dp, dm, dv), (wp, wm, wv)):
            assert _bits(got[:n], x), f"{what}: {name}"
        assert _bits(w.ratios[:w.nt], torch.tensor(wr)), f"{what}: ratios"
        assert all(_untouched(b[n:]) for b in bufs), f"{what}: a sentinel behind a flat changed"
        w.check(what)
        assert _bits(dg[:n], torch.zeros(n) if t == steps else g), f"{what}: gradients"
        want = (wp, wm, wv)
    return dp[:n].clone(), wr


def TM_scalars(hp, t):                                    # noqa: N802
    from dist_tuto.pth_b200.ops.optim import lamb_scalars
    return lamb_scalars(hp["lr"], hp["betas"], hp["eps"], hp["weight_decay"], t)


def run_lars(C, numels, adapt, seed, hp=LARS_HP, steps=2, clip=None, zero_p=None, zero_g=None):
    offsets, n, p, g, m, _ = _state(numels, seed, zero_p, zero_g)
    bufs = [_with_sentinel(x) for x in (p, g, m)]
    dp, dg, dm = bufs
    w = Work(C, offsets, numels, adapt, n)
    want = (p, m)
    for t in range(1, steps + 1):
        kw, coef = {}, None
        if clip is not None:
            sq = torch.zeros(1, dtype=torch.float64, device="cuda")
            ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
            C.grad_sqnorm(dg[:n], sq, 0, ws)
            coef = L.clip_coef(sq.cpu().tolist(), clip)
            assert coef < 1.0
            norm = torch.zeros(1, device="cuda")
            kw = dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=norm)
        C.lars_flat(dp[:n], dm[:n], dg[:n], *w.args(), hp["lr"], hp["momentum"], hp["weight_decay"], hp["trust_coefficient"],
                    hp["eps"], hp["nesterov"], t == steps, **kw)
        wp, wm, wr = L.lars_step(want[0], g, want[1], offsets, numels, adapt, hp, coef=coef)
        what = f"lars {len(numels)} tensors t {t}"
        assert _bits(dp[:n], wp) and _bits(dm[:n], wm), f"{what}: p / momentum"
        assert _bits(w.ratios[:w.nt], torch.tensor(wr)), f"{what}: ratios"
        assert all(_untouched(b[n:]) for b in bufs), f"{what}: a sentinel behind a flat changed"
        w.check(what)
        assert _bits(dg[:n], torch.zeros(n) if t == steps else g), f"{what}: gradients"
        if clip is not None:
            assert float(norm) == L.f32(math.sqrt(sum(sq.cpu().tolist())))
        want = (wp, wm)
    return dp[:n].clone(), wr


def test_chunk_size_is_the_models(C):
    assert C.layerwise_chunk_elems() == L.CHUNK


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_lamb_matches_the_model_bit_for_bit(C, name):
    numels = LAYOUTS[name]
    adapt = [i % 3 != 1 for i in range(len(numels))]            # every third tensor excluded
    run_lamb(C, numels, adapt, seed=len(numels))


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_lars_matches_the_model_bit_for_bit(C, name):
    numels = LAYOUTS[name]
    adapt = [i % 3 != 1 for i in range(len(numels))]
    run_lars(C, numels, adapt, seed=len(numels))
    run_lars(C, numels, adapt, seed=len(numels) + 1, hp=dict(LARS_HP, nesterov=True, weight_decay=0.0), steps=1)


def test_zero_tensor_and_zero_gradient_give_ratio_one(C):
    numels, adapt = [1000, 1001, 20000], [True, True, True]
    _, r = run_lars(C, numels, adapt, seed=1, zero_p=0, zero_g=1, steps=1)
    assert r[0] == 1.0 and r[1] == 1.0 and r[2] != 1.0
    _, r = run_lamb(C, numels, adapt, seed=1, hp=dict(LAMB_HP, weight_decay=0.0), zero_p=0, zero_g=1, steps=1)
    assert r[0] == 1.0 and r[2] != 1.0


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_clip_instance_with_a_coefficient_below_one(C, kind):
    numels = LAYOUTS["mixed"]
    adapt = [k > 64 for k in numels]
    (run_lamb if kind == "lamb" else run_lars)(C, numels, adapt, seed=3, clip=0.5)


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_two_runs_are_bit_identical(C, kind):
    numels = LAYOUTS["chunk_multiples"] + LAYOUTS["tiny_3000"][:500]
    adapt = [True] * len(numels)
    run = run_lamb if kind == "lamb" else run_lars
    a, ra = run(C, numels, adapt, seed=9, steps=1)
    b, rb = run(C, numels, adapt, seed=9, steps=1)
    assert _bits(a, b) and ra == rb


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_kernel_error_against_fp64_is_within_the_bound(C, kind):
    """50 updates of the model's layout through the kernel: within 4x the fp32 torch-op path's error of fp64, plus one ulp."""
    hp = TM._hp(kind, 0)
    offsets, numels, p0, grads = TM.inputs(21)
    n = p0.numel()
    ref, b = TM.bound(kind, hp, 21)
    w = Work(C, offsets, numels, TM.ADAPT, n)
    dp, dm, dv = p0.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for t, g in enumerate(grads, 1):
        dg = g.cuda()
        if kind == "lamb":
            C.lamb_flat(dp, dm, dv, dg, *w.args(), TM_scalars(hp, t), True)
        else:
            C.lars_flat(dp, dm, dg, *w.args(), hp["lr"], hp["momentum"], hp["weight_decay"], hp["trust_coefficient"],
                        hp["eps"], hp["nesterov"], True)
    err = float((dp.cpu().double() - ref).abs().max())
    assert err <= b, (err, b)


def test_refusals(C):
    offsets, n = _layout([10, 20])
    with pytest.raises(RuntimeError, match="multiple of 4"):
        C.layerwise_table([0, 11], [10, 20], [True, True], n, torch.device("cuda"))
    with pytest.raises(RuntimeError, match="inside the flat"):
        C.layerwise_table(offsets, [10, 20], [True, True], 20, torch.device("cuda"))
    w = Work(C, offsets, [10, 20], [True, True], n)
    p, g, m, v = (torch.zeros(n, device="cuda") for _ in range(4))
    with pytest.raises(RuntimeError, match="one size"):
        C.lamb_flat(p, m, v[:n - 4], g, *w.args(), TM_scalars(LAMB_HP, 1), True)
    with pytest.raises(RuntimeError, match="table"):
        C.lars_flat(p, m, g, w.table[:-3], w.nc, *w.args()[2:], 0.1, 0.9, 0.0, 1e-3, 1e-8, False, True)
    with pytest.raises(RuntimeError, match="scalars"):
        C.lamb_flat(p, m, v, g, *w.args(), TM_scalars(LAMB_HP, 1)[:7], True)
    with pytest.raises(RuntimeError, match="trust_coefficient"):
        C.lars_flat(p, m, g, *w.args(), 0.1, 0.9, 0.0, 0.0, 1e-8, False, True)


# ----------------------------------------------------------------------------------------------- module level
def test_ddp_resnet18_trains_with_lamb_and_lars_under_bf16_autocast():
    import dist_tuto.pth_b200 as b2
    import layerwise_workers as WK
    b2.launch(WK.w_resnet, size=1, backend="b200", join_timeout_s=600)
