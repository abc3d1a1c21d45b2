"""GPU-single tier: the one-GPU optimizer kernel reduce_sgd (csrc/sgd.cu, csrc/convnet_reduce.cuh) and det_reduce, bit
for bit against the rounding-exact model of tests/reduce_sgd_model.py.

* Every grid of ``R.grids()`` (``n_cta``: one CTA running all 124 units down to one unit per CTA) at every size of
  ``R.sizes(S)``: the local gradient, taken as the momentum of a plain launch with mu = 0 and lr = 0, equals the model at
  every grid and lies within the fp64 bound; small-integer data gives the exact sums; the clip instance's norm has the
  model's bits for that grid, and its update the model's.
* Every instance (plain, weight decay, Nesterov, both, each with a warmup-cosine schedule, and the clip instance clipping or
  not, with and without weight decay and Nesterov) with the step counter absent, at 4, 5 and 2^32 - 1, one or two gradient
  buckets or none: params, momentum, aux, loss_acc, grad_norm_out, the step counter and done_counter, with NaN or sentinel
  guard bands around everything that must not be written and NaN in everything that must not be read.
* FusedTrainer at batch 128 and 4S + 1 (slots carrying two samples): every step's update is the model of its launch.
* det_reduce at 1, 2, 31, 32, 33 and S slots, both parities, one or two buckets, with and without loss_acc.
"""
import pytest
import torch

import reduce_sgd_model as R
from engine_paths import _batches

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

NPAR, NPAR_ALLOC, DET, FAC = R.NPAR, 21888, R.DET_STRIDE, R.FAC_STRIDE
S = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
SIZES = R.sizes(S)
GRIDS = R.grids()
NAN = float("nan")
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def C():
    from dist_tuto.pth_b200.ops import _ext
    return _ext.C()


def _bits(t):
    return t.detach().cpu().float().contiguous().view(torch.int32)


def assert_bits(what, got, want, zeros_by_value=False):
    g, w = _bits(got), _bits(want)
    bad = g != w
    if zeros_by_value:                                     # fmaf(0, m, g) may turn a -0 into +0
        bad &= ~((got.detach().cpu().float() == 0) & (want.float() == 0))
    if bool(bad.any()):
        i = int(bad.nonzero()[0, 0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, first at {i}: got "
                             f"{float(got.reshape(-1)[i])} (0x{int(g[i]) & 0xffffffff:08x}), model {float(want[i])} "
                             f"(0x{int(w[i]) & 0xffffffff:08x})")


def _inputs(n_samples, n_slots, seed, ints=False):
    """Slots and factor rows, one slot and one row more than used, NaN wherever the kernel must not read: each slot's
    fc1.weight range and the words past its loss terms, the extra slot, factor columns [50, FAC_P2) and the extra row."""
    g = torch.Generator().manual_seed(seed)
    if ints:
        slots = torch.randint(-4, 5, (n_slots + 1, DET), generator=g).float()
        fac = torch.randint(-3, 4, (n_samples + 1, FAC), generator=g).float()
    else:
        slots, fac = torch.randn(n_slots + 1, DET, generator=g), torch.randn(n_samples + 1, FAC, generator=g)
    slots[:, R.W3:R.W3 + R.FC1] = NAN
    slots[:, NPAR + 2:] = NAN
    slots[n_slots:] = NAN
    fac[:, 50:R.FAC_P2] = NAN
    fac[n_samples:] = NAN
    return slots, fac


class Case:
    """One (samples, slots) size: random and small-integer inputs on the device and the model of their gradient."""

    def __init__(self, n_samples, n_slots):
        self.n_samples, self.n_slots = n_samples, n_slots
        seed = n_samples * 1009 + n_slots
        self.slots, self.fac = _inputs(n_samples, n_slots, seed)
        self.g = R.local_grad(self.slots, n_slots, self.fac, n_samples)
        self.loss = R.loss_terms(self.slots, n_slots)
        self.ref, self.bound, _, _ = R.fp64_bound(self.slots, n_slots, self.fac, n_samples)
        islots, ifac = _inputs(n_samples, n_slots, seed + 1, ints=True)
        self.int_exact = R.fp64_bound(islots, n_slots, ifac, n_samples)[0].float()
        self.d = {k: v.cuda() for k, v in dict(slots=self.slots, fac=self.fac, islots=islots, ifac=ifac).items()}


_CASES = {}


def case(n_samples, n_slots):
    key = (n_samples, n_slots)
    if key not in _CASES:
        _CASES[key] = Case(n_samples, n_slots)
    return _CASES[key]


def _flat(seed, n=NPAR_ALLOC):
    """Random params / momentum with NaN past NPAR (never written)."""
    t = torch.randn(n, generator=torch.Generator().manual_seed(seed))
    t[NPAR:] = NAN
    return t


# ---------------------------------------------------------------------------------------------------------- every grid
@pytest.mark.parametrize("n_samples,n_slots", SIZES, ids=[f"{a}x{b}" for a, b in SIZES])
def test_every_grid_reduces_in_the_model_order(C, n_samples, n_slots):
    c = case(n_samples, n_slots)
    d = c.d
    params = torch.randn(NPAR_ALLOC, generator=torch.Generator().manual_seed(1)).cuda()
    p0, m0 = _flat(2), _flat(3)
    ws = torch.zeros(C.clip_workspace_numel(NPAR_ALLOC), device="cuda")
    norm = torch.zeros(1, device="cuda")
    big = 1e30                                             # max_norm that never clips: coefficient 1
    for n_cta in GRIDS:
        m = torch.zeros(NPAR_ALLOC, device="cuda")
        C.reduce_sgd(d["slots"], n_slots, d["fac"], n_samples, params.clone(), m, None, None, 0.0, 0.0, n_cta=n_cta)
        assert_bits(f"gradient at grid {n_cta}", m[:NPAR], c.g, zeros_by_value=True)
        if n_cta == GRIDS[0]:
            err = (m[:NPAR].cpu().double() - c.ref).abs()
            assert bool((err <= c.bound).all()), f"kernel outside the fp64 bound: {float((err / c.bound).max())}"
        mi = torch.zeros(NPAR_ALLOC, device="cuda")
        C.reduce_sgd(d["islots"], n_slots, d["ifac"], n_samples, params.clone(), mi, None, None, 0.0, 0.0, n_cta=n_cta)
        assert torch.equal(mi[:NPAR].cpu(), c.int_exact), f"integer data not exact at grid {n_cta}"
        pc, mc = p0.cuda(), m0.cuda()
        C.reduce_sgd(d["slots"], n_slots, d["fac"], n_samples, pc, mc, None, None, 0.05, 0.5, max_grad_norm=big,
                     clip_workspace=ws, grad_norm_out=norm, n_cta=n_cta)
        want_n = R.clip_norm(c.g, n_cta)
        assert_bits(f"clip norm at grid {n_cta}", norm, torch.tensor([float(want_n)]))
        pw, mw = R.update(c.g, p0, m0, 0.5, 0.05, max_norm=big, norm=want_n)
        assert_bits(f"clip params at grid {n_cta}", pc[:NPAR], pw)
        assert_bits(f"clip momentum at grid {n_cta}", mc[:NPAR], mw)
        assert bool(pc[NPAR:].isnan().all() and mc[NPAR:].isnan().all())


# ---------------------------------------------------------------------------------------------------------- every instance
def _sched():
    from dist_tuto.pth_b200.ops.optim import LRSchedule, schedule_tuple
    return schedule_tuple(LRSchedule(warmup_steps=3, decay="cosine", total_steps=40, min_factor=0.1))


#        name                  wd     nesterov sched  max_norm
CONFIGS = [("plain", 0.0, False, False, None), ("wd", 1e-2, False, False, None), ("nesterov", 0.0, True, False, None),
           ("wd+nesterov", 1e-2, True, False, None)]
CONFIGS += [(n + "+cosine", wd, ne, True, None) for n, wd, ne, _, _ in CONFIGS]
CONFIGS += [("clip", 0.0, False, False, 1.0), ("clip-no-op", 0.0, False, False, 1e9),
            ("clip+wd+nesterov", 1e-2, True, False, 1.0), ("clip-no-op+wd+nesterov", 1e-2, True, False, 1e9)]
# (step counter or None, gradient buffer: its grad_stride, or None for no buffer)
VARIANTS = [(None, NPAR_ALLOC), (4, NPAR_ALLOC), (5, 0), (2 ** 32 - 1, NPAR_ALLOC), (4, None), (5, NPAR_ALLOC)]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_every_instance_matches_the_model_with_guard_bands(C, cfg):
    name, wd, nesterov, use_sched, max_norm = cfg
    sched = _sched() if use_sched else None
    ws = torch.zeros(C.clip_workspace_numel(NPAR_ALLOC), device="cuda")
    lr, mu = 0.05, 0.9
    for i, (st, stride) in enumerate(VARIANTS):
        k = (CONFIGS.index(cfg) * len(VARIANTS) + i) * 5
        n_samples, n_slots = SIZES[k % len(SIZES)]
        n_cta = GRIDS[(k // len(SIZES) + 3 * i) % len(GRIDS)]
        c = case(n_samples, n_slots)
        what = f"{name}, step {st}, grad_stride {stride}, {n_samples} samples, {n_slots} slots, grid {n_cta}"
        p0, m0 = _flat(10 + i), _flat(20 + i)
        aux0 = torch.full((13000,), NAN)                     # w2b's pad lanes stay NaN
        loss0 = torch.tensor([1.5, 7.0, SENTINEL, SENTINEL])
        grads0 = None
        if stride is not None:                               # sentinel buckets with NaN tails past NPAR
            grads0 = torch.full((NPAR_ALLOC if stride == 0 else 2 * NPAR_ALLOC,), SENTINEL).view(-1, NPAR_ALLOC)
            grads0[:, NPAR:] = NAN
            grads0 = grads0.reshape(-1)
        p, m, aux, loss = p0.cuda(), m0.cuda(), aux0.cuda(), loss0.cuda()
        grads = grads0.cuda() if grads0 is not None else None
        step = torch.tensor([st], dtype=torch.int64, device="cuda") if st is not None else None
        done = torch.zeros(1, dtype=torch.int32, device="cuda") if st is not None else None
        norm = torch.full((1,), NAN, device="cuda")
        kw = dict(lr_schedule=sched, weight_decay=wd, nesterov=nesterov, n_cta=n_cta)
        if max_norm is not None:
            kw.update(max_grad_norm=max_norm, clip_workspace=ws, grad_norm_out=norm)
        C.reduce_sgd(c.d["slots"], n_slots, c.d["fac"], n_samples, p, m, step, done, lr, mu, aux, loss, grads,
                     stride if stride is not None else 0, **kw)
        torch.cuda.synchronize()
        s = st if st is not None else 0
        lr_s = lr if sched is None else float(C.lr_schedule_eval(sched, lr, torch.tensor([s], device="cuda"))[0])
        want_n = None
        if max_norm is not None:
            want_n = R.clip_norm(c.g, n_cta)
            assert_bits(f"{what}: grad_norm_out", norm, torch.tensor([float(want_n)]))
        pw, mw = R.update(c.g, p0, m0, mu, lr_s, wd, nesterov, max_norm=max_norm, norm=want_n)
        assert_bits(f"{what}: params", p[:NPAR], pw)
        assert_bits(f"{what}: momentum", m[:NPAR], mw)
        assert bool(p[NPAR:].isnan().all() and m[NPAR:].isnan().all()), f"{what}: params / momentum written past NPAR"
        pn = p0.clone()
        pn[:NPAR] = pw
        assert_bits(f"{what}: aux", aux, R.aux_after(aux0, pn))
        assert_bits(f"{what}: loss_acc", loss, R.loss_after(loss0, c.loss))
        if grads is not None:
            assert_bits(f"{what}: gradient buckets", grads, R.bucket_after(grads0, s, stride))
        if st is not None:
            assert int(step.item()) == st + 1 and int(done.item()) == 0, what
        if max_norm is not None and max_norm < 1e3:
            assert float(want_n) > max_norm, f"{what}: the case was meant to clip"


# ---------------------------------------------------------------------------------------------------------- trainer
class _SlotSpy:
    """Wraps a trainer's extension handle: each reduce_sgd launch is recorded with copies of its slots and factors and the
    params and momentum before and after it."""

    def __init__(self, tr):
        self._C, self.log = tr.C, []
        tr.C = self

    def __getattr__(self, name):
        return getattr(self._C, name)

    def reduce_sgd(self, slots, n_slots, factors, n_samples, params, momentum, step, done, lr, mu, *a, **k):
        torch.cuda.current_stream().synchronize()
        rec = dict(slots=slots[:n_slots * DET].view(n_slots, DET).cpu(), fac=factors[:n_samples * FAC].view(n_samples, FAC).cpu(),
                   n_slots=n_slots, n_samples=n_samples, p0=params.cpu(), m0=momentum.cpu(), lr=lr, mu=mu, kw=k)
        self._C.reduce_sgd(slots, n_slots, factors, n_samples, params, momentum, step, done, lr, mu, *a, **k)
        torch.cuda.current_stream().synchronize()
        rec.update(p1=params.cpu(), m1=momentum.cpu())
        self.log.append(rec)


@pytest.mark.parametrize("bsz", [128, 4 * S + 1])
def test_trainer_steps_are_the_model_of_their_launches(bsz):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    tr = FusedTrainer(bsz, lr=0.05, seed=7, device="cuda", raw_uint8=True)
    assert tr.cluster == 1 and tr.grad_slots is not None
    spy = _SlotSpy(tr)
    for x, y in _batches(3, bsz, 17):
        tr.step(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    assert len(spy.log) == 3
    for i, r in enumerate(spy.log):
        assert r["n_samples"] == bsz and r["n_slots"] == min(bsz, 4 * S)
        assert not r["kw"].get("lr_schedule") and not r["kw"].get("max_grad_norm") and not r["kw"].get("weight_decay")
        g = R.local_grad(r["slots"], r["n_slots"], r["fac"], r["n_samples"])
        pw, mw = R.update(g, r["p0"], r["m0"], r["mu"], r["lr"])
        assert_bits(f"batch {bsz} step {i}: params", r["p1"][:NPAR], pw)
        assert_bits(f"batch {bsz} step {i}: momentum", r["m1"][:NPAR], mw)


# ---------------------------------------------------------------------------------------------------------- det_reduce
@pytest.mark.parametrize("n_slots", [1, 2, 31, 32, 33, S])
def test_det_reduce_sums_in_slot_order(C, n_slots):
    g = torch.Generator().manual_seed(n_slots)
    parts = torch.randn(n_slots + 1, DET, generator=g)
    parts[:, NPAR + 2:] = NAN
    parts[n_slots:] = NAN
    gm, lm = R.det_reduce(parts, n_slots)
    pd = parts.cuda()
    for st, stride, with_loss in [(None, 0, True), (0, NPAR_ALLOC, True), (1, NPAR_ALLOC, False), (1, 0, True),
                                  (None, NPAR_ALLOC, False)]:
        what = f"det_reduce {n_slots} slots, step {st}, grad_stride {stride}, loss_acc {with_loss}"
        grads0 = torch.full((2 * NPAR_ALLOC + 64,), NAN)
        grads0[1::2] = SENTINEL
        grads = grads0.cuda()
        step = torch.tensor([st], dtype=torch.int64, device="cuda") if st is not None else None
        loss0 = torch.tensor([0.25, 3.0, SENTINEL, SENTINEL])
        loss = loss0.cuda() if with_loss else None
        C.det_reduce(pd, n_slots, grads, step, stride, loss)
        torch.cuda.synchronize()
        want = grads0.clone()
        off = ((st or 0) & 1) * stride
        want[off:off + NPAR] = gm
        assert_bits(what + ": buckets", grads, want)
        if with_loss:
            want_l = loss0.clone()
            want_l[:2] = want_l[:2] + lm
            assert_bits(what + ": loss_acc", loss, want_l)
        if step is not None:
            assert int(step.item()) == st, what


# ---------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("n_cta", [-1, R.RED_UNITS + 1])
def test_grids_outside_the_units_are_refused_on_the_host(C, n_cta):
    c = case(*SIZES[0])
    p, m = _flat(1).cuda(), _flat(2).cuda()
    p0, m0 = p.clone(), m.clone()
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="n_cta"):
        C.reduce_sgd(c.d["slots"], c.n_slots, c.d["fac"], c.n_samples, p, m, step, done, 0.05, 0.5, n_cta=n_cta)
    torch.cuda.synchronize()
    assert torch.equal(_bits(p), _bits(p0)) and torch.equal(_bits(m), _bits(m0)) and int(step.item()) == 0
