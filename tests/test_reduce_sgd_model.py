"""CPU tier: the rounding-exact model of reduce_sgd and det_reduce (tests/reduce_sgd_model.py) -- the constants it reads
from the kernel headers, the model within the fp64 bound at every size, size and grid tables without gaps, and planted
faults in the summation order or routing that the bit-exact check (and for routing faults the bound) reports."""
import numpy as np
import pytest
import torch

import reduce_sgd_model as R


def _data(n_samples, n_slots, seed, ints=False):
    g = torch.Generator().manual_seed(seed)
    if ints:
        return (torch.randint(-4, 5, (n_slots, R.DET_STRIDE), generator=g).float(),
                torch.randint(-3, 4, (n_samples, R.FAC_STRIDE), generator=g).float())
    return torch.randn(n_slots, R.DET_STRIDE, generator=g), torch.randn(n_samples, R.FAC_STRIDE, generator=g)


def _bits_equal(a, b):
    return torch.equal(a.float().contiguous().view(torch.int32), b.float().contiguous().view(torch.int32))


def _within(got, ref, bound):
    return bool(((got.double() - ref).abs() <= bound).all())


# ---------------------------------------------------------------------------------------------------------- constants
def test_constants_match_the_header_and_the_parse_refuses_a_mangled_header():
    k = R.K
    assert (k["RKS"], k["RSS"], k["RSLOT_BATCH"] * k["RSS"], k["RED_FC1_TILES"], k["RED_OTHER"], k["RED_UNITS"]) == \
        (6, 25, 150, 50, 1462, 124)
    # the header's own static_asserts
    assert k["RKS"] * k["RED_TILE_VEC"] <= k["RED_T"] - 32
    assert 50 % k["RJ"] == 0 and 320 % k["RI"] == 0 and k["RJ"] % 2 == 0 and k["RI"] % 4 == 0
    assert k["W3"] % 4 == 0 and k["FAC_STRIDE"] % 4 == 0 and k["FAC_P2"] >= 50 and k["FAC_P2"] + 320 <= k["FAC_STRIDE"]
    assert k["NPAR"] + 2 <= k["DET_STRIDE"]
    with open(R.CSRC + "/convnet_reduce.cuh") as f:
        red = f.read()
    with open(R.CSRC + "/convnet_args.cuh") as f:
        args = f.read()
    assert R.parse_constants(red, args) == k
    with pytest.raises(ValueError, match="RKC"):
        R.parse_constants(red.replace("RKC = 128;", "RKC = kPass;"), args)
    with pytest.raises(ValueError, match="FAC_STRIDE"):
        R.parse_constants(red, args.replace("FAC_STRIDE = 384", "FAC_STRIDE=384"))


@pytest.mark.parametrize("S", [132, 114])
def test_size_and_grid_tables_have_no_gaps(S):
    assert R.gaps(S) == []
    assert R.gaps(S, table=R.sizes(S)[1:]) != []                       # (1 sample, 1 slot) is the only 1-sample row
    assert R.gaps(S, grid_table=[g for g in R.grids() if g != 1]) != []
    assert R.gaps(S, grid_table=[g for g in R.grids() if g > 3]) != []
    assert max(R.grids()) == R.RED_UNITS


def test_units_cover_every_unit_once_at_every_grid():
    for n in R.grids():
        got = sorted(u for c in R.units(n) for u in c)
        assert got == list(range(R.RED_UNITS))
    # every float4 vector of the gradient is emitted by exactly one thread of one unit
    v = torch.cat([R.unit_vectors(u) for u in range(R.RED_UNITS)])
    v = v[v >= 0]
    assert v.numel() == R.NPAR // 4 and torch.equal(v.sort().values, torch.arange(R.NPAR // 4))


# ---------------------------------------------------------------------------------------------------------- the bound
@pytest.mark.parametrize("n_samples,n_slots", R.sizes(132))
def test_model_is_within_the_fp64_bound(n_samples, n_slots):
    slots, factors = _data(n_samples, n_slots, seed=n_samples * 7 + n_slots)
    g = R.local_grad(slots, n_slots, factors, n_samples)
    ref, bound, lref, lbound = R.fp64_bound(slots, n_slots, factors, n_samples)
    assert _within(g, ref, bound)
    assert _within(R.loss_terms(slots, n_slots), lref, lbound)
    gd, ld = R.det_reduce(slots, n_slots)
    assert _within(gd[R.OTHER], ref[R.OTHER], bound[R.OTHER]) and _within(ld, lref, lbound)
    n64 = float(ref.norm())
    for n_cta in (1, 50, 124):
        assert abs(float(R.clip_norm(g, n_cta)) - n64) <= 2 ** -14 * n64


def test_small_integers_are_exact():
    slots, factors = _data(1000, 301, seed=3, ints=True)
    ref, _, lref, _ = R.fp64_bound(slots, 301, factors, 1000)
    assert torch.equal(R.local_grad(slots, 301, factors, 1000).double(), ref)
    assert torch.equal(R.loss_terms(slots, 301).double(), lref)


# ---------------------------------------------------------------------------------------------------------- planted faults
N_SMP, N_SL = 300, 151                # several passes, several slot rounds, a partial load batch


@pytest.fixture(scope="module")
def case():
    slots, factors = _data(N_SMP, N_SL, seed=11)
    return slots, factors, R.local_grad(slots, N_SL, factors, N_SMP), R.fp64_bound(slots, N_SL, factors, N_SMP)


SUM_FAULTS = {
    "a pass of 127 samples": dict(rkc=127),
    "a sample-group stride of 5": dict(stride=5),
    "the group partials added in reverse": dict(group_order=list(range(R.RKS))[::-1]),
    "24 slot groups": dict(rss=24),
}


@pytest.mark.parametrize("name", list(SUM_FAULTS))
def test_planted_order_fault_is_caught(case, name):
    slots, factors, good, _ = case
    bad = R.local_grad(slots, N_SL, factors, N_SMP, **SUM_FAULTS[name])
    assert not _bits_equal(bad, good), name


@pytest.mark.parametrize("name", ["the last slot dropped", "the slots rotated by one", "an fc1 column offset by one vector"])
def test_planted_input_fault_is_caught(case, name):
    slots, factors, good, (ref, bound, _, _) = case
    if name == "the last slot dropped":
        bad = R.local_grad(slots, N_SL - 1, factors, N_SMP)
    elif name == "the slots rotated by one":
        bad = R.local_grad(torch.roll(slots[:N_SL], 1, 0), N_SL, factors, N_SMP)
    else:
        f = factors.clone()
        f[:, R.FAC_P2:R.FAC_P2 + 320] = torch.roll(f[:, R.FAC_P2:R.FAC_P2 + 320], -4, 1)
        bad = R.local_grad(slots, N_SL, f, N_SMP)
    assert not _bits_equal(bad, good), name
    if name != "the slots rotated by one":                # a routing fault: outside the bound as well
        assert not _within(bad, ref, bound), name


def test_planted_loss_butterfly_fault_is_caught():
    slots, _ = _data(1, 301, seed=5)
    assert not _bits_equal(R.loss_terms(slots, 301, butterfly=False), R.loss_terms(slots, 301))


def test_planted_bucket_fault_is_caught():
    grads = torch.full((2 * 21888,), 3.0)
    good = R.bucket_after(grads, 5, 21888)
    bad = R.bucket_after(grads, 5, 21888, zero="current")
    assert not torch.equal(bad, good)
    want = grads.clone()
    want[:R.NPAR] = 0.0                                    # step 5: parity 1, bucket 0 is the other one
    assert torch.equal(good, want) and not torch.equal(bad, want)


def test_planted_aux_fault_is_caught():
    g = torch.Generator().manual_seed(2)
    params = torch.randn(21888, generator=g)
    aux = torch.full((13000,), float("nan"))
    good, bad = R.aux_after(aux, params), R.aux_after(aux, params, swap=True)
    assert not _bits_equal(bad, good)
    w = params[264:5264].view(20, 10, 25)                  # the fp64-free reference: conv2.weight permuted by torch
    assert torch.equal(good[:5000], w.permute(1, 2, 0).reshape(-1))
    assert not torch.equal(bad[:5000], w.permute(1, 2, 0).reshape(-1))
    wb = good[5000:].view(20, 25, 2, 8)
    assert torch.equal(wb[..., :5], w.view(20, 2, 5, 25).permute(0, 3, 1, 2)) and bool(wb[..., 5:].isnan().all())


def test_planted_clip_chain_fault_is_caught(case):
    _, _, good, _ = case
    assert any(R.clip_norm(good, n, per="cta") != R.clip_norm(good, n) for n in (1, 2, 3))


def test_planted_det_reduce_order_fault_is_caught():
    slots, _ = _data(1, 64, seed=9)
    g, l = R.det_reduce(slots, 64)
    gr, lr = R.det_reduce(slots[:64].flip(0), 64)
    assert not _bits_equal(gr, g) and not _bits_equal(torch.cat([g, l]), torch.cat([gr, lr]))


def test_clip_norm_depends_on_the_grid_only_through_the_squares_order(case):
    _, _, good, _ = case
    norms = {n: R.clip_norm(good, n) for n in R.grids()}
    ref = float(good.double().norm())
    assert all(abs(float(v) - ref) <= 2 ** -20 * ref for v in norms.values())
    assert all(isinstance(v, np.float32) for v in norms.values())
