"""The sharded LAMB / LARS model of tests/sharded_layerwise_model.py: within the unsharded model's bound against fp64,
bit for bit the unsharded model on every tensor that lies inside one slice, and planted faults that the checks catch.

The bound is tests/layerwise_cases.py's: after 50 updates the largest parameter error against fp64 is at most 4x the
error of the fp32 torch-op path on the same inputs, plus one fp32 ulp of the largest parameter.  In the bound test rank 0
holds the whole gradient and the other ranks zeros (scale 1), so the averaged gradient is exact and the fp64 reference is the
unsharded one; the rank-order average itself is tested with W different gradients in the bit-for-bit tests."""
import pytest
import torch

import layerwise_cases as TL
import sharded_layerwise_model as S

WORLDS = [2, 3, 5, 8]


def padded(n, world):
    return (n + 4 * world - 1) // (4 * world) * (4 * world)


def states0(kind, n):
    return [torch.zeros(n) for _ in range(2 if kind == "lamb" else 1)]


def run_sharded(kind, hp, seed, world, fault=None, chunk=TL.CHUNK, steps=TL.STEPS):
    """``steps`` sharded updates of tests/layerwise_cases.py's inputs; returns (params of rank 0, ratios per rank)."""
    offsets, numels, p0, grads = TL.inputs(seed, steps)
    n = padded(p0.numel(), world)
    p = torch.cat([p0, torch.zeros(n - p0.numel())])
    st = states0(kind, n)
    for t, g in enumerate(grads, 1):
        g = torch.cat([g, torch.zeros(n - g.numel())])
        out = S.step(kind, [g] + [torch.zeros(n)] * (world - 1), p, st, offsets, numels, TL.ADAPT, hp, 1.0, t=t, fault=fault,
                     chunk=chunk)
        p, st = out["params"][0], out["states"]
    return p[:p0.numel()], out["ratios"]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind,k", TL.CASES)
def test_within_the_bound_of_the_unsharded_model(kind, k, world):
    hp = TL._hp(kind, k)
    ref, b = TL.bound(kind, hp, 10 + k)
    p, ratios = run_sharded(kind, hp, 10 + k, world)
    err = float((p.double() - ref).abs().max())
    assert err <= b, (err, b)
    assert all(r == ratios[0] for r in ratios), "the ranks' ratios differ"


def _layout(world):
    """Tiny tensors in the first slice, one tensor that spans every slice, then TL's shapes and lengths at chunk multiples
    +- 1 around the last slice boundaries: tensors inside one slice and tensors that straddle one boundary at every world."""
    shapes = [(2,), (3,), (1000 * (world - 1),)] + TL.SHAPES + [(TL.CHUNK - 1,), (TL.CHUNK + 1,), (5,)]
    return TL.layout(shapes)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_tensors_inside_one_slice_equal_the_unsharded_model_bit_for_bit(kind, world):
    offsets, numels, n0 = _layout(world)
    adapt = [k > 3 for k in numels]
    n = padded(n0, world)
    gen = torch.Generator().manual_seed(world)
    p = torch.randn(n, generator=gen)
    st = states0(kind, n)
    up, ust = p.clone(), [s.clone() for s in st]
    inside = S.tensors_inside_one_slice(offsets, numels, n, world)
    spans = [t for t, (o, k) in enumerate(zip(offsets, numels)) if o // (n // world) == 0 and (o + k - 1) // (n // world) == world - 1]
    assert inside and spans and len(inside) < len(offsets)
    hp = TL._hp(kind, 1)
    for t in range(1, 6):
        grads = [torch.randn(n, generator=gen) * 0.1 for _ in range(world)]
        out = S.step(kind, grads, p, st, offsets, numels, adapt, hp, 1.0 / world, t=t, chunk=TL.CHUNK)
        up, ust, ur = S.unsharded_step(kind, out["g"], up, ust, offsets, numels, adapt, hp, t=t, chunk=TL.CHUNK)
        p, st = out["params"][0], out["states"]
        assert all(r == out["ratios"][0] for r in out["ratios"])
        for i in inside:
            s = slice(offsets[i], offsets[i] + numels[i])
            assert out["ratios"][0][i] == ur[i], (t, i)
            assert torch.equal(p[s], up[s]), (t, i)
            for a, b in zip(st, ust):
                assert torch.equal(a[s], b[s]), (t, i)


def test_rank_tables_cut_at_tensor_and_slice_boundaries():
    world = 3
    offsets, numels, n0 = _layout(world)
    n = padded(n0, world)
    per = n // world
    covered = torch.zeros(n, dtype=torch.int64)
    for r, tab in enumerate(S.rank_tables(offsets, numels, n, world, TL.CHUNK)):
        for s, ln, t in tab:
            assert s % 4 == 0 and 0 < ln <= TL.CHUNK
            assert r * per <= s and s + ln <= (r + 1) * per
            assert offsets[t] <= s and s + ln <= offsets[t] + numels[t]
            covered[s:s + ln] += 1
    want = torch.zeros(n, dtype=torch.int64)
    for o, k in zip(offsets, numels):
        want[o:o + k] = 1
    assert torch.equal(covered, want)


def test_a_slice_of_padding_only_has_no_chunk():
    tabs = S.rank_tables([0], [8], 32, 4)
    assert tabs[0] == [(0, 8, 0)] and tabs[1:] == [[], [], []]


MATHS_FAULTS = [f for f in S.FAULTS if f != "rank_dependent_order"]


@pytest.mark.parametrize("kind", ["lamb", "lars"])
@pytest.mark.parametrize("fault", MATHS_FAULTS)
def test_planted_faults_are_caught(kind, fault):
    """Each fault changes the model's bits (what the GPU test compares) and leaves the bound of fp64.  At W = 8 both adapted
    tensors of TL's layout straddle a slice boundary."""
    hp, world = TL._hp(kind, 1), 8
    ref, b = TL.bound(kind, hp, 7)
    clean, _ = run_sharded(kind, hp, 7, world)
    bad, _ = run_sharded(kind, hp, 7, world, fault)
    assert not torch.equal(clean, bad), f"{fault}: the bit-for-bit check would not see it"
    err = float((bad.double() - ref).abs().max())
    assert err > b, f"{fault}: error {err} within the bound {b}"


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_every_rank_adds_the_same_totals_and_a_rank_dependent_order_is_caught(kind):
    """The fp64 totals every rank forms from the W ranks' sums are the same bits on every rank.  A rank-dependent order
    (each rank starting from its own sums) breaks that.  It shows only where the ranks' sums use all 53 bits (an fp64 sum
    of a few fp32 partials of similar size is exact in any order), so each chunk of the parameters is scaled by its own
    power of two here; the fp32 ratio rarely shows such a difference of a few fp64 ulps, so the check is on the totals."""
    world = 8
    offsets, numels, n0 = _layout(world)
    adapt = [k > 3 for k in numels]
    n = padded(n0, world)
    gen = torch.Generator().manual_seed(5)
    p = torch.randn(n, generator=gen)
    p *= (2.0 ** torch.randint(-20, 21, (n // TL.CHUNK + 1,), generator=gen).float()).repeat_interleave(TL.CHUNK)[:n]
    hp = TL._hp(kind, 1)
    grads = [torch.randn(n, generator=gen) * 0.1 for _ in range(world)]
    clean = S.step(kind, grads, p, states0(kind, n), offsets, numels, adapt, hp, 1.0 / world, chunk=TL.CHUNK)
    bad = S.step(kind, grads, p, states0(kind, n), offsets, numels, adapt, hp, 1.0 / world, chunk=TL.CHUNK,
                 fault="rank_dependent_order")
    assert all(t == clean["totals"][0] for t in clean["totals"])
    assert any(t != bad["totals"][0] for t in bad["totals"]), "the ranks' totals agree under a rank-dependent order"
