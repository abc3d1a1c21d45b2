"""CPU tier: the references of tests/step_oracle.py -- the host Philox dropout stream, the per-sample fp64 oracle and the
per-sample checker -- against published known answers, against ``Net`` autograd, and against planted faults that the
checker must report at least 10x over its bound."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import step_oracle as O
from dist_tuto.pth_b200.models.convnet import Net
from dist_tuto.pth_b200.ops.convnet_fused import pack_params


def _kat(ctr, key):
    off, sub, seed = ctr[0] | ctr[1] << 32, ctr[2] | ctr[3] << 32, key[0] | key[1] << 32
    return [int(v) for v in O.philox4x32_10(seed, sub, off)]


def test_philox_matches_the_random123_known_answers():
    assert _kat([0, 0, 0, 0], [0, 0]) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert _kat([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert _kat([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0]) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_philox_vectorises_over_subsequences_and_offsets():
    sub = np.array([0, 1, 2 ** 32 + 5], dtype=np.uint64)[:, None]
    off = np.array([0, 7, 2 ** 40 + 3], dtype=np.uint64)[None, :]
    got = O.philox4x32_10(0xDEADBEEF01234567, sub, off)
    for i in range(3):
        for j in range(3):
            assert (got[i, j] == O.philox4x32_10(0xDEADBEEF01234567, int(sub[i, 0]), int(off[0, j]))).all()


@pytest.mark.parametrize("p", [0.0, 0.25, 0.5, 0.9])
def test_mask_values_and_keep_rate(p):
    m = O.dropout_masks(seed=3, sample_base=0, B=4096, step=5, p_drop=p).numpy()
    scale = np.float32(1) / (np.float32(1) - np.float32(p))
    assert set(np.unique(m).tolist()) <= {0.0, float(scale)}
    kept = float((m > 0).mean())                     # 286720 draws: 5 sigma of the keep rate is < 0.005
    assert abs(kept - (1 - p)) < 0.005, kept
    # channels and units draw independently: both halves keep at the same rate, and no column is stuck
    assert abs(float((m[:, :20] > 0).mean()) - (1 - p)) < 0.01 and abs(float((m[:, 20:] > 0).mean()) - (1 - p)) < 0.01
    if 0 < p:
        assert ((m > 0).mean(axis=0) < 1).all()
    assert (O.dropout_masks(3, 0, 8, 5, p, training=False).numpy() == 1).all()


def test_uniform_k_comes_from_counter_step_times_32_plus_k_div_4_word_k_mod_4():
    seed, base, step = 0x0123456789ABCDEF, 1000, 2 ** 40 + 3
    u = O.uniforms(seed, base, 3, step, 70)
    for b in range(3):
        for k in (0, 3, 4, 19, 20, 37, 69):
            w = O.philox4x32_10(seed, base + b, step * 32 + k // 4)[k % 4]
            assert u[b, k] == np.float32(int(w)) * np.float32(2.0 ** -32)


def test_high_words_of_step_seed_and_sample_change_the_stream():
    ref = O.dropout_masks(7, 5, 16, 1, 0.5)
    assert not torch.equal(ref, O.dropout_masks(7, 5, 16, 2 ** 32 + 1, 0.5))        # step's high word
    assert not torch.equal(ref, O.dropout_masks(7 + 2 ** 32, 5, 16, 1, 0.5))        # seed's high word
    assert not torch.equal(ref, O.dropout_masks(7, 5 + 2 ** 32, 16, 1, 0.5))        # sample index's high word
    assert torch.equal(ref, O.dropout_masks(7, 5, 16, 1, 0.5))


def test_masks_are_a_function_of_the_global_sample_index():
    a = O.dropout_masks(11, 0, 64, 9, 0.25)
    assert torch.equal(a, torch.cat([O.dropout_masks(11, 0, 32, 9, 0.25), O.dropout_masks(11, 32, 32, 9, 0.25)]))


def test_boundary_draw_is_exactly_p_and_kept():
    seed, sample, step, k = O.find_boundary_draw(0.5)
    u = O.uniforms(seed, sample, 1, step, 70)
    assert u[0, k] == np.float32(0.5) and k < 70
    assert float(O.dropout_masks(seed, sample, 1, step, 0.5)[0, k]) == 2.0


# ------------------------------------------------------------------------------------------------ oracle vs Net autograd
def _case(B, seed=0, p=0.5, step=3, training=True):
    torch.manual_seed(seed)
    net = Net()
    flat = pack_params(net)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(B, 1, 28, 28, generator=g)
    y = torch.randint(0, 10, (B,), generator=g)
    m = O.dropout_masks(seed, 0, B, step, p, training)
    return net.double(), flat, x, y, m


def test_per_sample_gradients_sum_to_the_batch_gradient_of_net():
    net, flat, x, y, m = _case(9, p=0.25)
    ref = O.per_sample_reference(flat, x, y, m)
    # Net's own layers on the whole batch, dropout replaced by the same scales
    h = F.relu(F.max_pool2d(net.conv1(x.double()), 2))
    h = F.relu(F.max_pool2d(net.conv2(h) * m[:, :20, None, None].double(), 2)).reshape(-1, 320)
    logp = F.log_softmax(net.fc2(F.relu(net.fc1(h)) * m[:, 20:].double()), dim=1)
    F.nll_loss(logp, y, reduction="sum").backward()
    for name, p in net.named_parameters():
        assert torch.allclose(ref[name].sum(0), p.grad, rtol=1e-10, atol=1e-13), name
    assert torch.allclose(ref["logp"], logp.detach(), rtol=1e-12, atol=1e-12)
    assert torch.equal(ref["argmax"], logp.argmax(1))


def test_with_masks_of_one_the_oracle_is_net_eval():
    net, flat, x, y, _ = _case(5)
    net.eval()
    ref = O.per_sample_reference(flat, x, y, None)
    out = net(x.double())
    assert torch.allclose(ref["logp"], out.detach(), rtol=1e-12, atol=1e-12)
    F.nll_loss(out, y, reduction="sum").backward()
    for name, p in net.named_parameters():
        assert torch.allclose(ref[name].sum(0), p.grad, rtol=1e-10, atol=1e-13), name


def test_uint8_input_is_normalised_as_in_the_kernels():
    xu = torch.tensor([0, 1, 128, 255], dtype=torch.uint8).repeat(196).reshape(1, 1, 28, 28)
    xf = O.model_input(xu)
    want = (xu.float() * (np.float32(1) / np.float32(255)) - np.float32(0.1307)) * (np.float32(1) / np.float32(0.3081))
    assert xf.dtype == torch.float32 and torch.equal(xf, want)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_max_pool_ties_go_to_the_first_element_in_row_major_order(dtype):
    for vals, first in (([3, 3, 3, 3], 0), ([1, 3, 3, 3], 1), ([1, 2, 3, 3], 2), ([0, 0, 0, 0], 0)):
        x = torch.tensor(vals, dtype=dtype).reshape(1, 1, 2, 2).requires_grad_()
        F.max_pool2d(x, 2).sum().backward()
        assert x.grad.flatten().tolist() == [1.0 if i == first else 0.0 for i in range(4)], vals
    # and the relu at exactly 0 passes no gradient
    z = torch.zeros(3, dtype=dtype, requires_grad=True)
    F.relu(z).sum().backward()
    assert z.grad.tolist() == [0.0, 0.0, 0.0]


# ---------------------------------------------------------------------------------------------------- the checker
def _refs(flat, x, y, m):
    return O.per_sample_reference(flat, x, y, m), O.per_sample_reference(flat, x, y, m, torch.float32)


def _faulty_masks(kind, seed, base, B, step, p):
    if kind == "scale 1/p":
        u = O.uniforms(seed, base, B, step, 70)
        return torch.from_numpy(np.where(u >= np.float32(p), np.float32(1) / np.float32(p), 0).astype(np.float32))
    if kind == "keep test inverted":
        u = O.uniforms(seed, base, B, step, 70)
        return torch.from_numpy(np.where(u < np.float32(p), O.keep_scale(p), 0).astype(np.float32))
    if kind == "> at the boundary draw":
        u = O.uniforms(seed, base, B, step, 70)
        return torch.from_numpy(np.where(u > np.float32(p), O.keep_scale(p), 0).astype(np.float32))
    if kind == "rnd index off by one":
        u = O.uniforms(seed, base, B, step, 72)[:, 1:71]
        return torch.from_numpy(np.where(u >= np.float32(p), O.keep_scale(p), 0).astype(np.float32))
    if kind == "step truncated to 32 bits":
        return O.dropout_masks(seed, base, B, step % 2 ** 32, p)
    raise ValueError(kind)


def _pool_last(x, k):
    """max-pool whose ties go to the LAST element of the window (flipping both axes reverses the row-major order)."""
    return torch.flip(F.max_pool2d(torch.flip(x, (-2, -1)), k), (-2, -1))


def _relu_open(x):
    """relu whose derivative at exactly 0 is 1."""
    return torch.where(x >= 0, x, torch.zeros_like(x))


def _planted(kind):
    """(got, ref64, ref32, masks, labels) for one planted fault."""
    torch.manual_seed(1)
    net = Net()
    g = torch.Generator().manual_seed(2)
    B = 6
    x = torch.randn(B, 1, 28, 28, generator=g)
    y = torch.randint(0, 10, (B,), generator=g)
    seed, base, step, p = 5, 0, 3, 0.25
    if kind in ("ties routed to the last element", "relu'(0) = 1"):
        with torch.no_grad():
            net.conv1.weight.zero_()                 # every pool1 window is an exact 4-way tie
            if kind == "relu'(0) = 1":
                net.conv1.bias.zero_()               # and every relu of conv1 sits at exactly 0
        flat = pack_params(net)
        r64, r32 = _refs(flat, x, y, None)
        kw = {"pool": _pool_last} if kind.startswith("ties") else {"relu": _relu_open}
        return O.per_sample_reference(flat, x, y, None, torch.float32, **kw), r64, r32, None, None
    if kind == "> at the boundary draw":
        seed, base, step, _ = O.find_boundary_draw(0.5)
        p, B = 0.5, 1
        x, y = x[:1], y[:1]
    if kind == "step truncated to 32 bits":
        step = 2 ** 32 + 1
    flat = pack_params(net)
    m = O.dropout_masks(seed, base, B, step, p)
    r64, r32 = _refs(flat, x, y, m)
    if kind in ("scale 1/p", "keep test inverted", "> at the boundary draw", "rnd index off by one",
                "step truncated to 32 bits"):
        bad = _faulty_masks(kind, seed, base, B, step, p)
        got = O.per_sample_reference(flat, x, y, bad, torch.float32)
        got["masks"] = bad                              # what such a kernel would report in mask_out
        return got, r64, r32, m, None
    if kind == "two samples' gradients swapped":
        got = {k: v.clone() for k, v in r32.items()}
        for n in O.NAMES:
            got[n][[1, 4]] = got[n][[4, 1]]
        return got, r64, r32, m, None
    if kind == "one sample's fc1.weight term dropped from its slot":
        groups = [[0, 3], [1, 4], [2, 5]]               # 6 samples on 3 CTAs
        f64, f32 = O.fold(r64, groups), O.fold(r32, groups)
        got = {k: v.clone() for k, v in f32.items()}
        got["fc1.weight"][1] -= r32["fc1.weight"][4]
        return got, f64, f32, None, [f"slot {i}" for i in range(3)]
    if kind == "loss without inv_bsz":
        s64, s32 = O.scaled(r64, 1 / B), O.scaled(r32, 1 / B)
        got = {k: v.clone() for k, v in s32.items()}
        got["loss"] = r32["loss"].clone()
        return got, s64, s32, m, None
    raise ValueError(kind)


FAULTS = ["two samples' gradients swapped", "ties routed to the last element", "relu'(0) = 1", "scale 1/p",
          "keep test inverted", "> at the boundary draw", "rnd index off by one", "step truncated to 32 bits",
          "one sample's fc1.weight term dropped from its slot", "loss without inv_bsz"]


@pytest.mark.parametrize("kind", FAULTS)
def test_checker_catches_the_planted_fault(kind):
    got, r64, r32, m, labels = _planted(kind)
    rep = O.check_per_sample(got, r64, r32, masks=m, labels=labels)
    print(f"planted fault {kind!r}: caught, worst {rep.worst:.3g}x the bound at {rep.worst_at}")
    assert rep.failures and rep.worst >= 10, rep.message()
    if "masks" in got:      # a kernel that reported the right masks but applied these would fail on its gradients alone
        rep = O.check_per_sample({k: v for k, v in got.items() if k != "masks"}, r64, r32, masks=m, labels=labels)
        print(f"    without the mask comparison: worst {rep.worst:.3g}x the bound at {rep.worst_at}")
        assert rep.failures and rep.worst >= 10, rep.message()


def test_checker_passes_a_one_ulp_perturbation_of_every_nonzero_entry():
    """Exact zeros stay zero (a kernel that flushes denormals cannot produce a 1-ulp neighbour of 0 either)."""
    torch.manual_seed(3)
    flat = pack_params(Net())
    g = torch.Generator().manual_seed(4)
    x, y = torch.randn(8, 1, 28, 28, generator=g), torch.randint(0, 10, (8,), generator=g)
    m = O.dropout_masks(9, 0, 8, 1, 0.5)
    r64, r32 = _refs(flat, x, y, m)
    rng = np.random.default_rng(5)
    got = {}
    for k in O.FLOAT_KEYS:
        a = r32[k].numpy()
        towards = np.where(rng.random(a.shape) < 0.5, np.float32(np.inf), np.float32(-np.inf))
        got[k] = torch.from_numpy(np.where(a != 0, np.nextafter(a, towards), a).astype(np.float32))
    got["masks"] = m.clone()
    rep = O.check_per_sample(got, r64, r32, masks=m)
    assert not rep.failures, rep.message()
    assert rep.worst < 0.5, rep.message()


def test_a_second_plain_fp32_implementation_passes_the_bound():
    """Net's batched fp32 autograd (other convolution algorithms and summation orders than the per-sample vmap) summed over
    a 16-sample batch: a plain fp32 implementation that the bound, set by the per-sample one, must accept."""
    torch.manual_seed(6)
    net = Net()
    flat = pack_params(net)
    g = torch.Generator().manual_seed(7)
    x, y = torch.randn(16, 1, 28, 28, generator=g), torch.randint(0, 10, (16,), generator=g)
    m = O.dropout_masks(2, 0, 16, 4, 0.5)
    r64, r32 = _refs(flat, x, y, m)
    p = {k: v.clone().requires_grad_() for k, v in O._params(flat, torch.float32).items()}
    logp = F.log_softmax(O.masked_forward(p, x, m[:, :20], m[:, 20:]), dim=1)
    F.nll_loss(logp, y, reduction="sum").backward()
    got = {k: p[k].grad[None] for k in O.NAMES}
    rep = O.check_per_sample(got, O.fold(r64, [range(16)]), O.fold(r32, [range(16)]), labels=["batch"])
    assert not rep.failures, rep.message()
    rep = O.check_per_sample({"logp": logp.detach()}, r64, r32)
    assert not rep.failures, rep.message()


def test_where_both_references_are_exactly_zero_any_nonzero_fails_and_nan_fails():
    zero64, zero32 = {"loss": torch.zeros(2, dtype=torch.float64)}, {"loss": torch.zeros(2)}
    assert math.isinf(O.check_per_sample({"loss": torch.tensor([0.0, 1e-30])}, zero64, zero32).worst)
    assert not O.check_per_sample({"loss": torch.zeros(2)}, zero64, zero32).failures
    one64, one32 = {"loss": torch.ones(2, dtype=torch.float64)}, {"loss": torch.ones(2)}
    assert math.isinf(O.check_per_sample({"loss": torch.tensor([1.0, float("nan")])}, one64, one32).worst)
