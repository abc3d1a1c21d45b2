"""GPU tier: the evaluation kernel (csrc/convnet_eval.cu) sample by sample against fp64 (tests/eval_checks.py), at the
sample counts where its persistent grid, group residues and mbarrier phases change, with guard bands around every output;
bit-for-bit invariance of a sample's row to where it sits; constructed edges (tied pools, ReLU zeros, exact logit ties,
saturated softmax); invalid labels; argument refusals; and evaluation sharded over emulated and real ranks."""
import math

import pytest
import torch

import dist_tuto.pth_b200 as b2
import eval_checks as E
import eval_workers as W
from dist_tuto.pth_b200.data import MNIST_MEAN, MNIST_STD, SyntheticMNIST, TensorImageDataset, eval_shard_range
from dist_tuto.pth_b200.models.convnet import Net
from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.ops.convnet_eval import Evaluator, convnet_evaluate
from dist_tuto.pth_b200.ops.convnet_fused import pack_params, unpack_params

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

PAD = 16
SENT_F64 = -1234.5678                   # fills the fp64 buffer around `result`
SENT_I32 = 0x5A5A5A5A                   # fills the slot words the kernel may not touch
NAN_BITS = 0x7FC00000                   # the NaN around `out_logp`
NONMNIST = (0.5, 0.25)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def geo(dev):
    C = _ext.C()
    return (C.convnet_eval_slot_words(dev.index) - 2) // 2, C.convnet_eval_samples_per_cta()


@pytest.fixture(scope="module")
def params(dev):
    torch.manual_seed(2024)
    return pack_params(Net(), dev)


def _images(n, u8, seed):
    if u8:
        ds = SyntheticMNIST(n=n, seed=seed)
        return ds.images, ds.labels
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 1, 28, 28, generator=g), torch.randint(0, 10, (n,), generator=g)


def run(params, x, y, mean=MNIST_MEAN, std=MNIST_STD, logp=True):
    """One call of the binding with guard bands: ``out_logp`` a ``[:N]`` view of a NaN-filled ``[N + 16, 10]`` buffer,
    ``result`` a view inside a sentinel-filled fp64 buffer, ``slots`` longer than the device needs and sentinel-filled
    past the ticket.  After the call no sentinel has changed, the ticket is 0 again and no slot word past the grid's was
    written (none at all for N = 0: nothing launched).  Returns (result, out_logp or None) on the CPU."""
    C, dev = _ext.C(), params.device
    N = y.numel()
    lp_buf = torch.full((N + PAD, 10), math.nan, device=dev)
    res_buf = torch.full((2 * PAD + 3,), SENT_F64, dtype=torch.float64, device=dev)
    slots = torch.full((C.convnet_eval_slot_words(dev.index) + 64,), SENT_I32, dtype=torch.int32, device=dev)
    slots[0] = 0
    C.convnet_eval(params, x.to(dev), y.to(dev), res_buf[PAD:PAD + 3], slots, float(mean), float(std),
                   lp_buf[:N] if logp else None)
    torch.cuda.synchronize()
    lp_buf, res_buf, slots = lp_buf.cpu(), res_buf.cpu(), slots.cpu()
    G, S = (slots.numel() - 64 - 2) // 2, C.convnet_eval_samples_per_cta()
    grid = E.schedule(N, G, S)["grid"]
    tail = lp_buf[N:] if logp else lp_buf
    assert bool((tail.view(torch.int32) == NAN_BITS).all()), f"N={N}: out_logp written past row N"
    guard = torch.cat([res_buf[:PAD], res_buf[PAD + 3:]])
    assert bool((guard == SENT_F64).all()), f"N={N}: result's neighbours overwritten"
    assert int(slots[0]) == 0, f"N={N}: ticket left at {int(slots[0])}"
    assert bool((slots[1 + 2 * grid:] == SENT_I32).all()), f"N={N}: slot words past the grid of {grid} written"
    res = res_buf[PAD:PAD + 3]
    if N == 0:
        assert res.tolist() == [0.0, 0.0, 0.0]
    return res, (lp_buf[:N] if logp else None)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _assert_checks(res, lp, y, r64, r32, geo, where=""):
    rep = E.check_eval(res, lp, y, r64, r32, *geo, where=where)
    assert not rep.failures, rep.message()
    return rep


# --------------------------------------------------------------------------------------------------- the size table
@pytest.mark.parametrize("u8", [True, False], ids=["uint8", "fp32"])
def test_size_table_against_fp64_with_guards_and_position_invariance(dev, geo, params, u8):
    """Every N of eval_sizes(G, S) on prefixes of one image pool: all checks, guard bands, the result without out_logp
    bit-equal to the one with it, and each sample's row bit-equal to its row in the largest call (other grid, other CTA,
    other group slot)."""
    G, S = geo
    table = sorted(E.eval_sizes(G, S), reverse=True)
    x, y = _images(table[0], u8, seed=101 + u8)
    r64, r32 = E.reference(params, x, y, MNIST_MEAN, MNIST_STD), E.reference(params, x, y, MNIST_MEAN, MNIST_STD,
                                                                             torch.float32)
    xd, yd = x.to(dev), y.to(dev)
    full = None
    worst = {}
    for n in table:
        res, lp = run(params, xd[:n], yd[:n])
        rep = _assert_checks(res, lp, y[:n], E.sliced(r64, 0, n), E.sliced(r32, 0, n), geo, where=f"N={n}: ")
        for k, v in rep.ratios.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if full is None:
            full = lp
        assert _same_bits(lp, full[:n]), f"N={n}: rows differ from the same samples' rows at N={table[0]}"
        res_nolp, _ = run(params, xd[:n], yd[:n], logp=False)
        assert torch.equal(res_nolp, res), f"N={n}: result without out_logp {res_nolp.tolist()} != {res.tolist()}"
    print(f"\n[eval edges] {'uint8' if u8 else 'fp32'}: G = {G}, S = {S}, {len(table)} sizes up to {table[0]}; worst "
          f"error / bound: logp {worst['logp']:.3g}, loss {worst['loss']:.3g}, sum {worst['sum']:.3g}, "
          f"sum64 {worst['sum64']:.3g}")


@pytest.mark.parametrize("u8", [True, False], ids=["uint8", "fp32"])
def test_rows_do_not_depend_on_the_offset_into_x(dev, geo, params, u8):
    """Slices of one pool starting at 0 .. 7 and at 8k + 3: every group's bulk copy starts elsewhere and every sample
    sits in another group slot, yet each row is bit-equal to the same sample's row in the unshifted call."""
    G, S = geo
    M = S * G + 13
    starts = list(range(8)) + [8 * k + 3 for k in (1, 40, 131)]
    x, y = _images(M + max(starts), u8, seed=202 + u8)
    xd, yd = x.to(dev), y.to(dev)
    _, whole = run(params, xd, yd)
    r64, r32 = E.reference(params, x, y, MNIST_MEAN, MNIST_STD), E.reference(params, x, y, MNIST_MEAN, MNIST_STD,
                                                                             torch.float32)
    for o in starts:
        res, lp = run(params, xd[o:o + M], yd[o:o + M])
        assert _same_bits(lp, whole[o:o + M]), f"offset {o}: rows differ"
        if o in (3, 8 * 131 + 3):
            _assert_checks(res, lp, y[o:o + M], E.sliced(r64, o, o + M), E.sliced(r32, o, o + M), geo, f"offset {o}: ")
        else:
            lo, hi = E.prediction_range(lp, y[o:o + M], E.sliced(r64, o, o + M))
            assert lo <= res[1] <= hi and res[2] == M


def test_mean_and_std_passed_are_used(dev, geo, params):
    """uint8 input normalised with a non-MNIST mean / std, and with a small std (inputs up to ~100): the checks hold on the
    fp32 image the kernel computes on.  Float32 input ignores mean / std: its rows are the same bits for any."""
    G, S = geo
    x, y = _images(S * G + 5, True, seed=303)
    for (mean, std), n in ((NONMNIST, S * G + 5), ((0.2, 0.01), 77)):
        r64, r32 = E.reference(params, x[:n], y[:n], mean, std), E.reference(params, x[:n], y[:n], mean, std, torch.float32)
        res, lp = run(params, x[:n], y[:n], mean, std)
        _assert_checks(res, lp, y[:n], r64, r32, geo, f"mean {mean}, std {std}: ")
    xf = E.normalize_u8(x[:77], *NONMNIST)
    _, a = run(params, xf, y[:77], *NONMNIST)
    _, b = run(params, xf, y[:77], MNIST_MEAN, MNIST_STD)
    assert _same_bits(a, b)


def test_uint8_and_fp32_paths_agree_within_the_bound(dev, geo, params):
    """The uint8 path and the fp32 path fed the reference's fp32 image both pass against the same reference.  They need
    not be bit-equal: --use_fast_math may contract the normalisation into an fma."""
    G, S = geo
    x, y = _images(S * G + 5, True, seed=404)
    r64, r32 = E.reference(params, x, y, *NONMNIST), E.reference(params, x, y, *NONMNIST, dtype=torch.float32)
    res_u8, lp_u8 = run(params, x, y, *NONMNIST)
    res_f32, lp_f32 = run(params, E.normalize_u8(x, *NONMNIST), y, *NONMNIST)
    _assert_checks(res_u8, lp_u8, y, r64, r32, geo, "uint8: ")
    _assert_checks(res_f32, lp_f32, y, r64, r32, geo, "fp32: ")
    assert res_u8[2] == res_f32[2] == y.numel()


# ------------------------------------------------------------------------------------------------ constructed edges
def _edge(params, x, y, geo, mean=MNIST_MEAN, std=MNIST_STD, where=""):
    r64, r32 = E.reference(params, x, y, mean, std), E.reference(params, x, y, mean, std, torch.float32)
    res, lp = run(params, x, y, mean, std)
    _assert_checks(res, lp, y, r64, r32, geo, where)
    return res, lp, r64


def test_constant_images_tie_every_max_pool_window(dev, geo, params):
    n = 2 * geo[1] + 3
    y = torch.arange(n) % 10
    cases = [("blank", torch.zeros(n, 28, 28, dtype=torch.uint8)), ("saturated", torch.full((n, 28, 28), 255, dtype=torch.uint8)),
             ("fp32 0.7", torch.full((n, 1, 28, 28), 0.7)), ("fp32 -1.3", torch.full((n, 1, 28, 28), -1.3))]
    for name, x in cases:
        _, lp, _ = _edge(params, x, y, geo, where=name + ": ")
        assert _same_bits(lp, lp[:1].expand(n, 10).contiguous()), f"{name}: equal images, different rows"


def test_zero_conv1_weights_leave_bias_only_and_relu_zeros(dev, geo, params):
    p = params.clone()
    v = unpack_params(p)
    v["conv1.weight"].zero_()
    v["conv1.bias"].copy_(torch.linspace(-0.3, 0.3, 10, device=dev))      # channels 0 .. 4 sit at ReLU exactly 0
    x, y = _images(77, True, seed=505)
    _, lp, _ = _edge(p, x, y, geo)
    assert _same_bits(lp, lp[:1].expand(77, 10).contiguous())


def test_exact_logit_ties_go_to_the_lowest_index(dev, geo, params):
    """fc2 rows a < b identical with a dominant shared bias: every sample's top logits tie exactly at a and b.  Label a
    counts as correct, label b does not."""
    G, S = geo
    a, b = 2, 7
    p = E.tie_fc2(params, a, b)
    n = S * G + 5
    x, _ = _images(n, True, seed=606)
    y = torch.tensor([a, b, 0, a, b, 9])[torch.arange(n) % 6]
    res, lp, r64 = _edge(p, x, y, geo)
    assert bool((r64["margin"] == 0).all())
    assert _same_bits(lp[:, a].contiguous(), lp[:, b].contiguous())
    assert res[1] == int((y == a).sum())


def test_flat_fc2_gives_uniform_log_probs_and_class_0(dev, geo, params):
    p = params.clone()
    v = unpack_params(p)
    v["fc2.weight"].zero_()
    v["fc2.bias"].fill_(0.3)
    x, y = _images(45, True, seed=707)
    res, lp, r64 = _edge(p, x, y, geo)
    assert bool((lp == lp[:, :1]).all())
    assert torch.allclose(lp.double(), torch.full_like(lp, -math.log(10)).double(), rtol=0, atol=1e-6)
    assert res[1] == int((y == 0).sum())


def test_saturated_softmax(dev, geo, params):
    p = params.clone()
    v = unpack_params(p)
    v["fc2.weight"].mul_(1e3)
    v["fc2.bias"].mul_(1e3)
    x, y = _images(geo[0] * geo[1] + 5, True, seed=808)
    _, lp, r64 = _edge(p, x, y, geo)
    assert float(r64["zmax"].max()) > 100 and float(lp.min()) < -50


# --------------------------------------------------------------------------------------------- labels and refusals
def test_labels_outside_0_to_9_give_infinite_loss_and_count_only_valid_samples(dev, params):
    x, y = _images(37, True, seed=909)
    xd = x.to(dev)
    lp0 = torch.empty(37, 10, device=dev)
    res0 = convnet_evaluate(params, xd, y.to(dev), out_logp=lp0).tolist()
    lp0 = lp0.cpu()
    right = (lp0 == lp0.max(1, keepdim=True).values).sum(1).eq(1) & lp0.argmax(1).eq(y)
    bad_at = [0, 17, 36]
    for bad in (-1, 10, 2 ** 40):
        y2 = y.clone()
        y2[bad_at] = bad
        lp = torch.empty(37, 10, device=dev)
        res = convnet_evaluate(params, xd, y2.to(dev), out_logp=lp).tolist()
        assert res[0] == math.inf, (bad, res)
        assert res[1] == res0[1] - int(right[bad_at].sum()) and res[2] == 37, (bad, res, res0)
        assert _same_bits(lp.cpu(), lp0)
        with pytest.raises(ValueError, match=r"\[0, 10\)"):
            Evaluator(dev).run(params, TensorImageDataset(x, y2))


def test_exact_npar_params_and_alignment_refusals(dev, params):
    C = _ext.C()
    for u8 in (True, False):
        x, y = _images(45, u8, seed=111)
        xd, yd = x.to(dev), y.to(dev)
        want, want_lp = run(params, xd, yd)
        got, got_lp = run(params[:C.convnet_npar()].clone(), xd, yd)
        assert torch.equal(got, want) and _same_bits(got_lp, want_lp)
        slots = torch.zeros(C.convnet_eval_slot_words(dev.index), dtype=torch.int32, device=dev)
        result = torch.zeros(3, dtype=torch.float64, device=dev)
        buf = torch.empty(xd.numel() + 16, dtype=xd.dtype, device=dev)
        xm = buf[1:1 + xd.numel()].view(xd.shape)
        xm.copy_(xd)
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            C.convnet_eval(params, xm, yd, result, slots, MNIST_MEAN, MNIST_STD, None)
        pbuf = torch.zeros(params.numel() + 4, device=dev)
        pm = pbuf[1:1 + params.numel()]
        pm.copy_(params)
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            C.convnet_eval(pm, xd, yd, result, slots, MNIST_MEAN, MNIST_STD, None)
        assert int(slots[0]) == 0
        lp = torch.empty(45, 10, device=dev)
        assert torch.equal(convnet_evaluate(params, xm, yd, out_logp=lp).cpu(), want)
        assert _same_bits(lp.cpu(), want_lp)


# ------------------------------------------------------------------------------------------------------------ sharding
def test_sharding_over_emulated_ranks(dev, geo, params):
    """Each rank's eval_shard_range slice through convnet_evaluate, worlds 1 .. 8: its rows are the whole set's rows bit
    for bit, the counts add up exactly, the shard sums stay within the sum rule, and an empty shard launches nothing."""
    G, S = geo
    Ns = [0, 1, 7, 1001, S * G + 5]
    x, y = _images(max(Ns), True, seed=121)
    xd, yd = x.to(dev), y.to(dev)
    for N in Ns:
        whole, whole_lp = run(params, xd[:N], yd[:N])
        nll = -whole_lp.double().gather(1, y[:N, None])[:, 0]
        for world in range(1, 9):
            correct, n, loss, tol = 0.0, 0.0, 0.0, 0.0
            for rank in range(world):
                lo, hi = eval_shard_range(N, rank, world)
                lp = torch.empty(hi - lo, 10, device=dev)
                res = convnet_evaluate(params, xd[lo:hi], yd[lo:hi], out_logp=lp).cpu()
                if hi == lo:
                    assert res.tolist() == [0.0, 0.0, 0.0]
                    run(params, xd[lo:hi], yd[lo:hi])          # asserts that no slot word was touched
                    continue
                assert _same_bits(lp.cpu(), whole_lp[lo:hi]), (N, world, rank)
                correct, n, loss = correct + float(res[1]), n + float(res[2]), loss + float(res[0])
                k = int(E.schedule(hi - lo, G, S)["samples"].max())
                tol += k * 2.0 ** -24 * float(nll[lo:hi].abs().sum())
            assert correct == float(whole[1]) and n == N, (N, world, correct, n, whole.tolist())
            own = math.fsum(nll.tolist())
            assert abs(loss - own) <= tol, (N, world, loss, own, tol)


def test_evaluate_over_three_gloo_processes_sharing_one_gpu():
    """Evaluator.run -> _group_sum with three ranks on cuda:0, N = 10 and N = 2 (one rank's shard is empty)."""
    b2.launch(W.w_evaluate_cuda_net_gloo, size=3, backend="gloo", join_timeout_s=600)


@pytest.mark.multigpu
def test_evaluate_on_cuda1_with_cuda0_current():
    """The kernel's shared-memory opt-in and occupancy are set up on the device evaluated on, not the current one."""
    b2.launch(W.w_evaluate_on_second_gpu, size=1, backend="gloo", join_timeout_s=600)
