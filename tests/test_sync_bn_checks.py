"""CPU checks of the SyncBatchNorm test helpers (tests/sync_bn_checks.py).

* The fp64 reference equals torch's fp64 ``F.batch_norm`` and its autograd for every weight / bias / running-stat /
  momentum configuration, ``momentum=None`` included.
* The kernels' numerics, as the CPU path of ``SyncBatchNormFunction`` computes them (fp64 sums, coefficients rounded once
  to fp32, outputs in the input's dtype, parameters and running stats each in their own dtype), pass every bound.
* Each of the faults below, planted in fp64 reference outputs rounded as a kernel would round them, misses a bound by at
  least 10x: a biased running var, ``momentum=None`` taken as 0 or as 0.1, a missing weight taken as 1, a bias ignored,
  ``dx`` without its ``sum dy / N`` or its ``(x - mean) sum dy (x - mean)`` term, running stats stored in the parameters'
  dtype, ``grad_weight`` without ``invstd``, and one channel's statistics swapped with its neighbour's.
"""
import pytest
import torch
import torch.nn.functional as F

import sync_bn_checks as S
from dist_tuto.pth_b200.parallel.sync_bn import SyncBatchNormFunction

DT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _data(shape=(16, 6, 5), dtype=torch.float32, pdtype=torch.float32, rdtype=torch.float32, seed=0):
    """Channels with distinct means, std 2 (invstd far from 1), dy with a nonzero mean, weights far from 1 and biases far
    from 0, so that every term of the forward and backward is visible."""
    g = torch.Generator().manual_seed(seed)
    C = shape[1]
    off = torch.linspace(-1.0, 1.0, C).view([1, C] + [1] * (len(shape) - 2))
    x = (torch.randn(shape, generator=g, dtype=torch.float64) * 2 + off).to(dtype)
    dy = (torch.randn(shape, generator=g, dtype=torch.float64) + 0.5).to(dtype)
    w = (torch.rand(C, generator=g, dtype=torch.float64) + 1.5).to(pdtype)
    sign = torch.tensor([1.0, -1.0], dtype=torch.float64).repeat(C)[:C]
    b = ((torch.rand(C, generator=g, dtype=torch.float64) * 0.5 + 0.25) * sign).to(pdtype)
    rm = torch.rand(C, generator=g, dtype=torch.float64).to(rdtype)
    rv = (torch.rand(C, generator=g, dtype=torch.float64) + 0.5).to(rdtype)
    return x, dy, w, b, rm, rv


@pytest.mark.parametrize("affine", [(True, True), (True, False), (False, True), (False, False)],
                         ids=["w+b", "w", "b", "none"])
@pytest.mark.parametrize("momentum", [0.1, None])
@pytest.mark.parametrize("track", [True, False])
def test_reference_is_torch_fp64_batch_norm(affine, momentum, track):
    x, dy, w, b, rm, rv = _data()
    w = w if affine[0] else None
    b = b if affine[1] else None
    rm, rv = (rm.double(), rv.double()) if track else (None, None)
    nbt = 3
    fwd = S.forward_ref(x, w, b, rm, rv, momentum, nbt)
    xr = x.double().clone().requires_grad_(True)
    wr = None if w is None else w.double().clone().requires_grad_(True)
    br = None if b is None else b.double().clone().requires_grad_(True)
    rmr, rvr = (None, None) if rm is None else (rm.clone(), rv.clone())
    yr = F.batch_norm(xr, rmr, rvr, wr, br, True, 1.0 / nbt if momentum is None else momentum, 1e-5)
    torch.testing.assert_close(fwd["y"], yr.detach(), rtol=1e-12, atol=1e-12)
    if track:
        torch.testing.assert_close(fwd["rm"], rmr, rtol=1e-14, atol=1e-14)
        torch.testing.assert_close(fwd["rv"], rvr, rtol=1e-14, atol=1e-14)
    else:
        assert fwd["rm"] is None and fwd["rv"] is None
    bwd = S.backward_ref(x, dy, fwd, w)
    grads = torch.autograd.grad(yr, [t for t in (xr, wr, br) if t is not None], dy.double())
    torch.testing.assert_close(bwd["dx"], grads[0], rtol=1e-10, atol=1e-12)
    k = 1
    if wr is not None:
        torch.testing.assert_close(bwd["gw"], grads[k], rtol=1e-12, atol=1e-12)
        k += 1
    if br is not None:
        torch.testing.assert_close(bwd["gb"], grads[k], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("dtype,pdtype,rdtype", [("fp32", "fp32", "fp32"), ("bf16", "fp32", "fp32"),
                                                 ("bf16", "bf16", "fp32"), ("bf16", "fp32", "bf16"),
                                                 ("fp16", "fp16", "fp32"), ("fp16", "fp32", "fp16"),
                                                 ("fp16", "fp16", "fp16")])
@pytest.mark.parametrize("shape", [(16, 6, 5), (9, 5), (4, 3, 2, 3)])
def test_kernel_numerics_on_cpu_pass_every_bound(dtype, pdtype, rdtype, shape):
    dt, pd, rd = DT[dtype], DT[pdtype], DT[rdtype]
    for affine, track, momentum in ((True, True, 0.1), (False, True, None), (True, False, 0.1), (False, False, None)):
        x, dy, w, b, rm0, rv0 = _data(shape, dt, pd, rd, seed=len(shape))
        w = w.clone().requires_grad_(True) if affine else None
        b = b.clone().requires_grad_(True) if affine else None
        rm, rv = (rm0.clone(), rv0.clone()) if track else (None, None)
        nbt = torch.tensor(4) if momentum is None and track else None
        xr = x.clone().requires_grad_(True)
        y = SyncBatchNormFunction.apply(xr, w, b, rm, rv, nbt, 0.0 if momentum is None else momentum, 1e-5, None, None)
        stats = y.grad_fn.saved_tensors[2]
        C = shape[1]
        fwd = S.forward_ref(x, w, b, rm0 if track else None, rv0 if track else None, momentum, 4)
        got = dict(y=y, mean=stats[:C], invstd=stats[C:2 * C], rm=rm, rv=rv)
        ratios = S.forward_checks(got, x, fwd, dt, rd)
        grads = torch.autograd.grad(y, [t for t in (xr, w, b) if t is not None], dy)
        bwd = S.backward_ref(x, dy, fwd, w)
        gotb = dict(dx=grads[0], gw=grads[1] if affine else None, gb=grads[2] if affine else None)
        ratios.update(S.backward_checks(gotb, x, dy, fwd, bwd, dt, pd))
        assert not S.failures(ratios), (affine, track, momentum, ratios)


# ------------------------------------------------------------------------------------------------------ planted faults
DTYPE, PDTYPE, RDTYPE = torch.bfloat16, torch.bfloat16, torch.float32
NBT = 3                                               # momentum=None: factor 1/3


def _case():
    x, dy, w, b, rm0, rv0 = _data((24, 6, 7), DTYPE, PDTYPE, RDTYPE, seed=11)
    fwd = S.forward_ref(x, w, b, rm0, rv0, None, NBT)
    bwd = S.backward_ref(x, dy, fwd, w)
    return dict(x=x, dy=dy, w=w, b=b, rm0=rm0, rv0=rv0, fwd=fwd, bwd=bwd)


def _outputs(fwd, bwd):
    """What a correct kernel writes: fp64 statistics, y / dx in the input's dtype, gradients in the parameters' dtype and
    running stats in their own."""
    return dict(y=fwd["y"].to(DTYPE), mean=fwd["mean"], invstd=fwd["invstd"], rm=fwd["rm"].to(RDTYPE),
                rv=fwd["rv"].to(RDTYPE), dx=bwd["dx"].to(DTYPE), gw=bwd["gw"].to(PDTYPE), gb=bwd["gb"].to(PDTYPE))


def _ratios(c, out):
    r = S.forward_checks({k: out[k] for k in ("y", "mean", "invstd", "rm", "rv")}, c["x"], c["fwd"], DTYPE, RDTYPE)
    r.update(S.backward_checks({k: out[k] for k in ("dx", "gw", "gb")}, c["x"], c["dy"], c["fwd"], c["bwd"], DTYPE, PDTYPE))
    return r


def _swap(v, i):
    v = v.clone()
    v[[i, i + 1]] = v[[i + 1, i]]
    return v


def _fault(name, c):
    fwd, bwd, x, dy = c["fwd"], c["bwd"], c["x"], c["dy"]
    out = _outputs(fwd, bwd)
    m = 1.0 / NBT
    N = fwd["N"]
    if name == "biased running var":
        out["rv"] = ((1 - m) * c["rv0"].double() + m * fwd["var"]).to(RDTYPE)
    elif name == "momentum None as 0":
        out["rm"], out["rv"] = c["rm0"].clone(), c["rv0"].clone()
    elif name == "momentum None as 0.1":
        f = S.forward_ref(x, c["w"], c["b"], c["rm0"], c["rv0"], 0.1)
        out["rm"], out["rv"] = f["rm"].to(RDTYPE), f["rv"].to(RDTYPE)
    elif name == "missing weight as 1":
        f = S.forward_ref(x, None, c["b"], c["rm0"], c["rv0"], None, NBT)
        out["y"], out["dx"] = f["y"].to(DTYPE), S.backward_ref(x, dy, f, None)["dx"].to(DTYPE)
    elif name == "bias ignored":
        out["y"] = S.forward_ref(x, c["w"], None)["y"].to(DTYPE)
    elif name == "dx without sum dy / N":
        kc = -bwd["kb"] * fwd["mean"]
        out["dx"] = (dy.double() * S.bview(x, bwd["ka"]) + x.double() * S.bview(x, bwd["kb"]) + S.bview(x, kc)).to(DTYPE)
    elif name == "dx without the (x - mean) term":
        out["dx"] = (dy.double() * S.bview(x, bwd["ka"]) + S.bview(x, -bwd["ka"] * bwd["sdy"] / N)).to(DTYPE)
    elif name == "running stats in the parameter dtype":
        out["rm"], out["rv"] = fwd["rm"].to(PDTYPE).to(RDTYPE), fwd["rv"].to(PDTYPE).to(RDTYPE)
    elif name == "grad_weight without invstd":
        out["gw"] = bwd["sdx"].to(PDTYPE)
    elif name == "neighbouring channels' statistics swapped":
        f = dict(fwd)
        for k in ("mean", "var", "invstd"):
            f[k] = _swap(fwd[k], 2)
        f["k1"] = c["w"].double() * f["invstd"]
        f["k0"] = c["b"].double() - f["mean"] * f["k1"]
        out["mean"], out["invstd"] = f["mean"], f["invstd"]
        out["y"] = (x.double() * S.bview(x, f["k1"]) + S.bview(x, f["k0"])).to(DTYPE)
        out["rm"] = ((1 - m) * c["rm0"].double() + m * f["mean"]).to(RDTYPE)
        out["rv"] = ((1 - m) * c["rv0"].double() + m * f["var"] * N / (N - 1)).to(RDTYPE)
        out["dx"] = S.backward_ref(x, dy, f, c["w"])["dx"].to(DTYPE)
    else:
        raise KeyError(name)
    return out


FAULTS = ["biased running var", "momentum None as 0", "momentum None as 0.1", "missing weight as 1", "bias ignored",
          "dx without sum dy / N", "dx without the (x - mean) term", "running stats in the parameter dtype",
          "grad_weight without invstd", "neighbouring channels' statistics swapped"]


def test_correct_outputs_pass():
    c = _case()
    ratios = _ratios(c, _outputs(c["fwd"], c["bwd"]))
    assert not S.failures(ratios), ratios


@pytest.mark.parametrize("name", FAULTS)
def test_planted_fault_is_caught(name):
    c = _case()
    ratios = _ratios(c, _fault(name, c))
    caught = S.failures(ratios)
    print(f"{name}: caught by {caught}, worst ratio {max(ratios.values()):.3g}")
    assert caught, (name, ratios)
    assert max(ratios.values()) >= 10.0, (name, ratios)
