"""fp64 reference and error bounds of the SyncBatchNorm kernels (csrc/batchnorm.cu), shared by tests/test_gpu_sync_bn.py and
tests/test_gpu_sync_bn_configs.py, and shown to catch planted faults by tests/test_sync_bn_checks.py (CPU).

The kernels compute the statistics in fp64 and round each per-channel coefficient once to fp32, so against the fp64
reference of the same operation:

* ``y = fmaf(x, k1, k0)``: ``|y - y64| <= C_BOUND 2^-24 (|x k1| + |k0|)`` plus the output's rounding (``OUT_EPS |y64|``)
  and its subnormal spacing (``OUT_SUB``);
* ``dx = fmaf(dy, ka, fmaf(x, kb, kc))``: the same form over ``|dy ka| + |x kb| + |kc|``, plus ``2^-22 |kb mean|`` for the
  cancellation inside ``kc``;
* mean within ``1e-12`` and invstd within ``rtol = 1e-9`` of fp64 (inputs within a few standard deviations of zero; the
  one-pass variance loses ``(mean / std)^2`` ulps, see DESIGN.md §4h);
* running stats, ``grad_weight`` and ``grad_bias`` rounded once from fp64 to their own dtype: ``PARAM_EPS`` of that dtype
  relative, and for the gradients ``1e-12`` of the sums' magnitude.

``weight=None`` / ``bias=None`` mean 1 / 0, ``running_mean=None`` means no running stats, and ``momentum=None`` takes the
factor ``1 / num_batches_tracked``.  Every check returns the worst ratio of error to bound (``<= 1`` passes; ``inf`` for a
NaN where the reference has none), so a test can also show by how much a planted fault misses.
"""
import torch

C_BOUND = 3.0
OUT_EPS = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
OUT_SUB = {dt: torch.finfo(dt).tiny * torch.finfo(dt).eps for dt in OUT_EPS}   # subnormal spacing of the output
PARAM_EPS = {torch.float32: 2.0 ** -23, torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}
MEAN_TOL = 1e-12
INVSTD_RTOL, INVSTD_ATOL = 1e-9, 1e-8


def dims(x):
    """The reduced dimensions: all but the channel dimension 1."""
    return [0] + list(range(2, x.dim()))


def bview(x, v):
    """A per-channel vector broadcast against x."""
    return v.view([1, -1] + [1] * (x.dim() - 2))


def _d(t):
    return None if t is None else t.detach().double().cpu()


def forward_ref(x, weight=None, bias=None, running_mean=None, running_var=None, momentum=0.1, nbt=None, eps=1e-5):
    """fp64 training forward of the global batch ``x``.  ``running_*`` are the values before the step; ``nbt`` is
    ``num_batches_tracked`` after its increment and gives the factor when ``momentum`` is None.  Returns fp64 CPU tensors:
    N, mean, var (biased), invstd, k1, k0, y and, when tracked, the new running_mean / running_var."""
    xd = _d(x)
    C = xd.shape[1]
    N = xd.numel() // C
    mean = xd.mean(dims(xd))
    var = xd.var(dims(xd), unbiased=False)
    invstd = 1.0 / torch.sqrt(var + eps)
    w = _d(weight) if weight is not None else torch.ones(C, dtype=torch.float64)
    b = _d(bias) if bias is not None else torch.zeros(C, dtype=torch.float64)
    k1 = w * invstd
    k0 = b - mean * k1
    out = dict(N=N, mean=mean, var=var, invstd=invstd, k1=k1, k0=k0, y=xd * bview(xd, k1) + bview(xd, k0), rm=None, rv=None)
    if running_mean is not None:
        m = 1.0 / float(nbt) if momentum is None else float(momentum)
        out["rm"] = (1.0 - m) * _d(running_mean) + m * mean
        out["rv"] = (1.0 - m) * _d(running_var) + m * (var * N / (N - 1.0))
    return out


def grad_sums(x, dy, mean, invstd):
    """fp64 per-channel ``sum dy`` (= grad_bias), ``sum dy (x - mean)``, grad_weight and the magnitude that bounds their
    summation error, over the rows of ``x`` / ``dy`` (one rank's local batch, or the global one)."""
    xd, dyd = _d(x), _d(dy)
    xmu = xd - bview(xd, mean)
    sdy, sdx = dyd.sum(dims(xd)), (dyd * xmu).sum(dims(xd))
    if xd.numel():
        scale = dyd.abs().sum(dims(xd)) * (1 + xmu.abs().amax(dims(xd)))
    else:
        scale = torch.zeros_like(mean)
    return dict(sdy=sdy, sdx=sdx, gb=sdy, gw=sdx * invstd, scale=scale)


def backward_ref(x, dy, fwd, weight=None):
    """fp64 input gradient of the global batch from ``forward_ref``'s statistics: the coefficients ka, kb, kc and dx."""
    xd, dyd = _d(x), _d(dy)
    C = xd.shape[1]
    s = grad_sums(xd, dyd, fwd["mean"], fwd["invstd"])
    w = _d(weight) if weight is not None else torch.ones(C, dtype=torch.float64)
    ka = w * fwd["invstd"]
    kb = -ka * fwd["invstd"] * fwd["invstd"] * s["sdx"] / fwd["N"]
    kc = -ka * s["sdy"] / fwd["N"] - kb * fwd["mean"]
    s.update(ka=ka, kb=kb, kc=kc, dx=dyd * bview(xd, ka) + xd * bview(xd, kb) + bview(xd, kc))
    return s


# ------------------------------------------------------------------------------------------------------------ bounds
def y_bound(x, fwd, dtype):
    xd, y = _d(x), fwd["y"]
    return (C_BOUND * 2.0 ** -24 * (xd.abs() * bview(xd, fwd["k1"].abs()) + bview(xd, fwd["k0"].abs()))
            + OUT_EPS[dtype] * y.abs() + OUT_SUB[dtype])


def dx_bound(x, dy, fwd, bwd, dtype):
    xd, dyd = _d(x), _d(dy)
    ka, kb, kc = (bview(xd, bwd[k]) for k in ("ka", "kb", "kc"))
    return (C_BOUND * 2.0 ** -24 * (dyd.abs() * ka.abs() + xd.abs() * kb.abs() + kc.abs())
            + OUT_EPS[dtype] * bwd["dx"].abs() + OUT_SUB[dtype] + 2.0 ** -22 * (kb * bview(xd, fwd["mean"])).abs())


def worst(got, ref, bound):
    """max |got - ref| / bound, with NaN matching NaN counted as exact and any other NaN as inf; 0 for empty tensors."""
    g = got.detach().double().cpu()
    ref = ref.double().cpu()
    if g.shape != ref.shape:
        return float("inf")
    if g.numel() == 0:
        return 0.0
    d = (g - ref).abs()
    r = d / bound
    exact = (d == 0) | (torch.isnan(g) & torch.isnan(ref))
    r = torch.where(exact, torch.zeros_like(r), r)
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    return float(r.max())


def check_y(y, x, fwd, dtype):
    return worst(y, fwd["y"], y_bound(x, fwd, dtype))


def check_dx(dx, x, dy, fwd, bwd, dtype):
    return worst(dx, bwd["dx"], dx_bound(x, dy, fwd, bwd, dtype))


def check_mean(mean, fwd):
    return worst(mean, fwd["mean"], MEAN_TOL + MEAN_TOL * fwd["mean"].abs())


def check_invstd(invstd, fwd):
    return worst(invstd, fwd["invstd"], INVSTD_ATOL + INVSTD_RTOL * fwd["invstd"].abs())


def check_running(got, ref, rdtype):
    """A running stat rounded once from fp64 to its own dtype ``rdtype``."""
    pe = PARAM_EPS[rdtype]
    return worst(got, ref, pe + pe * ref.abs())


def check_grad_bias(gb, sums, pdtype):
    return worst(gb, sums["gb"], PARAM_EPS[pdtype] * sums["gb"].abs() + 1e-12 * sums["scale"])


def check_grad_weight(gw, sums, invstd, pdtype):
    return worst(gw, sums["gw"], PARAM_EPS[pdtype] * sums["gw"].abs() + 1e-12 * sums["scale"] * invstd)


def forward_checks(got, x, fwd, dtype, rdtype=torch.float32):
    """Worst ratios of every forward output present in ``got`` (keys y, mean, invstd, rm, rv)."""
    out = {}
    if "y" in got:
        out["y"] = check_y(got["y"], x, fwd, dtype)
    if "mean" in got:
        out["mean"] = check_mean(got["mean"], fwd)
    if "invstd" in got:
        out["invstd"] = check_invstd(got["invstd"], fwd)
    for k in ("rm", "rv"):
        if got.get(k) is not None or fwd[k] is not None:
            out[k] = float("inf") if got.get(k) is None or fwd[k] is None else check_running(got[k], fwd[k], rdtype)
    return out


def backward_checks(got, x, dy, fwd, bwd, dtype, pdtype=torch.float32, local=None):
    """Worst ratios of dx, grad_weight and grad_bias in ``got``; ``local``: the ``grad_sums`` the gradients of the
    parameters are checked against (default: the global batch's)."""
    sums = bwd if local is None else local
    out = {}
    if got.get("dx") is not None:
        out["dx"] = check_dx(got["dx"], x, dy, fwd, bwd, dtype)
    if got.get("gw") is not None:
        out["gw"] = check_grad_weight(got["gw"], sums, fwd["invstd"], pdtype)
    if got.get("gb") is not None:
        out["gb"] = check_grad_bias(got["gb"], sums, pdtype)
    return out


def failures(ratios):
    """The names of the checks whose error exceeds the bound."""
    return sorted(k for k, v in ratios.items() if not v <= 1.0)
