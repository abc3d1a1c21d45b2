"""Rounding-exact model of FlatLAMB's and FlatLARS's kernels (csrc/layerwise.cu), the fp64 references of both optimizers,
and the torch-op path ``FlatLAMB`` / ``FlatLARS`` run on CPU tensors and bf16 buckets; shared by tests/test_layerwise_model.py,
the CPU tier (tests/layerwise_workers.py) and the GPU tier (tests/test_gpu_layerwise.py).

A bucket is a flat fp32 tensor with tensors at ``offsets`` (multiples of 4) of ``numels`` elements.  The model follows the
kernels: the chunk table (each tensor cut into chunks of at most CHUNK elements), per chunk each of THREADS threads sums
its float4 vectors (i = thread, thread + THREADS, ...) and then its tail element with one-rounding fmaf in fp32, the warps
add by xor butterflies and thread 0 adds the warps in order in fp32; the chunk partials of a tensor are added in chunk order
in fp64, the roots taken in fp64 and the ratio rounded once to fp32.  ``fault`` plants one defect a kernel could have.
"""
import math

import torch

from adamw_model import clip_coef, f32, sqrt32  # noqa: F401 - clip_coef is used by the tests through this module
from sgd_options_model import fma32

CHUNK = 16384
THREADS = 256
FAULTS_LAMB = ("ratio_inverted", "bucket_norm", "decay_on_excluded", "decay_outside_u", "bias_correction_off_by_one",
               "chunk_crosses_tensor")
FAULTS_LARS = ("ratio_inverted", "bucket_norm", "decay_on_excluded", "chunk_crosses_tensor", "no_eps", "no_wd_norm")


def chunk_table(offsets, numels, chunk=CHUNK, fault=None):
    """[(start, length, tensor)] in table order.  The fault ``chunk_crosses_tensor`` cuts the whole laid-out range instead,
    each chunk counted to the tensor its first element belongs to."""
    if fault == "chunk_crosses_tensor":
        end = offsets[-1] + numels[-1]
        out = []
        for s in range(0, end, chunk):
            t = max(i for i, o in enumerate(offsets) if o <= s)
            out.append((s, min(chunk, end - s), t))
        return out
    return [(o + s, min(chunk, k - s), t) for t, (o, k) in enumerate(zip(offsets, numels)) for s in range(0, k, chunk)]


def chunk_sqsum(x: torch.Tensor) -> float:
    """The fp32 partial of one chunk's values ``x`` (sum of squares, the kernel's order), as a Python float."""
    n = x.numel()
    nv, tail = n // 4, n % 4
    iters = (nv + THREADS - 1) // THREADS
    body = torch.zeros(iters * THREADS * 4)
    body[:nv * 4] = x[:nv * 4]
    body = body.view(iters, THREADS, 4)              # zero padding: fmaf(0, 0, s) == s
    s = torch.zeros(THREADS)
    for it in range(iters):
        for e in range(4):
            s = fma32(body[it, :, e], body[it, :, e], s)
    if tail:
        xt = x[nv * 4:]
        s[:tail] = fma32(xt, xt, s[:tail])
    w = s.view(THREADS // 32, 32)
    lane = torch.arange(32)
    for d in (16, 8, 4, 2, 1):
        w = w + w[:, lane ^ d]
    tot = torch.zeros((), dtype=torch.float32)
    for k in range(THREADS // 32):
        tot = tot + w[k, 0]
    return float(tot)


def tensor_sums(a: torch.Tensor, b: torch.Tensor, table, n_tensors: int, fault=None):
    """Per tensor the fp64 sums of the chunk partials of a^2 and b^2, in chunk order."""
    sa, sb = [0.0] * n_tensors, [0.0] * n_tensors
    for start, ln, t in table:
        sa[t] += chunk_sqsum(a[start:start + ln])
        sb[t] += chunk_sqsum(b[start:start + ln])
    if fault == "bucket_norm":
        sa, sb = [sum(sa)] * n_tensors, [sum(sb)] * n_tensors
    return sa, sb


def _segments(offsets, numels):
    return [slice(o, o + k) for o, k in zip(offsets, numels)]


def lamb_step(p, g, m, v, offsets, numels, adapt, hp, t, coef=None, fault=None, chunk=CHUNK):
    """(p, m, v, ratios) after LAMB update ``t`` of the bucket; ``hp``: lr, betas, eps, weight_decay."""
    p, g, m, v = (x.float().cpu().clone() for x in (p, g, m, v))
    if coef is not None:
        g = g * torch.tensor(coef, dtype=torch.float32)
    b1, b2 = hp["betas"]
    tb = t + 1 if fault == "bias_correction_off_by_one" else t
    w1, beta2, c2, sbc2, eps, rbc1, lr, wd = (f32(x) for x in (1 - b1, b2, 1 - b2, (1 - b2 ** tb) ** 0.5, hp["eps"],
                                                                1 / (1 - b1 ** tb), hp["lr"], hp["weight_decay"]))
    segs = _segments(offsets, numels)
    u = torch.zeros_like(p)
    for i, s in enumerate(segs):
        wd_l = wd if adapt[i] or fault == "decay_on_excluded" else 0.0
        if fault == "decay_outside_u":
            wd_l = 0.0
        d = g[s] - m[s]
        m[s] = fma32(w1, d, m[s]) if w1 < 0.5 else fma32(-d, f32(1.0 - w1), g[s])
        v[s] = fma32(torch.tensor(c2) * g[s], g[s], v[s] * torch.tensor(beta2))
        den = sqrt32(v[s]) / torch.tensor(sbc2) + torch.tensor(eps)
        u[s] = fma32(wd_l, p[s], (m[s] / den) * torch.tensor(rbc1))
    table = chunk_table(offsets, numels, chunk, fault)
    sp, su = tensor_sums(p, u, table, len(segs), fault)
    ratios = []
    for i, s in enumerate(segs):
        W, U = math.sqrt(sp[i]), math.sqrt(su[i])
        r = 1.0
        if adapt[i] and W > 0.0 and U > 0.0:
            r = f32(U / W) if fault == "ratio_inverted" else f32(W / U)
        ratios.append(r)
        q = p[s]
        if fault == "decay_outside_u" and adapt[i]:
            q = q * torch.tensor(f32(1.0 - hp["lr"] * hp["weight_decay"]))
        p[s] = fma32(-(torch.tensor(lr) * torch.tensor(r)), u[s], q)
    return p, m, v, ratios


def lars_step(p, g, mom, offsets, numels, adapt, hp, coef=None, fault=None, chunk=CHUNK):
    """(p, momentum, ratios) after one LARS update; ``hp``: lr, momentum, weight_decay, trust_coefficient, eps, nesterov."""
    p, g, mom = (x.float().cpu().clone() for x in (p, g, mom))
    if coef is not None:
        g = g * torch.tensor(coef, dtype=torch.float32)
    lr, mu, wd32 = f32(hp["lr"]), f32(hp["momentum"]), f32(hp["weight_decay"])
    eta, wd, eps = hp["trust_coefficient"], hp["weight_decay"], hp["eps"]
    segs = _segments(offsets, numels)
    table = chunk_table(offsets, numels, chunk, fault)
    sp, sg = tensor_sums(p, g, table, len(segs), fault)
    ratios = []
    for i, s in enumerate(segs):
        W, G = math.sqrt(sp[i]), math.sqrt(sg[i])
        r = 1.0
        if adapt[i] and W > 0.0 and G > 0.0:
            den = (G + (0.0 if fault == "no_wd_norm" else wd * W)) + (0.0 if fault == "no_eps" else eps)
            r = f32(den / (eta * W)) if fault == "ratio_inverted" else f32((eta * W) / den)
        ratios.append(r)
        wd_l = wd32 if adapt[i] or fault == "decay_on_excluded" else 0.0
        d = torch.tensor(r) * fma32(wd_l, p[s], g[s])
        mom[s] = fma32(mu, mom[s], d)
        p[s] = fma32(-lr, fma32(mu, mom[s], d) if hp["nesterov"] else mom[s], p[s])
    return p, mom, ratios


# ----------------------------------------------------------------------------------------------- the torch-op path
def _norm64(x):
    return float(torch.linalg.vector_norm(x, dtype=torch.float64))


def torch_lamb_tensor(p, g, m, v, adapt, hp, t):
    """FlatLAMB's torch-op update of one tensor in place (update t); returns its ratio."""
    b1, b2 = hp["betas"]
    m.lerp_(g, 1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    u = (m / (v.sqrt() / (1 - b2 ** t) ** 0.5).add_(hp["eps"])).mul_(1 / (1 - b1 ** t))
    if adapt and hp["weight_decay"] != 0.0:
        u.add_(p, alpha=hp["weight_decay"])
    r = 1.0
    if adapt:
        wn, un = _norm64(p), _norm64(u)
        if wn > 0.0 and un > 0.0:
            r = f32(wn / un)
    p.add_(u, alpha=-f32(f32(hp["lr"]) * r))
    return r


def torch_lars_ratio(p, g, adapt, hp):
    """FlatLARS's torch-op ratio of one tensor."""
    if not adapt:
        return 1.0
    wn, gn = _norm64(p), _norm64(g)
    if wn > 0.0 and gn > 0.0:
        return f32(hp["trust_coefficient"] * wn / (gn + hp["weight_decay"] * wn + hp["eps"]))
    return 1.0


def torch_lars_direction(p, g, adapt, hp, r):
    """d = r * (g + wd_l * p) as FlatLARS's torch-op path forms it."""
    d = g.add(p, alpha=hp["weight_decay"]) if adapt and hp["weight_decay"] != 0.0 else g.clone()
    if r != 1.0:
        d.mul_(r)
    return d


def torch_sgd(p, d, m, hp):
    """torch.optim.SGD(foreach=False)'s update of one tensor on the direction ``d`` (momentum buffer ``m``, in place)."""
    from torch.optim.sgd import sgd

    sgd([p], [d], [m], foreach=False, weight_decay=0.0, momentum=hp["momentum"], lr=hp["lr"], dampening=0.0,
        nesterov=hp["nesterov"], maximize=False)


# ----------------------------------------------------------------------------------------------- fp64 references
def lamb_fp64(p0, grads, offsets, numels, adapt, hp):
    """LAMB in fp64 over the gradient sequence (the bucket's tensors only)."""
    b1, b2 = hp["betas"]
    out = p0.double().clone()
    for s, ad in zip(_segments(offsets, numels), adapt):
        p, m, v = out[s].clone(), torch.zeros(s.stop - s.start, dtype=torch.float64), torch.zeros(s.stop - s.start, dtype=torch.float64)
        wd = hp["weight_decay"] if ad else 0.0
        for t, g in enumerate(grads, 1):
            gg = g[s].double()
            m = b1 * m + (1 - b1) * gg
            v = b2 * v + (1 - b2) * gg * gg
            u = (m / (v.sqrt() / math.sqrt(1 - b2 ** t) + hp["eps"])) / (1 - b1 ** t) + wd * p
            W, U = float(p.norm()), float(u.norm())
            r = W / U if ad and W > 0 and U > 0 else 1.0
            p = p - hp["lr"] * r * u
        out[s] = p
    return out


def lars_fp64(p0, grads, offsets, numels, adapt, hp):
    """LARS in fp64 over the gradient sequence (the bucket's tensors only)."""
    out = p0.double().clone()
    mu = hp["momentum"]
    for s, ad in zip(_segments(offsets, numels), adapt):
        p, m = out[s].clone(), torch.zeros(s.stop - s.start, dtype=torch.float64)
        wd = hp["weight_decay"] if ad else 0.0
        for g in grads:
            gg = g[s].double()
            W, G = float(p.norm()), float(gg.norm())
            r = hp["trust_coefficient"] * W / (G + wd * W + hp["eps"]) if ad and W > 0 and G > 0 else 1.0
            d = r * (gg + wd * p)
            m = mu * m + d
            p = p - hp["lr"] * (d + mu * m if hp["nesterov"] else m)
        out[s] = p
    return out
