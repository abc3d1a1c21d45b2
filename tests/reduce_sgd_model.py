"""Rounding-exact model of the one-GPU optimizer kernel ``reduce_sgd_kernel`` (csrc/sgd.cu) and its fixed-order reduction
``reduce_local_grad`` / ``reduce_loss`` (csrc/convnet_reduce.cuh), and of ``det_reduce_kernel`` (csrc/sgd.cu).

* ``local_grad``: the fp32 local gradient, every sum in the kernel's order.  fc1.weight: per pass of RKC samples, sample
  group ks chains ``fmaf`` over the pass's samples ks, ks + RKS, ... from 0; the RKS group partials are added to the tile
  total in group order, and the total carries across passes.  The other vectors: slot group sg adds slots sg, sg + RSS, ...
  from 0, and the total is part[0] + part[1] + ... + part[RSS - 1].  The gradient does not depend on the grid.
* ``loss_terms``: lane l sums the loss words of slots l, l + 32, ..., then an xor butterfly (d = 16 .. 1) runs per word.
* ``update`` / ``aux_after`` / ``bucket_after``: the update of sgd_options_model / grad_clip_model, conv2.weight's two
  pre-arranged copies, and the gradient bucket after the kernel re-zeroed the other step parity.
* ``clip_norm``: the clip instance's pre-clip norm, which does depend on the grid: each thread chains ``fmaf`` over the
  squares of its vectors in unit order (unit u runs on CTA u % n_cta), a warp butterfly, the 16 warps in fp32, the CTA
  partials in fp64 in CTA order, the root in fp64 rounded once.
* ``det_reduce``: the slots added in slot order, per element and for the two loss words.
* ``fp64_bound``: kept apart from the model, the fp64 sums and the error bound of any plain-fp32 evaluation of them, so
  that a model wrong in the same way as the kernel still fails.
* ``sizes(S)`` / ``grids()`` / ``gaps()``: the sample counts, slot counts and grids where the kernel's loops change shape.

The constants are read from the kernel headers (``constants()``), so a change to the tiling moves the model with it.
"""
import math
import os
import re

import numpy as np
import torch

import grad_clip_model as GM
import sgd_options_model as SM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dist_tuto.pth_b200", "csrc")
U32 = 2.0 ** -24                       # unit roundoff of fp32


# ---------------------------------------------------------------------------------------------------------- constants
def _need(pattern, text, where):
    m = re.search(pattern, text)
    if m is None:
        raise ValueError(f"{pattern!r} not found in {where}")
    return [int(g) for g in m.groups()]


def parse_constants(reduce_src: str, args_src: str) -> dict:
    """The reduction's constants from the texts of convnet_reduce.cuh and convnet_args.cuh, and the ones the header derives
    from them.  A pattern that is not found raises ValueError."""
    (red_t,) = _need(r"constexpr int RED_T = (\d+);", reduce_src, "convnet_reduce.cuh")
    rj, ri, rv, rkc = _need(r"constexpr int RJ = (\d+), RI = (\d+), RV = (\d+), RKC = (\d+);", reduce_src, "convnet_reduce.cuh")
    (npar,) = _need(r"constexpr int NPAR = (\d+);", args_src, "convnet_args.cuh")
    (w3,) = _need(r"\bW3 = (\d+),", args_src, "convnet_args.cuh")
    (det_stride,) = _need(r"constexpr int DET_STRIDE = (\d+);", args_src, "convnet_args.cuh")
    fac_stride, fac_p2 = _need(r"constexpr int FAC_STRIDE = (\d+), FAC_P2 = (\d+);", args_src, "convnet_args.cuh")
    tile_vec = rj * ri // 4
    k = dict(RED_T=red_t, RJ=rj, RI=ri, RV=rv, RKC=rkc, NPAR=npar, W3=w3, DET_STRIDE=det_stride, FAC_STRIDE=fac_stride,
             FAC_P2=fac_p2, RED_TILE_VEC=tile_vec)
    k["RKS"] = red_t // tile_vec
    k["RSS"] = red_t // rv
    k["RSLOT_BATCH"] = (rkc + k["RSS"] - 1) // k["RSS"]
    k["RED_FC1_TILES"] = (50 // rj) * (320 // ri)
    k["RED_OTHER"] = (npar - 16000) // 4
    k["RED_UNITS"] = k["RED_FC1_TILES"] + (k["RED_OTHER"] + rv - 1) // rv
    return k


def constants() -> dict:
    with open(os.path.join(CSRC, "convnet_reduce.cuh")) as f:
        red = f.read()
    with open(os.path.join(CSRC, "convnet_args.cuh")) as f:
        args = f.read()
    return parse_constants(red, args)


K = constants()
NPAR, W3, DET_STRIDE, FAC_STRIDE, FAC_P2 = K["NPAR"], K["W3"], K["DET_STRIDE"], K["FAC_STRIDE"], K["FAC_P2"]
RKC, RKS, RSS, RV, RJ, RI = K["RKC"], K["RKS"], K["RSS"], K["RV"], K["RJ"], K["RI"]
RED_FC1_TILES, RED_OTHER, RED_UNITS, RSLOT_BATCH = K["RED_FC1_TILES"], K["RED_OTHER"], K["RED_UNITS"], K["RSLOT_BATCH"]
FC1 = 50 * 320
OTHER = torch.cat([torch.arange(0, W3), torch.arange(W3 + FC1, NPAR)])     # flat elements outside fc1.weight


# ---------------------------------------------------------------------------------------------------------- the sums
def fc1_grad(factors: torch.Tensor, n_samples: int, rkc: int = RKC, stride: int = RKS, group_order=None) -> torch.Tensor:
    """fc1.weight's gradient [50, 320] in the kernel's order.  ``rkc`` (samples per pass), ``stride`` (sample step of a
    group) and ``group_order`` (the order the group partials are added) are the kernel's unless a test plants a fault."""
    f = factors[:n_samples].float()
    dh, p2 = f[:, :50], f[:, FAC_P2:FAC_P2 + 320]
    order = range(RKS) if group_order is None else group_order
    total = torch.zeros(50, 320)
    for k0 in range(0, max(n_samples, 1), rkc):
        kn = min(rkc, n_samples - k0)
        acc = torch.zeros(RKS, 50, 320)
        for i in range((rkc + RKS - 1) // RKS):
            k = torch.arange(RKS) + i * stride
            live = k < kn
            if not bool(live.any()):
                break
            kk = k0 + k[live]
            acc[live] = SM.fma32(dh[kk][:, :, None], p2[kk][:, None, :], acc[live])
        for g in order:
            total = total + acc[g]
    return total


def other_grad(slots: torch.Tensor, n_slots: int, rss: int = RSS) -> torch.Tensor:
    """The gradient outside fc1.weight [NPAR - 16000] in the kernel's order (``rss`` slot groups)."""
    s = slots[:n_slots].float().reshape(n_slots, -1)[:, OTHER]
    rounds = -(-n_slots // rss)
    pad = torch.zeros(rounds * rss - n_slots, s.shape[1])          # + 0 leaves a partial that never is -0 unchanged
    s = torch.cat([s, pad]).view(rounds, rss, -1)
    part = torch.zeros(rss, s.shape[2])
    for r in range(rounds):
        part = part + s[r]
    total = part[0].clone()
    for g in range(1, rss):
        total = total + part[g]
    return total


def local_grad(slots, n_slots: int, factors, n_samples: int, **fault) -> torch.Tensor:
    """The fp32 local gradient [NPAR] the kernel reduces from the first ``n_slots`` slots and ``n_samples`` factor rows.
    ``fault``: fc1_grad's / other_grad's knobs, for the tests that plant faults."""
    g = torch.empty(NPAR)
    g[OTHER] = other_grad(slots.cpu(), n_slots, **{k: v for k, v in fault.items() if k == "rss"})
    g[W3:W3 + FC1] = fc1_grad(factors.cpu(), n_samples, **{k: v for k, v in fault.items() if k != "rss"}).reshape(-1)
    return g


def _butterfly(x: torch.Tensor) -> torch.Tensor:
    """x [..., 32] after ``x += shfl_xor(x, d)`` for d = 16, 8, 4, 2, 1; every lane holds the same sum."""
    lane = torch.arange(32)
    for d in (16, 8, 4, 2, 1):
        x = x + x[..., lane ^ d]
    return x


def loss_terms(slots, n_slots: int, butterfly: bool = True) -> torch.Tensor:
    """{sum of the slots' loss words, sum of their count words} [2] fp32 as reduce_loss computes them."""
    w = slots[:n_slots].cpu().float().reshape(n_slots, -1)[:, NPAR:NPAR + 2]
    rounds = -(-n_slots // 32)
    w = torch.cat([w, torch.zeros(rounds * 32 - n_slots, 2)]).view(rounds, 32, 2)
    lanes = torch.zeros(32, 2)
    for r in range(rounds):
        lanes = lanes + w[r]
    if not butterfly:                                   # a planted fault: the lanes added one after the other
        t = torch.zeros(2)
        for i in range(32):
            t = t + lanes[i]
        return t
    return _butterfly(lanes.t())[:, 0]


def loss_after(loss_acc: torch.Tensor, terms: torch.Tensor) -> torch.Tensor:
    """loss_acc with ``loss_acc[i] = prev + terms[i]`` for i < 2, the rest unchanged."""
    out = loss_acc.clone().float()
    out[:2] = out[:2] + terms
    return out


# ---------------------------------------------------------------------------------------------------------- the update
def update(g, p, m, mu: float, lr: float, wd: float = 0.0, nesterov: bool = False, max_norm=None, norm=None):
    """(params, momentum) [NPAR] after the kernel's update from the local gradient ``g``; ``lr``: the step's lr.  With
    ``max_norm`` (the clip instance) the gradient is first scaled by the coefficient of the pre-clip ``norm``."""
    p, m = p[:NPAR].cpu().float(), m[:NPAR].cpu().float()
    if max_norm is None:
        return SM.sgd_update(g, p, m, mu, lr, wd, nesterov)
    return GM.clip_update(g, p, m, mu, lr, wd, nesterov, norm, max_norm)


def aux_after(aux: torch.Tensor, params: torch.Tensor, swap: bool = False) -> torch.Tensor:
    """aux after the kernel wrote conv2.weight of ``params`` into it: w2f [ci][ky][kx][co] at 0 and w2b
    [co][ky][kx][half][8] at 5000, lanes 5..7 of every w2b row untouched.  ``swap``: a planted fault, w2f written as
    [co][ky][kx][ci]."""
    out = aux.cpu().clone()
    i = torch.arange(5000)
    co, r = i // 250, i % 250
    ci, kk = r // 25, r % 25
    w = params[264:264 + 5000].cpu()
    out[(co * 25 + kk) * 10 + ci if swap else (ci * 25 + kk) * 20 + co] = w
    out[5000 + ((co * 25 + kk) * 2 + ci // 5) * 8 + ci % 5] = w
    return out


def bucket_after(grads: torch.Tensor, step: int, grad_stride: int, zero: str = "other") -> torch.Tensor:
    """The gradient buffer after the kernel: [0, NPAR) of the other step parity's bucket zeroed (the only bucket when
    grad_stride is 0), everything else unchanged.  ``zero="current"``: a planted fault."""
    out = grads.cpu().clone()
    par = step & 1
    z = (par ^ 1 if zero == "other" else par) * grad_stride if grad_stride > 0 else 0
    out[z:z + NPAR] = 0.0
    return out


# ---------------------------------------------------------------------------------------------------------- the clip norm
def units(n_cta: int) -> list:
    """The units of each CTA in the order it runs them."""
    return [list(range(c, RED_UNITS, n_cta)) for c in range(n_cta)]


def unit_vectors(u: int, n_threads: int = 512) -> torch.Tensor:
    """The float4 vector each thread of unit u emits, -1 for a thread that emits none."""
    tid = torch.arange(n_threads)
    v = torch.full((n_threads,), -1, dtype=torch.long)
    if u < RED_FC1_TILES:
        j0, i0 = (u // (320 // RI)) * RJ, (u % (320 // RI)) * RI
        live = tid < RJ * RI // 4
        v[live] = W3 // 4 + (j0 + tid[live] // (RI // 4)) * 80 + i0 // 4 + tid[live] % (RI // 4)
    else:
        o0 = (u - RED_FC1_TILES) * RV
        nv = min(RV, RED_OTHER - o0)
        o = o0 + tid[:nv]
        v[:nv] = torch.where(o < W3 // 4, o, o + FC1 // 4)
    return v


def clip_norm(g: torch.Tensor, n_cta: int, per: str = "thread") -> np.float32:
    """The pre-clip norm the clip instance writes to grad_norm_out at grid ``n_cta``.  ``per="cta"``: a planted fault, one
    fmaf chain per CTA over all its squares."""
    g4 = torch.cat([g.float().reshape(-1, 4), torch.zeros(1, 4)])        # row -1: the zeros of an idle thread
    sched = units(n_cta)
    sq = torch.zeros(n_cta, 512)
    for r in range(len(sched[0])):
        idx = torch.full((n_cta, 512), -1, dtype=torch.long)
        for c in range(n_cta):
            if r < len(sched[c]):
                idx[c] = unit_vectors(sched[c][r])
        vals = g4[idx]                                                    # [n_cta, 512, 4]
        for e in range(4):
            sq = SM.fma32(vals[..., e], vals[..., e], sq)
    if per == "cta":
        cta = torch.zeros(n_cta)
        for c in range(n_cta):
            for r in range(len(sched[c])):
                for t in unit_vectors(sched[c][r]).tolist():
                    if t >= 0:
                        for e in range(4):
                            cta[c] = SM.fma32(g4[t, e], g4[t, e], cta[c])
    else:
        warp = _butterfly(sq.view(n_cta, 16, 32))[..., 0]                # lane 0 of each warp
        cta = torch.zeros(n_cta)
        for w in range(16):
            cta = cta + warp[:, w]
    s = 0.0
    for c in range(n_cta):
        s += float(cta[c])
    return np.float32(math.sqrt(s))


# ---------------------------------------------------------------------------------------------------------- det_reduce
def det_reduce(partials, n_slots: int):
    """(gradient [NPAR], loss terms [2]) det_reduce_kernel computes from the first ``n_slots`` slots: each element and each
    loss word summed in slot order from 0."""
    s = partials[:n_slots].cpu().float().reshape(n_slots, -1)[:, :NPAR + 2]
    acc = torch.zeros(NPAR + 2)
    for i in range(n_slots):
        acc = acc + s[i]
    return acc[:NPAR], acc[NPAR:]


# ---------------------------------------------------------------------------------------------------------- fp64 bound
def _gamma(n: int) -> float:
    return n * U32 / (1 - n * U32)


def fp64_bound(slots, n_slots: int, factors, n_samples: int):
    """(fp64 gradient [NPAR], bound [NPAR], fp64 loss terms [2], bound [2]): the exact sums of the same terms and the error
    bound of any fp32 evaluation that adds them in some order with one rounding per addition (an fma rounds once):
    gamma_n * sum |term|, n the number of terms, plus the fp32 rounding of the result."""
    s = slots[:n_slots].cpu().double().reshape(n_slots, -1)
    f = factors[:n_samples].cpu().double()
    dh, p2 = f[:, :50], f[:, FAC_P2:FAC_P2 + 320]
    ref = s[:, :NPAR].sum(0)
    mag = s[:, :NPAR].abs().sum(0)
    ref[W3:W3 + FC1] = (dh.t() @ p2).reshape(-1)
    mag[W3:W3 + FC1] = (dh.abs().t() @ p2.abs()).reshape(-1)
    n = torch.full((NPAR,), float(n_slots + 1), dtype=torch.float64)
    n[W3:W3 + FC1] = n_samples + 1
    bound = mag * (n * U32 / (1 - n * U32))
    lref, lmag = s[:, NPAR:NPAR + 2].sum(0), s[:, NPAR:NPAR + 2].abs().sum(0)
    return ref, bound, lref, lmag * _gamma(n_slots + 1)


# ---------------------------------------------------------------------------------------------------------- the tables
def sample_edges(S: int) -> list:
    return sorted({1, RKS - 1, RKS, RKS + 1, RKC - 1, RKC, RKC + 1, 2 * RKC - 1, 2 * RKC + 1, 4 * S, 4 * S + 1, 1000})


def slot_edges() -> list:
    b = RSLOT_BATCH * RSS
    return sorted({1, RSS - 1, RSS, RSS + 1, b - 1, b + 1, 2 * b - 1, 2 * b + 1})


def trainer_pairs(S: int) -> list:
    """(n_samples, n_slots) of FusedTrainer's slot path at batch B: min(B, 4S) step CTAs."""
    return [(B, min(B, 4 * S)) for B in (65, 128, 4 * S, 4 * S + 1, 1000)]


# the six (samples, slots) pairs the kernel has been tested at since the slot path was written
LEGACY = [(65, 65), (127, 127), (128, 128), (129, 129), (300, 151), (200, 320)]


def sizes(S: int) -> list:
    """(n_samples, n_slots) pairs: every sample edge and every slot edge at least once, the trainer's pairs on an S-SM card
    and the legacy pairs."""
    smp, sl = sample_edges(S), slot_edges()
    out = [(smp[i % len(smp)], sl[i % len(sl)]) for i in range(max(len(smp), len(sl)))]
    for pr in trainer_pairs(S) + LEGACY:
        if pr not in out:
            out.append(pr)
    return out


def grids() -> list:
    """Grids from one CTA running every unit to one unit per CTA: the fc1 tile count and half the unit count, each +-1 (a
    CTA's units then start with an fc1 tile and end with another kind, or the reverse), the 114 SMs of an H100 PCIe."""
    h = RED_UNITS // 2
    return sorted({1, 2, 3, RED_FC1_TILES - 1, RED_FC1_TILES, RED_FC1_TILES + 1, h - 1, h, h + 1, 114, RED_UNITS - 1,
                   RED_UNITS})


def gaps(S: int, table=None, grid_table=None) -> list:
    """What the tables miss: each sample and slot edge, the trainer's pairs, the legacy pairs, and grids where one CTA
    runs every unit, where some CTAs run one unit and others two, of one unit per CTA, and where a CTA runs two fc1 tiles,
    an fc1 tile and then another unit, and two other units (units run in increasing order, so no CTA runs another unit
    before an fc1 tile)."""
    table = sizes(S) if table is None else table
    grid_table = grids() if grid_table is None else grid_table
    smp = {n for n, _ in table}
    sl = {k for _, k in table}
    out = [f"{n} samples never run" for n in sample_edges(S) if n not in smp]
    out += [f"{k} slots never run" for k in slot_edges() if k not in sl]
    out += [f"the pair {pr} never runs" for pr in trainer_pairs(S) + LEGACY if pr not in table]
    scheds = [units(n) for n in grid_table]
    if not any(len(s) == 1 for s in scheds):
        out.append("no grid where one CTA runs every unit")
    if not any(min(map(len, s)) == 1 and max(map(len, s)) == 2 for s in scheds):
        out.append("no grid where some CTAs run one unit and others two")
    if not any(max(map(len, s)) == 1 for s in scheds):
        out.append("no grid of one unit per CTA")
    kinds = lambda s: {(u[i] < RED_FC1_TILES, u[i + 1] < RED_FC1_TILES) for u in s for i in range(len(u) - 1)}   # noqa: E731
    seen = set().union(*[kinds(s) for s in scheds]) if scheds else set()
    for pair, what in (((True, True), "two fc1 tiles"), ((True, False), "an fc1 tile and then another unit"),
                       ((False, False), "two units outside fc1.weight")):
        if pair not in seen:
            out.append(f"no CTA runs {what}")
    if 114 not in grid_table:
        out.append("the grid of a 114-SM card never runs")
    return out
