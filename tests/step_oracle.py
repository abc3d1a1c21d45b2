"""Plain references for the per-sample step kernels (csrc/convnet.cu, csrc/convnet_cluster.cu), shared by the CPU test of
the references themselves (tests/test_step_oracle.py) and the GPU test of the kernels (tests/test_gpu_step_per_sample.py).

* ``philox4x32_10`` / ``dropout_masks``: the kernels' dropout stream, bit for bit, in uint32 / fp32 numpy.  Sample b of a
  launch draws from Philox4x32-10 with key = seed, counter = (step * 32 + q, sample_base + b), q = 0..17; uniform
  k = 4q + w is float32(word w) * 2^-32, channel c of Dropout2d uses uniform c and fc1 unit j uniform 20 + j.  A unit is
  kept iff its uniform >= float32(p), and kept units are scaled by float32(1) / (float32(1) - float32(p)).
* ``per_sample_reference``: every sample's log-probabilities, loss, argmax and the gradient of its own loss with respect
  to every parameter, through ``torch.func.vmap(grad(...))`` of the masked forward of ``Net`` (conv1 -> pool -> relu ->
  conv2 * m2 -> pool -> relu -> fc1 -> relu * mh -> fc2 -> log_softmax), on the CPU, in fp64 (the oracle) or fp32.
* ``check_per_sample``: compares each (row, tensor) pair of a kernel result with the fp64 oracle against a bound set by the
  error of the same computation in plain fp32 (see ``C_BOUND`` / ``EPS_BOUND``); a row is one sample, or one slot that
  summed several samples (``fold``).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from batched_checks import normalize_u8
from dist_tuto.pth_b200.models.convnet import PARAM_SHAPES
from dist_tuto.pth_b200.ops.convnet_fused import unpack_params

NAMES = [n for n, _ in PARAM_SHAPES]

# ------------------------------------------------------------------------------------------------------------ Philox
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(seed: int, subseq, offset) -> np.ndarray:
    """Philox4x32-10 of common.cuh (``Philox::gen``): key = (seed lo, seed hi), counter = (offset lo, offset hi, subseq lo,
    subseq hi).  ``subseq`` and ``offset`` broadcast against each other; returns uint32 [..., 4]."""
    sub = np.asarray(subseq, dtype=np.uint64)
    off = np.asarray(offset, dtype=np.uint64)
    sub, off = np.broadcast_arrays(sub, off)
    c0, c1 = off & _LO, off >> _S32
    c2, c3 = sub & _LO, sub >> _S32
    k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2                      # 32 x 32 -> 64-bit products, exact in uint64
        c0, c1, c2, c3 = ((p1 >> _S32) ^ c1 ^ np.uint64(k0), p1 & _LO, (p0 >> _S32) ^ c3 ^ np.uint64(k1), p0 & _LO)
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def uniforms(seed: int, sample_base: int, B: int, step: int, n: int = 72) -> np.ndarray:
    """The kernels' first ``n`` uniforms of samples sample_base .. sample_base + B - 1 at ``step``: float32 [B, n]."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    off = (np.uint64(int(step) % 2 ** 64) * np.uint64(32) + q)[None, :]      # step * 32 + q in uint64, as the kernel
    sub = (np.uint64(int(sample_base) % 2 ** 64) + np.arange(B, dtype=np.uint64))[:, None]
    words = philox4x32_10(seed, sub, off).reshape(B, -1)[:, :n]
    return words.astype(np.float32) * np.float32(2.0 ** -32)              # round-to-nearest conversion, exact scaling


def keep_scale(p_drop: float) -> np.float32:
    return np.float32(1.0) / (np.float32(1.0) - np.float32(p_drop))


def dropout_masks(seed: int, sample_base: int, B: int, step: int, p_drop: float, training: bool = True) -> torch.Tensor:
    """The [B, 70] scales the kernels apply and report in ``mask_out``: columns 0-19 Dropout2d channels, 20-69 fc1 units."""
    if not training:
        return torch.ones(B, 70, dtype=torch.float32)
    u = uniforms(seed, sample_base, B, step, 70)
    m = np.where(u >= np.float32(p_drop), keep_scale(p_drop), np.float32(0.0)).astype(np.float32)
    return torch.from_numpy(m)


@functools.lru_cache(maxsize=None)
def find_boundary_draw(p_drop: float = 0.5, seed: int = 0x5EED, step: int = 11, chunk: int = 1 << 16,
                       limit: int = 1 << 24):
    """(seed, sample, step, k): the first sample index whose uniform k (< 70) at ``step`` is exactly float32(p_drop), so
    that ``>=`` keeps the unit and ``>`` would drop it.  At p = 0.5 about 193 of the 2^32 words round to 0.5: one sample in
    ~3 * 10^5 has such a draw among its 70."""
    pf = np.float32(p_drop)
    for base in range(0, limit, chunk):
        u = uniforms(seed, base, chunk, step, 70)
        hit = np.argwhere(u == pf)
        if len(hit):
            b, k = (int(v) for v in hit[0])
            return seed, base + b, step, k
    raise RuntimeError(f"no uniform equal to {p_drop} in the first {limit} samples")


# ------------------------------------------------------------------------------------------------- per-sample oracle
def _params(params, dtype) -> Dict[str, torch.Tensor]:
    views = unpack_params(params) if isinstance(params, torch.Tensor) else params
    return {n: views[n].detach().to("cpu", dtype).clone() for n in NAMES}


def model_input(x: torch.Tensor) -> torch.Tensor:
    """The fp32 image the kernels compute on: uint8 pixels normalised as in the kernels, fp32 input as given."""
    x = x.detach().cpu()
    return normalize_u8(x).reshape(-1, 1, 28, 28) if x.dtype == torch.uint8 else x.float().reshape(-1, 1, 28, 28)


def masked_forward(p, x, m2, mh, pool=F.max_pool2d, relu=F.relu):
    """Net's forward with explicit dropout scales: m2 [N,20] per conv2 channel, mh [N,50] per fc1 unit.  Returns the
    logits.  ``pool`` / ``relu`` exist so that tests can plant faults in the reference."""
    h = relu(pool(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]), 2))
    h = F.conv2d(h, p["conv2.weight"], p["conv2.bias"]) * m2[:, :, None, None]
    h = relu(pool(h, 2)).reshape(-1, 320)
    h = relu(F.linear(h, p["fc1.weight"], p["fc1.bias"])) * mh
    return F.linear(h, p["fc2.weight"], p["fc2.bias"])


def per_sample_reference(params, x, y, masks: Optional[torch.Tensor] = None, dtype=torch.float64, pool=F.max_pool2d,
                         relu=F.relu) -> Dict[str, torch.Tensor]:
    """Each sample's ``logp`` [B,10], ``loss`` [B] (its nll), ``argmax`` [B] (first index of the largest logit), ``lse``
    [B] (log-sum-exp of its logits), ``zmax`` [B] (largest |logit|) and, per parameter name, the gradient of its own loss [B, *shape], in ``dtype`` on the
    CPU.  ``masks``: [B,70] dropout scales (None: dropout off)."""
    p = _params(params, dtype)
    xin = model_input(x).to(dtype)
    B = xin.shape[0]
    yy = y.detach().cpu().long().reshape(B)
    m = torch.ones(B, 70, dtype=dtype) if masks is None else masks.detach().cpu().to(dtype).reshape(B, 70)

    def loss_one(pp, xb, yb, mb):
        logits = masked_forward(pp, xb[None], mb[None, :20], mb[None, 20:], pool, relu)[0]
        logp = F.log_softmax(logits, dim=0)
        return -logp.gather(0, yb[None])[0], (logp, logits)

    grads, (logp, logits) = torch.func.vmap(torch.func.grad(loss_one, has_aux=True), in_dims=(None, 0, 0, 0))(p, xin, yy, m)
    out = {n: grads[n] for n in NAMES}
    out["logp"] = logp
    out["loss"] = -logp.gather(1, yy[:, None])[:, 0]
    out["argmax"] = logits.argmax(dim=1)
    out["lse"] = torch.logsumexp(logits, dim=1)
    out["zmax"] = logits.abs().amax(dim=1)
    return out


FLOAT_KEYS = NAMES + ["logp", "loss"]


def scaled(ref: Dict[str, torch.Tensor], inv_bsz: float) -> Dict[str, torch.Tensor]:
    """The kernels' per-sample terms at ``inv_bsz``: gradients and loss times inv_bsz (log-probs and argmax unscaled).  The
    factor is rounded to fp32 first, as the kernels receive it."""
    s = float(np.float32(inv_bsz))
    return {k: (v * s if k in NAMES or k in ("loss", "lse") else v) for k, v in ref.items()}


def fold(ref: Dict[str, torch.Tensor], groups: Sequence[Sequence[int]]) -> Dict[str, torch.Tensor]:
    """Row g = the sum of the rows in groups[g], added one sample after the other in the tensor's own dtype (fp32: the
    plain sequential accumulation a slot of the kernel does)."""
    out = {}
    for k in NAMES + ["loss", "lse"]:
        v = ref[k].abs() if k == "lse" else ref[k]
        rows = []
        for g in groups:
            acc = torch.zeros_like(v[0])
            for b in g:
                acc = acc + v[b]
            rows.append(acc)
        out[k] = torch.stack(rows)
    out["zmax"] = torch.stack([ref["zmax"][list(g)].max() for g in groups])
    return out


# ---------------------------------------------------------------------------------------------------------- checker
# Bound on each (row, tensor) error:  ||got - ref64|| <= max(C_BOUND * ||ref32 - ref64||, EPS_BOUND * ||ref64||).
# ref32 is the same computation in plain fp32 (per-sample vmap on the CPU; slot sums accumulated sample by sample in
# fp32), so ||ref32 - ref64|| is what fp32 rounding costs on that row.  A kernel sums in other orders, contracts to fma
# and uses __expf / __logf (a few ulp each, and 2^-21 absolute for log near 1): C_BOUND = 16 leaves an order of
# magnitude over one plain fp32 evaluation for that.  EPS_BOUND = 2^-20 (16 fp32 ulp of the row's norm) is the floor for
# rows where fp32 happens to be almost exact.  Log-probs and losses are differences logit - logsumexp: an fp32
# implementation that forms the log-sum-exp first (max + log sum exp, as the kernels and torch.logsumexp do) rounds at
# the size of the log-sum-exp, not of the difference, so their floor is EPS_BOUND times that size (``lse``).  Likewise
# the logits themselves carry an fp32 rounding error of the size of the largest logit (``zmax``), which exp() turns into
# a relative error of that size in the softmax and in every gradient behind it: the gradients' floor is EPS_BOUND *
# max(1, zmax) times their norm (it only differs from EPS_BOUND when logits exceed 1, e.g. a saturated softmax).  Exact
# zeros are required where the masks make the reference exactly zero.
C_BOUND = 16.0
EPS_BOUND = 2.0 ** -20


@dataclass
class Report:
    failures: List[str] = field(default_factory=list)
    worst: float = 0.0
    worst_at: str = ""
    ratios: Dict[str, float] = field(default_factory=dict)      # per tensor name: largest error / bound over the rows

    def note(self, where: str, name: str, ratio: float):
        if ratio > self.ratios.get(name, -1.0):
            self.ratios[name] = ratio
        if ratio > self.worst or not self.worst_at:
            self.worst, self.worst_at = ratio, f"{where}: {name}"

    def message(self, n: int = 12) -> str:
        head = f"{len(self.failures)} failures; worst {self.worst:.3g}x the bound at {self.worst_at}"
        return "\n".join([head] + self.failures[:n])


def _norm(t: torch.Tensor) -> float:
    return float(t.double().norm())


def _exact_zero_views(got_row: Dict[str, torch.Tensor], mask_row: torch.Tensor):
    """(what, tensor) pairs that must be exactly zero in a sample whose dropout scales are ``mask_row``."""
    for co in torch.nonzero(mask_row[:20] == 0).flatten().tolist():
        yield f"conv2.weight[{co}] (channel dropped)", got_row["conv2.weight"][co]
        yield f"conv2.bias[{co}] (channel dropped)", got_row["conv2.bias"][co]
    for j in torch.nonzero(mask_row[20:70] == 0).flatten().tolist():
        yield f"fc1.weight[{j}] (unit dropped)", got_row["fc1.weight"][j]
        yield f"fc1.bias[{j}] (unit dropped)", got_row["fc1.bias"][j]
        yield f"fc2.weight[:, {j}] (unit dropped)", got_row["fc2.weight"][:, j]


def check_per_sample(got: Dict[str, torch.Tensor], ref64: Dict[str, torch.Tensor], ref32: Dict[str, torch.Tensor],
                     masks: Optional[torch.Tensor] = None, labels: Optional[Sequence[str]] = None,
                     keys: Optional[Sequence[str]] = None, C: float = C_BOUND, eps: float = EPS_BOUND) -> Report:
    """Compare every row of every tensor in ``keys`` (default: those ``got`` has among the parameters, logp and loss).
    ``masks`` [rows, 70]: each row is one sample with these dropout scales, and the entries they zero must be exactly 0.
    ``got["masks"]``, if present, must equal ``masks`` bit for bit.  A missing row (NaN, wrong shape) is a failure like any
    other."""
    rep = Report()
    keys = [k for k in (keys or FLOAT_KEYS) if k in got]
    rows = ref64[keys[0]].shape[0]
    labels = labels or [f"sample {i}" for i in range(rows)]
    if "masks" in got:
        bad = torch.nonzero(got["masks"].detach().cpu().float() != masks.cpu().float())
        if len(bad):
            i, k = (int(v) for v in bad[0])
            rep.note(labels[i], "masks", math.inf)
            rep.failures.append(f"masks: {len(bad)} scales differ from the host Philox reference, first at {labels[i]}, "
                                f"column {k}: {float(got['masks'][i, k])} != {float(masks[i, k])}")
    for k in keys:
        g, r64, r32 = got[k].detach().cpu().double(), ref64[k].double(), ref32[k].double()
        if g.shape != r64.shape:
            rep.failures.append(f"{k}: shape {tuple(g.shape)} != {tuple(r64.shape)}")
            rep.note("all rows", k, math.inf)
            continue
        lse = ref64["lse"].double().abs() if k in ("logp", "loss") and "lse" in ref64 else None
        zmax = ref64["zmax"].double() if k in NAMES and "zmax" in ref64 else None
        for i in range(rows):
            err = _norm(g[i] - r64[i]) if bool(torch.isfinite(g[i]).all()) else math.inf
            size = _norm(r64[i]) if lse is None else max(_norm(r64[i]), float(lse[i]) * math.sqrt(r64[i].numel()))
            if zmax is not None:
                size *= max(1.0, float(zmax[i]))
            bound = max(C * _norm(r32[i] - r64[i]), eps * size)
            ratio = 0.0 if err == 0.0 else (err / bound if bound > 0 else math.inf)
            rep.note(labels[i], k, ratio)
            if ratio > 1.0:
                rep.failures.append(f"{labels[i]}: {k}: |got - fp64| = {err:.3e} is {ratio:.3g}x the bound {bound:.3e}")
    if masks is not None and all(n in got for n in ("conv2.weight", "conv2.bias", "fc1.weight", "fc1.bias", "fc2.weight")):
        for i in range(rows):
            row = {n: got[n][i].detach().cpu() for n in NAMES if n in got}
            for what, t in _exact_zero_views(row, masks[i].cpu()):
                nz = int(torch.count_nonzero(t))
                if nz:
                    rep.note(labels[i], what.split("[")[0], math.inf)
                    rep.failures.append(f"{labels[i]}: {what}: {nz} nonzero entries where the mask zeroes the gradient")
    return rep
