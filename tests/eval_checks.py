"""Plain references and checks for the forward-only evaluation kernel (csrc/convnet_eval.cu), shared by the CPU test of the
checks themselves (tests/test_eval_checks.py) and the GPU test of the kernel (tests/test_gpu_eval_edges.py).

* ``reference``: every sample's log-probabilities, nll, log-sum-exp, largest |logit|, fp64 argmax and top-2 logit margin of
  ``Net.eval()`` (``step_oracle.masked_forward`` with all-ones dropout scales, forward only), on the fp32 image the kernel
  computes on, in fp64 (the oracle) or plain fp32.
* ``check_eval``: one call's ``out_logp`` and ``result`` against those references -- each row with
  ``step_oracle.check_per_sample`` and its bounds, the prediction count against the kernel's own log-probabilities and
  against fp64, the loss sum against the fp32 accumulation of a CTA's slot, and the sample count exactly.
* ``eval_sizes`` / ``gaps``: sample counts chosen from the kernel's geometry (G resident CTAs walking groups of S samples),
  and the (groups per CTA, last-group residue) pairs a table leaves out.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

import step_oracle as O
from dist_tuto.pth_b200.ops.convnet_fused import unpack_params

# ------------------------------------------------------------------------------------------------------------ reference


def normalize_u8(xu: torch.Tensor, mean: float, std: float) -> torch.Tensor:
    """The kernel's normalisation of raw pixels with the caller's mean / std, in fp32:
    (u * f32(1/255) - f32(mean)) * (f32(1) / f32(std)).  [N,1,28,28]."""
    f32 = torch.float32
    inv255 = torch.tensor(1.0, dtype=f32) / torch.tensor(255.0, dtype=f32)
    inv_std = torch.tensor(1.0, dtype=f32) / torch.tensor(std, dtype=f32)
    return ((xu.detach().cpu().to(f32) * inv255 - torch.tensor(mean, dtype=f32)) * inv_std).reshape(-1, 1, 28, 28)


def model_input(x: torch.Tensor, mean: float, std: float) -> torch.Tensor:
    """The fp32 image the kernel computes on: uint8 normalised as the kernel does, float32 as given."""
    x = x.detach().cpu()
    return normalize_u8(x, mean, std) if x.dtype == torch.uint8 else x.float().reshape(-1, 1, 28, 28)


def reference(params, x: torch.Tensor, y: torch.Tensor, mean: float, std: float, dtype=torch.float64,
              chunk: int = 2048) -> Dict[str, torch.Tensor]:
    """Per sample, in ``dtype`` on the CPU: ``logp`` [N,10], ``loss`` [N] (its nll; +inf for a label outside [0, 10)),
    ``lse`` [N] (log-sum-exp of the logits), ``zmax`` [N] (largest |logit|), ``argmax`` [N] (first index of the largest
    logit) and ``margin`` [N] (largest minus second-largest logit; 0 for an exact tie)."""
    p = O._params(params, dtype)
    xin = model_input(x, mean, std)
    yy = y.detach().cpu().long().reshape(-1)
    logits = []
    with torch.no_grad():
        for s in range(0, xin.shape[0], chunk):
            xc = xin[s:s + chunk].to(dtype)
            n = xc.shape[0]
            logits.append(O.masked_forward(p, xc, torch.ones(n, 20, dtype=dtype), torch.ones(n, 50, dtype=dtype)))
    z = torch.cat(logits) if logits else torch.empty(0, 10, dtype=dtype)
    logp = F.log_softmax(z, dim=1)
    valid = (yy >= 0) & (yy < 10)
    loss = -logp.gather(1, yy.clamp(0, 9)[:, None])[:, 0]
    loss = torch.where(valid, loss, torch.full_like(loss, math.inf))
    top2 = z.topk(2, dim=1).values
    return {"logp": logp, "loss": loss, "lse": torch.logsumexp(z, dim=1), "zmax": z.abs().amax(dim=1),
            "argmax": z.argmax(dim=1), "margin": top2[:, 0] - top2[:, 1]}


def sliced(ref: Dict[str, torch.Tensor], lo: int, hi: int) -> Dict[str, torch.Tensor]:
    return {k: v[lo:hi] for k, v in ref.items()}


def tie_fc2(params: torch.Tensor, a: int, b: int, bias: float = 8.0) -> torch.Tensor:
    """A copy of the flat ``params`` whose fc2 rows a and b are identical and share a bias that dominates every other
    logit: every sample's two largest logits are then exactly equal, at a and b."""
    out = params.detach().clone()
    v = unpack_params(out)
    v["fc2.weight"][b].copy_(v["fc2.weight"][a])
    v["fc2.bias"].zero_()
    v["fc2.bias"][a] = v["fc2.bias"][b] = bias
    return out


# --------------------------------------------------------------------------------------------------------- geometry


def schedule(N: int, G: int, S: int) -> Dict:
    """How the kernel spreads N samples: ``grid = min(groups, G)`` CTAs, CTA c runs groups c, c + grid, ...  Returns the
    grid, each CTA's group and sample counts, the group count of the CTA that runs the last group, and N mod S."""
    groups = (N + S - 1) // S
    grid = min(groups, G)
    if groups == 0:
        return {"grid": 0, "groups": np.zeros(0, np.int64), "samples": np.zeros(0, np.int64), "last_cta_groups": 0,
                "residue": 0}
    sizes = np.full(groups, S, np.int64)
    sizes[-1] = N - (groups - 1) * S
    cta = np.arange(groups) % grid
    return {"grid": grid, "groups": np.bincount(cta, minlength=grid), "samples": np.bincount(cta, sizes, minlength=grid)
            .astype(np.int64), "last_cta_groups": (groups - 1) // grid + 1, "residue": N % S}


def eval_sizes(G: int, S: int) -> List[int]:
    """Sample counts for a device with G resident CTAs and groups of S samples:
    * 0 .. 9: no launch, one partial group, one full group, a full and a partial group on two CTAs;
    * S*G - 1, S*G, S*G + 1: one group per CTA with a partial last one, exactly one wave, and CTA 0 running a second group;
    * S*G + S*(G//2) + 3: half the CTAs run two groups, the others one;
    * S*G + S*j + r and 2*S*G + S*j + r, r = 1 .. S: the last group, of every residue, is its CTA's 2nd / 3rd group;
    * 3*S*G + S*(G//3) + 5 and 4*S*G + 7: every CTA runs three or four groups (the mbarrier phase wraps twice and more)."""
    SG = S * G
    out = list(range(10)) + [SG - 1, SG, SG + 1, SG + S * (G // 2) + 3]
    out += [SG + S * ((11 * r) % G) + r for r in range(1, S + 1)]
    out += [2 * SG + S * ((7 * r) % G) + r for r in range(1, S + 1)]
    out += [3 * SG + S * (G // 3) + 5, 4 * SG + 7]
    return out


def gaps(G: int, S: int, table: Optional[List[int]] = None) -> List[str]:
    """What ``table`` (default ``eval_sizes(G, S)``) misses: the fixed counts, a mix of CTAs running one and two groups,
    a case where every CTA runs three or more, and each (groups of the CTA that runs the last group: 1, 2 or 3+, N mod S)
    pair."""
    table = eval_sizes(G, S) if table is None else table
    SG = S * G
    out = [f"N = {n} never runs" for n in list(range(10)) + [SG - 1, SG, SG + 1] if n not in table]
    scheds = [schedule(n, G, S) for n in table if n > 0]
    if not any(s["groups"].min() == 1 and s["groups"].max() == 2 for s in scheds):
        out.append("no case where some CTAs run one group and others two")
    if not any(s["groups"].min() >= 3 for s in scheds):
        out.append("no case where every CTA runs three or more groups")
    have = {(min(s["last_cta_groups"], 3), s["residue"]) for s in scheds}
    out += [f"the last group is never its CTA's {'3rd or later' if k == 3 else ('1st', '2nd')[k - 1]} group with "
            f"N mod {S} = {r}" for k in (1, 2, 3) for r in range(S) if (k, r) not in have]
    return out


# ---------------------------------------------------------------------------------------------------------- checks


def kernel_rows(out_logp: torch.Tensor, y: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The kernel's per-sample results: its log-probabilities and the nll it adds, ``-out_logp[i, y_i]``."""
    lp = out_logp.detach().cpu().float()
    return {"logp": lp, "loss": -lp.gather(1, y.detach().cpu().long().reshape(-1, 1))[:, 0]}


def row_bounds(key: str, ref64: Dict[str, torch.Tensor], ref32: Dict[str, torch.Tensor]) -> torch.Tensor:
    """``check_per_sample``'s bound on each row of ``key`` ("logp" or "loss"), vectorised: max(C * |ref32 - ref64|,
    EPS * max(|ref64|, lse * sqrt(width)))."""
    r64, r32 = ref64[key].double(), ref32[key].double()
    if r64.dim() == 1:
        r64, r32 = r64[:, None], r32[:, None]
    size = torch.maximum(r64.norm(dim=1), ref64["lse"].double().abs() * math.sqrt(r64.shape[1]))
    return torch.maximum(O.C_BOUND * (r32 - r64).norm(dim=1), O.EPS_BOUND * size)


def prediction_range(out_logp: torch.Tensor, y: torch.Tensor, ref64: Dict[str, torch.Tensor]):
    """(lo, hi) for ``result[1]`` from the kernel's own log-probabilities.  ``logp = logit - c`` is monotone, so a row with
    a unique top entry predicts that entry.  A row with a tied top predicts the lowest tied index when its fp64 logits tie
    exactly too (margin 0), and is undecided otherwise: it may count if its label is among the tied entries."""
    lp = out_logp.detach().cpu().float()
    yy = y.detach().cpu().long().reshape(-1)
    if lp.shape[0] == 0:
        return 0, 0
    valid = (yy >= 0) & (yy < 10)
    is_top = lp == lp.max(dim=1, keepdim=True).values
    unique = is_top.sum(dim=1) == 1
    y_top = is_top.gather(1, yy.clamp(0, 9)[:, None])[:, 0] & valid
    exact_tie = ~unique & (ref64["margin"] == 0)
    lo = int((unique & y_top).sum()) + int((exact_tie & (ref64["argmax"] == yy) & valid).sum())
    return lo, lo + int((~unique & ~exact_tie & y_top).sum())


def check_eval(result, out_logp: torch.Tensor, y: torch.Tensor, ref64: Dict[str, torch.Tensor],
               ref32: Dict[str, torch.Tensor], G: int, S: int, where: str = "") -> O.Report:
    """Every check of one call with valid labels.  Ratios (error / bound) per check: "logp", "loss" (per row), "margin"
    (fp64 prediction rule), "correct", "n" (exact: inf on a miss), "sum" (against the kernel's own nll) and "sum64"
    (against the fp64 loss)."""
    res = [float(v) for v in (result.tolist() if isinstance(result, torch.Tensor) else result)]
    N = int(y.numel())
    got = kernel_rows(out_logp, y)
    labels = [f"{where}sample {i}" for i in range(N)]
    rep = O.check_per_sample(got, ref64, ref32, labels=labels, keys=["logp", "loss"]) if N else O.Report()
    lp = got["logp"]

    # fp64 prediction rule: a sample whose fp64 margin exceeds twice its logp bound has the fp64 argmax as unique top
    if N:
        sure = ref64["margin"] > 2 * row_bounds("logp", ref64, ref32)
        top = lp.max(dim=1, keepdim=True).values
        ok = (lp == top).sum(dim=1).eq(1) & lp.gather(1, ref64["argmax"][:, None])[:, 0].eq(top[:, 0])
        bad = torch.nonzero(sure & ~ok).flatten().tolist()
        rep.note(where + "predictions", "margin", math.inf if bad else 0.0)
        if bad:
            rep.failures.append(f"{where}{len(bad)} samples clear of a near-tie predict other than the fp64 argmax, "
                                f"first sample {bad[0]}: logp {lp[bad[0]].tolist()}, fp64 argmax "
                                f"{int(ref64['argmax'][bad[0]])}")

    lo, hi = prediction_range(lp, y, ref64)
    if not lo <= res[1] <= hi:
        rep.note(where + "result[1]", "correct", math.inf)
        rep.failures.append(f"{where}result[1] = {res[1]} outside [{lo}, {hi}] from the kernel's own log-probabilities")
    if res[2] != N:
        rep.note(where + "result[2]", "n", math.inf)
        rep.failures.append(f"{where}result[2] = {res[2]} != N = {N}")

    # sum rule: the kernel's own nll added in fp32 per CTA (k samples at most), the slots in fp64
    nll = got["loss"].double()
    k = int(schedule(N, G, S)["samples"].max()) if N else 0
    own = math.fsum(nll.tolist())
    tol = k * 2.0 ** -24 * float(nll.abs().sum())
    _ratio(rep, where + "result[0]", "sum", abs(res[0] - own), tol,
           f"{where}result[0] = {res[0]!r} vs the fp64 sum of its own nll {own!r}")
    if N:
        want = math.fsum(ref64["loss"].tolist())
        tol64 = tol + float(row_bounds("loss", ref64, ref32).sum())
        _ratio(rep, where + "result[0]", "sum64", abs(res[0] - want), tol64,
               f"{where}result[0] = {res[0]!r} vs the fp64 loss sum {want!r}")
    return rep


def _ratio(rep: O.Report, at: str, name: str, err: float, bound: float, what: str):
    ratio = 0.0 if err == 0.0 else (err / bound if bound > 0 else math.inf)
    if not math.isfinite(err):
        ratio = math.inf
    rep.note(at, name, ratio)
    if ratio > 1.0:
        rep.failures.append(f"{what}: error {err:.3e} is {ratio:.3g}x the bound {bound:.3e}")
