"""Plain-PyTorch fp32 model of the batched tensor-core engine (csrc/convnet_batched.cu), rounding point for rounding point.

The tensor-core kernels read bf16 operands and accumulate in fp32; this module performs the SAME computation with fp32
torch ops on operands rounded to bf16 at the places where the kernels round (activations between kernels, weight operand
copies, the data-gradient staging tile).  What is left between the two is fp32 summation order (~1e-6), so GPU tests can
use a tolerance that catches any indexing / layout bug instead of the loose "bf16 vs fp32" bounds of round 1; and on CPU
this model itself is checked against autograd of the reference ``Net`` (train_dist.py:53-71) within bf16 accuracy.

All functions take the flat fp32 parameter vector of ``ops.convnet_fused`` (same layout as the per-sample engine).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .convnet_fused import NPAR_ALLOC, pack_params, unpack_params  # noqa: F401  (re-exported for tests)

__all__ = ["rbf", "pool_codes", "forward_backward"]


def rbf(t: torch.Tensor) -> torch.Tensor:
    """Round to bf16 and back (fp32 container)."""
    return t.to(torch.bfloat16).to(torch.float32)


def pool_codes(indices: torch.Tensor, pooled: torch.Tensor, width: int) -> torch.Tensor:
    """The engine's 2x2 max-pool code of each pooled cell: bits 0..1 = argmax (0 top-left, 1 right, 2 below, 3 both),
    bit 2 = dead (the pooled maximum is not > 0, so relu passes no gradient).  ``indices`` come from
    ``F.max_pool2d(..., return_indices=True)`` over an input ``width`` columns wide."""
    code = ((indices // width) % 2) * 2 + (indices % width) % 2
    return code | ((pooled <= 0).to(code.dtype) * 4)


def _unpool_index(code: torch.Tensor, width: int) -> torch.Tensor:
    """Inverse of :func:`pool_codes` for the argmax bits: flat index into the un-pooled [2h, width] map."""
    code = code.to(torch.int64)
    h, w = code.shape[-2], code.shape[-1]
    py = torch.arange(h, device=code.device).view(h, 1)
    px = torch.arange(w, device=code.device).view(1, w)
    return (2 * py + ((code >> 1) & 1)) * width + 2 * px + (code & 1)


def forward_backward(params: torch.Tensor, x: torch.Tensor, target: torch.Tensor, m2: Optional[torch.Tensor] = None,
                     dm: Optional[torch.Tensor] = None, emulate_bf16: bool = True, p1_override: Optional[torch.Tensor] = None,
                     a1_override: Optional[torch.Tensor] = None, a2_override: Optional[torch.Tensor] = None,
                     p2_override: Optional[torch.Tensor] = None,
                     hrelu_override: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Mean-NLL loss and flat gradients of one batch.

    ``x`` [B,1,28,28] fp32 (normalised), ``m2`` [B,20] Dropout2d scales, ``dm`` [B,50] dropout scales (None = eval).
    ``emulate_bf16=False`` gives the same maths without any rounding (used to validate the formulas against autograd).
    ``p1_override`` [B,10,12,12] / ``a1_override`` [B,10,12,12] (2x2 argmax code 0..3): continue from the engine's OWN
    conv1 output -- conv1 is summed in a different fp32 order than ``F.conv2d``, so ~0.1 % of the bf16 values differ by
    one ulp, which flips a few conv2 pool arg-maxes downstream; with the override every later tensor is compared on
    bit-identical inputs.  The same holds further down: ``a2_override`` [B,20,4,4] (conv2 pool codes of
    :func:`pool_codes`, dead bit included) fixes the gradient routing and the relu decision of conv2, ``p2_override``
    [B,320] the fc1 input, and ``hrelu_override`` [B,50] (the fc1 GEMM output) the head and its relu decision."""
    r = rbf if emulate_bf16 else (lambda t: t)
    p = unpack_params(params)
    B = x.shape[0]
    x = x.to(torch.float32).view(B, 1, 28, 28)
    w1, b1, w2, b2 = p["conv1.weight"], p["conv1.bias"], p["conv2.weight"], p["conv2.bias"]
    w3, b3, w4, b4 = p["fc1.weight"], p["fc1.bias"], p["fc2.weight"], p["fc2.bias"]
    m2 = torch.ones(B, 20, dtype=torch.float32, device=x.device) if m2 is None else m2.to(torch.float32)
    dm = torch.ones(B, 50, dtype=torch.float32, device=x.device) if dm is None else dm.to(torch.float32)

    # ---------------------------------------------------------------- forward
    c1 = F.conv2d(x, w1, b1)                                             # fp32 SIMT
    m1, a1 = F.max_pool2d(c1, 2, return_indices=True)
    p1 = r(m1.clamp_min(0))                                              # P1 is stored as bf16
    if p1_override is not None:
        p1 = p1_override.to(torch.float32)
    if a1_override is not None:
        a1 = _unpool_index(a1_override.view(B, 10, 12, 12), 24)
    col = F.unfold(p1, 5)                                                # [B, 250, 64], k = ci*25 + tap
    c2 = (r(w2).view(20, 250) @ col).view(B, 20, 8, 8) + b2.view(1, 20, 1, 1)
    c2 = c2 * m2.view(B, 20, 1, 1)
    mp2, a2 = F.max_pool2d(c2, 2, return_indices=True)
    alive = (mp2.view(B, 320) > 0).to(torch.float32)                    # relu' (a dropped channel pools to 0: dead as well)
    if a2_override is not None:
        a2 = _unpool_index(a2_override.view(B, 20, 4, 4), 8)
        alive = ((a2_override.view(B, 320).to(torch.int64) & 4) == 0).to(torch.float32)
    p2 = r(mp2.clamp_min(0)).view(B, 320)                                # P2 is stored as bf16
    if p2_override is not None:
        p2 = p2_override.to(torch.float32).view(B, 320)
    hrelu = (p2 @ r(w3).t() + b3).clamp_min(0)                           # fp32 out of the fc1 GEMM
    if hrelu_override is not None:
        hrelu = hrelu_override.to(torch.float32).view(B, 50)
    h = hrelu * dm
    logits = h @ w4.t() + b4
    logp = F.log_softmax(logits, dim=1)
    loss = F.nll_loss(logp, target)

    # ---------------------------------------------------------------- backward
    dlog = (logp.exp() - F.one_hot(target, 10).to(torch.float32)) / B
    dh = r((dlog @ w4) * dm * (hrelu > 0).to(torch.float32))             # relu' * dropout scale; DH is stored as bf16
    hb = r(h)                                                            # H is stored as bf16
    g = {}
    g["fc2.weight"] = dlog.t() @ hb
    g["fc2.bias"] = dlog.sum(0)
    g["fc1.weight"] = dh.t() @ p2
    g["fc1.bias"] = dh.sum(0)
    dp2 = r(dh @ r(w3))                                                  # bf16 out of the fc1 data-gradient GEMM
    gp =r(dp2 * m2.repeat_interleave(16, dim=1)) * alive                # dropout2d scale; dC values are bf16
    dc = F.max_unpool2d(gp.view(B, 20, 4, 4), a2, 2, output_size=(8, 8))  # [B,20,8,8], one position per pooled cell
    g["conv2.weight"] = torch.einsum("bkp,bcp->ck", col, dc.view(B, 20, 64)).view(20, 10, 5, 5)
    g["conv2.bias"] = dc.sum((0, 2, 3))
    da = r(torch.einsum("ck,bcp->bkp", r(w2).view(20, 250), dc.view(B, 20, 64)))   # staging tile is bf16
    dp1 = F.fold(da, (12, 12), 5)                                        # col2im, fp32 sums
    g1 = dp1 * ((p1 if p1_override is not None else m1) > 0).to(torch.float32)
    dc1 = F.max_unpool2d(g1, a1, 2, output_size=(24, 24))
    g["conv1.weight"] = torch.einsum("bkp,bcp->ck", F.unfold(x, 5), dc1.view(B, 10, 576)).view(10, 1, 5, 5)
    g["conv1.bias"] = dc1.sum((0, 2, 3))
    flat = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=x.device)
    views = unpack_params(flat)
    for k, v in g.items():
        views[k].copy_(v)
    return {"loss": loss, "grads": flat, "p1": p1, "m1": m1, "p2": p2, "a1": a1, "c2": c2, "mp2": mp2, "a2": a2,
            "hrelu": hrelu, "logp": logp, "dlog": dlog, "dh": dh, "dp2": dp2, "dc": dc, "g1": g1, "named": g}
