"""wgmma bf16 GEMM entry points (csrc/gemm_tcgen05.cu).

``linear_bf16(x, w, bias)`` computes ``x @ w.T + bias`` like ``F.linear`` (the op
behind fc1/fc2, train_dist.py:61-62,68,70) on the Hopper tensor cores: TMA-fed
128B-swizzled smem tiles, ``wgmma.mma_async`` with fp32 accumulators in registers,
bias/ReLU fused in the register epilogue.  No cuBLAS on this path.

``linear_tc`` / ``TcLinear`` make it trainable: the data gradient ``dY @ W`` and the weight
gradient ``dY^T @ X`` are two more launches of the same kernel (it multiplies two K-major
operands, so the backward operands are re-laid out K-major first: ``W^T``, ``dY^T``, ``X^T``
-- bf16 transposes, memory-bound and small next to the GEMMs), the bias gradient is a
column sum.  Forward/backward accumulate in fp32; operands are rounded to bf16 once."""
from __future__ import annotations

from typing import Optional

import torch

from . import _ext

__all__ = ["linear_bf16", "linear_tc", "TcLinear"]


def linear_bf16(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
                out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``relu?(x[M,K] @ w[N,K]^T + bias[N])``; x, w bf16 (cast if needed), fp32 accumulate."""
    C = _ext.C()
    x2 = x.reshape(-1, x.shape[-1])
    if x2.dtype != torch.bfloat16:
        x2 = x2.to(torch.bfloat16)
    if w.dtype != torch.bfloat16:
        w = w.to(torch.bfloat16)
    K = x2.shape[1]
    if K % 8:                                  # TMA needs 16-byte rows
        pad = 8 - K % 8
        x2 = torch.nn.functional.pad(x2, (0, pad))
        w = torch.nn.functional.pad(w, (0, pad))
    b = None if bias is None else bias.to(torch.float32).contiguous()
    out = C.gemm_bf16(x2.contiguous(), w.contiguous(), b, relu, out_dtype == torch.bfloat16)
    return out.view(*x.shape[:-1], w.shape[0])


def _pad_to(t: torch.Tensor, dim: int, mult: int) -> torch.Tensor:
    r = t.shape[dim] % mult
    if r == 0:
        return t
    pad = [0, 0] * t.dim()
    pad[2 * (t.dim() - 1 - dim) + 1] = mult - r
    return torch.nn.functional.pad(t, pad)


class _LinearTC(torch.autograd.Function):
    """y = x @ w^T + b with all three GEMMs (forward, dgrad, wgrad) on csrc/gemm_tcgen05.cu."""

    @staticmethod
    def forward(ctx, x, w, bias):
        C = _ext.C()
        x2 = x.reshape(-1, x.shape[-1])
        xb = _pad_to(x2.to(torch.bfloat16), 1, 8).contiguous()           # [M, K8]
        wb = _pad_to(w.to(torch.bfloat16), 1, 8).contiguous()            # [N, K8]
        b = None if bias is None else bias.to(torch.float32).contiguous()
        y = C.gemm_bf16(xb, wb, b, False, False)                         # fp32 out
        ctx.save_for_backward(xb, wb)
        ctx.meta = (x.shape, x.dtype, w.shape, w.dtype, None if bias is None else bias.dtype)
        return y.view(*x.shape[:-1], w.shape[0]).to(x.dtype if x.dtype != torch.bfloat16 else torch.float32)

    @staticmethod
    def backward(ctx, gy):
        C = _ext.C()
        xb, wb = ctx.saved_tensors
        xshape, xdtype, wshape, wdtype, bdtype = ctx.meta
        N, K = wshape
        g2 = gy.reshape(-1, N)
        gb = g2.to(torch.bfloat16)
        gx = gw = gbias = None
        if ctx.needs_input_grad[0]:
            # dX[M,K] = dY[M,N] @ W[N,K]:  A = dY (inner dim N), B = W^T [K8, N]  (inner dim N, padded to 8)
            a = _pad_to(gb, 1, 8).contiguous()
            bt = _pad_to(wb.t(), 1, 8).contiguous()
            gx = C.gemm_bf16(a, bt, None, False, False)[:, :K].reshape(xshape).to(xdtype)
        if ctx.needs_input_grad[1]:
            # dW[N,K] = dY^T[N,M] @ X[M,K]:  A = dY^T (inner dim M), B = X^T [K8, M]
            at = _pad_to(gb.t(), 1, 8).contiguous()
            bt = _pad_to(xb.t(), 1, 8).contiguous()
            gw = C.gemm_bf16(at, bt, None, False, False)[:, :K].to(wdtype)
        if bdtype is not None and ctx.needs_input_grad[2]:
            gbias = g2.to(torch.float32).sum(0).to(bdtype)
        return gx, gw, gbias


def linear_tc(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable ``F.linear`` on the wgmma GEMM (CUDA tensors; falls back to ``F.linear`` on the CPU)."""
    if not x.is_cuda:
        return torch.nn.functional.linear(x, w, bias)
    return _LinearTC.apply(x, w, bias)


class TcLinear(torch.nn.Linear):
    """``nn.Linear`` whose forward, data-gradient and weight-gradient GEMMs run on ``wgmma.mma_async`` (bf16 operands, fp32
    accumulation, fp32 master weights stay in ``self.weight``).  State-dict compatible with ``nn.Linear``."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return linear_tc(x, self.weight, self.bias)
