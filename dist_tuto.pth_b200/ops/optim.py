"""Momentum SGD over flat buffers -- one launch per gradient bucket instead of one per tensor.

Parity: ``optim.SGD(model.parameters(), lr=0.01, momentum=0.5)`` + ``optimizer.step()`` + ``optimizer.zero_grad()``
of the reference's training loop (train_dist.py:110,118,123; tuto.md:283,291,296).  Same update rule as
``torch.optim.SGD`` (``buf = mu*buf + (g + wd*p)``, ``p -= lr*buf``, dampening 0, no Nesterov).

GPU-first: the gradients of a model already live in flat (symmetric-memory) buckets
(:class:`~dist_tuto.pth_b200.parallel.ddp.GradBucket`); this optimizer lays the parameters and the momentum out in flat
buffers with the *same* offsets and strides (``p.data`` becomes a view), so a whole bucket is updated -- and its
gradients re-zeroed for the next backward -- by ONE ``sgd_flat_kernel`` launch (csrc/sgd.cu) that streams the three
arrays once.  (The ConvNet goes further and fuses the all-reduce into the same kernel: ``allreduce_sgd_kernel``.)
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

__all__ = ["FlatSGD"]


class FlatSGD:
    """``FlatSGD(model)`` where ``model`` is a plain module, a module carrying ``_grad_bucket`` or a
    :class:`DistributedDataParallel` wrapper.

    ``step()`` expects averaged gradients (call ``average_gradients(model)`` first, as the tutorial loop does) and,
    with ``zero_grad=True`` (default), leaves the buckets zeroed so no separate ``zero_grad()`` pass is needed;
    ``zero_grad()`` exists for loop compatibility and is then a no-op apart from re-arming the DDP hooks."""

    def __init__(self, model: nn.Module, lr: float = 0.01, momentum: float = 0.5, weight_decay: float = 0.0,
                 zero_grad: bool = True, group=None):
        from ..parallel.ddp import DistributedDataParallel, GradBucket, flatten_params

        self.lr, self.momentum, self.weight_decay = float(lr), float(momentum), float(weight_decay)
        self.fused_zero = bool(zero_grad)
        self._engine = model if isinstance(model, DistributedDataParallel) else getattr(model, "_ddp_engine", None)
        if self._engine is not None:
            self.buckets: List[GradBucket] = self._engine.buckets
        else:
            gb = getattr(model, "_grad_bucket", None)
            if gb is None:
                gb = GradBucket(flatten_params(model), group=group)
                object.__setattr__(model, "_grad_bucket", gb)
            self.buckets = [gb]
        self.param_flats: List[torch.Tensor] = []
        self.momentum_flats: List[torch.Tensor] = []
        for gb in self.buckets:
            p0 = gb.params[0]
            if any(p.dtype != torch.float32 for p in gb.params):
                raise TypeError("FlatSGD keeps fp32 master parameters; cast activations (autocast), not the parameters")
            pf = torch.zeros(gb.numel, dtype=torch.float32, device=p0.device)
            with torch.no_grad():
                for p, o, gv in zip(gb.params, gb.offsets, gb.views):
                    pv = pf[o:o + p.numel()].as_strided(gv.shape, gv.stride())   # same layout as the gradient view
                    pv.copy_(p.data)
                    p.data = pv
            self.param_flats.append(pf)
            self.momentum_flats.append(torch.zeros_like(pf))
        self._native = None

    # ------------------------------------------------------------------ update
    def _kernel(self):
        if self._native is None:
            from . import _ext

            self._native = _ext.C()        # raises if the extension is missing: no silent fallback on a GPU box
        return self._native

    @torch.no_grad()
    def step(self) -> None:
        """``optimizer.step()`` (train_dist.py:124) for every bucket, and -- with ``zero_grad=True`` -- the
        ``optimizer.zero_grad()`` of the next iteration (train_dist.py:118) in the same pass."""
        for gb, pf, mf in zip(self.buckets, self.param_flats, self.momentum_flats):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if pf.is_cuda and g.dtype == torch.float32:
                self._kernel().sgd_flat(pf, mf, g, self.lr, self.momentum, self.weight_decay, self.fused_zero)
                continue
            # CPU ranks (gloo) and reduced-precision gradient buckets: the same flat update with tensor ops
            gf = g.to(torch.float32)
            if self.weight_decay:
                gf = gf.add(pf, alpha=self.weight_decay)
            mf.mul_(self.momentum).add_(gf)
            pf.add_(mf, alpha=-self.lr)
            if self.fused_zero:
                g.zero_()
        if self.fused_zero and self._engine is not None:
            self._engine._reset()

    def zero_grad(self, set_to_none: bool = False) -> None:  # noqa: ARG002 - gradients stay views of the bucket
        """Loop-compatibility call (train_dist.py:118): the buckets are already zero after ``step()``; re-arms the DDP hooks."""
        if self._engine is not None:
            self._engine.zero_grad() if not self.fused_zero else self._engine._reset()
        elif not self.fused_zero:
            for gb in self.buckets:
                gb.zero_()

    # ------------------------------------------------------------------ checkpointing
    def state_dict(self) -> dict:
        """Hyper-parameters + the flat momentum buffers (CPU copies), for ``utils.checkpoint.save_checkpoint``."""
        return {"lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay,
                "momentum_buffers": [m.detach().cpu().clone() for m in self.momentum_flats]}

    def named_momentum(self, model: nn.Module) -> dict:
        """Momentum per parameter NAME (CPU copies) -- the canonical, engine-independent form written to checkpoints: the
        fused trainer stores exactly this (``state_dict()['momentum']``), so checkpoints cross engines with momentum."""
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        out = {}
        for gb, mf in zip(self.buckets, self.momentum_flats):
            for p, o, gv in zip(gb.params, gb.offsets, gb.views):
                if id(p) in names:
                    out[names[id(p)]] = mf[o:o + p.numel()].as_strided(gv.shape, gv.stride()).detach().cpu().clone()
        return out

    @torch.no_grad()
    def load_named_momentum(self, model: nn.Module, named: dict) -> int:
        """Inverse of :meth:`named_momentum`; returns how many tensors were restored."""
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        done = 0
        for gb, mf in zip(self.buckets, self.momentum_flats):
            for p, o, gv in zip(gb.params, gb.offsets, gb.views):
                src = named.get(names.get(id(p)))
                if src is not None:
                    mf[o:o + p.numel()].as_strided(gv.shape, gv.stride()).copy_(src)
                    done += 1
        return done

    def load_state_dict(self, sd: dict) -> None:
        """Inverse of :meth:`state_dict` (same model => same bucket layout)."""
        self.lr, self.momentum, self.weight_decay = float(sd["lr"]), float(sd["momentum"]), float(sd["weight_decay"])
        for m, src in zip(self.momentum_flats, sd["momentum_buffers"]):
            m.copy_(src)
