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

import math
import struct
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

__all__ = ["FlatSGD", "LRSchedule"]

_KINDS = {"constant": 1, "multistep": 2, "cosine": 3}      # csrc/lr_schedule.h: LRS_CONSTANT, LRS_MULTISTEP, LRS_COSINE
MAX_MILESTONES = 8


def _f32(x: float) -> float:
    """``x`` rounded once to the nearest fp32 value (ties to even), as a Python float."""
    return struct.unpack("f", struct.pack("f", x))[0]


class LRSchedule:
    """Learning-rate warmup and decay as a closed-form multiplier of the base lr, evaluated per optimizer update.

    The argument ``s`` of the schedule is the number of updates applied before this one -- the device step counter's value
    when the update runs -- so the fused engines compute the lr inside their optimizer kernels (csrc/lr_schedule.h holds
    the same formula) and captured graphs, the native executor and resumed runs follow it without re-capture.

    * warmup: for ``s < warmup_steps`` (W) the multiplier is ``warmup_start + (1 - warmup_start) * s / W``
      (``torch.optim.lr_scheduler.LinearLR``'s ramp; default start 1/3 like LinearLR);
    * then ``decay``: ``"constant"`` (1); ``"multistep"``: ``gamma ** #{m in milestones : m <= s}`` (absolute update
      indices, sorted, at most 8); ``"cosine"``: ``min_factor + (1 - min_factor) * (1 + cos(pi * d / (T - W))) / 2`` with
      ``d = min(s - W, T - W)`` and ``T = total_steps > W``.

    All arithmetic is fp64 and ``base * factor`` is rounded to fp32 once (:meth:`lr_at`).  With ``unit="epoch"`` the
    counts (warmup, milestones, total) are epochs; :meth:`resolve` turns them into updates.  Trainers take step units only.
    Arbitrary callables are not supported: the fused engines replay fixed launches and compute the lr on the device."""

    def __init__(self, warmup_steps: float = 0, warmup_start: float = 1.0 / 3.0, decay: str = "constant",
                 milestones: Sequence[float] = (), gamma: float = 0.1, total_steps: Optional[float] = None,
                 min_factor: float = 0.0, unit: str = "step"):
        if unit not in ("step", "epoch"):
            raise ValueError(f"LRSchedule.unit must be 'step' or 'epoch', got {unit!r}")
        if decay not in _KINDS:
            raise ValueError(f"LRSchedule.decay must be one of {sorted(_KINDS)}, got {decay!r}")
        whole = (lambda v: float(v) == int(v)) if unit == "step" else (lambda v: True)
        if warmup_steps < 0 or not whole(warmup_steps):
            raise ValueError(f"LRSchedule.warmup_steps must be a non-negative {'integer' if unit == 'step' else 'count'}")
        if not 0.0 < warmup_start <= 1.0:
            raise ValueError("LRSchedule.warmup_start must be in (0, 1]")
        milestones = tuple(milestones)
        if decay == "multistep":
            if len(milestones) > MAX_MILESTONES:
                raise ValueError(f"LRSchedule: at most {MAX_MILESTONES} milestones")
            if any(m < 0 or not whole(m) for m in milestones):
                raise ValueError("LRSchedule.milestones must be non-negative step indices")
            if list(milestones) != sorted(milestones):
                raise ValueError("LRSchedule.milestones must be sorted")
            if not 0.0 < gamma <= 1.0:
                raise ValueError("LRSchedule.gamma must be in (0, 1]")
        elif milestones:
            raise ValueError("LRSchedule.milestones are used by decay='multistep' only")
        if decay == "cosine":
            if total_steps is None or total_steps <= warmup_steps or not whole(total_steps):
                raise ValueError("LRSchedule: decay='cosine' needs total_steps > warmup_steps")
            if not 0.0 <= min_factor <= 1.0:
                raise ValueError("LRSchedule.min_factor must be in [0, 1]")
        self.warmup_steps, self.warmup_start, self.decay = warmup_steps, float(warmup_start), decay
        self.milestones, self.gamma, self.total_steps = milestones, float(gamma), total_steps
        self.min_factor, self.unit = float(min_factor), unit

    def resolve(self, steps_per_epoch: int) -> "LRSchedule":
        """The same schedule in step units (itself if it already is); epoch counts are rounded to the nearest step."""
        if self.unit == "step":
            return self
        if steps_per_epoch < 1:
            raise ValueError("LRSchedule.resolve: steps_per_epoch must be >= 1")
        r = lambda v: int(round(v * steps_per_epoch))   # noqa: E731
        return LRSchedule(r(self.warmup_steps), self.warmup_start, self.decay, tuple(r(m) for m in self.milestones),
                          self.gamma, None if self.total_steps is None else r(self.total_steps), self.min_factor)

    def _steps(self) -> "LRSchedule":
        if self.unit != "step":
            raise ValueError("LRSchedule in epoch units: call resolve(steps_per_epoch) first")
        return self

    def factor(self, s: int) -> float:
        """Multiplier of the base lr for the update applied after ``s`` updates (fp64, same operations as the kernels)."""
        self._steps()
        W = int(self.warmup_steps)
        if s < W:
            return self.warmup_start + (1.0 - self.warmup_start) * float(s) / float(W)
        f = 1.0
        if self.decay == "multistep":
            for m in self.milestones:
                if int(m) <= s:
                    f = f * self.gamma
        elif self.decay == "cosine":
            span = int(self.total_steps) - W
            d = min(s - W, span)
            f = self.min_factor + (1.0 - self.min_factor) * (1.0 + math.cos(math.pi * float(d) / float(span))) / 2.0
        return f

    def lr_at(self, base: float, s: int) -> float:
        """fp32 lr of the update applied after ``s`` updates: ``base`` (rounded to fp32) times :meth:`factor`, rounded once."""
        return _f32(_f32(float(base)) * self.factor(int(s)))

    def as_tuple(self) -> tuple:
        """The plain form the native bindings take: ``(kind, warmup, total, start, gamma, min_factor, milestones)``."""
        self._steps()
        return (_KINDS[self.decay], int(self.warmup_steps), int(self.total_steps or 0), self.warmup_start, self.gamma,
                self.min_factor, [int(m) for m in self.milestones])

    def to_dict(self) -> dict:
        return {"warmup_steps": self.warmup_steps, "warmup_start": self.warmup_start, "decay": self.decay,
                "milestones": list(self.milestones), "gamma": self.gamma, "total_steps": self.total_steps,
                "min_factor": self.min_factor, "unit": self.unit}

    @classmethod
    def from_dict(cls, d: dict) -> "LRSchedule":
        return cls(**d)

    def __eq__(self, other):
        return isinstance(other, LRSchedule) and self.to_dict() == other.to_dict()

    def __repr__(self):
        return "LRSchedule(" + ", ".join(f"{k}={v!r}" for k, v in self.to_dict().items()) + ")"


def schedule_tuple(schedule: Optional[LRSchedule]):
    """``schedule.as_tuple()`` for the native bindings, ``None`` without a schedule; rejects epoch units."""
    if schedule is None:
        return None
    if not isinstance(schedule, LRSchedule):
        raise TypeError(f"lr_schedule must be an LRSchedule or None, got {type(schedule).__name__}")
    if schedule.unit != "step":
        raise ValueError("trainers take an LRSchedule in step units: resolve(steps_per_epoch) it first")
    return schedule.as_tuple()


class FlatSGD:
    """``FlatSGD(model)`` where ``model`` is a plain module, a module carrying ``_grad_bucket`` or a
    :class:`DistributedDataParallel` wrapper.

    ``step()`` expects averaged gradients (call ``average_gradients(model)`` first, as the tutorial loop does) and,
    with ``zero_grad=True`` (default), leaves the buckets zeroed so no separate ``zero_grad()`` pass is needed;
    ``zero_grad()`` exists for loop compatibility and is then a no-op apart from re-arming the DDP hooks."""

    def __init__(self, model: nn.Module, lr: float = 0.01, momentum: float = 0.5, weight_decay: float = 0.0,
                 zero_grad: bool = True, group=None, lr_schedule: Optional[LRSchedule] = None):
        from ..parallel.ddp import DistributedDataParallel, GradBucket, flatten_params

        self.lr, self.momentum, self.weight_decay = float(lr), float(momentum), float(weight_decay)
        # lr_schedule: update k (k = `steps`, the updates applied so far) uses lr_schedule.lr_at(lr, k), computed on the host
        schedule_tuple(lr_schedule)
        self.lr_schedule, self.steps = lr_schedule, 0
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
        lr = self.lr_at()
        for gb, pf, mf in zip(self.buckets, self.param_flats, self.momentum_flats):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if pf.is_cuda and g.dtype == torch.float32:
                self._kernel().sgd_flat(pf, mf, g, lr, self.momentum, self.weight_decay, self.fused_zero)
                continue
            # CPU ranks (gloo) and reduced-precision gradient buckets: the same flat update with tensor ops
            gf = g.to(torch.float32)
            if self.weight_decay:
                gf = gf.add(pf, alpha=self.weight_decay)
            mf.mul_(self.momentum).add_(gf)
            pf.add_(mf, alpha=-lr)
            if self.fused_zero:
                g.zero_()
        self.steps += 1
        if self.fused_zero and self._engine is not None:
            self._engine._reset()

    def lr_at(self, step: Optional[int] = None) -> float:
        """The lr of the update applied after ``step`` updates (default: the next one, ``steps``)."""
        if self.lr_schedule is None:
            return self.lr
        return self.lr_schedule.lr_at(self.lr, self.steps if step is None else step)

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
        return {"lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay, "steps": self.steps,
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
        self.steps = int(sd.get("steps", self.steps))
        for m, src in zip(self.momentum_flats, sd["momentum_buffers"]):
            m.copy_(src)
