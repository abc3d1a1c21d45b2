"""Momentum SGD over flat buffers -- one launch per gradient bucket instead of one per tensor.

Parity: ``optim.SGD(model.parameters(), lr=0.01, momentum=0.5)`` + ``optimizer.step()`` + ``optimizer.zero_grad()``
of the reference's training loop (train_dist.py:110,118,123; tuto.md:283,291,296).  Same update rule as
``torch.optim.SGD`` (``buf = mu*buf + (g + wd*p)``, ``p -= lr*buf``, or ``p -= lr*(g + wd*p + mu*buf)`` with Nesterov;
dampening 0).

GPU-first: the gradients of a model already live in flat (symmetric-memory) buckets
(:class:`~dist_tuto.pth_b200.parallel.ddp.GradBucket`); this optimizer lays the parameters and the momentum out in flat
buffers with the *same* offsets and strides (``p.data`` becomes a view), so a whole bucket is updated -- and its
gradients re-zeroed for the next backward -- by ONE ``sgd_flat_kernel`` launch (csrc/sgd.cu) that streams the three
arrays once.  (The ConvNet goes further and fuses the all-reduce into the same kernel: ``allreduce_sgd_kernel``.)

``FlatSGD(..., sharded=True)`` does the same for generic models: per bucket ONE ``sharded_sgd_kernel`` launch
(csrc/sharded_sgd.cu) reduce-scatters the gradients, updates the slice of the parameters this rank owns and stores the new
parameters into every rank's flat, so the momentum exists for the owned slice only (optimizer state is 1/W per GPU) and no
separate update kernel runs.

``FlatAdamW`` is ``torch.optim.AdamW`` on the same flat layout: one ``adamw_flat_kernel`` launch per bucket (csrc/adamw.cu),
and with ``sharded=True`` the AdamW instance of the same sharded kernel, with both moments sharded.  Both optimizers share
the layout, the sharding, the exchange hooks and the step bookkeeping (``_FlatOptimizer``).

``FlatRMSprop`` is ``torch.optim.RMSprop`` on the same layout: one ``rmsprop_flat_kernel`` launch per bucket (csrc/rmsprop.cu),
and with ``sharded=True`` the RMSprop instances of the sharded kernel, with every state sharded.

``FlatSGD`` and ``FlatAdamW`` take torch-style ``param_groups`` (per-group lr and weight decay): the same launches with a
per-vector group map and the groups' scalars in the kernel arguments.

``FlatSGD(..., capturable=True)`` and ``FlatAdamW(..., capturable=True)`` keep the step counter, the lr schedule and AdamW's bias
corrections on the device (csrc/flat_scalars.cuh), so a whole DDP step can be captured in a CUDA graph and replayed.

``FlatAdafactor`` is ``torch.optim.Adafactor`` on the same layout: factored second moments (a row and a column vector per
weight matrix) and per-tensor step sizes, in three launches per bucket (csrc/adafactor.cu) over a chunk table of the layout.

``FlatLAMB`` and ``FlatLARS`` are the large-batch optimizers with a trust ratio per parameter tensor: per bucket two kernels
(csrc/layerwise.cu) form every tensor's norms in a fixed order over a chunk table of the flat layout, then apply the update.

``FlatEMA`` keeps an exponential moving average of the weights of any of them: one ``ema_update`` launch (csrc/ema.cu) over
the parameter flats (or this rank's slices of them when sharded) and the fp32 buffers per update.
"""
from __future__ import annotations

import contextlib
import math
import struct
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

__all__ = ["FlatSGD", "FlatAdamW", "FlatRMSprop", "FlatAdafactor", "FlatLAMB", "FlatLARS", "FlatEMA", "LRSchedule", "adamw_scalars",
           "rmsprop_scalars", "check_adafactor_options", "lamb_scalars", "exclude_1d", "check_sgd_options", "check_max_grad_norm", "MAX_PARAM_GROUPS"]

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


def check_sgd_options(momentum: float, weight_decay: float, nesterov: bool) -> None:
    """``torch.optim.SGD``'s rules for the options every engine shares (dampening is always 0 here)."""
    if not float(weight_decay) >= 0.0:
        raise ValueError(f"weight_decay must be >= 0, got {weight_decay}")
    if nesterov and float(momentum) == 0.0:
        raise ValueError("nesterov momentum needs a nonzero momentum")


def check_max_grad_norm(max_grad_norm) -> Optional[float]:
    """``torch.nn.utils.clip_grad_norm_``'s ``max_norm`` for every engine (the L2 norm only): ``None`` (no clipping) or a
    finite value > 0 that stays > 0 in fp32.  Returns it as a float (or ``None``)."""
    if max_grad_norm is None:
        return None
    if isinstance(max_grad_norm, bool) or not isinstance(max_grad_norm, (int, float)):
        raise ValueError(f"max_grad_norm must be None or a finite number > 0, got {max_grad_norm!r}")
    c = float(max_grad_norm)
    c32 = float(torch.tensor(c, dtype=torch.float32))
    if not (math.isfinite(c) and c > 0.0 and math.isfinite(c32) and c32 > 0.0):
        raise ValueError(f"max_grad_norm must be None or a finite number > 0, got {max_grad_norm!r}")
    return c


MAX_PARAM_GROUPS = 64                                        # csrc/param_groups.h: kMaxGroups
_GROUP_KEYS = ("params", "lr", "weight_decay")


def _check_param_groups(name: str, model: nn.Module, param_groups, lr: float, weight_decay: float, check) -> list:
    """``param_groups`` of :class:`FlatSGD` / :class:`FlatAdamW` checked before anything is allocated or laid out: a list of
    ``{"params", "lr", "weight_decay"}`` dicts, absent keys taking the constructor's values and ``check(lr, weight_decay)``
    applied to every group.  Raises ``ValueError`` for a parameter that is in no bucket of ``model`` or in two groups, an
    empty ``"params"``, any other key, a bad value, more than :data:`MAX_PARAM_GROUPS` groups (the default group of the
    parameters named in no group included), or a CUDA bucket with a tensor at an offset that is not a multiple of 4."""
    from ..parallel.ddp import DistributedDataParallel, flatten_params

    if isinstance(param_groups, dict) or not isinstance(param_groups, (list, tuple)):
        raise ValueError(f"{name}: param_groups must be a list of dicts, got {type(param_groups).__name__}")
    engine = model if isinstance(model, DistributedDataParallel) else getattr(model, "_ddp_engine", None)
    buckets = engine.buckets if engine is not None else [gb for gb in [getattr(model, "_grad_bucket", None)] if gb is not None]
    laid = [p for gb in buckets for p in gb.params] if buckets else flatten_params(model)
    known = {id(p) for p in laid}
    seen, out = set(), []
    for i, g in enumerate(param_groups):
        if not isinstance(g, dict):
            raise ValueError(f"{name}: param_groups[{i}] must be a dict, got {type(g).__name__}")
        for key in g:
            if key not in _GROUP_KEYS:
                raise ValueError(f"{name}: param_groups[{i}] has the key {key!r}; a group sets only 'lr' and 'weight_decay' "
                                 "(every other hyper-parameter is the optimizer's)")
        if "params" not in g:
            raise ValueError(f"{name}: param_groups[{i}] has no 'params'")
        params = [g["params"]] if isinstance(g["params"], torch.Tensor) else list(g["params"])
        if not params:
            raise ValueError(f"{name}: param_groups[{i}]['params'] is empty")
        for p in params:
            if id(p) not in known:
                raise ValueError(f"{name}: param_groups[{i}] names a parameter that is in no gradient bucket of the model")
            if id(p) in seen:
                raise ValueError(f"{name}: a parameter appears twice in param_groups (again in group {i})")
            seen.add(id(p))
        glr, gwd = float(g.get("lr", lr)), float(g.get("weight_decay", weight_decay))
        check(glr, gwd)
        out.append({"params": params, "lr": glr, "weight_decay": gwd})
    n = len(out) + (1 if len(seen) < len(known) else 0)
    if n > MAX_PARAM_GROUPS:
        raise ValueError(f"{name}: at most {MAX_PARAM_GROUPS} parameter groups, the default group of the parameters named in "
                         f"no group included; got {n}")
    for gb in buckets:
        if gb.flat.is_cuda and any(o % 4 for o in gb.offsets):
            raise ValueError(f"{name}: param_groups on CUDA need every tensor of a bucket at a multiple of 4 elements (the "
                             "group map has one id per 16-byte parameter vector); build the buckets with align=4")
    return out


def _group_attr(key: str):
    """``lr`` / ``weight_decay`` of FlatSGD and FlatAdamW: the default group's values (``param_groups[-1]``)."""
    return property(lambda self: self._default_group[key], lambda self, v: self._default_group.__setitem__(key, float(v)))


def _fp32_grad(g: torch.Tensor, grad_scale: Optional[torch.Tensor]) -> torch.Tensor:
    """The gradient a torch-op update reads: ``g`` in fp32, and with GradScaler's ``grad_scale`` S times
    ``inv = fp32(1 / double(S))``, computed as ``GradScaler.unscale_`` computes it (a new tensor: ``g`` keeps the scaled
    values)."""
    gf = g.to(torch.float32)
    return gf if grad_scale is None else gf * grad_scale.double().reciprocal().float()


def _peer_world(gb) -> bool:
    """Does this gradient bucket live in the symmetric memory of ONE peer-memory world (not the two-level world of several
    machines), in a dtype ``sharded_sgd_kernel`` reduces?"""
    if gb.symm_handle is None or not gb.flat.is_cuda or gb.flat.dtype not in (torch.float32, torch.bfloat16):
        return False
    from ..parallel import symm

    return isinstance(gb.world, symm.SymmWorld)


class _FlatOptimizer:
    """What :class:`FlatSGD` and :class:`FlatAdamW` share: the flat fp32 parameter layout over the gradient buckets (``p.data``
    becomes a view with the gradient view's offset and strides), the shard padding and the symmetric parameter flats of
    ``sharded=True``, the registration of the sharded update with the buckets' exchange, the ``step()`` bookkeeping, the lr
    schedule, on-device gradient-norm clipping, and the gathering and slicing of per-bucket optimizer state.  A subclass
    allocates its state flats (:meth:`_state_flat`) and updates a whole bucket (``_update``), a bucket in one peer-memory
    kernel (``_sharded_kernel``) or the owned slice of a bucket with torch ops (``_update_slice``).

    fp16 loss scaling: ``torch.amp.GradScaler.step(opt)`` sees ``_step_supports_amp_scaling`` and, after its own check for
    non-finite gradients, sets ``grad_scale`` (the loss scale S, or ``None`` after an explicit ``scaler.unscale_(opt)``) and
    ``found_inf`` on the optimizer, calls :meth:`step` and deletes both; see :meth:`step`."""

    # torch.amp.GradScaler hands this optimizer grad_scale / found_inf instead of unscaling and syncing itself
    _step_supports_amp_scaling = True

    def __init__(self, model: nn.Module, zero_grad: bool, group, lr_schedule: Optional[LRSchedule],
                 max_grad_norm: Optional[float], sharded: bool, param_groups: Optional[list] = None,
                 capturable: bool = False):
        from .. import comm
        from ..parallel.ddp import DistributedDataParallel, GradBucket, flatten_params

        name = type(self).__name__
        self.capturable = bool(capturable)
        self.sharded = bool(sharded)
        if self.sharded and max_grad_norm is not None:
            raise ValueError(f"{name}(sharded=True) cannot clip: the total norm needs every bucket reduced before any update, "
                             "and the sharded update runs bucket by bucket during backward; use sharded=False with max_grad_norm")
        self.max_grad_norm = check_max_grad_norm(max_grad_norm)
        self._grad_norm = None           # the last update's pre-clip norm (a 0-dim / [1] tensor), see grad_norm()
        self._clip_bufs = None           # kernel path: (fp64 [buckets] squares, grad_sqnorm workspace, fp32 [1] norm)
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
        # sharded over more than one rank: "kernel" (one peer-memory kernel per bucket on a symmetric CUDA world) or "torch";
        # None: every rank holds and updates everything
        self._group = self._engine.group if self._engine is not None else self.buckets[0].group
        self._world, self._rank = comm.get_world_size(self._group), comm.get_rank(self._group)
        self._shard_mode = None
        if self.sharded and self._world > 1:
            self._shard_mode = "kernel" if all(_peer_world(gb) for gb in self.buckets) else "torch"
        self._check_shard_mode()         # before any parameter is rebound or hook registered
        self._shards: List[tuple] = []   # per bucket: (gradient vectors, padded elements, elements per rank, whole parameter flat, its handle)
        self._done = [False] * len(self.buckets)
        for gb in self.buckets:
            p0 = gb.params[0]
            if any(p.dtype != torch.float32 for p in gb.params):
                raise TypeError(f"{name} keeps fp32 master parameters; cast activations (autocast), not the parameters")
            if self._shard_mode is None:
                pf = torch.zeros(gb.numel, dtype=torch.float32, device=p0.device)
            else:
                # padded like the gradient bucket to W equal slices of whole 16-byte gradient vectors
                es = gb.flat.element_size()
                n_vec = ((gb.flat.numel() * es + 15) // 16 + self._world - 1) // self._world * self._world
                n_pad = n_vec * (16 // es)
                handle = None
                if self._shard_mode == "kernel":     # symmetric, so that the owners of the other slices can store into it
                    handle = gb.world.alloc_bytes(n_pad * 4, ll=False)
                    full = handle.view(torch.float32, n_pad)
                else:
                    full = torch.zeros(n_pad, dtype=torch.float32, device=p0.device)
                self._shards.append((n_vec, n_pad, n_pad // self._world, full, handle))
                pf = full[:gb.numel]
            with torch.no_grad():
                for p, o, gv in zip(gb.params, gb.offsets, gb.views):
                    pv = pf[o:o + p.numel()].as_strided(gv.shape, gv.stride())   # same layout as the gradient view
                    pv.copy_(p.data)
                    p.data = pv
            self.param_flats.append(pf)
            if self._shard_mode is not None:
                gb.sharded_step = lambda max_blocks=None, k=len(self.param_flats) - 1: self._sharded_step(k, max_blocks)
        self._native = None
        self._names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        self._set_groups(param_groups)
        if self.capturable:
            self._init_capturable(name)

    def _check_shard_mode(self) -> None:
        """Raise if this optimizer has no update for ``_shard_mode``; every mode is supported here."""

    # ------------------------------------------------------------------ capturable: step counter and scalars on the device
    def _init_capturable(self, name: str) -> None:
        """``capturable=True``: refuse every bucket a torch-op path would update (its host scalars would be frozen by a graph),
        then allocate the extension, the clip buffers, the device step counter, the hyper-parameter table and the scalar
        block (csrc/flat_scalars.h), and fill the block of the first update."""
        for gb, pf in zip(self.buckets, self.param_flats):
            if not pf.is_cuda:
                raise ValueError(f"{name}(capturable=True) needs CUDA parameters; CPU (gloo) updates run torch ops on the host")
            if self._shard_mode is None and gb.flat.dtype != torch.float32:
                raise ValueError(f"{name}(capturable=True) needs fp32 gradient buckets unless sharded=True: a {gb.flat.dtype} "
                                 "bucket is updated by torch ops whose scalars a CUDA graph would freeze")
        if self._shard_mode == "torch":
            raise ValueError(f"{name}(capturable=True, sharded=True) needs one peer-memory world (backend 'b200' on one "
                             "machine): elsewhere the sharded update runs torch ops whose scalars a CUDA graph would freeze")
        C = self._kernel()
        lay = C.flat_scalars_layout()
        dev = self.param_flats[0].device
        if self.max_grad_norm is not None:
            self._clip_bufs = (torch.zeros(len(self.buckets), dtype=torch.float64, device=dev),
                               torch.zeros(C.grad_sqnorm_workspace_numel(), dtype=torch.float32, device=dev),
                               torch.zeros(1, dtype=torch.float32, device=dev))
        self._cap_counter = torch.zeros(1, dtype=torch.int64, device=dev)
        self._cap_table = torch.zeros(lay["table_bytes"], dtype=torch.uint8, device=dev)
        self._cap_block = torch.zeros(lay["block_bytes"], dtype=torch.uint8, device=dev)
        self._cap_synced = None
        self._sync_device(steps=self._steps)

    def _hyper(self) -> tuple:
        """What the device table holds: every group's base lr and weight decay, the AdamW constants and the schedule."""
        groups = self._group_list
        b1, b2 = getattr(self, "betas", (0.0, 0.0))
        return ([float(g["lr"]) for g in groups], [float(g["weight_decay"]) for g in groups], float(b1), float(b2),
                float(getattr(self, "eps", 0.0)), schedule_tuple(self.lr_schedule))

    def _sync_device(self, steps: Optional[int] = None) -> None:
        """Upload the table (and with ``steps`` the counter) and refill the block; refused inside a capture, which would
        replay this call's values."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"{type(self).__name__}: the hyper-parameters and the step counter of a capturable optimizer are "
                               "uploaded outside a CUDA-graph capture (call sync_hyperparameters() or set steps before "
                               "capturing or between replays)")
        h = self._hyper()
        self._kernel().flat_scalars_sync(self._cap_table, self._cap_counter, self._cap_block, *h, steps=steps)
        self._cap_synced = h

    def _cap_refresh(self) -> None:
        """Before an eager capturable update: upload the hyper-parameters if one changed since the last upload.  Inside a
        capture nothing is uploaded (the replays use the table as it stands)."""
        if not torch.cuda.is_current_stream_capturing() and self._hyper() != self._cap_synced:
            self._sync_device()

    @property
    def steps(self) -> int:
        """Updates applied so far.  With ``capturable=True`` it is the device counter (reading it synchronises; assigning it
        writes the counter and recomputes the next update's scalars, and raises ``RuntimeError`` inside a capture), so it
        counts graph replays too."""
        if getattr(self, "_cap_counter", None) is not None:
            return int(self._cap_counter.item())
        return self._steps

    @steps.setter
    def steps(self, value: int) -> None:
        if getattr(self, "_cap_counter", None) is not None:
            self._sync_device(steps=int(value))
        else:
            self._steps = int(value)

    # ------------------------------------------------------------------ parameter groups
    def _set_groups(self, given: Optional[list]) -> None:
        """The group layout of ``given`` (checked groups, or None: no groups).  ``_group_list`` holds the groups the updates
        read -- the given ones in order, then the default group if any parameter is in none; without ``given`` the default
        group alone -- and per bucket ``_tensor_groups[k]`` the group of each tensor and ``_runs[k]`` cuts ``[0, numel)``
        into ``(lo, hi, group)`` runs: each tensor's padded segment takes its tensor's group, and adjacent segments of one
        group merge (without ``given``, one run ``(0, numel, 0)``).  With ``given``, the kernel paths also get a uint8 group
        map with one id per fp32 parameter vector: the whole bucket, or this rank's slice of the padded flat (padding in the
        last group)."""
        self._grouped = given is not None
        given = list(given or [])
        self._runs, self._tensor_groups, self._maps = [], [], []
        gid = {}
        for i, g in enumerate(given):
            for p in g["params"]:
                gid[id(p)] = i
        rest = [p for gb in self.buckets for p in gb.params if id(p) not in gid]
        self._default_group["params"] = rest
        self._group_list = given + ([self._default_group] if rest else [])
        for p in rest:
            gid[id(p)] = len(given)
        n_groups = len(self._group_list)
        for k, (gb, pf) in enumerate(zip(self.buckets, self.param_flats)):
            runs = []
            for i, (p, o) in enumerate(zip(gb.params, gb.offsets)):
                lo, hi = (0 if i == 0 else o), (gb.offsets[i + 1] if i + 1 < len(gb.params) else gb.numel)
                if runs and runs[-1][2] == gid[id(p)]:
                    runs[-1][1] = hi
                else:
                    runs.append([lo, hi, gid[id(p)]])
            self._runs.append([tuple(r) for r in runs])
            self._tensor_groups.append([gid[id(p)] for p in gb.params])
            if not self._grouped:
                continue
            if self._shard_mode == "kernel":
                n_pad, per = self._shards[k][1], self._shards[k][2]
                whole = self._group_map(runs + [[gb.numel, n_pad, n_groups - 1]], n_pad // 4, n_groups)
                self._maps.append(whole[self._rank * per // 4:(self._rank + 1) * per // 4].to(pf.device))
            elif self._shard_mode is None and pf.is_cuda and gb.flat.dtype == torch.float32:
                self._maps.append(self._group_map(runs, (gb.numel + 3) // 4, n_groups).to(pf.device))
            else:
                self._maps.append(None)

    @staticmethod
    def _group_map(runs: list, n_vec: int, n_groups: int) -> torch.Tensor:
        """One uint8 group id per 16-byte fp32 vector of ``runs`` (element runs at multiples of 4), checked against the
        number of groups before it is used."""
        ids = torch.tensor([r[2] for r in runs if r[1] > r[0]], dtype=torch.int64)
        lens = torch.tensor([(min(r[1], 4 * n_vec) + 3) // 4 - r[0] // 4 for r in runs if r[1] > r[0]], dtype=torch.int64)
        m = torch.repeat_interleave(ids, lens)
        if m.numel() != n_vec or (m.numel() and not (0 <= int(m.min()) and int(m.max()) < n_groups <= MAX_PARAM_GROUPS)):
            raise ValueError(f"group map of {m.numel()} ids for {n_vec} vectors, or an id outside [0, {n_groups})")
        return m.to(torch.uint8)

    def _group_values(self) -> list:
        """``(lr, weight_decay)`` of every group for the next update: ``lr_schedule.lr_at(group lr, steps)`` with a schedule."""
        s = self.lr_schedule
        return [(s.lr_at(g["lr"], self.steps) if s is not None else float(g["lr"]), float(g["weight_decay"]))
                for g in self._group_list]

    def _slice_runs(self, k: int, lo: int, n: int) -> list:
        """Bucket ``k``'s runs cut to ``[lo, lo + n)``, as ``(start, end, group)`` relative to ``lo``."""
        out = []
        for a, b, g in self._runs[k]:
            a, b = max(a, lo), min(b, lo + n)
            if a < b:
                out.append((a - lo, b - lo, g))
        return out

    def _run_views(self, runs: list, flats: list):
        """Per group in group order, as torch's optimizers step their groups: ``(lr, weight_decay, views)``, ``views[j]`` the
        group's ``(lo, hi, group)`` runs of ``flats[j]`` (``[]`` for a ``None`` flat)."""
        for gi, (lr, wd) in enumerate(self._group_values()):
            mine = [(lo, hi) for lo, hi, g in runs if g == gi]
            if mine:
                yield lr, wd, [[f[lo:hi] for lo, hi in mine] if f is not None else [] for f in flats]

    def _tensor_views(self, k: int, flats: list, nonempty: bool = False):
        """Per group in group order: ``(lr, weight_decay, idx, views)``, ``idx`` the group's tensors of bucket ``k``
        (``nonempty``: those with an element) and ``views[j]`` their views of ``flats[j]`` (``[]`` for a ``None`` flat), each
        with its tensor's own shape and strides, as torch's optimizers see the tensors."""
        gb = self.buckets[k]
        views = [[f[o:o + p.numel()].as_strided(gv.shape, gv.stride()) for p, o, gv in zip(gb.params, gb.offsets, gb.views)]
                 if f is not None else None for f in flats]
        for gi, (lr, wd) in enumerate(self._group_values()):
            idx = [i for i, x in enumerate(self._tensor_groups[k]) if x == gi and (gb.params[i].numel() > 0 or not nonempty)]
            if idx:
                yield lr, wd, idx, [[vs[i] for i in idx] if vs is not None else [] for vs in views]

    @property
    def param_groups(self) -> list:
        """The parameter groups, as torch's optimizers list them: the ``param_groups`` given to the constructor in order,
        then the default group of the parameters named in none (``lr`` / ``weight_decay`` are the optimizer's ``lr`` /
        ``weight_decay``).  Each is a dict with ``"params"``, ``"lr"`` and ``"weight_decay"``; every update reads the values,
        so assigning to them works as in torch.  Without ``param_groups`` it is the one default group."""
        return list(self._group_list)

    def _group_state(self) -> dict:
        """What a state_dict records of the groups: ``{"param_groups": [{"params": [names], "lr", "weight_decay"}]}``."""
        if not self._grouped:
            return {}
        return {"param_groups": [{"params": [self._names.get(id(p), "") for p in g["params"]], "lr": float(g["lr"]),
                                  "weight_decay": float(g["weight_decay"])} for g in self._group_list]}

    def _load_group_state(self, sd: dict, apply: bool = True) -> None:
        """The groups' lr / weight_decay from ``sd["param_groups"]``; ``ValueError`` if its membership is not this optimizer's
        (``apply=False``: only that check).  A state_dict without the key (written without groups) leaves the groups as built."""
        saved = sd.get("param_groups")
        if saved is None:
            return
        mine = self.param_groups if hasattr(self, "_default_group") else [{"params": [p for gb in self.buckets for p in gb.params]}]
        names = [sorted(self._names.get(id(p), "") for p in g["params"]) for g in mine]
        if names != [sorted(g["params"]) for g in saved]:
            raise ValueError(f"{type(self).__name__}.load_state_dict: the state_dict's parameter groups hold other parameters "
                             f"than this optimizer's ({len(saved)} saved groups, {len(mine)} here)")
        if not apply:
            return
        if not self._grouped:                  # one group with every parameter: the optimizer's own lr / weight_decay
            self.lr, self.weight_decay = float(saved[0]["lr"]), float(saved[0]["weight_decay"])
            return
        for g, s in zip(self._group_list, saved):
            g["lr"], g["weight_decay"] = float(s["lr"]), float(s["weight_decay"])

    def _state_flat(self, k: int) -> torch.Tensor:
        """A zero fp32 state flat for bucket ``k``: the whole flat, or this rank's shard of it when sharded."""
        pf = self.param_flats[k]
        if self._shard_mode is None:
            return torch.zeros_like(pf)
        return torch.zeros(self._shards[k][2], dtype=torch.float32, device=pf.device)

    # ------------------------------------------------------------------ update
    def _kernel(self):
        if self._native is None:
            from . import _ext

            self._native = _ext.C()        # raises if the extension is missing: no silent fallback on a GPU box
        return self._native

    @torch.no_grad()
    def step(self) -> None:
        """``optimizer.step()`` (train_dist.py:124) for every bucket, and -- with ``zero_grad=True`` -- the
        ``optimizer.zero_grad()`` of the next iteration (train_dist.py:118) in the same pass.  Called by
        ``torch.amp.GradScaler.step`` (``grad_scale`` / ``found_inf`` set), it is torch's ``unscale_`` + step:
        every gradient the update reads -- the clipping norm and the LAMB / LARS norms included -- is ``g * inv`` with
        ``inv = fp32(1 / double(S))``, and when ``found_inf != 0`` the step is skipped: no parameter, state, trust ratio or
        ``grad_norm`` is written and ``steps`` does not advance, but with ``zero_grad=True`` the buckets are still zeroed
        and the hooks re-armed.  ``capturable=True`` decides on the device with no host synchronisation; otherwise
        ``found_inf`` is read once (one synchronisation, as GradScaler makes with a ``torch.optim`` optimizer).  Sharded
        over more than one rank it raises ``RuntimeError``."""
        if getattr(self, "_ema_swapped", False):
            raise RuntimeError(f"{type(self).__name__}.step() inside FlatEMA.average_parameters(): the parameters hold the "
                               "EMA values there; step after the block")
        scale, found_inf = getattr(self, "grad_scale", None), getattr(self, "found_inf", None)
        if self._shard_mode is not None and (scale is not None or found_inf is not None):
            raise RuntimeError(f"{type(self).__name__}(sharded=True) over {self._world} ranks cannot take GradScaler's step: the "
                               "gradient exchange already applied this step's update with the scaled gradient during backward, "
                               "before any overflow check.  fp16 loss scaling needs sharded=False")
        if self._shard_mode is not None:      # the buckets' exchanges applied the update already
            if not all(self._done):
                raise RuntimeError(f"{type(self).__name__}(sharded=True).step(): this step's gradient buckets were not "
                                   "exchanged; call average_gradients(model) after backward() (one average_gradients per step)")
            self._done = [False] * len(self.buckets)
            if self.capturable:
                self._advance()
            else:
                self.steps += 1
            if self._engine is not None:
                self._engine._reset()
            return
        if self._engine is not None and self._engine._unexchanged():
            raise RuntimeError(f"{type(self).__name__}.step(): gradients accumulated under no_sync() were never exchanged; "
                               "run the last micro-batch's backward outside no_sync(), or call average_gradients(model), "
                               "before step()")
        # Unsharded, every rank holds the same averaged gradient bit for bit (the exchange sums in a fixed rank order), so
        # GradScaler's check finds the same found_inf on every rank and all ranks skip or apply together, with no collective.
        if self.capturable:
            self._cap_refresh()
            kw = {} if found_inf is None else dict(grad_scale=scale, found_inf=found_inf)
            if self.max_grad_norm is not None:
                kw.update(self._clip_on_device(scale))
            self._update_capturable(kw)
            self._advance(found_inf)
            if self.fused_zero and self._engine is not None:
                self._engine._reset()
            return
        if found_inf is not None and float(found_inf) != 0.0:      # the one host synchronisation of an eager scaled step
            if self.fused_zero:
                for gb in self.buckets:
                    gb.flat[:gb.numel].zero_()
                if self._engine is not None:
                    self._engine._reset()
            return
        kernel = [pf.is_cuda and gb.flat.dtype == torch.float32 for gb, pf in zip(self.buckets, self.param_flats)]
        kw = {} if scale is None else {"grad_scale": scale}
        if self.max_grad_norm is not None:
            if all(kernel):
                kw.update(self._clip_on_device(scale))
            else:                        # every bucket by torch itself, before any update
                params = []
                for gb in self.buckets:
                    gb.attach()          # p.grad is the bucket's view, so the clip scales the bucket in place
                    params += gb.params
                    if scale is not None:                  # GradScaler.unscale_'s own op, in place, before the clip
                        torch._amp_foreach_non_finite_check_and_unscale_(
                            [gb.flat[:gb.numel]], torch.zeros((), device=scale.device), scale.double().reciprocal().float())
                kw = {}
                self._grad_norm = torch.nn.utils.clip_grad_norm_(params, self.max_grad_norm, foreach=False)
                kernel = [False] * len(kernel)
        self._update(kernel, kw)
        self.steps += 1
        if self.fused_zero and self._engine is not None:
            self._engine._reset()

    @torch.no_grad()
    def _sharded_step(self, k: int, max_blocks: Optional[int] = None) -> None:
        """Bucket ``k``'s gradient exchange and update in sharded mode (``GradBucket.exchange_`` calls it on the stream the
        all-reduce would run on): afterwards every rank holds the updated parameters of the whole bucket."""
        from .. import comm

        if getattr(self, "_ema_swapped", False):
            raise RuntimeError(f"{type(self).__name__}(sharded=True): a gradient exchange inside FlatEMA.average_parameters() "
                               "would update the EMA values the parameters hold there; run backward after the block")
        if self._done[k]:
            raise RuntimeError(f"{type(self).__name__}(sharded=True): a gradient bucket was exchanged twice in one step, which "
                               "would apply its update twice; one average_gradients(model) goes with one step()")
        gb = self.buckets[k]
        per, full = self._shards[k][2], self._shards[k][3]
        if self._shard_mode == "kernel":
            if self.capturable:                 # the scalars the previous step() computed, with any new group values
                self._cap_refresh()
            self._sharded_kernel(k, gb.world.max_blocks if max_blocks is None else max_blocks)
        else:
            gb.all_reduce_average_(max_blocks)
            lo = self._rank * per
            n = min(lo + per, gb.flat.numel()) - lo          # the rest of the slice is padding no gradient exists for
            if n > 0:                                        # the unsharded update (step()), on the owned slice
                self._update_slice(k, lo, n)
            comm.all_gather_into_tensor(full, full[lo:lo + per].clone(), group=self._group)
            if self.fused_zero:
                gb.flat.zero_()
        self._done[k] = True

    def _sync_hyperparameters(self) -> None:
        """``capturable=True``: upload the groups' ``lr`` / ``weight_decay`` (and ``lr_schedule``) to the device table and
        recompute the next update's scalars from it: two non-blocking copies from pinned memory and one launch on the current
        stream.  An eager ``step()`` does this by itself when a value changed; a CUDA graph replays the table as it stands, so
        after assigning a new lr between replays call this outside the capture (as with torch's capturable optimizers, whose
        lr must be a tensor to change under a graph).  ``RuntimeError`` inside a capture.  Without ``capturable`` it does
        nothing."""
        if self.capturable:
            self._sync_device()

    def _advance(self, found_inf: Optional[torch.Tensor] = None) -> None:
        """capturable: counter += 1 and the scalars of the next update, one single-CTA launch after this step's updates;
        with GradScaler's ``found_inf`` nothing changes when it is nonzero."""
        self._kernel().flat_scalars_advance(self._cap_table, self._cap_counter, self._cap_block, found_inf=found_inf)

    def _cap_map(self, k: int) -> Optional[torch.Tensor]:
        return self._maps[k] if self._grouped else None

    def shard_range(self, k: int) -> tuple:
        """``(lo, hi)``: the elements of bucket ``k``'s flat this rank owns (updates, and holds the optimizer state of);
        everything when the optimizer is not sharded over several ranks."""
        numel = self.buckets[k].numel
        if self._shard_mode is None:
            return 0, numel
        per = self._shards[k][2]
        return min(self._rank * per, numel), min((self._rank + 1) * per, numel)

    # ------------------------------------------------------------------ checkpointing
    # A subclass declares what differs: _state_pairs() gives (state_dict key, flats) of every state buffer (flats empty for
    # a state its configuration does not keep); _options names the options a state_dict records besides max_grad_norm and
    # steps; _check_options(sd) raises ValueError unless its constructor would take the options of sd, and returns the
    # attributes loading them sets; _defaults() and _state_views() where they differ from these.
    _noun = "state"                                        # what the buffers hold, in the refusal of another rank's shard
    _carry = "named_state() / load_named_state()"          # the per-name form that crosses world sizes and layouts
    # the per-name loader's refusal of an entry without a part its tensor's state needs
    _lacks = "{cls}.load_named_state: the entry of {name!r} has no {key!r}; the state is not this optimizer's"

    def _defaults(self) -> dict:
        """The values of the keys that state_dicts written before their option existed lack."""
        return {"max_grad_norm": None}

    def state_dict(self) -> dict:
        """The options, ``max_grad_norm``, ``steps`` and the state flats (CPU copies), for
        ``utils.checkpoint.save_checkpoint``.  Sharded over several ranks, the buffers are this rank's shards, and
        ``sharded`` / ``world`` / ``rank`` say so; with ``param_groups`` the groups are recorded by parameter name.  The form
        that crosses world sizes and engines is the per-name one (``named_state`` or ``named_momentum``)."""
        sd = {key: getattr(self, key) for key in self._options}
        sd.update(max_grad_norm=self.max_grad_norm, steps=self.steps)
        sd.update((key, [f.detach().cpu().clone() for f in flats]) for key, flats in self._state_pairs())
        sd.update(self._shard_tags())
        sd.update(self._group_state())
        return sd

    def load_state_dict(self, sd: dict) -> None:
        """Inverse of :meth:`state_dict` (same model => same bucket layout); a state_dict with ``param_groups`` restores each
        group's lr / weight_decay.  ``ValueError``, before anything is loaded, if its groups hold other parameters than this
        optimizer's, its options are ones the constructor refuses or that decide other states, its buffers are the shards of
        another rank or world size, or they have other numbers or sizes."""
        sd = {**self._defaults(), **sd}
        self._load_group_state(sd, apply=False)
        options = self._check_options(sd)
        max_grad_norm, steps = check_max_grad_norm(sd["max_grad_norm"]), int(sd["steps"])
        self._check_shard_tags(sd, self._noun, self._carry)
        whole = self._shard_mode is not None and not sd.get("sharded")    # each rank will take its slice of whole buffers
        for key, flats in self._state_pairs():
            if [s.numel() for s in sd[key]] != [self.buckets[k].numel if whole else f.numel() for k, f in enumerate(flats)]:
                raise ValueError(f"{type(self).__name__}.load_state_dict: the state flats have other sizes than this "
                                 f"optimizer's (another model or bucket layout); carry the state with {self._carry}")
        self._load_flats(sd, [(flats, sd[key]) for key, flats in self._state_pairs()], self._noun, self._carry)
        for attr, value in options.items():
            setattr(self, attr, value)
        self.max_grad_norm, self.steps = max_grad_norm, steps
        self._load_group_state(sd)
        self._sync_hyperparameters()

    def _full_flat(self, k: int, flat: torch.Tensor) -> torch.Tensor:
        """Bucket ``k``'s whole state flat of which ``flat`` is this rank's part; collective in sharded mode (gathers)."""
        from .. import comm

        if self._shard_mode is None:
            return flat
        full = torch.empty_like(self._shards[k][3])
        comm.all_gather_into_tensor(full, flat, group=self._group)
        return full

    def _flat_views(self, k: int, flat: torch.Tensor, i: int, key: str) -> dict:
        """``{key: tensor i's part of flat}``, ``flat`` a whole flat of bucket ``k`` laid out as the parameters, the part with
        the tensor's shape and strides."""
        gb = self.buckets[k]
        o, gv = gb.offsets[i], gb.views[i]
        return {key: flat[o:o + gv.numel()].as_strided(gv.shape, gv.stride())}

    _state_views = _flat_views           # the per-tensor parts of a state flat, as the per-name forms hold them

    def _named_parts(self, model: nn.Module, pairs: list, views) -> dict:
        """``{parameter name: {part: CPU copy}}`` of the parts ``views(k, whole flat, i, key)`` of every tensor in the flats of
        ``pairs`` = ``[(key, flats)]``; collective in sharded mode (gathers the flats)."""
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        out = {}
        for key, flats in pairs:
            for k, gb in enumerate(self.buckets):
                full = self._full_flat(k, flats[k])
                for i, p in enumerate(gb.params):
                    if id(p) in names:
                        parts = views(k, full, i, key).items()
                        out.setdefault(names[id(p)], {}).update((x, v.detach().cpu().clone()) for x, v in parts)
        return out

    @torch.no_grad()
    def _load_parts(self, model: nn.Module, named: dict, pairs: list, views) -> int:
        """Inverse of :meth:`_named_parts`; returns how many tensors were restored.  ``ValueError`` (:attr:`_lacks`), before
        anything is written, if an entry lacks a part of its tensor.  Sharded over several ranks, each rank keeps its slice of
        the full tensors (not collective)."""
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        sharded = self._shard_mode is not None
        for check in (True, False):            # every entry is checked before the first write
            for key, flats in pairs:
                for k, (gb, mf) in enumerate(zip(self.buckets, flats)):
                    if sharded:                    # lay the tensors out in a whole flat, then cut this rank's slice out
                        shard = mf             # (the check needs the parts' names and shapes only: a meta flat)
                        mf = torch.zeros_like(self._shards[k][3], device="meta" if check else None)
                        given = torch.zeros_like(mf, dtype=torch.bool)
                    for i, (p, o) in enumerate(zip(gb.params, gb.offsets)):
                        src = named.get(names.get(id(p)))
                        parts = views(k, mf, i, key) if src is not None else {}
                        missing = [x for x in parts if x not in src]
                        if missing:
                            raise ValueError(self._lacks.format(cls=type(self).__name__, name=names[id(p)], key=missing[0],
                                                                keys=" / ".join(parts)))
                        if parts and not check:
                            for x, v in parts.items():
                                v.copy_(src[x])
                            if sharded:
                                given[o:o + p.numel()] = True
                    if sharded and not check:
                        lo, per = self._rank * self._shards[k][2], self._shards[k][2]
                        shard.copy_(torch.where(given[lo:lo + per], mf[lo:lo + per], shard))
        return sum(named.get(names.get(id(p))) is not None for gb in self.buckets for p in gb.params)

    def _named(self, model: nn.Module, flats: List[torch.Tensor]) -> dict:
        """``{parameter name: its part of the flats}`` (CPU copies), the flats laid out as the parameters; collective in
        sharded mode."""
        return {n: parts["flat"] for n, parts in self._named_parts(model, [("flat", flats)], self._flat_views).items()}

    def _load_named(self, model: nn.Module, named: dict, flats: List[torch.Tensor]) -> int:
        """Inverse of :meth:`_named`; returns how many tensors were restored.  Sharded over several ranks, each rank keeps its
        slice of the full tensors (not collective)."""
        return self._load_parts(model, {n: {"flat": t} for n, t in named.items()}, [("flat", flats)], self._flat_views)

    def _named_state(self, model: nn.Module) -> dict:
        """``{name: {"step", <state>: tensor, ...}}`` (CPU copies), the torch optimizer's per-parameter state by parameter
        name: the form that crosses world sizes, bucket layouts, sharded and unsharded runs and the torch optimizer.  Sharded
        over several ranks this is collective: every rank calls it and gets the full tensors."""
        step = float(self.steps)
        parts = self._named_parts(model, [(key, flats) for key, flats in self._state_pairs() if flats], self._state_views)
        return {n: {"step": torch.tensor(step), **s} for n, s in parts.items()}

    def _load_named_state(self, model: nn.Module, named: dict) -> int:
        """Inverse of :meth:`named_state`; returns how many parameters' state was restored and sets ``steps`` from their
        (common) ``step``.  ``ValueError``, before anything is loaded, if the steps differ or an entry lacks a state its
        parameter needs.  Sharded over several ranks, each rank keeps its slice (not collective)."""
        steps = {int(s["step"]) for s in named.values()}
        if len(steps) > 1:
            raise ValueError(f"{type(self).__name__} keeps one step count for all parameters; this state has steps "
                             f"{sorted(steps)}")
        pairs = [(key, flats) for key, flats in self._state_pairs() if flats]
        for key, _ in pairs if self._state_views == self._flat_views else []:     # states kept whole: every entry has each
            lacking = [n for n, s in named.items() if key not in s]
            if lacking:
                raise ValueError(self._lacks.format(cls=type(self).__name__, name=lacking[0], key=key, keys=key))
        done = self._load_parts(model, named, pairs, self._state_views)
        if done and steps:
            self.steps = steps.pop()
        return done

    def _shard_tags(self) -> dict:
        """What a state_dict records when its buffers are one rank's shards."""
        return dict(sharded=True, world=self._world, rank=self._rank) if self._shard_mode is not None else {}

    def _check_shard_tags(self, sd: dict, noun: str, carry: str) -> None:
        """``ValueError`` if the buffers of ``sd`` are shards that do not load here: shards load on their own rank of their
        own world size only.  ``noun`` names the state and ``carry`` the per-name methods that cross world sizes."""
        if sd.get("sharded") and (self._shard_mode is None or (sd["world"], sd["rank"]) != (self._world, self._rank)):
            raise ValueError(f"this state_dict holds the {noun} shard of rank {sd['rank']} of {sd['world']}; it loads "
                             f"into a sharded {type(self).__name__} on that rank of a world of that size only.  To change "
                             f"the world size or the engine, carry the {noun} with {carry}")

    @torch.no_grad()
    def _load_flats(self, sd: dict, pairs: list, noun: str, carry: str) -> None:
        """The buffers of ``sd`` into the state flats, ``pairs`` = [(flats, saved buffers)]: shards load on their own rank of
        their own world size only (:meth:`_check_shard_tags`); whole buffers of an unsharded optimizer load into a sharded
        one as this rank's slice."""
        self._check_shard_tags(sd, noun, carry)
        if self._shard_mode is not None and not sd.get("sharded"):   # whole buffers of an unsharded optimizer: the slice
            for flats, saved in pairs:
                for k, (m, src) in enumerate(zip(flats, saved)):
                    per = self._shards[k][2]
                    whole = torch.zeros(self._shards[k][1], dtype=torch.float32)
                    whole[:src.numel()].copy_(src)
                    m.copy_(whole[self._rank * per:(self._rank + 1) * per])
            return
        for flats, saved in pairs:
            for m, src in zip(flats, saved):
                m.copy_(src)

    def _clip_on_device(self, grad_scale: Optional[torch.Tensor] = None) -> dict:
        """Every bucket's sum of squares (of the unscaled gradient with GradScaler's ``grad_scale``) into the fp64 device array
        (grad_sqnorm, one launch per bucket); the update kernel's arguments that take the norm and the coefficient from it."""
        C = self._kernel()
        if self._clip_bufs is None:
            dev = self.param_flats[0].device
            self._clip_bufs = (torch.zeros(len(self.buckets), dtype=torch.float64, device=dev),
                               torch.zeros(C.grad_sqnorm_workspace_numel(), dtype=torch.float32, device=dev),
                               torch.zeros(1, dtype=torch.float32, device=dev))
        sq, ws, norm = self._clip_bufs
        for k, gb in enumerate(self.buckets):
            C.grad_sqnorm(gb.flat[:gb.numel], sq, k, ws, grad_scale=grad_scale)
        self._grad_norm = norm
        return dict(max_grad_norm=self.max_grad_norm, sqnorms=sq, grad_norm_out=norm)

    def grad_norm(self) -> Optional[float]:
        """The pre-clip total L2 norm of the gradient of the last update (what ``clip_grad_norm_`` returns); ``None``
        without clipping or before the first update.  Synchronises with the device."""
        return None if self._grad_norm is None else float(self._grad_norm.reshape(-1)[0].item())

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


class FlatSGD(_FlatOptimizer):
    """``FlatSGD(model)`` where ``model`` is a plain module, a module carrying ``_grad_bucket`` or a
    :class:`DistributedDataParallel` wrapper.

    ``step()`` expects averaged gradients (call ``average_gradients(model)`` first, as the tutorial loop does) and,
    with ``zero_grad=True`` (default), leaves the buckets zeroed so no separate ``zero_grad()`` pass is needed;
    ``zero_grad()`` exists for loop compatibility and is then a no-op apart from re-arming the DDP hooks.

    ``max_grad_norm=c`` clips the averaged gradient first, as ``torch.nn.utils.clip_grad_norm_(params, c)`` would: on CUDA
    fp32 buckets ``grad_sqnorm`` sums each bucket's squares on the device and ``sgd_flat`` takes the norm and the
    coefficient there (no host synchronisation); elsewhere ``clip_grad_norm_(..., foreach=False)`` itself runs.
    :meth:`grad_norm` returns the last update's pre-clip norm.

    ``sharded=True`` shards the optimizer over the ranks (ZeRO stage 1): every bucket is cut into W equal slices, rank r keeps
    the momentum of slice r only (``momentum_flats[k]`` is that shard, :meth:`shard_range` its element range) and updates
    only that slice of the parameters, which then reach every rank.  The update runs where the gradient exchange runs, not in
    ``step()``: the DDP hooks (or ``average_gradients(model)``) launch, per bucket, either ONE ``sharded_sgd`` kernel on a
    symmetric CUDA world (reduce-scatter in fp32 in rank order, update, parameter all-gather through peer stores; a bf16
    bucket's fp32 sum feeds the update unrounded) or, elsewhere (gloo, several machines, no symmetric world), the bucket's
    all-reduce, the update of the owned slice and an ``all_gather_into_tensor`` of the parameters.  So **after
    ``average_gradients(model)`` the parameters are already updated** and ``p.grad`` is zero (with ``zero_grad=False`` it
    holds this rank's local, unaveraged gradient on the kernel path and the averaged one elsewhere); ``step()`` launches
    nothing: it advances ``steps``, re-arms the hooks, and raises if the step's buckets were not exchanged.  One
    ``average_gradients`` goes with one ``step``.  With fp32 buckets the parameters are bit for bit those of
    ``sharded=False`` (given the all-reduce's fixed rank order).  ``max_grad_norm`` cannot be combined with it (the total
    norm needs every bucket reduced before any update) and raises ``ValueError``.  :meth:`named_momentum` is then collective
    (every rank calls it; it gathers the shards) and returns the same per-name tensors as an unsharded optimizer, so
    checkpoints stay engine-independent.  At world size 1 the flag changes nothing.

    ``param_groups=[{"params": [...], "lr": ..., "weight_decay": ...}, ...]`` gives groups of parameters their own lr and /
    or weight decay, as torch's parameter groups do (absent keys take the constructor's values; other keys raise
    ``ValueError``; at most 64 groups).  The parameters named in no group form the default group, last in
    :attr:`param_groups`, whose values are ``lr`` / ``weight_decay``.  Every update reads the groups' values, and
    ``lr_schedule`` scales each group's lr.  On CUDA the update stays one launch per bucket (``sgd_flat_grouped``,
    ``sharded_sgd_grouped``): a uint8 group map, one id per 16-byte parameter vector, picks each element's scalars.
    ``state_dict()`` records the groups by parameter name and ``load_state_dict`` restores their values.

    ``capturable=True`` lets a CUDA graph capture the whole step (forward, backward with the bucket exchanges, ``step()``),
    as ``torch.optim.SGD(capturable=True)`` does: the step counter lives on the device, and the update kernels read their
    scalars (the scheduled lr of every group and its weight decay) from a block on the device that a one-CTA kernel advances after every
    update, so replays follow the schedule.  ``step()`` then does no host synchronisation, allocation or host-to-device
    copy, apart from uploading group ``lr`` / ``weight_decay`` values that changed since the last eager step;
    :meth:`sync_hyperparameters` does that upload outside a capture (replays read the device table as it stands, so a
    value assigned between replays takes effect with that call).  ``steps``, :meth:`lr_at` and the checkpoints read or write the device counter.  Warm up with eager steps
    on a side stream before capturing, as torch requires.  Refused (``ValueError``) where a bucket would take a torch-op
    path: CPU (gloo), reduced-precision unsharded gradient buckets, and ``sharded=True`` without one peer-memory world.

    Gradient accumulation (every flat optimizer, sharded or not): run all but the last micro-batch's backward inside
    ``DistributedDataParallel.no_sync()``.  The buckets are exchanged once per optimizer step, so ``steps``, the schedule
    and the clipping norm see the accumulated, averaged gradient; ``step()`` raises ``RuntimeError`` while a bucket holds
    accumulated gradients no exchange has taken."""

    lr = _group_attr("lr")
    weight_decay = _group_attr("weight_decay")
    sync_hyperparameters = _FlatOptimizer._sync_hyperparameters

    def __init__(self, model: nn.Module, lr: float = 0.01, momentum: float = 0.5, weight_decay: float = 0.0,
                 zero_grad: bool = True, group=None, lr_schedule: Optional[LRSchedule] = None, nesterov: bool = False,
                 max_grad_norm: Optional[float] = None, sharded: bool = False, param_groups: Optional[list] = None,
                 capturable: bool = False):
        check_sgd_options(momentum, weight_decay, nesterov)
        if param_groups is not None:
            param_groups = _check_param_groups(type(self).__name__, model, param_groups, lr, weight_decay,
                                               lambda glr, gwd: check_sgd_options(momentum, gwd, nesterov))
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.momentum = float(momentum)
        self.nesterov = bool(nesterov)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded, param_groups, capturable)
        self.momentum_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]

    def _sgd_runs(self, runs: list, pv: torch.Tensor, mv: torch.Tensor, g: torch.Tensor) -> None:
        """The torch-op update of ``_update`` on each ``(lo, hi, group)`` run of the views, with the group's lr and decay."""
        vals = self._group_values()
        for lo, hi, gi in runs:
            lr, wd = vals[gi]
            p, m, gf = pv[lo:hi], mv[lo:hi], g[lo:hi].to(torch.float32)
            if wd:
                gf = gf.add(p, alpha=wd)
            m.mul_(self.momentum).add_(gf)
            p.add_(gf.add(m, alpha=self.momentum) if self.nesterov else m, alpha=-lr)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        vals = self._group_values()
        for k, (gb, pf, mf, kern) in enumerate(zip(self.buckets, self.param_flats, self.momentum_flats, kernel)):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if kern and self._grouped:
                self._kernel().sgd_flat_grouped(pf, mf, g, self._maps[k], [v[0] for v in vals], [v[1] for v in vals],
                                                self.momentum, self.fused_zero, self.nesterov, **clip)
            elif kern:
                lr, wd = vals[0]
                self._kernel().sgd_flat(pf, mf, g, lr, self.momentum, wd, self.fused_zero, self.nesterov, **clip)
            else:
                # CPU ranks (gloo) and reduced-precision gradient buckets: the same flat update with tensor ops, in
                # torch.optim.SGD's order (foreach=False)
                self._sgd_runs(self._runs[k], pf, mf, _fp32_grad(g, clip.get("grad_scale")))
                if self.fused_zero:
                    g.zero_()

    def _update_capturable(self, clip: dict) -> None:
        for k, (gb, pf, mf) in enumerate(zip(self.buckets, self.param_flats, self.momentum_flats)):
            self._kernel().sgd_flat_cap(pf, mf, gb.flat[:gb.numel], self._cap_map(k), self._cap_block, self.momentum,
                                        self.fused_zero, self.nesterov, **clip)

    def _sharded_kernel(self, k: int, max_blocks: int) -> None:
        gb, mf = self.buckets[k], self.momentum_flats[k]
        n_vec, handle, gh, W = self._shards[k][0], self._shards[k][4], gb.symm_handle, self._world
        if self.capturable:
            self._kernel().sharded_sgd_cap(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs, mf, self._cap_map(k),
                                           self._cap_block, n_vec, self.momentum, self.nesterov, 1.0 / W, self.fused_zero,
                                           gb.world.rank, W, max_blocks)
            return
        if self._grouped:
            vals = self._group_values()
            self._kernel().sharded_sgd_grouped(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs, mf, self._maps[k],
                                               n_vec, [v[0] for v in vals], [v[1] for v in vals], self.momentum, self.nesterov,
                                               1.0 / W, self.fused_zero, gb.world.rank, W, max_blocks)
            return
        self._kernel().sharded_sgd(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs, mf, n_vec, self.lr_at(),
                                   self.momentum, self.weight_decay, self.nesterov, 1.0 / W, self.fused_zero, gb.world.rank, W,
                                   max_blocks)

    def _update_slice(self, k: int, lo: int, n: int) -> None:
        self._sgd_runs(self._slice_runs(k, lo, n), self._shards[k][3][lo:lo + n], self.momentum_flats[k][:n],
                       self.buckets[k].flat[lo:lo + n])

    # ------------------------------------------------------------------ checkpointing
    _options = ("lr", "momentum", "weight_decay", "nesterov")
    _noun, _carry = "momentum", "named_momentum() / load_named_momentum()"

    def _state_pairs(self) -> list:
        return [("momentum_buffers", self.momentum_flats)]

    def _defaults(self) -> dict:
        # SGD state_dicts written before Nesterov, clipping and the step count: plain momentum, no clipping, steps as they are
        return {"nesterov": False, "max_grad_norm": None, "steps": self.steps}

    def _check_options(self, sd: dict) -> dict:
        check_sgd_options(sd["momentum"], sd["weight_decay"], sd["nesterov"])
        return {"lr": float(sd["lr"]), "momentum": float(sd["momentum"]), "weight_decay": float(sd["weight_decay"]),
                "nesterov": bool(sd["nesterov"])}

    def named_momentum(self, model: nn.Module) -> dict:
        """Momentum per parameter NAME (CPU copies) -- the canonical, engine-independent form written to checkpoints: the
        fused trainer stores exactly this (``state_dict()['momentum']``), so checkpoints cross engines with momentum.
        Sharded over several ranks this is collective: every rank calls it, the shards are gathered, and every rank gets the
        full tensors an unsharded optimizer would return."""
        return self._named(model, self.momentum_flats)

    def load_named_momentum(self, model: nn.Module, named: dict) -> int:
        """Inverse of :meth:`named_momentum`; returns how many tensors were restored.  Sharded over several ranks, each rank
        keeps its slice of the full tensors (not collective)."""
        return self._load_named(model, named, self.momentum_flats)


def check_adamw_options(lr: float, betas, eps: float, weight_decay: float) -> tuple:
    """``torch.optim.AdamW``'s rules for the hyper-parameters; returns ``(beta1, beta2)`` as floats."""
    if not float(lr) >= 0.0:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not float(eps) >= 0.0:
        raise ValueError(f"Invalid epsilon value: {eps}")
    b1, b2 = (float(b) for b in betas)
    if not 0.0 <= b1 < 1.0:
        raise ValueError(f"Invalid beta parameter at index 0: {b1}")
    if not 0.0 <= b2 < 1.0:
        raise ValueError(f"Invalid beta parameter at index 1: {b2}")
    if not float(weight_decay) >= 0.0:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    return b1, b2


def adamw_scalars(lr: float, betas: tuple, eps: float, weight_decay: float, t: int) -> list:
    """The scalars of AdamW update ``t`` (1-based) that the kernels take (csrc/adamw.h), in fp64 as torch's non-capturable
    single-tensor path computes them: ``[1 - lr*wd, 1 - beta1, beta2, 1 - beta2, lr / (1 - beta1^t), sqrt(1 - beta2^t), eps]``.
    The bindings round each once to fp32."""
    b1, b2 = betas
    return [1.0 - lr * weight_decay, 1.0 - b1, b2, 1.0 - b2, lr / (1.0 - b1 ** t), (1.0 - b2 ** t) ** 0.5, eps]


class FlatAdamW(_FlatOptimizer):
    """``torch.optim.AdamW`` (``amsgrad=False``, ``maximize=False``) over flat buffers: ``FlatAdamW(model)`` where ``model``
    is a plain module, a module carrying ``_grad_bucket`` or a :class:`DistributedDataParallel` wrapper, in the same loop as
    :class:`FlatSGD` (``backward(); average_gradients(model); opt.step()``).

    The first and second moments (``exp_avg_flats``, ``exp_avg_sq_flats``) have the parameter flats' layout, so on CUDA fp32
    buckets ONE ``adamw_flat`` launch per bucket (csrc/adamw.cu) streams the parameters, gradients and both moments once,
    and with ``zero_grad=True`` (default) re-zeroes the gradients in the same pass.  Update k (``steps`` before it) uses
    t = k + 1; ``1 - lr*wd``, ``lr / (1 - beta1^t)`` and ``sqrt(1 - beta2^t)`` are computed on the host in fp64, as torch
    does, with ``lr = lr_at()`` (:class:`LRSchedule`).  Elsewhere (CPU tensors, bf16 buckets) torch's own single-tensor
    AdamW runs on each parameter's views of the flats, so a CPU run is bit for bit ``torch.optim.AdamW(foreach=False)``.

    ``max_grad_norm=c`` clips first, as :class:`FlatSGD` does (``grad_sqnorm`` and the clip coefficient on the device, no
    host synchronisation; :meth:`grad_norm`).  ``sharded=True`` is :class:`FlatSGD`'s ZeRO stage 1 with both moments
    sharded (8/W bytes of state per parameter): per bucket ONE ``sharded_adamw`` kernel reduce-scatters the gradients in
    fp32 in rank order, applies AdamW to the owned slice and stores the new parameters into every rank's flat, inside
    ``average_gradients`` / the DDP hooks; ``step()`` only counts the step.  Without one peer-memory world torch ops run the
    same semantics; at world size 1 the flag changes nothing; with ``max_grad_norm`` it raises ``ValueError``.
    :meth:`named_state` (collective when sharded) is ``torch.optim.AdamW``'s per-parameter state by parameter name.

    ``param_groups`` are :class:`FlatSGD`'s (per-group ``lr`` / ``weight_decay``; e.g. no decay on biases and norm weights).
    The grouped kernels (``adamw_flat_grouped``, ``sharded_adamw_grouped``) take ``1 - lr_g*wd_g`` and ``lr_g / (1 - beta1^t)``
    per group (:meth:`group_scalars`); elsewhere torch's AdamW runs once per group, as ``torch.optim.AdamW`` does.

    ``capturable=True`` lets a CUDA graph capture the whole step (forward, backward with the bucket exchanges, ``step()``),
    as ``torch.optim.AdamW(capturable=True)`` does: the step counter lives on the device, and the update kernels read their
    scalars (the scheduled lr of every group, ``1 - lr*wd``, ``lr / (1 - beta1^t)`` and ``sqrt(1 - beta2^t)``) from a block
    on the device that a one-CTA kernel advances after every update, so replays follow the schedule.  ``step()`` then does no host synchronisation, allocation or host-to-device
    copy, apart from uploading group ``lr`` / ``weight_decay`` values that changed since the last eager step;
    :meth:`sync_hyperparameters` does that upload outside a capture (replays read the device table as it stands, so a
    value assigned between replays takes effect with that call).  ``steps``, :meth:`lr_at` and the checkpoints read or write the device counter.  Warm up with eager steps
    on a side stream before capturing, as torch requires.  Refused (``ValueError``) where a bucket would take a torch-op
    path: CPU (gloo), reduced-precision unsharded gradient buckets, and ``sharded=True`` without one peer-memory world."""

    lr = _group_attr("lr")
    weight_decay = _group_attr("weight_decay")
    sync_hyperparameters = _FlatOptimizer._sync_hyperparameters

    def __init__(self, model: nn.Module, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 1e-2, zero_grad: bool = True, group=None, lr_schedule: Optional[LRSchedule] = None,
                 max_grad_norm: Optional[float] = None, sharded: bool = False, param_groups: Optional[list] = None,
                 capturable: bool = False):
        self.betas = check_adamw_options(lr, betas, eps, weight_decay)
        if param_groups is not None:
            param_groups = _check_param_groups(type(self).__name__, model, param_groups, lr, weight_decay,
                                               lambda glr, gwd: check_adamw_options(glr, betas, eps, gwd))
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.eps = float(eps)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded, param_groups, capturable)
        self.exp_avg_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]
        self.exp_avg_sq_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]

    def scalars(self) -> list:
        """:func:`adamw_scalars` of the next update (t = ``steps`` + 1, lr = :meth:`lr_at`)."""
        return adamw_scalars(self.lr_at(), self.betas, self.eps, self.weight_decay, self.steps + 1)

    def group_scalars(self) -> tuple:
        """With parameter groups: ``(shared, decays, step_sizes)`` of the next update -- :meth:`scalars` (whose decay and
        step size the grouped kernels do not use), then ``1 - lr_g*wd_g`` and ``lr_g / (1 - beta1^t)`` of every group, each
        computed in fp64 by :func:`adamw_scalars` from the group's scheduled lr."""
        per = [adamw_scalars(lr, self.betas, self.eps, wd, self.steps + 1) for lr, wd in self._group_values()]
        return self.scalars(), [s[0] for s in per], [s[4] for s in per]

    def _torch_adamw(self, p: list, g: list, m: list, v: list, lr: float, weight_decay: float) -> None:
        """torch's single-tensor AdamW on the given views (update t = steps + 1) with one group's lr and weight decay."""
        from torch.optim.adamw import adamw

        steps = [torch.tensor(float(self.steps)) for _ in p]
        adamw(p, g, m, v, [], steps, foreach=False, capturable=False, differentiable=False, fused=None, amsgrad=False,
              beta1=self.betas[0], beta2=self.betas[1], lr=lr, weight_decay=weight_decay, eps=self.eps, maximize=False)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        sc = (self.group_scalars() if self._grouped else self.scalars()) if any(kernel) else None
        for k, (gb, pf, mf, vf, kern) in enumerate(zip(self.buckets, self.param_flats, self.exp_avg_flats,
                                                        self.exp_avg_sq_flats, kernel)):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if kern and self._grouped:
                self._kernel().adamw_flat_grouped(pf, mf, vf, g, self._maps[k], *sc, self.fused_zero, **clip)
            elif kern:
                self._kernel().adamw_flat(pf, mf, vf, g, sc, self.fused_zero, **clip)
            else:
                gf = _fp32_grad(g, clip.get("grad_scale"))
                for lr, wd, _, views in self._tensor_views(k, [pf, gf, mf, vf]):
                    self._torch_adamw(*views, lr=lr, weight_decay=wd)
                if self.fused_zero:
                    g.zero_()

    def _update_capturable(self, clip: dict) -> None:
        for k, (gb, pf, mf, vf) in enumerate(zip(self.buckets, self.param_flats, self.exp_avg_flats, self.exp_avg_sq_flats)):
            self._kernel().adamw_flat_cap(pf, mf, vf, gb.flat[:gb.numel], self._cap_map(k), self._cap_block, self.fused_zero,
                                          **clip)

    def _sharded_kernel(self, k: int, max_blocks: int) -> None:
        gb = self.buckets[k]
        n_vec, handle, gh, W = self._shards[k][0], self._shards[k][4], gb.symm_handle, self._world
        if self.capturable:
            self._kernel().sharded_adamw_cap(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs,
                                             self.exp_avg_flats[k], self.exp_avg_sq_flats[k], self._cap_map(k), self._cap_block,
                                             n_vec, 1.0 / W, self.fused_zero, gb.world.rank, W, max_blocks)
            return
        if self._grouped:
            self._kernel().sharded_adamw_grouped(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs,
                                                 self.exp_avg_flats[k], self.exp_avg_sq_flats[k], self._maps[k], n_vec,
                                                 *self.group_scalars(), 1.0 / W, self.fused_zero, gb.world.rank, W, max_blocks)
            return
        self._kernel().sharded_adamw(gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs, self.exp_avg_flats[k],
                                     self.exp_avg_sq_flats[k], n_vec, self.scalars(), 1.0 / W, self.fused_zero, gb.world.rank,
                                     W, max_blocks)

    def _update_slice(self, k: int, lo: int, n: int) -> None:
        gf = self.buckets[k].flat[lo:lo + n].to(torch.float32)
        flats = [self._shards[k][3][lo:lo + n], gf, self.exp_avg_flats[k][:n], self.exp_avg_sq_flats[k][:n]]
        for lr, wd, views in self._run_views(self._slice_runs(k, lo, n), flats):
            self._torch_adamw(*views, lr=lr, weight_decay=wd)

    # ------------------------------------------------------------------ checkpointing: torch.optim.AdamW's names
    _options = ("lr", "betas", "eps", "weight_decay")
    _noun = "AdamW state"
    named_state = _FlatOptimizer._named_state
    load_named_state = _FlatOptimizer._load_named_state

    def _state_pairs(self) -> list:
        return [("exp_avg", self.exp_avg_flats), ("exp_avg_sq", self.exp_avg_sq_flats)]

    def _check_options(self, sd: dict) -> dict:
        return {"betas": check_adamw_options(sd["lr"], sd["betas"], sd["eps"], sd["weight_decay"]), "lr": float(sd["lr"]),
                "eps": float(sd["eps"]), "weight_decay": float(sd["weight_decay"])}


def check_rmsprop_options(lr: float, alpha: float, eps: float, weight_decay: float, momentum: float) -> None:
    """``torch.optim.RMSprop``'s rules for the hyper-parameters, with its messages."""
    if not 0.0 <= float(lr):
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= float(eps):
        raise ValueError(f"Invalid epsilon value: {eps}")
    if not 0.0 <= float(momentum):
        raise ValueError(f"Invalid momentum value: {momentum}")
    if not 0.0 <= float(weight_decay):
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    if not 0.0 <= float(alpha):
        raise ValueError(f"Invalid alpha value: {alpha}")


def rmsprop_scalars(lr: float, alpha: float, eps: float, weight_decay: float, momentum: float) -> list:
    """The scalars of one RMSprop update that the kernels take (csrc/rmsprop.h), in fp64:
    ``[lr, weight_decay, alpha, 1 - alpha, eps, momentum]``.  The bindings round each once to fp32."""
    return [float(lr), float(weight_decay), float(alpha), 1.0 - float(alpha), float(eps), float(momentum)]


class FlatRMSprop(_FlatOptimizer):
    """``torch.optim.RMSprop`` (``maximize=False``) over flat buffers: ``FlatRMSprop(model)`` where ``model`` is a plain
    module, a module carrying ``_grad_bucket`` or a :class:`DistributedDataParallel` wrapper, in the same loop as
    :class:`FlatSGD` (``backward(); average_gradients(model); opt.step()``).  torchvision's classification recipes train
    with it as ``RMSprop(params, lr, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=wd)``.

    The state flats have the parameter flats' layout: ``square_avg_flats``, plus ``momentum_buffer_flats`` when
    ``momentum > 0`` and ``grad_avg_flats`` when ``centered`` (empty lists otherwise).  On CUDA fp32 buckets ONE
    ``rmsprop_flat`` launch per bucket (csrc/rmsprop.cu) streams the parameters, gradients and states once, and with
    ``zero_grad=True`` (default) re-zeroes the gradients in the same pass.  ``weight_decay`` is torch's coupled L2 decay
    (``g + wd * p`` before the square average).  Update k (``steps`` before it) uses ``lr = lr_at()`` (:class:`LRSchedule`).
    Elsewhere (CPU tensors, bf16 buckets) torch's own single-tensor RMSprop runs on each parameter's views of the flats, so a
    CPU run is bit for bit ``torch.optim.RMSprop(foreach=False)``.  ``maximize``, ``differentiable`` and ``foreach`` are not
    taken.

    Everything else is :class:`FlatAdamW`'s: ``max_grad_norm`` (on-device clipping, :meth:`grad_norm`); ``sharded=True``
    (ZeRO stage 1: per bucket ONE ``sharded_rmsprop`` kernel reduce-scatters the gradients in fp32 in rank order, applies
    RMSprop to the owned slice with every state sharded 1/W, and stores the new parameters into every rank's flat, inside
    ``average_gradients`` / the DDP hooks; torch ops without one peer-memory world; nothing changes at world size 1; refused
    with ``max_grad_norm``); ``param_groups`` (per-group ``lr`` / ``weight_decay``: ``rmsprop_flat_grouped``,
    ``sharded_rmsprop_grouped``); ``capturable=True`` (the scheduled lr and weight decay of every group come from the device
    scalar block, so a CUDA graph captures the whole step; RMSprop has no other step-dependent scalar); ``no_sync()``
    accumulation, :class:`FlatEMA` and ``torch.amp.GradScaler``.  :meth:`named_state` (collective when sharded) is
    ``torch.optim.RMSprop``'s per-parameter state by parameter name."""

    lr = _group_attr("lr")
    weight_decay = _group_attr("weight_decay")
    sync_hyperparameters = _FlatOptimizer._sync_hyperparameters

    def __init__(self, model: nn.Module, lr: float = 1e-2, alpha: float = 0.99, eps: float = 1e-8, weight_decay: float = 0.0,
                 momentum: float = 0.0, centered: bool = False, zero_grad: bool = True, group=None,
                 lr_schedule: Optional[LRSchedule] = None, max_grad_norm: Optional[float] = None, sharded: bool = False,
                 param_groups: Optional[list] = None, capturable: bool = False):
        check_rmsprop_options(lr, alpha, eps, weight_decay, momentum)
        if param_groups is not None:
            param_groups = _check_param_groups(type(self).__name__, model, param_groups, lr, weight_decay,
                                               lambda glr, gwd: check_rmsprop_options(glr, alpha, eps, gwd, momentum))
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.alpha, self.eps, self.momentum, self.centered = float(alpha), float(eps), float(momentum), bool(centered)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded, param_groups, capturable)
        nb = range(len(self.buckets))
        self.square_avg_flats: List[torch.Tensor] = [self._state_flat(k) for k in nb]
        self.momentum_buffer_flats: List[torch.Tensor] = [self._state_flat(k) for k in nb] if self.momentum > 0 else []
        self.grad_avg_flats: List[torch.Tensor] = [self._state_flat(k) for k in nb] if self.centered else []

    def scalars(self, lr: Optional[float] = None) -> list:
        """:func:`rmsprop_scalars` of the next update (lr = :meth:`lr_at` unless given)."""
        return rmsprop_scalars(self.lr_at() if lr is None else lr, self.alpha, self.eps, self.weight_decay, self.momentum)

    def _states(self, k: int) -> tuple:
        """Bucket ``k``'s ``(square_avg, grad_avg or None, momentum_buffer or None)`` flats, in the kernels' argument order."""
        return (self.square_avg_flats[k], self.grad_avg_flats[k] if self.centered else None,
                self.momentum_buffer_flats[k] if self.momentum > 0 else None)

    def _torch_rmsprop(self, p: list, g: list, sq: list, ga: list, buf: list, lr: float, weight_decay: float) -> None:
        """torch's single-tensor RMSprop on the given views with one group's lr and weight decay."""
        from torch.optim.rmsprop import rmsprop

        steps = [torch.tensor(float(self.steps)) for _ in p]
        rmsprop(p, g, sq, ga, buf, steps, foreach=False, maximize=False, differentiable=False, capturable=False, lr=lr,
                alpha=self.alpha, eps=self.eps, weight_decay=weight_decay, momentum=self.momentum, centered=self.centered)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        sc = self.scalars() if any(kernel) else None
        vals = self._group_values() if self._grouped else None
        for k, (gb, pf, kern) in enumerate(zip(self.buckets, self.param_flats, kernel)):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if kern and self._grouped:
                self._kernel().rmsprop_flat_grouped(pf, *self._states(k), g, self._maps[k], sc, self.centered,
                                                    [v[0] for v in vals], [v[1] for v in vals], self.fused_zero, **clip)
            elif kern:
                self._kernel().rmsprop_flat(pf, *self._states(k), g, sc, self.centered, self.fused_zero, **clip)
            else:
                gf = _fp32_grad(g, clip.get("grad_scale"))
                for lr, wd, _, views in self._tensor_views(k, [pf, gf, *self._states(k)]):
                    self._torch_rmsprop(*views, lr=lr, weight_decay=wd)
                if self.fused_zero:
                    g.zero_()

    def _update_capturable(self, clip: dict) -> None:
        sc = self.scalars(lr=self.lr)    # lr and weight decay come from the device block; reading steps would synchronise
        for k, (gb, pf) in enumerate(zip(self.buckets, self.param_flats)):
            self._kernel().rmsprop_flat_cap(pf, *self._states(k), gb.flat[:gb.numel], self._cap_map(k), self._cap_block, sc,
                                            self.centered, self.fused_zero, **clip)

    def _sharded_kernel(self, k: int, max_blocks: int) -> None:
        gb = self.buckets[k]
        n_vec, handle, gh, W = self._shards[k][0], self._shards[k][4], gb.symm_handle, self._world
        head = (gb.flat.dtype == torch.bfloat16, gh.ptrs, handle.ptrs, gh.sig_ptrs) + self._states(k)
        tail = (1.0 / W, self.fused_zero, gb.world.rank, W, max_blocks)
        if self.capturable:
            self._kernel().sharded_rmsprop_cap(*head, self._cap_map(k), self._cap_block, n_vec, self.scalars(lr=self.lr),
                                               self.centered, *tail)
        elif self._grouped:
            vals = self._group_values()
            self._kernel().sharded_rmsprop_grouped(*head, self._maps[k], n_vec, self.scalars(), self.centered,
                                                   [v[0] for v in vals], [v[1] for v in vals], *tail)
        else:
            self._kernel().sharded_rmsprop(*head, n_vec, self.scalars(), self.centered, *tail)

    def _update_slice(self, k: int, lo: int, n: int) -> None:
        gf = self.buckets[k].flat[lo:lo + n].to(torch.float32)
        states = [f[:n] if f is not None else None for f in self._states(k)]
        for lr, wd, views in self._run_views(self._slice_runs(k, lo, n), [self._shards[k][3][lo:lo + n], gf] + states):
            self._torch_rmsprop(*views, lr=lr, weight_decay=wd)

    # ------------------------------------------------------------------ checkpointing: torch.optim.RMSprop's names
    _options = ("lr", "alpha", "eps", "weight_decay", "momentum", "centered")
    _noun = "RMSprop state"
    _lacks = ("FlatRMSprop.load_named_state: an entry has no {key!r}; the state is of an RMSprop with another momentum or "
              "centered setting")
    named_state = _FlatOptimizer._named_state
    load_named_state = _FlatOptimizer._load_named_state

    def _state_pairs(self) -> list:
        return [("square_avg", self.square_avg_flats), ("momentum_buffer", self.momentum_buffer_flats),
                ("grad_avg", self.grad_avg_flats)]

    def _check_options(self, sd: dict) -> dict:
        if bool(sd["centered"]) != self.centered or (float(sd["momentum"]) > 0) != (self.momentum > 0):
            raise ValueError(f"FlatRMSprop.load_state_dict: the state_dict has centered={bool(sd['centered'])} and momentum "
                             f"{float(sd['momentum'])}, this optimizer centered={self.centered} and momentum {self.momentum}; "
                             "build it with the same centered and the same momentum > 0 (they decide which states exist)")
        check_rmsprop_options(sd["lr"], sd["alpha"], sd["eps"], sd["weight_decay"], sd["momentum"])
        return {"lr": float(sd["lr"]), "weight_decay": float(sd["weight_decay"]), "alpha": float(sd["alpha"]),
                "eps": float(sd["eps"]), "momentum": float(sd["momentum"])}


def check_adafactor_options(lr: float, beta2_decay: float, eps, d: float, weight_decay: float) -> tuple:
    """``torch.optim.Adafactor``'s rules for the hyper-parameters, with its messages.  Returns ``(eps1, eps2)`` with
    ``eps1=None`` taken as fp32 machine epsilon."""
    if not 0.0 <= float(lr):
        raise ValueError(f"Learning rate should be >= 0 but is: {lr}")
    if not 0.0 >= float(beta2_decay):
        raise ValueError(f"beta2_decay should be <= 0 but is: {beta2_decay}")
    if eps[0] is not None and not 0.0 <= float(eps[0]):
        raise ValueError(f"epsilon1 should be >= 0 but is: {eps[0]}")
    if not 0.0 <= float(eps[1]):
        raise ValueError(f"epsilon2 should be >= 0 but is: {eps[1]}")
    if not 1.0 <= float(d):
        raise ValueError(f"Clipping threshold d should be >= 1 but is: {d}")
    if not 0.0 <= float(weight_decay):
        raise ValueError(f"weight_decay should be >= 0 but is: {weight_decay}")
    return (torch.finfo(torch.float32).eps if eps[0] is None else float(eps[0])), float(eps[1])


def _factors(shape) -> Optional[tuple]:
    """``(B, R, C)`` of a tensor Adafactor factors (dim > 1: B the product of the leading sizes), ``None`` otherwise."""
    if len(shape) < 2:
        return None
    return math.prod(shape[:-2]), int(shape[-2]), int(shape[-1])


class FlatAdafactor(_FlatOptimizer):
    """``torch.optim.Adafactor`` (``maximize=False``) over flat buffers: ``FlatAdafactor(model)`` where ``model`` is a plain
    module, a module carrying ``_grad_bucket`` or a :class:`DistributedDataParallel` wrapper, in the loop of
    :class:`FlatSGD` (``backward(); average_gradients(model); opt.step()``).  Update t = ``steps + 1`` of each parameter
    tensor, with ``lr = lr_at()``:

    * ``beta2_t = t ** beta2_decay``, ``rho_t = min(lr, 1 / sqrt(t))``, ``alpha = max(eps2, ||p|| / sqrt(numel)) * rho_t``
      (``||p||`` before the decay), then ``p *= 1 - lr * weight_decay``;
    * dim > 1, factored over the last two dimensions: ``row_var.lerp_(mean(g^2, -1), beta2_t)``,
      ``col_var.lerp_(mean(g^2, -2), beta2_t)``, ``v = row_var * col_var / max(mean(row_var, -2), eps1)``; otherwise
      ``variance.lerp_(g * g, beta2_t)`` and ``v = variance``;
    * ``u = g / sqrt(max(v, eps1^2))``, ``p += (-alpha / max(1, ||u|| / (sqrt(numel) * d))) * u``.

    ``eps=(None, eps2)`` takes fp32 machine epsilon for eps1.  The state is one fp32 flat per bucket
    (``state_flats[k]``): for each tensor ``row_var`` then ``col_var`` (``B*R + B*C`` floats, B the product of the leading
    dimensions), or ``variance`` (its numel), so a factored tensor keeps ``R + C`` floats per slice where AdamW keeps ``2RC``.

    On CUDA fp32 buckets three launches per bucket (csrc/adafactor.cu) update it with no host synchronisation: a stats
    kernel (``||p||``, the row and column sums of g^2, the lerps, the row_var means and ``alpha``), a norm kernel (``||u||``
    and the step scalar) and an apply kernel (decay, step, re-zeroed gradients), every sum in an order fixed by the bucket's
    chunk table, so two runs are bit-identical.  Elsewhere (CPU tensors, bf16 buckets) torch's own single-tensor Adafactor
    runs on each parameter's views, so a CPU run is bit for bit ``torch.optim.Adafactor(foreach=False)``.

    Like :class:`FlatRMSprop` it takes ``lr_schedule`` (the scheduled lr feeds ``rho_t`` and the decay), ``param_groups``
    (per-group ``lr`` / ``weight_decay``), ``max_grad_norm`` (on-device clipping first, :meth:`grad_norm`), ``no_sync()``
    accumulation, :class:`FlatEMA` and ``torch.amp.GradScaler``.  ``maximize``, ``foreach``, ``capturable`` and
    ``differentiable`` are not taken; ``sharded=True`` raises ``ValueError``.  :meth:`named_state` is
    ``torch.optim.Adafactor``'s per-parameter state by parameter name."""

    lr = _group_attr("lr")
    weight_decay = _group_attr("weight_decay")

    def __init__(self, model: nn.Module, lr: float = 1e-2, beta2_decay: float = -0.8, eps=(None, 1e-3), d: float = 1.0,
                 weight_decay: float = 0.0, zero_grad: bool = True, group=None, lr_schedule: Optional[LRSchedule] = None,
                 max_grad_norm: Optional[float] = None, sharded: bool = False, param_groups: Optional[list] = None):
        eps = tuple(eps)
        self.eps1, self.eps2 = check_adafactor_options(lr, beta2_decay, eps, d, weight_decay)
        if sharded:
            raise ValueError("FlatAdafactor cannot be sharded: a factored tensor's state is its row and column vectors, which do "
                             "not split along the flat slices of the sharded exchange, and the update needs whole-tensor norms "
                             "before any element moves; use sharded=False")
        if param_groups is not None:
            param_groups = _check_param_groups(type(self).__name__, model, param_groups, lr, weight_decay,
                                               lambda glr, gwd: check_adafactor_options(glr, beta2_decay, eps, d, gwd))
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.beta2_decay, self.eps, self.d = float(beta2_decay), eps, float(d)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, False, param_groups)
        # per bucket: the state offset of each tensor, and the state flat
        self._state_offsets: List[List[int]] = []
        self.state_flats: List[torch.Tensor] = []
        for gb, pf in zip(self.buckets, self.param_flats):
            offs, n = [], 0
            for gv in gb.views:
                offs.append(n)
                f = _factors(gv.shape)
                n += gv.numel() if f is None else f[0] * (f[1] + f[2])
            self._state_offsets.append(offs)
            self.state_flats.append(torch.zeros(max(n, 1), dtype=torch.float32, device=pf.device))
        self._af = []                    # per bucket on the kernel path: the table and the workspaces, else None
        for k, (gb, pf) in enumerate(zip(self.buckets, self.param_flats)):
            if not (pf.is_cuda and gb.flat.dtype == torch.float32):
                self._af.append(None)
                continue
            table, n_chunks, n_rc, n_means = self._kernel().adafactor_table(
                list(gb.offsets), [list(gv.shape) for gv in gb.views], [list(gv.stride()) for gv in gb.views],
                self._state_offsets[k], self._tensor_groups[k], gb.numel, self.state_flats[k].numel(), len(self._group_list),
                pf.device)
            n_t, dev = len(gb.params), pf.device
            self._af.append(dict(table=table, n_chunks=n_chunks,
                                 partials=torch.zeros(2 * n_chunks, dtype=torch.float32, device=dev),
                                 rc=torch.zeros(max(n_rc, 1), dtype=torch.float32, device=dev),
                                 means=torch.zeros(max(n_means, 1), dtype=torch.float32, device=dev),
                                 tickets=torch.zeros(n_t, dtype=torch.int32, device=dev),
                                 alpha=torch.zeros(n_t, dtype=torch.float64, device=dev),
                                 step=torch.zeros(n_t, dtype=torch.float32, device=dev)))

    def scalars(self) -> tuple:
        """What ``adafactor_flat`` takes for the next update (t = ``steps + 1``), in fp64: ``([t ** beta2_decay, eps1, eps2,
        d], [rho_t per group], [1 - lr * weight_decay per group])``."""
        t = float(self.steps + 1)
        vals = self._group_values()
        return ([t ** self.beta2_decay, self.eps1, self.eps2, self.d], [min(lr, 1 / (t ** 0.5)) for lr, _ in vals],
                [1 - lr * wd for lr, wd in vals])

    def _state_views(self, k: int, flat: torch.Tensor, i: int, key: str = "state") -> dict:
        """Tensor ``i`` of bucket ``k``'s state in ``flat`` (the one state flat, ``key`` ``"state"``), as torch's shaped
        views: ``row_var`` / ``col_var`` or ``variance``."""
        gv, so = self.buckets[k].views[i], self._state_offsets[k][i]
        f = _factors(gv.shape)
        if f is None:
            return {"variance": flat[so:so + gv.numel()].as_strided(gv.shape, gv.stride())}
        B, R, C = f
        lead = tuple(gv.shape[:-2])
        return {"row_var": flat[so:so + B * R].view(*lead, R, 1), "col_var": flat[so + B * R:so + B * (R + C)].view(*lead, 1, C)}

    def _torch_adafactor(self, p: list, g: list, states: list, lr: float, weight_decay: float) -> None:
        from torch.optim._adafactor import adafactor

        steps = [torch.tensor(float(self.steps)) for _ in p]
        adafactor(p, g, [s.get("row_var") for s in states], [s.get("col_var") for s in states],
                  [s.get("variance") for s in states], steps, foreach=False, d=self.d, lr=lr, beta2_decay=self.beta2_decay,
                  weight_decay=weight_decay, eps1=self.eps[0], eps2=self.eps2, maximize=False)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        sc = self.scalars() if any(kernel) else None
        for k, (gb, pf, sf, kern) in enumerate(zip(self.buckets, self.param_flats, self.state_flats, kernel)):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if kern:
                w = self._af[k]
                self._kernel().adafactor_flat(pf, sf, g, w["table"], w["n_chunks"], w["partials"], w["rc"], w["means"],
                                              w["tickets"], w["alpha"], w["step"], *sc, self.fused_zero, **clip)
                continue
            gf = _fp32_grad(g, clip.get("grad_scale"))
            for lr, wd, idx, (pv, gv) in self._tensor_views(k, [pf, gf], nonempty=True):
                self._torch_adafactor(pv, gv, [self._state_views(k, sf, i) for i in idx], lr, wd)
            if self.fused_zero:
                g.zero_()

    # ------------------------------------------------------------------ checkpointing: torch.optim.Adafactor's names
    _options = ("lr", "beta2_decay", "eps", "d", "weight_decay")
    _lacks = ("FlatAdafactor.load_named_state: the entry of {name!r} has no {keys}; its parameter has another number of "
              "dimensions")
    named_state = _FlatOptimizer._named_state
    load_named_state = _FlatOptimizer._load_named_state

    def _state_pairs(self) -> list:
        return [("state", self.state_flats)]

    def _check_options(self, sd: dict) -> dict:
        eps = tuple(sd["eps"])
        eps1, eps2 = check_adafactor_options(sd["lr"], sd["beta2_decay"], eps, sd["d"], sd["weight_decay"])
        return {"lr": float(sd["lr"]), "weight_decay": float(sd["weight_decay"]), "beta2_decay": float(sd["beta2_decay"]),
                "eps": eps, "d": float(sd["d"]), "eps1": eps1, "eps2": eps2}


def exclude_1d(name: str, param: torch.Tensor) -> bool:      # noqa: ARG001 - the name is there for custom rules
    """The default ``exclude_from_adaptation`` of :class:`FlatLAMB` and :class:`FlatLARS`: biases and norm weights
    (``param.ndim <= 1``) get no weight decay and a trust ratio of 1, as in the usual LARS and BERT-LAMB recipes."""
    return param.ndim <= 1


def lamb_scalars(lr: float, betas: tuple, eps: float, weight_decay: float, t: int) -> list:
    """The scalars of LAMB update ``t`` (1-based) that ``lamb_flat`` takes (csrc/layerwise.h), in fp64:
    ``[1 - beta1, beta2, 1 - beta2, sqrt(1 - beta2^t), eps, 1 / (1 - beta1^t), lr, weight_decay]``.  The binding rounds
    each once to fp32."""
    b1, b2 = betas
    return [1.0 - b1, b2, 1.0 - b2, (1.0 - b2 ** t) ** 0.5, eps, 1.0 / (1.0 - b1 ** t), lr, weight_decay]


class _LayerwiseOptimizer(_FlatOptimizer):
    """What :class:`FlatLAMB` and :class:`FlatLARS` share: the per-tensor adaptation flags, the trust ratios of the last
    update, and on CUDA fp32 buckets the chunk table and the workspaces of the layer-wise kernels (csrc/layerwise.cu).
    :attr:`param_groups` is one group with every parameter, whose ``lr`` / ``weight_decay`` are the optimizer's.

    ``sharded=True`` over several ranks of one peer-memory world: per bucket the two kernels of csrc/sharded_layerwise.cu run
    in place of the all-reduce, on this rank's chunk table (its slice of the bucket), with a symmetric fp64 buffer of the
    per-tensor sums that the ranks add in rank order.  Elsewhere (gloo, several machines, NCCL) ``sharded=True`` over
    several ranks raises ``ValueError``."""

    lr = _group_attr("lr")
    weight_decay = _group_attr("weight_decay")

    def __init__(self, model: nn.Module, zero_grad: bool, group, lr_schedule: Optional[LRSchedule],
                 max_grad_norm: Optional[float], sharded: bool, exclude_from_adaptation):
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded)
        exclude = exclude_1d if exclude_from_adaptation is None else exclude_from_adaptation
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        self.adapt: List[List[bool]] = [[not bool(exclude(names.get(id(p), ""), p)) for p in gb.params] for gb in self.buckets]
        # the trust ratio of every tensor of a bucket (bucket order) in the last update; 1 before the first
        self.ratio_flats = [torch.ones(len(gb.params), dtype=torch.float32, device=pf.device)
                            for gb, pf in zip(self.buckets, self.param_flats)]
        # per bucket on a kernel path: (table, chunks, partials, tickets, sums), else None.  Sharded, the table is this rank's
        # slice's (a ShardedLwTable) and `sums` the symmetric handle of the [2 * tensors] fp64 sums every rank reads.
        self._lw = []
        for k, (gb, pf, adapt) in enumerate(zip(self.buckets, self.param_flats, self.adapt)):
            n_t, numels = len(gb.params), [p.numel() for p in gb.params]
            if self._shard_mode == "kernel":
                table = self._kernel().sharded_layerwise_table(gb.offsets, numels, adapt, self._shards[k][1], gb.world.rank,
                                                               self._world, pf.device)
                n_chunks = table.n_chunks
                sums = gb.world.alloc_bytes(16 * n_t, ll=False)
            elif self._shard_mode is None and pf.is_cuda and gb.flat.dtype == torch.float32:
                table, n_chunks = self._kernel().layerwise_table(gb.offsets, numels, adapt, gb.numel, pf.device)
                sums = torch.zeros(2 * n_t, dtype=torch.float64, device=pf.device)
            else:
                self._lw.append(None)
                continue
            self._lw.append((table, n_chunks, torch.zeros(2 * n_chunks, dtype=torch.float32, device=pf.device),
                             torch.zeros(n_t, dtype=torch.int32, device=pf.device), sums))

    def _check_shard_mode(self) -> None:
        if self._shard_mode == "torch":
            raise ValueError(f"{type(self).__name__}(sharded=True) over several ranks needs one peer-memory world (backend "
                             "'b200' on one machine): the norms of the tensors that straddle shard boundaries are exchanged "
                             "between the ranks inside the sharded kernels; use sharded=False")

    def _sharded_args(self, k: int) -> tuple:
        """The leading arguments of ``sharded_lamb`` / ``sharded_lars`` for bucket ``k``: dtype flag and per-rank pointers."""
        gb = self.buckets[k]
        return (gb.flat.dtype == torch.bfloat16, gb.symm_handle.ptrs, self._shards[k][4].ptrs, self._lw[k][4].ptrs,
                gb.symm_handle.sig_ptrs)

    def _tensors(self, k: int, flats: list):
        """Per tensor of bucket ``k``: (index, adapted?, its 1-D slice of each flat in ``flats``)."""
        gb = self.buckets[k]
        for i, (p, o) in enumerate(zip(gb.params, gb.offsets)):
            yield i, self.adapt[k][i], [f[o:o + p.numel()] for f in flats]

    def trust_ratios(self, model: nn.Module) -> dict:
        """``{parameter name: trust ratio of the last update}`` (1.0 before the first update and for excluded tensors).
        Synchronises with the device."""
        names = {id(p): n for n, p in getattr(model, "module", model).named_parameters()}
        out = {}
        for gb, r in zip(self.buckets, self.ratio_flats):
            for p, x in zip(gb.params, r.tolist()):
                if id(p) in names:
                    out[names[id(p)]] = x
        return out


def _norm64(x: torch.Tensor) -> float:
    return float(torch.linalg.vector_norm(x, dtype=torch.float64))


class FlatLAMB(_LayerwiseOptimizer):
    """LAMB (You et al. 2020, as Apex ``FusedLAMB`` with ``use_nvlamb=False``) over flat buffers, in the loop of
    :class:`FlatSGD` (``backward(); average_gradients(model); opt.step()``).  Update t = ``steps + 1``:

    * ``m``, ``v``: AdamW's moments;  ``u = (m / (sqrt(v) / sqrt(1 - beta2^t) + eps)) / (1 - beta1^t) + wd_l * p``;
    * ``r_l = ||p_l|| / ||u_l||`` per parameter tensor (1 if the tensor is excluded or a norm is 0);  ``p -= (lr * r_l) * u``.

    ``exclude_from_adaptation(name, param) -> bool`` picks the tensors with ``wd_l = 0`` and ``r_l = 1`` (default
    :func:`exclude_1d`: biases and norm weights).  On CUDA fp32 buckets two kernels per bucket (csrc/layerwise.cu) form the
    per-tensor norms in a fixed order (fp32 per thread and CTA, fp64 over the chunks of a tensor) and apply the update with
    no host synchronisation; elsewhere (CPU tensors, bf16 buckets) torch ops run the same semantics on each tensor.
    ``max_grad_norm`` clips first, as in :class:`FlatAdamW`.  :meth:`trust_ratios` gives the last update's ratios.  The
    checkpoint forms are :class:`FlatAdamW`'s, so LAMB state loads into ``FlatAdamW`` and back.  ``sharded=True`` is ZeRO
    stage 1 on one peer-memory world (both moments 1/W per rank, the per-tensor norms exchanged between the ranks inside the
    sharded kernels, csrc/sharded_layerwise.cu); over several ranks elsewhere it raises ``ValueError``."""

    def __init__(self, model: nn.Module, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6,
                 weight_decay: float = 0.01, zero_grad: bool = True, group=None, lr_schedule: Optional[LRSchedule] = None,
                 max_grad_norm: Optional[float] = None, sharded: bool = False, exclude_from_adaptation=None):
        self.betas = check_adamw_options(lr, betas, eps, weight_decay)
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.eps = float(eps)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded, exclude_from_adaptation)
        self.exp_avg_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]
        self.exp_avg_sq_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]

    def scalars(self) -> list:
        """:func:`lamb_scalars` of the next update (t = ``steps`` + 1, lr = :meth:`lr_at`)."""
        return lamb_scalars(self.lr_at(), self.betas, self.eps, self.weight_decay, self.steps + 1)

    def _sharded_kernel(self, k: int, max_blocks: int) -> None:
        table, _, partials, tickets, _ = self._lw[k]
        self._kernel().sharded_lamb(*self._sharded_args(k), self.exp_avg_flats[k], self.exp_avg_sq_flats[k], table, partials,
                                    tickets, self.ratio_flats[k], self._shards[k][0], self.scalars(), 1.0 / self._world,
                                    self.fused_zero, self.buckets[k].world.rank, self._world, max_blocks)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        sc = self.scalars()
        w1, b2, c2, sbc2, eps, rbc1, lr, wd = sc
        for k, (gb, pf, mf, vf, kern) in enumerate(zip(self.buckets, self.param_flats, self.exp_avg_flats,
                                                        self.exp_avg_sq_flats, kernel)):
            g = gb.flat[:gb.numel]       # a symmetric-memory bucket is padded beyond the laid-out elements
            if kern:
                self._kernel().lamb_flat(pf, mf, vf, g, *self._lw[k], self.ratio_flats[k], sc, self.fused_zero, **clip)
                continue
            gf = _fp32_grad(g, clip.get("grad_scale"))
            ratios = []
            for _, adapt, (p, gt, m, v) in self._tensors(k, [pf, gf, mf, vf]):
                m.lerp_(gt, w1)
                v.mul_(b2).addcmul_(gt, gt, value=c2)
                u = (m / (v.sqrt() / sbc2).add_(eps)).mul_(rbc1)
                if adapt and wd != 0.0:
                    u.add_(p, alpha=wd)
                r = 1.0
                if adapt:
                    wn, un = _norm64(p), _norm64(u)
                    if wn > 0.0 and un > 0.0:
                        r = _f32(wn / un)
                p.add_(u, alpha=-_f32(_f32(lr) * r))
                ratios.append(r)
            self.ratio_flats[k].copy_(torch.tensor(ratios, dtype=torch.float32))
            if self.fused_zero:
                g.zero_()

    # ------------------------------------------------------------------ checkpointing: FlatAdamW's forms
    _options, _noun = FlatAdamW._options, FlatAdamW._noun
    _state_pairs, _check_options = FlatAdamW._state_pairs, FlatAdamW._check_options
    named_state = _FlatOptimizer._named_state
    load_named_state = _FlatOptimizer._load_named_state


def check_lars_options(lr: float, momentum: float, weight_decay: float, trust_coefficient: float, eps: float,
                       nesterov: bool) -> None:
    """The hyper-parameter rules of :class:`FlatLARS`."""
    if not float(lr) >= 0.0:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not float(momentum) >= 0.0:
        raise ValueError(f"Invalid momentum value: {momentum}")
    if not (math.isfinite(float(trust_coefficient)) and float(trust_coefficient) > 0.0):
        raise ValueError(f"trust_coefficient must be a finite value > 0, got {trust_coefficient}")
    if not float(eps) >= 0.0:
        raise ValueError(f"Invalid epsilon value: {eps}")
    check_sgd_options(momentum, weight_decay, nesterov)


class FlatLARS(_LayerwiseOptimizer):
    """LARS (You, Gitman, Ginsburg 2017) over flat buffers, in the loop of :class:`FlatSGD`:

    * ``r_l = trust_coefficient * ||p_l|| / (||g_l|| + wd_l * ||p_l|| + eps)`` per parameter tensor (1 if the tensor is
      excluded or a norm is 0);
    * ``d = r_l * (g + wd_l * p)``, then ``torch.optim.SGD(momentum, dampening=0, nesterov, weight_decay=0)`` on ``d``.

    ``exclude_from_adaptation(name, param) -> bool`` picks the tensors with ``wd_l = 0`` and ``r_l = 1`` (default
    :func:`exclude_1d`).  On CUDA fp32 buckets two kernels per bucket (csrc/layerwise.cu) form the norms and apply
    :class:`FlatSGD`'s fmaf sequence to ``d``; elsewhere the ratio is formed with torch ops and
    ``torch.optim.SGD(foreach=False)``'s update runs on ``d``.  ``max_grad_norm`` clips ``g`` first.  The checkpoint forms
    are :class:`FlatSGD`'s (``named_momentum``), so LARS momentum loads into ``FlatSGD`` and back.  ``sharded=True`` is
    :class:`FlatLAMB`'s: ZeRO stage 1 on one peer-memory world (momentum 1/W per rank), ``ValueError`` over several ranks
    elsewhere."""

    def __init__(self, model: nn.Module, lr: float = 0.1, momentum: float = 0.9, weight_decay: float = 1e-4,
                 trust_coefficient: float = 1e-3, eps: float = 1e-8, nesterov: bool = False, zero_grad: bool = True,
                 group=None, lr_schedule: Optional[LRSchedule] = None, max_grad_norm: Optional[float] = None,
                 sharded: bool = False, exclude_from_adaptation=None):
        check_lars_options(lr, momentum, weight_decay, trust_coefficient, eps, nesterov)
        self._default_group = {"params": [], "lr": float(lr), "weight_decay": float(weight_decay)}
        self.momentum = float(momentum)
        self.trust_coefficient, self.eps, self.nesterov = float(trust_coefficient), float(eps), bool(nesterov)
        super().__init__(model, zero_grad, group, lr_schedule, max_grad_norm, sharded, exclude_from_adaptation)
        self.momentum_flats: List[torch.Tensor] = [self._state_flat(k) for k in range(len(self.buckets))]
        # sharded kernel path: the averaged gradient of this rank's slice, kept between the two kernels
        self._grad_shards = [self._state_flat(k) for k in range(len(self.buckets))] if self._shard_mode == "kernel" else None

    def _sharded_kernel(self, k: int, max_blocks: int) -> None:
        table, _, partials, tickets, _ = self._lw[k]
        self._kernel().sharded_lars(*self._sharded_args(k), self.momentum_flats[k], self._grad_shards[k], table, partials,
                                    tickets, self.ratio_flats[k], self._shards[k][0], self.lr_at(), self.momentum, self.weight_decay,
                                    self.trust_coefficient, self.eps, self.nesterov, 1.0 / self._world, self.fused_zero,
                                    self.buckets[k].world.rank, self._world, max_blocks)

    def _update(self, kernel: List[bool], clip: dict) -> None:
        from torch.optim.sgd import sgd

        lr, wd, eta, eps = self.lr_at(), self.weight_decay, self.trust_coefficient, self.eps
        for k, (gb, pf, mf, kern) in enumerate(zip(self.buckets, self.param_flats, self.momentum_flats, kernel)):
            g = gb.flat[:gb.numel]
            if kern:
                self._kernel().lars_flat(pf, mf, g, *self._lw[k], self.ratio_flats[k], lr, self.momentum, wd, eta, eps,
                                         self.nesterov, self.fused_zero, **clip)
                continue
            gf = _fp32_grad(g, clip.get("grad_scale"))
            ratios = []
            for _, adapt, (p, gt, m) in self._tensors(k, [pf, gf, mf]):
                r = 1.0
                if adapt:
                    wn, gn = _norm64(p), _norm64(gt)
                    if wn > 0.0 and gn > 0.0:
                        r = _f32(eta * wn / (gn + wd * wn + eps))
                d = gt.add(p, alpha=wd) if adapt and wd != 0.0 else gt.clone()
                if r != 1.0:
                    d.mul_(r)
                sgd([p], [d], [m], foreach=False, weight_decay=0.0, momentum=self.momentum, lr=lr, dampening=0.0,
                    nesterov=self.nesterov, maximize=False)
                ratios.append(r)
            self.ratio_flats[k].copy_(torch.tensor(ratios, dtype=torch.float32))
            if self.fused_zero:
                g.zero_()

    # ------------------------------------------------------------------ checkpointing: FlatSGD's forms
    _options = FlatSGD._options + ("trust_coefficient", "eps")
    _noun, _carry, _state_pairs = FlatSGD._noun, FlatSGD._carry, FlatSGD._state_pairs

    def _defaults(self) -> dict:
        # a FlatSGD state_dict loads too: the LARS options stay
        return dict(FlatSGD._defaults(self), trust_coefficient=self.trust_coefficient, eps=self.eps)

    def _check_options(self, sd: dict) -> dict:
        check_lars_options(sd["lr"], sd["momentum"], sd["weight_decay"], sd["trust_coefficient"], sd["eps"], sd["nesterov"])
        return dict(FlatSGD._check_options(self, sd), trust_coefficient=float(sd["trust_coefficient"]), eps=float(sd["eps"]))

    named_momentum = FlatSGD.named_momentum
    load_named_momentum = FlatSGD.load_named_momentum


def check_ema_options(decay, every, warmup_steps) -> tuple:
    """:class:`FlatEMA`'s rules: ``decay`` a finite number in [0, 1], ``every`` an int >= 1, ``warmup_steps`` an int >= 0.
    Returns them as ``(float, int, int)``."""
    if isinstance(decay, bool) or not isinstance(decay, (int, float)) or not math.isfinite(float(decay)) \
            or not 0.0 <= float(decay) <= 1.0:
        raise ValueError(f"FlatEMA: decay must be a finite number in [0, 1], got {decay!r}")
    if isinstance(every, bool) or not isinstance(every, int) or every < 1:
        raise ValueError(f"FlatEMA: every must be an int >= 1, got {every!r}")
    if isinstance(warmup_steps, bool) or not isinstance(warmup_steps, int) or warmup_steps < 0:
        raise ValueError(f"FlatEMA: warmup_steps must be an int >= 0, got {warmup_steps!r}")
    return float(decay), int(every), int(warmup_steps)


class FlatEMA:
    """An exponential moving average of the weights of a model trained by a flat optimizer (:class:`FlatSGD`,
    :class:`FlatAdamW`, :class:`FlatRMSprop`, :class:`FlatAdafactor`, :class:`FlatLAMB`, :class:`FlatLARS`), for evaluation and the final checkpoint: torchvision's
    ``--model-ema``, timm's ``ModelEma``, ``AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=True)``.

    ``ema = FlatEMA(optimizer, decay=0.9999, every=1, warmup_steps=0)`` copies the current parameters, and the floating-point
    buffers of the model (BatchNorm running statistics), into EMA storage.  The model is the module inside the optimizer's
    :class:`DistributedDataParallel`; an optimizer built on a plain module needs ``model=`` (that module, or a
    :class:`DistributedDataParallel` around it), and ``ValueError`` says so.  Call :meth:`update`
    after every ``optimizer.step()``.  With ``t`` the optimizer's ``steps`` after that step, the update

    * does nothing unless ``t % every == 0``;
    * copies the live values if ``t - every <= warmup_steps`` (the first update, as ``AveragedModel``'s ``n_averaged == 0``,
      and torchvision's reset of the average during lr warmup);
    * otherwise lerps: ``ema = lerp(ema, live, w)`` with ``w = fp32(1 - decay)``, ``1 - decay`` in fp64 as Python computes it
      for ``torch._foreach_lerp_(..., 1 - decay)``, and torch's roundings: ``fma(w, p - e, e)`` for ``w < 0.5``, else
      ``fma(-(p - e), 1 - w, p)``, subnormals kept.

    fp32 buffers are averaged by the same rule.  Integer buffers (``num_batches_tracked``) are neither averaged nor swapped:
    that is the one difference from ``AveragedModel(use_buffers=True)``, which averages them in integer arithmetic.  Buffers
    are followed in place, so a buffer the model replaces by a new tensor is no longer followed.

    On CUDA one launch of ``ema_update`` (csrc/ema.cu) updates the whole model per :meth:`update`: a table built here lists
    every bucket's parameter flat (or this rank's slice of it when the optimizer is sharded) and every fp32 buffer.  With a
    ``capturable=True`` optimizer the kernel reads the optimizer's device step counter and decides skip / copy / lerp itself,
    so ``update()`` can sit in the CUDA graph of the step and replays follow ``every`` and ``warmup_steps``; otherwise the host
    decides, launches nothing on a skipped step, and ``update()`` inside a capture raises ``RuntimeError``.  On CPU (gloo)
    ``torch._foreach_copy_`` / ``torch._foreach_lerp_`` apply the same rule.

    With ``sharded=True`` over several ranks a rank keeps the EMA of the slice of each bucket it owns (:meth:`shard_range` of
    the optimizer, padding included), so the EMA costs 4/W bytes per parameter as the optimizer state does.  No
    communication: the owned slice is the one this rank's own update wrote.

    ``with ema.average_parameters():`` puts the EMA into the model's parameters and fp32 buffers and on exit restores the live
    values bit for bit.  Sharded, it swaps the owned slices and all-gathers the parameter flats, on entry and on exit
    (collective: every rank enters).  Inside the block ``update()``, ``optimizer.step()`` and, when sharded, the gradient
    exchange of ``average_gradients`` / the DDP hooks raise ``RuntimeError`` before anything changes, and entering the block
    during a CUDA-graph capture does too.  ``state_dict()`` and :meth:`named_ema` work there and give the EMA, which the
    model holds inside the block.

    ``decay``, ``every`` and ``warmup_steps`` are read-only.  ``state_dict()`` / ``load_state_dict()`` follow the optimizers'
    rules (a shard loads only on its own rank of its own world size; a whole EMA loads into a sharded one as each rank's
    slice) and refuse a state with other settings; :meth:`named_ema` / :meth:`load_named_ema` cross world sizes."""

    def __init__(self, optimizer, decay: float = 0.9999, every: int = 1, warmup_steps: int = 0,
                 model: Optional[nn.Module] = None):
        self._decay, self._every, self._warmup = check_ema_options(decay, every, warmup_steps)
        if not isinstance(optimizer, _FlatOptimizer):
            raise ValueError(f"FlatEMA needs a flat optimizer (FlatSGD, FlatAdamW, FlatRMSprop, FlatAdafactor, FlatLAMB, FlatLARS), got "
                             f"{type(optimizer).__name__}")
        from ..parallel.ddp import DistributedDataParallel

        opt = optimizer
        self._kernel_path = opt.param_flats[0].is_cuda
        if model is None:
            if opt._engine is None:
                raise ValueError("FlatEMA: the optimizer was built on a plain module; pass model= (that module) so that its "
                                 "floating buffers are averaged too")
            model = opt._engine.module
        module = model.module if isinstance(model, DistributedDataParallel) else model
        mine = {id(p) for p in module.parameters()}
        if any(id(p) not in mine for gb in opt.buckets for p in gb.params):
            raise ValueError("FlatEMA: model= is not the module the optimizer updates (it lacks some of its parameters)")
        bufs = [(n, b) for n, b in module.named_buffers() if torch.is_floating_point(b)]
        for n, b in bufs:
            if self._kernel_path and (not b.is_cuda or b.dtype != torch.float32 or b.device != opt.param_flats[0].device):
                raise ValueError(f"FlatEMA averages floating buffers in fp32 on the parameters' device; the buffer {n!r} is "
                                 f"{b.dtype} on {b.device}")
        self._opt = opt
        self._swapped = False
        self._w = 1.0 - self._decay                  # rounded once to fp32 by the kernel's binding, by torch on CPU
        self._buf_names = [n for n, _ in bufs]
        self._bufs = [b for _, b in bufs]
        with torch.no_grad():
            self.ema_flats: List[torch.Tensor] = [self._live(k).clone() for k in range(len(opt.buckets))]
            self.ema_buffers: List[torch.Tensor] = [b.detach().clone() for b in self._bufs]
        self._table = None
        if self._kernel_path:
            self._table = opt._kernel().ema_table(self.ema_flats + self.ema_buffers,
                                                  [self._live(k) for k in range(len(opt.buckets))] + self._bufs)

    decay = property(lambda self: self._decay, doc="The decay (read-only).")
    every = property(lambda self: self._every, doc="Update every this many optimizer steps (read-only).")
    warmup_steps = property(lambda self: self._warmup, doc="Copy instead of averaging up to this step (read-only).")

    def _live(self, k: int) -> torch.Tensor:
        """Bucket ``k``'s live parameters that this rank averages: the whole flat, or its owned slice of the padded flat."""
        opt = self._opt
        if opt._shard_mode is None:
            return opt.param_flats[k]
        per = opt._shards[k][2]
        return opt._shards[k][3][opt._rank * per:(opt._rank + 1) * per]

    def _ema_tensors(self) -> tuple:
        """(EMA of every bucket, EMA of every buffer): the EMA storage, or inside :meth:`average_parameters` the model's own
        parameter flats (owned slices when sharded) and buffers, which hold the EMA there."""
        if self._swapped:
            return [self._live(k) for k in range(len(self.ema_flats))], list(self._bufs)
        return self.ema_flats, self.ema_buffers

    def _refuse_inside(self, what: str) -> None:
        if self._swapped:
            raise RuntimeError(f"FlatEMA.{what} inside average_parameters(): the model holds the EMA values there")

    @torch.no_grad()
    def update(self) -> None:
        """The EMA update after ``optimizer.step()`` (see the class): skip, copy or lerp, decided from the optimizer's
        ``steps``.  One kernel launch on CUDA, none on a skipped step unless the optimizer is capturable."""
        self._refuse_inside("update()")
        opt = self._opt
        if self._kernel_path and opt.capturable:
            opt._kernel().ema_update(*self._table, self._w, counter=opt._cap_counter, every=self._every,
                                     warmup_steps=self._warmup)
            return
        if self._kernel_path and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FlatEMA.update() in a CUDA-graph capture needs a capturable=True optimizer: otherwise the "
                               "host decides skip / copy / lerp, and the graph would replay the capture's decision")
        t = opt.steps
        if t % self._every:
            return
        copy = t - self._every <= self._warmup
        if self._kernel_path:
            opt._kernel().ema_update(*self._table, self._w, copy=copy)
            return
        emas = self.ema_flats + self.ema_buffers
        lives = [self._live(k) for k in range(len(opt.buckets))] + self._bufs
        if copy:
            torch._foreach_copy_(emas, lives)
        else:
            torch._foreach_lerp_(emas, lives, self._w)

    @torch.no_grad()
    def _swap(self) -> None:
        """Exchange the live values and the EMA (owned slices, then an all-gather of every parameter flat when sharded)."""
        from .. import comm

        opt = self._opt
        for k, e in enumerate(self.ema_flats):
            live = self._live(k)
            tmp = live.clone()
            live.copy_(e)
            e.copy_(tmp)
            if opt._shard_mode is not None:
                comm.all_gather_into_tensor(opt._shards[k][3], live.clone(), group=opt._group)
        for b, e in zip(self._bufs, self.ema_buffers):
            tmp = b.clone()
            b.copy_(e)
            e.copy_(tmp)

    @contextlib.contextmanager
    def average_parameters(self):
        """``with ema.average_parameters():`` evaluates the EMA model: the parameters and fp32 buffers hold the EMA inside
        the block and the live values, bit for bit, after it.  Collective when the optimizer is sharded over several ranks.
        ``RuntimeError`` when nested or entered during a CUDA-graph capture."""
        self._refuse_inside("average_parameters()")
        if self._kernel_path and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FlatEMA.average_parameters() cannot be entered during a CUDA-graph capture")
        self._swap()
        self._swapped = self._opt._ema_swapped = True
        try:
            yield self
        finally:
            self._swap()
            self._swapped = self._opt._ema_swapped = False

    # ------------------------------------------------------------------ checkpointing
    def _settings(self) -> dict:
        return {"decay": self._decay, "every": self._every, "warmup_steps": self._warmup}

    def state_dict(self) -> dict:
        """The settings, the EMA flats (CPU copies; this rank's shards when sharded, with ``sharded`` / ``world`` / ``rank``)
        and the fp32 buffers by name."""
        flats, bufs = self._ema_tensors()
        sd = dict(self._settings(), ema=[e.detach().cpu().clone() for e in flats],
                  buffers={n: e.detach().cpu().clone() for n, e in zip(self._buf_names, bufs)})
        sd.update(self._opt._shard_tags())
        return sd

    def _check_loadable(self, sd: dict, what: str) -> None:
        self._refuse_inside(what)
        saved = {k: sd.get(k) for k in self._settings()}
        if saved != self._settings():
            raise ValueError(f"FlatEMA.{what}: the state was written with {saved}, this EMA has {self._settings()}")

    @torch.no_grad()
    def load_state_dict(self, sd: dict) -> None:
        """Inverse of :meth:`state_dict`.  ``ValueError`` (before anything is loaded) for other settings, other buffers, or a
        shard of another rank or world size; ``RuntimeError`` inside :meth:`average_parameters`."""
        self._check_loadable(sd, "load_state_dict()")
        if sorted(sd["buffers"]) != sorted(self._buf_names):
            raise ValueError(f"FlatEMA.load_state_dict: the state holds the buffers {sorted(sd['buffers'])}, this EMA "
                             f"{sorted(self._buf_names)}")
        self._opt._load_flats(sd, [(self.ema_flats, sd["ema"])], "EMA", "named_ema() / load_named_ema()")
        for n, e in zip(self._buf_names, self.ema_buffers):
            e.copy_(sd["buffers"][n])

    def named_ema(self, model: nn.Module) -> dict:
        """``{name: EMA tensor}`` (CPU copies) for every parameter and averaged buffer, the form that crosses world sizes and
        sharded and unsharded runs (keys as in the module's ``state_dict()``).  Collective when sharded: every rank calls it
        and gets the whole tensors."""
        flats, bufs = self._ema_tensors()
        out = self._opt._named(model, flats)
        out.update({n: e.detach().cpu().clone() for n, e in zip(self._buf_names, bufs)})
        return out

    @torch.no_grad()
    def load_named_ema(self, model: nn.Module, named: dict) -> int:
        """Inverse of :meth:`named_ema`; returns how many tensors were restored.  Sharded, each rank keeps its slice."""
        self._refuse_inside("load_named_ema()")
        done = self._opt._load_named(model, named, self.ema_flats)
        for n, e in zip(self._buf_names, self.ema_buffers):
            if n in named:
                e.copy_(named[n])
                done += 1
        return done
