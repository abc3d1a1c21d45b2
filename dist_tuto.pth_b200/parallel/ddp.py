"""Synchronous data-parallel gradient averaging (layer L4, the hot path).

Parity: ``average_gradients(model)`` of train_dist.py:94-100 / tuto.md:310-314:
after the call every ``param.grad`` holds the mean over ranks.  (The committed
reference never communicates -- SURVEY §2.6 D1 -- we implement the documented
semantics.)

GPU-first design instead of "one blocking all_reduce + one divide per tensor":
  * :class:`GradBucket` -- all gradients of a model live in ONE flat buffer
    (``param.grad`` are views into it).  On a CUDA symmetric world the buffer is
    allocated in peer-mapped symmetric memory, so the all-reduce kernel reads
    the peers' gradients directly over NVSwitch: 1 launch instead of 16.
  * the reduction, the ``1/world_size`` scale and the dtype cast are fused in
    that one kernel (``ops/allreduce``), one-shot / two-shot / NVLS by size.
  * :class:`DistributedDataParallel` -- size-capped buckets in reverse
    parameter order; a post-accumulate-grad hook launches a bucket's all-reduce
    on a side stream as soon as its last gradient is written, overlapping
    communication with the rest of backward (tuto.md:216,320 points at the
    "official" DDP for this; here it is part of the library).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist
import torch.nn as nn

from .. import comm

__all__ = ["GradBucket", "average_gradients", "DistributedDataParallel", "broadcast_parameters",
           "flatten_params"]


def _symm_world(group, device):
    if device.type != "cuda":
        return None
    try:
        from . import symm
    except Exception:
        return None
    return symm.lookup_world(comm._g(group))


class GradBucket:
    """One flat gradient buffer; ``p.grad`` of every member is a view into it."""

    def __init__(self, params: Sequence[nn.Parameter], group=None, dtype: Optional[torch.dtype] = None,
                 align: int = 4, symmetric: bool = True):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("GradBucket needs at least one parameter that requires grad")
        self.group = group
        dev = self.params[0].device
        self.dtype = dtype or self.params[0].dtype
        for p in self.params:
            # reduced-precision gradient bucket (e.g. bf16 on the wire for fp32 master weights): autograd accumulates
            # straight into the bucket's dtype when the parameter says so (torch >= 2.x `Tensor.grad_dtype`)
            if p.dtype != self.dtype:
                if not hasattr(p, "grad_dtype"):
                    raise RuntimeError("a gradient bucket dtype different from the parameter dtype needs Tensor.grad_dtype")
                p.grad_dtype = self.dtype
        self.offsets, n = [], 0
        for p in self.params:
            if p.device != dev:
                raise ValueError("all parameters of a bucket must live on one device")
            self.offsets.append(n)
            n += (p.numel() + align - 1) // align * align
        self.numel = n
        self.world = _symm_world(group, dev) if symmetric else None
        self.symm_handle = None
        if self.world is not None:
            self.symm_handle = self.world.alloc(n, self.dtype)
            self.flat = self.symm_handle.local
            self.flat.zero_()
        else:
            self.flat = torch.zeros(n, dtype=self.dtype, device=dev)
        # a view has the parameter's own strides (e.g. channels_last conv weights), so autograd accumulates
        # straight into the bucket without a layout-converting copy
        self.views = []
        for o, p in zip(self.offsets, self.params):
            seg = self.flat[o:o + p.numel()]
            dense = p.is_contiguous() or p.numel() == 0
            if not dense and torch._debug_has_internal_overlap(p) == 0 and self._dense_strides(p):
                self.views.append(seg.as_strided(p.shape, p.stride()))
            else:
                self.views.append(seg.view(p.shape))
        self.attach()

    @staticmethod
    def _dense_strides(p) -> bool:
        """True when ``p`` covers exactly numel() elements under some dimension permutation."""
        dims = sorted(range(p.dim()), key=lambda d: (p.stride(d), p.size(d)))
        expect = 1
        for d in dims:
            if p.size(d) == 1:
                continue
            if p.stride(d) != expect:
                return False
            expect *= p.size(d)
        return expect == p.numel()

    def attach(self) -> None:
        """(Re)point every ``p.grad`` at its view (keeps current values)."""
        for p, v in zip(self.params, self.views):
            if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
            p.grad = v

    def zero_(self) -> None:
        """``optimizer.zero_grad()`` for the bucket: one memset of the flat buffer; re-attaches detached ``p.grad``."""
        self.flat.zero_()
        for p, v in zip(self.params, self.views):
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                p.grad = v

    def all_reduce_average_(self, max_blocks: Optional[int] = None) -> None:
        """flat <- mean over ranks (in place).  ``max_blocks`` caps the comm kernel's CTAs (overlap mode)."""
        size = comm.get_world_size(self.group)
        if size == 1:
            return
        if self.world is not None:
            self.world.all_reduce_(self.flat, scale=1.0 / size, handle=self.symm_handle, max_blocks=max_blocks)
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=comm._g(self.group))
            self.flat.div_(size)


def flatten_params(model: nn.Module) -> List[nn.Parameter]:
    """The trainable parameters in definition order (what ``model.parameters()`` of train_dist.py:97 iterates)."""
    return [p for p in model.parameters() if p.requires_grad]


def average_gradients(model: nn.Module, group=None) -> None:
    """Gradient averaging (tuto.md:310-314): ``p.grad <- mean_ranks(p.grad)``.

    * a model wrapped in :class:`DistributedDataParallel` (or carrying a
      :class:`GradBucket` as ``model._grad_bucket``) finishes / runs its fused
      bucketed all-reduce;
    * any other model: gradients are coalesced into one flat message (one
      collective instead of one per tensor), averaged and scattered back."""
    if isinstance(model, DistributedDataParallel):        # the wrapper itself (the natural call; FlatSGD accepts it too)
        model.finish()
        return
    eng = getattr(model, "_ddp_engine", None)             # the wrapped inner module
    if eng is not None:
        eng.finish()
        return
    bucket = getattr(model, "_grad_bucket", None)
    if bucket is not None:
        bucket.attach()
        bucket.all_reduce_average_()
        return
    size = comm.get_world_size(group)
    if size == 1:
        return
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    if not grads:
        return
    by_key = {}
    for g in grads:
        by_key.setdefault((g.device, g.dtype), []).append(g)
    for (dev, _), gs in by_key.items():
        flat = torch._utils._flatten_dense_tensors(gs) if len(gs) > 1 else gs[0].contiguous().view(-1)
        w = _symm_world(group, dev)
        if w is not None and w.supports(flat):
            w.all_reduce_(flat, scale=1.0 / size)
        else:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=comm._g(group))
            flat.div_(size)
        if len(gs) > 1:
            for g, r in zip(gs, torch._utils._unflatten_dense_tensors(flat, gs)):
                g.copy_(r)
        elif gs[0].data_ptr() != flat.data_ptr():
            gs[0].copy_(flat.view_as(gs[0]))


def broadcast_parameters(model: nn.Module, src: int = 0, group=None) -> None:
    """Make replicas identical without relying on equal seeds (the reference only
    has ``torch.manual_seed(1234)``, train_dist.py:105)."""
    if comm.get_world_size(group) == 1:
        return
    tensors = [p.data for p in model.parameters()] + [b.data for b in model.buffers()]
    by_key = {}
    for t in tensors:
        by_key.setdefault((t.device, t.dtype), []).append(t)
    for ts in by_key.values():
        flat = torch._utils._flatten_dense_tensors(ts)
        dist.broadcast(flat, src=src, group=comm._g(group))
        for t, r in zip(ts, torch._utils._unflatten_dense_tensors(flat, ts)):
            t.copy_(r)


class _Bucket:
    __slots__ = ("gb", "pending", "ready_event", "launched")

    def __init__(self, gb: GradBucket):
        self.gb, self.pending, self.ready_event, self.launched = gb, 0, None, False


class DistributedDataParallel(nn.Module):
    """Bucketed, overlapped gradient averaging around any ``nn.Module``.

    ``bucket_cap_bytes`` bounds each flat bucket; buckets are filled in reverse
    parameter order (the order backward produces gradients).  When the last
    gradient of a bucket has been accumulated, the bucket's fused all-reduce is
    enqueued on ``comm_stream`` behind an event, so it runs while autograd keeps
    producing earlier layers' gradients.  ``finish()`` (called by
    ``average_gradients(model)`` or ``optimizer`` glue) joins the streams."""

    def __init__(self, module: nn.Module, group=None, bucket_cap_bytes: int = 8 << 20,
                 overlap: bool = True, broadcast: bool = True, grad_dtype: Optional[torch.dtype] = None,
                 comm_blocks: int = 32):
        super().__init__()
        self.module = module
        self.group = group
        self.world_size = comm.get_world_size(group)
        params = flatten_params(module)
        if not params:
            raise ValueError("module has no trainable parameters")
        self.device = params[0].device
        self.overlap = bool(overlap) and self.device.type == "cuda" and self.world_size > 1
        # while backward kernels are running the comm kernel gets a slice of the SMs, not all of them
        self.comm_blocks = comm_blocks if self.overlap else None
        if broadcast:
            broadcast_parameters(module, 0, group)
        self._buckets: List[_Bucket] = []
        self._bucket_of = {}
        self._view_of = {}
        cur, cur_bytes = [], 0
        for p in reversed(params):
            nbytes = p.numel() * (torch.empty((), dtype=grad_dtype or p.dtype).element_size())
            if cur and cur_bytes + nbytes > bucket_cap_bytes:
                self._add_bucket(cur, grad_dtype)
                cur, cur_bytes = [], 0
            cur.append(p)
            cur_bytes += nbytes
        if cur:
            self._add_bucket(cur, grad_dtype)
        self.comm_stream = torch.cuda.Stream(self.device) if self.device.type == "cuda" else None
        self._hooks = []
        for p in params:
            self._hooks.append(p.register_post_accumulate_grad_hook(self._on_grad))
        object.__setattr__(module, "_ddp_engine", self)   # not a submodule (would be a cycle)
        self._reset()

    # -- construction -------------------------------------------------------
    def _add_bucket(self, params, grad_dtype):
        gb = GradBucket(params, group=self.group, dtype=grad_dtype)
        b = _Bucket(gb)
        for p, v in zip(gb.params, gb.views):
            self._bucket_of[p] = b
            self._view_of[p] = v
        self._buckets.append(b)

    @property
    def buckets(self) -> List[GradBucket]:
        """The flat gradient buckets, in the order backward completes them."""
        return [b.gb for b in self._buckets]

    def forward(self, *a, **kw):
        """Runs the wrapped module; gradient communication is driven by the hooks during ``backward()``."""
        return self.module(*a, **kw)

    # -- per-step state -----------------------------------------------------
    def _reset(self):
        for b in self._buckets:
            b.pending = len(b.gb.params)
            b.launched = False

    def zero_grad(self, set_to_none: bool = False):  # noqa: ARG002 - grads stay views
        """Zero every bucket (gradients stay views of the flat buffers) and re-arm the per-step hook bookkeeping."""
        for b in self._buckets:
            b.gb.zero_()
        self._reset()

    def _launch(self, b: _Bucket):
        b.launched = True
        if self.world_size == 1:
            return
        if self.overlap:
            cur = torch.cuda.current_stream(self.device)
            ev = torch.cuda.Event()
            ev.record(cur)
            self.comm_stream.wait_event(ev)
            with torch.cuda.stream(self.comm_stream):
                b.gb.all_reduce_average_(self.comm_blocks)
        else:
            b.gb.all_reduce_average_()

    def _on_grad(self, p: nn.Parameter):
        b = self._bucket_of[p]
        v = self._view_of[p]
        if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
            v.copy_(p.grad)       # optimizer.zero_grad(set_to_none=True) detached the view
            p.grad = v
        b.pending -= 1
        if b.pending == 0 and not b.launched:
            self._launch(b)

    def finish(self):
        """Complete all outstanding bucket all-reduces for this step."""
        for b in self._buckets:
            if not b.launched:      # unused parameters / hooks not fired
                self._launch(b)
        if self.overlap:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        self._reset()

    def remove_hooks(self):
        """Detach the engine from the module (hooks and the ``_ddp_engine`` back-reference)."""
        for h in self._hooks:
            h.remove()
        self._hooks = []
        if getattr(self.module, "_ddp_engine", None) is self:
            object.__delattr__(self.module, "_ddp_engine")
