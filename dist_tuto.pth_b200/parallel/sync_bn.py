"""SyncBatchNorm: batch statistics over the global batch of a data-parallel job, computed by sm_90a kernels.

:class:`SyncBatchNorm` is a drop-in for ``torch.nn.SyncBatchNorm`` (a subclass that overrides ``forward`` only, so
``isinstance``, the state-dict keys and ``load_state_dict`` are torch's) and follows its ``forward`` branch for branch.  What
differs is how a training step computes and exchanges the statistics:

* forward, per channel: the local count, ``S1 = sum x`` and ``S2 = sum x^2`` in fp64 (``bn_stats_kernel``), one fp64 SUM
  all-reduce of ``[count | S1 | S2]``, then ``bn_apply_kernel``: ``mean = S1/N``, ``var = max(S2/N - mean^2, 0)``,
  ``invstd = 1/sqrt(var + eps)`` in fp64, the running stats updated (with the unbiased ``var * N / (N - 1)``; the
  ``momentum=None`` factor ``1 / num_batches_tracked`` read on the device), and ``y = fmaf(x, k1, k0)`` with
  ``k1 = w invstd`` and ``k0 = b - mean k1`` rounded once to fp32;
* backward: the local ``sum dy`` and ``sum dy (x - mean)`` in fp64 (``bn_backward_reduce_kernel``, which also writes the local
  ``grad_bias`` / ``grad_weight``), one fp64 SUM all-reduce of the pair when the input gradient is wanted, and
  ``bn_backward_apply_kernel``: ``dx = dy ka + x kb + kc`` with coefficients rounded once from fp64.

The all-reduce is summed in rank order, so every rank ends a forward with bit-identical mean, invstd and running stats.  On a
peer-memory world (:class:`~.symm.SymmWorld`) it is ``SymmWorld.all_reduce_`` on the current stream; otherwise
``torch.distributed.all_reduce`` on the group (the two-level world, NCCL, gloo).  At world size 1 the exchange is skipped but
the same kernels run, so one GPU and eight share one numerics.  Nothing synchronises the host, so the step can be captured
in a CUDA graph.  On CPU tensors torch ops compute the same fp64 sums.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as tdist
import torch.nn.functional as F

from .. import comm

__all__ = ["SyncBatchNorm", "sync_batch_norm", "SyncBatchNormFunction", "exchange_numel"]

_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def exchange_numel(n: int, world: int) -> int:
    """``n`` fp64 values padded to a multiple of 16 x world bytes, so that the peer-memory all-reduce takes its staged,
    fused path (no copy around the kernel)."""
    m = 2 * max(1, world)
    return -(-n // m) * m


def _world_size(comm_) -> int:
    if comm_ is None:
        return 1
    if hasattr(comm_, "all_reduce_"):
        return comm_.world
    return tdist.get_world_size(comm_)


def _exchange(buf: torch.Tensor, comm_) -> None:
    """In-place fp64 SUM over the ranks: nothing for ``None``, the peer-memory kernel for a :class:`SymmWorld`, else
    ``torch.distributed.all_reduce`` on the process group ``comm_``."""
    if comm_ is None:
        return
    if hasattr(comm_, "all_reduce_"):
        comm_.all_reduce_(buf)
    else:
        tdist.all_reduce(buf, tdist.ReduceOp.SUM, group=comm_)


def _memory_format(x: torch.Tensor):
    if x.dim() == 4 and not x.is_contiguous() and x.is_contiguous(memory_format=torch.channels_last):
        return torch.channels_last
    if x.dim() == 5 and not x.is_contiguous() and x.is_contiguous(memory_format=torch.channels_last_3d):
        return torch.channels_last_3d
    return torch.contiguous_format


def _same_layout(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Same shape and the same strides on every dimension longer than 1 (the kernels' addressing)."""
    return a.shape == b.shape and all(n == 1 or sa == sb for n, sa, sb in zip(a.shape, a.stride(), b.stride()))


def _max_blocks(comm_, device) -> int:
    if comm_ is not None and hasattr(comm_, "max_blocks"):
        return int(comm_.max_blocks)
    return torch.cuda.get_device_properties(device).multi_processor_count


class SyncBatchNormFunction(torch.autograd.Function):
    """``y = batch_norm(x)`` with statistics over every rank of ``comm_`` (``None``: this rank alone; a
    :class:`~.symm.SymmWorld`; or a ``torch.distributed`` process group).  ``tickets``: an int32 tensor of at least C zeros on
    x's device that the kernels leave zero (CUDA only; one per module, used by one stream at a time)."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, num_batches_tracked, momentum, eps, comm_, tickets):
        if not x.is_contiguous(memory_format=_memory_format(x)):
            x = x.contiguous()
        C = x.shape[1]
        W = _world_size(comm_)
        ex = torch.empty(exchange_numel(1 + 2 * C, W), dtype=torch.float64, device=x.device)
        if x.is_cuda:
            from ..ops import _ext
            K = _ext.C()
            stats = torch.empty(2 * C + 1, dtype=torch.float64, device=x.device)
            mb = _max_blocks(comm_, x.device)
            K.bn_launch(0, x, None, None, ex, stats, tickets, None, None, None, None, None, None, None, 0.0, 0.0, mb)
            _exchange(ex, comm_)
            y = torch.empty_like(x)                          # x's strides, also for an empty local batch
            K.bn_launch(1, x, None, y, ex, stats, None, weight, bias, running_mean, running_var, num_batches_tracked, None,
                        None, float(momentum), float(eps), mb)
        else:
            y, stats = _cpu_forward(x, weight, bias, running_mean, running_var, num_batches_tracked, momentum, eps, ex,
                                    comm_)
        ctx.save_for_backward(x, weight, stats)
        ctx.comm_, ctx.W = comm_, W
        ctx.tickets = tickets
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, stats = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        if not _same_layout(dy, x):
            dy = torch.empty_like(x).copy_(dy)
        C = x.shape[1]
        gw = torch.empty_like(weight) if need_w and weight is not None else None
        gb = torch.empty_like(weight) if need_b and weight is not None else None
        dx = None
        if not (need_x or gw is not None or gb is not None):
            return (None,) * 10
        ex = torch.empty(exchange_numel(2 * C, ctx.W), dtype=torch.float64, device=x.device)
        if x.is_cuda:
            from ..ops import _ext
            K = _ext.C()
            mb = _max_blocks(ctx.comm_, x.device)
            K.bn_launch(2, x, dy, None, ex, stats, ctx.tickets, None, None, None, None, None, gw, gb, 0.0, 0.0, mb)
            if need_x:
                _exchange(ex, ctx.comm_)
                dx = torch.empty_like(x)
                K.bn_launch(3, x, dy, dx, ex, stats, None, weight, None, None, None, None, None, None, 0.0, 0.0, mb)
        else:
            dx = _cpu_backward(x, dy, weight, stats, ex, gw, gb, need_x, ctx.comm_)
        return dx, gw, gb, None, None, None, None, None, None, None


def _dims(x):
    return [0] + list(range(2, x.dim()))


def _bshape(x):
    return [1, -1] + [1] * (x.dim() - 2)


def _cpu_forward(x, weight, bias, running_mean, running_var, nbt, momentum, eps, ex, comm_):
    """The kernels' numerics on torch ops (CPU tensors): fp64 sums, fp64 statistics, fp32 coefficients."""
    C = x.shape[1]
    xd = x.double()
    ex.zero_()
    ex[0] = x.numel() // C if C else 0
    ex[1:1 + C] = xd.sum(_dims(x))
    ex[1 + C:1 + 2 * C] = (xd * xd).sum(_dims(x))
    _exchange(ex, comm_)
    N = ex[0]
    mean = ex[1:1 + C] / N
    var = (ex[1 + C:1 + 2 * C] / N - mean * mean).clamp_min(0.0)
    invstd = 1.0 / torch.sqrt(var + eps)
    w = weight.double() if weight is not None else torch.ones_like(mean)
    b = bias.double() if bias is not None else torch.zeros_like(mean)
    d1 = w * invstd
    k1, k0 = d1.float(), (b - mean * d1).float()
    y = torch.addcmul(k0.view(_bshape(x)), x.float(), k1.view(_bshape(x))).to(x.dtype)
    if running_mean is not None:
        with torch.no_grad():
            m = 1.0 / nbt.double() if nbt is not None else torch.tensor(float(momentum), dtype=torch.float64)
            running_mean.copy_(((1.0 - m) * running_mean.double() + m * mean).to(running_mean.dtype))
            running_var.copy_(((1.0 - m) * running_var.double() + m * (var * N / (N - 1.0))).to(running_var.dtype))
    stats = torch.cat([mean, invstd, N.view(1)])
    return y, stats


def _cpu_backward(x, dy, weight, stats, ex, gw, gb, need_x, comm_):
    C = x.shape[1]
    mean, invstd, N = stats[:C], stats[C:2 * C], stats[2 * C]
    dyd = dy.double()
    ex.zero_()
    ex[:C] = dyd.sum(_dims(x))
    ex[C:2 * C] = (dyd * (x.double() - mean.view(_bshape(x)))).sum(_dims(x))
    if gb is not None:
        gb.copy_(ex[:C])
    if gw is not None:
        gw.copy_(ex[C:2 * C] * invstd)
    if not need_x:
        return None
    _exchange(ex, comm_)
    w = weight.double() if weight is not None else torch.ones_like(mean)
    da = w * invstd
    db = -da * invstd * invstd * (ex[C:2 * C] / N)
    dc = -da * (ex[:C] / N) - db * mean
    s = _bshape(x)
    return (dy.float() * da.float().view(s) + (x.float() * db.float().view(s) + dc.float().view(s))).to(x.dtype)


def sync_batch_norm(x, weight, bias, running_mean, running_var, num_batches_tracked, momentum, eps, comm_=None,
                    tickets: Optional[torch.Tensor] = None):
    """Functional form of :class:`SyncBatchNorm`'s training path (see :class:`SyncBatchNormFunction`)."""
    if x.is_cuda and tickets is None:
        tickets = torch.zeros(x.shape[1], dtype=torch.int32, device=x.device)
    return SyncBatchNormFunction.apply(x, weight, bias, running_mean, running_var, num_batches_tracked, momentum, eps, comm_,
                                       tickets)


class SyncBatchNorm(torch.nn.SyncBatchNorm):
    """``torch.nn.SyncBatchNorm`` with the statistics computed and exchanged by this library's kernels.

    Same constructor, parameters, buffers and state dict as torch's.  Inputs of rank >= 2 in fp32, bf16 or fp16; weight,
    bias and running stats fp32 or the input's dtype.  Training uses the global batch's statistics over ``process_group``
    (default: the whole world); ``model.eval()`` with running stats runs plain ``F.batch_norm`` and communicates nothing.
    Local batch sizes may differ between ranks, including 0: every rank still takes part in both exchanges.
    ``grad_weight`` / ``grad_bias`` are the local sums, as in torch; data parallelism averages them."""

    def _tickets(self, x: torch.Tensor) -> Optional[torch.Tensor]:
        if not x.is_cuda:
            return None
        t = getattr(self, "_bn_tickets", None)
        if t is None or t.device != x.device or t.numel() < x.shape[1]:
            t = torch.zeros(x.shape[1], dtype=torch.int32, device=x.device)
            self._bn_tickets = t
        return t

    def _comm(self, x: torch.Tensor):
        """The exchange of a training forward: None when this rank is alone, the peer-memory world serving the group when
        one was built on CUDA, else the process group."""
        if not (tdist.is_available() and tdist.is_initialized()):
            return None
        group = self.process_group if self.process_group is not None else tdist.group.WORLD
        if tdist.get_world_size(group) == 1:
            return None
        if x.is_cuda:
            from . import symm
            w = symm.lookup_world(comm._g(self.process_group))
            if isinstance(w, symm.SymmWorld):
                return w
        return group

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        self._check_input_dim(input)
        self._check_non_zero_input_channels(input)
        factor = 0.0 if self.momentum is None else self.momentum
        nbt = None
        if self.training and self.track_running_stats:
            self.num_batches_tracked.add_(1)
            if self.momentum is None:
                nbt = self.num_batches_tracked
        bn_training = self.training or (self.running_mean is None and self.running_var is None)
        running_mean = self.running_mean if not self.training or self.track_running_stats else None
        running_var = self.running_var if not self.training or self.track_running_stats else None
        if not bn_training:
            return F.batch_norm(input, running_mean, running_var, self.weight, self.bias, False, factor, self.eps)
        comm_ = self._comm(input) if self.training else None
        if comm_ is None and input.numel() // input.shape[1] == 1:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size {input.size()}")
        if input.is_cuda and input.dtype not in _CODES:
            raise TypeError(f"SyncBatchNorm takes fp32, bf16 or fp16 CUDA inputs, got {input.dtype}")
        return sync_batch_norm(input, self.weight, self.bias, running_mean, running_var, nbt, factor, self.eps, comm_,
                               self._tickets(input))

    @classmethod
    def convert_sync_batchnorm(cls, module, process_group=None):
        """Replace every ``_BatchNorm`` of ``module`` (torch's ``SyncBatchNorm`` included) by a :class:`SyncBatchNorm`
        sharing its ``Parameter`` and buffer objects, ``training`` flag and ``requires_grad``; returns the new module when
        ``module`` itself is one."""
        out = module
        if isinstance(module, torch.nn.modules.batchnorm._BatchNorm):
            out = cls(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats,
                      process_group)
            if module.affine:
                with torch.no_grad():
                    out.weight = module.weight
                    out.bias = module.bias
            out.running_mean = module.running_mean
            out.running_var = module.running_var
            out.num_batches_tracked = module.num_batches_tracked
            out.training = module.training
            if hasattr(module, "qconfig"):
                out.qconfig = module.qconfig
        for name, child in module.named_children():
            out.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        del module
        return out
