"""Test-set evaluation of the tutorial ConvNet: loss and accuracy over a dataset, sharded over the ranks of a group.

The device path is one launch of the forward-only sm_90a kernel ``convnet_eval`` (csrc/convnet_eval.cu): fp32, eval mode,
deterministic (two calls on the same device and input are bit-equal), result ``{nll sum, #correct, #samples}`` in a
float64 device tensor.  Every rank evaluates its contiguous shard (``data.partition_eval_dataset``) and the three sums
are added over the group with one ``all_reduce`` of float64, so counts stay exact and every rank gets the same result.

    from dist_tuto.pth_b200 import evaluate
    evaluate(trainer)                      # FusedTrainer / BatchedTrainer / Net; default test set
    trainer.evaluate(test_set)

A ``Net`` on CPU is evaluated with torch ops (``Net.eval()``, in chunks), with the same sharding and cross-rank sum.
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import comm
from ..data import MNIST_MEAN, MNIST_STD, default_eval_dataset, eval_shard_range
from . import _ext

__all__ = ["convnet_evaluate", "Evaluator", "evaluate"]

_CPU_CHUNK = 2048


def convnet_evaluate(params: torch.Tensor, x: torch.Tensor, target: torch.Tensor, mean: float = MNIST_MEAN,
                     std: float = MNIST_STD, out_logp: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One launch of the eval kernel on the current stream.  ``x``: uint8 ``[N,28,28]`` (normalised in the kernel with
    ``mean`` / ``std``) or normalised float32 ``[N,1,28,28]``; ``target``: int64 ``[N]``.  Returns the device float64
    tensor ``[nll sum, #correct, N]``; ``out_logp`` (float32 ``[N,10]``) receives the log-probabilities."""
    C = _ext.C()
    dev = params.device
    x = x.contiguous()
    if x.data_ptr() % 16:                    # the kernel bulk-copies each group of images: 16-byte aligned source
        x = x.clone()
    result = torch.empty(3, dtype=torch.float64, device=dev)
    slots = torch.zeros(C.convnet_eval_slot_words(params.get_device()), dtype=torch.int32, device=dev)
    C.convnet_eval(params, x, target.contiguous(), result, slots, float(mean), float(std), out_logp)
    return result


def _shard_tensors(dataset, rank: int, world: int) -> Tuple[torch.Tensor, torch.Tensor, float, float]:
    """This rank's shard on the host: tensor-backed datasets as raw uint8 images (with their mean / std), any other
    dataset of ``(image, label)`` items gathered into normalised float32."""
    lo, hi = eval_shard_range(len(dataset), rank, world)
    if hasattr(dataset, "images") and hasattr(dataset, "labels"):
        x, y = dataset.images[lo:hi], dataset.labels[lo:hi].to(torch.int64)
        mean, std = float(getattr(dataset, "mean", MNIST_MEAN)), float(getattr(dataset, "std", MNIST_STD))
    else:
        items = [dataset[i] for i in range(lo, hi)]
        x = torch.stack([torch.as_tensor(it[0], dtype=torch.float32).reshape(1, 28, 28) for it in items]) if items else \
            torch.empty(0, 1, 28, 28, dtype=torch.float32)
        y = torch.as_tensor([int(it[1]) for it in items], dtype=torch.int64)
        mean, std = MNIST_MEAN, MNIST_STD
    if y.numel() and (int(y.min()) < 0 or int(y.max()) > 9):
        raise ValueError("evaluation labels must lie in [0, 10)")
    return x.contiguous(), y.contiguous(), mean, std


def _group_sum(t: torch.Tensor, group) -> torch.Tensor:
    """Sum a float64 ``[3]`` tensor over the group (NCCL takes it on the device, gloo on the host)."""
    if comm.is_initialized() and comm.get_world_size(group) > 1:
        if t.is_cuda and dist.get_backend(comm._g(group)) != "nccl":
            t = t.cpu()
        comm.all_reduce(t, group=group)
    return t


def _as_dict(total) -> Dict:
    loss, correct, n = (float(v) for v in total)
    n, correct = int(n), int(correct)
    return {"loss": loss / n if n else float("nan"), "accuracy": correct / n if n else float("nan"),
            "correct": correct, "n": n}


def _rank_world(group) -> Tuple[int, int]:
    if not comm.is_initialized():
        return 0, 1
    return comm.group_ranks(group).index(comm.get_rank()), comm.get_world_size(group)


class Evaluator:
    """What a repeated evaluation on one device needs: the rank's shard of the last dataset evaluated, copied to the
    device once and reused while the same dataset object comes back; the slot and result buffers of the kernel; the
    cross-rank sum.  Collective over ``group`` when the group has more than one rank."""

    def __init__(self, device, group=None):
        self.device = torch.device(device)
        self.group = group
        C = _ext.C()
        self.result = torch.zeros(3, dtype=torch.float64, device=self.device)
        self.slots = torch.zeros(C.convnet_eval_slot_words(self.device.index if self.device.index is not None
                                                           else torch.cuda.current_device()),
                                 dtype=torch.int32, device=self.device)
        self._dataset = None
        self._shard = None

    def shard(self, dataset):
        """``(x, target, mean, std)`` of this rank's shard on the device (cached for the same dataset object)."""
        if self._dataset is not dataset:
            rank, world = _rank_world(self.group)
            x, y, mean, std = _shard_tensors(dataset, rank, world)
            self._shard = (x.to(self.device), y.to(self.device), mean, std)
            torch.cuda.current_stream(self.device).synchronize()
            self._dataset = dataset
        return self._shard

    def run(self, params: torch.Tensor, dataset=None, stream: Optional[torch.cuda.Stream] = None) -> Dict:
        """Evaluate the flat parameters ``params`` on ``dataset`` (default: ``default_eval_dataset()``), launched on
        ``stream`` (default: the current stream), so it is ordered after the work already queued there."""
        ds = default_eval_dataset() if dataset is None else dataset
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            x, y, mean, std = self.shard(ds)
            _ext.C().convnet_eval(params, x, y, self.result, self.slots, mean, std, None)
            total = _group_sum(self.result.clone(), self.group)
            return _as_dict(total.tolist())


_NET_EVALUATORS: Dict[Tuple[str, int], Evaluator] = {}


def _evaluate_cpu(net: torch.nn.Module, dataset, group) -> Dict:
    """``Net.eval()`` in chunks with torch ops; same sharding and cross-rank sum as the kernel path."""
    rank, world = _rank_world(group)
    lo, hi = eval_shard_range(len(dataset), rank, world)
    was_training = net.training
    net.eval()
    loss, correct = torch.zeros((), dtype=torch.float64), 0
    try:
        with torch.no_grad():
            for s in range(lo, hi, _CPU_CHUNK):
                e = min(hi, s + _CPU_CHUNK)
                if hasattr(dataset, "gather"):
                    x, y = dataset.gather(torch.arange(s, e))
                else:
                    items = [dataset[i] for i in range(s, e)]
                    x = torch.stack([torch.as_tensor(it[0], dtype=torch.float32).reshape(1, 28, 28) for it in items])
                    y = torch.as_tensor([int(it[1]) for it in items], dtype=torch.int64)
                out = net(x)
                loss += F.nll_loss(out.double(), y, reduction="sum")
                correct += int((out.argmax(1) == y).sum())
    finally:
        net.train(was_training)
    total = torch.tensor([float(loss), float(correct), float(hi - lo)], dtype=torch.float64)
    return _as_dict(_group_sum(total, group).tolist())


def evaluate(model, dataset=None, group=None) -> Dict:
    """Test loss and accuracy of ``model`` on ``dataset`` (default: the MNIST test split, or its synthetic stand-in):
    ``{"loss": mean nll, "accuracy": correct / n, "correct": int, "n": int}``.

    Collective over ``group``: every rank passes the full dataset and evaluates its own contiguous shard; the sums are
    added over the ranks, so every rank returns the same dict.  ``model`` is a ``FusedTrainer``, a ``BatchedTrainer`` or
    a ``Net``: trainers and a ``Net`` on CUDA run the sm_90a eval kernel, a ``Net`` on CPU runs torch ops.  An empty
    dataset gives ``n == 0`` and NaN loss and accuracy."""
    if dataset is None:
        dataset = default_eval_dataset()
    if isinstance(model, torch.nn.Module):
        p = next(model.parameters())
        if not p.is_cuda:
            return _evaluate_cpu(model, dataset, group)
        from .convnet_fused import pack_params
        key = (str(p.device), id(group))
        ev = _NET_EVALUATORS.get(key)
        if ev is None or ev.group is not group:
            ev = _NET_EVALUATORS[key] = Evaluator(p.device, group)
        return ev.run(pack_params(model), dataset)
    if not (hasattr(model, "params") and hasattr(model, "stream")):
        raise TypeError(f"evaluate() takes a FusedTrainer, BatchedTrainer or Net, not {type(model).__name__}")
    if group is None or group is model.group:
        return model.evaluate(dataset)
    return Evaluator(model.device, group).run(model.params, dataset, stream=model.stream)
