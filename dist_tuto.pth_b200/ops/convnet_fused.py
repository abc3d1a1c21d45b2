"""Fused sm_90a training engine for the tutorial ConvNet.

One training step of the reference (train_dist.py:118-124:
``zero_grad -> model(data) -> nll_loss -> backward -> average_gradients -> step``)
is TWO kernels here, replayed as one CUDA graph:

  1. ``convnet_step``   (csrc/convnet.cu, csrc/convnet_cluster.cu)  forward + loss +
     backward, one CTA (or one 2/4/8-CTA cluster) per sample, gradients
     ``red.add``-ed into a flat fp32 bucket that lives in symmetric peer memory;
     on one GPU at one CTA per sample instead stored to per-CTA slots and per-sample
     fc1 factors, which ``reduce_sgd`` (csrc/sgd.cu) sums in a fixed order and feeds
     straight into the SGD update (no bucket, no atomics);
  2. ``allreduce_sgd``  (csrc/sgd.cu)      every rank stores its bucket, flag-in-data,
     into every peer's inbox over NVSwitch (or, ``B200DIST_SGD_PUSH=0``: flag barrier
     + loads of the peers' buckets), averages in fixed rank order, applies momentum
     SGD to the flat fp32 parameters, re-zeroes the bucket of the other step parity
     and bumps the RNG step counter.

The graph also contains the H2D copy of the batch from a pinned staging slot
and the D2H copy of the running loss, so the host issues ONE launch per step.

Parameter names/shapes/order follow the reference ``Net`` (state_dicts
interchange with ``models.convnet.Net``).
"""
from __future__ import annotations

import os
from collections import deque
from typing import Dict, Optional

import torch
import torch.distributed as dist

from .. import comm
from ..models.convnet import PARAM_SHAPES, Net
from . import _ext
from .optim import LRSchedule, schedule_tuple

__all__ = ["LAYOUT", "NPAR", "pack_params", "unpack_params", "convnet_loss_and_grads", "convnet_forward",
           "FusedTrainer"]

# padded flat layout: must match csrc/convnet.cu
LAYOUT: Dict[str, int] = {"conv1.weight": 0, "conv1.bias": 252, "conv2.weight": 264, "conv2.bias": 5264,
                          "fc1.weight": 5284, "fc1.bias": 21284, "fc2.weight": 21336, "fc2.bias": 21836}
NPAR = 21848
NPAR_ALLOC = 21888          # multiple of 64 elements (two-shot / NVLS slicing for any world <= 8)
FAC_STRIDE = 384            # per-sample fc1 factors of the step kernel: dh at [0, 50), p2 at [64, 384) (csrc/convnet_args.cuh)


def unpack_params(flat: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Named views (reference parameter names) into a flat buffer."""
    out = {}
    for name, shape in PARAM_SHAPES:
        n = 1
        for s in shape:
            n *= s
        out[name] = flat[LAYOUT[name]:LAYOUT[name] + n].view(shape)
    return out


def pack_params(src, device=None) -> torch.Tensor:
    """Flat fp32 buffer from a ``Net`` / state_dict (padding zero)."""
    sd = src.state_dict() if hasattr(src, "state_dict") else src
    dev = device if device is not None else next(iter(sd.values())).device
    flat = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=dev)
    views = unpack_params(flat)
    for name, _ in PARAM_SHAPES:
        views[name].copy_(sd[name].detach().to(torch.float32))
    return flat


def pick_cluster(bsz: int) -> int:
    """CTAs per sample for the fused step.

    With the reference's fixed global batch of 128 a GPU holds 128/N samples; a cluster per sample turns idle SMs into
    a shorter per-sample latency (csrc/convnet_cluster.cu).  Every choice keeps batch x cluster within one wave of the
    132 SMs of an H100; clusters of 8 are used only when the batch is <= 8.  ``B200DIST_CONVNET_CLUSTER`` overrides."""
    env = os.environ.get("B200DIST_CONVNET_CLUSTER")
    if env is not None:
        return int(env)
    if bsz <= 8:
        return 8
    if bsz <= 32:
        return 4
    if bsz <= 64:
        return 2
    return 1


def convnet_loss_and_grads(params: torch.Tensor, x: torch.Tensor, target: torch.Tensor, training: bool = False,
                           seed: int = 0, step: Optional[torch.Tensor] = None, sample_base: int = 0,
                           p_drop: float = 0.5, return_masks: bool = False, grads: Optional[torch.Tensor] = None,
                           cluster: int = 1):
    """Functional entry: returns ``(mean_nll, grads_flat[, masks])`` for one batch (used by tests)."""
    C = _ext.C()
    B = target.numel()
    if grads is None:
        grads = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=params.device)
    acc = torch.zeros(2, dtype=torch.float32, device=params.device)
    masks = torch.empty(B, 70, dtype=torch.float32, device=params.device) if return_masks else None
    C.convnet_step(params, grads, x.contiguous(), target.contiguous(), acc, None, masks, step, seed, sample_base,
                   training, 1.0 / B, p_drop, 0, 0, cluster)
    return (acc[0], grads, masks) if return_masks else (acc[0], grads)


def convnet_forward(params: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """Eval-mode forward: log-probabilities ``[B,10]`` (same semantics as ``Net.eval()(x)``)."""
    C = _ext.C()
    B = x.shape[0]
    out = torch.empty(B, 10, dtype=torch.float32, device=params.device)
    dummy_t = torch.zeros(B, dtype=torch.int64, device=params.device)
    C.convnet_step(params, None, x.contiguous(), dummy_t, None, out, None, None, 0, 0, False, 1.0 / max(B, 1), 0.5, 0)
    return out


class _Slot:
    __slots__ = ("x_pin", "y_pin", "loss_pin", "graph", "event", "busy")


class FusedTrainer:
    """Synchronous data-parallel SGD for the ConvNet, fully fused (see module docstring)."""

    def __init__(self, bsz: int, lr: float = 0.01, momentum: float = 0.5, seed: int = 1234, device=None,
                 p_drop: float = 0.5, group=None, raw_uint8: bool = False, num_slots: int = 4,
                 use_graph: bool = True, init_from: Optional[Net] = None, cluster: Optional[int] = None,
                 deterministic: bool = False, grad_wire: Optional[torch.dtype] = None,
                 lr_schedule: Optional[LRSchedule] = None):
        self.C = _ext.C()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.bsz, self._lr, self.mu, self.seed, self.p_drop = int(bsz), float(lr), float(momentum), int(seed), p_drop
        # lr_schedule (ops/optim.LRSchedule, step units): the optimizer kernels compute each update's lr from the device step
        # counter (csrc/lr_schedule.h), so graph replays and run_native follow it with fixed launch arguments
        self._sched = schedule_tuple(lr_schedule)
        self.lr_schedule = lr_schedule
        self.group = group
        # grad_wire=torch.bfloat16: the push exchange sends the locally reduced gradients as bf16 (one 16-byte line per
        # float4 instead of two: half the NVLink bytes, stores and polling loads); accumulation and master weights stay fp32
        # and all ranks sum the same rounded values, so replicas remain bit-identical (BASELINE config #2 "bf16 <-> fp32 cast").
        env_wire = os.environ.get("B200DIST_WIRE", "").lower()
        if grad_wire is None and env_wire in ("bf16", "fp32"):
            grad_wire = torch.bfloat16 if env_wire == "bf16" else torch.float32
        if grad_wire is None and comm.get_world_size(group) >= 4:
            # the exchange is what separates many GPUs from 1, so from 4 ranks up the wire is bf16 by default (half the bytes
            # per line, fp32 accumulation); pass grad_wire=torch.float32 for an exact fp32 exchange
            grad_wire = torch.bfloat16
        if grad_wire not in (None, torch.float32, torch.bfloat16):
            raise ValueError("grad_wire must be None/float32 or bfloat16")
        self.wire_bf16 = grad_wire == torch.bfloat16
        self.world = comm.get_world_size(group)
        self.rank = comm.group_ranks(group).index(comm.get_rank()) if comm.is_initialized() else 0
        self.raw_uint8 = raw_uint8
        self.training = True
        self.cluster = pick_cluster(self.bsz) if cluster is None else int(cluster)
        # identical replicas: same seed AND an explicit broadcast (the reference relies on the seed only)
        if init_from is None:
            torch.manual_seed(seed)
            init_from = Net(p_drop)
        self.params = pack_params(init_from, self.device)
        if self.world > 1:
            dist.broadcast(self.params, src=comm.group_ranks(group)[0], group=comm._g(group))
        self.momentum = torch.zeros_like(self.params)
        # conv2.weight pre-arranged in the two shared-memory layouts of the kernels; kept current by the SGD kernel
        self.aux = torch.zeros(13000, dtype=torch.float32, device=self.device)
        self._refresh_aux()
        self.symm = None
        self.grad_handle = None
        if self.world > 1:
            from ..parallel import symm
            self.symm = symm.lookup_world(comm._g(group)) or symm.init_world(comm._g(group))
            if not isinstance(self.symm, symm.SymmWorld):     # parallel/hier.HierWorld: the job spans several machines
                raise RuntimeError("the fused gradient exchange runs inside ONE NVSwitch domain; on several machines use "
                                   "train(engine='torch') / DistributedDataParallel (two-level all-reduce, parallel/hier.py)")
            self.grad_handle = self.symm.alloc(2 * NPAR_ALLOC, torch.float32)
            self.grads = self.grad_handle.local
            self.grads.zero_()
            self._grad_ptrs, self._sig_ptrs = self.grad_handle.ptrs, self.grad_handle.sig_ptrs
        else:
            self.grads = torch.zeros(2 * NPAR_ALLOC, dtype=torch.float32, device=self.device)
            self._grad_ptrs, self._sig_ptrs = [self.grads.data_ptr()], [0]
        # push exchange (csrc/sgd.cu, allreduce_sgd_push_kernel): every rank stores its bucket, flag-in-data, into every
        # peer's inbox and then reduces out of local memory -- one NVLink crossing instead of flag barrier + load round trip
        self.inbox_handle, self._inbox_ptrs = None, []
        if self.world > 1 and os.environ.get("B200DIST_SGD_PUSH", "1") != "0":
            self.inbox_handle = self.symm.alloc(2 * self.world * (NPAR_ALLOC // 4) * 8, torch.int32)
            self._inbox_ptrs = self.inbox_handle.ptrs
            self._reset_exchange()
        # two gradient buckets, selected by (step & 1) inside the kernels: the all-reduce kernel re-zeroes the bucket
        # of the previous step, which needs no second cross-GPU barrier (see csrc/sgd.cu)
        self.grad_stride = NPAR_ALLOC
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.done_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.loss_acc = torch.zeros(2, dtype=torch.float32, device=self.device)   # [sum of batch-mean nll, #correct]
        xdt = torch.uint8 if raw_uint8 else torch.float32
        self.x_dev = torch.zeros(self.bsz, 1, 28, 28, dtype=xdt, device=self.device)
        self.y_dev = torch.zeros(self.bsz, dtype=torch.int64, device=self.device)
        self.use_graph = use_graph
        self.stream = torch.cuda.Stream(self.device)
        self.slots = []
        for _ in range(max(2, num_slots)):
            s = _Slot()
            s.x_pin = torch.zeros(self.bsz, 1, 28, 28, dtype=xdt).pin_memory()
            s.y_pin = torch.zeros(self.bsz, dtype=torch.int64).pin_memory()
            s.loss_pin = torch.zeros(2, dtype=torch.float32).pin_memory()
            s.graph, s.event, s.busy = None, torch.cuda.Event(), False
            self.slots.append(s)
        self._executors = {}                        # id(loader) -> (C++ StepExecutor, training flag)
        self._ext_slots: Dict[int, _Slot] = {}      # loader-owned pinned buffers -> their graphs
        self._order = deque()                       # slots in flight, oldest first
        self._nstep = 0
        self._loss_read = 0.0                       # cumulative loss already returned by pop_loss_sum
        self._last_loss_cum = 0.0
        # deterministic=True: every step CTA stores its gradient sums to a private slot and `det_reduce` adds the slots in
        # CTA order (instead of float red.add into one bucket) => two runs with the same seed are bit-identical, at the
        # price of one more small kernel per step.  Used with several GPUs or clusters, by step() / the graph path only (the
        # C++ executor keeps the atomic flush there).  One GPU at one CTA per sample needs no flag: that path
        # has no atomics (below), in step() and in the executor alike.
        self.deterministic = bool(deterministic)
        self.sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        self.det_partials = None
        if deterministic and not (self.world == 1 and self.cluster == 1):
            self.det_partials = torch.zeros(self.sms * NPAR_ALLOC, dtype=torch.float32, device=self.device)
        # One GPU, one CTA per sample (the flagship, batch >= 65): no atomics at all.  Every step CTA stores its gradient sums
        # to its own slot and each sample its fc1 factors dh and p2 (plain stores); the optimizer kernel (`reduce_sgd`) sums
        # them in a fixed order and applies SGD from registers.  Bit-reproducible without `deterministic`.  The buffers
        # belong to the trainer so that captured graphs see fixed addresses, and are allocated here for every trainer whose
        # full batch can take this path (cluster 1, or clusters that do not fit one wave and fall back to one CTA per sample).
        self.grad_slots, self.factors = None, None
        if self.world == 1 and (self.cluster == 1 or self.bsz * self.cluster > self.sms):
            self._work_buffers(self.bsz)
        # Read by bench.py, whose result line names the step's kernels and counts its launches: every step is the step
        # kernel followed by one optimizer kernel.
        self.fused_tail = False
        self.gpu_launches_per_step = 2
        self._evaluator = None                      # ops/convnet_eval.Evaluator, made on the first evaluate()
        self._warm()

    def _reset_exchange(self):
        """Collective: bring the cross-step exchange state back to 'before the first step' -- both gradient buckets zero
        (the kernels only re-zero the bucket of the previous parity) and the push inbox empty (epoch 0).  Called at
        construction and whenever the step counter, which selects the bucket and is the epoch source, is rewritten.
        The barriers make sure no peer is still reading our bucket / writing our inbox, and that nobody starts stepping
        before everyone has cleaned up."""
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            comm.barrier(self.group)
        self.grads.zero_()
        if self.inbox_handle is not None:
            self.inbox_handle.local.zero_()
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            comm.barrier(self.group)

    def _refresh_aux(self):
        """(Re)build the pre-arranged conv2.weight copies from the flat parameters (init / load_state_dict)."""
        w2 = self.params[LAYOUT["conv2.weight"]:LAYOUT["conv2.weight"] + 5000].view(20, 10, 25)
        self.aux[:5000].copy_(w2.permute(1, 2, 0).reshape(-1))                       # w2f [ci][k][co]
        wb = torch.zeros(20, 25, 2, 8, dtype=torch.float32, device=self.device)
        wb[:, :, :, :5] = w2.view(20, 2, 5, 25).permute(0, 3, 1, 2)                  # w2b [co][k][half][8]
        self.aux[5000:].copy_(wb.reshape(-1))

    # ------------------------------------------------------------------ kernels
    def _step_ctas(self, B):
        """CTAs of the one-CTA-per-sample step kernel at batch ``B`` (= slots): one per sample, at most 4 per SM beyond that."""
        return min(B, 4 * self.sms)

    def _work_buffers(self, B):
        """Slots and factor rows for batch ``B`` (grown, never shrunk).  The full batch's buffers exist from construction;
        only eager batches larger than it grow them, and never inside graph capture."""
        n = self._step_ctas(B)
        grow = (self.grad_slots is None or self.grad_slots.numel() < n * NPAR_ALLOC or self.factors is None
                or self.factors.numel() < B * FAC_STRIDE)
        if grow and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"FusedTrainer: slot buffers for batch {B} must exist before graph capture")
        if self.grad_slots is None or self.grad_slots.numel() < n * NPAR_ALLOC:
            self.grad_slots = torch.zeros(n * NPAR_ALLOC, dtype=torch.float32, device=self.device)
        if self.factors is None or self.factors.numel() < B * FAC_STRIDE:
            self.factors = torch.zeros(B * FAC_STRIDE, dtype=torch.float32, device=self.device)

    def _native_slots(self):
        """(slots, factors) for the C++ executor when it runs the no-atomics one-GPU path (same condition as ``_kernels``)."""
        if self.world == 1 and self.cluster == 1 and self._step_ctas(self.bsz) == self.bsz:
            return self.grad_slots, self.factors
        return None, None

    def _kernels(self, x, y, B, input_ready=True):
        """Enqueue one step.  ``input_ready``: ``x`` and ``y`` were not written by the kernel enqueued right before this
        step (they come from copies or from work that finished earlier), so the step kernel may load them while it waits
        for the previous step's optimizer kernel."""
        cl = self.cluster if B * self.cluster <= self.sms else 1
        if self.world == 1 and cl == 1:
            self._work_buffers(B)
            n = self._step_ctas(B)
            self.C.convnet_step(self.params, self.grads, x, y, self.loss_acc, None, None, self.step_counter, self.seed,
                                self.rank * self.bsz, self.training, 1.0 / B, self.p_drop, n if n < B else 0, self.grad_stride,
                                1, self.aux, det_partials=self.grad_slots, factors=self.factors, input_ready=input_ready)
            # grads: re-zeroes the other-parity bucket, which a bucket step (the executor's) may use next
            self.C.reduce_sgd(self.grad_slots, n, self.factors, B, self.params, self.momentum, self.step_counter,
                              self.done_counter, self.lr, self.mu, self.aux, self.loss_acc, self.grads, self.grad_stride,
                              lr_schedule=self._sched)
            return
        if self.deterministic and B * cl <= self.sms:
            self.C.convnet_step(self.params, self.grads, x, y, self.loss_acc, None, None, self.step_counter, self.seed,
                                self.rank * self.bsz, self.training, 1.0 / B, self.p_drop, 0, self.grad_stride, cl, self.aux,
                                det_partials=self.det_partials)
            self.C.det_reduce(self.det_partials, B * cl, self.grads, self.step_counter, self.grad_stride, self.loss_acc)
        else:
            self.C.convnet_step(self.params, self.grads, x, y, self.loss_acc, None, None, self.step_counter, self.seed,
                                self.rank * self.bsz, self.training, 1.0 / B, self.p_drop, 0, self.grad_stride, cl, self.aux)
        self.C.allreduce_sgd(self._grad_ptrs, self._sig_ptrs, self.params, self.momentum, self.step_counter,
                             self.lr, self.mu, 1.0 / self.world, self.rank, self.world, True, self.grad_stride,
                             self.done_counter, self.aux, self._inbox_ptrs, self.wire_bf16, lr_schedule=self._sched)

    def _warm(self):
        # forward-only launch: sets the kernel's dynamic-smem attribute outside of graph capture
        with torch.cuda.stream(self.stream):
            self.C.convnet_step(self.params, None, self.x_dev, self.y_dev, None, None, None, None, 0, 0, False,
                                1.0 / self.bsz, self.p_drop, 0)
        self.stream.synchronize()

    def _capture(self, slot: _Slot):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=self.stream):
            self.x_dev.copy_(slot.x_pin, non_blocking=True)
            self.y_dev.copy_(slot.y_pin, non_blocking=True)
            self._kernels(self.x_dev, self.y_dev, self.bsz)
            slot.loss_pin.copy_(self.loss_acc, non_blocking=True)
        slot.graph = g

    # ------------------------------------------------------------------ stepping
    def _retire_oldest(self):
        s = self._order.popleft()
        s.event.synchronize()
        s.busy = False
        self._last_loss_cum = float(s.loss_pin[0])
        return s

    def sync_lag(self, keep: int = 0):
        """Block until at most ``keep`` steps are still in flight (bounds host run-ahead)."""
        while len(self._order) > keep:
            self._retire_oldest()

    def _slot_for(self, data: torch.Tensor, target: torch.Tensor) -> _Slot:
        key = data.data_ptr()
        s = self._ext_slots.get(key)
        if s is not None:
            return s
        if data.device.type == "cpu" and data.is_pinned() and target.is_pinned() and \
                data.dtype == self.x_dev.dtype and data.numel() == self.x_dev.numel() and len(self._ext_slots) < 16:
            # a loader-owned pinned buffer: adopt it as a graph source (zero extra host copies)
            s = _Slot()
            s.x_pin, s.y_pin = data.view(self.bsz, 1, 28, 28), target
            s.loss_pin = torch.zeros(2, dtype=torch.float32).pin_memory()
            s.graph, s.event, s.busy = None, torch.cuda.Event(), False
            self._ext_slots[key] = s
            return s
        # generic tensor: stage through one of our own pinned slots
        s = self.slots[self._nstep % len(self.slots)]
        if s.busy:
            while s.busy:
                self._retire_oldest()
        if data.device.type == "cpu":
            s.x_pin.copy_(data.view_as(s.x_pin))
            s.y_pin.copy_(target)
        return s

    def step(self, data: torch.Tensor, target: torch.Tensor) -> None:
        """One synchronous-SGD step on this rank's mini-batch (async; see ``sync_lag``)."""
        B = target.numel()
        if B != self.bsz or not self.use_graph or data.is_cuda:
            self._eager_step(data, target, B)
            return
        s = self._slot_for(data, target)
        if s.busy:
            while s.busy:
                self._retire_oldest()
        if s.graph is None:
            self.sync_lag(0)
            self._capture(s)
        if torch.cuda.current_stream(self.device) == self.stream:     # fast path: caller already runs on our stream
            s.graph.replay()
            s.event.record(self.stream)
        else:
            with torch.cuda.stream(self.stream):
                s.graph.replay()
                s.event.record(self.stream)
        s.busy = True
        self._order.append(s)
        self._nstep += 1
        if len(self._order) > len(self.slots) - 2:
            self._retire_oldest()

    def _eager_step(self, data, target, B):
        self.sync_lag(0)
        with torch.cuda.stream(self.stream):
            x = data.to(self.device, non_blocking=True).contiguous()
            y = target.to(self.device, non_blocking=True).contiguous()
            if x.dtype not in (torch.uint8, torch.float32):
                x = x.to(torch.float32)
            self._kernels(x, y, B, input_ready=False)   # x may come from a conversion kernel right before the step
        self.stream.synchronize()
        self._last_loss_cum = float(self.loss_acc[0].item())
        self._nstep += 1

    def active(self):
        """Context manager that makes the trainer's stream current (removes per-step stream switching)."""
        return torch.cuda.stream(self.stream)

    # ------------------------------------------------------------------ native hot loop
    def run_native(self, loader, max_steps: Optional[int] = None, new_epoch: bool = True):
        """Run (part of) an epoch with the C++ step executor (csrc/executor.cpp): no Python in the loop.

        ``loader`` is a :class:`data.NativeBatchLoader` with ``batch_size == bsz`` and a dtype matching
        ``raw_uint8``.  Returns ``(steps_done, epoch_finished)``.  A short tail batch is processed eagerly."""
        self.sync_lag(0)
        self.stream.synchronize()
        ex = self._executors.get(id(loader))
        if ex is None or ex[1] != self.training:
            if loader.batch_size != self.bsz:
                raise ValueError("loader batch size != trainer batch size")
            block = (int(loader._l.block_bytes()) + 255) // 256 * 256
            # every step: plain PDL stream launches (csrc/executor.cpp), one device block + loss snapshot per loader slot
            in_dev = torch.zeros(loader.num_buffers * block, dtype=torch.uint8, device=self.device)
            loss_hist = torch.zeros(2 * loader.num_buffers, dtype=torch.float32, device=self.device)
            ex = (self.C.StepExecutor(loader._l, self.params, self.momentum, self.grads, self._grad_ptrs, self._sig_ptrs,
                                      self.step_counter, self.done_counter, self.loss_acc, in_dev, self.raw_uint8,
                                      self.training, self.rank, self.world, self.seed, self.rank * self.bsz,
                                      self.grad_stride, self.lr, self.mu, self.p_drop, max(1, loader.num_buffers - 2),
                                      self.cluster, self.aux, self._inbox_ptrs, loss_hist, self.wire_bf16,
                                      *self._native_slots(), lr_schedule=self._sched),
                  self.training)
            self._executors[id(loader)] = ex
        if new_epoch:
            loader.begin_epoch()
        done, tail, finished = ex[0].run(-1 if max_steps is None else int(max_steps))
        self._nstep += done
        ex[0].drain()
        if done:
            self._last_loss_cum = ex[0].last_loss_cumulative()
        if tail is not None:                     # the eager step reads the loss itself: it must come AFTER the executor's value
            self._eager_step(tail[0], tail[1], tail[1].numel())
            loader._l.release()
            done += 1
            finished = True                      # a short batch is always the last one of the epoch
        return done, finished

    def pop_loss_sum(self) -> float:
        """Sum of per-batch mean losses since the previous call (one sync)."""
        self.sync_lag(0)
        self.stream.synchronize()
        cum = float(self.loss_acc[0].item())
        out = cum - self._loss_read
        self._loss_read = cum
        return out

    def last_loss_cumulative(self) -> float:
        """Cumulative loss as of the most recently *retired* step (read from the pinned D2H copy)."""
        return self._last_loss_cum

    # ------------------------------------------------------------------ learning rate
    def _relaunch(self):
        """Drop what baked the lr in: captured graphs and native executors are rebuilt on their next use."""
        self.sync_lag(0)
        self.stream.synchronize()
        for s in list(self.slots) + list(self._ext_slots.values()):
            s.graph = None
        self._executors = {}

    @property
    def lr(self) -> float:
        """Base learning rate.  Assigning it takes effect from the next step on every path (graphs are re-captured)."""
        return self._lr

    @lr.setter
    def lr(self, value: float) -> None:
        self._relaunch()
        self._lr = float(value)

    def set_lr_schedule(self, schedule: Optional[LRSchedule]) -> None:
        """Replace the lr schedule (``None``: constant ``lr``) from the next step on."""
        tup = schedule_tuple(schedule)
        self._relaunch()
        self._sched, self.lr_schedule = tup, schedule

    def lr_at(self, step: Optional[int] = None) -> float:
        """The lr the optimizer kernels apply when the step counter reads ``step`` (default: its current value)."""
        if step is None:
            self.sync_lag(0)
            self.stream.synchronize()
            step = int(self.step_counter.item())
        return self._lr if self.lr_schedule is None else self.lr_schedule.lr_at(self._lr, step)

    # ------------------------------------------------------------------ nn.Module-like surface
    def train(self, mode: bool = True):
        """``model.train()`` / ``model.eval()``: dropout on/off (captured graphs are dropped, the flag is baked in)."""
        if mode != self.training:
            self.sync_lag(0)
            self.training = mode
            for s in list(self.slots) + list(self._ext_slots.values()):
                s.graph = None          # dropout on/off is baked into the captured launch
        return self

    def eval(self):
        """``model.eval()``."""
        return self.train(False)

    def parameters(self):
        """Views of the flat fp32 parameter buffer, in the reference ``Net``'s order (train_dist.py:53-62)."""
        return list(unpack_params(self.params).values())

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        self.sync_lag(0)
        self.stream.synchronize()
        x = x.to(self.device)
        if x.dtype != torch.uint8:
            x = x.to(torch.float32)
        return convnet_forward(self.params, x)

    def evaluate(self, dataset=None) -> Dict:
        """Test loss and accuracy of the current parameters (``ops.convnet_eval.evaluate``; collective over the trainer's
        group).  Launched on the trainer's stream, so it follows every step issued so far (graph replays, eager steps;
        ``run_native`` returns drained), and it reads only the parameters: momentum, step counter, loss terms, exchange
        state, captured graphs and the train / eval mode are left as they are."""
        from .convnet_eval import Evaluator
        if self._evaluator is None:
            self._evaluator = Evaluator(self.device, self.group)
        return self._evaluator.run(self.params, dataset, stream=self.stream)

    def state_dict(self):
        """``{'model': ..., 'momentum': ..., 'steps': ...}`` with the reference's parameter names (CPU copies)."""
        self.sync_lag(0)
        self.stream.synchronize()
        p, m = unpack_params(self.params), unpack_params(self.momentum)
        return {"model": {k: v.detach().cpu().clone() for k, v in p.items()},
                "momentum": {k: v.detach().cpu().clone() for k, v in m.items()},
                "steps": int(self.step_counter.item()), "lr": self.lr, "mu": self.mu,
                "lr_schedule": None if self.lr_schedule is None else self.lr_schedule.to_dict()}

    def load_state_dict(self, sd):
        """Accepts a trainer checkpoint or a plain ``Net`` state_dict.  Collective when ``steps`` is present (the bucket
        parity and the exchange epochs derive from the step counter, see :meth:`_reset_exchange`).  The lr and the lr
        schedule stay the constructor's: ``steps`` is where a schedule continues from."""
        self.sync_lag(0)
        model = sd.get("model", sd)
        views = unpack_params(self.params)
        for k, v in model.items():
            views[k].copy_(v)
        if "momentum" in sd:
            mv = unpack_params(self.momentum)
            for k, v in sd["momentum"].items():
                mv[k].copy_(v)
        if "steps" in sd:
            self.step_counter.fill_(int(sd["steps"]))
            self._reset_exchange()               # bucket parity and push epochs derive from the step counter
        self._refresh_aux()
        torch.cuda.synchronize(self.device)

    def to_module(self) -> Net:
        """A torch ``Net`` holding copies of the current parameters."""
        net = Net(self.p_drop)
        net.load_state_dict(self.state_dict()["model"])
        return net
