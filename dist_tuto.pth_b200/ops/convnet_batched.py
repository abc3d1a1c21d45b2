"""Batched tensor-core training engine for the tutorial ConvNet (large per-GPU batches).

The per-sample engine (:mod:`.convnet_fused`) serves the reference's latency-bound configuration (global batch 128,
train_dist.py:85).  This engine is the throughput path -- BASELINE.md B1 "large-batch variant": the same network,
the same flat fp32 parameter / gradient-bucket layout and the same fused all-reduce + SGD kernel, but the batch flows
layer by layer through kernels in which the GEMM-shaped layers (conv2 forward / data gradient / weight gradient, fc1
forward and data gradient) run on the wgmma tensor cores with TMA-fed operands and register accumulators
(csrc/convnet_batched.cu has the kernel-by-kernel map; reference ops: train_dist.py:58-71,120-124).

Parity oracle: :mod:`.batched_reference` (plain PyTorch, same rounding points).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .. import comm
from ..models.convnet import Net
from . import _ext
from .optim import LRSchedule, check_max_grad_norm, check_sgd_options, schedule_tuple
from .convnet_fused import LAYOUT, NPAR, NPAR_ALLOC, pack_params, unpack_params  # noqa: F401

__all__ = ["BatchedBuffers", "batched_loss_and_grads", "batched_forward", "BatchedTrainer", "STAGES"]

# stage_mask bits of C.bt_step (tests run the pipeline prefix by prefix)
STAGES = {"conv1_fwd": 1, "conv2_fwd": 2, "head": 4, "fc1_dgrad": 8, "conv2_wgrad": 16, "conv2_dgrad": 32,
          "conv1_wgrad": 64, "fc_wgrad": 128, "all": 255}


class BatchedBuffers:
    """Activation / operand buffers of one batch size (bf16 unless noted); order = ``BtBuffers`` in csrc/bindings.cpp.

    ``P1`` relu(pool(conv1)) channel-last [B,12,12,16] (one 32-byte pixel = one TMA row): channels 11..15 are zero padding,
    channel 10 is a constant 1 so that the conv2 bias gradient is one row of the weight-gradient GEMM; ``DC`` conv2-output
    gradient [B,32,8,8] (channels 20..31 stay zero)."""

    def __init__(self, B: int, device):
        bf, u8, f32 = torch.bfloat16, torch.uint8, torch.float32
        z = lambda n, dt: torch.zeros(n, dtype=dt, device=device)   # noqa: E731
        self.B = int(B)
        self.P1, self.P2, self.H, self.DH, self.dP2 = z(B * 2304, bf), z(B * 320, bf), z(B * 64, bf), z(B * 64, bf), z(B * 320, bf)
        self.DC = z(B * 2048, bf)
        self.W2K, self.W2R, self.W3K, self.W3T = z(32 * 448, bf), z(400 * 64, bf), z(64 * 320, bf), z(320 * 64, bf)
        self.A1, self.A2 = z(B * 1440, u8), z(B * 320, u8)
        self.Hrelu, self.DLOG, self.G1, self.B3P = z(B * 64, f32), z(B * 16, f32), z(B * 1440, f32), z(64, f32)
        self.P1.view(B, 12, 12, 16)[..., 10].fill_(1.0)           # the constant-one input channel (bias gradient row)

    def as_list(self) -> List[torch.Tensor]:
        return [self.P1, self.P2, self.H, self.DH, self.dP2, self.DC, self.W2K, self.W2R, self.W3K, self.W3T,
                self.A1, self.A2, self.Hrelu, self.DLOG, self.G1, self.B3P]


def batched_loss_and_grads(params: torch.Tensor, x: torch.Tensor, target: torch.Tensor, training: bool = False,
                           seed: int = 0, step: Optional[torch.Tensor] = None, sample_base: int = 0, p_drop: float = 0.5,
                           bufs: Optional[BatchedBuffers] = None, stage_mask: int = 255, grads: Optional[torch.Tensor] = None):
    """Functional entry (tests / benches): ``(mean_nll, grads_flat, bufs)`` of one batch."""
    C = _ext.C()
    B = target.numel()
    bufs = bufs or BatchedBuffers(B, params.device)
    C.bt_pack_weights(params, bufs.as_list())
    if grads is None:
        grads = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=params.device)
    acc = torch.zeros(2, dtype=torch.float32, device=params.device)
    C.bt_step(params, grads, x.contiguous(), target.contiguous(), bufs.as_list(), acc, None, step, seed, sample_base,
              training, 1.0 / B, p_drop, stage_mask)
    return acc[0], grads, bufs


def batched_forward(params: torch.Tensor, x: torch.Tensor, bufs: Optional[BatchedBuffers] = None) -> torch.Tensor:
    """Eval-mode forward: log-probabilities ``[B,10]`` (``Net.eval()(x)`` semantics, bf16 tensor-core operands)."""
    C = _ext.C()
    B = x.shape[0]
    bufs = bufs or BatchedBuffers(B, params.device)
    C.bt_pack_weights(params, bufs.as_list())
    out = torch.empty(B, 10, dtype=torch.float32, device=params.device)
    dummy = torch.zeros(B, dtype=torch.int64, device=params.device)
    C.bt_step(params, None, x.contiguous(), dummy, bufs.as_list(), None, out, None, 0, 0, False, 1.0 / max(B, 1), 0.5, 7)
    return out


class BatchedTrainer:
    """Synchronous data-parallel SGD for the ConvNet with the batched tensor-core engine.

    One step = 8 forward/backward kernels + 2 wgmma GEMM launches + the fused [peer-memory all-reduce + 1/world +
    momentum SGD + re-zero] kernel of the per-sample engine (csrc/sgd.cu) + the bf16 weight re-pack, replayed as one CUDA
    graph.  Same constructor / ``step`` / ``state_dict`` surface as :class:`.convnet_fused.FusedTrainer`; state_dicts
    interchange (same flat layout and parameter names)."""

    def __init__(self, bsz: int, lr: float = 0.01, momentum: float = 0.5, seed: int = 1234, device=None,
                 p_drop: float = 0.5, group=None, raw_uint8: bool = False, use_graph: bool = True,
                 init_from: Optional[Net] = None, lr_schedule: Optional[LRSchedule] = None, weight_decay: float = 0.0,
                 nesterov: bool = False, max_grad_norm: Optional[float] = None):
        check_sgd_options(momentum, weight_decay, nesterov)
        max_grad_norm = check_max_grad_norm(max_grad_norm)
        self.C = _ext.C()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.bsz, self._lr, self.mu, self.seed, self.p_drop = int(bsz), float(lr), float(momentum), int(seed), p_drop
        self.weight_decay, self.nesterov = float(weight_decay), bool(nesterov)     # torch.optim.SGD's, fixed per trainer
        self._sched = schedule_tuple(lr_schedule)       # computed per update by the optimizer kernel (csrc/lr_schedule.h)
        self.lr_schedule = lr_schedule
        self.group = group
        self.world = comm.get_world_size(group)
        self.rank = comm.group_ranks(group).index(comm.get_rank()) if comm.is_initialized() else 0
        self.raw_uint8, self.training, self.use_graph = raw_uint8, True, use_graph
        if init_from is None:
            torch.manual_seed(seed)
            init_from = Net(p_drop)
        self.params = pack_params(init_from, self.device)
        if self.world > 1:
            dist.broadcast(self.params, src=comm.group_ranks(group)[0], group=comm._g(group))
        self.momentum = torch.zeros_like(self.params)
        self.symm, self.grad_handle = None, None
        if self.world > 1:
            from ..parallel import symm
            self.symm = symm.lookup_world(comm._g(group)) or symm.init_world(comm._g(group))
            if not isinstance(self.symm, symm.SymmWorld):     # parallel/hier.HierWorld: the job spans several machines
                raise RuntimeError("the fused gradient exchange runs inside ONE NVSwitch domain; on several machines use "
                                   "train(engine='torch') / DistributedDataParallel (two-level all-reduce, parallel/hier.py)")
            self.grad_handle = self.symm.alloc(NPAR_ALLOC, torch.float32)
            self.grads = self.grad_handle.local
            self.grads.zero_()
            self._grad_ptrs, self._sig_ptrs = self.grad_handle.ptrs, self.grad_handle.sig_ptrs
        else:
            self.grads = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=self.device)
            self._grad_ptrs, self._sig_ptrs = [self.grads.data_ptr()], [0]
        self.bufs = BatchedBuffers(self.bsz, self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.done_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        # max_grad_norm: clip_grad_norm_ of every update in allreduce_sgd's clip instance (see FusedTrainer)
        self.max_grad_norm = max_grad_norm
        self._clip_kw = {}
        if max_grad_norm is not None:
            self._grad_norm = torch.zeros(1, dtype=torch.float32, device=self.device)
            self._clip_kw = dict(max_grad_norm=max_grad_norm, grad_norm_out=self._grad_norm,
                                 clip_workspace=torch.zeros(self.C.clip_workspace_numel(NPAR_ALLOC), dtype=torch.float32,
                                                            device=self.device))
        self.loss_acc = torch.zeros(2, dtype=torch.float32, device=self.device)
        xdt = torch.uint8 if raw_uint8 else torch.float32
        self.x_dev = torch.zeros(self.bsz, 1, 28, 28, dtype=xdt, device=self.device)
        self.y_dev = torch.zeros(self.bsz, dtype=torch.int64, device=self.device)
        self.stream = torch.cuda.Stream(self.device)
        self._graph = None
        self._loss_read = 0.0
        self.gpu_launches_per_step = 12       # 8 engine kernels + 2 wgmma GEMMs + allreduce_sgd + pack_weights
        self._evaluator = None                # ops/convnet_eval.Evaluator, made on the first evaluate()
        with torch.cuda.stream(self.stream):
            self.C.bt_pack_weights(self.params, self.bufs.as_list())
        self.stream.synchronize()
        if self.world > 1:
            comm.barrier(self.group)

    # ------------------------------------------------------------------ kernels of one step (on the current stream)
    def _kernels(self, x, y, B):
        self.C.bt_step(self.params, self.grads, x, y, self.bufs.as_list(), self.loss_acc, None, self.step_counter, self.seed,
                       self.rank * self.bsz, self.training, 1.0 / B, self.p_drop, 255)
        # single gradient bucket: the barrier flavour of the fused exchange (flag barrier, peer loads, second barrier,
        # re-zero) -- at >= 100 us per step the exchange latency is irrelevant, the fusion (no separate /world, SGD,
        # zero_grad passes) is what is kept
        self.C.allreduce_sgd(self._grad_ptrs, self._sig_ptrs, self.params, self.momentum, self.step_counter,
                             self.lr, self.mu, 1.0 / self.world, self.rank, self.world, True, 0, self.done_counter, None, [],
                             lr_schedule=self._sched, weight_decay=self.weight_decay, nesterov=self.nesterov, **self._clip_kw)
        self.C.bt_pack_weights(self.params, self.bufs.as_list())

    def step_device(self, x: torch.Tensor, y: torch.Tensor) -> None:
        """One step on device-resident tensors (eager launches on the trainer's stream)."""
        with torch.cuda.stream(self.stream):
            self._kernels(x.contiguous(), y.contiguous(), y.numel())

    def step(self, data: torch.Tensor, target: torch.Tensor) -> None:
        """One synchronous-SGD step on this rank's mini-batch: H2D into the static input block, then the step graph."""
        B = target.numel()
        with torch.cuda.stream(self.stream):
            if B != self.bsz or not self.use_graph:
                x = data.to(self.device, non_blocking=True).contiguous()
                yy = target.to(self.device, non_blocking=True).contiguous()
                if x.dtype not in (torch.uint8, torch.float32):
                    x = x.to(torch.float32)
                self._kernels(x, yy, B)
                return
            self.x_dev.copy_(data.view_as(self.x_dev), non_blocking=True)
            self.y_dev.copy_(target, non_blocking=True)
            if self._graph is None:
                self._kernels(self.x_dev, self.y_dev, self.bsz)          # eager once: func attributes, lazy module load
                self.stream.synchronize()
                # the eager step advanced the model: capture replays exactly the same launches from here on
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    self._kernels(self.x_dev, self.y_dev, self.bsz)
                self._graph = g
                return
            self._graph.replay()

    def pop_loss_sum(self) -> float:
        """Sum of per-batch mean losses since the previous call (one sync)."""
        self.stream.synchronize()
        cum = float(self.loss_acc[0].item())
        out = cum - self._loss_read
        self._loss_read = cum
        return out

    # ------------------------------------------------------------------ learning rate
    @property
    def lr(self) -> float:
        """Base learning rate.  Assigning it takes effect from the next step (the step graph is re-captured)."""
        return self._lr

    @lr.setter
    def lr(self, value: float) -> None:
        self.stream.synchronize()
        self._lr, self._graph = float(value), None

    def set_lr_schedule(self, schedule: Optional[LRSchedule]) -> None:
        """Replace the lr schedule (``None``: constant ``lr``) from the next step on."""
        tup = schedule_tuple(schedule)
        self.stream.synchronize()
        self._sched, self.lr_schedule, self._graph = tup, schedule, None

    def lr_at(self, step: Optional[int] = None) -> float:
        """The lr the optimizer kernel applies when the step counter reads ``step`` (default: its current value)."""
        if step is None:
            self.stream.synchronize()
            step = int(self.step_counter.item())
        return self._lr if self.lr_schedule is None else self.lr_schedule.lr_at(self._lr, step)

    def grad_norm(self) -> Optional[float]:
        """The pre-clip total L2 norm of the averaged gradient of the last update; ``None`` without ``max_grad_norm``.
        Synchronises like :meth:`lr_at`."""
        if self.max_grad_norm is None:
            return None
        self.stream.synchronize()
        return float(self._grad_norm.item())

    # ------------------------------------------------------------------ nn.Module-like surface
    def train(self, mode: bool = True):
        if mode != self.training:
            self.stream.synchronize()
            self.training, self._graph = mode, None
        return self

    def eval(self):
        return self.train(False)

    def parameters(self):
        return list(unpack_params(self.params).values())

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        self.stream.synchronize()
        x = x.to(self.device)
        if x.dtype != torch.uint8:
            x = x.to(torch.float32)
        return batched_forward(self.params, x)

    def evaluate(self, dataset=None) -> Dict:
        """Test loss and accuracy of the current parameters on the fp32 eval kernel (``ops.convnet_eval.evaluate``;
        collective over the trainer's group), ordered after every step issued on the trainer's stream.  Reads only the
        parameters; the bf16 forward of ``__call__`` is not used, since it flips near-tie argmaxes."""
        from .convnet_eval import Evaluator
        if self._evaluator is None:
            self._evaluator = Evaluator(self.device, self.group)
        return self._evaluator.run(self.params, dataset, stream=self.stream)

    def state_dict(self) -> Dict:
        self.stream.synchronize()
        p, m = unpack_params(self.params), unpack_params(self.momentum)
        return {"model": {k: v.detach().cpu().clone() for k, v in p.items()},
                "momentum": {k: v.detach().cpu().clone() for k, v in m.items()},
                "steps": int(self.step_counter.item()), "lr": self.lr, "mu": self.mu,
                "lr_schedule": None if self.lr_schedule is None else self.lr_schedule.to_dict(),
                "weight_decay": self.weight_decay, "nesterov": self.nesterov, "max_grad_norm": self.max_grad_norm}

    def load_state_dict(self, sd) -> None:
        """Parameters, momentum and step counter; the lr, its schedule, the weight decay, Nesterov and max_grad_norm stay
        the constructor's."""
        self.stream.synchronize()
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
        self.C.bt_pack_weights(self.params, self.bufs.as_list())
        torch.cuda.synchronize(self.device)
