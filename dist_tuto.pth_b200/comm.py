"""Communication primitives (layer L2 of the tutorial).

Parity map (reference = /root/reference):
  * blocking ``send``/``recv``                      tuto.md:77-97
  * non-blocking ``isend``/``irecv`` + ``wait()``   tuto.md:97-120
  * ``all_reduce, reduce, broadcast, scatter, gather, all_gather``  tuto.md:176-202
  * ``reduce_op.{SUM,PRODUCT,MAX,MIN}``             tuto.md:188-193
  * ``new_group(ranks)``                            tuto.md:176,182
  * ``get_rank()/get_world_size()``                 train_dist.py:84,88,96

Design (GPU-first, not a port):
  * plumbing (rendezvous, p2p, the non-hot collectives) rides on
    ``torch.distributed`` -- NCCL for CUDA tensors (NVLink 5 / NVSwitch),
    gloo for CPU tensors;
  * when a symmetric world has been set up for the group (``backend="b200"``),
    blocking ``all_reduce`` and ``reduce`` (SUM, PRODUCT, MAX, MIN on CUDA
    fp32 / bf16) and ``broadcast`` and ``all_gather`` (CUDA, any dtype, copied
    bit for bit) run on our own fused peer-memory kernels (``parallel.symm``);
    that path never calls NCCL.  ``async_op=True``, CPU tensors, other dtypes
    and ops, ``scatter`` and ``gather`` go to NCCL / gloo, and so does every op
    but SUM on a world that serves only the sum (no ``supports_op``).
  * ``group=0`` (the 2017 spelling of "world", train_dist.py:99, ptp.py:26)
    is accepted and mapped to the default group (fixes defect D2).
"""
from __future__ import annotations

import warnings
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

__all__ = [
    "reduce_op", "ReduceOp", "send", "recv", "isend", "irecv", "broadcast", "reduce",
    "all_reduce", "scatter", "gather", "gather_to_root", "all_gather", "barrier", "new_group",
    "get_rank", "get_world_size", "is_initialized", "Request", "group_ranks",
]


class reduce_op:  # noqa: N801 - tutorial spelling (tuto.md:188-193)
    """Element-wise commutative reduction operators (``dist.reduce_op.*``)."""
    SUM = dist.ReduceOp.SUM
    PRODUCT = dist.ReduceOp.PRODUCT
    MAX = dist.ReduceOp.MAX
    MIN = dist.ReduceOp.MIN


ReduceOp = reduce_op


class _World:
    """Marker for the default group (``dist.group.WORLD`` analogue)."""


class group:  # noqa: N801 - mirrors ``dist.group.WORLD`` (ptp.py:14)
    """``dist.group.WORLD`` of the 2017 API (ptp.py:14): the default group, spelled ``None`` here."""
    WORLD = None


def _g(grp):
    """Normalise a user supplied group: ``None``/``0``/``group.WORLD`` -> world."""
    if grp is None or (isinstance(grp, int) and grp == 0):
        return None
    return grp


def is_initialized() -> bool:
    """True inside ``init_processes`` / after ``init_process_group`` (single-process use is allowed: rank 0 of 1)."""
    return dist.is_available() and dist.is_initialized()


def get_rank(group=None) -> int:
    """``dist.get_rank()`` (tuto.md:46, ptp.py:22); 0 when no process group exists."""
    return dist.get_rank(_g(group)) if is_initialized() else 0


def get_world_size(group=None) -> int:
    """``dist.get_world_size()`` (train_dist.py:84,95; ptp.py:23); 1 when no process group exists."""
    return dist.get_world_size(_g(group)) if is_initialized() else 1


def group_ranks(group=None) -> List[int]:
    """Global ranks of the members of ``group`` (world if None), in group order."""
    g = _g(group)
    if not is_initialized():
        return [0]
    if g is None:
        return list(range(dist.get_world_size()))
    return list(dist.get_process_group_ranks(g))


def new_group(ranks: Optional[Sequence[int]] = None, **kw):
    """Create a sub-group (``dist.new_group([0, 1])``, tuto.md:182).

    Must be called by *every* rank of the world, like the original."""
    return dist.new_group(ranks=None if ranks is None else list(ranks), **kw)


class Request:
    """Handle returned by ``isend``/``irecv`` (tuto.md:97-120).

    The tensor must not be read (irecv) or written (isend) before ``wait()``
    returns.  For CUDA tensors ``wait()`` orders the *current stream* after the
    transfer (NCCL semantics); ``wait(sync=True)`` additionally blocks the host.
    """

    def __init__(self, work, tensor: torch.Tensor):
        self._work = work
        self._tensor = tensor

    def wait(self, sync: bool = False) -> bool:
        """``req.wait()`` of tuto.md:108-116: after it the buffer may be reused (send) / read (recv).  On CUDA the
        transfer is ordered on the current stream; ``sync=True`` additionally blocks the host until it has finished."""
        if self._work is not None:
            self._work.wait()
            self._work = None
        if sync and self._tensor.is_cuda:
            torch.cuda.current_stream(self._tensor.device).synchronize()
        return True

    def is_completed(self) -> bool:
        """Non-blocking completion test."""
        return self._work is None or self._work.is_completed()


def _check(t: torch.Tensor):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"expected a torch.Tensor, got {type(t).__name__}")
    if not t.is_contiguous():
        raise ValueError("communication primitives need contiguous tensors")


# ----------------------------------------------------------------- p2p -------
def send(tensor: torch.Tensor, dst: int, group=None, tag: int = 0) -> None:
    """Blocking send (tuto.md:87).  Returns when the buffer may be reused."""
    _check(tensor)
    dist.send(tensor, dst=dst, group=_g(group), tag=tag)


def recv(tensor: torch.Tensor, src: Optional[int] = None, group=None, tag: int = 0) -> int:
    """Blocking receive into a pre-allocated tensor (tuto.md:90)."""
    _check(tensor)
    return dist.recv(tensor, src=src, group=_g(group), tag=tag)


def isend(tensor: torch.Tensor, dst: int, group=None, tag: int = 0) -> Request:
    """Non-blocking send (tuto.md:108)."""
    _check(tensor)
    return Request(dist.isend(tensor, dst=dst, group=_g(group), tag=tag), tensor)


def irecv(tensor: torch.Tensor, src: Optional[int] = None, group=None, tag: int = 0) -> Request:
    """Non-blocking receive (tuto.md:112)."""
    _check(tensor)
    return Request(dist.irecv(tensor, src=src, group=_g(group), tag=tag), tensor)


# --------------------------------------------------------- collectives -------
def _symm_world_for(tensor: torch.Tensor, group):
    """Return the fused peer-memory world serving ``group`` or None."""
    if not tensor.is_cuda:
        return None
    try:
        from .parallel import symm
    except Exception:  # extension not importable on a CPU-only box
        return None
    return symm.lookup_world(_g(group))


def _reduces(w, tensor: torch.Tensor, op) -> bool:
    """Does world ``w`` run this reduction natively?  SUM on any world that takes the tensor; the other ops only on a
    world that says it supports them (a hierarchical world reduces SUM only)."""
    if w is None or not w.supports(tensor):
        return False
    if op == reduce_op.SUM:
        return True
    return hasattr(w, "supports_op") and w.supports_op(op)


def all_reduce(tensor: torch.Tensor, op=reduce_op.SUM, group=None, async_op: bool = False):
    """In-place all-reduce; result on every rank (tuto.md:176-186,199).

    CUDA fp32 / bf16 tensors go through the fused sm_90a peer-memory kernels
    (variant picked by size) for SUM, PRODUCT, MAX and MIN when a symmetric
    world exists for the group; everything else goes to NCCL / gloo."""
    _check(tensor)
    if not async_op:
        w = _symm_world_for(tensor, group)
        if _reduces(w, tensor, op):
            if op == reduce_op.SUM:
                w.all_reduce_(tensor, scale=1.0)
            else:
                w.all_reduce_(tensor, op=op)
            return None
    return dist.all_reduce(tensor, op=op, group=_g(group), async_op=async_op)


def reduce(tensor: torch.Tensor, dst: int, op=reduce_op.SUM, group=None):
    """Reduce to ``dst`` only (tuto.md:198); ``dst`` is a global rank.  Other ranks' tensors are left as they were.
    Routed like ``all_reduce``."""
    _check(tensor)
    w = _symm_world_for(tensor, group)
    if _reduces(w, tensor, op) and hasattr(w, "reduce_"):
        w.reduce_(tensor, dst, op)
        return None
    return dist.reduce(tensor, dst=dst, op=op, group=_g(group))


def broadcast(tensor: torch.Tensor, src: int, group=None):
    """Copy ``tensor`` from global rank ``src`` to all ranks (tuto.md:197).  On a symmetric world any CUDA dtype is
    copied bit for bit by the peer-memory kernels."""
    _check(tensor)
    w = _symm_world_for(tensor, group)
    if w is not None and hasattr(w, "broadcast_") and w.supports_raw(tensor):
        w.broadcast_(tensor, src)
        return None
    return dist.broadcast(tensor, src=src, group=_g(group))


def scatter(tensor: torch.Tensor, src: int = 0, scatter_list: Optional[List[torch.Tensor]] = None,
            group=None):
    """i-th element of ``scatter_list`` on ``src`` goes to rank i (tuto.md:200).

    Unlike modern torch, a ``scatter_list`` passed on non-source ranks is
    ignored (the tutorial era accepted it)."""
    _check(tensor)
    g = _g(group)
    if dist.get_rank() != src:
        scatter_list = None
    return dist.scatter(tensor, scatter_list=scatter_list, src=src, group=g)


def gather(tensor: torch.Tensor, dst: int = 0, gather_list: Optional[List[torch.Tensor]] = None,
           group=None):
    """All ranks' tensors land in ``gather_list`` on ``dst`` (tuto.md:201, ptp.py:26).

    The reference passes ``gather_list`` on every rank (ptp.py:25-26); modern
    torch rejects that, so it is dropped on non-destination ranks here."""
    _check(tensor)
    g = _g(group)
    if dist.get_rank() != dst:
        gather_list = None
    elif gather_list is not None and len({id(t) for t in gather_list}) != len(gather_list):
        raise ValueError("gather_list must hold distinct tensors ([zeros(1)] * n aliases one buffer)")
    return dist.gather(tensor, gather_list=gather_list, dst=dst, group=g)


def gather_to_root(tensor: torch.Tensor, rank: int, tensor_list: Optional[List[torch.Tensor]] = None, root: int = 0,
                   group=None):
    """The ``gather(tensor, rank, tensor_list=None, root=0, group=None)`` helper of ptp.py:9-19, same argument order.

    "Sends tensor to root process, which store it in tensor_list."  The 2017 internals it called
    (``dist.gather_recv`` / ``dist.gather_send``, ptp.py:17,19) no longer exist; both map onto one ``gather`` collective
    here.  The root must pass ``tensor_list`` (the reference asserts the same, ptp.py:16)."""
    if rank == root:
        assert tensor_list is not None, "the root rank must provide tensor_list"
        return gather(tensor, dst=root, gather_list=tensor_list, group=group)
    return gather(tensor, dst=root, gather_list=None, group=group)


def all_gather(tensor_list: List[torch.Tensor], tensor: torch.Tensor, group=None):
    """Every rank receives every rank's tensor (tuto.md:202).  On a symmetric world, CUDA tensors of any dtype are gathered
    bit for bit by the peer-memory kernels."""
    _check(tensor)
    w = _symm_world_for(tensor, group)
    if w is not None and hasattr(w, "all_gather_") and w.supports_raw(tensor) and \
            all(isinstance(t, torch.Tensor) and w.supports_raw(t) and t.dtype == tensor.dtype and t.numel() == tensor.numel()
                for t in tensor_list) and len(tensor_list) == w.world:
        w.all_gather_(tensor_list, tensor)
        return None
    return dist.all_gather(tensor_list, tensor, group=_g(group))


def barrier(group=None):
    """Block until every rank of ``group`` got here (absent from the reference, which never synchronises explicitly --
    SURVEY §5; used by tests, benches and the symmetric-memory setup).  No-op without a process group."""
    g = _g(group)
    if not is_initialized():
        return
    if dist.get_backend(g) == "nccl" and torch.cuda.is_available():
        return dist.barrier(group=g, device_ids=[torch.cuda.current_device()])
    return dist.barrier(group=g)


def _warn_once(msg: str, _seen=set()):
    if msg not in _seen:
        _seen.add(msg)
        warnings.warn(msg, stacklevel=3)
