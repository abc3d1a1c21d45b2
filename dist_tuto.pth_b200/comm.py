"""Communication primitives (layer L2 of the tutorial).

Parity map (reference = /root/reference):
  * blocking ``send``/``recv``                      tuto.md:77-97
  * non-blocking ``isend``/``irecv`` + ``wait()``   tuto.md:97-120
  * ``all_reduce, reduce, broadcast, scatter, gather, all_gather``  tuto.md:176-202
  * ``reduce_op.{SUM,PRODUCT,MAX,MIN}``             tuto.md:188-193
  * ``new_group(ranks)``                            tuto.md:176,182
  * ``get_rank()/get_world_size()``                 train_dist.py:84,88,96

Design (GPU-first, not a port):
  * plumbing (rendezvous, anything without a symmetric world) rides on
    ``torch.distributed`` -- NCCL for CUDA tensors (NVLink 5 / NVSwitch),
    gloo for CPU tensors;
  * when a symmetric world has been set up for the group (``backend="b200"``),
    blocking ``all_reduce`` and ``reduce`` (SUM, PRODUCT, MAX, MIN on CUDA
    fp32, bf16, fp16, fp64, int8, uint8, int32, int64 and bool -- torch's NCCL
    dtypes; integers wrap and a bool SUM is a MAX, as with NCCL) and
    ``broadcast``, ``all_gather``, ``scatter`` and ``gather`` (CUDA, any
    dtype, copied bit for bit) run on our own fused peer-memory kernels
    (``parallel.symm``); that path never calls NCCL.
    ``async_op=True``, CPU tensors, AVG and other dtypes (int16, the wider
    unsigned types, complex, fp8) go to NCCL / gloo, and so does every op but
    SUM on a world that serves only the sum (no ``supports_op``), every dtype
    but fp32 / bf16 on a world without ``supports_reduction``, and
    ``scatter`` / ``gather`` on a world without ``scatter_`` / ``gather_``
    (the two-level world of several machines has none of the three).
  * beyond the tutorial, torch's ``reduce_scatter_tensor`` and
    ``reduce_scatter`` (the ops and dtypes of ``all_reduce``) and the
    equal-segment ``all_to_all_single`` (any dtype) run on peer-memory
    kernels of their own on such a world, and ``all_gather_into_tensor`` on
    the all-gather's; ``all_to_all_single`` with split sizes and the list form
    ``all_to_all`` (any sizes, any dtype) run on a variable-segment kernel;
    ``async_op=True``, AVG, other dtypes, CPU tensors and the two-level world
    go to torch.distributed.
  * on such a world ``send``, ``recv``, ``isend`` and ``irecv`` of a CUDA
    tensor (any dtype, bit for bit) run on our own point-to-point kernels
    (``csrc/p2p.cu``) when the peer is given: messages between a pair are
    matched in issue order and ``tag`` is ignored, as NCCL ignores it.
    ``recv(src=None)``, CPU tensors and the two-level world (no ``send_``)
    stay on torch.  ``batch_isend_irecv`` gives each op the route ``isend`` /
    ``irecv`` would, and runs all its peer-memory ops in one launch
    (``SymmWorld.batch_p2p_``), the rest in one ``dist.batch_isend_irecv``.
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
    "get_rank", "get_world_size", "is_initialized", "Request", "group_ranks", "reduce_scatter", "reduce_scatter_tensor",
    "all_to_all_single", "all_gather_into_tensor", "all_to_all", "P2POp", "batch_isend_irecv",
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
# On a symmetric world (``backend="b200"``) a CUDA tensor with a given peer goes through the peer-memory mailbox of
# ``SymmWorld.send_`` / ``recv_`` / ``isend_`` / ``irecv_``: both sides must use this module with the same byte count, and
# messages between one pair are matched in the order they are issued (``tag`` is ignored there, as NCCL ignores it).
def _p2p_world(tensor: torch.Tensor, group, peer: Optional[int]):
    """The symmetric world whose point-to-point kernels take this call, or None (torch.distributed)."""
    if peer is None:
        return None
    w = _symm_world_for(tensor, group)
    if w is None or not hasattr(w, "send_") or not w.supports_raw(tensor):
        return None
    return w


def send(tensor: torch.Tensor, dst: int, group=None, tag: int = 0) -> None:
    """Blocking send (tuto.md:87).  Returns when the buffer may be reused: on CUDA, as with NCCL, once the current stream is
    ordered after the transfer (the host is not synchronised).  ``dst`` is a global rank."""
    _check(tensor)
    w = _p2p_world(tensor, group, dst)
    if w is not None:
        w.send_(tensor, dst)
        return None
    dist.send(tensor, dst=dst, group=_g(group), tag=tag)


def recv(tensor: torch.Tensor, src: Optional[int] = None, group=None, tag: int = 0) -> int:
    """Blocking receive into a pre-allocated tensor (tuto.md:90); returns the sender's rank.  ``src=None`` (any source)
    always goes to torch.distributed."""
    _check(tensor)
    w = _p2p_world(tensor, group, src)
    if w is not None:
        w.recv_(tensor, src)
        return src
    return dist.recv(tensor, src=src, group=_g(group), tag=tag)


def isend(tensor: torch.Tensor, dst: int, group=None, tag: int = 0) -> Request:
    """Non-blocking send (tuto.md:108)."""
    _check(tensor)
    w = _p2p_world(tensor, group, dst)
    if w is not None:
        return Request(w.isend_(tensor, dst), tensor)
    return Request(dist.isend(tensor, dst=dst, group=_g(group), tag=tag), tensor)


def irecv(tensor: torch.Tensor, src: Optional[int] = None, group=None, tag: int = 0) -> Request:
    """Non-blocking receive (tuto.md:112)."""
    _check(tensor)
    w = _p2p_world(tensor, group, src)
    if w is not None:
        return Request(w.irecv_(tensor, src), tensor)
    return Request(dist.irecv(tensor, src=src, group=_g(group), tag=tag), tensor)


class P2POp:
    """One send or receive of :func:`batch_isend_irecv` (torch's ``P2POp``): ``op`` is ``isend`` or ``irecv`` of this
    module or of torch.distributed, ``peer`` a global rank."""

    def __init__(self, op, tensor: torch.Tensor, peer: int, group=None, tag: int = 0):
        if op not in (isend, irecv, dist.isend, dist.irecv):
            raise ValueError("P2POp takes isend or irecv (of this module or of torch.distributed) as its op")
        self.op, self.tensor, self.peer, self.group, self.tag = op, tensor, peer, group, tag


def _p2p_op(op):
    """(send, tensor, peer, group, tag) of a ``P2POp`` of this module or of torch.distributed; the group is None for the
    default group however it was spelled (torch's P2POp stores the default process group itself)."""
    if isinstance(op, (P2POp, dist.P2POp)):
        group = _g(op.group)
        if group is not None and is_initialized() and group is dist.group.WORLD:
            group = None
        return op.op in (isend, dist.isend), op.tensor, op.peer, group, op.tag
    raise ValueError("batch_isend_irecv takes a list of P2POp (of this module or of torch.distributed), got an element of "
                     f"type {type(op).__name__}")


def batch_isend_irecv(p2p_op_list: List[P2POp]) -> List[Request]:
    """Issue a list of sends and receives at once (torch's ``batch_isend_irecv``); one :class:`Request` per op, in list
    order.  Exchanges with several peers (rings, halo exchanges, pipeline stages) may list their sends before their
    receives: all of a batch's transfers progress together.

    Each op takes the route :func:`isend` / :func:`irecv` would give its tensor and peer, so the two sides of a pair agree
    whether each uses batches or single calls.  On a symmetric world (``backend="b200"``) all the ops that take the
    peer-memory kernels go out in one launch (``SymmWorld.batch_p2p_``; their Requests share its completion, as NCCL's
    coalesced works do, and ``tag`` is ignored); the rest go to one ``dist.batch_isend_irecv``.  Both sides of a pair pass
    the same byte count, as with :func:`isend`.  Raises ValueError before anything is issued for anything but a non-empty
    list of P2POp, ops of different groups, a non-contiguous tensor, or an op with this rank as its peer on the peer-memory
    path."""
    if not isinstance(p2p_op_list, list) or not p2p_op_list:
        raise ValueError("batch_isend_irecv takes a non-empty list of P2POp")
    ops = [_p2p_op(op) for op in p2p_op_list]
    if any(g != ops[0][3] for _, _, _, g, _ in ops):
        raise ValueError("All ops need to use the same group.")
    for _, t, _, _, _ in ops:
        _check(t)
    mine, theirs = [], []                                   # (position, op) on the peer-memory kernels / on torch
    world = None
    for i, (send, t, peer, group, tag) in enumerate(ops):
        w = _p2p_world(t, group, peer)
        if w is None:
            theirs.append(i)
            continue
        if peer == get_rank():
            raise ValueError(f"batch_isend_irecv: rank {peer} cannot {'send' if send else 'recv'} to itself")
        world = w
        mine.append(i)
    reqs: List[Optional[Request]] = [None] * len(ops)
    if mine:
        works = world.batch_p2p_([(ops[i][0], ops[i][1], ops[i][2]) for i in mine])
        for i, work in zip(mine, works):
            reqs[i] = Request(work, ops[i][1])
    if theirs:
        torch_ops = []
        for i in theirs:
            op = p2p_op_list[i]
            if not isinstance(op, dist.P2POp):
                send, t, peer, group, tag = ops[i]
                op = dist.P2POp(dist.isend if send else dist.irecv, t, peer, group=group, tag=tag)
            torch_ops.append(op)
        works = dist.batch_isend_irecv(torch_ops)
        for k, i in enumerate(theirs):                       # NCCL coalesces the batch into one work
            reqs[i] = Request(works[k] if len(works) == len(theirs) else (works[-1] if works else None), ops[i][1])
    return reqs


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
    world that says it supports them (a hierarchical world reduces SUM only).  A world with ``supports_reduction`` takes
    the dtypes beyond fp32 / bf16 too; one without it (the hierarchical world) only what ``supports`` takes."""
    if w is None:
        return False
    if not (w.supports_reduction if hasattr(w, "supports_reduction") else w.supports)(tensor):
        return False
    if op == reduce_op.SUM:
        return True
    return hasattr(w, "supports_op") and w.supports_op(op)


def all_reduce(tensor: torch.Tensor, op=reduce_op.SUM, group=None, async_op: bool = False):
    """In-place all-reduce; result on every rank (tuto.md:176-186,199).

    CUDA tensors go through the fused sm_90a peer-memory kernels (variant
    picked by size) for SUM, PRODUCT, MAX and MIN when a symmetric world
    exists for the group: fp32 / bf16 (fp32 accumulator), fp16 (fp32
    accumulator, rounded once), fp64, int8, uint8, int32 and int64 (SUM and
    PRODUCT wrap, as NCCL's do) and bool (SUM is MAX, as torch maps it for
    NCCL).  Everything else (AVG, other dtypes, CPU tensors, ``async_op``)
    goes to NCCL / gloo."""
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
    Routed like ``all_reduce``, with the same ops and dtypes."""
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
    ignored (the tutorial era accepted it).

    On a symmetric world a CUDA ``tensor`` of any dtype is scattered bit for bit by the peer-memory kernels.  Whether the
    call takes that path depends on ``tensor`` and the group alone, never on ``scatter_list``, which only ``src`` holds:
    every rank must enter the same kernel.  A ``scatter_list`` of the wrong length, dtype or size raises on ``src``, as
    torch does; its peers are then left waiting inside the kernel until its spin limit reports them."""
    _check(tensor)
    g = _g(group)
    if dist.get_rank() != src:
        scatter_list = None
    w = _symm_world_for(tensor, group)
    if w is not None and hasattr(w, "scatter_") and w.supports_raw(tensor):
        w.scatter_(tensor, scatter_list, src)
        return None
    return dist.scatter(tensor, scatter_list=scatter_list, src=src, group=g)


def gather(tensor: torch.Tensor, dst: int = 0, gather_list: Optional[List[torch.Tensor]] = None,
           group=None):
    """All ranks' tensors land in ``gather_list`` on ``dst`` (tuto.md:201, ptp.py:26).

    The reference passes ``gather_list`` on every rank (ptp.py:25-26); modern
    torch rejects that, so it is dropped on non-destination ranks here.

    On a symmetric world a CUDA ``tensor`` of any dtype is gathered bit for bit by the peer-memory kernels, routed by
    ``tensor`` and the group alone as in ``scatter``; a ``gather_list`` of the wrong length, dtype or size raises on
    ``dst``, and its peers are then left waiting inside the kernel until its spin limit reports them."""
    _check(tensor)
    g = _g(group)
    if dist.get_rank() != dst:
        gather_list = None
    elif gather_list is not None and len({id(t) for t in gather_list}) != len(gather_list):
        raise ValueError("gather_list must hold distinct tensors ([zeros(1)] * n aliases one buffer)")
    w = _symm_world_for(tensor, group)
    if w is not None and hasattr(w, "gather_") and w.supports_raw(tensor):
        w.gather_(tensor, gather_list, dst)
        return None
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


def _reduce_scatter_world(output: torch.Tensor, op, group, async_op: bool):
    """The symmetric world whose reduce-scatter kernels take this call, or None (torch.distributed).  The route depends on
    ``output``, ``op``, the group and ``async_op`` alone -- the same on every rank of a correct call -- never on the input,
    whose faults raise inside ``reduce_scatter_`` on the rank that has them."""
    if async_op:
        return None
    w = _symm_world_for(output, group)
    if w is None or not hasattr(w, "reduce_scatter_") or not _reduces(w, output, op):
        return None
    return w


def reduce_scatter_tensor(output: torch.Tensor, input: torch.Tensor, op=reduce_op.SUM, group=None,  # noqa: A002
                          async_op: bool = False):
    """``input`` holds world equal segments of ``output``'s size; rank r's ``output`` receives segment r of their reduction
    over the ranks (torch's ``reduce_scatter_tensor``).

    On a symmetric world (``backend="b200"``) a CUDA ``output`` takes the peer-memory kernels for the ops and dtypes of
    ``all_reduce`` (a bool SUM is a MAX), bit for bit slice r of what ``all_reduce`` leaves; AVG, other dtypes, CPU tensors
    and ``async_op=True`` go to torch.distributed."""
    _check(output)
    _check(input)
    w = _reduce_scatter_world(output, op, group, async_op)
    if w is not None:
        w.reduce_scatter_(output, input, op)
        return None
    return dist.reduce_scatter_tensor(output, input, op=op, group=_g(group), async_op=async_op)


def reduce_scatter(output: torch.Tensor, input_list: List[torch.Tensor], op=reduce_op.SUM, group=None,
                   async_op: bool = False):
    """``input_list[p]`` of every rank is reduced into rank p's ``output`` (torch's ``reduce_scatter``).  Routed like
    :func:`reduce_scatter_tensor`, by ``output`` alone: an ``input_list`` of the wrong length, dtype or size raises on the rank
    that passed it, before any launch, and its peers are then left waiting inside the kernel until its spin limit reports
    them.  A list of consecutive views of one 16-byte aligned block is read in place; any other list is copied into the
    staging buffer first."""
    _check(output)
    w = _reduce_scatter_world(output, op, group, async_op)
    if w is not None:
        w.reduce_scatter_(output, list(input_list), op)
        return None
    return dist.reduce_scatter(output, list(input_list), op=op, group=_g(group), async_op=async_op)


def all_to_all_single(output: torch.Tensor, input: torch.Tensor, output_split_sizes=None,  # noqa: A002
                      input_split_sizes=None, group=None, async_op: bool = False):
    """Segment p of rank r's ``output`` receives segment r of rank p's ``input`` (torch's ``all_to_all_single``); the split
    lists cut dim 0 into the ranks' segments (``None``: equal segments).

    On a symmetric world the equal-segment form (both split lists ``None``) of a CUDA tensor of any dtype is copied bit for
    bit by the peer-memory kernels.  Given either split list, a blocking call of two CUDA tensors runs on the variable-segment
    kernel (``SymmWorld.all_to_all_v_``), bit for bit, whatever the splits.  The form of the call picks the kernel, so:

    * every rank must use the same form: a rank that passes split sizes while a peer passes none is a caller error (it waits
      inside the kernel until its spin limit reports it), although torch.distributed would accept the mix;
    * ``async_op=True``, CPU tensors and the two-level world of several machines stay on torch.distributed;
    * splits that disagree between ranks give truncated segments (each receiver takes the shorter of what was sent and what
      it expects, and leaves the rest of its segment alone), not a hang."""
    _check(output)
    _check(input)
    if not async_op:
        w = _symm_world_for(output, group)
        if output_split_sizes is None and input_split_sizes is None:
            if w is not None and hasattr(w, "all_to_all_") and w.supports_raw(output):
                w.all_to_all_(output, input)
                return None
        elif w is not None and hasattr(w, "all_to_all_v_") and w.supports_raw(output) and w.supports_raw(input):
            w.all_to_all_v_(output, input, output_split_sizes, input_split_sizes)
            return None
    return dist.all_to_all_single(output, input, output_split_sizes=output_split_sizes,
                                  input_split_sizes=input_split_sizes, group=_g(group), async_op=async_op)


def all_to_all(output_tensor_list: List[torch.Tensor], input_tensor_list: List[torch.Tensor], group=None,
               async_op: bool = False):
    """``output_tensor_list[p]`` of rank r receives ``input_tensor_list[r]`` of rank p (torch's ``all_to_all``); the
    tensors may have any sizes.

    On a symmetric world a blocking call whose tensors are all CUDA runs on the variable-segment kernel
    (``SymmWorld.all_to_all_v_``), bit for bit; a list of the wrong length or of mixed dtypes raises there, on the rank that
    passed it.  The rules of :func:`all_to_all_single` with split sizes hold: every rank must call the list form,
    ``async_op=True``, CPU tensors and the two-level world stay on torch.distributed (whose gloo backend has no
    ``all_to_all``), and sizes that disagree between ranks give truncated segments, not a hang."""
    outs, ins = list(output_tensor_list), list(input_tensor_list)
    for t in outs + ins:
        _check(t)
    if not async_op and outs + ins:
        w = _symm_world_for((outs + ins)[0], group)
        if w is not None and hasattr(w, "all_to_all_v_") and all(w.supports_raw(t) for t in outs + ins):
            w.all_to_all_v_(outs, ins)
            return None
    return dist.all_to_all(outs, ins, group=_g(group), async_op=async_op)


def all_gather_into_tensor(output_tensor: torch.Tensor, input_tensor: torch.Tensor, group=None, async_op: bool = False):
    """Rank r's ``input_tensor`` lands at segment r of every rank's ``output_tensor`` (torch's ``all_gather_into_tensor``).
    On a symmetric world the CUDA tensors go through :func:`all_gather`'s peer-memory kernels, with ``output_tensor``'s
    segments as the (contiguous) output list.  As in :func:`all_gather`, the route also looks at ``output_tensor``: one
    whose dtype or size does not fit (world x the input's elements) goes to torch.distributed, which raises on that rank,
    while its peers are left waiting inside the kernel until its spin limit reports them (B2_SPIN_LIMIT)."""
    _check(output_tensor)
    _check(input_tensor)
    if not async_op:
        w = _symm_world_for(input_tensor, group)
        if w is not None and hasattr(w, "all_gather_") and w.supports_raw(input_tensor) and w.supports_raw(output_tensor) \
                and output_tensor.dtype == input_tensor.dtype and output_tensor.numel() == w.world * input_tensor.numel():
            w.all_gather_(list(output_tensor.view(w.world, -1).unbind(0)), input_tensor.view(-1))
            return None
    return dist.all_gather_into_tensor(output_tensor, input_tensor, group=_g(group), async_op=async_op)


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
