"""Symmetric peer memory worlds + fused all-reduce dispatch (the "b200" comm backend).

What replaces gloo/tcp/mpi for the gradient path (SURVEY §5.1; reference call
site train_dist.py:99, X1 in SURVEY §2.5b):

  * ``torch.distributed`` (NCCL/gloo) is used ONLY to bootstrap: ranks agree on
    a job token and synchronise set-up steps over the store;
  * every rank creates GPU memory with the CUDA VMM API (``csrc/symm_mem.cpp``),
    the POSIX file descriptors are exchanged over unix sockets (SCM_RIGHTS,
    here), and every rank maps every peer's allocation -> kernels load/store
    peer HBM over NVLink 5 / NVSwitch;
  * the same memory is bound to an NVSwitch multicast object when the host
    exposes it (NVLS: ``multimem.ld_reduce`` / ``multimem.st``);
  * ``cudaIpc`` handles are the fallback when fd export is not permitted.

A :class:`SymmHandle` is one symmetric allocation = [8 KiB signal pad | data].
Each allocation owns its signal pad, so collectives on different buffers may be
in flight on different streams at once.  All collectives must be issued in the
same order on every rank of the world (as with any communicator).

Collectives: ``all_reduce_`` and ``reduce_`` (SUM, PRODUCT, MAX, MIN on fp32,
bf16, fp16, fp64, int8, uint8, int32, int64 and bool), ``broadcast_``, ``all_gather_``, ``scatter_`` and ``gather_`` (raw
bytes, any dtype).  Each call picks its kernel variant with
:func:`plan_variant` (scatter and gather by the all-gather rule, on one rank's
segment) and never synchronises the host.

Point-to-point: ``send_``, ``recv_``, ``isend_`` and ``irecv_`` (raw bytes, any dtype) move messages through a mailbox
every world of more than one rank allocates when it is built (``csrc/p2p.cu``).  Each (peer, direction) pair has its own
stream, so a receive is never queued behind a send that waits for its peer; like NCCL they never synchronise the host.
``batch_p2p_`` runs a whole list of sends and receives in one launch (torch's ``batch_isend_irecv``), ordered against the
single calls through those pair streams.
"""
from __future__ import annotations

import array
import os
import socket
import struct
import threading
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import _ext

__all__ = ["SymmWorld", "SymmHandle", "P2PWork", "init_world", "lookup_world", "destroy_all", "VARIANTS", "COLLECTIVES",
           "op_code", "plan_variant", "DTYPE_CODES"]

PAD_BYTES = 8192                      # signal pad at the head of every allocation (B2_SIGNAL_WORDS*4 = 6016 B)
VARIANTS = {"oneshot": 0, "twoshot": 1, "nvls": 2, "ll": 3}
LL_CAP_VEC = 4096                     # LL (flag-in-data) inbox capacity per (parity, source): 4096 x 16 B = 64 KB messages
_TABLE_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "allreduce_table.json")


def _load_table():
    """Per-world variant thresholds measured by bench/allreduce_sweep.py --emit-table (wire bytes)."""
    try:
        import json
        with open(_TABLE_PATH) as f:
            return {int(k): v for k, v in json.load(f).get("worlds", {}).items()}
    except Exception:
        return {}
_WORLDS: Dict[object, "SymmWorld"] = {}
_DTYPES = (torch.float32, torch.bfloat16)
# The reductions' dtypes (torch's NCCL process group table) -> the kernels' wire dtype code (csrc/allreduce.cu).  Beyond fp32
# and bf16 the local dtype is the wire dtype: no scale, no bf16 wire, no NVLS.
DTYPE_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.float64: 3, torch.int8: 4, torch.uint8: 5,
               torch.int32: 6, torch.int64: 7, torch.bool: 8}
COLLECTIVES = ("allreduce", "reduce", "broadcast", "allgather", "reducescatter", "alltoall")
_OPS = {dist.ReduceOp.SUM: 0, dist.ReduceOp.PRODUCT: 1, dist.ReduceOp.MAX: 2, dist.ReduceOp.MIN: 3}


def op_code(op) -> Optional[int]:
    """The kernels' code of a reduction (0 SUM, 1 PRODUCT, 2 MAX, 3 MIN) for a ``torch.distributed.ReduceOp`` or one of
    those codes; ``None`` for any other op (e.g. AVG, or a pre-multiplied sum)."""
    if isinstance(op, int) and not isinstance(op, bool):
        return op if 0 <= op <= 3 else None
    try:
        return _OPS.get(op)
    except TypeError:                                      # an unhashable op object
        return None


def plan_variant(collective: str, op: int, nbytes: int, world: int, ll_max: int, oneshot_max: int, nvls_min: int,
                 multicast: bool, forced: Optional[str] = None) -> int:
    """Kernel variant (0 one-shot, 1 two-shot, 2 NVLS, 3 LL) of one collective from the measured thresholds.

    ``nbytes`` is the message: the wire bytes of a reduction or broadcast, one rank's input for an all-gather.  An all-gather
    uses LL while one rank's input is at most ``ll_max`` (which never exceeds the LL inbox), one-shot while its whole output
    is at most ``oneshot_max``, two-shot above.  NVLS reduces in the switch and so serves only the SUM all-reduce; ``forced``
    (``B200DIST_AR_VARIANT``) names a variant, and NVLS falls back to two-shot where it cannot run.  A reduce-scatter or an
    all-to-all (``nbytes``: one rank's segment) is LL (3) or pull (0) only, and any forced variant but LL runs pull."""
    if collective not in COLLECTIVES:
        raise ValueError(f"unknown collective {collective!r}")
    if world == 1:
        return 0
    if collective in ("reducescatter", "alltoall"):
        # Two kernels only: pull (0) and LL (3); a forced one-shot, two-shot or NVLS runs pull.  ``nbytes`` is one rank's
        # segment.  LL while it fits ll_max, pull above: unmeasured starting values, to be replaced by a sweep of
        # bench/allreduce_sweep.py --collective reducescatter|alltoall on a multi-GPU H100 machine.
        if forced in VARIANTS:
            return 3 if forced == "ll" else 0
        return 3 if nbytes <= ll_max else 0
    nvls_ok = multicast and collective == "allreduce" and op == 0
    if forced in VARIANTS:
        v = VARIANTS[forced]
        return v if (v != 2 or nvls_ok) else 1
    if collective == "allgather":
        return 3 if nbytes <= ll_max else 0 if world * nbytes <= oneshot_max else 1
    if nbytes <= ll_max:
        return 3
    if nbytes <= oneshot_max:
        return 0
    return 2 if (nvls_ok and nbytes >= nvls_min) else 1


def _env_int(name, default):
    try:
        return int(os.environ.get(name, default))
    except ValueError:
        return default


class SymmHandle:
    """One symmetric allocation, mapped on every rank of the world."""

    def __init__(self, world, nbytes, size, ptrs, mc_ptr, mem_handles, mc_handle, mode):
        self.world, self.nbytes, self.size = world, nbytes, size
        self.ll: Optional["SymmHandle"] = None               # inbox of the LL (flag-in-data) variant, if any
        self.base_ptrs: List[int] = ptrs                     # allocation bases (signal pads) per rank
        self.ptrs: List[int] = [p + PAD_BYTES for p in ptrs]  # data bases per rank
        self.sig_ptrs: List[int] = ptrs
        self.mc_base = mc_ptr
        self.mc_ptr = mc_ptr + PAD_BYTES if mc_ptr else 0
        self._mem_handles, self._mc_handle, self._mode = mem_handles, mc_handle, mode
        self.local: Optional[torch.Tensor] = None
        self.dtype = None

    def view(self, dtype, numel=None) -> torch.Tensor:
        """This rank's buffer as a 1-D tensor of ``dtype`` (no ownership: the handle keeps the mapping alive)."""
        es = torch.empty((), dtype=dtype).element_size()
        n = self.nbytes // es if numel is None else numel
        return _ext.C().tensor_from_ptr(self.ptrs[self.world.rank], n, dtype, self.world.device.index)

    def peer_view(self, r: int, dtype, numel=None) -> torch.Tensor:
        """Tensor aliasing rank ``r``'s buffer through the peer mapping (tests / debugging)."""
        es = torch.empty((), dtype=dtype).element_size()
        n = self.nbytes // es if numel is None else numel
        return _ext.C().tensor_from_ptr(self.ptrs[r], n, dtype, self.world.device.index)


class P2PWork:
    """The work object of :meth:`SymmWorld.isend_` / :meth:`SymmWorld.irecv_` (``comm.Request`` wraps it)."""

    def __init__(self, event: torch.cuda.Event, device: torch.device):
        self.event, self.device = event, device

    def wait(self) -> bool:
        """Order the current stream after the transfer (the host is not synchronised), as NCCL's work objects do."""
        torch.cuda.current_stream(self.device).wait_event(self.event)
        return True

    def is_completed(self) -> bool:
        """Has the transfer finished on the GPU?  (Never blocks.)"""
        return self.event.query()


class SymmWorld:
    """Symmetric-memory communicator over the ranks of a process group (<= 8 GPUs, one node)."""

    def __init__(self, group=None, multicast: Optional[bool] = None, mode: Optional[str] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("SymmWorld needs CUDA")
        self.C = _ext.C()
        self.group = group
        self.ranks = list(range(dist.get_world_size())) if group is None else list(dist.get_process_group_ranks(group))
        self.world = len(self.ranks)
        if self.world > 8:
            raise RuntimeError("symmetric worlds span one NVSwitch domain (<= 8 GPUs)")
        self.global_rank = dist.get_rank()
        self.rank = self.ranks.index(self.global_rank)
        self.device = torch.device("cuda", torch.cuda.current_device())
        torch.zeros(1, device=self.device)                       # make sure the primary context exists
        caps = self.C.symm_caps(self.device.index)
        want_mode = mode or os.environ.get("B200DIST_SYMM_MODE", "auto")
        self.mode = "vmm" if (caps[0] and caps[1] and want_mode in ("auto", "vmm")) else "ipc"
        if want_mode == "ipc":
            self.mode = "ipc"
        mc_env = os.environ.get("B200DIST_NVLS", "auto")
        want_mc = (mc_env != "0") if multicast is None else multicast
        self.multicast = bool(want_mc and caps[2] and self.mode == "vmm" and self.world > 1)
        # agree on mode / multicast across ranks (min)
        flags = [None] * self.world
        dist.all_gather_object(flags, (self.mode, self.multicast), group=group)
        if any(f[0] == "ipc" for f in flags):
            self.mode = "ipc"
        self.multicast = self.multicast and all(f[1] for f in flags) and self.mode == "vmm"
        tok = [os.urandom(6).hex() if self.rank == 0 else None]
        dist.broadcast_object_list(tok, src=self.ranks[0], group=group)
        self._token = tok[0]
        self._sock = None
        self._tag = 0
        if self.mode == "vmm" and self.world > 1:
            self._sock = socket.socket(socket.AF_UNIX, socket.SOCK_DGRAM)
            self._sock.bind(self._addr(self.rank))
            self._sock.settimeout(120.0)
            dist.barrier(group=group)
        self.gran = self.C.symm_granularity(self.device.index, self.world, self.multicast) if self.mode == "vmm" else 2 << 20
        self._handles: List[SymmHandle] = []
        self._staging: Dict[torch.dtype, SymmHandle] = {}
        self._lock = threading.Lock()
        # every CTA of a comm kernel spins on peer flags, so the grid never exceeds what is co-resident (1 CTA / SM)
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        self.max_blocks = _env_int("B200DIST_AR_BLOCKS", 0) or sms
        # size thresholds (wire bytes) from sweeps with bench/allreduce_sweep.py:
        #   2 GPUs : one-shot wins up to ~64 KB, two-shot above; NVLS never beats two-shot (no fan-in to amortise)
        #   8 GPUs : one-shot wins up to ~8 KB; above that NVLS (in-switch reduction) wins at every size, two-shot next
        # ... superseded per world size by the table bench/allreduce_sweep.py --emit-table writes (nearest measured world)
        defaults = {"ll_max": 32 << 10, "oneshot_max": (64 << 10) if self.world <= 2 else (8 << 10),
                    "nvls_min": (1 << 62) if self.world <= 2 else (8 << 10) + 1}
        table = _load_table()
        if table:
            near = min(table, key=lambda k: (abs(k - self.world), -k))
            defaults.update({k: int(v) for k, v in table[near].items() if k in defaults})
            self.table_world = near
        else:
            self.table_world = None
        self.ll_max = min(_env_int("B200DIST_LL_MAX", defaults["ll_max"]), LL_CAP_VEC * 16)
        self.oneshot_max = _env_int("B200DIST_ONESHOT_MAX", defaults["oneshot_max"])
        self.nvls_min = _env_int("B200DIST_NVLS_MIN", defaults["nvls_min"])
        self.nvls_error: Optional[str] = None
        # point-to-point mailbox (csrc/p2p.cu): allocated here because allocation is collective and a send involves two
        # ranks only; one stream per (peer, direction), as NCCL point-to-point has one communicator stream per pair
        self.p2p: Optional[SymmHandle] = None
        self._p2p_streams: Dict[tuple, torch.cuda.Stream] = {}
        if self.world > 1:
            ctas, slots, chunk, _ = self.C.p2p_config()
            self.p2p = self.alloc_bytes((self.world - 1) * ctas * slots * chunk, ll=False)

    # ------------------------------------------------------------------ plumbing
    def _addr(self, r: int) -> bytes:
        return b"\0b2dist-" + self._token.encode() + b"-%d" % r

    def _exchange_fds(self, fd: int, only_from: Optional[int] = None) -> Dict[int, int]:
        """Send ``fd`` to every peer (or only from rank ``only_from``); returns {src_rank: fd}."""
        self._tag += 1
        tag = self._tag
        senders = [only_from] if only_from is not None else list(range(self.world))
        if self.rank in senders:
            for r in range(self.world):
                if r != self.rank:
                    # (socket.send_fds ignores its address argument on CPython <= 3.12, so use sendmsg directly)
                    self._sock.sendmsg([struct.pack("ii", tag, self.rank)],
                                       [(socket.SOL_SOCKET, socket.SCM_RIGHTS, array.array("i", [fd]))], 0, self._addr(r))
        got: Dict[int, int] = {}
        expect = [s for s in senders if s != self.rank]
        while len(got) < len(expect):
            data, fds, _, _ = socket.recv_fds(self._sock, 8, 4)
            t, src = struct.unpack("ii", data)
            if t != tag or not fds:
                for f in fds:
                    os.close(f)
                raise RuntimeError(f"symmetric fd exchange out of order (tag {t} != {tag})")
            got[src] = fds[0]
        dist.barrier(group=self.group)
        return got

    # ------------------------------------------------------------------ allocation
    def alloc_bytes(self, nbytes: int, ll: bool = True) -> SymmHandle:
        """Collective: allocate ``nbytes`` of symmetric data (+ a private signal pad; + with ``ll`` the 2 MB inbox of the
        small-message flag-in-data variant, allocated here rather than lazily so that no collective set-up can land inside a
        CUDA-graph capture)."""
        C, dev = self.C, self.device.index
        nbytes = (int(nbytes) + 255) // 256 * 256 + 256       # slack for world-multiple vector padding
        size = (PAD_BYTES + nbytes + self.gran - 1) // self.gran * self.gran
        mem_handles, mc_handle, mc_ptr = [], 0, 0
        if self.world == 1:
            if self.mode == "vmm":
                h, fd = C.symm_create(dev, size)
                os.close(fd)
                ptrs = [C.symm_map(dev, h, size, self.gran)]
                mem_handles = [h]
            else:
                p, _ = C.ipc_alloc(size)
                ptrs = [p]
        elif self.mode == "vmm":
            h, fd = C.symm_create(dev, size)
            peers = self._exchange_fds(fd)
            os.close(fd)
            ptrs = []
            for r in range(self.world):
                if r == self.rank:
                    hr = h
                else:
                    hr = C.symm_import(peers[r])
                    os.close(peers[r])
                mem_handles.append(hr)
                ptrs.append(C.symm_map(dev, hr, size, self.gran))
            if self.multicast:
                # collective and failure-agreed: every rank gets a mapping or every rank degrades to two-shot together
                mc_handle, mc_ptr = self._setup_multicast(h, size)
                if not mc_ptr:
                    self.multicast = False
        else:
            p, hbytes = C.ipc_alloc(size)
            allh = [None] * self.world
            dist.all_gather_object(allh, hbytes, group=self.group)
            ptrs = [p if r == self.rank else C.ipc_open(allh[r]) for r in range(self.world)]
        hd = SymmHandle(self, nbytes, size, ptrs, mc_ptr, mem_handles, mc_handle, self.mode)
        C.tensor_from_ptr(ptrs[self.rank], size // 4, torch.int32, dev).zero_()
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        self._handles.append(hd)
        if ll and self.world > 1:
            hd.ll = self.alloc_bytes(2 * self.world * LL_CAP_VEC * 32, ll=False)
        return hd

    def _agree(self, ok: bool) -> bool:
        """Collective AND over the ranks of this world (every multicast set-up stage ends with one)."""
        flags = [None] * self.world
        dist.all_gather_object(flags, bool(ok), group=self.group)
        return all(flags)

    def _setup_multicast(self, mem_handle: int, size: int):
        """Collective.  Binds this allocation to an NVSwitch multicast object; returns ``(mc_handle, mc_ptr)`` on every
        rank, or ``(0, 0)`` on EVERY rank when any stage failed on any rank (``self.nvls_error`` says where).

        Containers may report CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED without a fabric manager / IMEX behind it, so each
        stage (create, fd exchange + import, add_device, bind, map) is followed by an agreement step: no rank is ever
        left inside a collective the others skipped, and the fd-exchange tags advance on all ranks or on none."""
        C, dev = self.C, self.device.index
        mc, fd, err = 0, -1, None
        # ---- stage 1: rank 0 creates the object; everyone learns the outcome BEFORE any fd exchange is attempted
        if self.rank == 0:
            try:
                mc, fd = C.mc_create(self.world, size)
            except Exception as e:
                err = f"cuMulticastCreate: {e!r}"
        created = [err is None if self.rank == 0 else None]
        dist.broadcast_object_list(created, src=self.ranks[0], group=self.group)
        if not created[0]:
            self.nvls_error = err or "cuMulticastCreate failed on rank 0"
            return 0, 0
        # ---- stage 2: fd exchange (all ranks enter it: tags stay aligned) + import on the receivers
        try:
            if self.rank == 0:
                self._exchange_fds(fd, only_from=0)
            else:
                got = self._exchange_fds(-1, only_from=0)
                try:
                    mc = C.symm_import(got[0])
                finally:
                    os.close(got[0])
        except Exception as e:
            err = f"multicast handle exchange/import: {e!r}"
        finally:
            if fd >= 0:
                os.close(fd)
        stage = "import"
        mc_ptr = 0
        ok = self._agree(err is None)
        # ---- stages 3..5: add_device -> bind -> map, each agreed
        for stage, fn in (("cuMulticastAddDevice", lambda: C.mc_add_device(mc, dev)),
                          ("cuMulticastBindMem", lambda: C.mc_bind(mc, mem_handle, size)),
                          ("map", lambda: C.symm_map(dev, mc, size, self.gran))):
            if not ok:
                break
            res = None
            try:
                res = fn()
            except Exception as e:
                err = f"{stage}: {e!r}"
            if stage == "map" and err is None:
                mc_ptr = res
            ok = self._agree(err is None)
        if not ok:
            self.nvls_error = err or f"multicast set-up failed on a peer rank (stage <= {stage})"
            if mc_ptr:
                try:
                    C.symm_unmap(mc_ptr, size)
                except Exception:
                    pass
            if mc:
                try:
                    C.symm_release(mc)
                except Exception:
                    pass
            return 0, 0
        return mc, mc_ptr

    def alloc(self, numel: int, dtype: torch.dtype) -> SymmHandle:
        """Collective: a symmetric buffer of ``numel`` elements (padded to 64) on every rank; ``handle.local`` is this
        rank's tensor, ``handle.ptrs`` the same buffer of every rank as mapped into THIS process."""
        es = torch.empty((), dtype=dtype).element_size()
        numel_p = (numel + 63) // 64 * 64
        hd = self.alloc_bytes(numel_p * es)
        hd.dtype = dtype
        hd.numel = numel_p
        hd.local = hd.view(dtype, numel_p)
        return hd

    # ------------------------------------------------------------------ collectives
    def supports(self, t: torch.Tensor) -> bool:
        """Can ``all_reduce_`` / ``reduce_`` take this tensor with a scale or a bf16 wire (CUDA, this device, fp32/bf16,
        contiguous)?"""
        return t.is_cuda and t.device == self.device and t.dtype in _DTYPES and t.is_contiguous()

    def supports_reduction(self, t: torch.Tensor) -> bool:
        """Can ``all_reduce_`` / ``reduce_`` take this tensor at all (CUDA, this device, contiguous, one of
        :data:`DTYPE_CODES`)?  The dtypes beyond :meth:`supports` take no scale and no wire conversion."""
        return t.is_cuda and t.device == self.device and t.dtype in DTYPE_CODES and t.is_contiguous()

    def pick_variant(self, wire_bytes: int) -> int:
        """Message size -> kernel (0 one-shot, 1 two-shot, 2 NVLS) from the measured thresholds; ``B200DIST_AR_VARIANT``
        forces one."""
        return self.plan("allreduce", 0, wire_bytes)

    def plan(self, collective: str, op: int, nbytes: int) -> int:
        """:func:`plan_variant` with this world's thresholds and ``B200DIST_AR_VARIANT``."""
        return plan_variant(collective, op, nbytes, self.world, self.ll_max, self.oneshot_max, self.nvls_min,
                            self.multicast, os.environ.get("B200DIST_AR_VARIANT"))

    def _launch(self, hd: SymmHandle, bf16: bool, n_vec: int, scale: float, src, dst, variant: Optional[int],
                max_blocks: Optional[int] = None, collective: str = "allreduce", op: int = 0, root: int = -1,
                dtype: Optional[int] = None):
        """One kernel call on ``hd``.  ``n_vec``: 16-byte vectors of the message (of the output for an all-gather or a gather,
        of the root's input for a scatter, a multiple of world for those three); ``root``: local rank (-1 for the all-to-all
        collectives); ``dtype``: a reduction's code in :data:`DTYPE_CODES` beyond fp32 / bf16 (``None``: fp32 or bf16 by
        ``bf16``), which NVLS cannot reduce, so it runs two-shot instead."""
        segmented = collective in ("allgather", "gather", "scatter")
        n_push = n_vec // self.world if segmented else n_vec
        v = self.plan("allgather" if segmented else collective, op, n_push * 16) if variant is None else variant
        if v == 2 and (not hd.mc_ptr or collective != "allreduce" or op != 0 or dtype is not None):
            v = 1
        if v == 3 and (hd.ll is None or n_push > LL_CAP_VEC):
            v = 0
        if v in (1, 2):
            n_vec = (n_vec + self.world - 1) // self.world * self.world
        ll = (hd.ll.ptrs, LL_CAP_VEC) if v == 3 else ([], 0)
        mb = self.max_blocks if max_blocks is None else max_blocks
        if collective == "broadcast":
            self.C.broadcast(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, root, self.rank, self.world, mb, *ll)
        elif collective == "allgather":
            self.C.allgather(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, self.rank, self.world, mb, *ll)
        elif collective == "gather":
            self.C.gather(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, root, self.rank, self.world, mb, *ll)
        elif collective == "scatter":
            self.C.scatter(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, root, self.rank, self.world, mb, *ll)
        elif dtype is not None:
            self.C.allreduce(v, False, hd.ptrs, hd.sig_ptrs, hd.mc_ptr, src, dst, n_vec, float(scale), self.rank,
                             self.world, mb, *ll, op, root, dtype=dtype)
        else:
            self.C.allreduce(v, bf16, hd.ptrs, hd.sig_ptrs, hd.mc_ptr, src, dst, n_vec, float(scale), self.rank,
                             self.world, mb, *ll, op, root)
        return v

    def supports_op(self, op) -> bool:
        """Can ``all_reduce_`` / ``reduce_`` run this reduction (SUM, PRODUCT, MAX, MIN)?"""
        return op_code(op) is not None

    def supports_raw(self, t: torch.Tensor) -> bool:
        """Can ``broadcast_`` / ``all_gather_`` / ``scatter_`` / ``gather_`` take this tensor (CUDA, this device, contiguous,
        any dtype)?"""
        return t.is_cuda and t.device == self.device and t.is_contiguous()

    def local_rank(self, root: int) -> int:
        """The rank within this world of global rank ``root``."""
        if root not in self.ranks:
            raise ValueError(f"rank {root} is not in this world (global ranks {self.ranks})")
        return self.ranks.index(root)

    def all_reduce_(self, t: torch.Tensor, scale: float = 1.0, handle: Optional[SymmHandle] = None,
                    variant: Optional[int] = None, wire: Optional[torch.dtype] = None,
                    max_blocks: Optional[int] = None, op=dist.ReduceOp.SUM) -> torch.Tensor:
        """In-place ``t <- scale * sum_ranks t`` with the fused peer-memory kernels; ``op`` PRODUCT / MAX / MIN combine
        instead of summing (fp32 in rank order, IEEE maximum / minimum: NaN wins, -0 < +0) and take no scale.

        Beyond fp32 / bf16, ``t`` may be fp16 (fp32 accumulator, rounded once), fp64, int8, uint8, int32, int64 (wrapping
        SUM / PRODUCT, as NCCL) or bool (SUM is MAX, as torch.distributed maps it); those take no scale and no ``wire``.

        ``handle`` given and ``t`` aliasing its data  -> zero-copy symmetric path;
        otherwise ``t`` is staged through a world-owned symmetric buffer with the
        copy-in / copy-out fused into the same kernel.  ``wire=torch.bfloat16``
        sends fp32 tensors as bf16 over NVLink (fp32 accumulate, fp32 result; SUM only)."""
        return self._reduce(t, scale, handle, variant, wire, max_blocks, op, -1)

    def reduce_(self, t: torch.Tensor, root: int, op=dist.ReduceOp.SUM, handle: Optional[SymmHandle] = None,
                variant: Optional[int] = None, wire: Optional[torch.dtype] = None,
                max_blocks: Optional[int] = None) -> torch.Tensor:
        """In-place reduce to global rank ``root``: its ``t`` receives the all-reduce result, every other rank's ``t`` is
        left as it was."""
        return self._reduce(t, 1.0, handle, variant, wire, max_blocks, op, self.local_rank(root))

    def _reduce(self, t, scale, handle, variant, wire, max_blocks, op, root):
        code = op_code(op)
        if code is None:
            raise ValueError(f"the fused reductions are SUM, PRODUCT, MAX and MIN, got {op!r}")
        if code != 0 and scale != 1.0:
            raise ValueError("scale applies to SUM only")
        if not self.supports_reduction(t):
            raise TypeError(f"fused all_reduce needs a contiguous CUDA tensor on this device of one of "
                            f"{[str(d).replace('torch.', '') for d in DTYPE_CODES]}, got {t.dtype}")
        if not self.supports(t):
            return self._reduce_same_dtype(t, scale, handle, variant, wire, max_blocks, code, root)
        if code != 0 and wire is not None and wire != t.dtype:
            raise TypeError("a bf16 wire for an fp32 tensor is for SUM only")
        if self.world == 1:
            if scale != 1.0:
                t.mul_(scale)
            return t
        es = t.element_size()
        if handle is not None and handle.local is not None and t.data_ptr() >= handle.ptrs[self.rank] and \
                t.data_ptr() + t.numel() * es <= handle.ptrs[self.rank] + handle.nbytes and \
                t.data_ptr() == handle.ptrs[self.rank] and (wire is None or wire == t.dtype):
            nbytes = (t.numel() * es + 15) // 16 * 16
            self._launch(handle, t.dtype == torch.bfloat16, nbytes // 16, scale, None, None, variant, max_blocks,
                         "reduce" if root >= 0 else "allreduce", code, root)
            return t
        wire_dt = wire or t.dtype
        if wire_dt not in _DTYPES or (wire_dt == torch.float32 and t.dtype == torch.bfloat16):
            raise TypeError("wire dtype must be bf16 or the tensor dtype")
        wes = 2 if wire_dt == torch.bfloat16 else 4
        wire_bytes = t.numel() * wes
        st = self._staging_for(wire_dt, wire_bytes)
        flat = t.view(-1)
        kind = "reduce" if root >= 0 else "allreduce"
        if wire_bytes % (16 * self.world) == 0 and t.data_ptr() % 16 == 0:
            self._launch(st, wire_dt == torch.bfloat16, wire_bytes // 16, scale, flat, flat, variant, max_blocks, kind, code,
                         root)
        else:  # ragged size: torch copies around an in-place symmetric all-reduce
            buf = st.view(wire_dt, (wire_bytes + 15) // 16 * 16 // wes + 64 * 8)
            buf[:flat.numel()].copy_(flat)
            buf[flat.numel():].zero_()
            self._launch(st, wire_dt == torch.bfloat16, (wire_bytes + 15) // 16, scale, None, None, variant, max_blocks,
                         kind, code, root)
            if root < 0 or root == self.rank:
                flat.copy_(buf[:flat.numel()])
        return t

    def _reduce_same_dtype(self, t, scale, handle, variant, wire, max_blocks, code, root):
        """The reductions beyond fp32 / bf16: the wire dtype is ``t``'s, staged through the byte staging buffer the raw
        moves use."""
        if scale != 1.0:
            raise ValueError(f"scale applies to fp32 / bf16 SUM only, not to {t.dtype}")
        if wire is not None and wire != t.dtype:
            raise TypeError(f"a wire dtype conversion is for fp32 / bf16 tensors only, not {t.dtype}")
        if t.dtype == torch.bool and code == 0:
            code = 2                                           # torch.distributed's NCCL group reduces a bool SUM as MAX
        if self.world == 1:
            return t
        dt = DTYPE_CODES[t.dtype]
        kind = "reduce" if root >= 0 else "allreduce"
        nbytes = t.numel() * t.element_size()
        n_vec = (nbytes + 15) // 16
        if handle is not None and t.data_ptr() == handle.ptrs[self.rank] and n_vec * 16 <= handle.nbytes:
            self._launch(handle, False, n_vec, 1.0, None, None, variant, max_blocks, kind, code, root, dtype=dt)
            return t
        st = self._staging_for(torch.float32, nbytes)
        flat = t.view(-1)
        if nbytes % (16 * self.world) == 0 and t.data_ptr() % 16 == 0:
            self._launch(st, False, n_vec, 1.0, flat, flat, variant, max_blocks, kind, code, root, dtype=dt)
        else:  # ragged size: torch copies around an in-place symmetric reduction (nobody reads the padding's results)
            raw = flat.view(torch.uint8)
            buf = st.view(torch.uint8, st.nbytes)
            buf[:nbytes].copy_(raw)
            self._launch(st, False, n_vec, 1.0, None, None, variant, max_blocks, kind, code, root, dtype=dt)
            if root < 0 or root == self.rank:
                raw.copy_(buf[:nbytes])
        return t

    def broadcast_(self, t: torch.Tensor, root: int, handle: Optional[SymmHandle] = None, variant: Optional[int] = None,
                   max_blocks: Optional[int] = None) -> torch.Tensor:
        """In place: every rank's ``t`` receives global rank ``root``'s bytes (any dtype; copied bit for bit)."""
        r = self.local_rank(root)
        if not self.supports_raw(t):
            raise TypeError("fused broadcast needs a contiguous CUDA tensor on this device")
        if self.world == 1:
            return t
        nbytes = t.numel() * t.element_size()
        n_vec = (nbytes + 15) // 16
        if handle is not None and t.data_ptr() == handle.ptrs[self.rank] and n_vec * 16 <= handle.nbytes:
            self._launch(handle, False, n_vec, 1.0, None, None, variant, max_blocks, "broadcast", 0, r)
            return t
        st = self._staging_for(torch.float32, nbytes)
        flat = t.view(-1)
        if nbytes % (16 * self.world) == 0 and t.data_ptr() % 16 == 0:
            self._launch(st, False, n_vec, 1.0, flat, flat, variant, max_blocks, "broadcast", 0, r)
        else:  # ragged size: torch copies around an in-place symmetric broadcast
            raw = flat.view(torch.uint8)
            buf = st.view(torch.uint8, st.nbytes)
            if self.rank == r:
                buf[:nbytes].copy_(raw)
            self._launch(st, False, n_vec, 1.0, None, None, variant, max_blocks, "broadcast", 0, r)
            if self.rank != r:
                raw.copy_(buf[:nbytes])
        return t

    def all_gather_(self, outs: List[torch.Tensor], t: torch.Tensor, handle: Optional[SymmHandle] = None,
                    variant: Optional[int] = None, max_blocks: Optional[int] = None) -> List[torch.Tensor]:
        """``outs[r]`` <- rank r's ``t`` on every rank (any dtype; copied bit for bit).  With ``handle``, ``t`` may sit at
        byte ``rank * len`` of the handle's buffer (``len`` a multiple of 16): the call then gathers in place there, and
        ``outs`` entries that already alias their slice are not copied."""
        if len(outs) != self.world:
            raise ValueError(f"all_gather needs {self.world} output tensors, got {len(outs)}")
        if not self.supports_raw(t) or not all(self.supports_raw(o) for o in outs):
            raise TypeError("fused all_gather needs contiguous CUDA tensors on this device")
        if any(o.dtype != t.dtype or o.numel() != t.numel() for o in outs):
            raise ValueError("every output of all_gather must have the input's dtype and size")
        if self.world == 1:
            outs[0].copy_(t)
            return outs
        nbytes = t.numel() * t.element_size()
        seg = (nbytes + 15) // 16                              # vectors per rank
        n_vec = seg * self.world
        slot = seg * 16
        if handle is not None and nbytes % 16 == 0 and t.data_ptr() == handle.ptrs[self.rank] + self.rank * slot and \
                n_vec * 16 <= handle.nbytes:
            self._launch(handle, False, n_vec, 1.0, None, None, variant, max_blocks, "allgather")
            base, buf = handle.ptrs[self.rank], handle.view(torch.uint8)
        else:
            st = self._staging_for(torch.float32, n_vec * 16)
            base, buf = st.ptrs[self.rank], st.view(torch.uint8, st.nbytes)
            if nbytes % 16 == 0 and t.data_ptr() % 16 == 0:
                o0 = outs[0].data_ptr()
                contiguous = o0 % 16 == 0 and all(o.data_ptr() == o0 + r * nbytes for r, o in enumerate(outs))
                dst = self.C.tensor_from_ptr(o0, n_vec * 16, torch.uint8, self.device.index) if contiguous else None
                self._launch(st, False, n_vec, 1.0, t.view(-1), dst, variant, max_blocks, "allgather")
                if contiguous:
                    return outs
            else:  # ragged size: stage this rank's bytes at its slot, gather in place
                buf[self.rank * slot:self.rank * slot + nbytes].copy_(t.view(-1).view(torch.uint8))
                self._launch(st, False, n_vec, 1.0, None, None, variant, max_blocks, "allgather")
        for r, o in enumerate(outs):
            if o.data_ptr() != base + r * slot:
                o.view(-1).view(torch.uint8).copy_(buf[r * slot:r * slot + nbytes])
        return outs

    def _root_list(self, what: str, lst, t: torch.Tensor) -> None:
        """The root's list of a scatter or gather: ``world`` contiguous CUDA tensors on this device with ``t``'s dtype and
        size.  Raised on the root only, before any launch: its peers are then left inside the kernel until its spin limit
        reports them (B2_SPIN_LIMIT), as with a collective that one rank never joins."""
        if lst is None or len(lst) != self.world:
            raise ValueError(f"{what} needs {self.world} tensors on the root, got {None if lst is None else len(lst)}")
        if not all(isinstance(o, torch.Tensor) and self.supports_raw(o) for o in lst):
            raise TypeError(f"fused {what} needs contiguous CUDA tensors on this device")
        if any(o.dtype != t.dtype or o.numel() != t.numel() for o in lst):
            raise ValueError(f"every tensor of {what}'s list must have the tensor's dtype and size")

    def _one_block(self, lst: List[torch.Tensor], nbytes: int) -> Optional[torch.Tensor]:
        """``lst`` as one uint8 tensor when its entries are consecutive views of one 16-byte aligned block, else None."""
        o0 = lst[0].data_ptr()
        if o0 % 16 or any(o.data_ptr() != o0 + r * nbytes for r, o in enumerate(lst)):
            return None
        return self.C.tensor_from_ptr(o0, self.world * nbytes, torch.uint8, self.device.index)

    def scatter_(self, t: torch.Tensor, scatter_list: Optional[List[torch.Tensor]], root: int,
                 variant: Optional[int] = None, max_blocks: Optional[int] = None) -> torch.Tensor:
        """``t`` <- global rank ``root``'s ``scatter_list[rank]`` on every rank (any dtype; copied bit for bit).
        ``scatter_list`` is read on the root only.

        Whether src and dst are fused into the kernel depends on ``t``'s size alone, so every rank makes the same choice
        (the kernels' barriers depend on it) while only the root holds the list: a multiple of 16 bytes is fused (an
        unaligned ``t`` through an aligned scratch tensor, a root list that is not one block through the staging buffer),
        any other size goes through the staging buffer in place."""
        r0 = self.local_rank(root)
        if not self.supports_raw(t):
            raise TypeError("fused scatter needs a contiguous CUDA tensor on this device")
        if self.rank == r0:
            self._root_list("scatter", scatter_list, t)
        if self.world == 1:
            t.copy_(scatter_list[0])
            return t
        nbytes = t.numel() * t.element_size()
        seg = (nbytes + 15) // 16                              # vectors per rank
        n_vec, slot = seg * self.world, seg * 16
        st = self._staging_for(torch.float32, n_vec * 16)      # the same size on every rank: allocation is collective
        buf = st.view(torch.uint8, st.nbytes)
        block = self._one_block(scatter_list, nbytes) if self.rank == r0 and nbytes % 16 == 0 else None
        if self.rank == r0 and block is None:
            for r, o in enumerate(scatter_list):
                buf[r * slot:r * slot + nbytes].copy_(o.view(-1).view(torch.uint8))
        out = t.view(-1).view(torch.uint8)
        if nbytes % 16 == 0:
            dst = out if out.data_ptr() % 16 == 0 else torch.empty_like(out)
            src = block if block is not None else buf[:n_vec * 16]
            self._launch(st, False, n_vec, 1.0, src, dst, variant, max_blocks, "scatter", 0, r0)
            if dst is not out:
                out.copy_(dst)
        else:  # ragged size: scatter in place, then copy this rank's slot out
            self._launch(st, False, n_vec, 1.0, None, None, variant, max_blocks, "scatter", 0, r0)
            out.copy_(buf[self.rank * slot:self.rank * slot + nbytes])
        return t

    def gather_(self, t: torch.Tensor, gather_list: Optional[List[torch.Tensor]], root: int,
                variant: Optional[int] = None, max_blocks: Optional[int] = None) -> Optional[List[torch.Tensor]]:
        """Global rank ``root``'s ``gather_list[r]`` <- rank r's ``t`` (any dtype; copied bit for bit).  ``gather_list`` is
        read and written on the root only; the others' outputs are left alone.  src and dst are chosen as in
        :meth:`scatter_`, by ``t``'s size alone; a root list that is not one block is filled from the staging buffer."""
        r0 = self.local_rank(root)
        if not self.supports_raw(t):
            raise TypeError("fused gather needs a contiguous CUDA tensor on this device")
        if self.rank == r0:
            self._root_list("gather", gather_list, t)
        if self.world == 1:
            gather_list[0].copy_(t)
            return gather_list
        nbytes = t.numel() * t.element_size()
        seg = (nbytes + 15) // 16
        n_vec, slot = seg * self.world, seg * 16
        st = self._staging_for(torch.float32, n_vec * 16)
        buf = st.view(torch.uint8, st.nbytes)
        block = self._one_block(gather_list, nbytes) if self.rank == r0 and nbytes % 16 == 0 else None
        inp = t.view(-1).view(torch.uint8)
        if nbytes % 16 == 0:
            src = inp if inp.data_ptr() % 16 == 0 else inp.clone()
            dst = block if block is not None else buf[:n_vec * 16]
            self._launch(st, False, n_vec, 1.0, src, dst, variant, max_blocks, "gather", 0, r0)
        else:  # ragged size: stage this rank's bytes at its slot, gather in place
            buf[self.rank * slot:self.rank * slot + nbytes].copy_(inp)
            self._launch(st, False, n_vec, 1.0, None, None, variant, max_blocks, "gather", 0, r0)
        if self.rank != r0:
            return None
        if block is None:
            for r, o in enumerate(gather_list):
                o.view(-1).view(torch.uint8).copy_(buf[r * slot:r * slot + nbytes])
        return gather_list

    # ------------------------------------------------------------------ reduce-scatter / all-to-all
    def _launch_segments(self, kind: str, hd: SymmHandle, src, dst, seg_vec: int, variant: Optional[int],
                         max_blocks: Optional[int], op: int = 0, dtype: int = 0) -> int:
        """One reduce-scatter or all-to-all kernel on ``hd``: world segments of ``seg_vec`` vectors; ``src`` None reads this
        rank's buffer, ``dst`` None (reduce-scatter) leaves the result at segment ``rank`` of it."""
        v = self.plan(kind, op, seg_vec * 16) if variant is None else variant
        v = 3 if v == 3 and hd.ll is not None and seg_vec <= LL_CAP_VEC else 0
        ll = (hd.ll.ptrs, LL_CAP_VEC) if v == 3 else ([], 0)
        mb = self.max_blocks if max_blocks is None else max_blocks
        n_vec = seg_vec * self.world
        if kind == "reducescatter":
            self.C.reduce_scatter(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, self.rank, self.world, mb, *ll, op, dtype)
        else:
            self.C.alltoall(v, hd.ptrs, hd.sig_ptrs, src, dst, n_vec, self.rank, self.world, mb, *ll)
        return v

    def reduce_scatter_(self, out: torch.Tensor, inp, op=dist.ReduceOp.SUM, variant: Optional[int] = None,
                        max_blocks: Optional[int] = None) -> torch.Tensor:
        """``out`` <- segment ``rank`` of the reduction over the ranks of ``inp``: a tensor of world x ``out``'s elements, or
        a list of world tensors of ``out``'s size.  Ops and dtypes as :meth:`all_reduce_` without scale or wire (a bool SUM
        is a MAX); the result is bit for bit slice ``rank`` of the all-reduce of the same inputs.

        The kernel reads ``inp`` in place when it is one 16-byte aligned block of segments of a multiple of 16 bytes, and
        writes ``out`` directly when that is aligned too and is not a part of that block other than a whole segment;
        anything else goes through the staging buffer: the segments are
        copied to 16-byte aligned slots, and the result is copied out of slot ``rank``.  The staging size depends on
        ``out``'s size alone, so it is the same on every rank (allocation is collective), and no call allocates device
        memory.  A malformed ``inp`` raises before any launch, on this rank only: its peers are then left inside the kernel
        until its spin limit reports them (B2_SPIN_LIMIT)."""
        code = op_code(op)
        if code is None:
            raise ValueError(f"the fused reductions are SUM, PRODUCT, MAX and MIN, got {op!r}")
        if not self.supports_reduction(out):
            raise TypeError(f"fused reduce_scatter needs a contiguous CUDA tensor on this device of one of "
                            f"{[str(d).replace('torch.', '') for d in DTYPE_CODES]}, got {out.dtype}")
        if isinstance(inp, torch.Tensor):
            if not self.supports_raw(inp) or inp.dtype != out.dtype or inp.numel() != self.world * out.numel():
                raise ValueError(f"reduce_scatter needs a contiguous CUDA input of {out.dtype} with world x the output's "
                                 f"elements ({self.world * out.numel()}), got {inp.dtype} x {inp.numel()}")
            segs = list(inp.view(-1).view(self.world, -1).unbind(0)) if out.numel() else [inp.view(-1)] * self.world
        else:
            segs = list(inp) if inp is not None else []
            if len(segs) != self.world:
                raise ValueError(f"reduce_scatter needs {self.world} input tensors, got {len(segs)}")
            if not all(isinstance(s, torch.Tensor) and self.supports_raw(s) for s in segs):
                raise TypeError("fused reduce_scatter needs contiguous CUDA tensors on this device")
            if any(s.dtype != out.dtype or s.numel() != out.numel() for s in segs):
                raise ValueError("every tensor of reduce_scatter's list must have the output's dtype and size")
        if out.dtype == torch.bool and code == 0:
            code = 2                                           # torch.distributed's NCCL group reduces a bool SUM as MAX
        if self.world == 1:
            s0 = segs[0].view(out.shape)
            a0, b0, nb = s0.data_ptr(), out.data_ptr(), out.numel() * out.element_size()
            out.copy_(s0.clone() if a0 != b0 and a0 < b0 + nb and b0 < a0 + nb else s0)   # torch refuses a partial overlap
            return out
        dt = DTYPE_CODES[out.dtype]
        nbytes = out.numel() * out.element_size()
        seg = (nbytes + 15) // 16
        slot = seg * 16
        st = self._staging_for(torch.float32, self.world * slot)   # the same size on every rank: allocation is collective
        buf = st.view(torch.uint8, st.nbytes)
        raw_out = out.view(-1).view(torch.uint8)
        block = self._one_block(segs, nbytes) if nbytes % 16 == 0 else None
        src = block.view(out.dtype) if block is not None else None
        b0 = raw_out.data_ptr()
        dst = out.view(-1) if nbytes % 16 == 0 and b0 % 16 == 0 else None
        if dst is not None and src is not None:
            # an output inside the input block is safe only as a whole segment (vector j of every segment is read and
            # written by one thread); at any other offset a thread would overwrite input another thread still reads
            a0 = src.data_ptr()
            if a0 < b0 + nbytes and b0 < a0 + self.world * nbytes and (b0 - a0) % nbytes:
                dst = None
        if src is None:                                        # stage every segment at its aligned slot
            for r, s in enumerate(segs):
                buf[r * slot:r * slot + nbytes].copy_(s.reshape(-1).view(torch.uint8))
        self._launch_segments("reducescatter", st, src, dst, seg, variant, max_blocks, code, dt)
        if dst is None:                                        # the result is at this rank's slot of its buffer
            raw_out.copy_(buf[self.rank * slot:self.rank * slot + nbytes])
        return out

    def all_to_all_(self, out: torch.Tensor, inp: torch.Tensor, variant: Optional[int] = None,
                    max_blocks: Optional[int] = None) -> torch.Tensor:
        """Equal-segment all-to-all: segment p of ``out`` <- segment ``rank`` of rank p's ``inp`` (any dtype, copied bit for
        bit; ``out`` and ``inp`` have one size, a multiple of world elements; ``out`` may be ``inp``).  Segments of a
        multiple of 16 bytes are read from an aligned ``inp`` and written to an aligned ``out`` that does not partly overlap
        it; anything else goes through the staging buffer, whose first half holds the input segments at 16-byte aligned
        slots and whose second half receives the output.  The staging size depends on the size alone, and no call
        allocates device memory."""
        if not self.supports_raw(out) or not self.supports_raw(inp):
            raise TypeError("fused all_to_all needs contiguous CUDA tensors on this device")
        if inp.dtype != out.dtype or inp.numel() != out.numel() or out.numel() % self.world:
            raise ValueError(f"all_to_all needs an input and an output of one dtype and size, a multiple of world "
                             f"({self.world}) elements; got {inp.dtype} x {inp.numel()} and {out.dtype} x {out.numel()}")
        if self.world == 1:
            out.copy_(inp)
            return out
        raw_in, raw_out = inp.view(-1).view(torch.uint8), out.view(-1).view(torch.uint8)
        total = raw_out.numel()
        nbytes = total // self.world
        seg = (nbytes + 15) // 16
        slot = seg * 16
        n = self.world * slot
        st = self._staging_for(torch.float32, 2 * n)
        buf = st.view(torch.uint8, st.nbytes)
        a0, b0 = raw_in.data_ptr(), raw_out.data_ptr()
        overlap = a0 != b0 and a0 < b0 + total and b0 < a0 + total
        fused = nbytes % 16 == 0
        src = raw_in if fused and a0 % 16 == 0 else None
        dst = raw_out if fused and b0 % 16 == 0 and not overlap else buf[n:2 * n]
        if src is None:                                        # stage every segment at its aligned slot
            for p in range(self.world):
                buf[p * slot:p * slot + nbytes].copy_(raw_in[p * nbytes:(p + 1) * nbytes])
        self._launch_segments("alltoall", st, src, dst, seg, variant, max_blocks)
        if dst is not raw_out:
            # contiguous copies (memcpy, no kernel): ranks driven from one process, as on emulated ranks, must not load a
            # kernel module while a peer's kernel spins, since lazy loading may wait for it
            for p in range(self.world):
                raw_out[p * nbytes:(p + 1) * nbytes].copy_(dst[p * slot:p * slot + nbytes])
        return out

    def _splits(self, what: str, splits, t: torch.Tensor) -> List[int]:
        """Rows of ``t``'s dim 0 per rank: ``splits`` checked against it, or equal ones when it is None."""
        rows = t.shape[0]
        if splits is None:
            if rows % self.world:
                raise ValueError(f"all_to_all: the {what} has {rows} rows, which do not split equally over world "
                                 f"{self.world}; give {what}_split_sizes")
            return [rows // self.world] * self.world
        s = [int(x) for x in splits]
        if len(s) != self.world:
            raise ValueError(f"all_to_all: {what}_split_sizes needs {self.world} entries, got {len(s)}")
        if any(x < 0 for x in s):
            raise ValueError(f"all_to_all: {what}_split_sizes has a negative entry: {s}")
        if sum(s) != rows:
            raise ValueError(f"all_to_all: {what}_split_sizes sums to {sum(s)}, but the {what} has {rows} rows")
        return s

    def _segments(self, t: torch.Tensor, splits: List[int]) -> List[torch.Tensor]:
        """``t``'s rows cut by ``splits``, as uint8 views."""
        raw = t.reshape(-1).view(torch.uint8)
        row = raw.numel() // t.shape[0] if t.shape[0] else 0
        offs = [0]
        for n in splits:
            offs.append(offs[-1] + n * row)
        return [raw[offs[p]:offs[p + 1]] for p in range(self.world)]

    def all_to_all_v_(self, out, inp, output_split_sizes=None, input_split_sizes=None,
                      max_blocks: Optional[int] = None):
        """All-to-all with segments of any size, torch's ``all_to_all_single`` with split sizes and its list form
        ``all_to_all``, copied bit for bit (any dtype).

        Single-tensor form: ``out`` and ``inp`` are tensors of one dtype whose dim 0 is cut by ``output_split_sizes`` /
        ``input_split_sizes`` (``None``: equal splits); rows p of ``out`` receive rank p's rows for this rank.  List form:
        ``out`` and ``inp`` are lists of ``world`` tensors of one dtype and any sizes; ``out[p]`` receives rank p's
        ``inp[rank]``.  Every rank must use the same form.

        Every segment, of any length and alignment, is read and written in place by one kernel that moves fixed chunks per
        pair in rounds; the round count comes from the lengths every rank publishes, so the staging size and the grid depend on
        the world size alone.  A receiver takes min(what its peer sends, what it expects): splits that disagree between ranks
        truncate segments, and bytes beyond are left as they were.  An output that overlaps an input reads from a copy of that
        input made on the current stream, the only device memory a call allocates.

        A bad argument (a split list of the wrong length, a negative split or one that does not sum to dim 0, a list of the
        wrong length or of mixed dtypes, or a tensor that is not contiguous, not CUDA or on another device) raises before any
        launch, on this rank only: its peers are then left inside the kernel until its spin limit reports them
        (B2_SPIN_LIMIT)."""
        if isinstance(out, (list, tuple)) or isinstance(inp, (list, tuple)):
            if not isinstance(out, (list, tuple)) or not isinstance(inp, (list, tuple)):
                raise TypeError("all_to_all takes two lists of tensors or two tensors")
            if output_split_sizes is not None or input_split_sizes is not None:
                raise ValueError("all_to_all: split sizes belong to the single-tensor form")
            outs, ins = list(out), list(inp)
            for what, lst in (("output", outs), ("input", ins)):
                if len(lst) != self.world:
                    raise ValueError(f"all_to_all needs {self.world} {what} tensors, got {len(lst)}")
            if not all(isinstance(t, torch.Tensor) and self.supports_raw(t) for t in outs + ins):
                raise TypeError("fused all_to_all needs contiguous CUDA tensors on this device")
            if len({t.dtype for t in outs + ins}) != 1:
                raise ValueError(f"all_to_all needs tensors of one dtype, got {sorted({str(t.dtype) for t in outs + ins})}")
            dsts = [t.reshape(-1).view(torch.uint8) for t in outs]
            srcs = [t.reshape(-1).view(torch.uint8) for t in ins]
        else:
            if not isinstance(out, torch.Tensor) or not isinstance(inp, torch.Tensor):
                raise TypeError("all_to_all takes two lists of tensors or two tensors")
            if not self.supports_raw(out) or not self.supports_raw(inp):
                raise TypeError("fused all_to_all needs contiguous CUDA tensors on this device")
            if out.dtype != inp.dtype:
                raise ValueError(f"all_to_all needs an input and an output of one dtype, got {inp.dtype} and {out.dtype}")
            if out.dim() == 0 or inp.dim() == 0:
                raise ValueError("all_to_all with split sizes cuts dim 0, so it needs tensors of at least one dimension")
            dsts = self._segments(out, self._splits("output", output_split_sizes, out))
            srcs = self._segments(inp, self._splits("input", input_split_sizes, inp))
        overlap = lambda a, b: a.numel() and b.numel() and a.data_ptr() < b.data_ptr() + b.numel() and \
            b.data_ptr() < a.data_ptr() + a.numel()  # noqa: E731
        if any(overlap(s, d) for s in srcs for d in dsts):
            if isinstance(inp, torch.Tensor):                  # one copy of the whole input, then its segments
                srcs = self._segments(inp.clone(), self._splits("input", input_split_sizes, inp))
            else:
                srcs = [s.clone() if any(overlap(s, d) for d in dsts) else s for s in srcs]
        if self.world == 1:
            n = min(srcs[0].numel(), dsts[0].numel())
            if n:
                dsts[0][:n].copy_(srcs[0][:n])
            return out
        chunk, header = self.C.alltoallv_config()
        st = self._staging_for(torch.float32, header + 2 * self.world * chunk)   # the world size alone: allocation is collective
        mb = self.max_blocks if max_blocks is None else max_blocks
        self.C.alltoallv(st.ptrs, st.sig_ptrs, srcs, [s.numel() for s in srcs], dsts, [d.numel() for d in dsts], self.rank,
                         self.world, mb)
        return out

    # ------------------------------------------------------------------ point-to-point
    def send_(self, t: torch.Tensor, dst: int) -> None:
        """Send ``t``'s bytes to global rank ``dst`` (any dtype; copied bit for bit).  Like ``dist.send`` on NCCL it returns
        without synchronising the host: the current stream is ordered after the transfer, so ``t`` may then be reused.

        The receiver must post a receive of the same byte count from this rank; messages between one pair are matched in
        the order they are issued (there are no tags)."""
        self._p2p(True, t, dst).wait()

    def recv_(self, t: torch.Tensor, src: int) -> torch.Tensor:
        """Receive into ``t`` the bytes global rank ``src`` sends (same byte count); the current stream is ordered after
        the transfer, the host is not synchronised."""
        self._p2p(False, t, src).wait()
        return t

    def isend_(self, t: torch.Tensor, dst: int) -> "P2PWork":
        """Non-blocking :meth:`send_`: ``t`` must not be written before the returned work's ``wait()``."""
        return self._p2p(True, t, dst)

    def irecv_(self, t: torch.Tensor, src: int) -> "P2PWork":
        """Non-blocking :meth:`recv_`: ``t`` must not be read or written before the returned work's ``wait()``."""
        return self._p2p(False, t, src)

    def _p2p(self, send: bool, t: torch.Tensor, peer_rank: int) -> "P2PWork":
        """One transfer on the (peer, direction) stream: that stream waits for the current one, the kernel runs on it, and
        the returned work holds an event recorded after it.  A data pointer that is not 16-byte aligned goes through an
        aligned scratch copy made on the same stream."""
        what = "send" if send else "recv"
        peer = self.local_rank(peer_rank)
        if peer == self.rank:
            raise ValueError(f"{what}: rank {peer_rank} cannot {what} to itself")
        if not self.supports_raw(t):
            raise TypeError(f"peer-memory {what} needs a contiguous CUDA tensor on this device")
        stream = self._p2p_stream((peer, send))
        stream.wait_stream(torch.cuda.current_stream(self.device))
        raw = t.view(-1).view(torch.uint8)
        with torch.cuda.stream(stream):
            buf = raw if raw.data_ptr() % 16 == 0 else (raw.clone() if send else torch.empty_like(raw))
            if send:
                self.C.p2p_send(self.p2p.ptrs, self.p2p.sig_ptrs, buf, peer, self.rank, self.world)
            else:
                self.C.p2p_recv(self.p2p.ptrs, self.p2p.sig_ptrs, buf, peer, self.rank, self.world)
                if buf is not raw:
                    raw.copy_(buf)
        t.record_stream(stream)                                # t's memory is not reused while the transfer runs
        done = torch.cuda.Event()
        done.record(stream)
        return P2PWork(done, self.device)

    def _p2p_stream(self, key) -> torch.cuda.Stream:
        """The stream of a (peer, direction) pair, or of a batch's set of pairs: a CUDA stream of its own, created on first
        use, never one of torch's pooled ones (two of those can be one CUDA stream)."""
        stream = self._p2p_streams.get(key)
        if stream is None:
            stream = torch.cuda.ExternalStream(self.C.stream_create(self.device.index), device=self.device)
            self._p2p_streams[key] = stream
        return stream

    def batch_p2p_(self, ops) -> List["P2PWork"]:
        """Every transfer of ``ops`` -- ``[(send, tensor, global peer)]`` -- in one kernel launch (torch's
        ``batch_isend_irecv``); one :class:`P2PWork` per op, all on the batch's completion event, as NCCL's coalesced works.

        Messages of a pair match in issue order, whether either side uses batches or single ``isend_`` / ``irecv_``: the
        batch waits for the current stream and for the streams of every (peer, direction) it touches, and those streams
        wait for the batch before their next transfer.  It runs on a stream of its own per set of pairs, so it is only ever
        queued behind a batch with exactly its pairs, which it would have to follow anyway.  A list is never split: a batch
        that sends more than a pair's mailbox holds before it receives completes only because all its transfers run at once.
        Unaligned tensors go through aligned scratch copies on the batch's stream.  Raises before any launch for a peer
        equal to this rank, a peer outside the world, a tensor this world cannot take, or more ops than one launch holds."""
        ops = [(bool(send), t, peer_rank) for send, t, peer_rank in ops]
        cap = self.C.p2p_batch_capacity()
        if len(ops) > cap:
            raise ValueError(f"batch_isend_irecv: at most {cap} peer-memory ops per batch, got {len(ops)}")
        local = [(send, t, self.local_rank(peer_rank)) for send, t, peer_rank in ops]
        for (send, t, peer), (_, _, peer_rank) in zip(local, ops):
            if peer == self.rank:
                raise ValueError(f"batch_isend_irecv: rank {peer_rank} cannot {'send' if send else 'recv'} to itself")
        for send, t, _ in local:
            if not self.supports_raw(t):
                raise TypeError(f"peer-memory {'send' if send else 'recv'} needs a contiguous CUDA tensor on this device")
        pairs = sorted({(peer, send) for send, _, peer in local})
        stream = self._p2p_stream(("batch",) + tuple(pairs))
        stream.wait_stream(torch.cuda.current_stream(self.device))
        for key in pairs:
            stream.wait_stream(self._p2p_stream(key))          # earlier transfers of these pairs come first
        with torch.cuda.stream(stream):
            launch, back = [], []
            for send, t, peer in local:
                raw = t.view(-1).view(torch.uint8)
                buf = raw if raw.data_ptr() % 16 == 0 else (raw.clone() if send else torch.empty_like(raw))
                launch.append((send, buf, peer))
                if not send and buf is not raw:
                    back.append((raw, buf))
            self.C.p2p_batch(self.p2p.ptrs, self.p2p.sig_ptrs, launch, self.rank, self.world)
            for raw, buf in back:
                raw.copy_(buf)
        for _, t, _ in local:
            t.record_stream(stream)                            # no tensor's memory is reused while the batch runs
        done = torch.cuda.Event()
        done.record(stream)
        for key in pairs:
            self._p2p_streams[key].wait_event(done)            # later transfers of these pairs come after it
        return [P2PWork(done, self.device) for _ in local]

    def _staging_for(self, dtype, nbytes: int) -> SymmHandle:
        st = self._staging.get(dtype)
        if st is None or st.nbytes < nbytes + 2048:
            st = self.alloc_bytes(max(nbytes + 2048, 1 << 20) * (1 if st is None else 2))
            self._staging[dtype] = st
        return st

    def barrier(self, handle: Optional[SymmHandle] = None):
        """Device-side barrier over the world (flag kernel on the current stream; no host synchronisation)."""
        hd = handle or self._staging_for(torch.float32, 1 << 20)
        if self.world > 1:
            self.C.barrier(hd.sig_ptrs, self.rank, self.world)

    def describe(self) -> dict:
        """What was negotiated at setup (mapping mode, multicast, thresholds) -- recorded in bench / sweep outputs."""
        return {"world": self.world, "rank": self.rank, "mode": self.mode, "multicast": self.multicast,
                "granularity": self.gran, "nvls_error": self.nvls_error, "ll_max": self.ll_max,
                "oneshot_max": self.oneshot_max, "nvls_min": self.nvls_min, "table_world": self.table_world}

    def destroy(self):
        """Unmap and release every symmetric allocation of this world (idempotent; called by ``launch.shutdown``)."""
        try:
            torch.cuda.synchronize(self.device)
        except Exception:
            pass
        if self._sock is not None:
            try:
                self._sock.close()
            except Exception:
                pass
            self._sock = None
        # mappings are reclaimed with the process; explicit unmap keeps long-lived jobs tidy
        for hd in self._handles:
            try:
                if hd._mode == "vmm":
                    for p in hd.base_ptrs:
                        self.C.symm_unmap(p, hd.size)
                    if hd.mc_base:
                        self.C.symm_unmap(hd.mc_base, hd.size)
                    for h in hd._mem_handles:
                        self.C.symm_release(h)
                else:
                    for r, p in enumerate(hd.base_ptrs):
                        (self.C.ipc_free if r == self.rank else self.C.ipc_close)(p)
            except Exception:
                pass
        self._handles.clear()
        self._staging.clear()
        self.p2p = None
        for st in self._p2p_streams.values():
            try:
                self.C.stream_destroy(st.cuda_stream)
            except Exception:
                pass
        self._p2p_streams.clear()


def init_world(group=None, **kw) -> SymmWorld:
    """Collective over ``group`` (world if None): build (or return) its symmetric world."""
    key = group
    w = _WORLDS.get(key)
    if w is None:
        w = _WORLDS[key] = SymmWorld(group, **kw)
    return w


def lookup_world(group=None) -> Optional[SymmWorld]:
    """The symmetric world already built over ``group`` (``None`` = default group), or ``None``."""
    return _WORLDS.get(group)


def destroy_all():
    """Tear down every symmetric world of this process."""
    for w in list(_WORLDS.values()):
        w.destroy()
    _WORLDS.clear()
