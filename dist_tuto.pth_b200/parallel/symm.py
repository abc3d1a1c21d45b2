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

Collectives: ``all_reduce_`` and ``reduce_`` (SUM, PRODUCT, MAX, MIN on fp32 /
bf16), ``broadcast_`` and ``all_gather_`` (raw bytes, any dtype).  Each call
picks its kernel variant with :func:`plan_variant` and never synchronises the
host.
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

__all__ = ["SymmWorld", "SymmHandle", "init_world", "lookup_world", "destroy_all", "VARIANTS", "COLLECTIVES",
           "op_code", "plan_variant"]

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
COLLECTIVES = ("allreduce", "reduce", "broadcast", "allgather")
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
    (``B200DIST_AR_VARIANT``) names a variant, and NVLS falls back to two-shot where it cannot run."""
    if collective not in COLLECTIVES:
        raise ValueError(f"unknown collective {collective!r}")
    if world == 1:
        return 0
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
        """Can ``all_reduce_`` / ``reduce_`` take this tensor (CUDA, this device, fp32/bf16, contiguous)?"""
        return t.is_cuda and t.device == self.device and t.dtype in _DTYPES and t.is_contiguous()

    def pick_variant(self, wire_bytes: int) -> int:
        """Message size -> kernel (0 one-shot, 1 two-shot, 2 NVLS) from the measured thresholds; ``B200DIST_AR_VARIANT``
        forces one."""
        return self.plan("allreduce", 0, wire_bytes)

    def plan(self, collective: str, op: int, nbytes: int) -> int:
        """:func:`plan_variant` with this world's thresholds and ``B200DIST_AR_VARIANT``."""
        return plan_variant(collective, op, nbytes, self.world, self.ll_max, self.oneshot_max, self.nvls_min,
                            self.multicast, os.environ.get("B200DIST_AR_VARIANT"))

    def _launch(self, hd: SymmHandle, bf16: bool, n_vec: int, scale: float, src, dst, variant: Optional[int],
                max_blocks: Optional[int] = None, collective: str = "allreduce", op: int = 0, root: int = -1):
        """One kernel call on ``hd``.  ``n_vec``: 16-byte vectors of the message (of the output for an all-gather, a multiple
        of world there); ``root``: local rank (-1 for the all-to-all collectives)."""
        n_push = n_vec // self.world if collective == "allgather" else n_vec
        v = self.plan(collective, op, n_push * 16) if variant is None else variant
        if v == 2 and (not hd.mc_ptr or collective != "allreduce" or op != 0):
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
        else:
            self.C.allreduce(v, bf16, hd.ptrs, hd.sig_ptrs, hd.mc_ptr, src, dst, n_vec, float(scale), self.rank,
                             self.world, mb, *ll, op, root)
        return v

    def supports_op(self, op) -> bool:
        """Can ``all_reduce_`` / ``reduce_`` run this reduction (SUM, PRODUCT, MAX, MIN)?"""
        return op_code(op) is not None

    def supports_raw(self, t: torch.Tensor) -> bool:
        """Can ``broadcast_`` / ``all_gather_`` take this tensor (CUDA, this device, contiguous, any dtype)?"""
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
        if not self.supports(t):
            raise TypeError("fused all_reduce needs a contiguous CUDA float32/bfloat16 tensor on this device")
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
