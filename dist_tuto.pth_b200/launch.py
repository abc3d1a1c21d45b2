"""Launcher + rendezvous (layers L0/L1 of the tutorial).

Parity map (reference = /root/reference):
  * ``init_processes(rank, size, fn, backend)``   train_dist.py:130-135, gloo.py:50-55,
                                                  allreduce.py:49-55, ptp.py:30-35, tuto.md:31-36
  * fork-N-processes ``__main__`` launcher        train_dist.py:138-147, tuto.md:39-48
  * init methods env:// / file:// / tcp://        tuto.md:421-457
  * backends tcp / gloo / mpi                     tuto.md:363-398

What is different on purpose (GPU-first, fixes defect D8):
  * one process per GPU; ``backend="b200"`` (alias of nccl + our symmetric
    peer-memory world) binds ``cuda:LOCAL_RANK`` before the group is created,
    bootstraps NCCL for p2p and exchanges peer-memory handles over the store;
  * the launcher propagates child tracebacks and exit codes, kills the
    survivors when one rank dies, supports a join timeout, and every child
    tears its process group down (the reference ``join()``s forever);
  * ``backend="tcp"`` (removed from torch) maps to gloo; ``backend="mpi"``
    means "rank/size come from the external launcher" (mpirun / torchrun /
    srun environment), which keeps the tutorial's MPI recipe
    ``init_processes(0, 0, run, backend='mpi')`` (tuto.md:393-398) working.
"""
from __future__ import annotations

import datetime as _dt
import os
import socket
import sys
import time
import traceback
import warnings
from typing import Callable, Optional

import torch
import torch.distributed as dist

__all__ = ["init_processes", "init_process", "launch", "init_from_env", "shutdown",
           "find_free_port", "resolve_backend", "external_rank_size", "LaunchError"]

DEFAULT_ADDR = "127.0.0.1"   # train_dist.py:132
DEFAULT_PORT = 29500         # train_dist.py:133
_RANK_VARS = ("RANK", "OMPI_COMM_WORLD_RANK", "PMI_RANK", "PMIX_RANK", "SLURM_PROCID")
_SIZE_VARS = ("WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "SLURM_NTASKS")
_LOCAL_VARS = ("LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "MPI_LOCALRANKID", "SLURM_LOCALID")


class LaunchError(RuntimeError):
    """A child rank failed (carries rank, exit code and the child's traceback)."""

    def __init__(self, rank, exitcode, tb=""):
        self.rank, self.exitcode, self.child_traceback = rank, exitcode, tb
        super().__init__(f"rank {rank} exited with code {exitcode}\n{tb}".rstrip())


def find_free_port(addr: str = DEFAULT_ADDR) -> int:
    """A currently free TCP port on ``addr`` (the reference hard-codes 29500, train_dist.py:133)."""
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        s.bind((addr, 0))
        return s.getsockname()[1]


def _first_env(names):
    for n in names:
        v = os.environ.get(n)
        if v not in (None, ""):
            return int(v)
    return None


def external_rank_size():
    """(rank, size, local_rank) supplied by mpirun / torchrun / srun, or Nones."""
    return _first_env(_RANK_VARS), _first_env(_SIZE_VARS), _first_env(_LOCAL_VARS)


def resolve_backend(backend: str, want_cuda: Optional[bool] = None):
    """Map a tutorial backend name to (torch backend string, use_cuda, use_symm).

    tcp -> gloo (the THD TCP channel no longer exists, SURVEY §2.4);
    mpi -> gloo/nccl with rank+size taken from the environment;
    b200 -> nccl for plumbing + symmetric peer-memory world for the hot path."""
    b = (backend or "gloo").lower()
    cuda_ok = torch.cuda.is_available()
    if b == "tcp":
        warnings.warn("backend 'tcp' was removed from torch.distributed; using 'gloo'", stacklevel=3)
        return "gloo", False, False
    if b == "gloo":
        use_cuda = bool(want_cuda) and cuda_ok
        return "gloo", use_cuda, False
    if b == "mpi":
        if dist.is_mpi_available():
            return "mpi", bool(want_cuda) and cuda_ok, False
        use_cuda = cuda_ok if want_cuda is None else (want_cuda and cuda_ok)
        return ("cpu:gloo,cuda:nccl" if use_cuda else "gloo"), use_cuda, False
    if b in ("nccl", "b200", "nvlink"):
        if not cuda_ok:
            raise RuntimeError(f"backend '{backend}' needs a CUDA device (one process per GPU)")
        return "cpu:gloo,cuda:nccl", True, b != "nccl"
    raise ValueError(f"unknown backend '{backend}' (expected tcp|gloo|mpi|nccl|b200)")


def _init_method(init_method, master_addr, master_port):
    if init_method in (None, "env://"):
        os.environ["MASTER_ADDR"] = str(master_addr)
        os.environ["MASTER_PORT"] = str(master_port)
        return "env://"
    if init_method.startswith(("file://", "tcp://")):
        if "[ff" in init_method.lower():
            raise ValueError("multicast tcp:// rendezvous (tuto.md:450-457) no longer exists in torch; "
                             "use tcp://ip:port, file:// or env://")
        return init_method
    raise ValueError(f"unsupported init_method '{init_method}'")


def init_processes(rank: int, size: int, fn: Callable[[int, int], object], backend: str = "gloo", *,
                   master_addr: str = DEFAULT_ADDR, master_port: int = DEFAULT_PORT,
                   init_method: Optional[str] = None, group_name: str = "",
                   timeout_s: float = 600.0, device: Optional[int] = None,
                   symmetric: Optional[bool] = None, teardown: bool = True):
    """Initialise the distributed environment, then run ``fn(rank, size)``.

    Same call shape and defaults as the reference (train_dist.py:130-135):
    ``MASTER_ADDR=127.0.0.1``, ``MASTER_PORT=29500``, env:// rendezvous.
    With ``backend='mpi'`` (or ``size == 0``) rank/size/local-rank are read
    from the launcher environment (allreduce.py:49-54, tuto.md:393-398).
    Returns whatever ``fn`` returns."""
    e_rank, e_size, e_local = external_rank_size()
    if (backend or "").lower() == "mpi" or size in (0, None):
        if e_rank is None or e_size is None:
            if size in (0, None):
                raise RuntimeError("backend 'mpi'/size=0 needs RANK/WORLD_SIZE (or OMPI_*/PMI_*/SLURM_*) "
                                   "from an external launcher")
        else:
            rank, size = e_rank, e_size
            master_addr = os.environ.get("MASTER_ADDR", master_addr)
            master_port = int(os.environ.get("MASTER_PORT", master_port))
    tbackend, use_cuda, use_symm = resolve_backend(backend)
    if symmetric is not None:
        use_symm = bool(symmetric) and use_cuda
    if use_cuda:
        if device is None:
            device = e_local if e_local is not None else rank
            device %= max(1, torch.cuda.device_count())
        torch.cuda.set_device(device)
    method = _init_method(init_method, master_addr, master_port)
    kw = dict(backend=tbackend, init_method=method, rank=rank, world_size=size,
              timeout=_dt.timedelta(seconds=timeout_s))
    if group_name:
        kw["group_name"] = group_name
    if use_cuda and "nccl" in tbackend:
        kw["device_id"] = torch.device("cuda", device)
    try:
        dist.init_process_group(**kw)
    except TypeError:  # older/newer torch without device_id/group_name
        kw.pop("device_id", None)
        kw.pop("group_name", None)
        dist.init_process_group(**kw)
    try:
        if use_symm:
            from .parallel import hier, symm
            if _one_node():
                symm.init_world()                  # one NVSwitch domain: every GPU maps every other GPU's memory
            else:
                hier.init_hier_world()             # several machines: peer memory inside each, NCCL rails across
        return fn(rank, size)
    finally:
        if teardown:
            shutdown()


init_process = init_processes  # BASELINE.json spelling


def _one_node() -> bool:
    """Collective: do all ranks of the default group sit on one machine?"""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return True
    from .parallel.hier import hostname
    hosts = [None] * dist.get_world_size()
    dist.all_gather_object(hosts, hostname())
    return len(set(hosts)) == 1


def assert_one_node(backend: str = "b200") -> None:
    """Collective: the peer-memory world maps every GPU's memory into every process, which only exists inside one
    NVSwitch domain (one machine).  Fail with a clear message instead of a socket timeout deep in the setup."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    hosts = [None] * dist.get_world_size()
    dist.all_gather_object(hosts, socket.gethostname())
    if len(set(hosts)) > 1:
        raise RuntimeError(f"backend '{backend}' builds a symmetric peer-memory world over NVSwitch, which spans ONE machine; "
                           f"this job runs on {sorted(set(hosts))}.  Use backend='nccl' (or 'gloo') across machines.")


def init_from_env(fn: Callable[[int, int], object], backend: str = "b200", **kw):
    """torchrun / mpirun entry: rank, size and local rank come from the environment."""
    rank, size, _ = external_rank_size()
    if rank is None or size is None:
        rank, size = 0, 1
        kw.setdefault("master_port", find_free_port())
    else:
        kw.setdefault("master_addr", os.environ.get("MASTER_ADDR", DEFAULT_ADDR))
        kw.setdefault("master_port", int(os.environ.get("MASTER_PORT", DEFAULT_PORT)))
    return init_processes(rank, size, fn, backend, **kw)


def shutdown():
    """Tear down symmetric worlds and the process group (idempotent)."""
    try:
        from .parallel import symm
        symm.destroy_all()
    except Exception:
        pass
    if dist.is_available() and dist.is_initialized():
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def _child(rank, size, fn, backend, opts, err_q):
    try:
        if "OMP_NUM_THREADS" not in os.environ:
            torch.set_num_threads(max(1, (os.cpu_count() or 1) // max(1, size)))
        init_processes(rank, size, fn, backend, **opts)
    except KeyboardInterrupt:
        sys.exit(130)
    except BaseException:
        try:
            err_q.put((time.time(), rank, traceback.format_exc()))
        finally:
            sys.exit(1)


def launch(fn: Callable[[int, int], object], size: int = 2, backend: str = "gloo", *,
           master_addr: str = DEFAULT_ADDR, master_port="auto", join_timeout_s: Optional[float] = None,
           start_method: Optional[str] = None, **opts) -> None:
    """Spawn ``size`` local processes, each running ``init_processes(rank, size, fn, backend)``.

    Equivalent of the reference ``__main__`` blocks (train_dist.py:138-147) with
    failure detection: the first failing rank's traceback is re-raised as
    :class:`LaunchError`, the remaining ranks are terminated, and
    ``join_timeout_s`` bounds the whole run."""
    import torch.multiprocessing as mp
    if master_port in ("auto", None, 0):
        master_port = find_free_port(master_addr)
    if start_method is None:
        start_method = os.environ.get("B200DIST_START_METHOD", "spawn")
    ctx = mp.get_context(start_method)
    err_q = ctx.SimpleQueue()
    opts = dict(opts, master_addr=master_addr, master_port=int(master_port))
    procs = []
    for rank in range(size):
        p = ctx.Process(target=_child, args=(rank, size, fn, backend, opts, err_q), daemon=False)
        p.start()
        procs.append(p)
    deadline = None if join_timeout_s is None else time.monotonic() + join_timeout_s
    failed = None
    try:
        while True:
            alive = False
            for r, p in enumerate(procs):
                p.join(timeout=0.05)
                if p.exitcode is None:
                    alive = True
                elif p.exitcode != 0 and failed is None:
                    failed = (r, p.exitcode)
            if failed is not None or not alive:
                break
            if deadline is not None and time.monotonic() > deadline:
                failed = (-1, "timeout")
                break
    finally:
        if failed is not None:
            for p in procs:
                if p.exitcode is None:
                    p.terminate()
            for p in procs:
                p.join(timeout=5)
                if p.exitcode is None:
                    p.kill()
                    p.join()
    if failed is not None:
        tb, who = "", failed[0]
        tbs = []
        while not err_q.empty():
            tbs.append(err_q.get())
        if tbs:
            tbs.sort()                      # earliest failure first: it is the root cause
            _, who, tb = tbs[0]
            if len(tbs) > 1:
                tb += "".join(f"\n[also failed: rank {r}]\n{t}" for _, r, t in tbs[1:])
        if failed[1] == "timeout":
            raise LaunchError(who, "timeout", f"launch(): ranks still running after {join_timeout_s}s\n{tb}")
        raise LaunchError(who, failed[1], tb)
