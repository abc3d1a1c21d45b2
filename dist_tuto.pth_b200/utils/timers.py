"""Tracing / profiling helpers (absent from the reference, SURVEY §5).

* :class:`DeviceTimer`   -- CUDA-event timing on the launching stream (falls
  back to ``perf_counter`` on CPU); multi-GPU numbers are reduced with MAX
  over ranks by :func:`max_over_ranks`.
* :class:`PhaseTimers`   -- named phases (fwd/bwd/allreduce/step).
* :func:`nvtx_range`     -- NVTX ranges when CUDA is present, no-op otherwise.
* :class:`ClockSampler`  -- samples ``nvidia-smi`` SM clocks + throttle reasons
  in a background thread during a timed region (B200_PROFILING.md recipe).
* :func:`l2_flush`       -- writes a buffer larger than the L2 (50 MB on an H100).
"""
from __future__ import annotations

import contextlib
import statistics
import subprocess
import threading
import time
from typing import Dict, List, Optional

import torch

__all__ = ["DeviceTimer", "PhaseTimers", "nvtx_range", "ClockSampler", "l2_flush", "max_over_ranks"]


class DeviceTimer:
    """CUDA-event stopwatch on the current stream (``perf_counter`` on CPU)."""

    def __init__(self, device=None):
        self.cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda")
        self._t0 = self._e0 = self._e1 = None

    def start(self):
        if self.cuda:
            self._e0, self._e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self._e0.record()
        else:
            self._t0 = time.perf_counter()
        return self

    def stop(self) -> float:
        """Milliseconds since ``start`` (synchronises)."""
        if self.cuda:
            self._e1.record()
            self._e1.synchronize()
            return self._e0.elapsed_time(self._e1)
        return (time.perf_counter() - self._t0) * 1e3


def max_over_ranks(value: float, device=None) -> float:
    """MAX over ranks of a per-rank time: the number every multi-GPU measurement reports."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    dev = device or ("cuda" if "nccl" in str(dist.get_backend()) and torch.cuda.is_available() else "cpu")
    t = torch.tensor([float(value)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


class PhaseTimers:
    """Named device-timed phases with NVTX ranges: ``with timers.phase('allreduce'): ...``."""

    def __init__(self):
        self.ms: Dict[str, List[float]] = {}

    @contextlib.contextmanager
    def phase(self, name: str):
        t = DeviceTimer().start()
        with nvtx_range(name):
            yield
        self.ms.setdefault(name, []).append(t.stop())

    def summary(self) -> Dict[str, float]:
        return {k: statistics.mean(v) for k, v in self.ms.items()}


@contextlib.contextmanager
def nvtx_range(name: str):
    """NVTX push/pop around a block (no-op without CUDA)."""
    on = torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()


_Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
      "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
      "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    """Background ``nvidia-smi`` sampler; ``summary()`` -> bench.py ``clocks`` key."""

    def __init__(self, gpu_index: int = 0, period_s: float = 0.2):
        self.gpu, self.period = gpu_index, period_s
        self.rows: List[List[str]] = []
        self._stop = threading.Event()
        self._th: Optional[threading.Thread] = None

    def _loop(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={_Q}",
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True,
                                     timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.splitlines()[0].split(",")])
            except Exception:
                pass
            self._stop.wait(self.period)

    def __enter__(self):
        self._th = threading.Thread(target=self._loop, daemon=True)
        self._th.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        if self._th is not None:
            self._th.join(timeout=6)

    def summary(self) -> dict:
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
            except Exception:
                continue
            for nm, v in zip(names, r[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


_L2_BUF = {}


def l2_flush(device=None, nbytes: int = 256 << 20):
    """Overwrite a buffer larger than L2 (50 MB on an H100) so the next kernel starts cold."""
    if not torch.cuda.is_available():
        return
    dev = torch.device(device or torch.cuda.current_device())
    buf = _L2_BUF.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = _L2_BUF[dev] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    buf.fill_(1)
