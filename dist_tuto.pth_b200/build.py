"""In-tree build of the native extension ``dist_tuto.pth_b200/_C.so``.

* every ``.cu`` is compiled by nvcc for **sm_90a only**
  (``-gencode arch=compute_90a,code=sm_90a -lineinfo``) -- no torch headers in
  the kernels, so a file takes seconds and cross-compiles without a GPU;
* ``bindings.cpp`` (pybind11 + torch) and the host runtime (``symm_mem.cpp``,
  ``loader.cpp``) are compiled by g++;
* objects are cached under ``csrc/build/`` keyed by a content hash.

``python -m dist_tuto.pth_b200.build`` or ``__graft_entry__.build()``.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
TARGET = os.path.join(HERE, "_C.so")

CU_SOURCES = ["allreduce.cu", "convnet.cu", "convnet_cluster.cu", "sgd.cu", "gemm_tcgen05.cu", "tc_probe.cu", "convnet_batched.cu",
              "convnet_eval.cu"]
CPP_SOURCES = ["symm_mem.cpp", "loader.cpp", "executor.cpp", "bindings.cpp"]
HEADERS = ["common.cuh", "tc_common.cuh", "convnet_args.cuh", "convnet_reduce.cuh", "sgd_device.cuh", "lr_schedule.h", "loader.h", "executor.h"]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _cuda_home() -> str:
    return os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH") or "/usr/local/cuda"


def _hash(paths: List[str], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:16]


def _run(cmd: List[str], log: str) -> None:
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"build step failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")


def build(verbose: bool = True, force: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(OBJ, exist_ok=True)
    cuda = _cuda_home()
    nvcc = os.path.join(cuda, "bin", "nvcc")
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    torch_inc = ce.include_paths()
    py_inc = sysconfig.get_paths()["include"]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", "-Wno-unused-result", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                 "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    incs = [f"-I{p}" for p in torch_inc] + [f"-I{py_inc}", f"-I{cuda}/include", f"-I{CSRC}"]

    jobs, objs = [], []
    for src in CU_SOURCES:
        sp = os.path.join(CSRC, src)
        tag = _hash([sp] + hdrs, " ".join(ARCH + NVCC_FLAGS))
        obj = os.path.join(OBJ, f"{src}.{tag}.o")
        objs.append(obj)
        if force or not os.path.exists(obj):
            jobs.append(([nvcc] + ARCH + NVCC_FLAGS + [f"-I{CSRC}", "-c", sp, "-o", obj], obj + ".log"))
    for src in CPP_SOURCES:
        sp = os.path.join(CSRC, src)
        tag = _hash([sp] + hdrs, " ".join(cxx_flags) + torch.__version__)
        obj = os.path.join(OBJ, f"{src}.{tag}.o")
        objs.append(obj)
        if force or not os.path.exists(obj):
            jobs.append((["g++"] + cxx_flags + incs + ["-c", sp, "-o", obj], obj + ".log"))
    if verbose and jobs:
        print(f"[build] compiling {len(jobs)} object(s) for sm_90a ...", flush=True)
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        list(ex.map(lambda j: _run(*j), jobs))

    link_tag = _hash(objs, "link")
    stamp = os.path.join(OBJ, "link.stamp")
    prev = open(stamp).read().strip() if os.path.exists(stamp) else ""
    if force or jobs or not os.path.exists(TARGET) or prev != link_tag:
        lib_dirs = ce.library_paths() + [os.path.join(cuda, "lib64")]
        tmp_target = f"{TARGET}.tmp{os.getpid()}"
        cmd = ["g++", "-shared", "-o", tmp_target] + objs + [f"-L{d}" for d in lib_dirs] + \
              [f"-Wl,-rpath,{d}" for d in lib_dirs] + \
              ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart", "-lpthread"]
        _run(cmd, os.path.join(OBJ, "link.log"))
        os.replace(tmp_target, TARGET)              # atomic: a concurrent importer sees the old or the new library, never half
        with open(stamp, "w") as f:
            f.write(link_tag)
        if verbose:
            print(f"[build] linked {TARGET}", flush=True)
    # keep only the current objects
    keep = {os.path.basename(o) for o in objs}
    for f in os.listdir(OBJ):
        if f.endswith(".o") and f not in keep:
            os.remove(os.path.join(OBJ, f))
            if os.path.exists(os.path.join(OBJ, f + ".log")):
                os.remove(os.path.join(OBJ, f + ".log"))
    return TARGET


def _expected_objects():
    """(object paths, link tag) the current sources/flags hash to -- without compiling anything."""
    import torch
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", "-Wno-unused-result", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                 "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    objs = []
    for src in CU_SOURCES:
        tag = _hash([os.path.join(CSRC, src)] + hdrs, " ".join(ARCH + NVCC_FLAGS))
        objs.append(os.path.join(OBJ, f"{src}.{tag}.o"))
    for src in CPP_SOURCES:
        tag = _hash([os.path.join(CSRC, src)] + hdrs, " ".join(cxx_flags) + torch.__version__)
        objs.append(os.path.join(OBJ, f"{src}.{tag}.o"))
    return objs


def up_to_date() -> bool:
    """True when ``_C.so`` was linked from objects matching the CURRENT sources, headers and flags (content hashes)."""
    try:
        objs = _expected_objects()
        if not os.path.isfile(TARGET) or not all(os.path.exists(o) for o in objs):
            return False
        stamp = os.path.join(OBJ, "link.stamp")
        return os.path.exists(stamp) and open(stamp).read().strip() == _hash(objs, "link")
    except Exception:
        return False


def ptxas_report() -> str:
    """Registers / spills / smem per kernel, from the cached nvcc logs."""
    out = []
    for f in sorted(os.listdir(OBJ)):
        if f.endswith(".o.log") and ".cu." in f:
            out.append(f"== {f.split('.cu.')[0]}.cu")
            for line in open(os.path.join(OBJ, f)):
                if "Compiling entry" in line or "registers" in line or "spill" in line:
                    out.append(line.rstrip())
    return "\n".join(out)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    if "--report" in sys.argv:
        print(ptxas_report())
