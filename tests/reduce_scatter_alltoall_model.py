"""Bit-exact model of the reduce-scatter and the all-to-all (csrc/allreduce.cu segments_pull_kernel / segments_ll_kernel), in
the style of tests/scatter_gather_model.py and tests/reduce_dtypes_model.py.  Shared by
tests/test_gpu_reduce_scatter_alltoall_emulated.py and the CPU test tests/test_reduce_scatter_alltoall_model.py.

* Every rank's input holds world segments of ``seg`` elements.  Reduce-scatter: rank r's output is segment r of the
  reduction over the ranks, folded as the all-reduce folds it (identity, then every rank's term in rank order; fp32 / bf16 /
  fp16 through the fp32 accumulator, rounded once; a bool SUM is a MAX), so it is bit for bit slice r of the all-reduce.
  All-to-all: segment p of rank r's output is segment r of rank p's input, bit for bit (the model works on int32 words).
* Pull stages a given src into the rank's symmetric buffer; LL leaves the buffer alone.  In place (reduce-scatter only) the
  input is the buffer and the result lands at segment r of it.
* LL: ``ll_lines`` is what every line carries (``lines[s][d]``: segment d of rank s's input, pushed to rank d).
* Every function takes what each output and symmetric buffer held before the call and returns what they hold after it,
  whole (sentinels behind the message included).  Bool tensors travel as their uint8 bytes (``RM.as_bytes``).
* ``fault`` / ``keep`` plant known bugs; tests/test_reduce_scatter_alltoall_model.py shows the checker catches each.
"""
import torch

import collectives_model as CM
import comm_model as M
import reduce_dtypes_model as RM

SUM, PRODUCT, MAX, MIN = CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN
DTYPES = [torch.float32, torch.bfloat16] + RM.DTYPES
NAMES = {torch.float32: "fp32", torch.bfloat16: "bf16", **RM.NAMES}


def elems_per_vec(dtype: torch.dtype) -> int:
    return 16 // torch.empty((), dtype=dtype).element_size()


def make_inputs(op: int, dtype: torch.dtype, world: int, n: int, seed: int) -> list:
    """Per-rank inputs of n elements with the cases that tell the semantics apart (collectives_model's for fp32 / bf16,
    reduce_dtypes_model's for the others)."""
    if dtype in (torch.float32, torch.bfloat16):
        return CM.make_reduce_inputs(op, world, n, dtype, seed)
    return RM.make_inputs(op, dtype, world, n, seed)


def fold(op: int, terms: list, fault: str = None) -> torch.Tensor:
    """One segment's reduction over the ranks' terms, in the terms' dtype.  ``fault``: "order" (the terms combined in
    reverse rank order), "bool_wrap" (a bool SUM as a wrapping add: the SUM -> MAX mapping missing)."""
    if fault == "order":
        terms = terms[::-1]
    dtype = terms[0].dtype
    if dtype in (torch.float32, torch.bfloat16):
        return CM.fold(op, [t.float() for t in terms]).to(dtype)
    return RM.fold(op, terms, "bool_wrap" if fault == "bool_wrap" else None)


def segment(x: torch.Tensor, s: int, world: int) -> torch.Tensor:
    seg = x.numel() // world
    return x[s * seg:(s + 1) * seg]


def ll_lines(xs: list) -> list:
    """The data of the LL lines: ``lines[s][d]`` is segment d of rank s's input, which rank s pushes to rank d (d != s;
    ``None`` on the diagonal, where a rank takes its own segment from its input)."""
    world = len(xs)
    return [[segment(xs[s], d, world) if s != d else None for d in range(world)] for s in range(world)]


def reduce_scatter_result(op: int, xs: list, r: int, fault: str = None) -> torch.Tensor:
    """Rank r's output.  ``fault``: also "swap" (ranks 2k and 2k+1 receive each other's segment), "next_slice" (rank r
    reduces segment r + 1)."""
    world = len(xs)
    s = r
    if fault == "swap" and (r ^ 1) < world:
        s = r ^ 1
    elif fault == "next_slice":
        s = (r + 1) % world
    return fold(op, [segment(x, s, world) for x in xs], fault)


def reduce_scatter_model(variant: int, op: int, xs: list, mode: str, out_before: list, buf_before: list,
                         fault: str = None) -> dict:
    """Reduce-scatter of ``xs`` (world x seg elements per rank, one dtype).  ``mode``: "inplace" (the input is the
    symmetric buffer, the output its segment r) or "staged" (src and dst).  Returns the outputs and buffers whole, each
    rank's result, and for LL the lines."""
    world, n = len(xs), xs[0].numel()
    seg = n // world
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    results = []
    for r in range(world):
        res = RM.as_bytes(reduce_scatter_result(op, xs, r, fault))
        results.append(res)
        if mode == "inplace":
            bufs[r][:n] = RM.as_bytes(xs[r])
            bufs[r][r * seg:(r + 1) * seg] = res
            outs[r] = bufs[r]
        else:
            if variant != M.LL:
                bufs[r][:n] = RM.as_bytes(xs[r])                      # the staging copy of src
            outs[r][:seg] = res
    return {"out": outs, "buf": bufs, "result": results, "lines": ll_lines(xs) if variant == M.LL else None}


def alltoall_model(variant: int, xs: list, mode: str, out_before: list, buf_before: list, keep=None) -> dict:
    """All-to-all of int32 words (``xs[r]``: rank r's input, world x seg words): segment p of output r <- segment r of
    ``xs[p]``.  ``mode``: "staged" (src and dst) or "buffer" (the input already is the symmetric buffer, dst given).  LL
    stores at segment p the line from ``keep(r, p)`` (default p; planted faults only)."""
    world, n = len(xs), xs[0].numel()
    seg = n // world
    lines = ll_lines(xs)
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        if mode == "buffer":
            bufs[r][:n] = xs[r]
        elif variant != M.LL:
            bufs[r][:n] = xs[r]                                       # the staging copy of src
        for p in range(world):
            if variant == M.LL:
                q = p if keep is None else keep(r, p)
                got = segment(xs[r], r, world) if q == r else lines[q][r]
            else:
                got = segment(xs[p], r, world)
            outs[r][p * seg:(p + 1) * seg] = got
    return {"out": outs, "buf": bufs, "lines": lines if variant == M.LL else None}


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def stage_ragged(segs: list, slot: int, buf_before: torch.Tensor, fault: str = None) -> torch.Tensor:
    """``SymmWorld``'s ragged path: the uint8 bytes of segment p go to byte ``p * slot`` of the staging buffer.  ``fault``
    "drop_last": the last segment is never staged."""
    buf = buf_before.clone()
    for p, s in enumerate(segs):
        if fault == "drop_last" and p == len(segs) - 1:
            continue
        buf[p * slot:p * slot + s.numel()] = s
    return buf


def ragged_reduce_scatter(op: int, xs: list, dtype: torch.dtype, bufs_before: list, fault: str = None) -> list:
    """What ``SymmWorld.reduce_scatter_`` returns on every rank for a segment that is not a multiple of 16 bytes: every rank
    stages its segments at 16-byte slots, the kernel reduces slot r over the ranks' buffers, rank r copies slot r out."""
    world = len(xs)
    es = torch.empty((), dtype=dtype).element_size()
    nbytes = xs[0].numel() // world * es
    slot = (nbytes + 15) // 16 * 16
    staged = [stage_ragged([RM.as_bytes(segment(x, p, world)).contiguous().view(torch.uint8) for p in range(world)], slot,
                           bufs_before[r], fault) for r, x in enumerate(xs)]
    out = []
    for r in range(world):
        terms = [b[r * slot:r * slot + nbytes].clone().view(torch.uint8 if dtype == torch.bool else dtype) for b in staged]
        if dtype == torch.bool:
            terms = [t.view(torch.bool) for t in terms]
        out.append(fold(op, terms))
    return out
