"""Bit-exact model of the gather to a root and the scatter from a root (csrc/allreduce.cu), in the style of
tests/collectives_model.py and on top of tests/comm_model.py (launch geometry, the bit checker).  Shared by
tests/test_gpu_scatter_gather_emulated.py and the CPU test tests/test_scatter_gather_model.py.

* Gather and scatter move 16-byte vectors bit for bit, whatever the dtype, with one end fixed at a root, so the model works
  on int32 words (make the inputs with ``collectives_model.make_raw_inputs``).
* Every function takes what each output and symmetric buffer held before the call and returns what they hold after it,
  whole (sentinels behind the message included), so "left as it was" is checked bit for bit too.
"""
import torch

import comm_model as M


def gather_model(variant: int, xs: list, root: int, mode: str, out_before: list, buf_before: list) -> dict:
    """Gather of int32 words to ``root`` (``xs[r]``: rank r's input, seg words): the root's output receives ``cat(xs)``,
    every other output is left as it was.  In place, rank r's input sits at slot r of its buffer.  Staged, a rank stages its
    src at its own slot (one-shot, two-shot) and two-shot pushes every slot to the root only."""
    world, seg = len(xs), xs[0].numel()
    whole = torch.cat(xs)
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        if mode == "inplace":
            bufs[r][r * seg:(r + 1) * seg] = xs[r]
            if r == root:
                bufs[r][:world * seg] = whole
            outs[r] = bufs[r]
            continue
        if variant in (M.ONESHOT, M.TWOSHOT):
            bufs[r][r * seg:(r + 1) * seg] = xs[r]
        if variant == M.TWOSHOT and r == root:
            bufs[r][:world * seg] = whole
        if r == root:
            outs[r][:world * seg] = whole
    return {"out": outs, "buf": bufs}


def ll_scatter_lines(segs: list, root: int) -> list:
    """The data of the LL scatter's lines: ``lines[s][d]`` is what rank s pushes to rank d (d != s).  The root's line to d
    carries segment d; every other rank pushes zeros, the acknowledgements the parity argument needs."""
    world = len(segs)
    zero = torch.zeros_like(segs[0])
    return [[segs[d] if s == root else zero for d in range(world)] for s in range(world)]


def ll_scatter_receive(lines: list, segs: list, rank: int, root: int, keep: int) -> torch.Tensor:
    """What rank ``rank`` stores: the line from rank ``keep`` (the kernel keeps the root's), or its own segment when it is
    that rank and the root (a non-root's own "line" is its zeros)."""
    if keep == rank:
        return segs[rank] if rank == root else torch.zeros_like(segs[0])
    return lines[keep][rank]


def scatter_model(variant: int, xs: list, root: int, mode: str, out_before: list, buf_before: list,
                  keep=None) -> dict:
    """Scatter of int32 words from ``root`` (``xs[r]``: the root's segment for rank r, seg words): output r receives
    ``xs[r]``.  In place, the root's input fills its buffer and rank r receives its segment at slot r of its own buffer.
    Staged, the root stages its src (one-shot, two-shot), two-shot pushes slot r into rank r's buffer, and a non-root's src
    is never read.  LL delivers through ``ll_scatter_receive``; ``keep(rank)`` overrides whose line a rank keeps (planted
    faults only)."""
    world, seg = len(xs), xs[0].numel()
    whole = torch.cat(xs)
    lines = ll_scatter_lines(xs, root)
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        got = ll_scatter_receive(lines, xs, r, root, root if keep is None else keep(r)) if variant == M.LL else xs[r]
        if mode == "inplace":
            if r == root:
                bufs[r][:world * seg] = whole
            bufs[r][r * seg:(r + 1) * seg] = got
            outs[r] = bufs[r]
            continue
        if r == root and variant in (M.ONESHOT, M.TWOSHOT):
            bufs[r][:world * seg] = whole
        if variant == M.TWOSHOT:
            bufs[r][r * seg:(r + 1) * seg] = xs[r]
        outs[r][:seg] = got
    return {"out": outs, "buf": bufs}
