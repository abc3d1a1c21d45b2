"""Bit-exact model of the collectives beyond the SUM all-reduce (csrc/allreduce.cu): the PRODUCT / MAX / MIN reductions,
the reduce to one root, and the raw-bit broadcast and all-gather.  It builds on tests/comm_model.py (wire values, bf16
rounding, launch geometry, the bit checker) and is shared by tests/test_gpu_collectives_emulated.py and the CPU test
tests/test_collectives_model.py.

* Reductions: ``acc = identity``, then ``acc = combine(acc, wire_r)`` for r = 0, 1, ... in fp32 on every rank; SUM then
  multiplies by the fp32 scale, the other ops take none.  Identities: SUM +0, PRODUCT 1, MAX -Inf, MIN +Inf.  MAX and MIN
  are IEEE 754-2019 maximum / minimum: NaN if any term is NaN, and -0 < +0.  The result is rounded to the wire dtype where
  the SUM all-reduce rounds it (comm_model.allreduce_model); only SUM takes fp32 locals over a bf16 wire.
* PRODUCT runs under --use_fast_math (fp32 multiplies flush subnormal results to zero); this model does not, so inputs must
  keep every partial product clear of the subnormal range.
* Reduce (root >= 0): the root's output is the all-reduce's; every other rank's output is left as it was.  Symmetric
  buffers: two-shot pushes each reduced slice to the root only, so the others keep what was staged in them.
* Broadcast and all-gather move 16-byte vectors bit for bit, whatever the dtype, so the model works on int32 words.

Every function takes what each output and symmetric buffer held before the call and returns what they hold after it, whole
(sentinels behind the message included), so "left as it was" is checked bit for bit too.
"""
import math

import torch

import comm_model as M

SUM, PRODUCT, MAX, MIN = 0, 1, 2, 3
OP_NAMES = {SUM: "sum", PRODUCT: "product", MAX: "max", MIN: "min"}
IDENTITY = {SUM: 0.0, PRODUCT: 1.0, MAX: -math.inf, MIN: math.inf}
CANONICAL_NAN = 0x7FFFFFFF                # what max.NaN / min.NaN return for a NaN term


def _f2i(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.int32)


def ieee_maximum(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """IEEE 754-2019 maximum of fp32 tensors: NaN (canonical) if either is NaN; max(-0, +0) = +0."""
    r = torch.where(a > b, a, b)
    r = torch.where(a == b, (_f2i(a) & _f2i(b)).view(torch.float32), r)      # +-0: the sign bit only if both have it
    return torch.where(torch.isnan(a) | torch.isnan(b), torch.tensor(CANONICAL_NAN, dtype=torch.int32).view(torch.float32), r)


def ieee_minimum(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """IEEE 754-2019 minimum of fp32 tensors: NaN (canonical) if either is NaN; min(-0, +0) = -0."""
    r = torch.where(a < b, a, b)
    r = torch.where(a == b, (_f2i(a) | _f2i(b)).view(torch.float32), r)
    return torch.where(torch.isnan(a) | torch.isnan(b), torch.tensor(CANONICAL_NAN, dtype=torch.int32).view(torch.float32), r)


def combine(op: int, acc: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    if op == SUM:
        return acc + t
    if op == PRODUCT:
        return acc * t
    return ieee_maximum(acc, t) if op == MAX else ieee_minimum(acc, t)


def fold(op: int, terms: list, scale: float = 1.0) -> torch.Tensor:
    """The fp32 accumulator of one vector lane, identical on every rank: identity, then every term in rank order."""
    if op == SUM:
        return M.reduce_scaled(terms, scale)
    assert scale == 1.0, "scale applies to SUM only"
    acc = torch.full_like(terms[0], IDENTITY[op], dtype=torch.float32)
    for t in terms:
        acc = combine(op, acc, t.float())
    return acc


def reduce_model(variant: int, op: int, xs: list, wire: torch.dtype, scale: float, mode: str, root: int,
                 out_before: list, buf_before: list) -> dict:
    """All-reduce (root -1) or reduce of the locals ``xs`` (n elements each).  ``mode``: "inplace" (the output is the
    symmetric buffer), "staged" (src and dst) or "alias" (src is dst).  ``out_before`` / ``buf_before``: each rank's output
    and symmetric buffer before the call, as long as the tensors the test allocated."""
    world, n = len(xs), xs[0].numel()
    local = xs[0].dtype
    assert op == SUM or (wire == local and scale == 1.0), "PRODUCT / MAX / MIN: no scale, no fp32 locals over a bf16 wire"
    wires = [M.wire_values(x, wire) for x in xs]
    acc = fold(op, wires, scale)
    wire_rounded = acc.to(wire)
    staged = mode != "inplace"
    result = wire_rounded.to(local) if variant in (M.TWOSHOT, M.NVLS) or local == wire else acc
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        stores = root < 0 or r == root
        if staged:
            if variant in (M.ONESHOT, M.TWOSHOT):
                bufs[r][:n] = wires[r].to(wire)                               # the staging copy of src
            if variant == M.TWOSHOT and stores:
                bufs[r][:n] = wire_rounded                                    # every reduced slice is pushed here
            if stores:
                outs[r][:n] = result
        elif stores:
            bufs[r][:n] = wire_rounded
            outs[r] = bufs[r]
        else:
            outs[r] = bufs[r]
    return {"out": outs, "buf": bufs, "acc": acc}


def broadcast_model(variant: int, xs: list, root: int, mode: str, out_before: list, buf_before: list) -> dict:
    """Broadcast of int32 words: every output receives ``xs[root]``.  Staged, the root stages its src (one-shot, two-shot)
    and two-shot pushes slice s from rank s to every rank; nobody else stages anything."""
    world, n = len(xs), xs[0].numel()
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        if mode == "inplace":
            bufs[r][:n] = xs[root]
            outs[r] = bufs[r]
            continue
        if variant == M.TWOSHOT or (variant == M.ONESHOT and r == root):
            bufs[r][:n] = xs[root]
        outs[r][:n] = xs[root]
    return {"out": outs, "buf": bufs}


def allgather_model(variant: int, xs: list, mode: str, out_before: list, buf_before: list) -> dict:
    """All-gather of int32 words (``xs[r]``: rank r's input, seg words): every output receives ``cat(xs)``.  In place, rank
    r's input sits at slot r of its buffer.  Staged, a rank stages its src at its own slot (one-shot, two-shot), and
    two-shot pushes every slot to every rank."""
    world, seg = len(xs), xs[0].numel()
    whole = torch.cat(xs)
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        if mode == "inplace":
            bufs[r][:world * seg] = whole
            outs[r] = bufs[r]
            continue
        if variant == M.TWOSHOT:
            bufs[r][:world * seg] = whole
        elif variant == M.ONESHOT:
            bufs[r][r * seg:(r + 1) * seg] = xs[r]
        outs[r][:world * seg] = whole
    return {"out": outs, "buf": bufs}


# ------------------------------------------------------------------------------------------------------------ inputs
def make_reduce_inputs(op: int, world: int, n: int, dtype: torch.dtype, seed: int) -> list:
    """Per-rank locals for ``op``: comm_model's normals and specials (bf16 ties, +-0, +-Inf on one rank) plus, for MAX and
    MIN, NaN on exactly one rank at some positions, -0 / +0 mixes across ranks and all-equal lanes.  PRODUCT terms are
    drawn from [0.5, 2) with random signs, so no partial product of up to 8 terms is subnormal, plus +-0 and +-Inf (on
    exactly one rank, so no 0 x Inf) and a NaN on one rank."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.arange(n)
    xs = M.make_inputs(world, n, torch.float32, seed)
    out = []
    for r, x in enumerate(xs):
        if op == PRODUCT:
            mag = torch.rand(n, generator=g) * 1.5 + 0.5
            sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
            x = mag * sign
            x = torch.where((idx % 97 == 11) & ((idx // 97) % world == r), torch.full_like(x, -math.inf), x)
            x = torch.where((idx % 89 == 13) & (idx % 97 != 11), torch.full_like(x, -0.0 if r % 2 else 0.0), x)
        if op in (MAX, MIN):
            x = torch.where(idx % 61 == 9, torch.full_like(x, -0.0 if r % 2 else 0.0), x)           # mixed signs
            x = torch.where((idx % 61 == 10) & ((idx // 61) % 2 == 0), torch.full_like(x, 1.25), x)   # all ranks equal
            x = torch.where(idx % 67 == 17, torch.full_like(x, 0.0 if r == world // 2 else -0.0), x)
        if op != SUM:
            x = torch.where((idx % 53 == 29) & ((idx // 53) % world == r), torch.full_like(x, math.nan), x)
        out.append(x.to(dtype))
    return out


RAW_SPECIALS = [0x80000000, 0x00000000, 0x7FC01234, 0xFFC00001, 0x7F800001, 0x00000001, 0x807FFFFF, 0x7F800000,
                0xFF800000, 0xFFFFFFFF, 0x7FFFFFFF]


def make_raw_inputs(world: int, n: int, seed: int) -> list:
    """Per-rank int32 words: random bits (int64 patterns, so any 16-byte vector), with -0, quiet and signalling NaNs with
    payloads, subnormals, +-Inf and all-ones words at fixed positions.  Every rank's words differ."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.arange(n)
    special = torch.tensor([s - (1 << 32) if s >= 1 << 31 else s for s in RAW_SPECIALS], dtype=torch.int32)
    xs = []
    for r in range(world):
        x = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=g, dtype=torch.int64).to(torch.int32)
        x = torch.where(idx % 7 == 3, special[(idx // 7 + r) % len(special)], x)
        xs.append(x)
    return xs
