"""Bit-exact model of the all-reduce and reduce for the dtypes beyond fp32 / bf16 (csrc/allreduce.cu lane types): fp16,
fp64, int8, uint8, int32, int64 and bool.  It builds on tests/comm_model.py (launch geometry) and tests/collectives_model.py
(the fp32 fold and IEEE maximum / minimum), and is shared by tests/test_gpu_reduce_dtypes_emulated.py and the CPU test
tests/test_reduce_dtypes_model.py.

* The wire dtype is the local dtype: no scale, no conversion.
* fp16: the fp32 fold of collectives_model (identity, then every term in rank order; IEEE maximum / minimum) rounded once,
  RN-even, to fp16.  A NaN result is 0x7FFF.  PRODUCT runs under --use_fast_math, so, as for fp32, inputs keep every
  partial product clear of the fp32 subnormal range.
* fp64: the same fold in fp64.  MAX / MIN return 0x7FFFFFFFFFFFFFFF for a NaN result; the payload of a NaN that an fp64 add
  or multiply produces is the hardware's, so the checker takes any NaN for any NaN there (``nan_any``).
* int8, uint8, int32, int64: two's-complement SUM and PRODUCT mod 2^bits, signed or unsigned MAX / MIN.
* bool: the uint8 ops on 0 / 1 bytes; a SUM is a MAX (parallel/symm.py maps it, as torch's NCCL process group does).
* Reduce (root >= 0) and the symmetric buffers follow collectives_model.reduce_model: the root's output is the result, every
  other output is left as it was; staged one-shot and two-shot copy src into the buffer, and two-shot pushes each result slice
  to every storing rank's buffer.

Every function takes what each output and symmetric buffer held before the call and returns what they hold after it, whole
(sentinels behind the message included).
"""
import math

import torch

import collectives_model as CM
import comm_model as M

SUM, PRODUCT, MAX, MIN = CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN
DTYPES = [torch.float16, torch.float64, torch.int8, torch.uint8, torch.int32, torch.int64, torch.bool]
CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.float64: 3, torch.int8: 4, torch.uint8: 5,
         torch.int32: 6, torch.int64: 7, torch.bool: 8}
NAMES = {torch.float16: "fp16", torch.float64: "fp64", torch.int8: "int8", torch.uint8: "uint8", torch.int32: "int32",
         torch.int64: "int64", torch.bool: "bool"}
F16_NAN = 0x7FFF
F64_NAN = 0x7FFFFFFFFFFFFFFF
_BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def elems_per_vec(dtype: torch.dtype) -> int:
    return 16 // torch.empty((), dtype=dtype).element_size()


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(_BITS[t.element_size()])


def as_bytes(t: torch.Tensor) -> torch.Tensor:
    """A bool tensor as its uint8 bytes (torch's bool copies turn any nonzero byte into 1, which would hide a sentinel)."""
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def kernel_op(op: int, dtype: torch.dtype) -> int:
    """The op the kernels run: a bool SUM is a MAX."""
    return MAX if dtype == torch.bool and op == SUM else op


def _f64_minmax(op: int, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    ia, ib = a.view(torch.int64), b.view(torch.int64)
    r = torch.where(a > b, a, b) if op == MAX else torch.where(a < b, a, b)
    r = torch.where(a == b, (ia & ib if op == MAX else ia | ib).view(torch.float64), r)
    nan = torch.tensor(F64_NAN, dtype=torch.int64).view(torch.float64)
    return torch.where(torch.isnan(a) | torch.isnan(b), nan, r)


def fold(op: int, terms: list, fault: str = None) -> torch.Tensor:
    """The reduction of one element position over the ranks' terms, in the terms' dtype.  ``fault`` plants a known bug
    (tests/test_reduce_dtypes_model.py shows the checker catches each): "minmax_sign" (signed and unsigned MAX / MIN
    swapped), "saturate" (a saturating add), "f16_every_term" (fp16 rounded after every term), "f64_via_f32" (fp64 folded
    through fp32), "bool_wrap" (a bool SUM as a wrapping add), "lost_nan" (MAX / MIN that ignore a NaN term)."""
    dtype = terms[0].dtype
    if dtype == torch.bool:
        u = [t.view(torch.uint8) for t in terms]
        if fault == "bool_wrap" and op == SUM:
            return fold(SUM, u).view(torch.bool)
        return fold(kernel_op(op, dtype), u, fault).view(torch.bool)
    if dtype == torch.float16:
        if fault == "f16_every_term":
            acc = torch.full_like(terms[0], CM.IDENTITY[op], dtype=torch.float32)
            for t in terms:
                acc = CM.combine(op, acc, t.float()).half().float()
        elif fault == "lost_nan" and op in (MAX, MIN):
            acc = torch.stack([t.float() for t in terms]).nan_to_num(nan=-math.inf if op == MAX else math.inf,
                                                                     posinf=math.inf, neginf=-math.inf)
            acc = CM.fold(op, list(acc))
        else:
            acc = CM.fold(op, [t.float() for t in terms])
        out = acc.to(torch.float16)
        return torch.where(torch.isnan(acc), torch.tensor(F16_NAN, dtype=torch.int16).view(torch.float16), out)
    if dtype == torch.float64:
        if fault == "f64_via_f32":
            return CM.fold(op, [t.float() for t in terms]).double()
        acc = torch.full_like(terms[0], CM.IDENTITY[op])
        for t in terms:
            if fault == "lost_nan" and op in (MAX, MIN):
                t = t.nan_to_num(nan=-math.inf if op == MAX else math.inf, posinf=math.inf, neginf=-math.inf)
            acc = acc + t if op == SUM else acc * t if op == PRODUCT else _f64_minmax(op, acc, t)
        return acc
    if fault == "minmax_sign" and op in (MAX, MIN) and dtype in (torch.int8, torch.uint8):
        terms = [t.view(torch.uint8 if dtype == torch.int8 else torch.int8) for t in terms]
        return (torch.stack(terms).amax(0) if op == MAX else torch.stack(terms).amin(0)).view(dtype)
    if op in (MAX, MIN):
        s = torch.stack(terms)
        return s.amax(0) if op == MAX else s.amin(0)
    acc = torch.full_like(terms[0], 0 if op == SUM else 1, dtype=torch.int64)
    for t in terms:
        acc = acc + t.long() if op == SUM else acc * t.long()
        if fault == "saturate" and op == SUM:
            info = torch.iinfo(dtype)
            acc = acc.clamp(info.min, info.max)
    return acc.to(dtype)                               # truncation: the wrap mod 2^bits


def reduce_model(variant: int, op: int, xs: list, mode: str, root: int, out_before: list, buf_before: list,
                 fault: str = None) -> dict:
    """All-reduce (root -1) or reduce of the locals ``xs`` (n elements each, one dtype).  ``mode``: "inplace" (the output is
    the symmetric buffer), "staged" (src and dst) or "alias" (src is dst).  ``out_before`` / ``buf_before``: each rank's
    output and symmetric buffer before the call, as long as the tensors the test allocated (bool ones as uint8, see
    :func:`as_bytes`)."""
    world, n = len(xs), xs[0].numel()
    result = as_bytes(fold(op, xs, fault))
    xs = [as_bytes(x) for x in xs]
    outs, bufs = [o.clone() for o in out_before], [b.clone() for b in buf_before]
    for r in range(world):
        stores = root < 0 or r == root
        if mode != "inplace":
            if variant in (M.ONESHOT, M.TWOSHOT):
                bufs[r][:n] = xs[r]                                           # the staging copy of src
            if variant == M.TWOSHOT and stores:
                bufs[r][:n] = result                                          # every reduced slice is pushed here
            if stores:
                outs[r][:n] = result
        else:
            if stores:
                bufs[r][:n] = result
            outs[r] = bufs[r]
    return {"out": outs, "buf": bufs, "result": result}


def nan_any(op: int, dtype: torch.dtype) -> bool:
    """May a NaN result have any payload?  Only where an fp64 add or multiply makes it."""
    return dtype == torch.float64 and op in (SUM, PRODUCT)


def first_mismatch(got: list, want: list, any_nan: bool = False):
    """First (rank, element, got bits, want bits) where the bit patterns differ, or None; with ``any_nan`` any NaN equals
    any NaN."""
    for r, (g, w) in enumerate(zip(got, want)):
        g = g.detach().cpu()
        assert g.dtype == w.dtype and g.shape == w.shape, (r, g.dtype, w.dtype, g.shape, w.shape)
        bad = bits(g) != bits(w)
        if any_nan and g.is_floating_point():
            bad &= ~(torch.isnan(g) & torch.isnan(w))
        if bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            mask = (1 << (8 * g.element_size())) - 1
            return r, i, int(bits(g)[i]) & mask, int(bits(w)[i]) & mask
    return None


def assert_bits_equal(what: str, got: list, want: list, any_nan: bool = False):
    m = first_mismatch(got, want, any_nan)
    if m is not None:
        r, i, gb, wb = m
        raise AssertionError(f"{what}: rank {r}, element {i}: got 0x{gb:x}, model 0x{wb:x}")


# ------------------------------------------------------------------------------------------------------------ inputs
def make_inputs(op: int, dtype: torch.dtype, world: int, n: int, seed: int) -> list:
    """Per-rank locals of ``dtype`` with the cases that tell the semantics apart:

    * integers: random bits, the maximum on every rank (int8 127 + 127 wraps), 2^63 - 1 on rank 0 and 1 on the others
      (int64), -1 / 255 bytes on some ranks (signed and unsigned MAX differ), and products of random terms that wrap;
    * bool: random 0 / 1 bytes, all-zero and all-one positions;
    * fp16: normals, fp32 sums that are fp16 ties (1 on rank 0, 2^-11 on the others: rounding once and after every term
      differ at three ranks and more), 60000 on every rank (the sum overflows to Inf), +-0 mixes, +-Inf on one rank, NaN
      on one rank;
    * fp64: normals, +-0 mixes, +-Inf on one rank, NaN on one rank, and terms whose sum fp32 would round.
    PRODUCT terms are drawn from [0.5, 2) with random signs (no partial product of up to 8 terms leaves fp16's or fp32's
    normal range), plus +-0 and +-Inf on one rank (so no 0 x Inf) and NaN on one rank."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.arange(n)
    xs = []
    for r in range(world):
        if dtype == torch.bool:
            x = torch.rand(n, generator=g) < 0.5
            x = torch.where(idx % 13 == 1, torch.zeros_like(x), x)
            x = torch.where(idx % 13 == 2, torch.ones_like(x), x)
        elif not dtype.is_floating_point:
            info = torch.iinfo(dtype)
            x = torch.randint(info.min, info.max, (n,), generator=g, dtype=torch.int64)
            x = torch.where(idx % 17 == 3, torch.full_like(x, info.max), x)
            x = torch.where(idx % 17 == 4, torch.full_like(x, info.max if r == 0 else 1), x)
            x = torch.where(idx % 17 == 5, torch.full_like(x, -1 if dtype != torch.uint8 else 255), x)
            x = torch.where((idx % 17 == 6) & (r % 2 == 1), torch.full_like(x, 1), x)
            if op == PRODUCT:
                x = torch.where(idx % 17 == 7, torch.full_like(x, 3), x)
            x = x.to(dtype)
        else:
            if op == PRODUCT:
                x = (torch.rand(n, generator=g, dtype=torch.float64) * 1.5 + 0.5) * \
                    torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
                x = torch.where((idx % 97 == 11) & ((idx // 97) % world == r), torch.full_like(x, -math.inf), x)
                x = torch.where((idx % 89 == 13) & (idx % 97 != 11), torch.full_like(x, -0.0 if r % 2 else 0.0), x)
            else:
                x = torch.randn(n, generator=g, dtype=torch.float64) * 4
                x = torch.where(idx % 64 == 5, torch.full_like(x, -0.0), x)
                x = torch.where(idx % 61 == 9, torch.full_like(x, -0.0 if r % 2 else 0.0), x)
                x = torch.where(idx % 67 == 17, torch.full_like(x, 0.0 if r == world // 2 else -0.0), x)
                inf = torch.where((idx // 251) % 2 == 0, torch.full_like(x, math.inf), torch.full_like(x, -math.inf))
                x = torch.where((idx % 251 == 7) & ((idx // 251) % world == r), inf, x)
                if dtype == torch.float16:
                    x = torch.where(idx % 16 == 3, torch.full_like(x, 1.0 if r == 0 else 2.0 ** -11), x)
                    x = torch.where(idx % 71 == 23, torch.full_like(x, 60000.0), x)
                else:
                    x = torch.where(idx % 16 == 3, torch.full_like(x, 1.0 if r == 0 else 2.0 ** -30), x)
            x = torch.where((idx % 53 == 29) & ((idx // 53) % world == r), torch.full_like(x, math.nan), x)
            x = x.to(dtype)
        xs.append(x)
    return xs
