"""Bit-exact model of the peer-memory communication kernels (csrc/allreduce.cu, csrc/sgd.cu + csrc/sgd_device.cuh), shared by
the emulated-world GPU tests (tests/test_gpu_comm_emulated.py) and by the CPU test that checks the model and shows that the
checker catches planted faults (tests/test_comm_model.py).

The kernels are specified down to the bit, so the model reproduces them exactly from the per-rank inputs:

* wire values: ``wire_r = x_r``, or ``bf16_rn(x_r)`` when the local tensor is fp32 and the wire is bf16 (one RN-even rounding);
* ``acc = ((0 + wire_0) + wire_1) + ...`` in fp32, in rank order on every rank (the LL and push kernels take their own term
  from registers, at position ``rank``), then ONE fp32 multiply by the fp32 scale;
* output rounding per variant: one-shot and LL round to the wire dtype when the output is a wire-dtype buffer and keep fp32
  when the output is an fp32 ``dst`` over a bf16 wire; two-shot always packs the reduced slice to the wire dtype (it is
  pushed to every rank in that form), so an fp32 ``dst`` over a bf16 wire receives bf16-rounded values;
* the SGD exchange: ``g = scale * sum_r grad_r`` (terms bf16-rounded on the push kernel's bf16 wire, own term included; the
  barrier kernel and world 1 never round), ``m = fmaf(mu, m, g)``, ``p = fmaf(-lr, m, p)``.  With ``mu`` and ``lr`` powers of
  two, ``mu*m`` and ``lr*m`` are exact, each fmaf is one correctly rounded fp32 addition, and an fp64 addition rounded to fp32
  is correctly rounded (53 >= 2*24 + 2), so the fp64 model is exact.

The kernels are built with --use_fast_math, which flushes fp32 subnormals to zero; the inputs here stay clear of them.
"""
import math
import os
import re

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dist_tuto.pth_b200", "csrc")

ONESHOT, TWOSHOT, NVLS, LL = 0, 1, 2, 3
VARIANT_NAMES = {ONESHOT: "oneshot", TWOSHOT: "twoshot", NVLS: "nvls", LL: "ll"}
THREADS = 512                   # allreduce.cu kThreads, sgd_device.cuh kSgdThreads
UNROLL = 2                      # allreduce.cu kUnroll (one-shot and two-shot: vectors per thread and pass)
MAX_BLOCKS = 160                # common.cuh B2_MAX_BLOCKS
MAX_RANKS = 8
SIGNAL_WORDS = MAX_BLOCKS * MAX_RANKS + MAX_BLOCKS + 64     # common.cuh B2_SIGNAL_WORDS
EPOCH_WORD0 = MAX_BLOCKS * MAX_RANKS                        # per-block epoch words follow the flag words
LL_CAP_VEC = 4096               # parallel/symm.py: LL inbox capacity per (parity, source), in 16-byte vectors
SGD_MAX_BLOCKS = 64             # sgd.cu: grid of allreduce_sgd = min(64, ceil(n_vec / 512))
CONV2_OFF, CONV2_N = 264, 5000  # sgd_device.cuh sgd_apply_mp: conv2.weight in the flat parameter vector
AUX_N = 13000                   # aux = [w2f 5000 | w2b 8000]


def kernel_constants() -> dict:
    """The launch constants as the CUDA sources define them (so a change there is seen by tests/test_comm_model.py)."""
    common = open(os.path.join(CSRC, "common.cuh")).read()
    ar = open(os.path.join(CSRC, "allreduce.cu")).read()
    sgd = open(os.path.join(CSRC, "sgd_device.cuh")).read()

    def num(src, pat):
        return int(re.search(pat, src).group(1))
    return {"threads": num(ar, r"constexpr int kThreads = (\d+);"), "unroll": num(ar, r"constexpr int kUnroll = (\d+);"),
            "max_blocks": num(common, r"#define B2_MAX_BLOCKS (\d+)"), "max_ranks": num(common, r"#define B2_MAX_RANKS (\d+)"),
            "sgd_threads": num(sgd, r"constexpr int kSgdThreads = (\d+);")}


def elems_per_vec(wire: torch.dtype) -> int:
    return 8 if wire == torch.bfloat16 else 4


# ------------------------------------------------------------------------------------------------------------ geometry
def grid_blocks(variant: int, n_vec: int, world: int, max_blocks: int) -> int:
    """CTAs per rank of one b2_allreduce_launch.  The LL grid is sized by the message alone (a vector's block must not
    depend on the per-call cap, see DESIGN.md); the other variants are capped by ``max_blocks``."""
    if variant == LL:
        return max(1, min(math.ceil(n_vec / THREADS), MAX_BLOCKS))
    cap = max_blocks if 0 < max_blocks <= MAX_BLOCKS else MAX_BLOCKS
    work = n_vec if variant == ONESHOT else n_vec // world
    blocks = math.ceil(work / THREADS)
    if variant in (TWOSHOT, NVLS):
        blocks = (blocks + 1) // 2
    return min(max(blocks, 1), cap)


def sgd_grid_blocks(n_elems: int) -> int:
    return max(1, min(SGD_MAX_BLOCKS, math.ceil(n_elems // 4 / THREADS)))


def ll_block_of(v: int, n_vec: int) -> int:
    """The block of the LL kernel that handles vector ``v`` (grid-stride over the grid of ``grid_blocks``)."""
    return (v // THREADS) % grid_blocks(LL, n_vec, 1, 0)


# ------------------------------------------------------------------------------------------------------------ inputs
def make_inputs(world: int, n_elems: int, dtype: torch.dtype, seed: int, specials: bool = True) -> list:
    """Per-rank local tensors: normals, plus (``specials``) exact bf16 ties (fp32 halfway between two bf16 values, both
    mantissa parities and signs), -0 on every rank at some positions (the sum is +0: the accumulator starts at +0), +0,
    and +-Inf on exactly one rank at some positions (no Inf - Inf, so no NaN)."""
    g = torch.Generator().manual_seed(seed)
    xs = []
    idx = torch.arange(n_elems)
    for r in range(world):
        x = torch.randn(n_elems, generator=g, dtype=torch.float32)
        if specials:
            tie = (x.view(torch.int32) & -65536) | 0x8000          # bf16 truncation of x plus half a bf16 ulp
            x = torch.where(idx % 16 == 3, tie.view(torch.float32), x)
            x = torch.where(idx % 64 == 5, torch.full_like(x, -0.0), x)
            x = torch.where(idx % 64 == 6, torch.zeros_like(x), x)
            inf = torch.where((idx // 251) % 2 == 0, torch.full_like(x, math.inf), torch.full_like(x, -math.inf))
            x = torch.where((idx % 251 == 7) & ((idx // 251) % world == r), inf, x)
        xs.append(x.to(dtype))
    return xs


# ------------------------------------------------------------------------------------------------------------ model
def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 round-to-nearest-even -> fp32 (the kernels' __floats2bfloat162_rn)."""
    return x.float().to(torch.bfloat16).float()


def fp32_scale(scale: float) -> torch.Tensor:
    """The scale as the kernels get it: the binding's double rounded once to fp32."""
    return torch.tensor(scale, dtype=torch.float64).to(torch.float32)


def wire_values(x: torch.Tensor, wire: torch.dtype) -> torch.Tensor:
    """What rank r puts on the wire, as fp32."""
    if wire == torch.bfloat16:
        return bf16_rn(x) if x.dtype == torch.float32 else x.float()
    assert x.dtype == torch.float32, "an fp32 wire needs fp32 locals"
    return x.clone()


def reduce_scaled(terms: list, scale: float) -> torch.Tensor:
    """((0 + t_0) + t_1) + ... in fp32, in rank order, then one fp32 multiply by the fp32 scale."""
    acc = torch.zeros_like(terms[0], dtype=torch.float32)
    for t in terms:
        acc = acc + t.float()
    return acc * fp32_scale(scale)


def allreduce_model(variant: int, xs: list, wire: torch.dtype, scale: float, out_dtype: torch.dtype, staged: bool) -> dict:
    """Expected state after one all-reduce of the locals ``xs`` (one per rank, all the same dtype).

    ``staged``: the kernel got ``src`` and ``dst`` (``out_dtype`` is ``dst``'s); else it ran in place on the symmetric
    buffers (``out_dtype`` is the wire dtype).  Returns ``out`` (what each rank's output holds, in ``out_dtype``) and
    ``buf`` (each rank's symmetric buffer in the wire dtype; None for a buffer the call must leave as it was)."""
    world = len(xs)
    assert wire == out_dtype or (wire == torch.bfloat16 and out_dtype == torch.float32 and staged)
    wires = [wire_values(x, wire) for x in xs]
    acc = reduce_scaled(wires, scale)                                  # fp32, identical on every rank
    wire_rounded = acc.to(wire)
    if variant in (TWOSHOT, NVLS) or out_dtype == wire:
        out = wire_rounded.to(out_dtype)
    else:                                                              # one-shot / LL, fp32 dst over a bf16 wire
        out = acc
    if variant in (TWOSHOT, NVLS):
        bufs = [wire_rounded.clone() for _ in range(world)]            # every slice is pushed to every rank
    elif not staged:
        bufs = [wire_rounded.clone() for _ in range(world)]            # in place: the result is the buffer
    elif variant == ONESHOT:
        bufs = [w.to(wire) for w in wires]                             # the staging copy of src
    else:
        bufs = [None] * world                                          # LL reads src and writes dst directly
    return {"out": [out.clone() for _ in range(world)], "buf": bufs, "acc": acc}


def sgd_model(grads: list, params: torch.Tensor, mom: torch.Tensor, scale: float, mu: float, lr: float,
              bf16_terms: bool):
    """One exchange + momentum SGD step: (params, momentum) after it.  ``bf16_terms``: the push kernel's bf16 wire at
    world > 1 (every term, the own one included, rounded once)."""
    assert is_pow2(mu) and is_pow2(lr), "the fp64 model is exact only for power-of-two mu and lr"
    g = reduce_scaled([bf16_rn(t) if bf16_terms else t for t in grads], scale)
    m = (mu * mom.double() + g.double()).float()
    p = (params.double() - lr * m.double()).float()
    return p, m


def bucket_model(bucket: torch.Tensor, n: int, cur: int, zero_grads: bool, two: bool) -> torch.Tensor:
    """One rank's gradient bucket(s) after a step that read bucket ``cur``: with two buckets the current one is left as it
    is and the other one is zeroed; with one bucket that bucket is zeroed (the zeroing only with ``zero_grads``)."""
    b = bucket.clone()
    if zero_grads:
        z = (cur ^ 1) if two else 0
        b[z * n:(z + 1) * n] = 0.0
    return b


def is_pow2(x: float) -> bool:
    return x > 0 and math.frexp(x)[0] == 0.5


def aux_index() -> tuple:
    """For conv2.weight element i (flat offset CONV2_OFF + i): its slots in aux, w2f [ci][ky][kx][co] and w2b
    [co][ky][kx][half][8] (sgd_apply_mp)."""
    i = torch.arange(CONV2_N)
    co, r = i // 250, i % 250
    ci, kk = r // 25, r % 25
    return (ci * 25 + kk) * 20 + co, 5000 + ((co * 25 + kk) * 2 + ci // 5) * 8 + ci % 5


def aux_model(params: torch.Tensor, aux_before: torch.Tensor) -> torch.Tensor:
    w2f, w2b = aux_index()
    aux = aux_before.clone()
    w = params[CONV2_OFF:CONV2_OFF + CONV2_N]
    aux[w2f] = w
    aux[w2b] = w
    return aux


# ------------------------------------------------------------------------------------------------------------ checker
def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def first_mismatch(got: list, want: list, epv: int):
    """First (rank, vector, element, got bits, want bits) where the bit patterns differ (so -0 / +0 and Inf compare; any
    NaN equals any NaN), or None.  ``epv``: elements per 16-byte vector."""
    for r, (g, w) in enumerate(zip(got, want)):
        if w is None:
            continue
        g = g.detach().cpu()
        assert g.dtype == w.dtype and g.shape == w.shape, (r, g.dtype, w.dtype, g.shape, w.shape)
        bad = (_bits(g) != _bits(w)) & ~(torch.isnan(g) & torch.isnan(w))
        if bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            mask = 0xFFFF if g.element_size() == 2 else 0xFFFFFFFF
            return r, i // epv, i, int(_bits(g)[i]) & mask, int(_bits(w)[i]) & mask
    return None


def assert_bits_equal(what: str, got: list, want: list, epv: int):
    m = first_mismatch(got, want, epv)
    if m is not None:
        r, v, i, gb, wb = m
        raise AssertionError(f"{what}: rank {r}, vector {v} (element {i}): got 0x{gb:x}, model 0x{wb:x}")


def fp64_error_bound(xs: list, scale: float, wire: torch.dtype, out_rounded: bool) -> tuple:
    """The fp64 all-reduce of the unrounded locals and the bound any correct fp32 implementation of it meets: W-1 fp32
    additions and one multiply, plus one bf16 rounding per term on a bf16 wire and one of the result when it is packed."""
    world = len(xs)
    s = float(fp32_scale(scale))
    ref = torch.zeros(xs[0].numel(), dtype=torch.float64)
    mag = torch.zeros_like(ref)
    for x in xs:
        ref += x.double()
        mag += x.double().abs()
    ref, mag = ref * s, mag * abs(s)
    bound = mag * (world + 1) * 2.0 ** -24
    if wire == torch.bfloat16:
        bound = bound + mag * 2.0 ** -8
    if out_rounded:
        bound = bound + (ref.abs() + bound) * 2.0 ** -8
    return ref, bound * 1.01


def check_against_fp64(what: str, out: torch.Tensor, xs: list, scale: float, wire: torch.dtype, out_rounded: bool):
    """Sanity net for the model itself: within the bound of the fp64 result where that is finite, equal where it is not."""
    ref, bound = fp64_error_bound(xs, scale, wire, out_rounded)
    o = out.detach().cpu().double()
    fin = torch.isfinite(ref)
    err = (o - ref).abs()
    bad = fin & ~(err <= bound)
    assert not bool(bad.any()), f"{what}: element {int(bad.nonzero()[0, 0])} off the fp64 result by more than its bound"
    nf = ~fin
    assert torch.equal(o[nf].nan_to_num(), ref[nf].nan_to_num()), f"{what}: non-finite results differ from fp64"
