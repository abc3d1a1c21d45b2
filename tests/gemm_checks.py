"""Checks shared by the wgmma GEMM tests (tests/test_gpu_gemm.py) and by the CPU test that shows they catch planted faults
and that the case table reaches every dispatch path at its edges (tests/test_gemm_checks.py).

* Exact oracle: bf16 operands with integer values in [-4, 4] and an integer fp32 bias in [-64, 64].  Each product is an
  integer of magnitude <= 16, except one planted product of magnitude <= 1024 per planted tie (``int_operands``), so with
  K <= 4096 every partial sum stays below 2^17 in any order: any fp32 accumulator keeping >= 18 significant bits gets the
  exact integer.  fp32 output must equal relu?(A B^T + bias) computed in fp64; bf16 output must equal that rounded to
  nearest even.  Every case carries a planted tie that round-to-nearest-even rounds toward zero (257 between 256 and
  258, say), so a round-half-away or truncating epilogue cannot pass.
* fp64 bound: for randn operands rounded to bf16, |C - R| <= K 2^-22 (sum_k |a_ik b_jk| + |bias_j|), plus 2^-8 |R| for
  bf16 output: four times the worst-case bound of fp32 summation with round to nearest, which leaves room for a
  tensor-core accumulation that truncates.
* Case table: ``cases(S)`` mirrors the dispatch rule of ``b2_gemm_bf16_launch`` on a GPU with S SMs, and
  ``kernel_geometry()`` reads the ring depths, tile widths and dispatch thresholds out of the kernel source, so that
  ``coverage_gaps`` notices when a change to the kernel moves a case off the path or edge it was meant for.
* Guard bands: ``guarded_out`` places the output inside a buffer filled with a sentinel bit pattern, ``guard_faults``
  reports any guard element a store reached.
"""
import os
import re
from collections import namedtuple

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SRC = os.path.join(ROOT, "dist_tuto.pth_b200", "csrc", "gemm_tcgen05.cu")

# epilogues: (bias, relu, bf16 out); rotated over each path's cases so that every combination runs on every path
COMBOS = [(True, False, False), (False, False, True), (True, True, True), (False, True, False),
          (True, False, True), (False, False, False), (True, True, False), (False, True, True)]
M_EDGES = [1, 63, 64, 65, 127, 128, 129, 257]          # one row; warpgroup 2 empty / one row; one tile; a row of tile 2; 3 tiles
ENGINE_B = [1, 3, 2048, 8191]                           # batch sizes of the batched engine's fc1 launches
ENGINE_CALLS = [(64, 320, (True, True, False)),         # fc1 forward into Hrelu: bias, ReLU, fp32 out
                (320, 64, (False, False, True))]        # fc1 data gradient into dP2: no bias, bf16 out
EXISTING = [(128, 64, 64), (256, 50, 320), (1000, 10, 512), (300, 200, 136), (64, 32, 8), (4096, 512, 1024),
            (4096, 256, 512), (2000, 1000, 264), (8192, 1003, 520), (2500, 2048, 2056), (8192, 4096, 4096)]
PATHS = ["bn32", "bn64", "bn128", "persistent"]
KERNEL_NAME = {"bn32": "gemm_bf16_kernel<32>", "bn64": "gemm_bf16_kernel<64>", "bn128": "gemm_bf16_kernel<128>",
               "persistent": "gemm_bf16_persistent_kernel"}
MAX_K = 4096                                            # keeps every partial sum of the integer operands below 2^17

Case = namedtuple("Case", "group M N K bias relu out_bf16 path bn")


# ---------------------------------------------------------------------------------------------------------- geometry
def kernel_geometry(src: str = KERNEL_SRC) -> dict:
    """Tile shape, ring depths and dispatch thresholds of csrc/gemm_tcgen05.cu."""
    with open(src) as f:
        text = f.read()

    def need(pattern):
        m = re.search(pattern, text)
        assert m, f"{pattern!r} not found in {src}"
        return m

    bm, bk = map(int, need(r"constexpr int BM = (\d+), BK = (\d+);").groups())
    st = need(r"struct Cfg \{ static constexpr int STAGES = BN >= (\d+) \? (\d+) : (\d+); \};")
    pbn, pst = map(int, need(r"constexpr int PBN = (\d+), PSTAGES = (\d+);").groups())
    p = need(r"if \(mode && N >= (\d+) && K >= (\d+) && \(long long\)\(\(M \+ (\d+)\) / (\d+)\) \* "
             r"\(\(N \+ (\d+)\) / (\d+)\) >= gemm::sm_count\(\)\)\s*return gemm::launch_persistent")
    assert int(p.group(3)) + 1 == int(p.group(4)) == bm and int(p.group(5)) + 1 == int(p.group(6)) == pbn, \
        "the persistent rule counts tiles of another shape than the kernel's"
    rule = [(int(n), int(bn)) for n, bn in re.findall(r"if \(N <= (\d+)\) return gemm::launch<(\d+)>", text)]
    last = int(need(r"\n  return gemm::launch<(\d+)>\(a, b, c, bias, M, N, K, relu, out_bf16, stream\);").group(1))
    assert rule, "BN dispatch not found"
    st_min, st_big, st_small = map(int, st.groups())
    stages = {bn: (st_big if bn >= st_min else st_small) for bn in [b for _, b in rule] + [last]}
    return {"BM": bm, "BK": bk, "PBN": pbn, "PSTAGES": pst, "p_min_n": int(p.group(1)), "p_min_k": int(p.group(2)),
            "rule": rule, "last": last, "stages": stages}


def tiles(M: int, N: int, geo: dict) -> int:
    return -(-M // geo["BM"]) * -(-N // geo["PBN"])


def dispatch(M: int, N: int, K: int, S: int, geo: dict) -> str:
    """The kernel ``b2_gemm_bf16_launch`` picks on a GPU with S SMs."""
    if N >= geo["p_min_n"] and K >= geo["p_min_k"] and tiles(M, N, geo) >= S:
        return "persistent"
    for n_max, bn in geo["rule"]:
        if N <= n_max:
            return f"bn{bn}"
    return f"bn{geo['last']}"


def num_kb(K: int, geo: dict) -> int:
    return -(-K // geo["BK"])


def _case(group, M, N, K, combo, S, geo):
    path = dispatch(M, N, K, S, geo)
    bn = geo["PBN"] if path == "persistent" else int(path[2:])
    return Case(group, M, N, K, *combo, path, bn)


def bn_edges(geo: dict) -> dict:
    """Per 128xBN path: (the N values at its edges, the num_kb values around its ring depth).
    N: the three smallest N the dispatch sends to the path, BN - 1 and BN; on the widest path also BN + 1 and odd N
    with 3 N-tiles.  num_kb: 1, STAGES - 1, STAGES, STAGES + 1 (the ring wraps once) and 2 STAGES + 1."""
    out, lo = {}, 1
    for n_max, bn in geo["rule"] + [(None, geo["last"])]:
        ns = [lo, lo + 1, lo + 2, bn - 1, bn]
        if n_max is None:
            ns += [bn + 1, 2 * bn + 1, 3 * bn - 1]
        else:
            lo = n_max + 1
        st = geo["stages"][bn]
        out[f"bn{bn}"] = (ns, [1, st - 1, st, st + 1, 2 * st + 1])
    return out


def persistent_edges(S: int, geo: dict) -> dict:
    """Tile counts S, S + 1, 2S + 5 (CTAs run 1, 2 and 3 tiles), num_kb p .. p + PSTAGES - 1 from the first k-loop long
    enough (every residue mod PSTAGES)."""
    kb0 = num_kb(geo["p_min_k"], geo)
    return {"tiles": [S, S + 1, 2 * S + 5], "kb": list(range(kb0, kb0 + geo["PSTAGES"]))}


def cases(S: int, geo: dict = None) -> list:
    """The case table for a GPU with S SMs (see the module docstring)."""
    geo = geo or kernel_geometry()
    bk, out = geo["BK"], []
    for p, (path, (ns, kbs)) in enumerate(bn_edges(geo).items()):
        for i in range(2 * len(kbs)):                      # every num_kb twice: K a multiple of 64, then ragged (K % 64 = 8)
            kb = kbs[i % len(kbs)]
            K = bk * kb if i < len(kbs) else bk * (kb - 1) + 8
            out.append(_case(path, M_EDGES[i % len(M_EDGES)], ns[i % len(ns)], K, COMBOS[(i + p) % len(COMBOS)], S, geo))
    pe = persistent_edges(S, geo)
    kbs = pe["kb"]
    ks = [bk * kb if j == 0 else bk * (kb - 1) + 8 for j, kb in enumerate(kbs)]
    n_choices = [geo["PBN"] + 1, 200, 192, geo["PBN"]]        # odd N with a one-column second tile, ragged tiles, a full one
    m_short = [5, 0, 127, 64, 1, 100, 33, 0]                   # rows missing from the last M-tile
    for i in range(len(COMBOS)):
        T, K, N = pe["tiles"][i % 3], ks[i % len(ks)], n_choices[i % len(n_choices)]
        nt = -(-N // geo["PBN"])
        if T % nt:                                             # odd tile count: one N-tile, odd N
            N, nt = geo["PBN"] - 1, 1
        M = (T // nt) * geo["BM"] - m_short[i]
        out.append(_case("persistent", M, N, K, COMBOS[(i + 3) % len(COMBOS)], S, geo))
    for B in ENGINE_B:
        for N, K, combo in ENGINE_CALLS:
            out.append(_case("engine", B, N, K, combo, S, geo))
    for i, (M, N, K) in enumerate(EXISTING):
        out.append(_case("existing", M, N, K, COMBOS[i % len(COMBOS)], S, geo))
    return out


def coverage_gaps(table: list, S: int, geo: dict = None) -> list:
    """Every coverage condition the table misses on a GPU with S SMs (empty when it meets them all)."""
    geo = geo or kernel_geometry()
    gaps = []
    for c in table:
        if dispatch(c.M, c.N, c.K, S, geo) != c.path:
            gaps.append(f"{c} is dispatched to {dispatch(c.M, c.N, c.K, S, geo)}")
        if c.K > MAX_K or c.K % 8:
            gaps.append(f"{c}: K must be a multiple of 8 and <= {MAX_K}")
    by = {p: [c for c in table if c.path == p] for p in PATHS}
    for p, cs in by.items():
        have = {(c.bias, c.relu, c.out_bf16) for c in cs}
        gaps += [f"{p}: epilogue {e} never runs" for e in COMBOS if e not in have]
    for p, (ns, kbs) in bn_edges(geo).items():
        cs = by[p]
        gaps += [f"{p}: M = {m} never runs" for m in M_EDGES if m not in {c.M for c in cs}]
        gaps += [f"{p}: N = {n} never runs" for n in ns if n not in {c.N for c in cs}]
        gaps += [f"{p}: num_kb = {k} never runs" for k in kbs if k not in {num_kb(c.K, geo) for c in cs}]
        if not any(c.K % geo["BK"] == 8 for c in cs):
            gaps.append(f"{p}: no ragged K")
        if p == f"bn{geo['last']}" and not any(c.N % 2 and -(-c.N // c.bn) >= 2 for c in cs):
            gaps.append(f"{p}: no odd N with two or more N-tiles")
    pe, cs = persistent_edges(S, geo), by["persistent"]
    gaps += [f"persistent: {t} tiles never run" for t in pe["tiles"] if t not in {tiles(c.M, c.N, geo) for c in cs}]
    gaps += [f"persistent: num_kb = {k} never runs" for k in pe["kb"] if k not in {num_kb(c.K, geo) for c in cs}]
    if not any(c.N % geo["PBN"] for c in cs):
        gaps.append("persistent: no ragged N-tile")
    if not any(c.N % 2 for c in cs):
        gaps.append("persistent: no odd N")
    if not any(c.M % geo["BM"] for c in cs):
        gaps.append("persistent: no ragged M")
    for B in ENGINE_B:
        for N, K, combo in ENGINE_CALLS:
            if (B, N, K) + combo not in {(c.M, c.N, c.K, c.bias, c.relu, c.out_bf16) for c in table}:
                gaps.append(f"engine call M={B} N={N} K={K} {combo} missing")
    gaps += [f"shape {s} of the existing test missing" for s in EXISTING if s not in {(c.M, c.N, c.K) for c in table}]
    return gaps


# ---------------------------------------------------------------------------------------------------------- operands
def _tie_values(limit: int = 1 << 17):
    """Positive integers below ``limit`` that lie halfway between two bf16 neighbours: (rounded down by RNE, rounded up)."""
    v = torch.arange(1, limit, dtype=torch.float64)
    down, up = tie_masks(v)
    return v[down].long().tolist(), v[up].long().tolist()


_TIES = None


def _plant(A, B, bias, r, j, k, targets):
    """Set A[r, k] = a in [-4, 4] and B[j, k] = b in [-256, 256] (both exact in bf16) so that element (r, j) of
    A B^T + bias becomes one of ``targets``.  Flips the sign of row r of A first if the rest of the sum is negative."""
    def rest():
        x = int((A[r].long() * B[j].long()).sum()) - int(A[r, k]) * int(B[j, k])
        return x + (int(bias[j]) if bias is not None else 0)
    x = rest()
    if x < 0:
        A[r].neg_()
        x = rest()
    for a in (1, 3, 2, 4, -1, -3, -2, -4):
        for T in targets:
            if (T - x) % a == 0 and abs((T - x) // a) <= 256:
                A[r, k], B[j, k] = a, (T - x) // a
                return T
    raise AssertionError(f"no tie reachable from {x}")


def int_operands(c: Case, seed: int, device):
    """Integer-valued bf16 A [M, K], B [N, K] and fp32 bias [N] (or None) for the exact oracle.  Element (M-1, N-1)
    (through k = K-1, in the last k-block) is planted with a tie that RNE rounds toward zero, and for M, N >= 2
    element (0, 0) (through k = 0) with one that RNE rounds away from zero."""
    global _TIES
    if _TIES is None:
        _TIES = _tie_values()
    assert c.K <= MAX_K, c
    g = torch.Generator(device=device).manual_seed(seed)
    A = torch.randint(-4, 5, (c.M, c.K), generator=g, device=device, dtype=torch.int32)
    B = torch.randint(-4, 5, (c.N, c.K), generator=g, device=device, dtype=torch.int32)
    bias = torch.randint(-64, 65, (c.N,), generator=g, device=device, dtype=torch.int32) if c.bias else None
    down, up = _TIES
    _plant(A, B, bias, c.M - 1, c.N - 1, c.K - 1, down)
    if c.M >= 2 and c.N >= 2:
        _plant(A, B, bias, 0, 0, 0, up)
    return A.to(torch.bfloat16), B.to(torch.bfloat16), None if bias is None else bias.float()


def randn_operands(c: Case, seed: int, device):
    g = torch.Generator(device=device).manual_seed(seed)
    A = torch.randn(c.M, c.K, generator=g, device=device).to(torch.bfloat16)
    B = (torch.randn(c.N, c.K, generator=g, device=device) / c.K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(c.N, generator=g, device=device) if c.bias else None
    return A, B, bias


# ---------------------------------------------------------------------------------------------------------- references
def reference(A, B, bias, relu):
    """relu?(A B^T + bias) in fp64."""
    R = A.double() @ B.double().t()
    if bias is not None:
        R += bias.double()
    return R.clamp_(min=0) if relu else R


def exact_expected(R: torch.Tensor, out_bf16: bool) -> torch.Tensor:
    """What the kernel must store for an integer-valued fp64 result R (|R| < 2^24: exact in fp32): R itself, or R
    rounded to nearest even in bf16."""
    return R.float().to(torch.bfloat16) if out_bf16 else R.float()


def bound(A, B, bias, K: int, R: torch.Tensor, out_bf16: bool) -> torch.Tensor:
    b = A.double().abs() @ B.double().abs().t()
    if bias is not None:
        b += bias.double().abs()
    b *= K * 2.0 ** -22
    return b + 2.0 ** -8 * R.abs() if out_bf16 else b


def tie_masks(R: torch.Tensor):
    """fp64 values halfway between two bf16 neighbours: (those RNE rounds toward zero, those it rounds away from zero)."""
    v = R.abs()
    _, e = torch.frexp(v)
    ulp = torch.ldexp(torch.ones_like(v), e - 8)
    tie = (v > 0) & (torch.fmod(v, ulp) == ulp / 2)
    rounded = R.float().to(torch.bfloat16).double().abs()
    return tie & (rounded < v), tie & (rounded > v)


def check_ties(R: torch.Tensor, c: Case):
    """A bf16-output case must contain a tie that RNE rounds toward zero (and, from 2 x 2 up, one it rounds away), or its
    rounding mode is not tested."""
    down, up = tie_masks(R)
    assert bool(down.any()), f"{c}: no tie that rounds toward zero"
    assert bool(up.any()) or min(c.M, c.N) < 2, f"{c}: no tie that rounds away from zero"
    return int(down.sum()), int(up.sum())


# ---------------------------------------------------------------------------------------------------------- checkers
def locate(row: int, col: int, c: Case) -> str:
    half = int(row % 128 >= 64)
    return (f"(row {row}, col {col}): tile ({row // 128}, {col // c.bn}) of 128x{c.bn}, rows {64 * half}..{64 * half + 63} "
            f"of the tile (consumer warpgroup {half + 1})")


def _first(mask: torch.Tensor):
    i = int(mask.reshape(-1).nonzero()[0])
    return divmod(i, mask.shape[1])


def check_exact(got: torch.Tensor, want: torch.Tensor, c: Case):
    assert got.dtype == want.dtype and got.shape == want.shape, f"{c}: got {got.dtype} {tuple(got.shape)}"
    if torch.equal(got, want):
        return
    bad = got != want
    r, k = _first(bad)
    raise AssertionError(f"{c}: {int(bad.sum())} of {bad.numel()} elements differ; first at {locate(r, k, c)}: "
                         f"expected {float(want[r, k])!r}, got {float(got[r, k])!r}")


def check_bound(got: torch.Tensor, R: torch.Tensor, bnd: torch.Tensor, c: Case) -> float:
    """Asserts |got - R| <= bnd everywhere; returns the largest error / bound ratio."""
    err = (got.double() - R).abs()
    bad = ~(err <= bnd)                                   # NaN counts as bad
    if bool(bad.any()):
        r, k = _first(bad)
        raise AssertionError(f"{c}: {int(bad.sum())} of {bad.numel()} elements outside the fp64 bound; first at "
                             f"{locate(r, k, c)}: expected {float(R[r, k])!r} +- {float(bnd[r, k]):.3g}, "
                             f"got {float(got[r, k])!r}")
    return float((err / bnd.clamp_min(1e-300)).max())


# ---------------------------------------------------------------------------------------------------------- guards
SENTINEL = {torch.float32: 0x5EADBEEF, torch.bfloat16: 0x5EAD}     # finite bit patterns no result here can produce
_BITS = {torch.float32: torch.int32, torch.bfloat16: torch.int16}
GUARD_BEFORE = 64


def guard_after(N: int) -> int:
    return 128 * N + 64                                   # a whole tile of rows past M, and then some


def guarded_out(M: int, N: int, dtype, device):
    """(buffer, [M, N] view) with GUARD_BEFORE sentinel elements before the view and guard_after(N) after it."""
    buf = torch.full((GUARD_BEFORE + M * N + guard_after(N),), SENTINEL[dtype], dtype=_BITS[dtype], device=device).view(dtype)
    return buf, buf[GUARD_BEFORE:GUARD_BEFORE + M * N].view(M, N)


def guard_faults(buf: torch.Tensor, M: int, N: int):
    """None if both guards still hold the sentinel, else where the first overwritten guard element lies."""
    bits = buf.view(_BITS[buf.dtype])
    for name, g, base in (("before", bits[:GUARD_BEFORE], -GUARD_BEFORE), ("after", bits[GUARD_BEFORE + M * N:], M * N)):
        hit = (g != SENTINEL[buf.dtype]).nonzero()
        if hit.numel():
            i = base + int(hit[0])
            return f"guard {name} the output overwritten at element {i} (row {i // N}, col {i % N} of an [M, N] layout)"
    return None
