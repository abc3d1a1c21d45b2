"""CPU tier for the wgmma GEMM checks (tests/gemm_checks.py): the case table reaches every dispatch path of
csrc/gemm_tcgen05.cu at its edges, the integer operands are exact and carry bf16 ties, and the checkers catch each fault
a kernel could plausibly make, applied by a Python "faulty kernel" to the exact result."""
import pytest
import torch

import gemm_checks as G

GEO = G.kernel_geometry()


def test_geometry_read_from_the_kernel_source():
    assert GEO["BM"] == 128 and GEO["BK"] == 64
    assert set(GEO["stages"]) == {32, 64, 128} and all(s >= 2 for s in GEO["stages"].values())
    assert GEO["PBN"] % 2 == 0 and GEO["PSTAGES"] >= 2
    assert [bn for _, bn in GEO["rule"]] == [32, 64] and GEO["last"] == 128


@pytest.mark.parametrize("S", [132, 114])
def test_table_meets_every_coverage_condition(S):
    table = G.cases(S, GEO)
    assert G.coverage_gaps(table, S, GEO) == []
    assert {c.path for c in table} == set(G.PATHS)


def test_coverage_notices_a_moved_threshold():
    """A persistent threshold raised past the table's K takes its persistent cases off that path: the gaps say so."""
    moved = dict(GEO, p_min_k=4096)
    gaps = G.coverage_gaps(G.cases(132, GEO), 132, moved)
    assert any("dispatched to bn128" in g for g in gaps) and any(g.startswith("persistent: ") for g in gaps)
    deeper = dict(GEO, stages={**GEO["stages"], 64: 6})
    assert any(g.startswith("bn64: num_kb") for g in G.coverage_gaps(G.cases(132, GEO), 132, deeper))


def _small_table_cases():
    return [c for c in G.cases(132, GEO) if c.M * c.N * c.K <= 1 << 26]


@pytest.mark.parametrize("c", _small_table_cases(), ids=lambda c: f"{c.group}-{c.M}x{c.N}x{c.K}")
def test_integer_operands_are_exact_and_carry_ties(c):
    A, B, bias = G.int_operands(c, 7, "cpu")
    Af, Bf = A.float(), B.float()
    assert torch.equal(Af, Af.round()) and torch.equal(Bf, Bf.round())
    # one planted entry per tie: every other |a|, |b| <= 4
    assert int((Af.abs() > 4).sum()) == 0 and int((Bf.abs() > 4).sum()) <= 2 and float(Bf.abs().max()) <= 256
    # every partial sum, in any order, below 2^17: bounded by the sum of |products| per element
    assert float((Af.abs().double() @ Bf.abs().double().t()).max()) < 2 ** 17
    R = G.reference(A, B, bias, c.relu)
    down, up = G.check_ties(R, c)
    assert down >= 1


# -------------------------------------------------------------------------------------------- the faulty kernels
CASE = G._case("bn128", 129, 67, 136, (True, True, True), 132, GEO)            # odd N, two M-tiles, ragged last k-block
assert CASE.path == "bn128" and G.num_kb(CASE.K, GEO) == 3 and CASE.K % 64 == 8


def _operands(c=CASE):
    A, B, bias = G.int_operands(c, 11, "cpu")
    return A, B, bias, G.reference(A, B, bias, c.relu)


def _round_half_away(R):
    out = R.float().to(torch.bfloat16)
    down, _ = G.tie_masks(R)
    _, e = torch.frexp(R.abs())
    ulp = torch.ldexp(torch.ones_like(R), e - 8)
    away = (R + torch.sign(R) * ulp / 2).float().to(torch.bfloat16)
    return torch.where(down, away, out)


def _faulty(name, c, A, B, bias, R):
    """The output a kernel with fault ``name`` would store."""
    out = lambda R2: G.exact_expected(R2, c.out_bf16)                            # noqa: E731
    if name == "one_ulp":
        got = out(R).clone()
        got.view(torch.int16 if c.out_bf16 else torch.int32)[70, 3] += 1
        return got
    if name == "round_half_away":
        return _round_half_away(R)
    if name == "drop_last_kblock":
        k = (c.K - 1) // 64 * 64
        return out(G.reference(A[:, :k], B[:, :k], bias, c.relu))
    if name == "repeat_kstep":                                                  # k-step 1 of k-block 0 reads k-step 0
        A2, B2 = A.clone(), B.clone()
        A2[:, 16:32], B2[:, 16:32] = A[:, 0:16], B[:, 0:16]
        return out(G.reference(A2, B2, bias, c.relu))
    if name == "swap_halves":
        got = out(R).clone()
        got[0:64], got[64:128] = out(R)[64:128], out(R)[0:64]
        return got
    if name == "relu_before_bias":
        S = A.double() @ B.double().t()
        return out((S.clamp(min=0) if c.relu else S) + bias.double())
    if name == "tail_bias_shift":                                               # v0 += bias[col + 1] in the scalar tail
        b2 = bias.clone()
        b2[0:c.N - 1:2] = bias[1:c.N:2]
        return out(G.reference(A, B, b2, c.relu))
    if name == "fp32_through_bf16":
        return out(R).to(torch.bfloat16).float()
    raise KeyError(name)


FAULTS = {"one_ulp": CASE, "round_half_away": CASE, "drop_last_kblock": CASE, "repeat_kstep": CASE, "swap_halves": CASE,
          "relu_before_bias": CASE, "tail_bias_shift": CASE, "fp32_through_bf16": CASE._replace(out_bf16=False)}


def test_exact_kernel_passes():
    for c in (CASE, CASE._replace(out_bf16=False)):
        A, B, bias, R = _operands(c)
        G.check_exact(G.exact_expected(R, c.out_bf16), G.exact_expected(R, c.out_bf16), c)
        got = G.exact_expected(R, c.out_bf16).clone()
        got[R == 0] = -0.0                                                      # a signed zero is not a fault
        G.check_exact(got, G.exact_expected(R, c.out_bf16), c)


@pytest.mark.parametrize("name", sorted(FAULTS))
def test_exact_checker_catches_planted_fault(name):
    c = FAULTS[name]
    A, B, bias, R = _operands(c)
    got = _faulty(name, c, A, B, bias, R)
    with pytest.raises(AssertionError, match=r"elements differ; first at \(row \d+, col \d+\): tile \(\d+, \d+\) of 128x128"):
        G.check_exact(got, G.exact_expected(R, c.out_bf16), c)


def test_failure_message_locates_the_element():
    A, B, bias, R = _operands()
    got = _faulty("one_ulp", CASE, A, B, bias, R)
    with pytest.raises(AssertionError) as e:
        G.check_exact(got, G.exact_expected(R, True), CASE)
    msg = str(e.value)
    assert "1 of 8643 elements differ" in msg and "(row 70, col 3): tile (0, 0)" in msg and "warpgroup 2" in msg
    assert f"expected {float(G.exact_expected(R, True)[70, 3])!r}" in msg


def test_round_half_away_differs_only_at_the_planted_and_natural_ties():
    A, B, bias, R = _operands()
    down, _ = G.tie_masks(R)
    assert bool(down[CASE.M - 1, CASE.N - 1])                                   # the planted one
    assert torch.equal(_round_half_away(R) != G.exact_expected(R, True), down)


def test_store_past_row_M_hits_the_guard():
    A, B, bias, R = _operands()
    want = G.exact_expected(R, True)
    for dtype in (torch.bfloat16, torch.float32):
        buf, view = G.guarded_out(CASE.M, CASE.N, dtype, "cpu")
        view.copy_(want)
        assert G.guard_faults(buf, CASE.M, CASE.N) is None
        buf[G.GUARD_BEFORE + CASE.M * CASE.N + 5] = 1.0                         # row M, col 5
        assert G.guard_faults(buf, CASE.M, CASE.N).startswith(f"guard after the output overwritten at element "
                                                              f"{CASE.M * CASE.N + 5} (row {CASE.M}, col 5")
        buf, view = G.guarded_out(CASE.M, CASE.N, dtype, "cpu")
        buf[G.GUARD_BEFORE - 1] = 0.0
        assert "guard before" in G.guard_faults(buf, CASE.M, CASE.N)


# -------------------------------------------------------------------------------------------- the fp64 bound
def _randn_case(c):
    A, B, bias = G.randn_operands(c, 5, "cpu")
    R = G.reference(A, B, bias, c.relu)
    return A, B, bias, R, G.bound(A, B, bias, c.K, R, c.out_bf16)


def test_bound_admits_fp32_and_bf16_results():
    for c in (CASE, CASE._replace(out_bf16=False, relu=False)):
        A, B, bias, R, bnd = _randn_case(c)
        got = (A.float() @ B.float().t() + bias)
        got = got.relu() if c.relu else got
        got = got.to(torch.bfloat16) if c.out_bf16 else got
        assert G.check_bound(got, R, bnd, c) <= 1.0


@pytest.mark.parametrize("fault", ["twice_the_bound", "fp32_through_bf16", "drop_last_kblock", "nan"])
def test_bound_checker_catches_planted_fault(fault):
    c = CASE._replace(out_bf16=False, relu=False)
    A, B, bias, R, bnd = _randn_case(c)
    got = R.float().clone()
    if fault == "twice_the_bound":
        got[100, 66] = float(R[100, 66] + 2 * bnd[100, 66])
    elif fault == "fp32_through_bf16":
        got = got.to(torch.bfloat16).float()
    elif fault == "drop_last_kblock":
        got = G.reference(A[:, :128], B[:, :128], bias, False).float()
    else:
        got[128, 0] = float("nan")
    with pytest.raises(AssertionError, match="outside the fp64 bound; first at"):
        G.check_bound(got, R, bnd, c)
