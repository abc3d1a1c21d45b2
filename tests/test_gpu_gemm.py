"""GPU tier for the wgmma GEMM (csrc/gemm_tcgen05.cu): every case of the table in tests/gemm_checks.py, exact on integer
operands and within the fp64 bound on randn operands; the kernel each call launched, read from torch.profiler; guard bands
around the output; ``linear_tc`` exact on integer data; empty shapes; and a second device."""
import itertools
import re

import pytest
import torch
import torch.nn.functional as F

import gemm_checks as G
from emulated_ranks import C  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

GROUPS = ["bn32", "bn64", "bn128", "persistent", "engine", "existing"]


@pytest.fixture(scope="module")
def table():
    props = torch.cuda.get_device_properties(0)
    S = props.multi_processor_count
    print(f"\n[gemm] {props.name}, {S} SMs")
    return G.cases(S)


def _seed(c, salt=0):
    return (c.M * 1000003 + c.N * 1009 + c.K * 7 + salt) % (1 << 31)


def _run_exact(C, c, dev, out=None):
    A, B, bias = G.int_operands(c, _seed(c), dev)
    got = C.gemm_bf16(A, B, bias, c.relu, c.out_bf16, out=out)
    R = G.reference(A, B, bias, c.relu)
    if c.out_bf16:
        G.check_ties(R, c)
    G.check_exact(got, G.exact_expected(R, c.out_bf16), c)
    return got


@pytest.mark.parametrize("group", GROUPS)
def test_gemm_exact_and_within_fp64_bound(C, table, group):
    dev = torch.device("cuda", 0)
    cs = [c for c in table if c.group == group]
    worst = {False: (0.0, None), True: (0.0, None)}        # per output dtype: bf16 rounding alone reaches 2^-8 |R|
    for c in cs:
        _run_exact(C, c, dev)
        A, B, bias = G.randn_operands(c, _seed(c, 1), dev)
        got = C.gemm_bf16(A, B, bias, c.relu, c.out_bf16)
        R = G.reference(A, B, bias, c.relu)
        ratio = G.check_bound(got, R, G.bound(A, B, bias, c.K, R, c.out_bf16), c)
        if ratio >= worst[c.out_bf16][0]:
            worst[c.out_bf16] = (ratio, c)
        del A, B, bias, got, R
    print(f"\n[gemm] {group}: {len(cs)} cases exact; largest error/bound ratio on randn operands: "
          + "; ".join(f"{'bf16' if k else 'fp32'} out {r:.3g} at {c}" for k, (r, c) in worst.items() if c))


def test_each_call_launches_the_kernel_the_table_expects(C, table):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda", 0)
    ops = [G.int_operands(c, _seed(c), dev) for c in table if c.M * c.K < (1 << 26)]   # the large ones: made in the loop
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]):       # a first session starts the profiler before anything is counted
        torch.ones(1, device=dev).add_(1)
        torch.cuda.synchronize()
    pat = re.compile(r"gemm_bf16_kernel<\d+>|gemm_bf16_persistent_kernel")

    def launched(A, B, bias, c):
        """The GEMM kernels one call launched, from a profiler session around that call alone."""
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            # Once another process has used the GPU, a session loses kernel records at its start, and the profiler keeps
            # only the device activity inside its window.  After many sessions in one process (the whole suite) the loss
            # reaches past a single ~10 ms sleep kernel: twenty ~5 ms sleep kernels before the GEMM launch and one ~10 ms
            # after it keep the launch well inside the window.
            for _ in range(20):
                torch.cuda._sleep(10_000_000)
            torch.cuda.synchronize()
            C.gemm_bf16(A, B, bias, c.relu, c.out_bf16)
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)
            torch.cuda.synchronize()
        return [pat.search(e.name).group(0) for e in prof.events() if e.device_type == DeviceType.CUDA and pat.search(e.name)]

    small = iter(ops)
    for c in table:
        A, B, bias = next(small) if c.M * c.K < (1 << 26) else G.int_operands(c, _seed(c), dev)
        # A session that recorded no GEMM at all is run again; one call recorded as another kernel, or as more than one
        # launch, fails at once.
        for _ in range(3):
            ran = launched(A, B, bias, c)
            if ran:
                break
        assert ran == [G.KERNEL_NAME[c.path]], (c, ran)
    counts = {p: sum(1 for c in table if c.path == p) for p in G.PATHS}
    print(f"\n[gemm] profiler: calls per kernel {counts}")


def _guard_cases(table):
    """The first case of each path with each epilogue."""
    seen, out = set(), []
    for c in table:
        key = (c.path, c.bias, c.relu, c.out_bf16)
        if key not in seen and c.M * c.N < (1 << 24):
            seen.add(key)
            out.append(c)
    return out


def test_stores_stay_inside_the_output(C, table):
    dev = torch.device("cuda", 0)
    cs = _guard_cases(table)
    assert {(c.path, c.bias, c.relu, c.out_bf16) for c in cs} == {(p,) + e for p in G.PATHS for e in G.COMBOS}
    for c in cs:
        buf, view = G.guarded_out(c.M, c.N, torch.bfloat16 if c.out_bf16 else torch.float32, dev)
        got = _run_exact(C, c, dev, out=view)
        assert got.data_ptr() == view.data_ptr()
        fault = G.guard_faults(buf, c.M, c.N)
        assert fault is None, f"{c}: {fault}"


def test_out_argument_is_checked(C):
    dev = torch.device("cuda", 0)
    a = torch.ones(4, 8, device=dev, dtype=torch.bfloat16)
    b = torch.ones(6, 8, device=dev, dtype=torch.bfloat16)
    ok = torch.empty(4, 6, device=dev)
    assert C.gemm_bf16(a, b, None, False, False, out=ok).data_ptr() == ok.data_ptr() and bool((ok == 8).all())
    bad = {"dtype": torch.empty(4, 6, device=dev, dtype=torch.bfloat16), "shape": torch.empty(6, 4, device=dev),
           "contiguous": torch.empty(6, 4, device=dev).t(), "aligned": torch.empty(25, device=dev)[1:].view(4, 6),
           "device": torch.empty(4, 6)}
    for what, out in bad.items():
        with pytest.raises(RuntimeError, match="out must"):
            C.gemm_bf16(a, b, None, False, False, out=out)


def _ints(g, shape, lo, hi, dev):
    return torch.randint(lo, hi + 1, shape, generator=g).float().to(dev)


@pytest.mark.parametrize("M", [1, 7, 13, 129, 1000])
def test_linear_tc_exact_on_integer_data(M):
    """Forward, data gradient, weight gradient (inner dimension M, padded to 8) and bias gradient of ``linear_tc``, all
    integers: every one must equal the fp64 result exactly."""
    from dist_tuto.pth_b200.ops.gemm import linear_tc
    dev = torch.device("cuda", 0)
    lead = (8, 125) if M == 1000 else (M,)
    for K, N in itertools.product([3, 8, 50, 320], [1, 10, 50, 64]):
        g = torch.Generator().manual_seed(M * 100 + K + N)
        x = _ints(g, lead + (K,), -4, 4, dev).requires_grad_()
        w = _ints(g, (N, K), -4, 4, dev).requires_grad_()
        b = _ints(g, (N,), -64, 64, dev).requires_grad_()
        gy = _ints(g, lead + (N,), -4, 4, dev)
        y = linear_tc(x, w, b)
        y.backward(gy)
        x2, gy2 = x.detach().reshape(M, K).double(), gy.reshape(M, N).double()
        wd = w.detach().double()
        want = {"y": (x2 @ wd.t() + b.detach().double()).reshape(lead + (N,)), "dx": (gy2 @ wd).reshape(lead + (K,)),
                "dw": gy2.t() @ x2, "db": gy2.sum(0)}
        for name, got in (("y", y), ("dx", x.grad), ("dw", w.grad), ("db", b.grad)):
            assert got.dtype == torch.float32 and torch.equal(got, want[name].float()), \
                (M, K, N, name, float((got.double() - want[name]).abs().max()))


@pytest.mark.parametrize("M,N,K", [(0, 10, 16), (5, 0, 16), (5, 10, 0), (0, 0, 0), (0, 64, 320)])
def test_empty_shapes_match_f_linear(M, N, K):
    from dist_tuto.pth_b200.ops.gemm import TcLinear, linear_bf16, linear_tc
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(M, K, generator=g).to(dev)
    w = torch.randn(N, K, generator=g).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    for bias, relu, dt in itertools.product((b, None), (False, True), (torch.float32, torch.bfloat16)):
        ref = F.linear(x, w, bias)
        ref = (ref.relu() if relu else ref).to(dt)
        out = linear_bf16(x, w, bias, relu=relu, out_dtype=dt)
        assert out.shape == ref.shape and out.dtype == dt and torch.equal(out, ref)
    m = TcLinear(K, N).to(dev)
    ref = torch.nn.Linear(K, N).to(dev)
    ref.load_state_dict(m.state_dict())
    xm, xr = x.clone().requires_grad_(), x.clone().requires_grad_()
    y, yr = m(xm), ref(xr)
    assert y.shape == yr.shape and torch.equal(y, yr)
    y.sum().backward()
    yr.sum().backward()
    for got, want in ((xm.grad, xr.grad), (m.weight.grad, ref.weight.grad), (m.bias.grad, ref.bias.grad)):
        assert got.shape == want.shape and torch.equal(got, want)
    xl = x.clone().requires_grad_()
    yl = linear_tc(xl, w, None)
    yl.backward(torch.ones_like(yl))
    assert torch.equal(yl, F.linear(x, w)) and torch.equal(xl.grad, torch.ones(M, N, device=dev) @ w)


@pytest.mark.multigpu
def test_second_device_after_the_first(C, table):
    """The launchers configure each kernel's shared-memory limit per device: one case per path on cuda:0, then cuda:1."""
    picks = [next(c for c in table if c.path == p) for p in G.PATHS]
    for d in (0, 1):
        dev = torch.device("cuda", d)
        with torch.cuda.device(dev):
            S = torch.cuda.get_device_properties(d).multi_processor_count
            for c in picks:
                c = G._case(c.group, c.M, c.N, c.K, (c.bias, c.relu, c.out_bf16), S, G.kernel_geometry())
                got = _run_exact(C, c, dev)
                assert got.device == dev
