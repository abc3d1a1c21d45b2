"""Autograd wiring of the trainable wgmma linear (ops/gemm.py): the three GEMMs, their K-major re-layouts and paddings.

CPU tier: the extension's ``gemm_bf16`` is replaced by a plain fp32 ``A @ B^T`` of the same bf16 operands, so everything but
the kernel itself is checked here (shapes not multiples of 8, leading batch dims, no bias); the GPU tier
(tests/test_gpu_kernels.py::test_tc_linear_forward_backward_on_tcgen05) runs the real kernel."""
import pytest
import torch

from dist_tuto.pth_b200.ops import gemm as G


class _FakeExt:
    calls = []

    @staticmethod
    def gemm_bf16(a, b, bias, relu, out_bf16):
        assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.is_contiguous() and b.is_contiguous()
        assert a.shape[1] == b.shape[1] and a.shape[1] % 8 == 0           # the kernel's TMA constraint: 16-byte rows
        _FakeExt.calls.append((tuple(a.shape), tuple(b.shape)))
        c = a.float() @ b.float().t()
        if bias is not None:
            c = c + bias
        if relu:
            c = c.relu()
        return c.to(torch.bfloat16) if out_bf16 else c


@pytest.mark.parametrize("lead,K,N,use_bias", [((12,), 16, 8, True), ((5, 7), 50, 10, True), ((33,), 320, 50, False), ((1,), 3, 1, True)])
def test_linear_tc_autograd_matches_reference(monkeypatch, lead, K, N, use_bias):
    monkeypatch.setattr(G._ext, "C", lambda: _FakeExt)
    _FakeExt.calls.clear()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(*lead, K, generator=g, requires_grad=True)
    w = torch.randn(N, K, generator=g, requires_grad=True)
    b = torch.randn(N, generator=g, requires_grad=True) if use_bias else None
    gy = torch.randn(*lead, N, generator=g)
    y = G._LinearTC.apply(x, w, b)
    y.backward(gy)
    # reference: the same op on the same bf16-rounded operands, fp32 math
    xr = x.detach().to(torch.bfloat16).float().requires_grad_()
    wr = w.detach().to(torch.bfloat16).float().requires_grad_()
    br = b.detach().clone().requires_grad_() if use_bias else None
    yr = torch.nn.functional.linear(xr, wr, br)
    yr.backward(gy.to(torch.bfloat16).float())
    assert y.shape == yr.shape and torch.allclose(y, yr, atol=1e-4, rtol=1e-4)
    assert torch.allclose(x.grad, xr.grad, atol=1e-3, rtol=1e-3) and x.grad.shape == x.shape
    assert torch.allclose(w.grad, wr.grad, atol=1e-3, rtol=1e-3) and w.grad.shape == w.shape
    if use_bias:
        assert torch.allclose(b.grad, gy.reshape(-1, N).sum(0), atol=1e-4, rtol=1e-4)
    assert len(_FakeExt.calls) == 3                                       # forward, dgrad, wgrad: one launch each


def test_tc_linear_is_a_drop_in_linear_on_cpu():
    m = G.TcLinear(20, 7)
    ref = torch.nn.Linear(20, 7)
    ref.load_state_dict(m.state_dict())                                   # state-dict compatible
    x = torch.randn(4, 20)
    assert torch.allclose(m(x), ref(x))                                   # CPU tensors take F.linear


class _RefusingExt(_FakeExt):
    """The fake GEMM with the launcher's shape rule: M, N or K = 0 is refused."""

    @staticmethod
    def gemm_bf16(a, b, bias, relu, out_bf16):
        if 0 in (a.shape[0], a.shape[1], b.shape[0]):
            raise RuntimeError("gemm_bf16: bad shape (K must be a multiple of 8)")
        return _FakeExt.gemm_bf16(a, b, bias, relu, out_bf16)


@pytest.mark.parametrize("M,N,K", [(0, 10, 16), (5, 0, 16), (5, 10, 0), (0, 0, 0)])
@pytest.mark.parametrize("use_bias", [True, False])
def test_empty_shapes_launch_nothing_and_match_f_linear(monkeypatch, M, N, K, use_bias):
    monkeypatch.setattr(G._ext, "C", lambda: _RefusingExt)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(M, K, generator=g, requires_grad=True)
    w = torch.randn(N, K, generator=g, requires_grad=True)
    b = torch.randn(N, generator=g, requires_grad=True) if use_bias else None
    y = G._LinearTC.apply(x, w, b)
    yr = torch.nn.functional.linear(x.detach().requires_grad_(), w.detach().requires_grad_(), b)
    assert y.shape == yr.shape == (M, N) and y.dtype == torch.float32 and torch.equal(y, yr.detach())
    y.backward(torch.ones_like(y))
    assert x.grad.shape == x.shape and torch.equal(x.grad, torch.ones(M, N) @ w.detach())
    assert w.grad.shape == w.shape and torch.equal(w.grad, torch.ones(M, N).t() @ x.detach())
    if use_bias:
        assert torch.equal(b.grad, torch.full((N,), float(M)))
    for relu in (False, True):
        for dt in (torch.float32, torch.bfloat16):
            out = G.linear_bf16(x.detach(), w.detach(), b, relu=relu, out_dtype=dt)
            ref = torch.nn.functional.linear(x.detach(), w.detach(), b)
            ref = (ref.relu() if relu else ref).to(dt)
            assert out.shape == (M, N) and out.dtype == dt and torch.equal(out, ref.detach())
