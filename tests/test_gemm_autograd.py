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
