"""GPU-single tier: the one-GPU optimizer kernel reduce_sgd (csrc/sgd.cu, csrc/convnet_reduce.cuh) called directly on random
slots and fc1 factors, at batches and step grids that are not multiples of its load batches: fc1 passes of 128 samples
split over 480 loader threads, and batches of 6 slots per thread group (150 slots)."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

W3, FC1 = 5284, 50 * 320                # flat offset and size of fc1.weight (ops/convnet_fused.py LAYOUT)


@pytest.mark.parametrize("n_samples,n_slots", [(65, 65), (127, 127), (128, 128), (129, 129), (300, 151), (200, 320)])
def test_reduce_sgd_matches_fp64_and_zeroes_the_other_bucket(n_samples, n_slots):
    """SGD step from the fp64 sum of the slots and of dh (x) p2, the loss terms added to loss_acc, the step counter bumped and
    only the bucket of the other step parity zeroed."""
    from dist_tuto.pth_b200.ops import _ext
    from dist_tuto.pth_b200.ops.convnet_fused import FAC_STRIDE, NPAR, NPAR_ALLOC
    C = _ext.C()
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(n_samples * 1000 + n_slots)
    slots = torch.randn(n_slots, NPAR_ALLOC, generator=g)
    slots[:, W3:W3 + FC1] = float("nan")                   # the fc1.weight range of a slot is never read
    factors = torch.randn(n_samples, FAC_STRIDE, generator=g)
    params = torch.randn(NPAR_ALLOC, generator=g)
    momentum = torch.randn(NPAR_ALLOC, generator=g)
    loss_acc = torch.tensor([1.5, 7.0, 0.0, 0.0])
    lr, mu = 0.05, 0.5
    step = torch.tensor([5], dtype=torch.int64, device=dev)  # parity 1: bucket 0 is the other one
    done = torch.zeros(1, dtype=torch.int32, device=dev)
    grads = torch.full((2 * NPAR_ALLOC,), 3.0, device=dev)

    p_d, m_d, l_d = params.to(dev), momentum.to(dev), loss_acc.to(dev)
    C.reduce_sgd(slots.to(dev).reshape(-1), n_slots, factors.to(dev).reshape(-1), n_samples, p_d, m_d, step, done, lr, mu,
                 None, l_d, grads, NPAR_ALLOC)
    torch.cuda.synchronize()

    s64, f64 = slots.double(), factors.double()
    grad = s64[:, :NPAR].sum(0)
    grad[W3:W3 + FC1] = (f64[:, :50].t() @ f64[:, 64:384]).reshape(-1)
    m_ref = mu * momentum[:NPAR].double() + grad
    p_ref = params[:NPAR].double() - lr * m_ref
    tol = 1e-5 * max(n_slots, n_samples) ** 0.5
    assert torch.allclose(m_d[:NPAR].cpu().double(), m_ref, rtol=1e-5, atol=tol)
    assert torch.allclose(p_d[:NPAR].cpu().double(), p_ref, rtol=1e-5, atol=tol)
    loss_ref = loss_acc[:2].double() + s64[:, NPAR:NPAR + 2].sum(0)
    assert torch.allclose(l_d[:2].cpu().double(), loss_ref, rtol=1e-5, atol=tol)
    assert int(step.item()) == 6 and int(done.item()) == 0
    assert float(grads[:NPAR].abs().max()) == 0.0
    assert bool((grads[NPAR_ALLOC:] == 3.0).all())
