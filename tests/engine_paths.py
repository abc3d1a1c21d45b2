"""The engine-path helpers of the optimizer-option tests (tests/test_gpu_sgd_options.py, tests/test_gpu_grad_clip.py): a spy
on a trainer's optimizer launches, random batches, the one-GPU slot trainer and the state two runs are compared by."""
import torch

import comm_model as M


class Spy:
    """Wraps a trainer's extension handle: before each optimizer launch it records the parameters, the momentum and the
    averaged gradient that launch will apply -- the bucket of this step's parity for ``allreduce_sgd``, and for
    ``reduce_sgd`` (whose gradient never leaves registers) the momentum of a plain launch with mu = 0 and lr = 0 on copies,
    which is the fixed-order reduction of the same slots.  Eager steps only (graph capture would record the copies)."""

    def __init__(self, tr):
        self._C, self.tr, self.log = tr.C, tr, []
        tr.C = self

    def __getattr__(self, name):
        return getattr(self._C, name)

    def _grad_of_bucket(self, stride):
        from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC
        cur = int(self.tr.step_counter.item()) & 1 if stride > 0 else 0
        return M.reduce_scaled([self.tr.grads[cur * NPAR_ALLOC:cur * NPAR_ALLOC + NPAR_ALLOC]], 1.0)   # 0 + bucket, as the kernel

    def allreduce_sgd(self, grads, sigs, params, momentum, step, lr, mu, scale, rank, world, zero_grads, grad_stride, *a, **k):
        torch.cuda.current_stream().synchronize()
        assert world == 1 and scale == 1.0
        self.log.append((params.clone(), momentum.clone(), self._grad_of_bucket(grad_stride), int(step.item())))
        return self._C.allreduce_sgd(grads, sigs, params, momentum, step, lr, mu, scale, rank, world, zero_grads, grad_stride,
                                     *a, **k)

    def reduce_sgd(self, slots, n_slots, factors, n_samples, params, momentum, step, *a, **k):
        torch.cuda.current_stream().synchronize()
        g = torch.zeros_like(momentum)
        self._C.reduce_sgd(slots, n_slots, factors, n_samples, params.clone(), g, None, None, 0.0, 0.0)
        torch.cuda.current_stream().synchronize()
        self.log.append((params.clone(), momentum.clone(), g, int(step.item())))
        return self._C.reduce_sgd(slots, n_slots, factors, n_samples, params, momentum, step, *a, **k)


def _batches(n, bsz, seed, raw=True):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = torch.randint(0, 256, (bsz, 1, 28, 28), generator=g, dtype=torch.uint8) if raw else \
            torch.randn(bsz, 1, 28, 28, generator=g)
        out.append((x, torch.randint(0, 10, (bsz,), generator=g)))
    return out


def _slot_trainer(dev, **kw):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    return FusedTrainer(128, lr=0.05, seed=11, device=dev, raw_uint8=True, **kw)


def _state(tr):
    tr.sync_lag(0)
    torch.cuda.synchronize()
    return tr.params.clone(), tr.momentum.clone(), float(tr.loss_acc[0].item()), int(tr.step_counter.item())
