"""Model of gradient-norm clipping in the optimizer kernels (csrc/sgd_device.cuh clip_coef / clip_apply, csrc/sgd.cu
sgd_flat_clip_kernel): torch.nn.utils.clip_grad_norm_ with norm type 2.

* ``coef32(n, c)``: torch's coefficient ``clamp(c / (n + 1e-6), max=1)`` in fp32, where torch computes the division as
  ``reciprocal(n + 1e-6) * c`` -- three correctly rounded fp32 operations (numpy float32 arithmetic), NaN passing the clamp;
* ``clip_update``: ``g * coef`` (one fp32 multiply), then the update of sgd_options_model;
* ``NORM_REL_TOL``: how far the kernels' norm may be from the fp64 norm of the same fp32 gradient.  The kernels sum the
  squares in fp32 per thread (at most a few dozen terms here) and per CTA (a fixed tree of at most 16 warps x 5 levels),
  then in fp64: the relative error of the fp32 part is below (terms + 21) * 2^-24, well under 2^-14 for every size the
  tests use, and the square root halves it.

Shared by tests/test_grad_clip.py and tests/test_gpu_grad_clip.py.
"""
import numpy as np
import torch

import sgd_options_model as SM

NORM_REL_TOL = 2.0 ** -14


def coef32(n, c) -> np.float32:
    """The fp32 clip coefficient for total norm ``n`` (fp32) and max norm ``c`` (rounded to fp32 once)."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        d = np.float32(n) + np.float32(1e-6)
        k = (np.float32(1.0) / d) * np.float32(c)
    return k if not k > np.float32(1.0) else np.float32(1.0)


def clip_update(g, p, m, mu, lr, wd, nesterov, n, c):
    """(params, momentum) after clipping the averaged fp32 gradient ``g`` by the norm ``n`` and one update."""
    k = float(coef32(n, c))
    return SM.sgd_update(g * torch.tensor(k, dtype=torch.float32), p, m, mu, lr, wd, nesterov)


def norm64(g) -> float:
    """The fp64 L2 norm of the fp32 gradient ``g`` (one tensor or a list)."""
    ts = g if isinstance(g, (list, tuple)) else [g]
    return float(torch.sqrt(sum((t.double() ** 2).sum() for t in ts)))


def assert_norm_close(what, got, want):
    assert abs(got - want) <= NORM_REL_TOL * want + 1e-30, (what, got, want, abs(got - want) / max(want, 1e-300))
