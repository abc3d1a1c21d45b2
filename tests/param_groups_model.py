"""A rounding-exact CPU model of the grouped optimizer kernels (csrc/sgd.cu sgd_flat_grouped_kernel, csrc/adamw.cu
adamw_flat_grouped_kernel and the grouped instances of csrc/sharded_sgd.cu): element i takes the scalars of group
``gmap[i // 4]``, one uint8 id per 16-byte fp32 parameter vector.  Everything else is the ungrouped kernels' sequence
(tests/sgd_options_model.py ``sgd_update``, tests/adamw_model.py ``adamw_update``), so running those on each tensor's
segment with its group's scalars is the oracle.  ``fault`` plants the mistakes the tests must catch."""
import torch

from adamw_model import f32, scalars64, sqrt32
from sgd_options_model import fma32

FAULTS = ("map_shifted", "group0_everywhere", "decay_in_no_decay_group", "lr_after_bc1_rounding")


def expand(gmap: torch.Tensor, n: int, values: list, fault: str = None) -> torch.Tensor:
    """The fp32 per-element tensor of ``values[group of the element]`` for ``n`` elements."""
    ids = gmap.long().cpu()
    if fault == "map_shifted":
        ids = torch.roll(ids, 1)
    if fault == "group0_everywhere":
        ids = torch.zeros_like(ids)
    vals = torch.tensor([f32(v) for v in values], dtype=torch.float32)
    return vals[ids].repeat_interleave(4)[:n]


def _decays(wds: list, fault: str) -> list:
    return [max(wds) if (fault == "decay_in_no_decay_group" and w == 0.0) else w for w in wds]


def grouped_sgd(g, p, m, gmap, lrs: list, wds: list, mu: float, nesterov: bool, fault: str = None):
    """(p, m) after one grouped momentum-SGD update of the fp32 flats."""
    assert fault in (None,) + FAULTS
    g, p, m = (x.float().cpu() for x in (g, p, m))
    lr, wd = expand(gmap, g.numel(), lrs, fault), expand(gmap, g.numel(), _decays(wds, fault), fault)
    g = fma32(wd, p, g)
    m = fma32(mu, m, g)
    d = fma32(mu, m, g) if nesterov else m
    return fma32(-lr, d, p), m


def group_step_sizes(lrs: list, betas: tuple, t: int, fault: str = None) -> list:
    """lr_g / (1 - beta1^t) per group in fp64 (rounded once by the binding); the fault forms it from the rounded 1 / bc1."""
    if fault == "lr_after_bc1_rounding":
        return [f32(f32(lr) * f32(1.0 / (1.0 - betas[0] ** t))) for lr in lrs]
    return [lr / (1.0 - betas[0] ** t) for lr in lrs]


def grouped_adamw(g, p, m, v, gmap, lrs: list, wds: list, betas: tuple, eps: float, t: int, fault: str = None):
    """(p, m, v) after grouped AdamW update ``t``: ``1 - lr_g*wd_g`` and ``lr_g / bc1`` per group, the rest shared."""
    assert fault in (None,) + FAULTS
    g, p, m, v = (x.float().cpu() for x in (g, p, m, v))
    n = g.numel()
    wds = _decays(wds, fault)
    decay = expand(gmap, n, [1.0 - lr * wd for lr, wd in zip(lrs, wds)], fault)
    step = expand(gmap, n, group_step_sizes(lrs, betas, t, fault), fault)
    _, w1, b2, c2, _, sbc2, e = (torch.full_like(g, f32(x)) for x in scalars64(lrs[0], betas, eps, 0.0, t))
    p = p * decay
    d = g - m
    m = fma32(w1, d, m) if float(w1[0]) < 0.5 else fma32(-d, 1.0 - w1, g)
    v = fma32(c2 * g, g, v * b2)
    den = sqrt32(v) / sbc2 + e
    p = fma32(-step, m / den, p)
    return p, m, v
