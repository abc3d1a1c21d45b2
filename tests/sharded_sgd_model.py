"""Bit-exact model of the sharded optimizer kernel (csrc/sharded_sgd.cu), shared by the emulated-world GPU test
(tests/test_gpu_sharded_sgd_emulated.py) and by the CPU test that checks the model and shows that the checker catches planted
faults (tests/test_sharded_sgd_model.py).

One launch per rank on a gradient bucket of ``n_vec`` 16-byte vectors (4 fp32 or 8 bf16 gradients each), ``n_vec`` a multiple
of the world size W:

* rank r owns the elements ``[r * per, (r + 1) * per)``, ``per = n_vec / W`` vectors' worth;
* on its slice, ``g = (((0 + g_0) + g_1) + ...) * scale`` in fp32 in rank order (tests/comm_model.py ``reduce_scaled``: what
  the one-shot and two-shot all-reduce store for an fp32 bucket).  bf16 gradients are widened exactly and the fp32 result is
  NOT rounded back to bf16;
* the fmaf-exact update of tests/sgd_options_model.py (``sgd_update``) on the rank's own parameters of the slice and on its
  momentum shard (``per`` elements, indexed from 0);
* the new parameters of the slice land in EVERY rank's parameter flat; the momentum shard stays local;
* the rank's gradient bucket is zeroed (``zero_grad``) or left as it was, and it is zeroed only after every peer has read it.

``fault`` plants one defect a kernel could have; the CPU test shows that each changes what the checker sees.
"""
import struct

import torch

import comm_model as M
from sgd_options_model import sgd_update

FAULTS = ("wrong_owner", "sum_reversed", "scale_after_update", "momentum_global_offset", "zero_before_peers_read",
          "push_to_owner_only")


def f32(x: float) -> float:
    """A hyper-parameter as the kernel gets it: the binding's double rounded once to fp32."""
    return struct.unpack("f", struct.pack("f", x))[0]


def grid_blocks(n_vec: int, world: int, max_blocks: int) -> int:
    """CTAs per rank of one b2_sharded_sgd_launch: the two-shot all-reduce's grid."""
    return M.grid_blocks(M.TWOSHOT, n_vec, world, max_blocks)


def slice_of(rank: int, world: int, n_elems: int) -> tuple:
    per = n_elems // world
    return rank * per, (rank + 1) * per


def sharded_sgd_model(grads: list, params: list, momentum: list, scale: float, lr: float, mu: float, wd: float,
                      nesterov: bool, zero_grad: bool, fault: str = None) -> dict:
    """State after one step.  ``grads[r]``: rank r's bucket (fp32 or bf16, ``n`` elements, ``n`` a multiple of W x the
    elements of a vector); ``params[r]``: its fp32 parameter flat (``n`` elements); ``momentum[r]``: its fp32 shard
    (``n / W``).  Returns ``params``, ``momentum`` and ``grads``, one tensor per rank each."""
    world, n = len(grads), grads[0].numel()
    assert n % (world * M.elems_per_vec(grads[0].dtype)) == 0 and fault in (None,) + FAULTS
    lr, mu, wd = f32(lr), f32(mu), f32(wd)
    new_p = [p.clone() for p in params]
    new_m = [m.clone() for m in momentum]
    for r in range(world):
        lo, hi = slice_of((r + 1) % world if fault == "wrong_owner" else r, world, n)
        terms = [g[lo:hi].float() for g in grads]
        if fault == "zero_before_peers_read" and r > 0:          # rank 0 finished first and zeroed its bucket
            terms[0] = torch.zeros_like(terms[0])
        if fault == "sum_reversed":
            terms = terms[::-1]
        g = M.reduce_scaled(terms, 1.0 if fault == "scale_after_update" else scale)
        m_in = momentum[r]
        if fault == "momentum_global_offset" and r > 0:          # reads behind the shard, where nothing was ever stored
            m_in = torch.zeros_like(m_in)
        p, m = sgd_update(g, params[r][lo:hi], m_in, mu, lr, wd, nesterov)
        if fault == "scale_after_update":
            p = params[r][lo:hi] + (p - params[r][lo:hi]) * M.fp32_scale(scale)
        if fault != "momentum_global_offset" or r == 0:
            new_m[r] = m
        for q in range(world):
            if fault != "push_to_owner_only" or q == r:
                new_p[q][lo:hi] = p
    new_g = [torch.zeros_like(g) if zero_grad else g.clone() for g in grads]
    return {"params": new_p, "momentum": new_m, "grads": new_g}


def unsharded_model(variant: int, grads: list, params: torch.Tensor, momentum: torch.Tensor, scale: float, lr: float, mu: float,
                    wd: float, nesterov: bool) -> tuple:
    """The path the sharded kernel replaces, for fp32 buckets: the in-place all-reduce of tests/comm_model.py, then the
    unsharded update of the whole flat on every rank.  Returns (params, momentum), the same on every rank."""
    g = M.allreduce_model(variant, grads, torch.float32, scale, torch.float32, staged=False)["out"][0]
    return sgd_update(g, params, momentum, f32(mu), f32(lr), f32(wd), nesterov)


def make_state(world: int, n: int, seed: int) -> tuple:
    """Identical replicas of the parameters and a different momentum shard per rank."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    m = torch.randn(n, generator=g) * 0.1
    per = n // world
    return [p.clone() for _ in range(world)], [m[r * per:(r + 1) * per].clone() for r in range(world)], m
