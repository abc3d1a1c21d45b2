"""Rounding-exact model of the sharded FlatLAMB / FlatLARS kernels (csrc/sharded_layerwise.cu), shared by the CPU test
(tests/test_sharded_layerwise_model.py) and the emulated-rank GPU test (tests/test_gpu_sharded_layerwise_emulated.py).

A bucket of ``n`` elements (padded to W slices of whole 16-byte gradient vectors) holds tensors at ``offsets`` (multiples of
4) of ``numels`` elements.  Rank r owns ``[r * per, (r + 1) * per)``, ``per = n / W``.  One update:

* the averaged gradient ``(((0 + g_0) + g_1) + ...) * scale`` in fp32 in rank order (tests/comm_model.py ``reduce_scaled``;
  bf16 buckets are widened exactly);
* rank r's chunk table: each tensor's piece of its slice cut into chunks of at most CHUNK elements from the piece's start;
* per element the maths of tests/layerwise_model.py (LAMB's moments and u, LARS's direction and momentum step);
* rank r's per-tensor sums: its chunks' partials (``chunk_sqsum``, the kernel's fp32 order) added in chunk order in fp64;
* a tensor's two sums: the W ranks' sums added in rank order from +0 in fp64, the same on every rank; the ratio as in the
  unsharded model;
* the new parameters of every slice land in every rank's flat; the state shards stay with their rank.

``fault`` plants one defect a kernel could have; tests/test_sharded_layerwise_model.py shows that the checks catch each.
"""
import math

import torch

import comm_model as M
import layerwise_model as L
from layerwise_model import f32, fma32, sqrt32

CHUNK = L.CHUNK
FAULTS = ("local_ratio", "partial_twice", "partial_dropped", "chunk_crosses_slice", "decay_on_excluded",
          "rank_dependent_order")


def slice_table(offsets, numels, lo, hi, chunk=CHUNK):
    """[(start, length, tensor)]: rank's chunk table for the slice [lo, hi), starts in bucket coordinates."""
    out = []
    for t, (o, k) in enumerate(zip(offsets, numels)):
        a, b = max(o, lo), min(o + k, hi)
        out += [(s, min(chunk, b - s), t) for s in range(a, b, chunk)]
    return out


def rank_tables(offsets, numels, n, world, chunk=CHUNK, fault=None):
    """Every rank's table.  The fault ``chunk_crosses_slice`` gives each rank the unsharded table's chunks that start in its
    slice, uncut, so a chunk may run into the next slice."""
    per = n // world
    if fault == "chunk_crosses_slice":
        whole = L.chunk_table(offsets, numels, chunk)
        return [[c for c in whole if r * per <= c[0] < (r + 1) * per] for r in range(world)]
    return [slice_table(offsets, numels, r * per, (r + 1) * per, chunk) for r in range(world)]


def _tensor_ids(offsets, numels, n):
    tid = torch.full((n,), -1, dtype=torch.int64)
    for t, (o, k) in enumerate(zip(offsets, numels)):
        tid[o:o + k] = t
    return tid


def _ratio(kind, adapt, a, b, hp):
    W, Q = math.sqrt(a), math.sqrt(b)
    if not (adapt and W > 0.0 and Q > 0.0):
        return 1.0
    if kind == "lamb":
        return f32(W / Q)
    return f32((hp["trust_coefficient"] * W) / ((Q + hp["weight_decay"] * W) + hp["eps"]))


def step(kind, grads, p, states, offsets, numels, adapt, hp, scale, t=1, zero_grad=True, fault=None, chunk=CHUNK):
    """One sharded update of a bucket.  ``grads``: the W ranks' gradient buckets (n elements, fp32 or bf16); ``p``: the fp32
    parameter flat (n, the same on every rank); ``states``: the whole state flats, the ranks' shards in rank order (LAMB:
    [m, v], LARS: [momentum]); ``t``: LAMB's update number.

    Returns ``params`` (one flat per rank), ``states`` (whole flats), ``shards`` (per state, one shard per rank), ``ratios``
    (per rank, all tensors), ``sums`` (per rank: the [2 * tensors] fp64 sums over its chunks), ``totals`` (per rank: the
    [2 * tensors] fp64 sums it adds up from every rank's, the same on every rank), ``grads`` (after the update) and ``g``
    (the averaged gradient, fp32)."""
    assert kind in ("lamb", "lars") and fault in (None,) + FAULTS
    world, n, T = len(grads), p.numel(), len(offsets)
    per = n // world
    p = p.float().cpu().clone()
    states = [s.float().cpu().clone() for s in states]
    g = M.reduce_scaled([x.cpu() for x in grads], scale)
    tables = rank_tables(offsets, numels, n, world, chunk, fault)
    tid = _tensor_ids(offsets, numels, n)
    owner = torch.full((n,), -1, dtype=torch.int64)               # the rank whose chunk covers the element
    for r, tab in enumerate(tables):
        for s, ln, _ in tab:
            owner[s:s + ln] = r
    cov = owner >= 0
    inside = cov & (torch.arange(n) // per == owner)               # the owner holds the element's state
    ad = torch.tensor([bool(a) for a in adapt] + [False])[tid]       # tid -1 (padding) -> not adapted
    decay = ad | (cov & (fault == "decay_on_excluded"))
    st_in = [torch.where(inside, s, torch.zeros_like(s)) for s in states]   # state beyond a shard reads as 0
    if kind == "lamb":
        b1, b2 = hp["betas"]
        w1, beta2, c2, sbc2, eps, rbc1, lr, wd = (f32(x) for x in (1 - b1, b2, 1 - b2, (1 - b2 ** t) ** 0.5, hp["eps"],
                                                                    1 / (1 - b1 ** t), hp["lr"], hp["weight_decay"]))
        m, v = st_in
        d = g - m
        m = fma32(w1, d, m) if w1 < 0.5 else fma32(-d, f32(1.0 - w1), g)
        v = fma32(torch.tensor(c2) * g, g, v * torch.tensor(beta2))
        den = sqrt32(v) / torch.tensor(sbc2) + torch.tensor(eps)
        q = fma32(torch.where(decay, torch.tensor(wd), torch.tensor(0.0)), p, (m / den) * torch.tensor(rbc1))
        new_states = [m, v]
    else:
        q = g
        new_states = [st_in[0]]
    sums = []
    for tab in tables:
        sa, sb = L.tensor_sums(p, q, tab, T)
        sums.append([x for pair in zip(sa, sb) for x in pair])
    ratios, totals = [], []
    for r in range(world):
        order = list(range(world))
        if fault == "rank_dependent_order":          # each rank starts from its own sums
            order = [(r + i) % world for i in range(world)]
        if fault == "local_ratio":
            order = [r]
        if fault == "partial_twice":
            order = [0] + order
        if fault == "partial_dropped":
            order = order[1:]
        tot = [0.0] * (2 * T)
        for s in order:
            tot = [x + y for x, y in zip(tot, sums[s])]
        totals.append(tot)
        ratios.append([_ratio(kind, adapt[i], tot[2 * i], tot[2 * i + 1], hp) for i in range(T)])
    # every covered element is updated by its owner with the owner's ratio
    rt = torch.tensor(ratios + [[1.0] * T], dtype=torch.float32)     # row -1: uncovered elements (never written)
    r_el = rt[owner, tid.clamp(min=0)]
    new_p = p.clone()
    if kind == "lamb":
        new_p = fma32(-(torch.tensor(lr) * r_el), q, p)
    else:
        lr, mu, wd32 = f32(hp["lr"]), f32(hp["momentum"]), f32(hp["weight_decay"])
        dd = r_el * fma32(torch.where(decay, torch.tensor(wd32), torch.tensor(0.0)), p, g)
        mom = fma32(mu, st_in[0], dd)
        new_p = fma32(-lr, fma32(mu, mom, dd) if hp["nesterov"] else mom, p)
        new_states = [mom]
    p_out = torch.where(cov, new_p, p)
    st_out = [torch.where(inside, ns, s) for ns, s in zip(new_states, states)]
    return {"params": [p_out.clone() for _ in range(world)], "states": st_out,
            "shards": [[s[r * per:(r + 1) * per].clone() for r in range(world)] for s in st_out], "ratios": ratios,
            "sums": sums, "totals": totals, "g": g,
            "grads": [torch.zeros_like(x) if zero_grad else x.clone() for x in grads]}


def tensors_inside_one_slice(offsets, numels, n, world):
    """Indices of the tensors (with elements) that lie inside one rank's slice."""
    per = n // world
    return [t for t, (o, k) in enumerate(zip(offsets, numels)) if k > 0 and o // per == (o + k - 1) // per]


def unsharded_step(kind, g, p, states, offsets, numels, adapt, hp, t=1, chunk=CHUNK):
    """tests/layerwise_model.py's unsharded update on the averaged gradient ``g``: (p, states, ratios)."""
    if kind == "lamb":
        p2, m, v, r = L.lamb_step(p, g, states[0], states[1], offsets, numels, adapt, hp, t, chunk=chunk)
        return p2, [m, v], r
    p2, m, r = L.lars_step(p, g, states[0], offsets, numels, adapt, hp, chunk=chunk)
    return p2, [m], r
