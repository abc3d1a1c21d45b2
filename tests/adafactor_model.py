"""Rounding-exact model of FlatAdafactor's kernels (csrc/adafactor.cu) and the fp64 reference, shared by
tests/test_adafactor_model.py (CPU) and tests/test_gpu_adafactor.py.

A bucket is a flat fp32 tensor holding tensors at ``offset`` with a shape and strides (any dense layout).  The model follows
the kernels:

* the chunk table (``table``): unfactored tensors in runs of CHUNK columns; a factored tensor with R * C <= CHUNK in chunks
  of whole slices; a bigger one in tiles of TR x TC of one slice (TC = min(C, 256), TR = min(R, CHUNK // TC), then
  TC = min(C, CHUNK // TR)), in (slice, tile row, tile column) order;
* a chunk's sum of squares (``box_sqsum``): its values in logical order (columns fastest), thread i of THREADS adding
  values i, i + THREADS, ... with one-rounding fmaf in fp32, xor butterflies in each warp, the warps in order in fp32;
  a tensor's chunk partials added in chunk order in fp64, the root taken in fp64 and rounded once to fp32;
* a row's (column's) sum of g^2 inside a tile: fmaf in column (row) order in fp32; the tile partials added in tile order
  in fp64; the mean ``fp32(sqrt(sum))^2 / C`` in fp32;
* a slice's row_var mean: blocks of ceil(R / 256) rows, fp64 in row order within a block, then the blocks in order,
  divided by R in fp64, rounded once, clamped to eps1;
* torch's lerp as one fused multiply-add; ``u = (1 / sqrt(max(v, eps1^2))) * g`` with every operation rounded once;
* ``alpha``, the denominator and the step formed in fp64 from the fp32 norms, the step rounded once to fp32;
  ``p = fmaf(step, u, p * fp32(1 - lr * wd))``.

``fault`` plants one defect a kernel could have; tests/test_adafactor_model.py shows that the bound catches each.
"""
import math

import torch

from adamw_model import f32
from sgd_options_model import fma32

CHUNK = 8192
THREADS = 256
TILE_COLS = 256
FAULTS = ("rows_cols_swapped", "norm_after_decay", "eps1_not_squared", "mean_over_wrong_dim", "denom_without_d",
          "t_from_zero", "rho_unscheduled", "chunk_crosses_tensor")


def factors(shape):
    """(B, R, C) of a factored tensor (dim > 1), None otherwise."""
    if len(shape) < 2:
        return None
    return math.prod(shape[:-2]), int(shape[-2]), int(shape[-1])


def state_offsets(shapes):
    """Each tensor's first state element and the state's size: row_var then col_var (B*R + B*C) or variance (numel)."""
    out, n = [], 0
    for s in shapes:
        out.append(n)
        f = factors(s)
        n += math.prod(s) if f is None else f[0] * (f[1] + f[2])
    return out, n


def table(shapes):
    """Per tensor: (chunks [(b0, nb, r0, nr, c0, nc)], whole, TR, TC) as adafactor_table builds them."""
    out = []
    for s in shapes:
        n, f = math.prod(s), factors(s)
        chunks, whole, TR, TC = [], False, 0, 0
        if n > 0:
            if f is None:
                chunks = [(0, 1, 0, 1, c0, min(CHUNK, n - c0)) for c0 in range(0, n, CHUNK)]
            else:
                B, R, C = f
                if R * C <= CHUNK:
                    whole, per = True, CHUNK // (R * C)
                    chunks = [(b0, min(per, B - b0), 0, R, 0, C) for b0 in range(0, B, per)]
                else:
                    TC = min(C, TILE_COLS)
                    TR = min(R, CHUNK // TC)
                    TC = min(C, CHUNK // TR)
                    chunks = [(b, 1, r0, min(TR, R - r0), c0, min(TC, C - c0)) for b in range(B) for r0 in range(0, R, TR)
                              for c0 in range(0, C, TC)]
        out.append((chunks, whole, TR, TC))
    return out


def box_sqsum(rows: torch.Tensor) -> torch.Tensor:
    """The fp32 partial of each row of ``rows`` ([chunks, L], each chunk's values in logical order, zero padded; a zero adds
    nothing), in the kernels' order; fp64 results."""
    n, L = rows.shape
    it = (L + THREADS - 1) // THREADS
    x = torch.zeros(n, it * THREADS, dtype=torch.float32)
    x[:, :L] = rows
    x = x.view(n, it, THREADS)
    s = torch.zeros(n, THREADS, dtype=torch.float32)
    for i in range(it):
        s = fma32(x[:, i], x[:, i], s)
    w = s.view(n, THREADS // 32, 32)
    lane = torch.arange(32)
    for d in (16, 8, 4, 2, 1):
        w = w + w[:, :, lane ^ d]
    tot = torch.zeros(n, dtype=torch.float32)
    for k in range(THREADS // 32):
        tot = tot + w[:, k, 0]
    return tot.double()


def seq_sqsum(x: torch.Tensor, dim: int) -> torch.Tensor:
    """fp32 sum of squares along ``dim`` in index order, one fmaf per element."""
    x = x.movedim(dim, -1)
    s = torch.zeros(x.shape[:-1], dtype=torch.float32)
    for k in range(x.shape[-1]):
        s = fma32(x[..., k], x[..., k], s)
    return s


def seq_sum64(x: torch.Tensor) -> torch.Tensor:
    """fp64 sum along the last dimension in index order."""
    s = torch.zeros(x.shape[:-1], dtype=torch.float64)
    for k in range(x.shape[-1]):
        s = s + x[..., k]
    return s


def sq_mean(s64: torch.Tensor, n: int) -> torch.Tensor:
    """fp32(sqrt(s))^2 / n in fp32."""
    nrm = torch.sqrt(s64).float()
    return (nrm * nrm) / torch.tensor(float(n), dtype=torch.float32)


def lerp32(s: torch.Tensor, e: torch.Tensor, w: float) -> torch.Tensor:
    d = e - s
    return fma32(w, d, s) if w < 0.5 else fma32(f32(f32(w) - 1.0), d, e)


def slice_means(rv: torch.Tensor, eps1: float) -> torch.Tensor:
    """The clamped row_var mean of each slice of ``rv`` [B, R]."""
    B, R = rv.shape
    blk = (R + THREADS - 1) // THREADS
    K = (R + blk - 1) // blk
    x = torch.zeros(B, K * blk, dtype=torch.float64)
    x[:, :R] = rv.double()
    s = seq_sum64(seq_sum64(x.view(B, K, blk)).view(B, K))
    m = (s / float(R)).float()
    e = torch.tensor(f32(eps1), dtype=torch.float32)
    return torch.where(m < e, e, m)


def _index(offset, shape, stride):
    """Flat index of every element of the tensor as [B, R, C] in logical order (unfactored: [1, 1, numel])."""
    f = factors(shape)
    idx = torch.arange(offset + max(1, math.prod(shape)), dtype=torch.int64).as_strided(shape, stride, offset)
    if f is None:
        return idx.reshape(1, 1, -1)
    return idx.reshape(*f)


def adafactor_step(p, g, state, tensors, groups, hp, t, fault=None):
    """(p, state, alpha, step) after update ``t`` (1-based) of the bucket.  ``p``, ``g`` (the gradient the update reads, already
    unscaled and clipped), ``state``: flat fp32; ``tensors``: [(offset, shape, stride, group)]; ``groups``: per group
    ``(lr, weight_decay, base_lr)`` with the scheduled lr; ``hp``: beta2_decay, eps1, eps2, d."""
    assert fault in (None,) + FAULTS
    p, g, state = (x.float().cpu().clone() for x in (p, g, state))
    tt = t - 1 if fault == "t_from_zero" else t
    w = f32(float(tt) ** hp["beta2_decay"]) if tt > 0 else math.inf
    eps1, eps2, d = hp["eps1"], hp["eps2"], hp["d"]
    eps1sq = torch.tensor(f32(eps1) if fault == "eps1_not_squared" else f32(eps1 * eps1), dtype=torch.float32)
    shapes = [tuple(s) for _, s, _, _ in tensors]
    soff, _ = state_offsets(shapes)
    alphas, steps = [], []
    for (o, shape, stride, gi), so in zip(tensors, soff):
        n = math.prod(shape)
        if n == 0:
            alphas.append(None), steps.append(None)
            continue
        lr, wd, base = groups[gi]
        chunks, whole, TR, TC = table([tuple(shape)])[0]
        E = _index(o, shape, stride)
        B, R, C = E.shape
        P, G = p[E], g[E]
        boxes = [E[b0:b0 + nb, r0:r0 + nr, c0:c0 + nc].reshape(-1) for b0, nb, r0, nr, c0, nc in chunks]

        def chunk_norm(x):
            rows = torch.zeros(len(boxes), CHUNK, dtype=torch.float32)
            for i, bx in enumerate(boxes):
                rows[i, :bx.numel()] = x[bx]
            return f32(math.sqrt(float(seq_sum64(box_sqsum(rows).view(1, -1))[0])))

        if fault == "chunk_crosses_tensor":         # the tensor's last chunk runs on into the next tensors' elements
            end = min(p.numel(), o + (n + CHUNK - 1) // CHUNK * CHUNK)
            pn = f32(math.sqrt(float(seq_sum64(box_sqsum(p[o:end].view(-1, CHUNK) if (end - o) % CHUNK == 0 else
                                                         torch.nn.functional.pad(p[o:end], (0, -(end - o) % CHUNK)).view(-1, CHUNK)
                                                         ).view(1, -1))[0])))
        else:
            pn = chunk_norm(p * torch.tensor(f32(1 - lr * wd)) if fault == "norm_after_decay" else p)
        q = pn / math.sqrt(n)
        rho = min(base if fault == "rho_unscheduled" else lr, 1 / (tt ** 0.5) if tt > 0 else math.inf)
        alpha = (q if q > eps2 else eps2) * rho
        f = factors(shape)
        if f is None:
            var = state[so:so + n]
            var = lerp32(var, G.reshape(-1) * G.reshape(-1), w)
            state[so:so + n] = var
            V = var.view(1, 1, n)
        else:
            rv = state[so:so + B * R].view(B, R).clone()
            cv = state[so + B * R:so + B * (R + C)].view(B, C).clone()
            if whole:
                rs, cs = seq_sqsum(G, 2).double(), seq_sqsum(G, 1).double()
            else:
                ntr, ntc = (R + TR - 1) // TR, (C + TC - 1) // TC
                Gp = torch.zeros(B, ntr * TR, ntc * TC, dtype=torch.float32)
                Gp[:, :R, :C] = G
                rs = seq_sum64(seq_sqsum(Gp.view(B, ntr * TR, ntc, TC), 3).double())[:, :R]
                cs = seq_sum64(seq_sqsum(Gp.view(B, ntr, TR, ntc * TC), 2).double().transpose(1, 2))[:, :C]
            sw = fault == "rows_cols_swapped"             # each mean divided by the other dimension's size
            rv = lerp32(rv, sq_mean(rs, R if sw else C), w)
            cv = lerp32(cv, sq_mean(cs, C if sw else R), w)
            state[so:so + B * R] = rv.reshape(-1)
            state[so + B * R:so + B * (R + C)] = cv.reshape(-1)
            if fault == "mean_over_wrong_dim":            # over every row of the tensor, not per slice
                m = slice_means(rv.reshape(1, B * R), eps1).expand(B)
            else:
                m = slice_means(rv, eps1)
            V = (rv.view(B, R, 1) * cv.view(B, 1, C)) / m.view(B, 1, 1)
        U = (1.0 / torch.sqrt(torch.where(V < eps1sq, eps1sq, V).double()).float()) * G
        u_flat = torch.zeros_like(p)
        u_flat[E] = U
        un = chunk_norm(u_flat)
        q = un / (math.sqrt(n) * (1.0 if fault == "denom_without_d" else d))
        step = f32(-alpha / (q if q > 1.0 else 1.0))
        alphas.append(alpha), steps.append(step)
        p[E] = fma32(step, U, P * torch.tensor(f32(1 - lr * wd), dtype=torch.float32))
    return p, state, alphas, steps


def adafactor_fp64(params, grads, hp, lrs, wds):
    """``torch.optim.Adafactor`` in fp64 over the gradient sequence: ``params`` the tensors (shaped), ``grads`` per update a
    list of gradients, ``lrs`` / ``wds`` per update and tensor."""
    ws = [torch.nn.Parameter(q.detach().double().clone()) for q in params]
    opt = torch.optim.Adafactor([{"params": [w_]} for w_ in ws], lr=1e-2, beta2_decay=hp["beta2_decay"],
                                eps=(hp["eps1"], hp["eps2"]), d=hp["d"], foreach=False)
    for gs, lr, wd in zip(grads, lrs, wds):
        for grp, gg, l_, w_ in zip(opt.param_groups, gs, lr, wd):
            grp["lr"], grp["weight_decay"] = l_, w_
            grp["params"][0].grad = gg.detach().double().clone()
        opt.step()
    return [w_.detach() for w_ in ws]
