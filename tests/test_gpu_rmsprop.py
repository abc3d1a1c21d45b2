"""FlatRMSprop's kernels on one GPU: every instance of ``rmsprop_flat`` (csrc/rmsprop.cu) bit for bit against
tests/rmsprop_model.py with sentinels behind every buffer, the clip / scaled / grouped / capturable instances against the plain
one fed the same scalars, the kernel against ``torch.optim.RMSprop`` on CUDA and fp64, the RMSprop instances of the sharded
kernel (csrc/sharded_sgd.cu) at emulated worlds 1-8 (the harness of tests/emulated_ranks.py), a captured
DDP step against eager steps, and a ResNet-18 trained through ``DistributedDataParallel`` + ``FlatRMSprop`` under bf16
autocast."""
import math

import pytest
import torch

import comm_model as M
import rmsprop_model as R
import sharded_sgd_model as S
from adamw_model import clip_coef, f32
from emulated_ranks import CO_RESIDENT, C, World, _bits, _untouched, _with_sentinel, sms  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

SIZES = [1, 2, 3, 4, 5, 6, 7, 1023, 1024, 1025, 1026, 1027, 256 * 4 * 7 + 3, 1 << 20, (1 << 20) + 1, 3 * 1000003]
# (momentum, centered, weight decay): every momentum x centered combination, decay on in two of them
OPTIONS = [(0.0, False, 0.0), (0.9, False, 0.05), (0.0, True, 0.05), (0.9, True, 0.0)]
HP = dict(lr=0.01, alpha=0.9, eps=1e-3)


def _sc(opt, lr=HP["lr"]):
    mu, _, wd = opt
    return R.scalars64(lr, HP["alpha"], HP["eps"], wd, mu)


def _state(n, seed):
    """p, g, square_avg, grad_avg, momentum_buffer; a tenth of the elements has a zero gradient and empty states."""
    gen = torch.Generator().manual_seed(seed)
    p, g = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 0.1
    ga = torch.randn(n, generator=gen) * 0.01
    sq = ga * ga + torch.rand(n, generator=gen) * 1e-3
    buf = torch.randn(n, generator=gen) * 0.1
    z = torch.rand(n, generator=gen) < 0.1
    g[z], sq[z], ga[z], buf[z] = 0, 0, 0, 0
    return p, g, sq, ga, buf


def _model(opt, g, p, sq, ga, buf, lr=HP["lr"], wd=None):
    mu, centered, wd0 = opt
    return R.rmsprop_update(g, p, sq, ga if centered else None, buf if mu > 0 else None, lr, HP["alpha"], HP["eps"],
                            wd0 if wd is None else wd, mu, centered)


def _dev_states(opt, sq, ga, buf):
    """Sentinel-backed device copies of the states the options have (None for the others)."""
    mu, centered, _ = opt
    return _with_sentinel(sq), _with_sentinel(ga) if centered else None, _with_sentinel(buf) if mu > 0 else None


def _check_states(what, n, opt, dsq, dga, dbuf, want):
    _, wsq, wga, wbuf = want
    assert _bits(dsq[:n], wsq) and _untouched(dsq[n:]), f"{what}: square_avg"
    if dga is not None:
        assert _bits(dga[:n], wga) and _untouched(dga[n:]), f"{what}: grad_avg"
    if dbuf is not None:
        assert _bits(dbuf[:n], wbuf) and _untouched(dbuf[n:]), f"{what}: momentum_buffer"


def _views(n, *bufs):
    return [b[:n] if b is not None else None for b in bufs]


# ----------------------------------------------------------------------------------------------- rmsprop_flat
@pytest.mark.parametrize("n", SIZES)
def test_rmsprop_flat_matches_the_model_bit_for_bit(C, n):
    for k, opt in enumerate(OPTIONS):
        p, g, sq, ga, buf = _state(n, 4 * n + k)
        zero_grad = k % 2 == 0
        dp, dg = _with_sentinel(p), _with_sentinel(g)
        dsq, dga, dbuf = _dev_states(opt, sq, ga, buf)
        want = (p, sq, ga, buf)
        for t in (1, 2):
            C.rmsprop_flat(*_views(n, dp, dsq, dga, dbuf, dg), _sc(opt), opt[1], zero_grad)
            want = _model(opt, g, *want)
            what = f"n {n} options {opt} step {t}"
            assert _bits(dp[:n], want[0]) and _untouched(dp[n:]), f"{what}: p"
            _check_states(what, n, opt, dsq, dga, dbuf, want)
            assert _untouched(dg[n:]), f"{what}: a sentinel behind g changed"
            if zero_grad:
                assert not dg[:n].any(), what
                dg[:n].copy_(g)
            else:
                assert _bits(dg[:n], g), what


def _instances_case(C, n, opt, seed):
    p, g, sq, ga, buf = _state(n, seed)
    dev = [x.cuda() if x is not None else None for x in (p, g, sq, ga if opt[1] else None, buf if opt[0] > 0 else None)]
    return (p, g, sq, ga, buf), dev


def _plain(C, opt, dev_state, g, lr=HP["lr"], wd=None, zero_grad=True):
    """The plain instance on copies of the device state, fed gradient g and the given lr / weight decay."""
    p, _, sq, ga, buf = (x.clone() if x is not None else None for x in dev_state)
    mu, centered, wd0 = opt
    gg = g.clone()
    C.rmsprop_flat(p, sq, ga, buf, gg, R.scalars64(lr, HP["alpha"], HP["eps"], wd0 if wd is None else wd, mu), centered, zero_grad)
    return p, sq, ga, buf


def _same(a, b):
    return all((x is None and y is None) or _bits(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("n", [5, 1027, (1 << 20) + 3])
@pytest.mark.parametrize("k", range(len(OPTIONS)))
def test_clip_instance_equals_the_plain_instance_on_the_clipped_gradient(C, n, k):
    opt = OPTIONS[k]
    _, dev = _instances_case(C, n, opt, 3 * n + k)
    sqn = torch.zeros(2, dtype=torch.float64, device="cuda")
    ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
    C.grad_sqnorm(dev[1], sqn, 0, ws)
    C.grad_sqnorm(torch.randn(4096, device="cuda"), sqn, 1, ws)        # a second bucket's squares count towards the norm
    norm = torch.zeros(1, device="cuda")
    coef = clip_coef(sqn.cpu().tolist(), 0.5)
    assert coef < 1.0
    want = _plain(C, opt, dev, dev[1] * torch.tensor(coef, device="cuda"))
    p, g, sq, ga, buf = (x.clone() if x is not None else None for x in dev)
    C.rmsprop_flat(p, sq, ga, buf, g, _sc(opt), opt[1], True, max_grad_norm=0.5, sqnorms=sqn, grad_norm_out=norm)
    assert _same((p, sq, ga, buf), want) and not g.any()
    assert float(norm) == f32(math.sqrt(sum(sqn.cpu().tolist())))


@pytest.mark.parametrize("scale", [1024.0, 3000.0, 2.0 ** -24])
@pytest.mark.parametrize("k", range(len(OPTIONS)))
def test_scaled_instance_equals_the_plain_instance_on_the_unscaled_gradient(C, scale, k):
    """torch's CUDA multiply by fp32(1 / double(S)) keeps subnormals, as the scaled instances do."""
    opt, n = OPTIONS[k], 4099
    _, dev = _instances_case(C, n, opt, 11 + k)
    S_ = torch.tensor([scale], device="cuda")
    inv = S_.double().reciprocal().float()
    want = _plain(C, opt, dev, dev[1] * inv)
    p, g, sq, ga, buf = (x.clone() if x is not None else None for x in dev)
    C.rmsprop_flat(p, sq, ga, buf, g, _sc(opt), opt[1], True, grad_scale=S_)
    assert _same((p, sq, ga, buf), want) and not g.any()


def _group_map(n, n_groups, seed):
    ids = torch.randint(0, n_groups, ((n + 3) // 4,), generator=torch.Generator().manual_seed(seed), dtype=torch.int64)
    return ids.to(torch.uint8)


def _grouped_want(C, opt, dev, ids, lrs, wds):
    """Per element: the plain instance run with the element's group's lr and weight decay."""
    n = dev[0].numel()
    elem = ids.long().repeat_interleave(4)[:n].cuda()
    out = None
    for gi, (lr, wd) in enumerate(zip(lrs, wds)):
        r = _plain(C, opt, dev, dev[1], lr=lr, wd=wd)
        out = r if out is None else tuple(torch.where(elem == gi, a, b) if a is not None else None for a, b in zip(r, out))
    return out


@pytest.mark.parametrize("n", [3, 1027, (1 << 20) + 1])
@pytest.mark.parametrize("k", range(len(OPTIONS)))
def test_grouped_instance_equals_the_plain_instance_per_group(C, n, k):
    opt = OPTIONS[k]
    _, dev = _instances_case(C, n, opt, 5 * n + k)
    lrs, wds = [0.01, 0.003, 0.02], [0.0, 0.05, 0.2]
    ids = _group_map(n, 3, n)
    want = _grouped_want(C, opt, dev, ids, lrs, wds)
    p, g, sq, ga, buf = (x.clone() if x is not None else None for x in dev)
    C.rmsprop_flat_grouped(p, sq, ga, buf, g, ids.cuda(), _sc(opt), opt[1], lrs, wds, True)
    assert _same((p, sq, ga, buf), want) and not g.any()


def _block(C, lrs, wds, schedule=None, steps=0):
    lay = C.flat_scalars_layout()
    table = torch.zeros(lay["table_bytes"], dtype=torch.uint8, device="cuda")
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    block = torch.zeros(lay["block_bytes"], dtype=torch.uint8, device="cuda")
    C.flat_scalars_sync(table, counter, block, lrs, wds, schedule=schedule, steps=steps)
    return table, counter, block


@pytest.mark.parametrize("n", [5, 1027, (1 << 20) + 3])
@pytest.mark.parametrize("kind", ["plain", "grouped", "clip", "scaled", "scaled_grouped_clip"])
def test_capturable_instances_equal_the_eager_ones(C, n, kind):
    """The capturable instances fed the block's lr / weight decay compute the eager instances' bits, and a set found_inf
    writes only the zeroing."""
    for k, opt in enumerate(OPTIONS):
        _, dev = _instances_case(C, n, opt, 7 * n + k)
        grouped, clip, scaled = "grouped" in kind, "clip" in kind, "scaled" in kind
        lrs, wds = ([0.01, 0.003], [0.05, 0.0]) if grouped else ([0.007], [opt[2]])
        _, _, block = _block(C, lrs, wds)
        ids = _group_map(n, 2, n).cuda() if grouped else None
        kw, eager_kw = {}, {}
        if clip:
            sqn = torch.zeros(1, dtype=torch.float64, device="cuda")
            ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
            C.grad_sqnorm(dev[1], sqn, 0, ws, grad_scale=torch.tensor([512.0], device="cuda") if scaled else None)
            kw = eager_kw = dict(max_grad_norm=0.05, sqnorms=sqn)
        if scaled:
            S_ = torch.tensor([512.0], device="cuda")
            eager_kw = dict(eager_kw, grad_scale=S_)
            kw = dict(kw, grad_scale=S_, found_inf=torch.zeros(1, device="cuda"))
        want = [x.clone() if x is not None else None for x in dev]
        wp, wg, wsq, wga, wbuf = want
        if grouped:
            C.rmsprop_flat_grouped(wp, wsq, wga, wbuf, wg, ids, _sc(opt), opt[1], lrs, wds, True, **eager_kw)
        else:
            C.rmsprop_flat(wp, wsq, wga, wbuf, wg, _sc(opt, lr=lrs[0]), opt[1], True, **eager_kw)
        p, g, sq, ga, buf = (x.clone() if x is not None else None for x in dev)
        C.rmsprop_flat_cap(p, sq, ga, buf, g, ids, block, _sc(opt, lr=123.0), opt[1], True, **kw)
        assert _same((p, sq, ga, buf), (wp, wsq, wga, wbuf)) and not g.any(), (kind, opt)
        if scaled:                                     # a skipped step: only the zeroing
            p, g, sq, ga, buf = (x.clone() if x is not None else None for x in dev)
            kw["found_inf"] = torch.ones(1, device="cuda")
            C.rmsprop_flat_cap(p, sq, ga, buf, g, ids, block, _sc(opt), opt[1], True, **kw)
            assert _same((p, sq, ga, buf), (dev[0], dev[2], dev[3], dev[4])) and not g.any(), (kind, opt)


def test_kernel_error_against_fp64_is_within_4x_torch_fp32():
    """50 updates with fresh gradients; the kernel (through FlatRMSprop) and torch.optim.RMSprop on CUDA from the same
    inputs, for every option combination.  Bound: 4x torch's fp32 error against fp64 plus one ulp of the largest parameter."""
    from dist_tuto.pth_b200 import FlatRMSprop
    n, steps = 50001, 50
    gen = torch.Generator().manual_seed(5)
    p0 = torch.randn(n, generator=gen)
    grads = [torch.randn(n, generator=gen) * 0.1 + 0.01 for _ in range(steps)]
    for mu, centered, wd in OPTIONS:
        hp = dict(lr=HP["lr"], alpha=HP["alpha"], eps=HP["eps"], weight_decay=wd, momentum=mu, centered=centered)
        lin = torch.nn.Linear(n, 1, bias=False).cuda()
        with torch.no_grad():
            lin.weight.copy_(p0.view(1, n))
        opt = FlatRMSprop(lin, **hp)
        w = torch.nn.Parameter(p0.clone().cuda())
        topt = torch.optim.RMSprop([w], foreach=False, **hp)
        for g in grads:
            lin._grad_bucket.flat[:n].copy_(g)
            opt.step()
            w.grad = g.cuda()
            topt.step()
        ref = R.rmsprop_fp64(p0, grads, [HP["lr"]] * steps, HP["alpha"], HP["eps"], wd, mu, centered)
        e_k = float((lin.weight.detach().view(-1).double().cpu() - ref).abs().max())
        e_t = float((w.detach().double().cpu() - ref).abs().max())
        big = ref.abs().max().float()
        ulp = float(torch.nextafter(big, torch.tensor(float("inf"))) - big)
        assert e_k <= 4 * e_t + ulp, (mu, centered, wd, e_k, e_t, ulp)
        print(f"momentum {mu} centered {centered} wd {wd}: kernel error {e_k:.3e}, torch fp32 error {e_t:.3e}, bit-equal to "
              f"torch's CUDA RMSprop: {torch.equal(lin.weight.detach().view(-1), w.detach())}")


def test_refusals(C):
    p, g, sq, ga, buf = (torch.zeros(64, device="cuda") for _ in range(5))
    sc = _sc((0.9, True, 0.0))
    with pytest.raises(RuntimeError, match="grad_avg"):
        C.rmsprop_flat(p, sq, None, buf, g, sc, True, True)
    with pytest.raises(RuntimeError, match="momentum_buffer"):
        C.rmsprop_flat(p, sq, ga, None, g, sc, True, True)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        C.rmsprop_flat(p, sq[:60], ga, buf, g, sc, True, True)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        C.rmsprop_flat(p[1:], sq[1:], ga[1:], buf[1:], g[1:], sc, True, True)
    with pytest.raises(RuntimeError, match="scalars"):
        C.rmsprop_flat(p, sq, ga, buf, g, sc[:5], True, True)
    with pytest.raises(RuntimeError, match="grad_scale"):
        C.rmsprop_flat(p, sq, ga, buf, g, sc, True, True, grad_scale=torch.ones(2, device="cuda"))
    _, _, block = _block(C, [0.01], [0.0])
    with pytest.raises(RuntimeError, match="found_inf"):
        C.rmsprop_flat_cap(p, sq, ga, buf, g, None, block, sc, True, True, grad_scale=torch.ones(1, device="cuda"))
    pad = torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda")
    one = lambda t, k: [t.data_ptr()] * k          # noqa: E731
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.sharded_rmsprop(False, one(g, 3), one(p, 3), one(pad, 3), sq, ga, buf, 16, sc, True, 1.0, True, 0, 3)
    with pytest.raises(RuntimeError, match="world"):
        C.sharded_rmsprop(False, one(g, 9), one(p, 9), one(pad, 9), sq, ga, buf, 18, sc, True, 1.0, True, 0, 9)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        C.sharded_rmsprop(False, one(g, 2), one(p, 2), one(pad, 2), sq[:8], ga, buf, 16, sc, True, 1.0, True, 0, 2)


# ----------------------------------------------------------------------------------------------- emulated ranks
def _sharded_model(gs, params, states, opt, scale, kind, ids, lrs, wds):
    """Every rank's parameter flat and state shards after one sharded RMSprop step (as sharded_sgd_model); grouped kinds
    take each vector's group's lr / weight decay from this rank's ids."""
    world, n = len(gs), gs[0].numel()
    new_p = [p.clone() for p in params]
    new_s = [list(s) for s in states]
    for r in range(world):
        lo, hi = S.slice_of(r, world, n)
        g = M.reduce_scaled([x[lo:hi].float() for x in gs], scale)
        sq, ga, buf = states[r]
        if ids is None:
            out = _model(opt, g, params[r][lo:hi], sq, ga, buf, lr=lrs[0], wd=wds[0])
        else:
            elem = ids[r].long().repeat_interleave(4)[:hi - lo]
            out = None
            for gi, (lr, wd) in enumerate(zip(lrs, wds)):
                o = _model(opt, g, params[r][lo:hi], sq, ga, buf, lr=lr, wd=wd)
                out = o if out is None else tuple(torch.where(elem == gi, a, b) if a is not None else None for a, b in zip(o, out))
        p, new_s[r][0], nga, nbuf = out
        new_s[r][1] = nga if opt[1] else ga
        new_s[r][2] = nbuf if opt[0] > 0 else buf
        for q in range(world):
            new_p[q][lo:hi] = p
    return new_p, new_s


def run_sharded(C, W, n_vec, max_blocks, wire, zero_grad, opt, kind, seed, steps=3, against_kernels=False):
    """``steps`` sharded RMSprop steps over the emulated world, every buffer checked against the model; ``kind``: "plain",
    "grouped" (sharded_rmsprop_grouped), "cap" or "cap_grouped" (sharded_rmsprop_cap with the block).  against_kernels (fp32,
    plain): the parameters and states also equal the two-shot all-reduce followed by rmsprop_flat, bit for bit."""
    world = W.world
    mu, centered, wd = opt
    epv = M.elems_per_vec(wire)
    n, per = n_vec * epv, n_vec * epv // world
    scale = 1.0 / world
    blocks = S.grid_blocks(n_vec, world, max_blocks)
    p0, m0, m_full = S.make_state(world, n, seed)
    sq_full = m_full * m_full + 1e-4
    st0 = [[sq_full[r * per:(r + 1) * per].clone(), m0[r].clone() * 0.1 if centered else None, m0[r].clone() if mu > 0 else None]
           for r in range(world)]
    params = [_with_sentinel(p) for p in p0]
    dst = [[_with_sentinel(x) if x is not None else None for x in s] for s in st0]
    grads = [_with_sentinel(torch.zeros(n), wire) for _ in range(world)]
    gp, pp = [g.data_ptr() for g in grads], [p.data_ptr() for p in params]
    grouped, cap = "grouped" in kind, kind.startswith("cap")
    lrs, wds = ([0.01, 0.004, 0.02], [wd, 0.1, 0.0]) if grouped else ([HP["lr"]], [wd])
    ids = [_group_map(per, len(lrs), 31 * seed + r) for r in range(world)] if grouped else None
    dids = [i.cuda() for i in ids] if grouped else None
    block = _block(C, lrs, wds)[2] if cap else None
    what = f"sharded_rmsprop {kind} world {world} n_vec {n_vec} max_blocks {max_blocks} {wire} {opt} zero_grad {zero_grad}"
    if against_kernels:
        assert wire == torch.float32 and kind == "plain"
        ref = [p0[0].cuda(), sq_full.cuda(), torch.cat([s[1] for s in st0]).cuda() if centered else None,
               torch.cat([s[2] for s in st0]).cuda() if mu > 0 else None]
    for it in range(steps):
        gs = M.make_inputs(world, n, wire, 7919 * seed + it, specials=False)
        for r in range(world):
            if zero_grad and it > 0:
                assert not bool(grads[r][:n].any()), f"{what} step {it}: rank {r}'s bucket was not left zeroed"
            grads[r][:n].copy_(gs[r])
        if against_kernels:
            bufs = [g[:n].clone() for g in grads]
            bptr = [b.data_ptr() for b in bufs]
            W.launch(M.grid_blocks(M.TWOSHOT, n_vec, world, max_blocks),
                     lambda r: C.allreduce(M.TWOSHOT, False, bptr, W.sig_ptrs, 0, None, None, n_vec, scale, r, world, max_blocks))
            C.rmsprop_flat(ref[0], ref[1], ref[2], ref[3], bufs[0], _sc(opt), centered, False)

        def launch(r):
            sv = [x[:per] if x is not None else None for x in dst[r]]
            bf16 = wire == torch.bfloat16
            if cap:
                C.sharded_rmsprop_cap(bf16, gp, pp, W.sig_ptrs, *sv, dids[r] if grouped else None, block, n_vec, _sc(opt, lr=9.0),
                                      centered, scale, zero_grad, r, world, max_blocks)
            elif grouped:
                C.sharded_rmsprop_grouped(bf16, gp, pp, W.sig_ptrs, *sv, dids[r], n_vec, _sc(opt), centered, lrs, wds, scale,
                                          zero_grad, r, world, max_blocks)
            else:
                C.sharded_rmsprop(bf16, gp, pp, W.sig_ptrs, *sv, n_vec, _sc(opt), centered, scale, zero_grad, r, world, max_blocks)
        W.launch(blocks, launch)
        wp, ws = _sharded_model(gs, p0, st0, opt, scale, kind, ids, lrs, wds)
        M.assert_bits_equal(f"{what} step {it}: params", [p[:n] for p in params], wp, 4)
        for j, name in enumerate(("square_avg", "grad_avg", "momentum_buffer")):
            if dst[0][j] is not None:
                M.assert_bits_equal(f"{what} step {it}: {name}", [d[j][:per] for d in dst], [w[j] for w in ws], 4)
        M.assert_bits_equal(f"{what} step {it}: gradient buckets", [g[:n] for g in grads],
                            [torch.zeros_like(g) if zero_grad else g.clone() for g in gs], epv)
        for r in range(world):
            assert _untouched(params[r][n:]) and _untouched(grads[r][n:]) and \
                all(_untouched(x[per:]) for x in dst[r] if x is not None), f"{what} step {it}: rank {r} wrote behind a buffer"
        if against_kernels:
            name = f"{what} step {it}: two-shot all-reduce + rmsprop_flat"
            M.assert_bits_equal(name + ": params", [p[:n] for p in params], [ref[0].cpu()] * world, 4)
            for j in range(3):
                if ref[j + 1] is not None:
                    M.assert_bits_equal(f"{name}: state {j}", [torch.cat([d[j][:per] for d in dst])], [ref[j + 1].cpu()], 4)
        p0, st0 = wp, ws


KINDS = ["plain", "grouped", "cap", "cap_grouped"]


def _cases(world, sms):
    out = []
    for m, mb in enumerate([1, 3, sms // world]):
        tail = M.THREADS * mb                 # one pass of the RMSprop instances' loop (unroll 1) at mb CTAs
        for i, sl in enumerate([1, 511, 513, tail - 1, tail + 1, 3 * tail + 1]):
            k = 6 * m + i
            out.append((world * sl, mb, torch.bfloat16 if k % 2 else torch.float32, (k // 2) % 2 == 0, OPTIONS[k % 4],
                        KINDS[(k + world) % 4]))
    return out


@CO_RESIDENT
@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_rmsprop_matches_the_model_bit_for_bit(C, sms, world):
    for k, (n_vec, mb, wire, zero_grad, opt, kind) in enumerate(_cases(world, sms)):
        run_sharded(C, World(world, sms), n_vec, mb, wire, zero_grad, opt, kind, seed=100 * world + k)


@CO_RESIDENT
@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_rmsprop_fp32_equals_allreduce_then_rmsprop_flat(C, sms, world):
    big = (524288 + world - 1) // world * world
    for k, (n_vec, mb) in enumerate([(world * 513, 1), (world * 3073, 3), (big, sms // world)]):
        run_sharded(C, World(world, sms), n_vec, mb, torch.float32, k % 2 == 0, OPTIONS[(world + k) % 4], "plain",
                    seed=50 * world + k, against_kernels=True)


# ----------------------------------------------------------------------------------------------- module level
def test_captured_ddp_step_equals_eager_steps():
    """capturable=True: replays of one captured DDP step (forward, backward with the exchange, step()) equal eager steps bit
    for bit, for every option combination with groups, clipping and a schedule; an eager step does not synchronise."""
    import dist_tuto.pth_b200 as b2
    import capturable_workers as CW

    def make_for(mu, centered, wd):
        def make(ddp, m, **kw):
            groups = [{"params": [p for p in m.parameters() if p.ndim <= 1], "weight_decay": 0.0, "lr": 0.002}]
            return b2.FlatRMSprop(ddp, lr=3e-3, alpha=0.9, eps=0.0316, momentum=mu, centered=centered, weight_decay=wd,
                                  max_grad_norm=1.0, param_groups=groups,
                                  lr_schedule=b2.LRSchedule(decay="cosine", total_steps=12, min_factor=0.1), **kw)
        return make

    def state(m, opt):
        flats = opt.square_avg_flats + opt.grad_avg_flats + opt.momentum_buffer_flats
        return ([t.detach().clone(memory_format=torch.contiguous_format) for t in m.state_dict().values()],
                [f.clone() for f in flats], opt.grad_norm(), opt.state_dict()["steps"])

    dev = torch.device("cuda", 0)
    # the two runs compare bit for bit, so cuDNN's backward must not pick a nondeterministic algorithm (other test modules
    # turn TF32 off for the whole session, which changes cuDNN's choice)
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        for mu, centered, wd in OPTIONS:
            make = make_for(mu, centered, wd)
            eager = state(*CW.run(make, 12, False, dev))
            graph = state(*CW.run(make, 12, True, dev))
            what = (mu, centered, wd)
            assert CW._bits_equal(eager[0], graph[0]), (what, "parameters / buffers")
            assert CW._bits_equal(eager[1], graph[1]), (what, "optimizer state")
            assert eager[2:] == graph[2:], (what, eager[2:], graph[2:])
            assert graph[3] == 12
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved
    m = CW.net().cuda()
    ddp = b2.DistributedDataParallel(m)
    opt = make_for(0.9, True, 0.01)(ddp, m, capturable=True)
    x, y = torch.randn(4, 3, 8, 8, device="cuda"), torch.randint(0, 10, (4,), device="cuda")
    for it in range(3):
        torch.nn.functional.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        if it == 2:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    ddp.remove_hooks()


def test_ddp_resnet18_trains_like_torch_rmsprop_under_bf16_autocast():
    import dist_tuto.pth_b200 as b2
    import rmsprop_gpu_workers as WK
    b2.launch(WK.w_resnet, size=1, backend="b200", join_timeout_s=600)


def test_world_one_sharded_is_the_unsharded_path():
    import dist_tuto.pth_b200 as b2
    import rmsprop_gpu_workers as WK
    b2.launch(WK.w_world1, size=1, backend="b200", join_timeout_s=600)
