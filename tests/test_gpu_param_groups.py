"""The grouped optimizer kernels on one GPU.  Oracle: the existing ungrouped kernel run on each tensor's padded segment (or, for
the sharded kernel, on the whole world) with its group's scalars -- the grouped kernels must match it bit for bit, since the
per-element sequence is the same and only the scalars' source differs.  Sharded cases use the emulated world of
tests/emulated_ranks.py; the end-to-end case trains a ResNet-18 through the public API."""
import pytest
import torch

import adamw_model as A
import dist_tuto.pth_b200 as b2
import param_groups_gpu_workers as WK
from emulated_ranks import CO_RESIDENT, WRAP, C, World, _bits, _untouched, _with_sentinel  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

MU, BETAS, EPS = 0.9, (0.8, 0.95), 1e-6


def _layout(sizes, gids):
    """Offsets at multiples of 4, the flat's size, the group map (one id per vector) and the padded segments."""
    offs, n = [], 0
    for s in sizes:
        offs.append(n)
        n += (s + 3) // 4 * 4
    segs = [(o, offs[i + 1] if i + 1 < len(offs) else n, gids[i]) for i, o in enumerate(offs)]
    gmap = torch.cat([torch.full(((hi - lo) // 4,), g, dtype=torch.uint8) for lo, hi, g in segs])
    return n, segs, gmap


def _groups(n_groups, seed):
    g = torch.Generator().manual_seed(seed)
    lrs = (torch.rand(n_groups, generator=g, dtype=torch.float64) * 0.1 + 1e-3).tolist()
    wds = [0.0 if i % 3 == 1 else w for i, w in enumerate((torch.rand(n_groups, generator=g, dtype=torch.float64) * 0.1).tolist())]
    return lrs, wds


def _cases():
    rng = torch.Generator().manual_seed(5)
    tiny = torch.randint(1, 10, (3000,), generator=rng).tolist()
    return [("one group", [7, 1, 300, 4, 13], [0] * 5, 1),
            ("alternating", [5, 8, 1, 4, 9, 33, 2, 6], [0, 1] * 4, 2),
            ("64 groups", [3 + 5 * i for i in range(64)], list(range(64)), 64),
            ("3000 tensors of 1..9", tiny, [i * 7 % 5 for i in range(3000)], 5),
            ("2^20 + 4", [1 << 19, 3, (1 << 19) - 3], [2, 0, 1], 3)]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
@pytest.mark.parametrize("kind", ["sgd", "sgd_nesterov", "adamw"])
def test_grouped_flat_kernels_equal_the_ungrouped_kernel_per_segment(C, case, kind):
    name, sizes, gids, n_groups = case
    n, segs, gmap = _layout(sizes, gids)
    lrs, wds = _groups(n_groups, len(sizes))
    gmap_d = gmap.cuda()
    nesterov = kind == "sgd_nesterov"
    for clip in (None, 0.05):
        for zero_grad in (True, False):
            g = torch.Generator().manual_seed(n + len(sizes))
            p0, g0, m0, v0 = (torch.randn(n, generator=g) for _ in range(4))
            v0 = v0.abs()
            bufs = {k: _with_sentinel(x) for k, x in (("p", p0), ("g", g0), ("m", m0), ("v", v0))}
            refs = {k: x.clone() for k, x in bufs.items()}
            kw, rkw = {}, {}
            if clip is not None:
                sq = torch.zeros(1, dtype=torch.float64, device="cuda")
                C.grad_sqnorm(bufs["g"][:n], sq, 0, torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda"))
                gn, rgn = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
                kw, rkw = dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=gn), dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=rgn)
            f = {k: x[:n] for k, x in bufs.items()}
            if kind == "adamw":
                t = 3
                per = [A.scalars64(lr, BETAS, EPS, wd, t) for lr, wd in zip(lrs, wds)]
                C.adamw_flat_grouped(f["p"], f["m"], f["v"], f["g"], gmap_d, per[0], [s[0] for s in per], [s[4] for s in per],
                                     zero_grad, **kw)
                for lo, hi, gi in segs:
                    r = {k: x[lo:hi] for k, x in refs.items()}
                    C.adamw_flat(r["p"], r["m"], r["v"], r["g"], per[gi], zero_grad, **rkw)
            else:
                C.sgd_flat_grouped(f["p"], f["m"], f["g"], gmap_d, lrs, wds, MU, zero_grad, nesterov, **kw)
                for lo, hi, gi in segs:
                    r = {k: x[lo:hi] for k, x in refs.items()}
                    C.sgd_flat(r["p"], r["m"], r["g"], lrs[gi], MU, wds[gi], zero_grad, nesterov, **rkw)
            torch.cuda.synchronize()
            what = f"{name} {kind} clip {clip} zero_grad {zero_grad}"
            for k in ("p", "m", "g") + (("v",) if kind == "adamw" else ()):
                assert _bits(bufs[k][:n], refs[k][:n]), f"{what}: {k}"
                assert _untouched(bufs[k][n:]), f"{what}: wrote behind {k}"
            if clip is not None:
                assert _bits(kw["grad_norm_out"], rkw["grad_norm_out"])
            if n_groups == 1:                      # one group is today's bucket-wide launch
                w = {k: _with_sentinel(x) for k, x in (("p", p0), ("g", g0), ("m", m0), ("v", v0))}
                if kind == "adamw":
                    C.adamw_flat(w["p"][:n], w["m"][:n], w["v"][:n], w["g"][:n], per[0], zero_grad, **rkw)
                else:
                    C.sgd_flat(w["p"][:n], w["m"][:n], w["g"][:n], lrs[0], MU, wds[0], zero_grad, nesterov, **rkw)
                assert _bits(w["p"][:n], bufs["p"][:n]) and _bits(w["m"][:n], bufs["m"][:n]), what


def test_grouped_launch_refusals(C):
    p, m, g = (torch.zeros(8, device="cuda") for _ in range(3))
    gmap = torch.zeros(2, dtype=torch.uint8, device="cuda")
    for lrs, wds in (([], []), ([0.1] * 65, [0.0] * 65), ([0.1], [0.0, 0.0])):
        with pytest.raises(RuntimeError, match="groups"):
            C.sgd_flat_grouped(p, m, g, gmap, lrs, wds, MU, True)
    with pytest.raises(RuntimeError, match="group_map"):
        C.sgd_flat_grouped(p, m, g, gmap[:1], [0.1], [0.0], MU, True)
    with pytest.raises(RuntimeError, match="group_map"):
        C.sgd_flat_grouped(p, m, g, gmap.to(torch.int32), [0.1], [0.0], MU, True)


def _sharded_map(n_pvec, world, n_groups, seed):
    """Group ids of n_pvec fp32 parameter vectors: random runs, with a run crossing every even rank's first boundary and a
    group change exactly at every odd one."""
    g = torch.Generator().manual_seed(seed)
    ids, cur = [], 0
    while len(ids) < n_pvec:
        cur = int(torch.randint(0, n_groups, (1,), generator=g))
        ids += [cur] * int(torch.randint(1, 40, (1,), generator=g))
    ids = ids[:n_pvec]
    per = n_pvec // world
    for r in range(1, world):
        b = r * per
        if b < n_pvec:
            ids[b] = ids[b - 1] if r % 2 == 0 else (ids[b - 1] + 1) % n_groups
    return torch.tensor(ids, dtype=torch.uint8)


def _run_sharded(C, world, sms, kind, wire, n_vec, max_blocks, zero_grad, pad_start, seed):
    epv = 8 if wire == torch.bfloat16 else 4
    n, per = n_vec * epv, n_vec * epv // world
    n_groups = 5
    lrs, wds = _groups(n_groups, seed)
    gmap = _sharded_map(n // 4, world, n_groups, seed)
    elem_gid = gmap.long().repeat_interleave(4)
    gen = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=gen)
    s0 = [[torch.randn(per, generator=gen).abs() for _ in range(world)] for _ in range(2)]
    g0 = [torch.randn(n, generator=gen) for _ in range(world)]
    scale = 1.0 / world
    t = 4
    per_sc = [A.scalars64(lr, BETAS, EPS, wd, t) for lr, wd in zip(lrs, wds)]

    def launch(grouped_gid):
        """One sharded step over a fresh world: grouped (grouped_gid None) or the ungrouped kernel with group grouped_gid's
        scalars everywhere.  Returns (params, state shards, grads) per rank."""
        W = World(world, sms, pad_start=pad_start)
        params = [_with_sentinel(p0) for _ in range(world)]
        st = [[_with_sentinel(x) for x in s0[i]] for i in range(2)]
        grads = [_with_sentinel(g, wire) for g in g0]
        gp, pp = [x.data_ptr() for x in grads], [x.data_ptr() for x in params]
        maps = [gmap[r * per // 4:(r + 1) * per // 4].cuda() for r in range(world)]
        blocks = min(max_blocks, max(1, ((n_vec // world + 511) // 512 + 1) // 2))
        bf16 = wire == torch.bfloat16
        if kind == "sgd":
            if grouped_gid is None:
                fn = lambda r: C.sharded_sgd_grouped(bf16, gp, pp, W.sig_ptrs, st[0][r][:per], maps[r], n_vec, lrs, wds, MU, False,  # noqa: E731
                                                     scale, zero_grad, r, world, max_blocks)
            else:
                fn = lambda r: C.sharded_sgd(bf16, gp, pp, W.sig_ptrs, st[0][r][:per], n_vec, lrs[grouped_gid], MU,  # noqa: E731
                                             wds[grouped_gid], False, scale, zero_grad, r, world, max_blocks)
        else:
            if grouped_gid is None:
                fn = lambda r: C.sharded_adamw_grouped(bf16, gp, pp, W.sig_ptrs, st[0][r][:per], st[1][r][:per], maps[r], n_vec,  # noqa: E731
                                                       per_sc[0], [s[0] for s in per_sc], [s[4] for s in per_sc], scale,
                                                       zero_grad, r, world, max_blocks)
            else:
                fn = lambda r: C.sharded_adamw(bf16, gp, pp, W.sig_ptrs, st[0][r][:per], st[1][r][:per], n_vec,  # noqa: E731
                                               per_sc[grouped_gid], scale, zero_grad, r, world, max_blocks)
        W.launch(blocks, fn)
        for r in range(world):
            assert _untouched(params[r][n:]) and _untouched(grads[r][n:]) and all(_untouched(s[r][per:]) for s in st)
        return ([x[:n].cpu() for x in params], [[x[:per].cpu() for x in s] for s in st], [x[:n].cpu() for x in grads])

    got = launch(None)
    want_p = [torch.empty(n) for _ in range(world)]
    want_s = [[torch.empty(per) for _ in range(world)] for _ in range(2)]
    for gi in range(n_groups):
        ref = launch(gi)
        sel = elem_gid == gi
        for r in range(world):
            want_p[r][sel] = ref[0][r][sel]
            for i in range(2):
                want_s[i][r][sel[r * per:(r + 1) * per]] = ref[1][i][r][sel[r * per:(r + 1) * per]]
        for r in range(world):
            assert torch.equal(got[2][r].view(torch.int16 if wire == torch.bfloat16 else torch.int32),
                               ref[2][r].view(torch.int16 if wire == torch.bfloat16 else torch.int32))
    what = f"{kind} world {world} {wire} n_vec {n_vec} max_blocks {max_blocks}"
    for r in range(world):
        assert _bits(got[0][r], want_p[r]), f"{what}: params of rank {r}"
        for i in range(2 if kind == "adamw" else 1):
            assert _bits(got[1][i][r], want_s[i][r]), f"{what}: state {i} of rank {r}"


@CO_RESIDENT
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_sharded_grouped_equals_the_ungrouped_kernel_per_group(C, world, kind):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    k = 0
    for wire in (torch.float32, torch.bfloat16):
        for sl, mb in ((1, 1), (513, 3), (2 * 1024 * 3 + 1, sms // world)):
            _run_sharded(C, world, sms, kind, wire, world * sl, mb, k % 2 == 0, WRAP if k == 3 else 0, 100 * world + k)
            k += 1


def test_resnet18_with_no_decay_groups_trains_like_torch():
    b2.launch(WK.w_resnet_groups, size=1, backend="b200", join_timeout_s=600)
