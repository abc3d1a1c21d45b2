"""The all-to-all with variable segments (csrc/allreduce.cu alltoallv_kernel) on ONE GPU with W emulated ranks, bit for bit
against tests/all_to_all_v_model.py.

The harness is tests/emulated_ranks.py's: each rank has its own staging buffer, signal pad and stream, the W launches
go out back to back, and no case runs more CTAs than the GPU has SMs.  Every segment of every input and output sits between
random sentinel bytes; whole output buffers are compared with the model, every input buffer is checked unchanged, and the
per-block epochs must advance by the model's barrier count on every rank.  One staging buffer per rank serves all calls of a
test, so its header and both halves are reused.  The last tests drive ``SymmWorld.all_to_all_v_`` for W ranks built over
the emulated buffers.
"""
import pytest
import torch

import all_to_all_v_model as AM
import all_to_all_v_workers as AW
import collectives_model as CM
import comm_model as M
import emulated_ranks as E
import reduce_scatter_alltoall_model as RS
from emulated_ranks import C, _bytes, _unaligned, pytestmark, sms  # noqa: F401

GAP = 32                                         # sentinel bytes at least between two segments


class A2AV:
    """The staging buffers of W emulated ranks (header + 2 x W x chunk bytes each) and the kernel's grid."""

    def __init__(self, C, W):
        self.chunk, header = C.alltoallv_config()
        nbytes = header + 2 * W.world * self.chunk
        self.bufs = [torch.full((nbytes,), 0x77, dtype=torch.uint8, device="cuda") for _ in range(W.world)]
        self.ptrs = [b.data_ptr() for b in self.bufs]

    def grid(self, mb):
        return min(-(-self.chunk // 16 // M.THREADS), mb)


def _layout(sizes, mis):
    """Byte offsets of segments of ``sizes`` bytes in one buffer: each behind at least GAP sentinel bytes, at ``mis[i]`` bytes
    past a 16-byte boundary; and the buffer's length."""
    offs, at = [], 0
    for i, n in enumerate(sizes):
        at = (at + GAP + 15) // 16 * 16 + mis[i]
        offs.append(at)
        at += n
    return offs, at + GAP


def _epochs(W):
    return torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu().long() & 0xFFFFFFFF


def a2av_call(C, W, A, lens, expect, es, mis_src, mis_dst, mb, seed):
    """One call: ``lens[s][d]`` elements of ``es`` bytes from rank s to rank d, ``expect[r][p]`` elements rank r expects from
    p; segment i of every input (output) sits ``mis_src[i]`` (``mis_dst[i]``) bytes past a 16-byte boundary."""
    world = W.world
    g = torch.Generator().manual_seed(seed)
    sbytes = [[n * es for n in row] for row in lens]
    dbytes = [[n * es for n in row] for row in expect]
    ins, outs, srcs, dsts, sends, out_offs = [], [], [], [], [], []
    for r in range(world):
        so, sn = _layout(sbytes[r], mis_src)
        do, dn = _layout(dbytes[r], mis_dst)
        x = torch.randint(0, 256, (sn,), generator=g, dtype=torch.uint8)
        y = torch.randint(0, 256, (dn,), generator=g, dtype=torch.uint8)
        sends.append([x[so[d]:so[d] + sbytes[r][d]] for d in range(world)])
        out_offs.append(do)
        ins.append(x.cuda())
        outs.append(y.cuda())
        srcs.append([ins[r][so[d]:so[d] + sbytes[r][d]] for d in range(world)])
        dsts.append([outs[r][do[p]:do[p] + dbytes[r][p]] for p in range(world)])
    in_before = [x.cpu() for x in ins]
    want = AM.predict(sends, [y.cpu() for y in outs], out_offs, dbytes)
    ep0 = _epochs(W)
    blocks = A.grid(mb)
    W.launch(blocks, lambda r: C.alltoallv(A.ptrs, W.sig_ptrs, srcs[r], sbytes[r], dsts[r], dbytes[r], r, world, mb))
    what = f"all-to-allv world {world} max_blocks {mb} element {es} mis {mis_src[:2]} / {mis_dst[:2]} lens {lens}"[:400]
    for r in range(world):
        assert torch.equal(outs[r].cpu(), want[r]), f"{what}: rank {r}'s output"
        assert torch.equal(ins[r].cpu(), in_before[r]), f"{what}: rank {r}'s input changed"
    ep = _epochs(W)
    step = torch.zeros(M.MAX_BLOCKS, dtype=torch.long)
    step[:blocks] = AM.barriers(sbytes, A.chunk)
    for r in range(world):
        assert torch.equal(ep[r], (ep0[r] + step) & 0xFFFFFFFF), f"{what}: rank {r}'s per-block epochs"


def _matrix(pattern, world, n, g, choices):
    """A W x W matrix of element counts: "equal" (n everywhere), "zero", "silent" (one rank sends nothing), "hot" (every
    rank sends only to one destination), "random" (entries drawn from ``choices``)."""
    if pattern == "equal":
        return [[n] * world for _ in range(world)]
    if pattern == "zero":
        return [[0] * world for _ in range(world)]
    q = int(torch.randint(0, world, (1,), generator=g))
    if pattern == "silent":
        return [[0 if s == q else n for _ in range(world)] for s in range(world)]
    if pattern == "hot":
        return [[n if d == q else 0 for d in range(world)] for _ in range(world)]
    return [[choices[int(torch.randint(0, len(choices), (1,), generator=g))] for _ in range(world)] for _ in range(world)]


def _lengths(chunk, es):
    """Per-pair lengths in elements of ``es`` bytes: 0, 1, 15, 16 and 17 bytes (where the element size allows), one chunk
    and its neighbours, and more than three chunks, so both staging halves are reused at least twice."""
    small = [0, 1, 15, 16, 17] if es == 1 else [0, 1, 7, 8, 9]
    c = chunk // es
    return small + [c - 1, c, c + 1, 3 * c + 1]


def _mis(es, k):
    """Offsets past a 16-byte boundary, multiples of the element size: all aligned (k % 3 == 0) or a mix."""
    if k % 3 == 0:
        return [0] * 8
    return [(es * (i + k)) % 16 for i in range(8)]


PATTERNS = ["equal", "zero", "silent", "hot", "random"]
SIZES = [1, 2, 4, 8]


@pytest.mark.parametrize("world", range(1, 9))
def test_alltoallv_matches_the_model_bit_for_bit(C, sms, world):
    W = E.World(world, sms)
    A = A2AV(C, W)
    g = torch.Generator().manual_seed(world)
    k = 0
    for m, mb in enumerate([1, 3, sms // world]):
        for pattern in PATTERNS:
            es = SIZES[(k + m) % 4]
            choices = _lengths(A.chunk, es)
            n = choices[5 + (k % 4)] if pattern != "random" else 0
            lens = _matrix(pattern, world, n, g, choices)
            a2av_call(C, W, A, lens, lens, es, _mis(es, k), _mis(es, k + 1), mb, seed=1000 * world + k)
            k += 1


@pytest.mark.parametrize("es", SIZES)
def test_every_length_at_every_alignment(C, sms, es):
    """World 3, every per-pair length against every mix of aligned and unaligned sources and destinations."""
    world = 3
    W = E.World(world, sms)
    A = A2AV(C, W)
    choices = _lengths(A.chunk, es)
    for k in range(4):
        mis_src = [0] * 8 if k % 2 == 0 else [(es * (i + 1)) % 16 for i in range(8)]
        mis_dst = [0] * 8 if k < 2 else [(es * (3 * i + 1)) % 16 for i in range(8)]
        for j in range(0, len(choices), world * world):
            lens = [[choices[(j + world * s + d + k) % len(choices)] for d in range(world)] for s in range(world)]
            a2av_call(C, W, A, lens, lens, es, mis_src, mis_dst, 3, seed=50 * es + 10 * k + j)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_mismatched_splits_truncate(C, sms, world):
    """Receivers that expect more, fewer, or nothing against what was sent: the model's truncated bytes, nothing outside
    the segments, and the same epochs on every rank (the round count comes from the published lengths alone)."""
    W = E.World(world, sms)
    A = A2AV(C, W)
    g = torch.Generator().manual_seed(77 + world)
    for k in range(4):
        es = SIZES[k]
        choices = _lengths(A.chunk, es)
        lens = _matrix("random", world, 0, g, choices)
        expect = _matrix("random", world, 0, g, choices)             # rank r expects expect[r][p] from p
        a2av_call(C, W, A, lens, expect, es, _mis(es, k + 1), _mis(es, k), [1, 3, sms // world][k % 3], seed=900 + k)
    ep = _epochs(W)
    assert bool((ep == ep[0]).all())


@pytest.mark.parametrize("world", range(1, 9))
def test_alltoallv_shares_pads_and_inboxes_with_every_kind_through_the_epoch_wrap(C, sms, world):
    """One set of pads and inboxes, starting 5 before the uint32 wrap: all-to-allv calls between all-reduces,
    reduce-scatters, equal all-to-alls, broadcasts, scatters, gathers and barriers; every call matches its model and the
    per-block epochs agree on every rank at the end."""
    W = E.World(world, sms, pad_start=E.WRAP)
    A = A2AV(C, W)
    g = torch.Generator().manual_seed(5 * world)
    f32, b16 = torch.float32, torch.bfloat16
    last, mid = world - 1, world // 2
    c = A.chunk
    calls = [("v", "random", 1, 3), ("rs", M.LL, torch.int64, CM.SUM, 1000, 3, "inplace"), ("v", "hot", 4, 1),
             ("ar", M.LL, CM.MAX, 1000, 3, f32, "inplace", -1), ("v", "zero", 2, 3), ("a2a", M.ONESHOT, 2000, 2, "buffer"),
             ("v", "equal", 8, 2), "barrier", ("sc", M.LL, 1000, 3, "inplace", last), ("v", "silent", 1, sms // world),
             ("ga", M.TWOSHOT, 600, 2, "staged", 0), ("v", "random", 2, 1), ("bc", M.LL, 700, 1, "staged", last),
             ("a2a", M.LL, 700, 1, "staged"), ("v", "equal", 1, 3), ("rs", M.ONESHOT, torch.bfloat16, CM.MIN, 5000, 2,
                                                                     "inplace"),
             ("ar", M.TWOSHOT, CM.SUM, world * 900, 3, b16, "staged", mid), ("v", "random", 4, 3)]
    for k, call in enumerate(calls):
        seed = 171 * world + k
        if call == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
        elif call[0] == "v":
            _, pattern, es, mb = call
            choices = _lengths(c, es)
            lens = _matrix(pattern, world, choices[6 + k % 3], g, choices)
            a2av_call(C, W, A, lens, lens, es, _mis(es, k), _mis(es, k + 2), mb, seed)
        elif call[0] == "rs":
            _, variant, dtype, op, seg_vec, mb, mode = call
            E.reduce_scatter_call(C, W, variant, dtype, op, seg_vec, mb, mode, seed)
        elif call[0] == "a2a":
            _, variant, seg_vec, mb, mode = call
            E.alltoall_call(C, W, variant, seg_vec, mb, mode, seed)
        elif call[0] == "ar":
            _, variant, op, n_vec, mb, wire, mode, root = call
            E.reduce_call(C, W, variant, op, n_vec, mb, wire, mode, wire, root, seed)
        elif call[0] == "bc":
            _, variant, n_vec, mb, mode, root = call
            E.broadcast_call(C, W, variant, n_vec, mb, mode, root, seed)
        else:
            kind, variant, seg_vec, mb, mode, root = call
            (E.scatter_call if kind == "sc" else E.gather_call)(C, W, variant, seg_vec, mb, mode, root, seed)
    ep = _epochs(W)
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 1000                                   # block 0 went through the wrap


# ---------------------------------------------------------------------------------------------------------- SymmWorld
DTYPES = AW.DTYPES


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_all_to_all_v_single_and_list_forms(C, sms, world):
    """``all_to_all_v_`` of every dtype class, rows of several elements, skewed and empty splits, in the single-tensor form
    (aligned, unaligned, an output that is the input or overlaps it) and the list form (separate tensors, unaligned); the
    group's global ranks are not 0..W-1.  Every output equals plain slicing bit for bit, and inputs are unchanged."""
    worlds, keep = E.symm_worlds(world, sms, [10 + 3 * r for r in range(world)])
    forms = ["single", "list", "unaligned", "same", "overlap", "list_unaligned"]
    for k in range(2 * len(DTYPES)):
        dtype = DTYPES[k % len(DTYPES)]
        form = forms[k % len(forms)]
        tail = [(), (3,), (4, 2), (1,)][k % 4]
        S = AW.split_matrix(world, 40 * world + k, hot=k % 2 == 0, most=[5, 300, 4000][k % 3])
        if k % 7 == 3:
            S[world - 1] = [0] * world                                  # the last rank sends nothing ...
            for row in S:
                row[world - 1] = 0                                      # ... and receives nothing
        if form in ("same", "overlap"):
            S = [[S[s][d] + S[d][s] for d in range(world)] for s in range(world)]   # symmetric: as many rows out as in
        xs = [AW.rows_of(S, s, dtype, tail, 70 * k) for s in range(world)]
        want = AM.by_slicing(xs, S)
        out_splits = [[S[p][r] for p in range(world)] for r in range(world)]
        ins = [x.cuda() for x in xs]
        if form in ("single", "list"):
            outs = [torch.zeros_like(w_) for w_ in want]
            outs = [o.cuda() for o in outs]
        elif form == "unaligned":
            ins = [_unaligned(x) for x in ins]
            outs = [_unaligned(torch.zeros_like(w_)) for w_ in want]
        elif form == "same":
            outs = ins
        elif form == "overlap":                                         # out starts half way into the input
            bases = []
            for r, x in enumerate(xs):
                rows = x.shape[0]
                b = torch.zeros((rows + rows // 2,) + tail, dtype=dtype, device="cuda")
                b[:rows] = x.cuda()
                bases.append(b)
            ins = [b[:x.shape[0]] for b, x in zip(bases, xs)]
            outs = [b[x.shape[0] // 2:x.shape[0] // 2 + x.shape[0]] for b, x in zip(bases, xs)]
        else:                                                           # list_unaligned
            outs = [torch.zeros_like(w_).cuda() for w_ in want]
        if form.startswith("list"):
            unal = form == "list_unaligned"
            lin = [[(_unaligned(p) if unal else p.clone()) for p in torch.split(x, S[r])] for r, x in enumerate(ins)]
            lout = [[(_unaligned(p) if unal else p.clone()) for p in torch.split(o, out_splits[r])] for r, o in enumerate(outs)]
            E.on_ranks(worlds, lambda r, w: w.all_to_all_v_(lout[r], lin[r]))
            for r in range(world):
                got = torch.cat([_bytes(p) for p in lout[r]]) if lout[r] else torch.zeros(0, dtype=torch.uint8)
                assert torch.equal(got, _bytes(want[r])), ("all_to_all_v_ list", dtype, form, S, r)
                for s, p in enumerate(lin[r]):
                    assert torch.equal(_bytes(p), _bytes(torch.split(xs[r], S[r])[s])), ("input changed", dtype, r, s)
            continue
        E.on_ranks(worlds, lambda r, w: w.all_to_all_v_(outs[r], ins[r], out_splits[r], S[r]))
        for r in range(world):
            assert torch.equal(_bytes(outs[r]), _bytes(want[r])), ("all_to_all_v_", dtype, form, S, r)
            if form in ("single", "unaligned"):
                assert torch.equal(_bytes(ins[r]), _bytes(xs[r])), ("input changed", dtype, form, r)
    w0 = worlds[0]
    t = torch.zeros(2 * world, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match=f"needs {world} entries"):
        w0.all_to_all_v_(t, t.clone(), [2] * (world + 1), None)
    with pytest.raises(ValueError, match="negative"):
        w0.all_to_all_v_(t, t.clone(), None, [-1, 2 * world + 1] + [0] * (world - 2) if world > 1 else [-1])
    with pytest.raises(ValueError, match="sums to"):
        w0.all_to_all_v_(t, t.clone(), [1] * world, None)
    with pytest.raises(ValueError, match=f"needs {world} output tensors"):
        w0.all_to_all_v_([t] * (world + 1), [t] * world)
    with pytest.raises(ValueError, match="one dtype"):
        w0.all_to_all_v_([t] * world, [t.float()] + [t] * (world - 1))
    with pytest.raises(TypeError, match="contiguous CUDA"):
        w0.all_to_all_v_(t, t.cpu(), [2] * world, [2] * world)
    if world > 1:
        with pytest.raises(TypeError, match="contiguous CUDA"):
            w0.all_to_all_v_(t.view(2, world).t(), t.view(world, 2), [2] + [0] * (world - 1), [2] + [0] * (world - 1))
    del keep


@pytest.mark.parametrize("world", [2, 5, 8])
def test_symm_world_all_to_all_v_calls_share_the_staging_buffer(C, sms, world):
    """All-to-allv calls with splits that change from call to call, between equal all-to-alls and reduce-scatters on the
    same staging buffer and pads."""
    worlds, keep = E.symm_worlds(world, sms, list(range(world)))
    for k in range(6):
        S = AW.split_matrix(world, 500 + k, hot=k % 2 == 1, most=[3, 9000, 40000][k % 3])
        xs = [AW.rows_of(S, s, torch.int64, (2,), k) for s in range(world)]
        want = AM.by_slicing(xs, S)
        ins = [x.cuda() for x in xs]
        outs = [torch.zeros_like(w_).cuda() for w_ in want]
        E.on_ranks(worlds, lambda r, w: w.all_to_all_v_(outs[r], ins[r], [S[p][r] for p in range(world)], S[r]))
        for r in range(world):
            assert torch.equal(outs[r].cpu(), want[r]), (k, r)
        ys = [E._raw(torch.uint8, world * 3001, 10 * k + r).cuda() for r in range(world)]
        zs = [torch.zeros_like(y) for y in ys]
        E.on_ranks(worlds, lambda r, w: w.all_to_all_(zs[r], ys[r]))
        for r in range(world):
            assert torch.equal(zs[r].cpu(), torch.cat([y.view(world, -1)[r].cpu() for y in ys])), (k, r)
        us = RS.make_inputs(CM.SUM, torch.int32, world, world * 1000, k)
        vs = [u.cuda() for u in us]
        os_ = [torch.zeros(1000, dtype=torch.int32, device="cuda") for _ in range(world)]
        E.on_ranks(worlds, lambda r, w: w.reduce_scatter_(os_[r], vs[r]))
        for r in range(world):
            assert torch.equal(os_[r].cpu(), RS.reduce_scatter_result(CM.SUM, us, r)), (k, r)
    del keep
