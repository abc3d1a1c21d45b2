"""PRODUCT / MAX / MIN all-reduce, reduce to a root, broadcast and all-gather (csrc/allreduce.cu) on ONE GPU with W emulated
ranks, bit for bit against tests/collectives_model.py.

The harness is tests/test_gpu_comm_emulated.py's: each rank has its own buffers, signal pad, LL inbox and stream, the W
launches go out back to back, and no case runs more CTAs than the GPU has SMs (every CTA spins on its peers).  Outputs,
symmetric buffers and the sentinels behind them are compared whole, so "a non-root leaves its output alone" and "the raw
moves keep every bit" are checked as well.  The last tests drive ``SymmWorld``'s methods for W ranks built over the
emulated buffers, one rank per stream.
"""
import threading

import pytest
import torch

import collectives_model as CM
import comm_model as M
import test_gpu_comm_emulated as E

pytestmark = E.pytestmark

RAW_SENTINEL = 0x5EADBEEF
VARIANTS = [M.ONESHOT, M.TWOSHOT, M.LL]
VARIANT_IDS = ["oneshot", "twoshot", "ll"]
C = E.C
sms = E.sms


def _raw_sentinel(n, dev="cuda"):
    return torch.full((n,), RAW_SENTINEL, dtype=torch.int32, device=dev)


def _inbox(W, variant):
    return (W.inbox_ptrs, M.LL_CAP_VEC) if variant == M.LL else ([], 0)


def _check(what, got, want, epv):
    M.assert_bits_equal(what, [g.cpu() for g in got], want, epv)


# ---------------------------------------------------------------------------------------------------------- reductions
def reduce_call(C, W, variant, op, n_vec, mb, wire, mode, local, root, seed):
    world = W.world
    epv = M.elems_per_vec(wire)
    n = n_vec * epv
    scale = 0.3 if op == CM.SUM else 1.0
    xs = CM.make_reduce_inputs(op, world, n, local, seed)
    bufs = [E._sentinel(n + E.SENT_VECS * epv, wire) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], E._sentinel(E.SENT_VECS * epv, local, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [E._sentinel(n + E.SENT_VECS * epv, local) for _ in range(world)]
        outs = dst
    want = CM.reduce_model(variant, op, xs, wire, scale, mode, root, [o.cpu() for o in outs], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(M.grid_blocks(variant, n_vec, world, mb),
             lambda r: C.allreduce(variant, wire == torch.bfloat16, ptrs, W.sig_ptrs, 0, src[r], dst[r], n_vec, scale, r,
                                   world, mb, inbox, cap, op, root))
    what = (f"{CM.OP_NAMES[op]} root {root} {M.VARIANT_NAMES[variant]} world {world} n_vec {n_vec} max_blocks {mb} "
            f"wire {wire} {mode} {local}")
    _check(what + ": output", outs, want["out"], epv)
    _check(what + ": symmetric buffers", bufs, want["buf"], epv)


# (wire, mode, local): PRODUCT / MAX / MIN take the wire dtype locally; SUM (as a reduce) also fp32 over a bf16 wire
SAME_DTYPE = [c for c in E.COMBOS if c[0] == c[2]]


def reduce_cases(variant, world, sms):
    """(n_vec, max_blocks, op, root, combo) per case over comm_model's sizes: every grid and unroll tail at max_blocks 1, 3
    and SMs // world; ops, roots (all, 0, last, middle) and (wire, mode, local) cycle independently."""
    roots = [-1, 0, world - 1, world // 2]
    ops = [CM.PRODUCT, CM.MAX, CM.MIN, CM.SUM]
    out = []
    for k, (n_vec, mb, _, _) in enumerate(E.allreduce_cases(variant, world, sms)):
        op = ops[k % 4]
        root = roots[(k // 4 + k // 8) % 4]
        if op == CM.SUM and root < 0:
            root = world - 1                      # the SUM all-reduce is test_gpu_comm_emulated.py's
        combos = E.COMBOS if op == CM.SUM else SAME_DTYPE
        out.append((n_vec, mb, op, root, combos[(k // 2) % len(combos)]))
    return out


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_reductions_match_the_model_bit_for_bit(C, sms, world, variant):
    for k, (n_vec, mb, op, root, (wire, mode, local)) in enumerate(reduce_cases(variant, world, sms)):
        reduce_call(C, E.World(world, sms), variant, op, n_vec, mb, wire, mode, local, root,
                    seed=3000 * world + 100 * variant + k)


# ---------------------------------------------------------------------------------------------------------- raw moves
def broadcast_call(C, W, variant, n_vec, mb, mode, root, seed):
    world, n = W.world, n_vec * 4
    xs = CM.make_raw_inputs(world, n, seed)
    bufs = [_raw_sentinel(n + 4 * E.SENT_VECS) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _raw_sentinel(4 * E.SENT_VECS, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [_raw_sentinel(n + 4 * E.SENT_VECS) for _ in range(world)]
        outs = dst
    want = CM.broadcast_model(variant, xs, root, mode, [o.cpu() for o in outs], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(M.grid_blocks(variant, n_vec, world, mb),
             lambda r: C.broadcast(variant, ptrs, W.sig_ptrs, src[r], dst[r], n_vec, root, r, world, mb, inbox, cap))
    what = f"broadcast root {root} {M.VARIANT_NAMES[variant]} world {world} n_vec {n_vec} max_blocks {mb} {mode}"
    _check(what + ": output", outs, want["out"], 4)
    _check(what + ": symmetric buffers", bufs, want["buf"], 4)


def allgather_call(C, W, variant, seg_vec, mb, mode, seed):
    world, seg = W.world, seg_vec * 4
    n_vec = world * seg_vec
    xs = CM.make_raw_inputs(world, seg, seed)
    bufs = [_raw_sentinel(world * seg + 4 * E.SENT_VECS) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][r * seg:(r + 1) * seg].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _raw_sentinel(4 * E.SENT_VECS, "cpu")]).cuda() for r in range(world)]
        dst = [_raw_sentinel(world * seg + 4 * E.SENT_VECS) for _ in range(world)]
        outs = dst
    want = CM.allgather_model(variant, xs, mode, [o.cpu() for o in outs], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    blocks = M.grid_blocks(variant, seg_vec if variant == M.LL else n_vec, world, mb)
    W.launch(blocks, lambda r: C.allgather(variant, ptrs, W.sig_ptrs, src[r], dst[r], n_vec, r, world, mb, inbox, cap))
    what = f"allgather {M.VARIANT_NAMES[variant]} world {world} per-rank vectors {seg_vec} max_blocks {mb} {mode}"
    _check(what + ": output", outs, want["out"], 4)
    _check(what + ": symmetric buffers", bufs, want["buf"], 4)
    if src[0] is not None:
        for r in range(world):
            assert bool((src[r][seg:] == RAW_SENTINEL).all()), f"{what}: rank {r} wrote into src"


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_broadcast_matches_the_model_bit_for_bit(C, sms, world, variant):
    roots = [0, world - 1, world // 2]
    modes = ["inplace", "staged", "alias"]
    for k, (n_vec, mb, _, _) in enumerate(E.allreduce_cases(variant, world, sms)):
        broadcast_call(C, E.World(world, sms), variant, n_vec, mb, modes[k % 3], roots[(k // 3) % 3],
                       seed=5000 * world + 100 * variant + k)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_allgather_matches_the_model_bit_for_bit(C, sms, world, variant):
    """Per-rank sizes across the LL inbox's block boundaries, and (one-shot, two-shot) across every grid and unroll tail
    of the world x larger output."""
    k = 0
    for m, mb in enumerate([1, 3, sms // world]):
        tail = 2 * M.THREADS * mb
        if variant == M.LL:
            segs = [1, 511, 512, 513, 1025, 4095, M.LL_CAP_VEC]
        elif variant == M.ONESHOT:
            segs = [1, 511, 513, tail // world + 1, tail // world - 1, 700, (3 * tail + 700) // world]
        else:
            segs = [1, 511, 512, 513, tail - 1, tail + 1, 700, 3 * tail + 300]
        for seg_vec in segs:
            allgather_call(C, E.World(world, sms), variant, max(seg_vec, 1), mb, ["inplace", "staged"][(k + m) % 2],
                           seed=7000 * world + 100 * variant + k)
            k += 1


# ---------------------------------------------------------------------------------------------------------- sequences
@pytest.mark.parametrize("world", range(1, 9))
def test_every_kind_of_call_shares_pads_and_inboxes_through_the_epoch_wrap(C, sms, world):
    """One set of pads and inboxes, starting 5 before the uint32 wrap, runs SUM, the new ops, reduces, broadcasts,
    all-gathers and barriers in every variant; every call matches the model and the per-block epochs agree at the end."""
    W = E.World(world, sms, pad_start=E.WRAP)
    f32, b16 = torch.float32, torch.bfloat16
    last, mid = world - 1, world // 2
    calls = [("ar", M.LL, CM.MAX, 1000, 3, f32, "inplace", -1), ("bc", M.LL, 700, 1, "staged", last),
             ("ag", M.TWOSHOT, 300, 2, "inplace"), "barrier", ("ar", M.ONESHOT, CM.PRODUCT, 3000, 3, b16, "staged", mid),
             ("ag", M.LL, 4096, 1, "staged"), ("ar", M.LL, CM.SUM, 4096, 3, f32, "alias", -1),
             ("bc", M.ONESHOT, 5000, 2, "inplace", 0), ("ar", M.TWOSHOT, CM.MIN, world * 700, 2, b16, "inplace", 0),
             ("ag", M.ONESHOT, 600, 3, "staged"), ("ar", M.LL, CM.PRODUCT, 513, 3, f32, "inplace", last), "barrier",
             ("bc", M.TWOSHOT, world * 1500, 3, "alias", mid), ("ag", M.LL, 2000, 3, "inplace"),
             ("ar", M.TWOSHOT, CM.SUM, world * 900, 3, f32, "staged", mid), ("bc", M.LL, 4096, 3, "inplace", 0)]
    for k, c in enumerate(calls):
        seed = 91 * world + k
        if c == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
        elif c[0] == "ar":
            _, variant, op, n_vec, mb, wire, mode, root = c
            reduce_call(C, W, variant, op, n_vec, mb, wire, mode, wire, root, seed)
        elif c[0] == "bc":
            _, variant, n_vec, mb, mode, root = c
            broadcast_call(C, W, variant, n_vec, mb, mode, root, seed)
        else:
            _, variant, seg_vec, mb, mode = c
            allgather_call(C, W, variant, seg_vec, mb, mode, seed)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 100


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def symm_worlds(world, sms, global_ranks):
    """W SymmWorld objects over emulated buffers (no process group): world r has rank r, global rank global_ranks[r], and
    handles whose per-rank pointers are the W emulated allocations, [signal pad | data] as alloc_bytes lays them out."""
    from dist_tuto.pth_b200.ops import _ext
    from dist_tuto.pth_b200.parallel import symm

    keep = []

    def alloc(nbytes):
        ts = [torch.zeros((symm.PAD_BYTES + nbytes) // 4, dtype=torch.int32, device="cuda") for _ in range(world)]
        keep.extend(ts)
        return [t.data_ptr() for t in ts]

    staging_bytes = 4 << 20
    st_ptrs = {dt: alloc(staging_bytes) for dt in (torch.float32, torch.bfloat16)}
    ll_ptrs = {dt: alloc(2 * world * symm.LL_CAP_VEC * 32) for dt in st_ptrs}
    worlds = []
    for r in range(world):
        w = object.__new__(symm.SymmWorld)
        w.C, w.group, w.ranks, w.world = _ext.C(), None, list(global_ranks), world
        w.global_rank, w.rank = global_ranks[r], r
        w.device = torch.device("cuda", 0)
        w.multicast, w.mode, w.nvls_error, w.table_world = False, "emulated", None, None
        w._handles, w._lock, w._staging = [], threading.Lock(), {}
        w.max_blocks = sms // world
        w.ll_max, w.oneshot_max, w.nvls_min = 32 << 10, 256 << 10, 1 << 62
        for dt, ptrs in st_ptrs.items():
            hd = symm.SymmHandle(w, staging_bytes, staging_bytes, ptrs, 0, [], 0, "emulated")
            hd.ll = symm.SymmHandle(w, 0, 0, ll_ptrs[dt], 0, [], 0, "emulated")
            w._staging[dt] = hd
        worlds.append(w)
    return worlds, keep


def on_ranks(worlds, fn):
    """fn(r, world_r) for every rank, each on its own stream, issued back to back."""
    streams = [torch.cuda.Stream() for _ in worlds]
    torch.cuda.synchronize()
    for r, w in enumerate(worlds):
        with torch.cuda.stream(streams[r]):
            fn(r, w)
    torch.cuda.synchronize()


def _bits_equal(a, b):
    return torch.equal(a.cpu().view(-1).view(torch.uint8), b.cpu().view(-1).view(torch.uint8))


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_methods_route_stage_and_copy_out(C, sms, world):
    """Message sizes on both sides of every threshold (LL, one-shot, two-shot) and ragged ones; fp32 and bf16 reductions,
    int64 / bf16 / uint8 raw moves; roots given as global ranks of a group whose ranks are not 0..W-1."""
    globals_ = [10 + 3 * r for r in range(world)]
    worlds, keep = symm_worlds(world, sms, globals_)
    g = torch.Generator().manual_seed(world)
    ops = [CM.MAX, CM.MIN, CM.PRODUCT, CM.SUM]
    for k, numel in enumerate([5, 1024, 3001, 12288, 40000, 200003]):
        dtype = torch.float32 if k % 2 == 0 else torch.bfloat16
        op = ops[k % 4]
        xs = [x.to(dtype) for x in CM.make_reduce_inputs(op, world, numel, torch.float32, 100 * world + k)]
        want = CM.fold(op, [x.float() for x in xs]).to(dtype)
        ts = [x.cuda() for x in xs]
        on_ranks(worlds, lambda r, w: w.all_reduce_(ts[r], op=op))
        for r in range(world):
            assert _bits_equal(ts[r], want) or bool(((ts[r].cpu() == want) | (ts[r].cpu().isnan() & want.isnan())).all()), \
                (CM.OP_NAMES[op], numel, r)
        root_local = [0, world - 1, world // 2][k % 3]
        ts = [x.cuda() for x in xs]
        on_ranks(worlds, lambda r, w: w.reduce_(ts[r], globals_[root_local], op))
        for r in range(world):
            got = ts[r].cpu()
            if r == root_local:
                assert bool(((got == want) | (got.isnan() & want.isnan())).all()), ("reduce", numel, r)
            else:
                assert _bits_equal(got, xs[r]), ("reduce: a non-root changed its tensor", numel, r)
        raw_dtype = [torch.int64, torch.bfloat16, torch.uint8][k % 3]
        raw = [torch.randint(-2 ** 62, 2 ** 62, (numel,), generator=g, dtype=torch.int64).to(raw_dtype)
               if raw_dtype != torch.bfloat16 else CM.make_raw_inputs(1, numel, 100 * k + s)[0].view(torch.bfloat16)[:numel].clone()
               for s in range(world)]
        ts = [x.cuda() for x in raw]
        on_ranks(worlds, lambda r, w: w.broadcast_(ts[r], globals_[root_local]))
        for r in range(world):
            assert _bits_equal(ts[r], raw[root_local]), ("broadcast", raw_dtype, numel, r)
        ins = [x.cuda() for x in raw]
        contiguous = k % 2 == 0
        if contiguous:
            blocks = [torch.zeros(world * numel, dtype=raw_dtype, device="cuda") for _ in range(world)]
            outs = [list(b.view(world, numel).unbind(0)) for b in blocks]
        else:
            outs = [[torch.zeros(numel, dtype=raw_dtype, device="cuda") for _ in range(world)] for _ in range(world)]
        on_ranks(worlds, lambda r, w: w.all_gather_(outs[r], ins[r]))
        for r in range(world):
            for s in range(world):
                assert _bits_equal(outs[r][s], raw[s]), ("all_gather", raw_dtype, numel, r, s)
    with pytest.raises(ValueError, match="not in this world"):
        worlds[0].reduce_(torch.zeros(4, device="cuda"), 0, CM.MAX)
    with pytest.raises(ValueError, match="scale applies to SUM only"):
        worlds[0].all_reduce_(torch.zeros(4, device="cuda"), scale=0.5, op=CM.MAX)
    del keep
