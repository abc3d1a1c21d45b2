"""The emulated-rank harness: W "ranks" on ONE GPU, shared by every test of the peer-memory kernels that runs on one device.

The kernels take raw per-rank pointers, so W ranks can be W sets of buffers on one device: each rank gets its own data,
signal pad, LL inbox and stream, and its own launch.  What this cannot cover (the memory model across NVLink, NVLS and the
IPC / VMM mappings) stays in the ``_multi`` tests.

Every CTA of these kernels spins on its peers, so the W grids of one call must all be resident at once:

* the W launches are issued back to back on W streams between two device synchronisations, never one after another with a
  wait in between.  With serialized launches (CUDA_LAUNCH_BLOCKING=1, or a tool that serializes kernels) the first rank's
  grid spins alone until B2_SPIN_LIMIT and traps, so these tests are skipped under CUDA_LAUNCH_BLOCKING=1 and are not part
  of tools/sanitize.sh;
* the budget is one CTA per SM for all ranks together (``allreduce_oneshot_kernel<false>`` uses 128 registers x 512
  threads, the whole register file of an SM): the harness computes each launch's grid as the launcher does and refuses
  any case with ``world x blocks > SM count``.

A test module takes the fixtures by importing them (``from emulated_ranks import C, sms``) and the marks through
``pytestmark``.  Besides ``World`` this holds the call drivers of the collectives that several modules run on one set of pads
and inboxes, W ``SymmWorld`` objects over emulated allocations, and the point-to-point mailboxes.
"""
import os
import threading

import pytest
import torch

import collectives_model as CM
import comm_model as M
import reduce_dtypes_model as RM
import reduce_scatter_alltoall_model as RS
import scatter_gather_model as SG

SERIALIZED = os.environ.get("CUDA_LAUNCH_BLOCKING") == "1"
SERIAL_SKIP = pytest.mark.skipif(SERIALIZED, reason="serialized launches: every rank's grid would spin alone until it traps")
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900), SERIAL_SKIP]
# for the emulated-rank tests of a module whose other tests launch one kernel at a time
CO_RESIDENT = pytest.mark.skipif(SERIALIZED, reason="serialized launches: the ranks' grids must be co-resident")

SENT_VECS = 3                                   # sentinel vectors behind every buffer
SENTINEL = {torch.float32: 0x5EADBEEF, torch.bfloat16: 0x5EAD}     # finite bit patterns no kernel result can produce here
RAW_SENTINEL = 0x5EADBEEF                       # the word behind every buffer of a raw move
RAW_SENT = 4 * SENT_VECS                        # sentinel words behind every buffer of a raw move
SENTINEL_BYTE = 0x5E                            # 0x5E5E... is finite in fp16 and fp64, and no result here is all 0x5E bytes
WRAP = 2 ** 32 - 5                              # wrap tests: every pad's epoch and flag words (or p2p counters) start here
VARIANTS = [M.ONESHOT, M.TWOSHOT, M.LL]
VARIANT_IDS = ["oneshot", "twoshot", "ll"]


@pytest.fixture(scope="module")
def C():
    from dist_tuto.pth_b200.ops import _ext
    return _ext.C()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------- sentinels
def _typed_sentinel(n, dtype, dev="cuda"):
    """n fp32 / bf16 elements holding SENTINEL[dtype]."""
    bits = torch.full((n,), SENTINEL[dtype], dtype=torch.int32 if dtype == torch.float32 else torch.int16, device=dev)
    return bits.view(dtype)


def _raw_sentinel(n, dev="cuda"):
    """n 32-bit words holding RAW_SENTINEL."""
    return torch.full((n,), RAW_SENTINEL, dtype=torch.int32, device=dev)


def _byte_sentinel(n, dtype, dev="cuda"):
    """n elements of any dtype whose every byte is SENTINEL_BYTE."""
    es = torch.empty((), dtype=dtype).element_size()
    return torch.full((n * es,), SENTINEL_BYTE, dtype=torch.uint8, device=dev).view(dtype)


def _with_sentinel(x, dtype=None):
    """``x`` on the GPU followed by SENT_VECS sentinel vectors."""
    dtype = dtype or x.dtype
    epv = M.elems_per_vec(dtype)
    bits = torch.full((SENT_VECS * epv,), SENTINEL[dtype], dtype=torch.int32 if dtype == torch.float32 else torch.int16)
    return torch.cat([x.to(dtype), bits.view(dtype)]).cuda()


def _untouched(t):
    """Every fp32 / bf16 element of t still holds SENTINEL[t.dtype]."""
    ib = torch.int32 if t.dtype == torch.float32 else torch.int16
    return bool((t.view(ib) == SENTINEL[t.dtype]).all())


# ---------------------------------------------------------------------------------------------------------- the world
class World:
    """W emulated ranks on cuda:0: a zeroed signal pad (uint32 [B2_SIGNAL_WORDS]), an LL inbox
    ([2 parities][W sources][LL_CAP_VEC][2 lines of 16 B]) and a stream per rank."""

    def __init__(self, world, sms, pad_start=0):
        self.world, self.sms = world, sms
        self.pads = [torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda") for _ in range(world)]
        if pad_start:
            for p in self.pads:                   # per-block epoch words and every flag word
                p[:M.EPOCH_WORD0 + M.MAX_BLOCKS] = pad_start - 2 ** 32 if pad_start >= 2 ** 31 else pad_start
        self.inbox = [torch.zeros(2 * world * M.LL_CAP_VEC * 8, dtype=torch.int32, device="cuda") for _ in range(world)]
        self.streams = [torch.cuda.Stream() for _ in range(world)]
        self.sig_ptrs = [p.data_ptr() for p in self.pads]
        self.inbox_ptrs = [b.data_ptr() for b in self.inbox]

    def launch(self, blocks, fn):
        """fn(r) issues rank r's kernel.  All W launches go out back to back, each on its own stream."""
        assert self.world * blocks <= self.sms, (
            f"{self.world} ranks x {blocks} CTAs would not be co-resident on {self.sms} SMs; not launched")
        torch.cuda.synchronize()
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                fn(r)
        torch.cuda.synchronize()


def _inbox(W, variant):
    return (W.inbox_ptrs, M.LL_CAP_VEC) if variant == M.LL else ([], 0)


def _check(what, got, want, epv):
    M.assert_bits_equal(what, [g.cpu() for g in got], want, epv)


# ---------------------------------------------------------------------------------------------------------- reductions
# (wire dtype, mode, local dtype): in place on the symmetric buffers; src / dst; src aliasing dst (parallel/symm.py's
# staged path)
COMBOS = [(torch.float32, "inplace", torch.float32), (torch.float32, "staged", torch.float32),
          (torch.float32, "alias", torch.float32), (torch.bfloat16, "inplace", torch.bfloat16),
          (torch.bfloat16, "staged", torch.bfloat16), (torch.bfloat16, "staged", torch.float32),
          (torch.bfloat16, "alias", torch.float32), (torch.bfloat16, "alias", torch.bfloat16)]


def allreduce_cases(variant, world, sms):
    """(n_vec, max_blocks, combo, scale) per case: every size at max_blocks 1, 3 and SMs // world; every (wire, mode, local)
    combination once per max_blocks and so with every scale."""
    scales = [1.0, 1.0 / world, 0.3]
    out = []
    for m, mb in enumerate([1, 3, sms // world]):
        tail = 2 * M.THREADS * mb                 # one full pass of the unrolled peer-load loop at mb CTAs
        if variant == M.LL:
            sizes = [1, 511, 512, 513, 1023, 1025, 4095, M.LL_CAP_VEC]
        elif variant == M.ONESHOT:
            sizes = [1, 511, 512, 513, tail - 1, tail + 1, M.LL_CAP_VEC, 3 * tail + 700]
        else:                                     # two-shot: slices, several of them not multiples of 512
            sizes = [world * s for s in (1, 511, 512, 513, tail - 1, tail + 1, 700, 3 * tail + 300)]
        for i, n_vec in enumerate(sizes):
            out.append((n_vec, mb, COMBOS[(i + m) % len(COMBOS)], scales[m]))
    return out


def reduce_call(C, W, variant, op, n_vec, mb, wire, mode, local, root, seed):
    """One fp32 / bf16 all-reduce (root -1) or reduce of ``op`` over W with fresh inputs; checks every rank's output and
    symmetric buffer, sentinels included, against tests/collectives_model.py."""
    world = W.world
    epv = M.elems_per_vec(wire)
    n = n_vec * epv
    scale = 0.3 if op == CM.SUM else 1.0
    xs = CM.make_reduce_inputs(op, world, n, local, seed)
    bufs = [_typed_sentinel(n + SENT_VECS * epv, wire) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _typed_sentinel(SENT_VECS * epv, local, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [_typed_sentinel(n + SENT_VECS * epv, local) for _ in range(world)]
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


# ---------------------------------------------------------------------------------------------------------- raw moves
def broadcast_call(C, W, variant, n_vec, mb, mode, root, seed):
    world, n = W.world, n_vec * 4
    xs = CM.make_raw_inputs(world, n, seed)
    bufs = [_raw_sentinel(n + RAW_SENT) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _raw_sentinel(RAW_SENT, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [_raw_sentinel(n + RAW_SENT) for _ in range(world)]
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
    bufs = [_raw_sentinel(world * seg + RAW_SENT) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][r * seg:(r + 1) * seg].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _raw_sentinel(RAW_SENT, "cpu")]).cuda() for r in range(world)]
        dst = [_raw_sentinel(world * seg + RAW_SENT) for _ in range(world)]
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


def _launch_blocks(kind, variant, seg_vec, world, mb):
    """The scatter / gather launcher's grid: LL and the one-shot scatter by one segment, the rest like an all-gather of
    world segments."""
    by_seg = variant == M.LL or (kind == "scatter" and variant == M.ONESHOT)
    return M.grid_blocks(variant, seg_vec if by_seg else world * seg_vec, world, mb)


def gather_call(C, W, variant, seg_vec, mb, mode, root, seed):
    world, seg = W.world, seg_vec * 4
    n_vec = world * seg_vec
    xs = CM.make_raw_inputs(world, seg, seed)
    bufs = [_raw_sentinel(world * seg + RAW_SENT) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][r * seg:(r + 1) * seg].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([xs[r], _raw_sentinel(RAW_SENT, "cpu")]).cuda() for r in range(world)]
        dst = [_raw_sentinel(world * seg + RAW_SENT) for _ in range(world)]
        outs = dst
    src_before = [s.cpu() if s is not None else None for s in src]
    want = SG.gather_model(variant, xs, root, mode, [o.cpu() for o in outs], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(_launch_blocks("gather", variant, seg_vec, world, mb),
             lambda r: C.gather(variant, ptrs, W.sig_ptrs, src[r], dst[r], n_vec, root, r, world, mb, inbox, cap))
    what = f"gather root {root} {M.VARIANT_NAMES[variant]} world {world} per-rank vectors {seg_vec} max_blocks {mb} {mode}"
    _check(what + ": output", outs, want["out"], 4)
    _check(what + ": symmetric buffers", bufs, want["buf"], 4)
    if mode != "inplace":
        _check(what + ": src", src, src_before, 4)


def scatter_call(C, W, variant, seg_vec, mb, mode, root, seed):
    """The root's src holds the world segments; every other rank passes a src of the same size holding other words, which
    must neither be read (the outputs would show it) nor written."""
    world, seg = W.world, seg_vec * 4
    n_vec = world * seg_vec
    xs = CM.make_raw_inputs(world, seg, seed)
    decoy = CM.make_raw_inputs(world, seg, seed + 1)
    bufs = [_raw_sentinel(world * seg + RAW_SENT) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        bufs[root][:world * seg].copy_(torch.cat(xs))
        outs = bufs
    else:
        src = [torch.cat(xs + [_raw_sentinel(RAW_SENT, "cpu")]).cuda() if r == root else
               torch.cat(decoy + [_raw_sentinel(RAW_SENT, "cpu")]).cuda() for r in range(world)]
        dst = [_raw_sentinel(seg + RAW_SENT) for _ in range(world)]
        outs = dst
    src_before = [s.cpu() if s is not None else None for s in src]
    want = SG.scatter_model(variant, xs, root, mode, [o.cpu() for o in outs], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(_launch_blocks("scatter", variant, seg_vec, world, mb),
             lambda r: C.scatter(variant, ptrs, W.sig_ptrs, src[r], dst[r], n_vec, root, r, world, mb, inbox, cap))
    what = f"scatter root {root} {M.VARIANT_NAMES[variant]} world {world} per-rank vectors {seg_vec} max_blocks {mb} {mode}"
    _check(what + ": output", outs, want["out"], 4)
    _check(what + ": symmetric buffers", bufs, want["buf"], 4)
    if mode != "inplace":
        _check(what + ": src", src, src_before, 4)


# ---------------------------------------------------------------------------------------------------------- segments
def _grid(variant, seg_vec, mb):
    """The reduce-scatter / all-to-all launchers' grid: one thread per vector of a segment; LL never capped by max_blocks."""
    return M.grid_blocks(M.LL, seg_vec, 1, 0) if variant == M.LL else M.grid_blocks(M.ONESHOT, seg_vec, 1, mb)


def _any_nan(op, dtype):
    return dtype in (torch.float32, torch.bfloat16) or RM.nan_any(op, dtype)


def _bytes_cpu(ts):
    return [RM.as_bytes(t).cpu() for t in ts]


def reduce_scatter_call(C, W, variant, dtype, op, seg_vec, mb, mode, seed):
    world = W.world
    epv = RS.elems_per_vec(dtype)
    seg = seg_vec * epv
    n = world * seg
    xs = RS.make_inputs(op, dtype, world, n, seed)
    tail = SENT_VECS * epv
    bufs = [_byte_sentinel(n + tail, dtype) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            RM.as_bytes(bufs[r])[:n].copy_(RM.as_bytes(xs[r]))
        outs = bufs
    else:
        src = [torch.cat([RM.as_bytes(xs[r]), RM.as_bytes(_byte_sentinel(tail, dtype, "cpu"))]).cuda().view(dtype)
               for r in range(world)]
        dst = [_byte_sentinel(seg + tail, dtype) for _ in range(world)]
        outs = dst
    src_before = [RM.as_bytes(s).cpu() if s is not None else None for s in src]
    want = RS.reduce_scatter_model(variant, op, xs, mode, _bytes_cpu(outs), _bytes_cpu(bufs))
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(_grid(variant, seg_vec, mb),
             lambda r: C.reduce_scatter(variant, ptrs, W.sig_ptrs, src[r], dst[r], world * seg_vec, r, world, mb, inbox, cap,
                                        RM.kernel_op(op, dtype), RM.CODES[dtype]))
    what = (f"reduce-scatter {RS.NAMES[dtype]} {CM.OP_NAMES[op]} {M.VARIANT_NAMES[variant]} world {world} seg_vec {seg_vec} "
            f"max_blocks {mb} {mode}")
    any_nan = _any_nan(op, dtype)
    RM.assert_bits_equal(what + ": output", _bytes_cpu(outs), want["out"], any_nan)
    RM.assert_bits_equal(what + ": symmetric buffers", _bytes_cpu(bufs), want["buf"], any_nan)
    if mode != "inplace":
        RM.assert_bits_equal(what + ": src", _bytes_cpu(src), src_before)


def alltoall_call(C, W, variant, seg_vec, mb, mode, seed):
    world, seg = W.world, seg_vec * 4
    n = world * seg
    xs = CM.make_raw_inputs(world, n, seed)
    bufs = [_raw_sentinel(n + RAW_SENT) for _ in range(world)]
    src = [None] * world
    if mode == "buffer":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
    else:
        src = [torch.cat([xs[r], _raw_sentinel(RAW_SENT, "cpu")]).cuda() for r in range(world)]
    dst = [_raw_sentinel(n + RAW_SENT) for _ in range(world)]
    src_before = [s.cpu() if s is not None else None for s in src]
    want = RS.alltoall_model(variant, xs, mode, [d.cpu() for d in dst], [b.cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = _inbox(W, variant)
    W.launch(_grid(variant, seg_vec, mb),
             lambda r: C.alltoall(variant, ptrs, W.sig_ptrs, src[r], dst[r], n // 4, r, world, mb, inbox, cap))
    what = f"all-to-all {M.VARIANT_NAMES[variant]} world {world} seg_vec {seg_vec} max_blocks {mb} {mode}"
    _check(what + ": output", dst, want["out"], 4)
    _check(what + ": symmetric buffers", bufs, want["buf"], 4)
    if mode != "buffer":
        _check(what + ": src", src, src_before, 4)


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def symm_worlds(world, sms, global_ranks):
    """W SymmWorld objects over emulated buffers (no process group): world r has rank r, global rank global_ranks[r], and
    handles whose per-rank pointers are the W emulated allocations, [signal pad | data] as alloc_bytes lays them out.

    ``SymmWorld.__init__`` needs a process group, so this sets its attributes by hand and must follow it: ``C``, ``group``,
    ``ranks``, ``world``, ``global_rank``, ``rank``, ``device``, ``multicast``, ``mode``, ``nvls_error``, ``table_world``,
    ``_handles``, ``_lock``, ``_staging`` (an fp32 and a bf16 staging handle, each with its LL handle), ``max_blocks``,
    ``ll_max``, ``oneshot_max``, ``nvls_min``, ``p2p`` (the point-to-point mailbox, None at world 1) and ``_p2p_streams``."""
    from dist_tuto.pth_b200.ops import _ext
    from dist_tuto.pth_b200.parallel import symm

    C = _ext.C()
    keep = []

    def alloc(nbytes):
        ts = [torch.zeros((symm.PAD_BYTES + nbytes) // 4, dtype=torch.int32, device="cuda") for _ in range(world)]
        keep.extend(ts)
        return [t.data_ptr() for t in ts]

    staging_bytes = 4 << 20
    st_ptrs = {dt: alloc(staging_bytes) for dt in (torch.float32, torch.bfloat16)}
    ll_ptrs = {dt: alloc(2 * world * symm.LL_CAP_VEC * 32) for dt in st_ptrs}
    ctas, slots, chunk, _ = C.p2p_config()
    p2p_bytes = (world - 1) * ctas * slots * chunk
    p2p_ptrs = alloc(p2p_bytes) if world > 1 else None
    worlds = []
    for r in range(world):
        w = object.__new__(symm.SymmWorld)
        w.C, w.group, w.ranks, w.world = C, None, list(global_ranks), world
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
        w.p2p = symm.SymmHandle(w, p2p_bytes, p2p_bytes, p2p_ptrs, 0, [], 0, "emulated") if world > 1 else None
        w._p2p_streams = {}
        worlds.append(w)
    return worlds, keep


def on_ranks(worlds, fn, streams=None):
    """fn(r, world_r) for every rank, each on its own current stream, issued back to back.  Without ``streams`` it makes
    one stream per rank and synchronises the device before and after; with them it only issues the calls."""
    if streams is not None:
        for r, w in enumerate(worlds):
            with torch.cuda.stream(streams[r]):
                fn(r, w)
        return
    streams = [torch.cuda.Stream() for _ in worlds]
    torch.cuda.synchronize()
    on_ranks(worlds, fn, streams)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- point to point
P2P_SENT = 48                                   # sentinel bytes behind every point-to-point destination
P2P_SENT_BYTE = 0xA5


@pytest.fixture(scope="module")
def geo(C):
    """(CTAs per transfer, slots per CTA, bytes per slot, signal-pad words)."""
    return C.p2p_config()


def _stream(C):
    return torch.cuda.ExternalStream(C.stream_create(0), device=torch.device("cuda", 0))


class Mailboxes:
    """W emulated ranks' mailboxes on cuda:0 (data [W - 1 sources][G x S slots][CHUNK] after an 8 KB signal pad, as
    ``SymmWorld`` allocates them) and a stream per (rank, peer, direction).

    A rank runs a send and a receive at once, and each waits for its peer, so every (rank, peer, direction) gets a CUDA
    stream of its own (``stream_create``, never a pooled torch stream that could alias another)."""

    def __init__(self, C, world, sms, start=0):
        from dist_tuto.pth_b200.parallel import symm
        self.C, self.world, self.sms = C, world, sms
        self.G, self.S, self.CHUNK, self.pad_words = C.p2p_config()
        data = max(world - 1, 1) * self.G * self.S * self.CHUNK
        self.mem = [torch.zeros((symm.PAD_BYTES + data) // 4, dtype=torch.int32, device="cuda") for _ in range(world)]
        if start:
            for m in self.mem:
                m[:self.pad_words] = start - 2 ** 32 if start >= 2 ** 31 else start
        self.sig_ptrs = [m.data_ptr() for m in self.mem]
        self.box_ptrs = [p + symm.PAD_BYTES for p in self.sig_ptrs]
        self.streams = {}

    def stream(self, r, peer, send):
        if (r, peer, send) not in self.streams:
            self.streams[(r, peer, send)] = _stream(self.C)
        return self.streams[(r, peer, send)]

    def grid(self, nbytes):
        return min(self.G, (nbytes + self.CHUNK - 1) // self.CHUNK)

    def run(self, transfers):
        """transfers: [(src rank, dst rank, src tensor, dst tensor)], submitted in this order, each as the send on the
        sender's stream, then the receive on the receiver's."""
        busy = {}
        for a, b, x, y in transfers:
            g = self.grid(x.numel() * x.element_size())
            for key in ((a, b, True), (b, a, False)):
                busy[key] = max(busy.get(key, 0), g)
        assert sum(busy.values()) <= self.sms, f"{sum(busy.values())} CTAs would not be co-resident on {self.sms} SMs"
        torch.cuda.synchronize()
        for a, b, x, y in transfers:
            with torch.cuda.stream(self.stream(a, b, True)):
                self.C.p2p_send(self.box_ptrs, self.sig_ptrs, x, b, a, self.world)
            with torch.cuda.stream(self.stream(b, a, False)):
                self.C.p2p_recv(self.box_ptrs, self.sig_ptrs, y, a, b, self.world)
        torch.cuda.synchronize()

    def counters(self, r):
        """Rank r's signal-pad counters as uint32: {name: [peer][slot]}."""
        words = self.mem[r][:self.pad_words].cpu().to(torch.int64) % 2 ** 32
        per = self.G * self.S
        return {name: words[k * 8 * per:(k + 1) * 8 * per].view(8, per) for k, name in
                enumerate(("flag", "ack", "fills", "consumed"))}

    def close(self):
        torch.cuda.synchronize()
        for s in self.streams.values():
            self.C.stream_destroy(s.cuda_stream)
        self.streams.clear()


@pytest.fixture
def boxes(C, sms):
    made = []

    def make(world, start=0):
        made.append(Mailboxes(C, world, sms, start))
        return made[-1]
    yield make
    for m in made:
        m.close()


@pytest.fixture
def worlds(C, sms):
    """make(world, global_ranks) -> (symm_worlds' W worlds, one ``stream_create`` stream per rank); every stream they made
    is destroyed afterwards."""
    made = []

    def make(world, global_ranks):
        ws, keep = symm_worlds(world, sms, global_ranks)
        streams = [_stream(C) for _ in range(world)]
        made.append((ws, keep, streams))
        return ws, streams
    yield make
    torch.cuda.synchronize()
    for ws, keep, streams in made:
        for w in ws:
            for s in w._p2p_streams.values():
                C.stream_destroy(s.cuda_stream)
        for s in streams:
            C.stream_destroy(s.cuda_stream)


def _message(nbytes, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()


def _dest(nbytes):
    return torch.full((nbytes + P2P_SENT,), P2P_SENT_BYTE, dtype=torch.uint8, device="cuda")


def _check_message(what, x, x_before, y):
    n = x.numel()
    assert torch.equal(y[:n].cpu(), x_before), f"{what}: received bytes differ"
    assert bool((y[n:] == P2P_SENT_BYTE).all()), f"{what}: bytes written behind the destination"
    assert torch.equal(x.cpu(), x_before), f"{what}: the source changed"


def _agree(boxes, pairs):
    """After every message between a and b was received: fills (a) == ack (a) == flag (b) == consumed (b), slot by slot."""
    for a, b in pairs:
        ca, cb = boxes.counters(a), boxes.counters(b)
        for name, v in (("ack", ca["ack"][b]), ("flag", cb["flag"][a]), ("consumed", cb["consumed"][a])):
            assert torch.equal(v, ca["fills"][b]), (a, b, name, v, ca["fills"][b])


# ---------------------------------------------------------------------------------------------------------- raw data and bits
def _raw(dtype, numel, seed):
    """numel random elements of dtype: int64 draws cast to dtype, or random raw words seen as bf16."""
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.bfloat16:
        return CM.make_raw_inputs(1, (numel + 1) // 2, seed)[0].view(torch.bfloat16)[:numel].clone()
    return torch.randint(-2 ** 62, 2 ** 62, (numel,), generator=g, dtype=torch.int64).to(dtype)


def _values(dtype, numel, seed):
    """numel elements of dtype made of random bytes (bool: random 0 / 1)."""
    g = torch.Generator().manual_seed(seed)
    raw = torch.randint(0, 256, (numel * torch.empty((), dtype=dtype).element_size(),), generator=g, dtype=torch.uint8)
    return (raw % 2).to(torch.bool) if dtype == torch.bool else raw.view(dtype)


def _unaligned(x):
    """``x`` on the GPU as a view one element into its storage (a data pointer that is not 16-byte aligned for any dtype
    here)."""
    base = torch.zeros(x.numel() + 1, dtype=x.dtype, device="cuda")
    v = base[1:].view(x.shape)
    v.copy_(x)
    return v


def _bytes(t):
    """t's elements as bytes on the CPU, in order."""
    return t.detach().reshape(-1).view(torch.uint8).cpu()


def _bits_equal(a, b):
    """Two contiguous tensors hold the same bytes."""
    return torch.equal(a.cpu().view(-1).view(torch.uint8), b.cpu().view(-1).view(torch.uint8))


def _bits(a, b):
    """Two fp32 tensors of one shape (views may be strided) are equal bit for bit."""
    return torch.equal(a.cpu().view(torch.int32), b.cpu().view(torch.int32))
