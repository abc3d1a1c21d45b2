"""Point-to-point send / recv (csrc/p2p.cu) on ONE GPU with W emulated ranks, bit for bit.

The harness is tests/emulated_ranks.py's: each rank has its own mailbox (data and signal pad), and the kernels of
one batch go out back to back between two device synchronisations.  Unlike a collective, a rank runs a send and a receive at
once, and each waits for its peer, so every (rank, peer, direction) gets a CUDA stream of its own (``stream_create``, never a
pooled torch stream that could alias another).  Kernels that wait for each other are submitted so that whatever a kernel
waits for was submitted before it, or runs in a batch where every stream holds one kernel and nothing else.  No batch runs
more CTAs than the GPU has SMs.  Every destination has sentinels behind it, and every source is compared with its value
before the call.  The last tests drive ``SymmWorld.send_`` / ``recv_`` / ``isend_`` / ``irecv_`` for W ranks built over the
emulated mailboxes, one rank per stream.
"""
import random

import pytest
import torch

from emulated_ranks import (C, WRAP, _agree, _bytes, _check_message, _dest, _message, _unaligned, _values,  # noqa: F401
                            boxes, geo, on_ranks, pytestmark, sms, worlds)


def _transfer(boxes, pairs, seed):
    """One batch: pairs [(src, dst, nbytes)]; checks every destination, its sentinels and every source."""
    msgs = []
    for k, (a, b, n) in enumerate(pairs):
        x = _message(n, seed + k)
        msgs.append((a, b, x, x.cpu(), _dest(n)))
    boxes.run([(a, b, x, y[:n]) for (a, b, x, _, y), (_, _, n) in zip(msgs, pairs)])
    for a, b, x, xb, y in msgs:
        _check_message(f"rank {a} -> rank {b}, {x.numel()} bytes", x, xb, y)


def _agree(boxes, pairs):
    """After every message between a and b was received: fills (a) == ack (a) == flag (b) == consumed (b), slot by slot."""
    for a, b in pairs:
        ca, cb = boxes.counters(a), boxes.counters(b)
        for name, v in (("ack", ca["ack"][b]), ("flag", cb["flag"][a]), ("consumed", cb["consumed"][a])):
            assert torch.equal(v, ca["fills"][b]), (a, b, name, v, ca["fills"][b])


# ---------------------------------------------------------------------------------------------------------- sizes
def sizes(G, S, CHUNK):
    ring = G * S * CHUNK                        # one message of this size fills every slot once
    return [1, 15, 16, 17, 4096 + 3, CHUNK - 16, CHUNK, CHUNK + 16, 3 * CHUNK + 1, ring - 16, ring, ring + 16,
            2 * ring - 16, 2 * ring + 16, 3 * ring + 16 * 1021, 5 * ring + 16]


def test_message_sizes_across_the_chunk_and_the_slot_ring(C, boxes, geo):
    """One pair, one message per batch, on one mailbox: tails under 16 bytes, one piece, several pieces per CTA, and messages
    of several times G x S x CHUNK, whose sends wait for acknowledgements inside the message."""
    B = boxes(2)
    for k, n in enumerate(sizes(*geo[:3])):
        _transfer(B, [(0, 1, n)], seed=k)
    _agree(B, [(0, 1)])


@pytest.mark.parametrize("world", [3, 4])
def test_all_pairs_at_once(C, boxes, geo, world):
    """Every ordered pair of the world in one batch: each mailbox's source regions are written at the same time by
    different peers and must stay apart."""
    B = boxes(world)
    G, S, CHUNK = geo[:3]
    pairs = [(a, b) for a in range(world) for b in range(world) if a != b]
    # 2 x W x (W - 1) kernels run at once: full grids at world 3, grids of 5 at world 4
    for k, n in enumerate([G * S * CHUNK + 16, 3 * CHUNK + 5] if world == 3 else [5 * CHUNK - 16, 17]):
        _transfer(B, [(a, b, n + i) for i, (a, b) in enumerate(pairs)], seed=100 * world + 1000 * k)
    _agree(B, pairs)


def test_mixed_sizes_on_one_pair_without_host_synchronisation(C, boxes, geo):
    """60 messages of mixed sizes from rank 0 to rank 1 in one batch: each receive is submitted right after its send, and no
    host synchronisation separates them."""
    B = boxes(2)
    G, S, CHUNK = geo[:3]
    rng = random.Random(5)
    pick = [1, 15, 17, 4096, CHUNK - 16, CHUNK + 16, G * CHUNK + 3, G * S * CHUNK + 16, 2 * G * S * CHUNK - 16]
    ns = [rng.choice(pick) if k % 3 else rng.randint(1, 3 * G * S * CHUNK) for k in range(60)]
    _transfer(B, [(0, 1, n) for n in ns], seed=1000)
    _agree(B, [(0, 1)])


# ---------------------------------------------------------------------------------------------------------- rings and pairs
@pytest.mark.parametrize("world", range(2, 9))
def test_ring_every_rank_sends_right_and_receives_left(C, boxes, geo, world):
    """All ranks at once, every kernel at its full grid, then small and ragged messages on the same mailboxes."""
    B = boxes(world)
    G, S, CHUNK = geo[:3]
    for k, n in enumerate([3 * G * S * CHUNK + 16, 17, CHUNK + 48, 2 * G * S * CHUNK - 16]):
        _transfer(B, [(r, (r + 1) % world, n + r) for r in range(world)], seed=10 * world + 1000 * k)
    _agree(B, [(r, (r + 1) % world) for r in range(world)])


@pytest.mark.parametrize("world", [2, 4, 8])
def test_both_directions_of_each_pair_at_once(C, boxes, geo, world):
    B = boxes(world)
    G, S, CHUNK = geo[:3]
    for k, n in enumerate([2 * G * S * CHUNK + 16, 15, G * S * CHUNK + 4096]):
        pairs = []
        for r in range(0, world, 2):
            pairs += [(r, r + 1, n + r), (r + 1, r, n + 3 * r + 1)]
        _transfer(B, pairs, seed=20 * world + 1000 * k)
    _agree(B, [(r, r ^ 1) for r in range(world)])


# ---------------------------------------------------------------------------------------------------------- counter wrap
@pytest.mark.parametrize("world", [2, 5])
def test_counters_wrap_through_zero(C, boxes, geo, world):
    """Every counter word starts at 2^32 - 5; three rounds of a ring of 3 x G x S x CHUNK messages move every slot's
    counters through 0, and afterwards both sides agree on them."""
    B = boxes(world, start=WRAP)
    G, S, CHUNK = geo[:3]
    for k in range(3):
        _transfer(B, [(r, (r + 1) % world, 3 * G * S * CHUNK - 16 * k) for r in range(world)], seed=30 * world + k)
    _agree(B, [(r, (r + 1) % world) for r in range(world)])
    c = B.counters(0)["fills"][1 % world]
    assert bool(((c > 0) & (c < 100)).all()), c


# ---------------------------------------------------------------------------------------------------------- SymmWorld
CASES = [(torch.float32, 1), (torch.int64, 3), (torch.bfloat16, 4097), (torch.uint8, 17), (torch.bool, 1000),
         (torch.int16, 40000), (torch.float64, 0), (torch.int32, 100003), (torch.uint8, 1 << 20)]


@pytest.mark.parametrize("world", [2, 3, 5, 8])
@pytest.mark.parametrize("blocking", [False, True], ids=["isend_irecv", "send_recv"])
def test_symm_world_ring_any_dtype_aligned_or_not(C, sms, worlds, world, blocking):
    """A ring through the four methods with global ranks that are not 0..W-1: fp32 with NaN payloads and -0, integers,
    bool, bf16, zero elements, and up to G x S x CHUNK bytes per message; views that are not 16-byte aligned on either side.
    Every send of a batch is submitted before every receive."""
    globals_ = [3 + 2 * r for r in range(world)]
    ws, streams = worlds(world, globals_)
    for k, (dtype, numel) in enumerate(CASES):
        xs = [_values(dtype, numel, 100 * world + 10 * k + r).cuda() for r in range(world)]
        if dtype == torch.float32 and numel:
            xs[0][0] = float("nan")
        ys = [torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)]
        if k % 3 == 1:
            xs = [_unaligned(x) for x in xs]
        if k % 3 == 2:
            ys = [_unaligned(y) for y in ys]
        before = [_bytes(x) for x in xs]
        torch.cuda.synchronize()
        right = [globals_[(r + 1) % world] for r in range(world)]
        left = [globals_[(r - 1) % world] for r in range(world)]
        if blocking:
            on_ranks(ws, lambda r, w: w.send_(xs[r], right[r]), streams)
            on_ranks(ws, lambda r, w: w.recv_(ys[r], left[r]), streams)
        else:
            reqs = [None] * world
            on_ranks(ws, lambda r, w: reqs.__setitem__(r, [w.isend_(xs[r], right[r])]), streams)
            on_ranks(ws, lambda r, w: reqs[r].append(w.irecv_(ys[r], left[r])), streams)
            on_ranks(ws, lambda r, w: [q.wait() for q in reqs[r]], streams)
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(_bytes(ys[r]), before[(r - 1) % world]), (dtype, numel, r)
            assert torch.equal(_bytes(xs[r]), before[r]), ("source changed", dtype, numel, r)


def test_request_wait_orders_later_work_on_the_current_stream(C, worlds):
    """rank 1: irecv_, Request.wait(), then a copy on its current stream: the copy sees the received bytes, although the
    host never waited."""
    from dist_tuto.pth_b200 import comm
    ws, streams = worlds(2, [0, 1])
    G, S, CHUNK, _ = C.p2p_config()
    x = _values(torch.int32, G * S * CHUNK // 4, 7).cuda()
    y = torch.zeros_like(x)
    out = torch.zeros_like(x)
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        send = comm.Request(ws[0].isend_(x, 1), x)
    with torch.cuda.stream(streams[1]):
        req = comm.Request(ws[1].irecv_(y, 0), y)
        req.wait()
        out.copy_(y)
    with torch.cuda.stream(streams[0]):
        send.wait()
    torch.cuda.synchronize()
    assert torch.equal(out, x) and torch.equal(y, x)
    assert req.is_completed() and send.is_completed()


def test_is_completed_before_and_after_the_transfer(C, worlds):
    """A send queued behind a long kernel on the current stream has not completed when ``isend_`` returns; after the
    receive and a synchronisation both works report completion.  ``is_completed`` never blocks."""
    ws, streams = worlds(2, [0, 1])
    x = _values(torch.uint8, 1000, 9).cuda()
    y = torch.zeros_like(x)
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        torch.cuda._sleep(1_000_000_000)                    # ~0.5 s at H100 clocks: the send stream waits for it
        send = ws[0].isend_(x, 1)
    assert send.is_completed() is False
    with torch.cuda.stream(streams[1]):
        recv = ws[1].irecv_(y, 0)
    assert recv.is_completed() is False
    torch.cuda.synchronize()
    assert send.is_completed() and recv.is_completed()
    assert torch.equal(y, x)
