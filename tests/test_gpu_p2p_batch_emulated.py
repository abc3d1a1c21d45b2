"""The point-to-point batch kernel (``p2p_batch``, csrc/p2p.cu) on ONE GPU with W emulated ranks, bit for bit.

The harness is tests/emulated_ranks.py's mailboxes: each rank has its own mailbox, every (rank, peer, direction) and every
rank's batch gets a CUDA stream of its own (``stream_create``), destinations have sentinels behind them, sources are compared
with their values before the call, and no round runs more CTAs than the GPU has SMs.  A round is submitted so that no stream
holds a kernel that waits for one submitted after it behind another of its own: batches go first, and a rank that uses single
launches against another rank's batch waits only on that batch.

Besides the bytes, every test compares the counter words of every rank's signal pad with those of a second set of mailboxes
that ran the same messages as single sends and receives: after a batch every counter holds what the single launches leave.
The last tests drive ``SymmWorld.batch_p2p_`` for W ranks over the emulated mailboxes, one thread per rank, in phases where
each batch waits only for work submitted before it.
"""
import random
import threading

import pytest
import torch

import emulated_ranks as E
from emulated_ranks import C, WRAP, boxes, geo, pytestmark, sms, worlds  # noqa: F401


def _nbytes(t):
    return t.numel() * t.element_size()


class Round:
    """One round of messages: ``transfers`` [(src, dst, nbytes)] in per-pair order.  ``batched`` ranks issue all their ops
    of the round in one ``p2p_batch`` (``order``: "sends_first", "recvs_first" or a seeded shuffle that keeps each pair's
    order); the other ranks issue single ``p2p_send`` / ``p2p_recv`` launches on their pair streams."""

    def __init__(self, transfers, batched, order="sends_first", seed=0):
        self.transfers, self.batched, self.order, self.seed = transfers, set(batched), order, seed


def _ops(rnd, msgs, world):
    """Every rank's op list for the round: [(send, peer, tensor)]."""
    sends = {r: [] for r in range(world)}
    recvs = {r: [] for r in range(world)}
    for (a, b, _), (x, _, y) in zip(rnd.transfers, msgs):
        sends[a].append((True, b, x))
        recvs[b].append((False, a, y))
    ops = {}
    rng = random.Random(rnd.seed)
    for r in range(world):
        if rnd.order == "sends_first":
            ops[r] = sends[r] + recvs[r]
        elif rnd.order == "recvs_first":
            ops[r] = recvs[r] + sends[r]
        else:                                               # a random merge: each list keeps its order
            s, v, out = list(sends[r]), list(recvs[r]), []
            while s or v:
                out.append((s if s and (not v or rng.random() < 0.5) else v).pop(0))
            ops[r] = out
    return ops


def _run_round(B, rnd, msgs):
    ops = _ops(rnd, msgs, B.world)
    busy = {}
    for r in range(B.world):
        if r in rnd.batched:
            lanes = {(s, p) for s, p, t in ops[r] if _nbytes(t)}
            grid = max([B.grid(_nbytes(t)) for _, _, t in ops[r]] + [0])
            busy[(r, "batch")] = len(lanes) * grid
        else:
            for s, p, t in ops[r]:
                busy[(r, p, s)] = max(busy.get((r, p, s), 0), B.grid(_nbytes(t)))
    assert sum(busy.values()) <= B.sms, f"{sum(busy.values())} CTAs would not be co-resident on {B.sms} SMs"
    torch.cuda.synchronize()
    for r in sorted(rnd.batched):
        with torch.cuda.stream(B.stream(r, -1, "batch")):
            B.C.p2p_batch(B.box_ptrs, B.sig_ptrs, [(s, t, p) for s, p, t in ops[r]], r, B.world)
    for r in range(B.world):
        if r not in rnd.batched:
            for s, p, t in ops[r]:
                with torch.cuda.stream(B.stream(r, p, s)):
                    (B.C.p2p_send if s else B.C.p2p_recv)(B.box_ptrs, B.sig_ptrs, t, p, r, B.world)
    torch.cuda.synchronize()


def run_and_check(boxes, world, rounds, seed, start=0):
    """Run the rounds on one set of mailboxes, check every destination, its sentinels and every source, then run the same
    messages as single launches on a second set and compare every counter word of every rank."""
    B = boxes(world, start)
    k = 0
    for rnd in rounds:
        msgs = []
        for a, b, n in rnd.transfers:
            x = E._message(n, seed + k)
            k += 1
            msgs.append((x, x.cpu(), E._dest(n)))
        _run_round(B, rnd, [(x, xb, y[:_nbytes(x)]) for x, xb, y in msgs])
        for (a, b, n), (x, xb, y) in zip(rnd.transfers, msgs):
            E._check_message(f"rank {a} -> rank {b}, {n} bytes", x, xb, y)
    R = boxes(world, start)
    for rnd in rounds:
        R.run([(a, b, E._message(n, 0), torch.empty(n, dtype=torch.uint8, device="cuda")) for a, b, n in rnd.transfers])
    for r in range(world):
        got, want = B.counters(r), R.counters(r)
        for name in got:
            assert torch.equal(got[name], want[name]), (f"rank {r} {name} after the batches differs from the single "
                                                        f"launches", got[name], want[name])
    pairs = {(a, b) for rnd in rounds for a, b, n in rnd.transfers if n}
    E._agree(B, sorted(pairs))
    return B


def _grid_for(sms_, world, lanes_per_rank, G):
    """The largest grid (pieces per message, at most G) at which every rank's batch of this many lanes is co-resident."""
    return max(1, min(G, sms_ // (world * lanes_per_rank)))


# ---------------------------------------------------------------------------------------------------------- rings and pairs
@pytest.mark.parametrize("world", range(2, 9))
def test_ring_in_one_batch_per_rank(C, sms, boxes, geo, world):
    """Every rank sends right and receives left in one batch, at full grids, then ragged and tiny messages, with the
    receive listed first, sends first, and shuffled."""
    G, S, CHUNK = geo[:3]
    rounds = []
    for k, (n, order) in enumerate([(2 * G * S * CHUNK + 16, "sends_first"), (17, "recvs_first"),
                                    (CHUNK + 48, "shuffle"), (G * S * CHUNK - 16, "sends_first")]):
        rounds.append(Round([(r, (r + 1) % world, n + r) for r in range(world)], range(world), order, seed=k))
    run_and_check(boxes, world, rounds, seed=10 * world)


@pytest.mark.parametrize("world", range(2, 9))
def test_all_pairs_both_directions_in_one_batch_per_rank(C, sms, boxes, geo, world):
    """Every rank sends to and receives from every peer in one batch: 2 x (world - 1) lanes per rank, every mailbox region
    written by different peers at once.  Message sizes fill the grid the SMs allow (one piece per lane at 7-8 ranks)."""
    G, S, CHUNK = geo[:3]
    g = _grid_for(sms, world, 2 * (world - 1), G)
    pairs = [(a, b) for a in range(world) for b in range(world) if a != b]
    rounds = [Round([(a, b, g * CHUNK - 16 * i) for i, (a, b) in enumerate(pairs)], range(world), "sends_first"),
              Round([(a, b, 1 + i) for i, (a, b) in enumerate(pairs)], range(world), "shuffle", seed=3)]
    run_and_check(boxes, world, rounds, seed=100 * world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sends_listed_before_receives_beyond_the_mailbox(C, sms, boxes, geo, world):
    """Each rank lists its sends (to both neighbours) before its receives, every message larger than a pair's
    G x S x CHUNK slots: split into two launches on one stream these batches would wait for each other for ever."""
    G, S, CHUNK = geo[:3]
    ring = G * S * CHUNK
    g = _grid_for(sms, world, 4 if world > 2 else 2, G)
    n = 2 * ring + 16 if g == G else 3 * g * S * CHUNK + 16
    transfers = [(r, (r + 1) % world, n + 16 * r) for r in range(world)]
    if world > 2:
        transfers += [(r, (r - 1) % world, n + 3) for r in range(world)]
    else:
        transfers += [(1, 0, n + 5)]
    run_and_check(boxes, world, [Round(transfers, range(world), "sends_first")], seed=7 * world)


def sizes(G, S, CHUNK):
    return [0, 1, 15, 16, 17, 0, CHUNK - 16, CHUNK, CHUNK + 16, G * CHUNK, G * CHUNK + 16, G * S * CHUNK + 16, 33]


def test_several_ops_to_one_peer_in_one_batch(C, sms, boxes, geo):
    """Thirteen messages each way between two ranks in one batch per rank: zero bytes, tails under 16 bytes, chunk edges
    and more than G x CHUNK; the lanes carry them in list order."""
    G, S, CHUNK = geo[:3]
    ns = sizes(G, S, CHUNK)
    transfers = [(0, 1, n) for n in ns] + [(1, 0, n + 1 if n else 0) for n in reversed(ns)]
    rounds = [Round(transfers, [0, 1], "sends_first"), Round(transfers, [0, 1], "shuffle", seed=11)]
    run_and_check(boxes, 2, rounds, seed=500)


@pytest.mark.parametrize("world", [2, 3])
def test_a_batch_against_single_launches(C, sms, boxes, geo, world):
    """Rank 0 batches its messages to and from rank 1 (and rank 2); the peers issue one launch per message on their pair
    streams, in the same per-pair order."""
    G, S, CHUNK = geo[:3]
    ns = [17, G * S * CHUNK + 16, 0, CHUNK, 3 * G * S * CHUNK - 16, 1]
    transfers = []
    for p in range(1, world):
        transfers += [(0, p, n + p) for n in ns] + [(p, 0, 2 * n + p) for n in ns]
    run_and_check(boxes, world, [Round(transfers, [0], "shuffle", seed=world), Round(transfers, [0], "recvs_first")],
                  seed=900)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_mixed_sequences_through_the_counter_wrap(C, sms, boxes, geo, world):
    """Counters start at 2^32 - 5.  Rounds of single launches, batches on every rank, and batches on every other rank
    against single launches on the rest move every counter of a ring's pairs through 0; afterwards the counters equal those
    of the same messages sent one by one."""
    G, S, CHUNK = geo[:3]
    big = 2 * G * S * CHUNK + 16                            # a ring of these runs at full grids at every world
    g = _grid_for(sms, world, 4, G)                         # both directions: full grids up to 4 ranks
    nb = big if g == G else g * CHUNK - 16
    both = lambda n: [(r, (r + 1) % world, n + r) for r in range(world)] + \
        [(r, (r - 1) % world, n + 2 * r + 1) for r in range(world) if world > 2 or r == 1]
    even = [r for r in range(world) if r % 2 == 0]
    odd = [r for r in range(world) if r % 2 == 1]
    right = lambda n: [(r, (r + 1) % world, n + r) for r in range(world)]
    rounds = [Round(right(big), []), Round(both(nb), range(world), "sends_first"),
              Round(right(CHUNK + 1), even if world % 2 == 0 else range(world), "shuffle", seed=1),
              Round(right(big - 32), odd if world % 2 == 0 else range(world), "recvs_first"),
              Round(right(15), []), Round(both(nb - 48), range(world), "shuffle", seed=2),
              Round(right(big + 16), range(world), "sends_first")]
    B = run_and_check(boxes, world, rounds, seed=40 * world, start=WRAP)
    c = B.counters(0)["fills"][1 % world]
    assert bool(((c > 0) & (c < 100)).all()), c


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def _threads(ws, streams, fn):
    """fn(r, world_r) for every rank, each on its own thread with its own current stream; returns when all were issued."""
    errs = []

    def body(r, w):
        try:
            with torch.cuda.stream(streams[r]):
                fn(r, w)
        except BaseException as e:                           # noqa: BLE001 - re-raised on the main thread
            errs.append(e)
    ts = [threading.Thread(target=body, args=(r, w)) for r, w in enumerate(ws)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]


def _in_order(ws, streams, ranks, fn):
    """fn(r, world_r) for the given ranks one after another, each rank's calls on its own thread and current stream."""
    for r in ranks:
        _threads([ws[r]], [streams[r]], lambda _, w, r=r: fn(r, w))


CASES = [(torch.float32, 1), (torch.int64, 3), (torch.bfloat16, 4097), (torch.uint8, 17), (torch.bool, 1000),
         (torch.int16, 40000), (torch.float64, 0), (torch.int32, 100003), (torch.uint8, 1 << 20)]


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_symm_world_batches_any_dtype_aligned_or_not(C, sms, worlds, world):
    """Through ``SymmWorld.batch_p2p_`` with global ranks that are not 0..W-1, every dtype, zero elements and up to
    G x S x CHUNK bytes, on views that are not 16-byte aligned on either side.  Phase 1: every rank sends to both neighbours
    in one batch, all ranks on their own threads at once (each send fits its pair's slots, so every batch ends by itself).
    Phase 2: every rank receives from both neighbours in one batch, again all at once."""
    globals_ = [3 + 2 * r for r in range(world)]
    ws, streams = worlds(world, globals_)
    for k, (dtype, numel) in enumerate(CASES):
        xs = [E._values(dtype, numel, 100 * world + 10 * k + r).cuda() for r in range(world)]
        if dtype == torch.float32 and numel:
            xs[0][0] = float("nan")
        ys = {(r, d): torch.zeros(numel, dtype=dtype, device="cuda") for r in range(world) for d in (-1, 1)}
        if k % 3 == 1:
            xs = [E._unaligned(x) for x in xs]
        if k % 3 == 2:
            ys = {key: E._unaligned(y) for key, y in ys.items()}
        before = [E._bytes(x) for x in xs]
        torch.cuda.synchronize()
        works = {}
        nbrs = lambda r: sorted({(r + 1) % world, (r - 1) % world})
        _threads(ws, streams, lambda r, w: works.__setitem__(
            (r, "s"), w.batch_p2p_([(True, xs[r], globals_[q]) for q in nbrs(r)])))
        _threads(ws, streams, lambda r, w: works.__setitem__(
            (r, "r"), w.batch_p2p_([(False, ys[(r, 1 if q == (r + 1) % world else -1)], globals_[q]) for q in nbrs(r)])))
        _threads(ws, streams, lambda r, w: [x.wait() for x in works[(r, "s")] + works[(r, "r")]])
        torch.cuda.synchronize()
        for r in range(world):
            assert len(works[(r, "s")]) == len(nbrs(r)) and len(works[(r, "r")]) == len(nbrs(r))
            for q in nbrs(r):
                d = 1 if q == (r + 1) % world else -1
                assert torch.equal(E._bytes(ys[(r, d)]), before[q]), (dtype, numel, r, q)
            assert torch.equal(E._bytes(xs[r]), before[r]), ("source changed", dtype, numel, r)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_symm_world_ring_with_sends_and_receives_in_one_batch(C, sms, worlds, world):
    """Ranks 1..W-1 each run one batch [send right, receive left]; rank 0 sends with ``isend_`` before them and receives in
    a batch after them, so every batch waits only for work submitted before it.  Then the pairs go on with single calls,
    which come after the batches on the same pairs."""
    globals_ = list(range(world))
    ws, streams = worlds(world, globals_)
    G, S, CHUNK, _ = C.p2p_config()
    for k, (dtype, numel) in enumerate([(torch.float32, G * S * CHUNK // 4), (torch.int16, 12345), (torch.uint8, 3)]):
        xs = [E._values(dtype, numel, 1000 * world + 10 * k + r).cuda() for r in range(world)]
        ys = [torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)]
        zs = [torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)]
        torch.cuda.synchronize()
        reqs = {r: [] for r in range(world)}
        right = lambda r: (r + 1) % world
        left = lambda r: (r - 1) % world
        _in_order(ws, streams, [0], lambda r, w: reqs[r].append(w.isend_(xs[r], right(r))))
        _in_order(ws, streams, range(1, world), lambda r, w: reqs[r].extend(
            w.batch_p2p_([(True, xs[r], right(r)), (False, ys[r], left(r))])))
        _in_order(ws, streams, [0], lambda r, w: reqs[r].extend(w.batch_p2p_([(False, ys[r], left(r))])))
        _in_order(ws, streams, range(world), lambda r, w: [q.wait() for q in reqs[r]])
        # pass the received tensors on with single calls on the same pairs: sends first, then receives
        _in_order(ws, streams, range(world), lambda r, w: reqs[r].append(w.isend_(ys[r], right(r))))
        _in_order(ws, streams, range(world), lambda r, w: reqs[r].append(w.irecv_(zs[r], left(r))))
        _in_order(ws, streams, range(world), lambda r, w: [q.wait() for q in reqs[r]])
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(E._bytes(ys[r]), E._bytes(xs[left(r)])), (dtype, numel, r)
            assert torch.equal(E._bytes(zs[r]), E._bytes(xs[left(left(r))])), (dtype, numel, r)


def test_request_wait_orders_later_work_on_the_current_stream(C, worlds):
    """rank 0 sends in a batch; rank 1 receives in a batch, calls Request.wait(), then copies on its current stream: the
    copy sees the received bytes, although the host never waited."""
    from dist_tuto.pth_b200 import comm
    ws, streams = worlds(2, [0, 1])
    G, S, CHUNK, _ = C.p2p_config()
    x = E._values(torch.int32, G * CHUNK // 4, 7).cuda()     # with x2, fits the pair's slots: the send batch ends by itself
    x2 = E._values(torch.int8, 999, 8).cuda()
    y, y2 = torch.zeros_like(x), torch.zeros_like(x2)
    out = torch.zeros_like(x)
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        sends = [comm.Request(wk, t) for wk, t in zip(ws[0].batch_p2p_([(True, x, 1), (True, x2, 1)]), (x, x2))]
    with torch.cuda.stream(streams[1]):
        recvs = [comm.Request(wk, t) for wk, t in zip(ws[1].batch_p2p_([(False, y, 0), (False, y2, 0)]), (y, y2))]
        recvs[0].wait()
        out.copy_(y)
    with torch.cuda.stream(streams[0]):
        for s in sends:
            s.wait()
    torch.cuda.synchronize()
    assert torch.equal(out, x) and torch.equal(y, x) and torch.equal(y2, x2)
    assert all(r.is_completed() for r in sends + recvs)
    assert recvs[0]._work is None and recvs[1]._work is not None
    assert recvs[1].is_completed() and recvs[1]._work.event is not None


def test_is_completed_before_and_after_the_batch(C, worlds):
    """A batch queued behind a long kernel on the current stream has not completed when ``batch_p2p_`` returns, and its
    works share one event; after the peer's batch and a synchronisation every work reports completion."""
    ws, streams = worlds(2, [0, 1])
    x, x2 = E._values(torch.uint8, 1000, 9).cuda(), E._values(torch.uint8, 70000, 10).cuda()
    y, y2 = torch.zeros_like(x), torch.zeros_like(x2)
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        torch.cuda._sleep(1_000_000_000)                    # ~0.5 s at H100 clocks: the batch stream waits for it
        send = ws[0].batch_p2p_([(True, x, 1), (True, x2, 1)])
    assert [w.is_completed() for w in send] == [False, False]
    assert send[0].event is send[1].event
    with torch.cuda.stream(streams[1]):
        recv = ws[1].batch_p2p_([(False, y, 0), (False, y2, 0)])
    assert not any(w.is_completed() for w in recv)
    torch.cuda.synchronize()
    assert all(w.is_completed() for w in send + recv)
    assert torch.equal(y, x) and torch.equal(y2, x2)


def test_batch_streams_are_per_set_of_pairs_and_never_pooled(C, worlds):
    """A batch's stream is one of this world's own, shared only by batches with the same (peer, direction) pairs, and every
    pair it touched has a stream that later single calls use."""
    ws, streams = worlds(3, [0, 1, 2])
    x = [torch.zeros(64, dtype=torch.uint8, device="cuda") for _ in range(6)]
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        ws[0].batch_p2p_([(True, x[0], 1), (True, x[1], 2)])
    with torch.cuda.stream(streams[1]):
        ws[1].batch_p2p_([(False, x[2], 0)])
    with torch.cuda.stream(streams[2]):
        ws[2].batch_p2p_([(False, x[3], 0)])
    torch.cuda.synchronize()
    keys = set(ws[0]._p2p_streams)
    assert keys == {(1, True), (2, True), ("batch", (1, True), (2, True))}
    handles = {s.cuda_stream for w in ws for s in w._p2p_streams.values()}
    assert len(handles) == sum(len(w._p2p_streams) for w in ws)
