"""Model check of the point-to-point mailbox of csrc/p2p.cu (``p2p_send_kernel`` / ``p2p_recv_kernel``), in the abstract
machine style of tests/test_protocol_models.py.

The kernels' claim: a slot is a single-producer single-consumer channel between CTA c of the sender and CTA c of the
receiver.  The sender refills a slot only after the receiver's acknowledgement reached the slot's previous sequence number,
and the receiver reads a slot only after its flag reached the expected one.  Sender and receiver pick the same slot for every
piece from their own counters alone (round robin derived from the counts).  All counters are uint32 and compared wrap-safe.
So no receiver ever reads a stale or half-written slot, whatever the interleaving, message sizes and counter start.

Machine: every (rank, peer, direction) is a stream that runs its kernels one after the other (one kernel per message), and
inside a kernel every CTA is its own thread of control.  One atomic action is a flag or acknowledgement poll, the store of
one half of a slot (a slot is observed half old, half new while it is being written), the read of one half, a flag or
acknowledgement store, or a CTA's final store of its counters.  The scheduler interleaves all threads of all streams.  Every
interleaving is explored (depth-first over the reachable states) for 2 ranks, 1-2 CTAs and 1-2 slots; random skewed schedules
cover rings and bidirectional pairs at 3-8 ranks.  Negative controls: a sender that does not wait for the acknowledgement,
and a plain ``>=`` compare across the uint32 wrap, must both be caught.
"""
import random

import pytest

MOD = 1 << 32


def reached(have, want):
    """The kernels' wrap-safe compare: (int32_t)(have - want) >= 0."""
    return (have - want) % MOD < (1 << 31)


def plain_ge(have, want):
    """Negative control: a plain unsigned compare, wrong across the wrap."""
    return have >= want


def cursor(cnt):
    """The kernels' slot cursor (``load_counters``): the number of slots whose count equals slot 0's, mod S."""
    return sum(c == cnt[0] for c in cnt) % len(cnt)


class Mailbox:
    """The mailbox protocol over ``pairs``: {(src, dst): [pieces of message 0, message 1, ...]} (0 = a zero-byte message,
    which launches nothing).  ``ctas`` = G, ``slots`` = S, counters start at ``start``.  Streams are ("send", src, dst) and
    ("recv", dst, src)."""

    def __init__(self, pairs, ctas, slots, start=0, compare=reached, wait_for_ack=True):
        self.pairs, self.G, self.S = pairs, ctas, slots
        self.compare, self.wait_for_ack = compare, wait_for_ack
        self.streams = [("send", a, b) for (a, b) in pairs] + [("recv", b, a) for (a, b) in pairs]
        keys = []
        for (a, b) in pairs:
            for c in range(ctas):
                for s in range(slots):
                    keys += [("flag", b, a, c, s), ("ack", a, b, c, s), ("fills", a, b, c, s), ("consumed", b, a, c, s),
                             ("data", b, a, c, s, 0), ("data", b, a, c, s, 1)]
        self.index = {k: i for i, k in enumerate(keys)}
        mem = tuple(None if k[0] == "data" else start for k in keys)
        self.initial = (mem, self.normalize(mem, tuple((-1, ()) for _ in self.streams)))

    # ---------------------------------------------------------------------------------------------- kernels
    def kernel(self, mem, stream, m):
        """The CTAs (action tuples) of message m on `stream`, built from the counters as the kernel reads them."""
        kind, me, peer = stream
        a, b = (me, peer) if kind == "send" else (peer, me)
        n = self.pairs[(a, b)][m]
        ctas = []
        for c in range(min(self.G, n)):
            ckeys = [self.index[("fills" if kind == "send" else "consumed", me, peer, c, s)] for s in range(self.S)]
            cnt = [mem[k] for k in ckeys]
            s = cursor(cnt)
            acts = []
            for k in range(c, n, self.G):
                seq = (cnt[s] + 1) % MOD
                data = [self.index[("data", b, a, c, s, h)] for h in (0, 1)]
                if kind == "send":
                    if self.wait_for_ack:
                        acts.append(("wait", self.index[("ack", a, b, c, s)], (seq - 1) % MOD))
                    acts += [("store", data[0], (m, k, 0)), ("store", data[1], (m, k, 1)),
                             ("store", self.index[("flag", b, a, c, s)], seq)]
                else:
                    acts += [("wait", self.index[("flag", b, a, c, s)], seq), ("read", data[0], (m, k, 0)),
                             ("read", data[1], (m, k, 1)), ("store", self.index[("ack", a, b, c, s)], seq)]
                cnt[s] = seq
                s = (s + 1) % self.S
            acts += [("store", ckeys[q], cnt[q]) for q in range(self.S)]   # thread 0 writes the counters back
            ctas.append(tuple(acts))
        return tuple(ctas)

    def normalize(self, mem, streams):
        """Stream order: a stream whose kernel finished (or launched nothing) starts its next message's kernel."""
        out = []
        for i, (m, ctas) in enumerate(streams):
            st = self.streams[i]
            total = len(self.pairs[(st[1], st[2]) if st[0] == "send" else (st[2], st[1])])
            while not any(ctas) and m + 1 < total:
                m += 1
                ctas = self.kernel(mem, st, m)
            out.append((m, ctas))
        return tuple(out)

    # ---------------------------------------------------------------------------------------------- steps
    def enabled(self, state):
        mem, streams = state
        out = []
        for i, (_, ctas) in enumerate(streams):
            for c, acts in enumerate(ctas):
                if acts and (acts[0][0] != "wait" or self.compare(mem[acts[0][1]], acts[0][2])):
                    out.append((i, c))
        return out

    def step(self, state, i, c):
        """Run the next action of CTA c of stream i: (new state, violation or None)."""
        mem, streams = state
        m, ctas = streams[i]
        act, rest = ctas[c][0], ctas[c][1:]
        bad = None
        if act[0] == "store":
            mem = mem[:act[1]] + (act[2],) + mem[act[1] + 1:]
        elif act[0] == "read" and mem[act[1]] != act[2]:
            kind, me, peer = self.streams[i]
            bad = f"rank {me} read {mem[act[1]]} from rank {peer}'s slot while expecting {act[2]} (message, piece, half)"
        ctas = ctas[:c] + (rest,) + ctas[c + 1:]
        streams = streams[:i] + ((m, ctas),) + streams[i + 1:]
        return (mem, self.normalize(mem, streams)), bad

    def done(self, state):
        return not any(any(ctas) for _, ctas in state[1])

    # ---------------------------------------------------------------------------------------------- drivers
    def run(self, choose, max_ticks=10 ** 6):
        """One schedule: `choose(enabled (stream, cta) list) -> element`.  None when every transfer completed correctly."""
        state = self.initial
        for _ in range(max_ticks):
            if self.done(state):
                return None
            en = self.enabled(state)
            if not en:
                return "deadlock: streams at messages %s" % [m for m, _ in state[1]]
            state, bad = self.step(state, *choose(en))
            if bad:
                return bad
        return "did not terminate"

    def explore(self, limit=2_000_000):
        """Every interleaving: depth-first over the reachable states.  Returns (violation or None, states visited)."""
        seen, stack = {self.initial}, [self.initial]
        while stack:
            state = stack.pop()
            if self.done(state):
                continue
            en = self.enabled(state)
            if not en:
                return "deadlock: streams at messages %s" % [m for m, _ in state[1]], len(seen)
            for i, c in en:
                nxt, bad = self.step(state, i, c)
                if bad:
                    return bad, len(seen)
                if nxt not in seen:
                    seen.add(nxt)
                    stack.append(nxt)
            assert len(seen) <= limit, "state space larger than the exploration limit"
        return None, len(seen)


# ---------------------------------------------------------------------------------------------------------- every interleaving
# Message sizes in pieces; with G CTAs and S slots each sequence makes every CTA fill every one of its slots at least twice,
# and it includes a zero-byte message and a one-piece message between longer ones.
def reuse_sequence(ctas, slots):
    per = ctas * slots
    return [per + 1, 0, 1, per]


WRAP = MOD - 3                                  # counters that pass through 0 inside the sequences


@pytest.mark.parametrize("slots", [1, 2])
@pytest.mark.parametrize("ctas", [1, 2])
@pytest.mark.parametrize("start", [0, WRAP], ids=["zero", "wrap"])
def test_one_direction_every_interleaving_is_safe(ctas, slots, start):
    mb = Mailbox({(0, 1): reuse_sequence(ctas, slots)}, ctas, slots, start)
    bad, n = mb.explore()
    assert bad is None, bad
    assert n > 50                               # the search really branched


@pytest.mark.parametrize("ctas,slots", [(1, 1), (1, 2), (2, 1)])
def test_both_directions_of_a_pair_every_interleaving_is_safe(ctas, slots):
    seq = [ctas * slots + 1, 1]
    mb = Mailbox({(0, 1): seq, (1, 0): seq[::-1]}, ctas, slots, WRAP)
    bad, n = mb.explore()
    assert bad is None, bad
    assert n > 50


def test_every_slot_is_reused_by_the_sequences():
    """The exhaustive sequences really refill every slot: after them every counter advanced at least twice."""
    for ctas in (1, 2):
        for slots in (1, 2):
            mb = Mailbox({(0, 1): reuse_sequence(ctas, slots)}, ctas, slots)
            assert mb.run(lambda en: en[0]) is None
            pieces = [0] * ctas
            for n in reuse_sequence(ctas, slots):
                for k in range(n):
                    pieces[k % ctas] += 1
            assert min(pieces) >= 2 * slots


# ---------------------------------------------------------------------------------------------------------- random schedules
def _random_sizes(rng, n, max_pieces):
    return [rng.choice([0, 1, 1, 2, rng.randint(1, max_pieces)]) for _ in range(n)]


def _skewed(rng, world):
    """A scheduler where some ranks run much faster than others."""
    weights = [rng.choice([1, 1, 5, 25]) for _ in range(world)]

    def choose(en, mb):
        return rng.choices(en, weights=[weights[mb.streams[i][1]] for i, _ in en])[0]
    return choose


@pytest.mark.parametrize("world", [3, 4, 5, 8])
def test_random_schedules_of_rings_are_safe(world):
    """Every rank sends to its right and receives from its left at once, message sizes drawn per pair."""
    for seed in range(40):
        rng = random.Random(seed * 7919 + world)
        ctas, slots = rng.choice([(2, 2), (8, 2), (3, 1)])
        pairs = {(r, (r + 1) % world): _random_sizes(rng, 6, 3 * ctas * slots) for r in range(world)}
        mb = Mailbox(pairs, ctas, slots, rng.choice([0, WRAP, MOD - 1]))
        choose = _skewed(rng, world)
        bad = mb.run(lambda en: choose(en, mb))
        assert bad is None, (seed, bad)


@pytest.mark.parametrize("world", [3, 4, 6, 8])
def test_random_schedules_of_bidirectional_pairs_are_safe(world):
    """Ranks 2i and 2i + 1 exchange in both directions at once (and rank 0 also sends to the last rank at odd worlds)."""
    for seed in range(40):
        rng = random.Random(seed * 104729 + world)
        ctas, slots = rng.choice([(2, 2), (8, 2), (1, 2)])
        pairs = {}
        for r in range(0, world - 1, 2):
            pairs[(r, r + 1)] = _random_sizes(rng, 5, 3 * ctas * slots)
            pairs[(r + 1, r)] = _random_sizes(rng, 5, 3 * ctas * slots)
        if world % 2:
            pairs[(0, world - 1)] = _random_sizes(rng, 5, 3 * ctas * slots)
        mb = Mailbox(pairs, ctas, slots, rng.choice([0, WRAP]))
        choose = _skewed(rng, world)
        bad = mb.run(lambda en: choose(en, mb))
        assert bad is None, (seed, bad)


# ---------------------------------------------------------------------------------------------------------- negative controls
def test_a_sender_that_does_not_wait_for_the_ack_is_caught():
    """Without the acknowledgement wait a fast sender refills a slot its receiver has not read: the exhaustive search finds
    the stale read, and so does a schedule where the sender runs ahead."""
    mb = Mailbox({(0, 1): [3, 2]}, 1, 2, wait_for_ack=False)
    bad, _ = mb.explore()
    assert bad is not None and "read" in bad, bad
    sender_first = mb.run(lambda en: min(en, key=lambda e: mb.streams[e[0]][0] != "send"))
    assert sender_first is not None and "read" in sender_first, sender_first


def test_a_plain_compare_across_the_wrap_is_caught():
    """With ``>=`` on the raw uint32 values, a counter that wrapped to 0 looks already reached: the receiver reads a slot
    the sender has not written yet.  The same start with the wrap-safe compare is safe (tests above)."""
    mb = Mailbox({(0, 1): [3, 2]}, 1, 2, MOD - 1, compare=plain_ge)
    bad, _ = mb.explore()
    assert bad is not None and "read" in bad, bad
    assert Mailbox({(0, 1): [3, 2]}, 1, 2, 5, compare=plain_ge).explore()[0] is None     # far from the wrap it holds
