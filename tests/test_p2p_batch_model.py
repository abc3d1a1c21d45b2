"""Model of the lane schedule of the point-to-point batch kernel (``p2p_batch_kernel`` in csrc/p2p.cu), in the abstract
machine style of tests/test_p2p_protocol_model.py.

The kernel's claims: a batch is one launch whose CTA (c, lane) runs the ops of one (peer, direction) one after another, each
exactly as CTA c of the single-message kernel would (same pieces, same slot choice from its own counters, same stores), and
skips an op that has no piece for it.  So after a batch every counter word holds what the ops launched one by one in list
order leave, and a batch never waits on itself: its lanes progress independently, whatever the list order.  Splitting a
batch into two launches on one stream loses that.

Machine: a launch (a batch, or one single op) starts once every earlier launch of its rank that shares a (peer, direction)
with it has finished -- the order ``SymmWorld`` gives them through the pair streams -- or, for the planted split, every
earlier launch on the same stream.  Every CTA of a started launch is its own thread; one atomic action is an acknowledgement
or flag poll, the store of one half of a slot, the read of one half, a flag or acknowledgement store, or a counter store.
Every CTA builds an op's actions from the counters when it starts that op, as the kernel loads them.  Random skewed
schedules explore worlds 2..8 with G CTAs and S slots per pair; a stale or torn read, or a state where nothing can move
before everything finished, is reported.
"""
import random

import pytest

MOD = 1 << 32
WRAP = MOD - 3


def reached(have, want):
    return (have - want) % MOD < (1 << 31)


def cursor(cnt):
    return sum(c == cnt[0] for c in cnt) % len(cnt)


class Machine:
    """``programs``: {rank: [launch, ...]} in issue order; a launch is (keys, [(send, peer, pieces, msg id)]).  G CTAs and
    S slots per pair, every counter starting at ``start``."""

    def __init__(self, programs, G, S, start=0):
        self.G, self.S, self.start = G, S, start
        self.mem = {}
        self.programs = programs
        self.pending = {r: list(range(len(p))) for r, p in programs.items()}   # launches not started yet
        self.running = {}                                                      # (rank, launch) -> [thread]
        self.done = set()

    def word(self, key):
        return self.mem.get(key, None if key[0] == "data" else self.start)

    # ---------------------------------------------------------------------------------------------- launches
    def _can_start(self, r, i):
        keys = self.programs[r][i][0]
        return all((r, j) in self.done for j in range(i) if keys & self.programs[r][j][0])

    def _start_ready(self):
        started = True
        while started:                                      # a launch without pieces (zero-byte ops only) ends at once
            started = False
            for r, todo in self.pending.items():
                for i in list(todo):
                    if self._can_start(r, i):
                        todo.remove(i)
                        threads = self._threads(r, self.programs[r][i][1])
                        if threads:
                            self.running[(r, i)] = threads
                        else:
                            self.done.add((r, i))
                            started = True

    def _threads(self, r, ops):
        lanes = {}
        for send, peer, pieces, mid in ops:
            lanes.setdefault((send, peer), []).append((send, peer, pieces, mid))
        threads = []
        for lane_ops in lanes.values():
            for c in range(self.G):
                mine = [op for op in lane_ops if c < op[2]]            # an op with no piece for CTA c is skipped
                if mine:
                    threads.append({"rank": r, "c": c, "ops": mine, "acts": []})
        return threads

    def _op_actions(self, th):
        """The actions of the thread's next op, built from the counters as CTA c loads them when it starts the op."""
        send, peer, pieces, mid = th["ops"].pop(0)
        me, c, G, S = th["rank"], th["c"], self.G, self.S
        a, b = (me, peer) if send else (peer, me)
        own = [("fills" if send else "consumed", me, peer, c, s) for s in range(S)]
        cnt = [self.word(k) for k in own]
        s = cursor(cnt)
        acts = []
        for k in range(c, pieces, G):
            seq = (cnt[s] + 1) % MOD
            data = [("data", b, a, c, s, h) for h in (0, 1)]
            if send:
                acts += [("wait", ("ack", a, b, c, s), (seq - 1) % MOD), ("store", data[0], (mid, k, 0)),
                         ("store", data[1], (mid, k, 1)), ("store", ("flag", b, a, c, s), seq)]
            else:
                acts += [("wait", ("flag", b, a, c, s), seq), ("read", data[0], (mid, k, 0)),
                         ("read", data[1], (mid, k, 1)), ("store", ("ack", a, b, c, s), seq)]
            cnt[s] = seq
            s = (s + 1) % S
        acts += [("store", own[q], cnt[q]) for q in range(S)]
        return acts

    # ---------------------------------------------------------------------------------------------- steps
    def _enabled(self):
        out = []
        for key, threads in self.running.items():
            for t, th in enumerate(threads):
                while not th["acts"] and th["ops"]:
                    th["acts"] = self._op_actions(th)
                if th["acts"]:
                    act = th["acts"][0]
                    if act[0] != "wait" or reached(self.word(act[1]), act[2]):
                        out.append((key, t))
        return out

    def run(self, rng, max_ticks=10 ** 7):
        """One random skewed schedule.  None when every launch finished with every read correct, else what went wrong."""
        weight = {r: rng.choice([1, 1, 5, 25]) for r in self.programs}
        self._start_ready()
        for _ in range(max_ticks):
            en = self._enabled()
            if not en:
                if not self.running and not any(self.pending.values()):
                    return None
                return "deadlock: running launches %s, not started %s" % (sorted(self.running), self.pending)
            key, t = rng.choices(en, weights=[weight[k[0]] for k, _ in en])[0]
            th = self.running[key][t]
            act = th["acts"].pop(0)
            if act[0] == "store":
                self.mem[act[1]] = act[2]
            elif act[0] == "read" and self.word(act[1]) != act[2]:
                return f"rank {th['rank']} read {self.word(act[1])} where it expected {act[2]}"
            if all(not x["acts"] and not x["ops"] for x in self.running[key]):
                del self.running[key]
                self.done.add(key)
                self._start_ready()
        return "did not terminate"

    def counters(self):
        return {k: v for k, v in self.mem.items() if k[0] != "data"}


# ---------------------------------------------------------------------------------------------------------- programs
def random_pairs(rng, world, G, S, max_msgs=4):
    """{(src, dst): [pieces of message 0, 1, ...]} for a random subset of ordered pairs; 0 is a zero-byte message."""
    pairs = {}
    for a in range(world):
        for b in range(world):
            if a != b and rng.random() < 0.6:
                pairs[(a, b)] = [rng.choice([0, 1, 2, G, G * S + 1, rng.randint(1, 3 * G * S)])
                                 for _ in range(rng.randint(1, max_msgs))]
    return pairs


def op_lists(rng, world, pairs, order="shuffle"):
    """Every rank's ops [(send, peer, pieces, msg id)]: its sends and receives, each pair in message order, merged at
    random (or sends first)."""
    out = {}
    for r in range(world):
        sends = [(True, b, n, (r, b, m)) for (a, b), ns in sorted(pairs.items()) if a == r for m, n in enumerate(ns)]
        recvs = [(False, a, n, (a, r, m)) for (a, b), ns in sorted(pairs.items()) if b == r for m, n in enumerate(ns)]
        if order == "sends_first":
            out[r] = sends + recvs
            continue
        per = {}
        for op in sends + recvs:
            per.setdefault((op[0], op[1]), []).append(op)
        queues, merged = list(per.values()), []
        while any(queues):
            q = rng.choice([q for q in queues if q])
            merged.append(q.pop(0))
        out[r] = merged
    return out


def batches(ops):
    """One batch per rank, keyed by every (peer, direction) it touches."""
    return {r: [(frozenset((s, p) for s, p, _, _ in lst), lst)] for r, lst in ops.items()}


def singles(ops):
    """Every op its own launch on its pair's stream."""
    return {r: [(frozenset([(s, p)]), [op]) for op in lst for s, p in [op[:2]]] for r, lst in ops.items()}


# ---------------------------------------------------------------------------------------------------------- invariant
@pytest.mark.parametrize("world", range(2, 9))
def test_counters_after_a_batch_equal_the_ops_one_by_one(world):
    """Random op lists: one batch per rank leaves every counter word as the same ops launched one at a time in list order,
    and every read sees the piece it expects."""
    for seed in range(25):
        rng = random.Random(seed * 7919 + world)
        G, S = rng.choice([(2, 2), (3, 1), (2, 1), (4, 2)])
        start = rng.choice([0, WRAP, MOD - 1])
        pairs = random_pairs(rng, world, G, S)
        ops = op_lists(rng, world, pairs)
        batched = Machine(batches(ops), G, S, start)
        assert batched.run(rng) is None, (seed, world)
        one_by_one = Machine(singles(ops), G, S, start)
        assert one_by_one.run(random.Random(seed)) is None, (seed, world)
        assert batched.counters() == one_by_one.counters(), (seed, world)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_rounds_of_batches_and_single_ops_mixed_keep_the_counters(world):
    """Rounds in which each rank issues its ops as one batch or as single launches, at random, on counters that wrap:
    the same counters as every op one by one, and every round completes."""
    for seed in range(10):
        rng = random.Random(seed * 104729 + world)
        G, S = rng.choice([(2, 2), (3, 1)])
        rounds = [op_lists(rng, world, random_pairs(rng, world, G, S, max_msgs=2)) for _ in range(3)]
        mixed = {r: [] for r in range(world)}
        for ops in rounds:
            for r, lst in ops.items():
                launches = batches({r: lst}) if rng.random() < 0.5 else singles({r: lst})
                mixed[r] += launches[r]
        flat = {r: [op for ops in rounds for op in ops[r]] for r in range(world)}
        m = Machine(mixed, G, S, WRAP)
        assert m.run(rng) is None, (seed, world)
        ref = Machine(singles(flat), G, S, WRAP)
        assert ref.run(random.Random(seed)) is None
        assert m.counters() == ref.counters(), (seed, world)


# ---------------------------------------------------------------------------------------------------------- adversarial orders
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_sends_before_receives_beyond_the_mailbox_complete(world):
    """Every rank lists its sends to both neighbours before its receives, each message larger than a pair's G x S slots."""
    G, S = 2, 2
    for seed in range(15):
        rng = random.Random(seed + 31 * world)
        n = rng.randint(G * S + 1, 4 * G * S)
        pairs = {(r, (r + 1) % world): [n, 1] for r in range(world)}
        pairs.update({(r, (r - 1) % world): pairs.get((r, (r - 1) % world), []) + [n + 1] for r in range(world)})
        m = Machine(batches(op_lists(rng, world, pairs, "sends_first")), G, S, rng.choice([0, WRAP]))
        assert m.run(rng) is None, seed


def test_both_directions_with_one_peer_and_several_ops_per_lane_complete():
    G, S = 2, 2
    for seed in range(40):
        rng = random.Random(seed)
        pairs = {(0, 1): [rng.randint(0, 3 * G * S) for _ in range(4)], (1, 0): [rng.randint(0, 3 * G * S) for _ in range(4)]}
        m = Machine(batches(op_lists(rng, 2, pairs, rng.choice(["sends_first", "shuffle"]))), G, S, WRAP)
        assert m.run(rng) is None, seed


# ---------------------------------------------------------------------------------------------------------- negative control
def _split(ops):
    """The planted bug: each rank's batch cut into its sends, then its receives, as two launches on one stream."""
    out = {}
    for r, lst in ops.items():
        sends, recvs = [op for op in lst if op[0]], [op for op in lst if not op[0]]
        out[r] = [(frozenset(["stream"]), part) for part in (sends, recvs) if part]
    return out


def test_a_batch_split_into_two_launches_on_one_stream_deadlocks():
    """rank 0: [send to 1 | receive from 1], rank 1 the mirror, each message larger than a pair's slots: as two launches on
    one stream both sends fill the slots and wait for receives queued behind them.  As one batch it completes, and so does
    the split when the messages fit the slots (the deadlock is the slots running out, not the model)."""
    G, S = 2, 2
    for n in (G * S + 1, 3 * G * S):
        ops = op_lists(random.Random(0), 2, {(0, 1): [n], (1, 0): [n]}, "sends_first")
        bad = Machine(_split(ops), G, S).run(random.Random(1))
        assert bad is not None and bad.startswith("deadlock"), bad
        assert Machine(batches(ops), G, S).run(random.Random(1)) is None
    ops = op_lists(random.Random(0), 2, {(0, 1): [G * S], (1, 0): [G * S]}, "sends_first")
    assert Machine(_split(ops), G, S).run(random.Random(1)) is None


def test_a_lane_that_ignores_list_order_is_caught():
    """Negative control for the read check: a receiving lane that takes its ops in reverse order reads the wrong pieces."""
    G, S = 2, 2
    ops = op_lists(random.Random(0), 2, {(0, 1): [3, 1]}, "sends_first")
    ops[1] = ops[1][::-1]
    bad = Machine(batches(ops), G, S).run(random.Random(2))
    assert bad is not None and "read" in bad, bad
