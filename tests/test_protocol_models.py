"""Model checks of the two cross-GPU synchronisation protocols: the push ("flag-in-data") gradient exchange of csrc/sgd.cu
(`allreduce_sgd_push_kernel`, first part) and the one-slot flag barrier of csrc/common.cuh (second part).

The kernel's safety argument (SURVEY §7.4 hard part #1: no reset races across back-to-back steps) is: lines carry
epoch = step + 1, inboxes are double-buffered by step parity, and a peer can only overwrite parity p two steps later --
which needs my push of the step in between, which I issue only after I finished reading parity p.  Here that argument is
checked mechanically on an abstract machine: every store of an 8-byte half line and every poll is one atomic action,
ranks interleave arbitrarily (exhaustively for the small configuration, randomly for larger ones), 16-byte lines may
tear between their halves, and a reader accepts a line only when both halves carry the expected epoch -- exactly the
kernel's rule.  Checked: every value a rank consumes is the sender's value of THAT step, nobody deadlocks.
The same machine with a single-buffered inbox is shown to fail, so the model can see the bug the parity prevents.
"""
import random

import pytest


class Rank:
    def __init__(self, r, world, steps):
        self.r, self.world, self.steps = r, world, steps
        self.step = 0
        self.todo = []           # pending atomic actions of the current step
        self.reading = None      # index of the source being polled
        self.begin_step()

    def begin_step(self):
        s, w, r = self.step, self.world, self.r
        # push: two half-line stores per peer (a 16-byte line = two independently visible 8-byte halves)
        self.todo = [("store", (r + i) % w, half) for i in range(1, w) for half in (0, 1)]
        self.polls = [q for q in range(w) if q != r]      # fixed rank order, own contribution comes from registers

    def done(self):
        return self.step >= self.steps


def value(rank, step, half):
    return (rank, step, half)


def run(world, steps, choose, double_buffered=True, max_ticks=100000):
    """Runs the abstract machine under scheduler `choose(list_of_runnable_ranks) -> rank`.  Returns None when every rank
    finished all steps with correct data, else a string describing the violation."""
    nbuf = 2 if double_buffered else 1
    # inbox[dst][parity][src][half] = (value, epoch); epoch 0 = freshly zeroed
    inbox = [[[[(None, 0), (None, 0)] for _ in range(world)] for _ in range(nbuf)] for _ in range(world)]
    ranks = [Rank(r, world, steps) for r in range(world)]
    for _ in range(max_ticks):
        runnable = []
        for k in ranks:
            if k.done():
                continue
            if k.todo:
                runnable.append(k)
            else:                                    # polling: runnable only when the awaited line is complete
                q = k.polls[0]
                line = inbox[k.r][k.step % nbuf][q]
                if line[0][1] == k.step + 1 and line[1][1] == k.step + 1:
                    runnable.append(k)
        if all(k.done() for k in ranks):
            return None
        if not runnable:
            return "deadlock at steps %s" % [k.step for k in ranks]
        k = choose(runnable)
        if k.todo:
            _, dst, half = k.todo.pop(0)
            inbox[dst][k.step % nbuf][k.r][half] = (value(k.r, k.step, half), k.step + 1)
        else:
            q = k.polls.pop(0)
            line = inbox[k.r][k.step % nbuf][q]
            for half in (0, 1):
                if line[half][0] != value(q, k.step, half):
                    return f"rank {k.r} consumed {line[half][0]} for (rank {q}, step {k.step}, half {half})"
            if not k.polls:                          # all sources summed: SGD update, next step
                k.step += 1
                if not k.done():
                    k.begin_step()
    return "did not terminate"


def exhaustive(world, steps, double_buffered=True, limit=400000):
    """DFS over every interleaving (scheduler choice sequences), with replay."""
    stack, explored = [[]], 0
    while stack:
        prefix = stack.pop()
        trace = []

        def choose(runnable, prefix=prefix, trace=trace):
            i = len(trace)
            c = prefix[i] if i < len(prefix) else 0
            trace.append((c, len(runnable)))
            return runnable[c]

        bad = run(world, steps, choose, double_buffered)
        explored += 1
        if bad:
            return bad, explored
        if explored > limit:
            pytest.skip("state space larger than the exploration limit")
        # branch: for every choice point beyond the prefix, schedule the alternatives
        for i in range(len(prefix), len(trace)):
            for alt in range(1, trace[i][1]):
                stack.append([c for c, _ in trace[:i]] + [alt])
    return None, explored


def test_two_ranks_two_steps_every_interleaving_is_safe():
    bad, n = exhaustive(world=2, steps=2)
    assert bad is None, bad
    assert n > 100                                   # the search really branched


@pytest.mark.parametrize("world,steps", [(2, 6), (3, 5), (4, 4), (8, 3)])
def test_random_interleavings_are_safe(world, steps):
    for seed in range(300):
        rng = random.Random(seed * 7919 + world)
        # skewed schedulers (one rank much faster / slower than the others) are the interesting ones
        weights = [rng.choice([1, 1, 5, 25]) for _ in range(world)]
        bad = run(world, steps, lambda rs: rng.choices(rs, weights=[weights[k.r] for k in rs])[0])
        assert bad is None, (seed, bad)


def test_single_buffered_inbox_is_caught_by_the_model():
    """Without the parity double-buffer a fast rank overwrites a line its peer has not consumed: the peer then waits for
    an epoch that is gone (deadlock) -- the model must find such a schedule."""
    found = None
    for seed in range(400):
        rng = random.Random(seed)
        weights = [25, 1, 1]
        found = run(3, 4, lambda rs: rng.choices(rs, weights=[weights[k.r] for k in rs])[0], double_buffered=False)
        if found:
            break
    assert found is not None and ("deadlock" in found or "consumed" in found)


# ---------------------------------------------------------------------------------------------------------------------
# The flag barrier of csrc/common.cuh (`block_barrier_all_ranks`): ONE slot per (block, source rank), monotonically
# growing epochs, ">= epoch" wait.  Claim: one slot suffices because a peer can be at most one barrier ahead, and a rank
# that passes barrier k knows every peer has ARRIVED at barrier k (so its writes before the barrier are visible).
def run_barrier(world, rounds, choose, compare=lambda have, want: have >= want):
    flags = [[0] * world for _ in range(world)]          # flags[dst][src]
    arrived = [0] * world                                # highest barrier each rank has entered
    epoch = [0] * world
    todo = [[] for _ in range(world)]                    # pending stores of the barrier being executed
    passed = [0] * world
    for _ in range(200000):
        if all(p == rounds for p in passed):
            return None
        runnable = []
        for r in range(world):
            if passed[r] == rounds:
                continue
            if epoch[r] == passed[r]:                    # not inside a barrier: enter the next one
                runnable.append(r)
            elif todo[r]:
                runnable.append(r)
            elif all(compare(flags[r][q], epoch[r]) for q in range(world)):
                runnable.append(r)
        if not runnable:
            return "deadlock: passed=%s" % passed
        r = choose(runnable)
        if epoch[r] == passed[r]:
            epoch[r] += 1
            arrived[r] = epoch[r]
            todo[r] = list(range(world))                 # signal every peer (and itself)
        elif todo[r]:
            flags[todo[r].pop(0)][r] = epoch[r]
        else:
            k = epoch[r]
            if any(arrived[q] < k for q in range(world)):
                return f"rank {r} passed barrier {k} before everybody arrived: {arrived}"
            passed[r] = k
    return "did not terminate"


@pytest.mark.parametrize("world,rounds", [(2, 6), (3, 5), (8, 4)])
def test_flag_barrier_with_one_slot_per_source_is_safe(world, rounds):
    for seed in range(300):
        rng = random.Random(seed * 104729 + world)
        weights = [rng.choice([1, 1, 5, 25]) for _ in range(world)]
        bad = run_barrier(world, rounds, lambda rs: rng.choices(rs, weights=[weights[r] for r in rs])[0])
        assert bad is None, (seed, bad)


def test_flag_barrier_needs_the_monotonic_compare():
    """With an equality wait a fast peer that is already one barrier ahead overwrites the slot and the slow rank never
    sees 'its' epoch: the model must find the hang.  (The kernel waits for `>= epoch`, wrap-safe.)"""
    found = None
    for seed in range(400):
        rng = random.Random(seed)
        weights = [25, 1, 1]
        found = run_barrier(3, 5, lambda rs: rng.choices(rs, weights=[weights[r] for r in rs])[0], compare=lambda have, want: have == want)
        if found:
            break
    assert found is not None and "deadlock" in found


# ---------------------------------------------------------------------------------------------------------------------
# The generic LL all-reduce of csrc/allreduce.cu (`allreduce_ll_kernel`) shares its per-block call counter (the signal pad's
# epoch word) with the barrier-based variants, and consecutive calls may have different sizes and caps: a call only advances
# the epochs of the blocks it launches, and only exchanges the vectors below its n_vec.  Claim (kernel comment): sender and
# receiver of a line always agree on epoch and parity, and a line is never overwritten before its reader consumed it --
# for ANY call sequence mixing LL calls of different sizes and per-call caps (max_blocks) with barrier-type calls (one-shot /
# two-shot / NVLS / barrier kernel advance a block's epoch by 1..3 and are full cross-rank barriers for that block).
def launcher_ll_grid(n_vec, cap, vpb):
    """Grid of an LL call as b2_allreduce_launch sizes it: by the message alone, whatever the per-call cap."""
    return (n_vec + vpb - 1) // vpb


def capped_ll_grid(n_vec, cap, vpb):
    """A grid that follows the per-call cap (the launcher before it ignored the cap for LL): the negative control."""
    return min((n_vec + vpb - 1) // vpb, cap)


class LLRank:
    """One rank executing a fixed call list in stream order: call k+1 starts after every thread of call k finished.  Inside a
    call every vector (LL) / every block (barrier-type call) is its own thread of control: the GPU runs them concurrently,
    so the scheduler may interleave them freely."""

    def __init__(self, r, world, calls, nblocks, vec_per_block, ll_grid=launcher_ll_grid):
        self.r, self.world, self.calls = r, world, calls
        self.epoch = [0] * nblocks                      # per-block epoch word in this rank's signal pad
        self.vpb = vec_per_block
        self.ll_grid = ll_grid
        self.k = -1
        self.threads = {}                               # thread id -> pending atomic actions
        self.bumps = []
        self.next_call()

    def next_call(self):
        for b, ep in self.bumps:                        # barrier_epoch_store of the finished call
            self.epoch[b] = ep
        self.k += 1
        self.threads, self.bumps = {}, []
        if self.k >= len(self.calls):
            return
        kind, blocks, arg = self.calls[self.k]
        if kind == "ll":                                # blocks = the call's cap, arg = n_vec: vectors v < n_vec, grid-stride,
            grid = self.ll_grid(arg, blocks, self.vpb)  # so vector v lives in block (v // vpb) % grid
            for b in range(grid):
                vs = [v for v in range(arg) if (v // self.vpb) % grid == b]
                if not vs:
                    continue
                ep = self.epoch[b] + 1
                for v in vs:                            # per vector: store both half lines to every peer, then poll every peer
                    acts = [("store", b, v, (self.r + i) % self.world, half, ep) for i in range(1, self.world) for half in (0, 1)]
                    acts += [("poll", b, v, q, ep) for q in range(self.world) if q != self.r]
                    self.threads[("v", v)] = acts
                self.bumps.append((b, ep))
        else:                                           # barrier-type call: arg = number of barrier rounds (1..3)
            for b in range(blocks):
                acts = []
                for i in range(arg):
                    acts += [("arrive", b, self.epoch[b] + 1 + i), ("wait", b, self.epoch[b] + 1 + i)]
                self.threads[("b", b)] = acts
                self.bumps.append((b, self.epoch[b] + arg))

    def done(self):
        return self.k >= len(self.calls)


def run_ll(world, calls, nblocks, vpb, choose, max_ticks=400000, double_buffered=True, ll_grid=launcher_ll_grid):
    cap = nblocks * vpb
    par = (lambda ep: ep & 1) if double_buffered else (lambda ep: 0)
    # inbox[dst][parity][src][v][half] = (payload, flag); flags[dst][block][src] = barrier epochs
    inbox = [[[[[(None, 0), (None, 0)] for _ in range(cap)] for _ in range(world)] for _ in range(2)] for _ in range(world)]
    flags = [[[0] * world for _ in range(nblocks)] for _ in range(world)]
    ranks = [LLRank(r, world, calls, nblocks, vpb, ll_grid) for r in range(world)]
    for _ in range(max_ticks):
        for k in ranks:
            while not k.done() and not k.threads:       # call finished (or launched nothing): stream order -> next call
                k.next_call()
        if all(k.done() for k in ranks):
            return None
        runnable = []
        for k in ranks:
            for tid, acts in k.threads.items():
                a = acts[0]
                if a[0] == "poll":
                    _, b, v, q, ep = a
                    line = inbox[k.r][par(ep)][q][v]
                    ok = line[0][1] == ep and line[1][1] == ep
                elif a[0] == "wait":
                    _, b, ep = a
                    ok = all(flags[k.r][b][q] >= ep for q in range(world) if q != k.r)
                else:
                    ok = True
                if ok:
                    runnable.append((k, tid))
        if not runnable:
            return "deadlock at calls %s" % [k.k for k in ranks]
        k, tid = choose(runnable)
        a = k.threads[tid].pop(0)
        if not k.threads[tid]:
            del k.threads[tid]
        if a[0] == "store":
            _, b, v, dst, half, ep = a
            inbox[dst][par(ep)][k.r][v][half] = ((k.r, k.k, v, half), ep)
        elif a[0] == "poll":
            _, b, v, q, ep = a
            line = inbox[k.r][par(ep)][q][v]
            for half in (0, 1):
                if line[half][0] != (q, k.k, v, half):
                    return f"rank {k.r} call {k.k} consumed {line[half][0]} for (rank {q}, vector {v}, half {half})"
        elif a[0] == "arrive":
            _, b, ep = a
            for q in range(world):
                if q != k.r:
                    flags[q][b][k.r] = ep
    return "did not terminate"


def _random_calls(rng, nblocks, vpb, n):
    calls = []
    for _ in range(n):
        if rng.random() < 0.65:
            n_vec = rng.randint(1, nblocks * vpb)
            calls.append(("ll", rng.randint(1, nblocks), n_vec))        # per-call cap (max_blocks), n_vec
        else:
            calls.append(("bar", rng.randint(1, nblocks), rng.randint(1, 3)))
    return calls


@pytest.mark.parametrize("world", [2, 3, 4])
def test_ll_allreduce_mixed_sizes_and_variants_are_safe(world):
    nblocks, vpb = 3, 2
    for seed in range(120):
        rng = random.Random(seed * 104729 + world)
        calls = _random_calls(rng, nblocks, vpb, 7)
        weights = [rng.choice([1, 1, 5, 25]) for _ in range(world)]
        bad = run_ll(world, calls, nblocks, vpb, lambda rs: rng.choices(rs, weights=[weights[k.r] for k, _ in rs])[0])
        assert bad is None, (seed, calls, bad)


def test_ll_model_catches_a_single_buffered_inbox():
    """Negative control: without the parity double-buffer a fast rank's next call overwrites a line its peer is still polling
    for (the peer then waits for an epoch that is gone) -- the model must find such a schedule."""
    calls = [("ll", 2, 4)] * 4
    found = None
    for seed in range(300):
        rng = random.Random(seed)
        weights = [25, 1]
        found = run_ll(2, calls, 2, 2, lambda rs: rng.choices(rs, weights=[weights[k.r] for k, _ in rs])[0], double_buffered=False)
        if found:
            break
    assert found is not None and ("consumed" in found or "deadlock" in found), found


# The three calls of a cap that changes on one inbox (n_vec, cap), scaled to 2 vectors per block: the first gives blocks 0 and 1
# epoch 1; if the second call's grid followed its cap of 1, block 0 would take vector 2 at epoch 2, parity 0; in the third,
# block 1 would take vector 2 at ITS epoch 2, parity 0, and find the second call's line already carrying flag 2.
MIXED_CAP_CALLS = [("ll", 2, 4), ("ll", 1, 3), ("ll", 2, 3)]


def _first_runnable(rs):
    return rs[0]                                        # rank 0 runs whenever it can: it reaches the third call first


def test_ll_allreduce_with_a_cap_that_changes_between_calls_is_safe():
    assert run_ll(2, MIXED_CAP_CALLS, 2, 2, _first_runnable) is None
    for seed in range(200):
        rng = random.Random(seed)
        weights = [rng.choice([1, 5, 25]) for _ in range(3)]
        bad = run_ll(3, MIXED_CAP_CALLS, 2, 2, lambda rs: rng.choices(rs, weights=[weights[k.r] for k, _ in rs])[0])
        assert bad is None, (seed, bad)


def test_ll_model_catches_a_grid_that_follows_the_cap():
    """Negative control: with the grid capped per call, the third call accepts the second call's line for vector 2."""
    bad = run_ll(2, MIXED_CAP_CALLS, 2, 2, _first_runnable, ll_grid=capped_ll_grid)
    assert bad is not None and "call 2 consumed (1, 1, 2, 0)" in bad, bad
