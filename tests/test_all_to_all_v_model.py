"""CPU tier of the all-to-all with variable segments: the model of tests/all_to_all_v_model.py against plain slicing and
against gloo's ``all_to_all_single`` with split sizes, the planted faults it catches, ``SymmWorld.all_to_all_v_``'s argument
checks (each raises before any launch), the routing of ``comm.all_to_all_single`` / ``comm.all_to_all``, and the export."""
import pytest
import torch

import all_to_all_v_model as AM
import all_to_all_v_workers as AW

CHUNK = 128 << 10                                # the kernel's bytes per pair and round (checked on the GPU tier)


def _case(world, seed, dtype=torch.int32, tail=(3,), most=9, hot=False):
    S = AW.split_matrix(world, seed, hot, most)
    xs = [AW.rows_of(S, s, dtype, tail, seed) for s in range(world)]
    outs = [torch.zeros((sum(S[p][r] for p in range(world)),) + tail, dtype=dtype) for r in range(world)]
    return S, xs, outs


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_model_equals_plain_slicing(world):
    for k, (dtype, tail) in enumerate([(torch.int32, (3,)), (torch.uint8, ()), (torch.float64, (2, 2)),
                                       (torch.bool, (5,))]):
        S, xs, outs = _case(world, 10 * world + k, dtype, tail, hot=k % 2 == 1)
        got = AM.single_form(xs, S, outs, [[S[p][r] for p in range(world)] for r in range(world)])
        want = AM.by_slicing(xs, S)
        for r in range(world):
            assert torch.equal(got[r], want[r]), (world, dtype, r)


def _sends_and_buffers(world, lens, expect, seed, gap=16):
    """Random sends of lens[s][d] bytes; output buffers of random bytes with segments of expect[r][p] bytes, each behind
    ``gap`` sentinel bytes."""
    g = torch.Generator().manual_seed(seed)
    sends = [[torch.randint(0, 256, (lens[s][d],), generator=g, dtype=torch.uint8) for d in range(world)]
             for s in range(world)]
    offs, bufs = [], []
    for r in range(world):
        o, at = [], gap
        for p in range(world):
            o.append(at)
            at += expect[r][p] + gap
        offs.append(o)
        bufs.append(torch.randint(0, 256, (at,), generator=g, dtype=torch.uint8))
    return sends, bufs, offs


def test_model_truncates_mismatched_splits_and_leaves_the_rest():
    world = 3
    lens = [[5, 17, 0], [16, 1, 40], [33, 0, 15]]
    expect = [[9, 16, 20], [17, 0, 0], [0, 40, 15]]           # more, fewer, equal, and zero against non-zero
    sends, bufs, offs = _sends_and_buffers(world, lens, expect, 1)
    got = AM.predict(sends, bufs, offs, expect)
    for r in range(world):
        for p in range(world):
            m = min(lens[p][r], expect[r][p])
            at = offs[r][p]
            assert torch.equal(got[r][at:at + m], sends[p][r][:m])
            assert torch.equal(got[r][at + m:at + expect[r][p]], bufs[r][at + m:at + expect[r][p]])
        mask = torch.ones(bufs[r].numel(), dtype=torch.bool)
        for p in range(world):
            mask[offs[r][p]:offs[r][p] + expect[r][p]] = False
        assert torch.equal(got[r][mask], bufs[r][mask])


def test_round_count():
    assert AM.rounds([[0, 0], [0, 0]], CHUNK) == 1                # an all-empty call still runs one round
    assert AM.rounds([[1, 0], [0, 0]], CHUNK) == 1
    assert AM.rounds([[CHUNK, 0], [0, 0]], CHUNK) == 1
    assert AM.rounds([[0, 0], [CHUNK + 1, 0]], CHUNK) == 2
    assert AM.rounds([[0, 3 * CHUNK + 1], [0, 0]], CHUNK) == 4
    assert AM.barriers([[0]], CHUNK) == 2


@pytest.mark.parametrize("fault", ["sent", "expected", "swap", "tail"])
def test_the_checker_catches_planted_faults(fault):
    world = 4
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(0, 60, (world, world), generator=g).tolist()
    expect = [[lens[p][r] + (7 if (r + p) % 3 == 0 else -3 if lens[p][r] >= 3 and (r + p) % 3 == 1 else 0)
               for p in range(world)] for r in range(world)]
    sends, bufs, offs = _sends_and_buffers(world, lens, expect, 6)
    good = AM.predict(sends, bufs, offs, expect)
    bad = AM.predict(sends, bufs, offs, expect, fault)
    assert any(not torch.equal(a, b) for a, b in zip(good, bad)), fault


# ---------------------------------------------------------------------------------------------------------- gloo
@pytest.mark.timeout(240)
@pytest.mark.parametrize("world", [2, 3])
def test_model_equals_gloo_all_to_all_single_with_splits(world):
    import dist_tuto.pth_b200 as b2
    b2.launch(AW.w_gloo, size=world, backend="gloo", join_timeout_s=200)


# ---------------------------------------------------------------------------------------------------------- arguments
class _Kernels:
    """Stands in for the extension: records launches."""

    def __init__(self):
        self.calls = []

    def alltoallv_config(self):
        return CHUNK, 64

    def alltoallv(self, *a):
        self.calls.append(a)


def _meta_world(world, rank=1):
    """A SymmWorld whose tensors are "meta" tensors (standing in for CUDA ones) and whose kernels are recorded."""
    from dist_tuto.pth_b200.parallel import symm
    w = object.__new__(symm.SymmWorld)
    w.C, w.world, w.rank, w.ranks, w.max_blocks = _Kernels(), world, rank, list(range(world)), 16
    w.supports_raw = lambda t: t.device.type == "meta" and t.is_contiguous()
    hd = symm.SymmHandle(w, 1 << 30, 1 << 30, [0x10000 * (r + 1) for r in range(world)], 0, [], 0, "vmm")
    w._staging = {torch.float32: hd}
    return w


def _m(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_all_to_all_v_launches_the_byte_counts_of_the_splits():
    w = _meta_world(3)
    w.all_to_all_v_(_m(6, 4), _m(9, 4), [1, 2, 3], [4, 0, 5])
    (ptrs, sigs, srcs, sbytes, dsts, dbytes, rank, world, mb), = w.C.calls
    assert sbytes == [64, 0, 80] and dbytes == [16, 32, 48] and (rank, world, mb) == (1, 3, 16)
    w.all_to_all_v_(_m(6, dtype=torch.int16), _m(3, dtype=torch.int16))            # None: equal splits
    assert w.C.calls[-1][3] == [2, 2, 2] and w.C.calls[-1][5] == [4, 4, 4]
    w.all_to_all_v_([_m(2), _m(0), _m(7)], [_m(5), _m(1), _m(0)])
    assert w.C.calls[-1][3] == [20, 4, 0] and w.C.calls[-1][5] == [8, 0, 28]
    w.all_to_all_v_(_m(0, 3), _m(0, 3), [0, 0, 0], [0, 0, 0])                      # an empty rank still launches
    assert w.C.calls[-1][3] == [0, 0, 0] and len(w.C.calls) == 4


def test_every_bad_argument_raises_before_any_launch():
    """Each raises on the rank that passed it, with nothing launched; its peers would wait in the kernel until the spin
    limit reports them."""
    w = _meta_world(3)
    cases = [
        (lambda: w.all_to_all_v_(_m(6), _m(6), [1, 2], None), ValueError, "needs 3 entries"),
        (lambda: w.all_to_all_v_(_m(6), _m(6), None, [1, 2, 3, 0]), ValueError, "needs 3 entries"),
        (lambda: w.all_to_all_v_(_m(6), _m(6), [3, 4, -1], None), ValueError, "negative"),
        (lambda: w.all_to_all_v_(_m(6), _m(6), None, [1, 1, 1]), ValueError, "sums to 3"),
        (lambda: w.all_to_all_v_(_m(7), _m(6)), ValueError, "do not split equally"),
        (lambda: w.all_to_all_v_(_m(6), _m(6, dtype=torch.int32), [2, 2, 2], [2, 2, 2]), ValueError, "one dtype"),
        (lambda: w.all_to_all_v_(_m(6), torch.zeros(6), [2, 2, 2], [2, 2, 2]), TypeError, "contiguous CUDA"),
        (lambda: w.all_to_all_v_(_m(6, 2).t(), _m(2, 6), [2, 0, 0], [2, 0, 0]), TypeError, "contiguous CUDA"),
        (lambda: w.all_to_all_v_(_m(), _m(), [0, 0, 0], [0, 0, 0]), ValueError, "at least one dimension"),
        (lambda: w.all_to_all_v_([_m(1)] * 2, [_m(1)] * 3), ValueError, "needs 3 output tensors"),
        (lambda: w.all_to_all_v_([_m(1)] * 3, [_m(1)] * 4), ValueError, "needs 3 input tensors"),
        (lambda: w.all_to_all_v_([_m(1)] * 3, [_m(1), _m(1, dtype=torch.half), _m(1)]), ValueError, "one dtype"),
        (lambda: w.all_to_all_v_([_m(1)] * 3, [_m(1), torch.zeros(1), _m(1)]), TypeError, "contiguous CUDA"),
        (lambda: w.all_to_all_v_([_m(1)] * 3, _m(3)), TypeError, "two lists"),
        (lambda: w.all_to_all_v_([_m(1)] * 3, [_m(1)] * 3, [1, 1, 1]), ValueError, "single-tensor form"),
    ]
    for k, (call, exc, match) in enumerate(cases):
        with pytest.raises(exc, match=match):
            call()
        assert w.C.calls == [], k


def test_an_output_overlapping_the_input_reads_a_copy():
    w = _meta_world(2, rank=0)
    x = _m(8)
    w.all_to_all_v_(x, x, [3, 5], [4, 4])               # meta tensors all sit at address 0: every pair overlaps
    assert all(s._base is not x for s in w.C.calls[-1][2])                  # (the GPU tier checks the bytes)


# ---------------------------------------------------------------------------------------------------------- routing
class _StandIn:
    def __init__(self, world, v=True):
        self.world, self.calls = world, []
        self.all_to_all_ = lambda out, inp: self.calls.append("all_to_all_")
        if v:
            self.all_to_all_v_ = lambda out, inp, *splits: self.calls.append("all_to_all_v_")

    def supports_raw(self, t):
        return t.device.type == "meta"


def _route(monkeypatch, v, call):
    from dist_tuto.pth_b200 import comm
    w = _StandIn(4, v)
    torch_calls = []
    monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: w if tensor.device.type == "meta" else None)
    for name in ("all_to_all_single", "all_to_all"):
        monkeypatch.setattr(comm.dist, name, lambda *a, _n=name, **k: torch_calls.append(_n))
    call(comm)
    return w.calls + torch_calls


def test_comm_routes_split_sizes_and_the_list_form(monkeypatch):
    """With either split list, or the list form, a blocking call of device tensors reaches ``all_to_all_v_`` on a world
    that has it; both lists None keeps the equal-segment kernel; a world with only ``all_to_all_``, ``async_op=True`` and
    CPU tensors reach torch.distributed."""
    dev = lambda n, dtype=torch.float32: torch.empty(n, dtype=dtype, device="meta")  # noqa: E731
    cpu = lambda n: torch.zeros(n)  # noqa: E731
    # (call, route on a world with all_to_all_v_, route on one with all_to_all_ only)
    cases = [
        (lambda c: c.all_to_all_single(dev(16), dev(16)), "all_to_all_", "all_to_all_"),
        (lambda c: c.all_to_all_single(dev(16), dev(16), [4] * 4, [4] * 4), "all_to_all_v_", "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(10), dev(16), [1, 2, 3, 4], None), "all_to_all_v_", "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(16), dev(10), None, [1, 2, 3, 4]), "all_to_all_v_", "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(16), dev(16), [4] * 4, [4] * 4, async_op=True), "all_to_all_single",
         "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(16), dev(16), async_op=True), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_to_all_single(cpu(16), cpu(16), [4] * 4, [4] * 4), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(16), cpu(16), [4] * 4, [4] * 4), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_to_all([dev(2)] * 4, [dev(3)] * 4), "all_to_all_v_", "all_to_all"),
        (lambda c: c.all_to_all([dev(2)] * 3, [dev(3)] * 4), "all_to_all_v_", "all_to_all"),   # raises in the method
        (lambda c: c.all_to_all([dev(2)] * 4, [dev(3)] * 4, async_op=True), "all_to_all", "all_to_all"),
        (lambda c: c.all_to_all([cpu(2)] * 4, [cpu(3)] * 4), "all_to_all", "all_to_all"),
        (lambda c: c.all_to_all([dev(2)] * 4, [dev(3)] * 3 + [cpu(3)]), "all_to_all", "all_to_all"),
    ]
    for k, (call, with_v, without_v) in enumerate(cases):
        assert _route(monkeypatch, True, call) == [with_v], k
        assert _route(monkeypatch, False, call) == [without_v], k


def test_all_to_all_is_exported_from_the_package_root():
    import dist_tuto.pth_b200 as b2
    from dist_tuto.pth_b200 import comm
    assert b2.all_to_all is comm.all_to_all and "all_to_all" in comm.__all__
