"""``comm.batch_isend_irecv`` without a GPU: which ops reach ``SymmWorld.batch_p2p_`` and which ``dist.batch_isend_irecv``,
what both refuse before anything is issued, what the ``p2p_batch`` binding and ``b2_p2p_batch_launch`` refuse before any
launch, and one real gloo ring at worlds 2 and 3."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200 import comm


# ---------------------------------------------------------------------------------------------------------- routing
class _Work:
    def __init__(self, tag):
        self.tag = tag

    def wait(self):
        return True

    def is_completed(self):
        return True


class _StandInWorld:
    """A symmetric world as comm.py sees it: takes every tensor, has the point-to-point methods (the two-level world,
    ``with_methods=False``, has none) and records the batches it was asked to run."""

    def __init__(self, with_methods=True, with_batch=True):
        self.batches = []
        if with_methods:
            self.send_ = self.recv_ = self.isend_ = self.irecv_ = lambda t, peer: None
        if with_methods and with_batch:
            self.batch_p2p_ = self._batch

    def _batch(self, ops):
        self.batches.append([(send, t, peer) for send, t, peer in ops])
        return [_Work(("mine", k)) for k in range(len(ops))]

    def supports_raw(self, t):
        return True


class _TorchP2POp(dist.P2POp):
    """torch's P2POp without a process group: its constructor resolves the group and the peer's group rank, which needs
    one (the real class is driven by the gloo ring below)."""

    def __init__(self, op, tensor, peer=None, group=None, tag=0):
        self.op, self.tensor, self.peer, self.group, self.tag = op, tensor, peer, group, tag


@pytest.fixture
def routed(monkeypatch):
    """(patch(world, cuda_only), torch_batches): ``comm._symm_world_for`` returns ``world`` (for every tensor, or only for
    ``cuda_only`` tensors tagged by the test); torch.distributed's batch_isend_irecv is recorded."""
    batches = []

    def fake_batch(ops):
        batches.append(list(ops))
        return [_Work(("torch", k)) for k in range(len(ops))]
    monkeypatch.setattr(comm.dist, "batch_isend_irecv", fake_batch)
    monkeypatch.setattr(comm.dist, "P2POp", _TorchP2POp)

    def patch(world, only=None):
        monkeypatch.setattr(comm, "_symm_world_for",
                            lambda tensor, group: world if only is None or any(tensor is t for t in only) else None)
    return patch, batches


def _t(n=5, dtype=torch.float32):
    return torch.zeros(n, dtype=dtype)


def test_every_op_with_a_peer_reaches_one_batch_of_the_symmetric_world(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    xs = [_t(), _t(3, torch.int16), _t(0), _t(7, torch.bool)]
    ops = [comm.P2POp(comm.isend, xs[0], 1), comm.P2POp(comm.irecv, xs[1], 2, tag=7),
           comm.P2POp(dist.isend, xs[2], 3), comm.P2POp(dist.irecv, xs[3], 1, group=0)]
    reqs = comm.batch_isend_irecv(ops)
    assert len(w.batches) == 1 and nccl == []
    assert [(s, p) for s, _, p in w.batches[0]] == [(True, 1), (False, 2), (True, 3), (False, 1)]
    assert all(a is b for (_, a, _), b in zip(w.batches[0], xs))
    assert [r._work.tag for r in reqs] == [("mine", k) for k in range(4)]
    assert all(isinstance(r, comm.Request) and r.is_completed() and r.wait() for r in reqs)
    assert b2.batch_isend_irecv is comm.batch_isend_irecv and b2.P2POp is comm.P2POp


def test_torch_p2pop_elements_are_accepted(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    x, y = _t(), _t()
    reqs = comm.batch_isend_irecv([dist.P2POp(dist.isend, x, 1), dist.P2POp(dist.irecv, y, 1)])
    assert [(s, p) for s, _, p in w.batches[0]] == [(True, 1), (False, 1)] and nccl == []
    assert len(reqs) == 2


def test_cpu_tensors_and_any_source_go_to_one_torch_batch_in_list_order(routed):
    """CUDA-routed ops go to the world, the others (CPU tensors here) to one dist.batch_isend_irecv; the Requests come back
    in the order of the list."""
    patch, nccl = routed
    w = _StandInWorld()
    gpu = [_t(), _t()]
    patch(w, only=gpu)
    cpu = [_t(), _t()]
    theirs = dist.P2POp(dist.irecv, cpu[1], 3, tag=4)
    ops = [comm.P2POp(comm.isend, cpu[0], 2, tag=9), comm.P2POp(comm.isend, gpu[0], 1), theirs,
           comm.P2POp(comm.irecv, gpu[1], 1)]
    reqs = comm.batch_isend_irecv(ops)
    assert [(s, p) for s, _, p in w.batches[0]] == [(True, 1), (False, 1)]
    assert len(nccl) == 1 and len(nccl[0]) == 2
    first = nccl[0][0]
    assert isinstance(first, dist.P2POp) and first.op is dist.isend and first.tensor is cpu[0]
    assert first.peer == 2 and first.tag == 9 and first.group is None
    assert nccl[0][1] is theirs                                # a torch P2POp is passed on as it is
    assert [r._work.tag for r in reqs] == [("torch", 0), ("mine", 0), ("torch", 1), ("mine", 1)]


def test_a_coalesced_torch_batch_gives_every_request_its_work(routed, monkeypatch):
    patch, _ = routed
    patch(None)
    monkeypatch.setattr(comm.dist, "batch_isend_irecv", lambda ops: [_Work("one")])
    reqs = comm.batch_isend_irecv([comm.P2POp(comm.isend, _t(), 1), comm.P2POp(comm.irecv, _t(), 1)])
    assert [r._work.tag for r in reqs] == ["one", "one"]


def test_a_world_without_the_point_to_point_methods_stays_on_torch(routed):
    patch, nccl = routed
    patch(_StandInWorld(with_methods=False))
    comm.batch_isend_irecv([comm.P2POp(comm.isend, _t(), 1), comm.P2POp(comm.irecv, _t(), 1)])
    assert len(nccl) == 1 and len(nccl[0]) == 2


def test_cpu_tensors_never_reach_the_world_lookup(routed, monkeypatch):
    """With a symmetric world registered, CPU tensors still go to torch.distributed (gloo)."""
    _, nccl = routed
    try:
        from dist_tuto.pth_b200.parallel import symm
    except Exception:                                        # extension not importable here: the lookup returns None anyway
        symm = None
    w = _StandInWorld()
    if symm is not None:
        monkeypatch.setattr(symm, "lookup_world", lambda group=None: w)
    comm.batch_isend_irecv([comm.P2POp(comm.isend, _t(), 1), comm.P2POp(comm.irecv, _t(), 1)])
    assert w.batches == [] and len(nccl) == 1


# ---------------------------------------------------------------------------------------------------------- errors
def test_malformed_lists_are_refused_before_anything_is_issued(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    ok = comm.P2POp(comm.isend, _t(), 1)
    for bad in ((ok,), [], ok, [ok, "isend"], [ok, None]):
        with pytest.raises(ValueError):
            comm.batch_isend_irecv(bad)
    with pytest.raises(ValueError, match="same group"):
        comm.batch_isend_irecv([ok, comm.P2POp(comm.irecv, _t(), 1, group=object())])
    with pytest.raises(ValueError, match="contiguous"):
        comm.batch_isend_irecv([ok, comm.P2POp(comm.irecv, torch.zeros(4, 4).t(), 1)])
    with pytest.raises(ValueError, match="cannot send to itself"):
        comm.batch_isend_irecv([comm.P2POp(comm.irecv, _t(), 1), comm.P2POp(comm.isend, _t(), 0)])  # rank 0 here
    with pytest.raises(ValueError, match="isend or irecv"):
        comm.P2POp(comm.send, _t(), 1)
    assert w.batches == [] and nccl == []


def test_group_zero_is_the_default_group(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    comm.batch_isend_irecv([comm.P2POp(comm.isend, _t(), 1, group=0), comm.P2POp(comm.irecv, _t(), 1)])
    assert len(w.batches) == 1


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def _symm_world(world, rank, ranks):
    from dist_tuto.pth_b200.parallel import symm
    w = object.__new__(symm.SymmWorld)
    w.world, w.rank, w.ranks = world, rank, list(ranks)
    w.global_rank = ranks[rank]
    w.device = torch.device("cuda", 0)
    w.p2p, w._p2p_streams = None, {}
    return w


def test_symm_world_batch_refuses_before_touching_a_stream():
    C = _C()
    w = _symm_world(3, 1, [4, 6, 9])
    w.C = C
    t = torch.zeros(8)
    with pytest.raises(ValueError, match="cannot send to itself"):
        w.batch_p2p_([(False, t, 4), (True, t, 6)])
    with pytest.raises(ValueError, match="not in this world"):
        w.batch_p2p_([(True, t, 1)])
    with pytest.raises(TypeError, match="contiguous CUDA tensor"):
        w.batch_p2p_([(True, t, 9)])
    with pytest.raises(ValueError, match="at most 256"):
        w.batch_p2p_([(True, t, 9)] * 257)
    assert w._p2p_streams == {}


# ---------------------------------------------------------------------------------------------------------- bindings
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def test_batch_capacity():
    assert _C().p2p_batch_capacity() == 256


def test_p2p_batch_binding_refuses_bad_worlds_peers_and_lists():
    C = _C()
    b, s = [0x1000 * (i + 1) for i in range(4)], [0x2000 * (i + 1) for i in range(4)]
    t = torch.zeros(8)                                       # CPU: reaching the tensor check means every other check passed
    f = C.p2p_batch
    with pytest.raises(RuntimeError, match="world must be in 1..8"):
        f(b, s, [(True, t, 1)], 0, 9)
    with pytest.raises(RuntimeError, match="at least 2"):
        f(b[:1], s[:1], [(True, t, 0)], 0, 1)
    with pytest.raises(RuntimeError, match="one mailbox and one signal pad per rank"):
        f(b[:3], s, [(True, t, 1)], 0, 4)
    with pytest.raises(RuntimeError, match="at most 256 ops"):
        f(b, s, [(True, t, 1)] * 257, 0, 4)
    with pytest.raises(RuntimeError, match="peer 4 is outside"):
        f(b, s, [(True, t, 1), (False, t, 4)], 0, 4)
    with pytest.raises(RuntimeError, match="cannot be its own peer"):
        f(b, s, [(False, t, 2)], 2, 4)
    with pytest.raises(RuntimeError, match="contiguous CUDA tensor"):
        f(b, s, [(True, t, 1)], 0, 4)
    f(b, s, [], 0, 4)                                        # nothing to launch


def test_p2p_batch_launcher_refuses_without_a_launch():
    """b2_p2p_batch_launch returns cudaErrorInvalidValue (1) before any CUDA call for each of these, and 0 for a batch of
    zero-byte ops, which launches nothing (on a machine without a GPU a launch would return another error)."""
    from dist_tuto.pth_b200.ops import _ext
    _C()
    lib = ctypes.CDLL(_ext.so_path())
    i, p = ctypes.c_int, ctypes.c_void_p
    fn = lib.b2_p2p_batch_launch
    fn.restype = i
    fn.argtypes = [p, p, p, p, p, p, i, i, i, p]
    box = (ctypes.c_void_p * 8)(*[0x100000 * (r + 1) for r in range(4)])
    sig = (ctypes.c_void_p * 8)(*[0x200000 * (r + 1) for r in range(4)])

    def call(send, peer, msg, nbytes, rank=0, world=4, n=None, box_=box):
        n = len(send) if n is None else n
        k = max(len(send), 1)
        return fn(box_, sig, (ctypes.c_int * k)(*send), (ctypes.c_int * k)(*peer), (ctypes.c_void_p * k)(*msg),
                  (ctypes.c_size_t * k)(*nbytes), n, rank, world, None)
    m = 0x300000
    assert call([1], [1], [m], [64], world=1) == 1                    # world 1
    assert call([1], [1], [m], [64], world=9) == 1                    # world 9
    assert call([1], [1], [m], [64], rank=4) == 1                     # rank outside the world
    assert call([1, 0], [1, 4], [m, m], [64, 64]) == 1                # a peer outside the world
    assert call([0], [-1], [m], [64]) == 1
    assert call([1, 0], [2, 0], [m, m], [64, 64]) == 1                # peer == rank
    assert call([2], [1], [m], [64]) == 1                             # unknown direction
    assert call([1, 0], [1, 1], [m, None], [64, 64]) == 1             # no message
    assert call([1], [1], [m + 4], [64]) == 1                         # not 16-byte aligned
    assert call([1], [1], [m], [64], box_=None) == 1                  # no mailbox
    assert call([1], [1], [m], [64], n=257) == 1                      # more ops than the capacity
    assert call([1], [1], [m], [64], n=-1) == 1
    assert call([1, 0, 1], [1, 2, 3], [m, m, m], [0, 0, 0]) == 0      # zero bytes: nothing to launch
    assert call([], [], [], []) == 0                                  # an empty batch: nothing to launch


# ---------------------------------------------------------------------------------------------------------- gloo
@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ring(world):
    import p2p_batch_workers as W
    b2.launch(W.w_gloo_ring, size=world, backend="gloo", join_timeout_s=120)
