"""Point-to-point on the b200 backend without a GPU: which calls ``comm.send`` / ``recv`` / ``isend`` / ``irecv`` hand to a
symmetric world and which stay on ``torch.distributed``, what ``SymmWorld`` refuses before it touches a stream, and what the
``p2p_send`` / ``p2p_recv`` bindings and launchers refuse before any launch."""
import ctypes
import os

import pytest
import torch

from dist_tuto.pth_b200 import comm


# ---------------------------------------------------------------------------------------------------------- routing
class _Work:
    def __init__(self, calls):
        self.calls = calls

    def wait(self):
        self.calls.append("wait")
        return True

    def is_completed(self):
        return True


class _StandInWorld:
    """A symmetric world as comm.py sees it: takes every tensor and records the point-to-point method it was asked to run
    (``with_methods=False`` is the two-level world, which has none)."""

    def __init__(self, with_methods=True):
        self.calls = []
        if with_methods:
            self.send_ = lambda t, dst: self.calls.append(("send_", dst))
            self.recv_ = lambda t, src: self.calls.append(("recv_", src))
            self.isend_ = lambda t, dst: self.calls.append(("isend_", dst)) or _Work(self.calls)
            self.irecv_ = lambda t, src: self.calls.append(("irecv_", src)) or _Work(self.calls)

    def supports_raw(self, t):
        return True


@pytest.fixture
def routed(monkeypatch):
    """(patch(world), calls): ``comm._symm_world_for`` returns ``world``; torch.distributed's p2p calls are recorded."""
    calls = []
    for name in ("send", "recv", "isend", "irecv"):
        monkeypatch.setattr(comm.dist, name, lambda *a, _n=name, **k: calls.append((_n, k.get("src", k.get("dst")))) or 7)

    def patch(world):
        monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: world)
    return patch, calls


def test_send_recv_isend_irecv_reach_the_symmetric_world(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    t = torch.zeros(5, dtype=torch.int16)
    assert comm.send(t, 3) is None
    assert comm.recv(t, 2) == 2                              # the sender's rank, as torch returns it
    req = comm.isend(t, 1, tag=9)                            # tag is ignored on this path
    assert isinstance(req, comm.Request) and req.is_completed()
    assert req.wait() is True
    req = comm.irecv(t, 0, group=None)
    req.wait()
    assert w.calls == [("send_", 3), ("recv_", 2), ("isend_", 1), "wait", ("irecv_", 0), "wait"]
    assert nccl == []


def test_any_source_receive_stays_on_torch(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    t = torch.zeros(5)
    assert comm.recv(t) == 7
    comm.irecv(t, None)
    assert w.calls == [] and nccl == [("recv", None), ("irecv", None)]


def test_a_world_without_send_stays_on_torch(routed):
    """The two-level world of several machines has no point-to-point methods: every call goes to torch.distributed."""
    patch, nccl = routed
    patch(_StandInWorld(with_methods=False))
    t = torch.zeros(5)
    comm.send(t, 1)
    comm.recv(t, 1)
    comm.isend(t, 1)
    comm.irecv(t, 1)
    assert nccl == [("send", 1), ("recv", 1), ("isend", 1), ("irecv", 1)]


def test_cpu_tensors_stay_on_torch(routed, monkeypatch):
    """With a symmetric world registered, a CPU tensor still goes to torch.distributed (gloo): the world lookup is never
    reached for it."""
    _, nccl = routed
    try:
        from dist_tuto.pth_b200.parallel import symm
    except Exception:                                        # extension not importable here: the lookup returns None anyway
        symm = None
    w = _StandInWorld()
    if symm is not None:
        monkeypatch.setattr(symm, "lookup_world", lambda group=None: w)
    t = torch.zeros(5)
    comm.send(t, 1)
    assert comm.recv(t, 1) == 7
    comm.isend(t, 1)
    comm.irecv(t, 1)
    assert w.calls == [] and nccl == [("send", 1), ("recv", 1), ("isend", 1), ("irecv", 1)]


def test_non_contiguous_tensors_are_refused_before_routing(routed):
    patch, nccl = routed
    w = _StandInWorld()
    patch(w)
    t = torch.zeros(4, 4).t()
    for fn in (comm.send, comm.recv, comm.isend, comm.irecv):
        with pytest.raises(ValueError, match="contiguous"):
            fn(t, 1)
    assert w.calls == [] and nccl == []


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def _symm_world(world, rank, ranks):
    from dist_tuto.pth_b200.parallel import symm
    w = object.__new__(symm.SymmWorld)
    w.world, w.rank, w.ranks = world, rank, list(ranks)
    w.global_rank = ranks[rank]
    w.device = torch.device("cuda", 0)
    w.p2p, w._p2p_streams = None, {}
    return w


def test_symm_world_refuses_itself_strangers_and_cpu_tensors():
    pytest.importorskip("dist_tuto.pth_b200.parallel.symm")
    w = _symm_world(3, 1, [4, 6, 9])
    t = torch.zeros(8)
    for fn in (w.send_, w.recv_, w.isend_, w.irecv_):
        with pytest.raises(ValueError, match="cannot (send|recv) to itself"):
            fn(t, 6)                                         # global rank 6 is this rank
        with pytest.raises(ValueError, match="not in this world"):
            fn(t, 1)
        with pytest.raises(TypeError, match="contiguous CUDA tensor"):
            fn(t, 9)
    assert w._p2p_streams == {}                              # nothing reached a stream


# ---------------------------------------------------------------------------------------------------------- bindings
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def test_mailbox_geometry():
    ctas, slots, chunk, pad_words = _C().p2p_config()
    assert (ctas, slots, chunk) == (8, 2, 64 << 10)
    assert pad_words * 4 <= 8192                             # the counters fit the allocation's signal pad
    assert 2 * 7 * ctas <= 132                               # co-residency at 8 GPUs on an H100 SXM


def test_p2p_bindings_refuse_bad_worlds_peers_and_lists():
    C = _C()
    b, s = [0x1000 * (i + 1) for i in range(4)], [0x2000 * (i + 1) for i in range(4)]
    t = torch.zeros(8)                                       # CPU: reaching the tensor check means every other check passed
    for name in ("p2p_send", "p2p_recv"):
        f = getattr(C, name)
        with pytest.raises(RuntimeError, match="world must be in 1..8"):
            f(b, s, t, 1, 0, 9)
        with pytest.raises(RuntimeError, match="at least 2"):
            f(b[:1], s[:1], t, 0, 0, 1)
        with pytest.raises(RuntimeError, match="rank 4 is outside"):
            f(b, s, t, 1, 4, 4)
        with pytest.raises(RuntimeError, match="peer 4 is outside"):
            f(b, s, t, 4, 0, 4)
        with pytest.raises(RuntimeError, match="peer -1 is outside"):
            f(b, s, t, -1, 0, 4)
        with pytest.raises(RuntimeError, match="cannot be its own peer"):
            f(b, s, t, 2, 2, 4)
        with pytest.raises(RuntimeError, match="one mailbox and one signal pad per rank"):
            f(b[:3], s, t, 1, 0, 4)
        with pytest.raises(RuntimeError, match="one mailbox and one signal pad per rank"):
            f(b, s[:2], t, 1, 0, 4)
        with pytest.raises(RuntimeError, match="contiguous CUDA tensor"):
            f(b, s, t, 1, 0, 4)


def test_p2p_launchers_refuse_without_a_launch():
    """b2_p2p_send_launch / b2_p2p_recv_launch return cudaErrorInvalidValue (1) before any CUDA call for each of these, and
    0 for a zero-byte message, which launches nothing (on a machine without a GPU a launch would return another error)."""
    from dist_tuto.pth_b200.ops import _ext
    _C()
    lib = ctypes.CDLL(_ext.so_path())
    i, p, z = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
    box = (ctypes.c_void_p * 8)(*[0x100000 * (r + 1) for r in range(4)])
    sig = (ctypes.c_void_p * 8)(*[0x200000 * (r + 1) for r in range(4)])
    for name in ("b2_p2p_send_launch", "b2_p2p_recv_launch"):
        fn = getattr(lib, name)
        fn.restype = i
        fn.argtypes = [p, p, p, z, i, i, i, p]
        msg = 0x300000
        assert fn(box, sig, msg, 64, 0, 1, 1, None) == 1       # world 1
        assert fn(box, sig, msg, 64, 0, 1, 9, None) == 1       # world 9
        assert fn(box, sig, msg, 64, 4, 1, 4, None) == 1       # rank outside the world
        assert fn(box, sig, msg, 64, 0, 4, 4, None) == 1       # peer outside the world
        assert fn(box, sig, msg, 64, 2, 2, 4, None) == 1       # peer == rank
        assert fn(box, sig, None, 64, 0, 1, 4, None) == 1      # no message
        assert fn(box, sig, msg + 4, 64, 0, 1, 4, None) == 1   # not 16-byte aligned
        assert fn(None, sig, msg, 64, 0, 1, 4, None) == 1      # no mailbox
        assert fn(box, sig, msg, 0, 0, 1, 4, None) == 0        # zero bytes: nothing to launch
