"""The optimizer-update bindings refuse bad input before anything is launched, and every variant of one family (plain,
grouped, capturable; and the layer-wise pair) refuses the same input with the same message.  The tensors here are CPU
tensors and the per-rank pointers fake: every call must stop at a host check, so nothing is launched or dereferenced."""
import os

import pytest
import torch


def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


N = 64                                               # elements of every flat; 16 fp32 vectors
SC_ADAMW = [0.99, 0.1, 0.999, 0.001, 0.01, 0.03, 1e-8]
SC_RMSPROP = [0.01, 0.0, 0.99, 0.01, 1e-8, 0.0]
SC_LAMB = [0.1, 0.999, 0.001, 0.03, 1e-6, 10.0, 0.01, 0.01]


def _flats(k):
    return [torch.zeros(N) for _ in range(k)]


def _refusal(call, name):
    """The message ``call`` raises, without the binding's name in front of it (which must be ``name``)."""
    with pytest.raises(RuntimeError) as e:
        call()
    msg = str(e.value).splitlines()[0]
    assert msg.startswith(name + ": "), msg
    return msg[len(name) + 2:]


def _same_refusal(calls, match):
    """Every binding of ``calls`` ({name: call}) refuses with one message, and it contains ``match``."""
    msgs = {name: _refusal(call, name) for name, call in calls.items()}
    assert len(set(msgs.values())) == 1, msgs
    assert match in next(iter(msgs.values())), msgs


# ---------------------------------------------------------------------------------------------------- unsharded families
def _sgd_flat(C, wd=0.0, mu=0.5, nesterov=False, **kw):
    p, m, g = _flats(3)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    calls = {"sgd_flat": lambda: C.sgd_flat(p, m, g, 0.1, mu, wd, True, nesterov, **kw),
             "sgd_flat_grouped": lambda: C.sgd_flat_grouped(p, m, g, gmap, [0.1], [wd], mu, True, nesterov, **kw)}
    if wd == 0.0:                                    # the capturable form takes every weight decay from the block
        calls["sgd_flat_cap"] = lambda: C.sgd_flat_cap(p, m, g, gmap, block, mu, True, nesterov, **kw)
    return calls


def _adamw_flat(C, **kw):
    p, m, v, g = _flats(4)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    return {"adamw_flat": lambda: C.adamw_flat(p, m, v, g, SC_ADAMW, True, **kw),
            "adamw_flat_grouped": lambda: C.adamw_flat_grouped(p, m, v, g, gmap, SC_ADAMW, [0.99], [0.01], True, **kw),
            "adamw_flat_cap": lambda: C.adamw_flat_cap(p, m, v, g, gmap, block, True, **kw)}


def _rmsprop_flat(C, **kw):
    p, sq, g = _flats(3)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    return {"rmsprop_flat": lambda: C.rmsprop_flat(p, sq, None, None, g, SC_RMSPROP, False, True, **kw),
            "rmsprop_flat_grouped": lambda: C.rmsprop_flat_grouped(p, sq, None, None, g, gmap, SC_RMSPROP, False, [0.01], [0.0],
                                                                   True, **kw),
            "rmsprop_flat_cap": lambda: C.rmsprop_flat_cap(p, sq, None, None, g, gmap, block, SC_RMSPROP, False, True, **kw)}


def _caps(C, **kw):
    return {name: call for fam in (_sgd_flat, _adamw_flat, _rmsprop_flat) for name, call in fam(C, **kw).items()
            if name.endswith("_cap")}


def test_flat_sgd_refuses_nesterov_without_momentum():
    _same_refusal(_sgd_flat(_C(), mu=0.0, nesterov=True), "nesterov needs a nonzero momentum")


def test_flat_sgd_refuses_a_negative_weight_decay():
    _same_refusal(_sgd_flat(_C(), wd=-0.1), "weight_decay must be >= 0, got -0.1")


@pytest.mark.parametrize("family", [_sgd_flat, _adamw_flat, _rmsprop_flat])
def test_flat_updates_refuse_max_grad_norm_without_sqnorms(family):
    _same_refusal(family(_C(), max_grad_norm=1.0), "max_grad_norm needs sqnorms")


def test_capturable_updates_refuse_grad_scale_without_found_inf():
    _same_refusal(_caps(_C(), grad_scale=torch.ones(1)), "grad_scale comes with found_inf")


@pytest.mark.parametrize("family", [_sgd_flat, _adamw_flat, _rmsprop_flat])
def test_flat_updates_refuse_cpu_buffers(family):
    _same_refusal(family(_C()), f"16-byte aligned contiguous fp32 CUDA tensors on one device, of one size, {N} elements")


# ---------------------------------------------------------------------------------------------------- sharded families
def _peers(world, n=None):
    n = world if n is None else n
    return [[0x100000 * (r + 1) + 0x10000 * i for r in range(n)] for i in range(4)]


def _sharded_sgd(C, world=2, rank=0, n_vec=16, ptrs=None, wd=0.0, mu=0.5, nesterov=False):
    g, p, s, _ = _peers(world) if ptrs is None else ptrs
    (m,) = _flats(1)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    calls = {"sharded_sgd": lambda: C.sharded_sgd(False, g, p, s, m, n_vec, 0.1, mu, wd, nesterov, 0.5, True, rank, world),
             "sharded_sgd_grouped": lambda: C.sharded_sgd_grouped(False, g, p, s, m, gmap, n_vec, [0.1], [wd], mu, nesterov, 0.5,
                                                                  True, rank, world)}
    if wd == 0.0:
        calls["sharded_sgd_cap"] = lambda: C.sharded_sgd_cap(False, g, p, s, m, gmap, block, n_vec, mu, nesterov, 0.5, True, rank,
                                                             world)
    return calls


def _sharded_adamw(C, world=2, rank=0, n_vec=16, ptrs=None):
    g, p, s, _ = _peers(world) if ptrs is None else ptrs
    m, v = _flats(2)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    return {"sharded_adamw": lambda: C.sharded_adamw(False, g, p, s, m, v, n_vec, SC_ADAMW, 0.5, True, rank, world),
            "sharded_adamw_grouped": lambda: C.sharded_adamw_grouped(False, g, p, s, m, v, gmap, n_vec, SC_ADAMW, [0.99], [0.01], 0.5,
                                                                     True, rank, world),
            "sharded_adamw_cap": lambda: C.sharded_adamw_cap(False, g, p, s, m, v, gmap, block, n_vec, 0.5, True, rank, world)}


def _sharded_rmsprop(C, world=2, rank=0, n_vec=16, ptrs=None):
    g, p, s, _ = _peers(world) if ptrs is None else ptrs
    (sq,) = _flats(1)
    gmap, block = torch.zeros(N // 4, dtype=torch.uint8), torch.zeros(4096, dtype=torch.uint8)
    return {"sharded_rmsprop": lambda: C.sharded_rmsprop(False, g, p, s, sq, None, None, n_vec, SC_RMSPROP, False, 0.5, True, rank,
                                                         world),
            "sharded_rmsprop_grouped": lambda: C.sharded_rmsprop_grouped(False, g, p, s, sq, None, None, gmap, n_vec, SC_RMSPROP,
                                                                         False, [0.01], [0.0], 0.5, True, rank, world),
            "sharded_rmsprop_cap": lambda: C.sharded_rmsprop_cap(False, g, p, s, sq, None, None, gmap, block, n_vec, SC_RMSPROP,
                                                                 False, 0.5, True, rank, world)}


def _sharded_layerwise(C, world=2, rank=0, n_vec=16, ptrs=None):
    g, p, s, sums = _peers(world) if ptrs is None else ptrs
    m, v = _flats(2)
    # a table of rank 0 of 2 (the bindings check the world before the table); int64 / int32 / fp32 CPU workspaces
    table = C.sharded_layerwise_table([0], [N * 2], [True], N * 2, 0, 2, torch.device("cpu"))
    partials = torch.zeros(2 * table.n_chunks)
    tickets, ratios = torch.zeros(1, dtype=torch.int32), torch.zeros(1)
    return {"sharded_lamb": lambda: C.sharded_lamb(False, g, p, sums, s, m, v, table, partials, tickets, ratios, n_vec, SC_LAMB, 0.5,
                                                   True, rank, world),
            "sharded_lars": lambda: C.sharded_lars(False, g, p, sums, s, m, v, table, partials, tickets, ratios, n_vec, 0.1, 0.9, 0.0,
                                                   0.001, 0.0, False, 0.5, True, rank, world)}


SHARDED = [_sharded_sgd, _sharded_adamw, _sharded_rmsprop, _sharded_layerwise]


@pytest.mark.parametrize("family", SHARDED)
@pytest.mark.parametrize("rank,world", [(0, 0), (0, 9), (-1, 2), (2, 2)])
def test_sharded_updates_refuse_a_bad_world_or_rank(family, rank, world):
    C = _C()
    calls = family(C, world=world, rank=rank, ptrs=_peers(world, n=max(world, 1)))
    msgs = {name: _refusal(call, name) for name, call in calls.items()}
    assert len(set(msgs.values())) == 1, msgs
    assert "world must be in 1..8" in next(iter(msgs.values())) or "is outside" in next(iter(msgs.values()))


@pytest.mark.parametrize("family", SHARDED)
@pytest.mark.parametrize("which", range(4))
def test_sharded_updates_refuse_pointer_lists_of_the_wrong_length(family, which):
    ptrs = _peers(3)
    ptrs[which] = ptrs[which][:2]
    if family is not _sharded_layerwise and which == 3:      # only the layer-wise kernels take the sums buffers
        ptrs[2] = ptrs[2] + [0x9990000]
    _same_refusal(family(_C(), world=3, n_vec=30, ptrs=ptrs), "one gradient bucket, parameter flat")


@pytest.mark.parametrize("family", SHARDED)
def test_sharded_updates_refuse_a_slice_remainder(family):
    _same_refusal(family(_C(), world=3, n_vec=31), "n_vec must be a multiple of world")


@pytest.mark.parametrize("family", SHARDED)
@pytest.mark.parametrize("bad", [0, 0x100008])
def test_sharded_updates_refuse_a_null_or_misaligned_pointer(family, bad):
    for which in range(4 if family is _sharded_layerwise else 3):
        ptrs = _peers(2)
        ptrs[which][1] = bad
        _same_refusal(family(_C(), ptrs=ptrs), "null or misaligned per-rank pointer")


def test_sharded_sgd_refuses_nesterov_without_momentum():
    _same_refusal(_sharded_sgd(_C(), mu=0.0, nesterov=True), "nesterov needs a nonzero momentum")


def test_sharded_sgd_refuses_a_negative_weight_decay():
    _same_refusal(_sharded_sgd(_C(), wd=-0.1), "weight_decay must be >= 0, got -0.1")


@pytest.mark.parametrize("family", [_sharded_sgd, _sharded_adamw, _sharded_rmsprop])
def test_sharded_updates_refuse_cpu_state(family):
    _same_refusal(family(_C()), "16-byte aligned contiguous fp32 CUDA tensors on one device, of at least 32 elements")
