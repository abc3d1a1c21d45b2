"""The model of the sharded optimizer kernel (tests/sharded_sgd_model.py) against the models of the path it replaces, and the
planted faults the bit-for-bit checker has to catch.  No GPU."""
import re

import pytest
import torch

import comm_model as M
import sharded_sgd_model as S

OPTIONS = [(0.0, False), (0.01, False), (0.0, True), (0.01, True)]          # (weight decay, nesterov)


def _case(world, per_vec, dtype, seed):
    n = world * per_vec * M.elems_per_vec(dtype)
    grads = M.make_inputs(world, n, dtype, seed, specials=False)
    params, shards, full = S.make_state(world, n, seed + 1)
    return n, grads, params, shards, full


def test_constants_follow_the_cuda_source():
    src = open(M.CSRC + "/sharded_sgd.cu").read()
    assert int(re.search(r"constexpr int kShardThreads = (\d+);", src).group(1)) == M.THREADS
    assert int(re.search(r"constexpr int kShardUnroll = (\d+);", src).group(1)) == M.UNROLL
    assert S.grid_blocks(8 * 5000, 8, 3) == 3 and S.grid_blocks(8 * 5000, 8, 0) == 5 and S.grid_blocks(8, 8, 0) == 1


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("variant", [M.ONESHOT, M.TWOSHOT], ids=["oneshot", "twoshot"])
def test_fp32_equals_allreduce_then_unsharded_sgd(world, variant):
    for k, (wd, nesterov) in enumerate(OPTIONS):
        n, grads, params, shards, full = _case(world, 37 + k, torch.float32, 10 * world + k)
        scale, lr, mu = 1.0 / world, 0.07, 0.9
        for step in range(3):                                        # momentum carries from step to step
            out = S.sharded_sgd_model(grads, params, shards, scale, lr, mu, wd, nesterov, zero_grad=True)
            p_ref, m_ref = S.unsharded_model(variant, grads, params[0], full, scale, lr, mu, wd, nesterov)
            M.assert_bits_equal(f"world {world} step {step}: params", out["params"], [p_ref] * world, 4)
            M.assert_bits_equal(f"world {world} step {step}: momentum", [torch.cat(out["momentum"])], [m_ref], 4)
            assert all(not g.any() for g in out["grads"])
            params, shards, full = out["params"], out["momentum"], m_ref
            grads = M.make_inputs(world, n, torch.float32, 1000 + 10 * world + step, specials=False)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_slices_and_what_stays_local(world):
    n, grads, params, shards, _ = _case(world, 5, torch.float32, world)
    out = S.sharded_sgd_model(grads, params, shards, 1.0 / world, 0.1, 0.5, 0.0, False, zero_grad=False)
    assert [S.slice_of(r, world, n) for r in range(world)] == [(r * 20, r * 20 + 20) for r in range(world)]
    assert all(m.numel() == n // world for m in out["momentum"])
    M.assert_bits_equal("replicas", out["params"], [out["params"][0]] * world, 4)
    M.assert_bits_equal("zero_grad off keeps the local gradients", out["grads"], grads, 4)


def test_bf16_gradients_feed_the_update_unrounded():
    world = 4
    n, grads, params, shards, _ = _case(world, 16, torch.bfloat16, 3)
    out = S.sharded_sgd_model(grads, params, shards, 1.0 / world, 0.1, 0.5, 0.0, False, zero_grad=True)
    acc = M.reduce_scaled([g.float() for g in grads], 1.0 / world)
    rounded = M.bf16_rn(acc)
    assert not torch.equal(acc, rounded)                             # the round trip would lose bits here
    per = n // world
    for r in range(world):
        exact = S.sgd_update(acc[r * per:(r + 1) * per], params[r][r * per:(r + 1) * per], shards[r], S.f32(0.5), S.f32(0.1),
                             0.0, False)
        lossy = S.sgd_update(rounded[r * per:(r + 1) * per], params[r][r * per:(r + 1) * per], shards[r], S.f32(0.5),
                             S.f32(0.1), 0.0, False)
        assert torch.equal(out["momentum"][r], exact[1]) and not torch.equal(out["momentum"][r], lossy[1])
        assert torch.equal(out["params"][0][r * per:(r + 1) * per], exact[0])
    assert all(g.dtype == torch.bfloat16 and not g.any() for g in out["grads"])


@pytest.mark.parametrize("fault", S.FAULTS)
@pytest.mark.parametrize("world", [3, 5])                 # not 2: a sum of two terms has no order
def test_planted_faults_are_caught(world, fault):
    n, grads, params, shards, _ = _case(world, 9, torch.float32, 40 + world)
    args = (grads, params, shards, 1.0 / world, 0.1, 0.5, 0.01, True)
    want = S.sharded_sgd_model(*args, zero_grad=True)
    got = S.sharded_sgd_model(*args, zero_grad=True, fault=fault)
    caught = [k for k in ("params", "momentum", "grads") if M.first_mismatch(got[k], want[k], 4) is not None]
    assert caught, f"the checker does not see {fault}"
    with pytest.raises(AssertionError, match="rank"):
        M.assert_bits_equal(fault, got[caught[0]], want[caught[0]], 4)
