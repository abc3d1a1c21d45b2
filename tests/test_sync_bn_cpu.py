"""``SyncBatchNorm`` on gloo CPU ranks (worlds 2 and 3): outputs, gradients, running stats and ``num_batches_tracked`` against
fp64 ``F.batch_norm`` of the global batch, the converter and state dicts, and a subgroup.  Workers in
tests/sync_bn_workers.py."""
import pytest

import dist_tuto.pth_b200 as b2
import sync_bn_workers as W

pytestmark = pytest.mark.timeout(300)


def go(fn, size):
    b2.launch(fn, size=size, backend="gloo", join_timeout_s=250)


@pytest.mark.parametrize("size", [2, 3])
def test_matches_fp64_batch_norm_of_the_global_batch(size):
    go(W.w_matches_global_batch_norm, size)


def test_convert_sync_batchnorm_keeps_objects_and_state_dict_round_trips():
    go(W.w_convert_and_state_dict, 2)


def test_subgroup_process_group():
    go(W.w_subgroup, 3)


def test_exchange_is_padded_for_the_fused_path():
    from dist_tuto.pth_b200.parallel.sync_bn import exchange_numel
    for world in range(1, 9):
        for n in (3, 129, 1 + 2 * 2049):
            m = exchange_numel(n, world)
            assert m >= n and (m * 8) % (16 * world) == 0 and m - n < 2 * world
