"""FlatLAMB / FlatLARS(sharded=True) on backend "b200" at world 1: the unsharded optimizer, bit for bit."""
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def test_sharded_true_at_world_1_equals_sharded_false():
    import dist_tuto.pth_b200 as b2
    import sharded_layerwise_workers as WK
    b2.launch(WK.w_world1, size=1, backend="b200", join_timeout_s=600)
