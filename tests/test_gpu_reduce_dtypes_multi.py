"""``comm.all_reduce`` and ``comm.reduce`` of fp16, fp64, int8, uint8, int32, int64 and bool on ``backend="b200"``: the
peer-memory kernels through the public API, never NCCL, against NCCL at the available world sizes and on a sub-group.
Integer and bool results are bit-equal to NCCL's, MAX / MIN equal on NaN-free inputs, fp16 / fp64 SUM and PRODUCT within a
tolerance (NCCL rounds fp16 after every step)."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import reduce_dtypes_workers as W

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900), pytest.mark.multigpu]


def go(fn, size):
    b2.launch(fn, size=size, backend="b200", join_timeout_s=600)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_new_dtype_reductions_match_nccl(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    go(W.w_reduce_dtypes_vs_nccl, world)


def test_new_dtype_reductions_on_a_subgroup_match_nccl():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    go(W.w_reduce_dtypes_subgroup_vs_nccl, min(n, 4))


def test_evaluate_on_b200_equals_its_cpu_float64_reference():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    go(W.w_evaluate_takes_the_fp64_kernels, min(n, 4))
