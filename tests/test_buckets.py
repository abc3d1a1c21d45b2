"""Property tests for the flat gradient-bucket layout (SURVEY §4: "random sizes/offsets ... bucket layout")."""
import torch
import torch.nn as nn
from hypothesis import given, settings, strategies as st

from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel, GradBucket

shapes = st.lists(st.lists(st.integers(1, 7), min_size=1, max_size=4), min_size=1, max_size=8)


def _params(shape_list, channels_last=False):
    ps = []
    for s in shape_list:
        t = torch.randn(*s)
        if channels_last and len(s) == 4:
            t = t.contiguous(memory_format=torch.channels_last)
        ps.append(nn.Parameter(t))
    return ps


@settings(max_examples=60, deadline=None)
@given(shape_list=shapes, align=st.sampled_from([1, 4, 16]), cl=st.booleans())
def test_views_tile_the_flat_buffer_without_overlap(shape_list, align, cl):
    ps = _params(shape_list, cl)
    gb = GradBucket(ps, align=align, symmetric=False)
    assert gb.numel >= sum(p.numel() for p in ps) and gb.flat.numel() == gb.numel
    # offsets: aligned, increasing, segment i ends before segment i+1 starts
    for i, (o, p) in enumerate(zip(gb.offsets, ps)):
        assert o % align == 0
        if i + 1 < len(ps):
            assert o + p.numel() <= gb.offsets[i + 1]
    # every view aliases exactly its own segment and has the parameter's shape and strides
    gb.flat.zero_()
    for i, (v, p, o) in enumerate(zip(gb.views, ps, gb.offsets)):
        assert v.shape == p.shape and v.stride() == p.stride() and p.grad is v
        v.fill_(float(i + 1))
        seg = gb.flat[o:o + p.numel()]
        assert bool((seg == float(i + 1)).all())
    # nothing was written outside the segments (alignment padding stays zero)
    written = sum(p.numel() * (i + 1) for i, p in enumerate(ps))
    assert float(gb.flat.sum()) == float(written)


@settings(max_examples=40, deadline=None)
@given(shape_list=shapes, cap=st.integers(4, 4096))
def test_ddp_buckets_partition_the_parameters_in_reverse_order(shape_list, cap):
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.ps = nn.ParameterList(_params(shape_list))

        def forward(self, x):
            return sum((p * x).sum() for p in self.ps)

    m = M()
    ddp = DistributedDataParallel(m, bucket_cap_bytes=cap, broadcast=False)
    flat_order = [p for b in ddp.buckets for p in b.params]
    assert [id(p) for p in flat_order] == [id(p) for p in reversed(list(m.parameters()))]      # backward order
    for b in ddp.buckets:                       # a bucket only exceeds the cap when a single parameter does
        nbytes = sum(p.numel() * 4 for p in b.params)
        assert nbytes <= cap or len(b.params) == 1
    # one backward fills every bucket through the views; averaging at world 1 is the identity
    ddp.zero_grad()
    ddp(torch.tensor(2.0)).backward()
    ddp.finish()
    for p in m.parameters():
        assert torch.allclose(p.grad, torch.full_like(p, 2.0))
    ddp.remove_hooks()


def test_all_reduce_variant_selection_follows_the_threshold_table():
    """pick_variant(): size -> kernel from (ll_max, oneshot_max, nvls_min) -- the per-world thresholds that
    bench/allreduce_sweep.py --emit-table measures (parallel/allreduce_table.json) -- checked without a GPU."""
    from dist_tuto.pth_b200.parallel.symm import SymmWorld, VARIANTS

    def world(n, multicast, ll_max, oneshot_max, nvls_min):
        w = SymmWorld.__new__(SymmWorld)
        w.world, w.multicast = n, multicast
        w.ll_max, w.oneshot_max, w.nvls_min = ll_max, oneshot_max, nvls_min
        return w

    one, two, nvls, ll = VARIANTS["oneshot"], VARIANTS["twoshot"], VARIANTS["nvls"], VARIANTS["ll"]
    assert world(1, False, 0, 0, 0).pick_variant(1 << 20) == one
    # a 2-GPU sweep (bench/allreduce_sweep.py): LL wins to 64 KB, one-shot to 1 MB, two-shot above; NVLS never pays at 2
    w2 = world(2, True, 64 << 10, 1 << 20, 1 << 62)
    assert [w2.pick_variant(b) for b in (1 << 10, 64 << 10, (64 << 10) + 16, 1 << 20, (1 << 20) + 16, 1 << 30)] == [ll, ll, one, one, two, two]
    w8 = world(8, True, 32 << 10, 32 << 10, (32 << 10) + 1)
    assert [w8.pick_variant(b) for b in (1 << 10, 32 << 10, (32 << 10) + 16, 87360, 1 << 30)] == [ll, ll, nvls, nvls, nvls]
    w8n = world(8, False, 32 << 10, 32 << 10, (32 << 10) + 1)       # switch without multicast objects: two-shot takes over
    assert [w8n.pick_variant(b) for b in (1 << 10, 87360, 1 << 30)] == [ll, two, two]
    # the packaged table is well-formed and every entry is usable
    import json
    import os
    from dist_tuto.pth_b200.parallel import symm
    t = json.load(open(symm._TABLE_PATH))
    for k, v in t["worlds"].items():
        assert 2 <= int(k) <= 8 and set(v) >= {"ll_max", "oneshot_max", "nvls_min"} and v["ll_max"] <= symm.LL_CAP_VEC * 16


def test_bf16_gradient_bucket_for_fp32_master_weights():
    """`DistributedDataParallel(grad_dtype=torch.bfloat16)`: gradients are accumulated by autograd directly into a bf16
    flat bucket (half the bytes on the wire), parameters and momentum stay fp32 (`FlatSGD` casts at the update)."""
    import copy
    import torch.nn.functional as F
    import dist_tuto.pth_b200 as dist
    torch.manual_seed(0)
    ref = dist.Net().eval()
    mine = copy.deepcopy(ref)
    ddp = DistributedDataParallel(mine, bucket_cap_bytes=8192, broadcast=False, grad_dtype=torch.bfloat16)
    assert all(b.flat.dtype == torch.bfloat16 for b in ddp.buckets) and len(ddp.buckets) > 1
    opt = dist.FlatSGD(ddp, lr=0.05, momentum=0.5)
    ref_opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    for i in range(3):
        g = torch.Generator().manual_seed(i)
        x, y = torch.randn(16, 1, 28, 28, generator=g), torch.randint(0, 10, (16,), generator=g)
        for model, o in ((ref, ref_opt), (ddp, opt)):
            o.zero_grad()
            F.nll_loss(model(x), y).backward()
            if model is ddp:
                dist.average_gradients(mine)
            o.step()
    for p in mine.parameters():
        assert p.dtype == torch.float32 and p.grad.dtype == torch.bfloat16
    for (n, a), b in zip(ref.named_parameters(), mine.parameters()):
        assert torch.allclose(a, b, atol=3e-3, rtol=3e-2), n          # bf16 gradients: ~3 significant digits
    ddp.remove_hooks()
