"""Host-side layout contracts shared between Python and the CUDA kernels, checked without a GPU."""
import types

import torch

from dist_tuto.pth_b200.models.convnet import Net, PARAM_SHAPES
from dist_tuto.pth_b200.ops import convnet_fused as cf


def test_flat_parameter_layout_matches_the_kernel_constants():
    # csrc/convnet_args.cuh: W1 0, B1 252, W2 264, B2 5264, W3 5284, B3 21284, W4 21336, B4 21836, NPAR 21848
    assert cf.LAYOUT == {"conv1.weight": 0, "conv1.bias": 252, "conv2.weight": 264, "conv2.bias": 5264, "fc1.weight": 5284,
                         "fc1.bias": 21284, "fc2.weight": 21336, "fc2.bias": 21836}
    assert cf.NPAR == 21848 and cf.NPAR_ALLOC % 64 == 0 and cf.NPAR_ALLOC >= cf.NPAR
    for name, shape in PARAM_SHAPES:                       # every segment starts 16-byte aligned (float4 accesses)
        assert cf.LAYOUT[name] % 4 == 0, name
    total = sum(int(torch.tensor(s).prod()) for _, s in PARAM_SHAPES)
    assert total == 21840                                  # the reference Net (train_dist.py:53-62)


def test_pack_unpack_roundtrip_and_padding_is_zero():
    torch.manual_seed(0)
    net = Net()
    flat = cf.pack_params(net, torch.device("cpu"))
    assert flat.numel() == cf.NPAR_ALLOC
    views = cf.unpack_params(flat)
    covered = torch.zeros(cf.NPAR_ALLOC, dtype=torch.bool)
    for name, p in net.state_dict().items():
        assert torch.equal(views[name], p)
        covered[cf.LAYOUT[name]:cf.LAYOUT[name] + p.numel()] = True
    assert float(flat[~covered].abs().sum()) == 0.0        # alignment gaps + tail stay zero (SGD never moves them)


def test_prearranged_conv2_weights_match_the_kernel_indexing():
    """`aux` = conv2.weight in the two shared-memory layouts of the step kernels; the SGD kernels keep it current with
    (csrc/sgd.cu, sgd_apply):  w2f[(ci*25 + kk)*20 + co]  and  w2b[5000 + ((co*25 + kk)*2 + ci/5)*8 + ci%5]."""
    torch.manual_seed(1)
    net = Net()
    fake = types.SimpleNamespace(params=cf.pack_params(net, torch.device("cpu")), aux=torch.full((13000,), float("nan")),
                                 device=torch.device("cpu"))
    cf.FusedTrainer._refresh_aux(fake)
    w2 = net.conv2.weight.detach().reshape(20, 10, 25)     # [co][ci][ky*5+kx]
    expect = torch.zeros(13000)
    for co in range(20):
        for ci in range(10):
            for kk in range(25):
                v = w2[co, ci, kk]
                expect[(ci * 25 + kk) * 20 + co] = v
                expect[5000 + ((co * 25 + kk) * 2 + ci // 5) * 8 + ci % 5] = v
    assert torch.equal(fake.aux, expect)                   # including the zero padding lanes 5..7 of every w2b group


def test_cluster_policy_keeps_one_wave():
    # one CTA per sample above 64 samples, clusters below; C * B never exceeds the 132 SMs of an H100
    for b, c in ((128, 1), (64, 2), (32, 4), (16, 4), (8, 8), (1, 8)):
        assert cf.pick_cluster(b) == c and b * c <= 132


def test_tc_layout_model_swizzles_are_involutions_and_window_addresses_stay_inside_the_image():
    """ops/tc_layouts.py (host model of the TMA / wgmma shared-memory images used by csrc/convnet_batched.cu)."""
    import numpy as np
    from dist_tuto.pth_b200.ops import tc_layouts as L
    # 32B / 128B swizzles permute 16-byte chunks inside their repeat (256 B / 1024 B) and are their own inverse
    offs = [L.sw32_offset(r, c) for r in range(16) for c in (0, 16)]
    assert sorted(offs) == list(range(0, 512, 16))
    offs = [L.sw128_offset(r, c * 16) for r in range(8) for c in range(8)]
    assert sorted(offs) == list(range(0, 1024, 16))
    m = np.arange(64 * 16, dtype=np.uint16).reshape(64, 16)
    assert np.array_equal(L.image_rows32(m), L.expected_tma_image_sw32(m))
    # conv2-forward window descriptors: image [12 y][2 b][12 x] pixels of 32 B; tap (ky, kx) starts at ky*768 + kx*32 and walks
    # 16 row groups (oy, b) 384 B apart, 8 pixels each -> the last byte touched is exactly the end of the 9216-byte image
    last = max(ky * 768 + kx * 32 + g * 384 + ox * 32 + 31 for ky in range(5) for kx in range(5) for g in range(16) for ox in range(8))
    assert last == 12 * 2 * 12 * 32 - 1
    # conv2 weight-gradient windows: image [12 y][12 x] pixels; atoms kx = 0..7 (5 real), K-steps of two image rows;
    # the over-read past the 4608-byte image stays inside the 512-byte zero padding the kernel keeps behind it
    last = max(ky * 384 + ks * 768 + katom * 384 + pos * 32 + kx * 32 + 31
               for ky in range(5) for ks in range(4) for katom in range(2) for pos in range(8) for kx in range(8))
    assert 4608 <= last < 4608 + 512
    # descriptor fields
    d = L.smem_desc(0x1230, 32, 384, L.SW32)
    assert d & 0x3FFF == 0x123 and (d >> 16) & 0x3FFF == 2 and (d >> 32) & 0x3FFF == 24 and (d >> 62) == 3 and (d >> 46) & 0xFFFF == 0
    assert L.smem_desc(0, 16, 1024) >> 62 == 1 and (L.smem_desc(0, 16, 1024) >> 46) & 0xFFFF == 0
