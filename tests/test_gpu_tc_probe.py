"""Hardware probes for the tensor-core operand layouts the batched training kernels rely on (csrc/tc_probe.cu).

Each probe builds a shared-memory image (or a tensor map) on the host from the rules in ops/tc_layouts.py, lets the GPU
execute real ``cp.async.bulk.tensor`` / ``wgmma.mma_async`` instructions on it, and compares with plain fp32 matmuls.
A wgmma covers 64 accumulator rows; the 128-row tiles of the kernels are two warpgroups whose A descriptors start 64
rows apart, and the probes check exactly those two descriptors."""
import numpy as np
import pytest
import torch

from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.ops import tc_layouts as L

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def _rand_bits(rng, shape):
    return L.bf16_bits(rng.standard_normal(shape).astype(np.float32))


def _wgmma(a_img, b_img, ops, n, a_mn=False):
    """One warpgroup runs the (adesc, bdesc, accumulate) list; returns D [64, n]."""
    C = _ext.C()
    dev = torch.device("cuda", 0)
    flat = []
    for o in ops:
        flat += [int(o[0]), int(o[1]), int(o[2])]
    out = C.wgmma_probe(torch.from_numpy(a_img).to(dev), torch.from_numpy(b_img).to(dev), bool(a_mn), flat, n)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _rows128(a_img, b_img, ops_of_half, n, a_mn=False):
    """128 accumulator rows as two warpgroup-sized halves: ``ops_of_half(h)`` gives the op list of rows 64h..64h+63."""
    return np.concatenate([_wgmma(a_img, b_img, ops_of_half(h), n, a_mn) for h in range(2)])


def _tma(t, dims, strides, box, swz, coords):
    C = _ext.C()
    img = C.tma_probe(torch.from_numpy(t.view(np.int16)).to("cuda:0"), dims, strides, box, swz, coords)
    torch.cuda.synchronize()
    return img.cpu().numpy()


def test_tma_channel_last_boxes_are_address_swizzled():
    """The boxes the batched engine issues (NHWC activations, 32-byte pixels, SWIZZLE_32B): a shifted 8x8 window of two
    samples, the [y][b][x][c] image of the conv2-forward window descriptors, and zero fill past the batch.  (An x-innermost
    box shifted by an odd number of elements is not a legal box: TMA needs a 16-byte aligned innermost start.)"""
    B = 5
    t = (np.arange(B * 12 * 12 * 16, dtype=np.uint16) + 1).reshape(B, 12, 12, 16)
    got = _tma(t, [16, 12, 12, B], [32, 384, 4608], [16, 8, 8, 2], 1, [0, 3, 2, 1])
    assert np.array_equal(got, L.expected_tma_image_sw32(t[1:3, 2:10, 3:11, :]))
    got = _tma(t, [16, 12, B, 12], [32, 4608, 384], [16, 12, 2, 12], 1, [0, 0, 2, 0])
    assert np.array_equal(got, L.expected_tma_image_sw32(np.ascontiguousarray(t[2:4].transpose(1, 0, 2, 3))))
    got = _tma(t, [16, 12, 12, B], [32, 384, 4608], [16, 8, 8, 2], 1, [0, 1, 1, 4])
    box = np.zeros((2, 8, 8, 16), dtype=np.uint16)
    box[0] = t[4, 1:9, 1:9, :]
    assert np.array_equal(got, L.expected_tma_image_sw32(box))


def test_umma_shifted_window_descriptors():
    """conv2 forward: 25 taps = 25 K-major SWIZZLE_32B descriptors over ONE [y][b][x][c] image (start + ky*768 + kx*32,
    SBO = 384; rows 64..127 start 8 row groups later); conv2 weight gradient: MN-major with overlapping 16-channel atoms
    32 bytes apart (rows 64..127 start 4 atoms later)."""
    rng = np.random.default_rng(6)
    pix = _rand_bits(rng, (12, 2, 12, 16))
    b = _rand_bits(rng, (32, 64))
    ky, kx = 2, 3
    d = _rows128(L.expected_tma_image_sw32(pix), L.image_rows128(b),
                 lambda h: [(L.smem_desc(ky * 768 + kx * 32 + h * 8 * 384, 16, 384, L.SW32), L.smem_desc(0, 16, 1024), 0)], 32)
    pf, bf = L.bits_to_f32(pix), L.bits_to_f32(b)[:, :16]
    ref = np.zeros((128, 32), np.float32)
    for oy in range(8):
        for bb in range(2):
            for ox in range(8):
                ref[(oy * 2 + bb) * 8 + ox] = pf[oy + ky, bb, ox + kx] @ bf.T
    assert float(np.abs(d - ref).max() / np.abs(ref).max()) < 1e-3
    pix1 = _rand_bits(rng, (12, 12, 16))
    a_img = np.concatenate([L.expected_tma_image_sw32(pix1), np.zeros(1024, np.uint8)])
    ky = 1
    d = _rows128(a_img, L.image_rows128(b),
                 lambda h: [(L.smem_desc(h * 128 + ky * 384 + ks * 768, 32, 384, L.SW32), L.smem_desc(ks * 32, 16, 1024), int(ks > 0))
                            for ks in range(4)], 32, a_mn=True)
    pf1, bfull = L.bits_to_f32(pix1).reshape(144, 16), L.bits_to_f32(b)
    ref = np.zeros((80, 32), np.float32)
    for kx in range(5):
        for ci in range(16):
            row = np.array([pf1[(oy + ky) * 12 + ox + kx, ci] for oy in range(8) for ox in range(8)], np.float32)
            ref[kx * 16 + ci] = bfull @ row
    assert float(np.abs(d[:80] - ref).max() / np.abs(ref).max()) < 1e-3


def test_umma_kmajor_sw128_reference_mode():
    """The mode gemm_tcgen05.cu uses: A [128 x 64] and B [32 x 64] K-major, four K=16 steps, rows 64..127 8 KB later."""
    rng = np.random.default_rng(0)
    a, b = _rand_bits(rng, (128, 64)), _rand_bits(rng, (32, 64))
    d = _rows128(L.image_rows128(a), L.image_rows128(b),
                 lambda h: [(L.smem_desc(h * 8192 + k * 32, 16, 1024), L.smem_desc(k * 32, 16, 1024), int(k > 0)) for k in range(4)], 32)
    ref = L.bits_to_f32(a) @ L.bits_to_f32(b).T
    err = float(np.abs(d - ref).max() / np.abs(ref).max())
    assert err < 1e-3


def _mn_major_a_image(a_bits_mk, k_rows_per_atom):
    """A[m, k] (m = 128 = two 64-wide atoms) stored MN-major: per atom a [k][64 m] 128B-swizzled block."""
    M, K = a_bits_mk.shape
    blocks = []
    for atom in range(M // 64):
        blocks.append(L.image_rows128(np.ascontiguousarray(a_bits_mk[atom * 64:(atom + 1) * 64, :].T)))   # [k][64]
    return np.concatenate(blocks), blocks[0].size


def test_umma_mn_major_a_operand():
    """conv2 data-gradient: A is stored [k][64 positions] per sample (MN-major), B K-major; SBO = stride between 8-row K
    atoms (1024), the second sample (rows 64..127) one atom block later.  The swapped reading must not match."""
    rng = np.random.default_rng(1)
    K = 32
    a, b = _rand_bits(rng, (128, K)), _rand_bits(rng, (32, 64))
    a_img, atom_bytes = _mn_major_a_image(a, K)
    b_img = L.image_rows128(b)
    ref = L.bits_to_f32(a) @ L.bits_to_f32(b)[:, :K].T
    res = {}
    for name, lbo, sbo in (("cute", atom_bytes, 1024), ("swapped", 1024, atom_bytes)):
        d = _rows128(a_img, b_img, lambda h: [(L.smem_desc(h * atom_bytes + s * 2048, lbo, sbo), L.smem_desc(s * 32, 16, 1024), int(s > 0))
                                              for s in range(K // 16)], 32, a_mn=True)
        res[name] = float(np.abs(d - ref).max() / np.abs(ref).max())
    assert res["cute"] < 1e-3 and res["swapped"] > 1e-2, res


def test_umma_wide_n_from_row_offsets():
    """conv2 data-gradient: N = 400 as five instructions of N = 80 at B rows 0, 80, ..., 320 of one K-major B tile."""
    rng = np.random.default_rng(2)
    K = 32
    a, b = _rand_bits(rng, (128, K)), _rand_bits(rng, (400, 64))
    a_img, atom_bytes = _mn_major_a_image(a, K)
    b_img = L.image_rows128(b)
    ref = L.bits_to_f32(a) @ L.bits_to_f32(b)[:, :K].T
    for c0 in range(0, 400, 80):
        d = _rows128(a_img, b_img, lambda h: [(L.smem_desc(h * atom_bytes + s * 2048, atom_bytes, 1024),
                                               L.smem_desc(c0 * 128 + s * 32, 16, 1024), int(s > 0)) for s in range(K // 16)],
                     80, a_mn=True)
        err = float(np.abs(d - ref[:, c0:c0 + 80]).max() / np.abs(ref).max())
        assert err < 1e-3, (c0, err)
