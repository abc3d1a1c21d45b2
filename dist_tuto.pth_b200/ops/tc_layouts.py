"""Host-side model of the shared-memory operand layouts used by the sm_90a tensor-core kernels.

The kernels (csrc/convnet_batched.cu, csrc/gemm_tcgen05.cu) hard-code how TMA lays a box out in shared memory
(128-byte swizzle) and how a wgmma shared-memory descriptor walks it.  These functions state the same rules in numpy so that
(a) CPU tests can cross-check the index arithmetic of the kernels and (b) the hardware probes (tests/test_gpu_tc_probe.py,
csrc/tc_probe.cu) can compare what the GPU really does against them.

Canonical layouts (cute/atom/mma_traits_sm90_gmma.hpp, units of 16 bytes = 8 bf16):
  K-major  SW128  ((8,n),2):((8,SBO),1)            row r, 16-byte chunk c of a 128-byte row:
                                                    (r//8)*SBO + (r%8)*128 + ((c ^ (r%8)) * 16)
  MN-major SW128  ((8,n),(8,k)):((1,LBO),(8,SBO))  element (mn, k): the same image as the K-major tile of the transposed
                                                    [k][mn] matrix; 64-wide mn atoms LBO apart, 8-k-row atoms SBO apart.
"""
from __future__ import annotations

import numpy as np

__all__ = ["sw128_offset", "sw32_offset", "image_rows128", "image_rows32", "expected_tma_image_sw32", "smem_desc", "SW128", "SW32", "expected_tma_image", "bf16_bits", "bits_to_f32"]


def sw128_offset(row: int, byte_in_row: int, sbo: int = 1024) -> int:
    """Byte offset of ``byte_in_row`` (0..127) of 128-byte row ``row`` inside a 128B-swizzled tile (1024-byte aligned)."""
    c = byte_in_row >> 4
    return (row >> 3) * sbo + (row & 7) * 128 + (((c ^ (row & 7)) & 7) << 4) + (byte_in_row & 15)


def bf16_bits(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bit patterns (round to nearest even), as uint16."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u >> 16) & 1) + 0x7FFF
    return ((u + r) >> 16).astype(np.uint16)


def bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << 16).view(np.float32)


def image_rows128(mat_bits: np.ndarray, sbo: int = 1024) -> np.ndarray:
    """uint16 matrix [rows, 64] -> uint8 image of a 128B-swizzled tile (rows padded to a multiple of 8).

    This is both the K-major image of ``mat`` (rows = M or N index, columns = K) and the MN-major image of its transpose
    (rows = K index, columns = 64 consecutive MN elements)."""
    rows = mat_bits.shape[0]
    assert mat_bits.shape[1] == 64 and mat_bits.dtype == np.uint16
    rp = (rows + 7) // 8 * 8
    img = np.zeros(max(rp // 8 * sbo, rp * 128), dtype=np.uint8)
    raw = mat_bits.view(np.uint8).reshape(rows, 128)
    for r in range(rows):
        for c in range(8):
            o = sw128_offset(r, c * 16, sbo)
            img[o:o + 16] = raw[r, c * 16:(c + 1) * 16]
    return img


def sw32_offset(row: int, byte_in_row: int) -> int:
    """Byte offset inside a 32B-swizzled tile of 32-byte rows (Swizzle<1,4,3>: address bit 4 ^= address bit 7)."""
    o = row * 32 + byte_in_row
    return o ^ (((o >> 7) & 1) << 4)


def image_rows32(mat_bits: np.ndarray) -> np.ndarray:
    """uint16 matrix [rows, 16] -> uint8 image of a 32B-swizzled tile: the K-major image of ``mat`` (rows = M/N index, 16 K
    elements per row) and the MN-major image of its transpose (rows = K index, 16 consecutive MN elements per row)."""
    rows = mat_bits.shape[0]
    assert mat_bits.shape[1] == 16 and mat_bits.dtype == np.uint16 and rows % 8 == 0
    img = np.zeros(rows * 32, dtype=np.uint8)
    raw = mat_bits.view(np.uint8).reshape(rows, 32)
    for r in range(rows):
        for c in range(2):
            o = sw32_offset(r, c * 16)
            img[o:o + 16] = raw[r, c * 16:(c + 1) * 16]
    return img


def expected_tma_image_sw32(box_vals: np.ndarray) -> np.ndarray:
    """SWIZZLE_32B counterpart of :func:`expected_tma_image` (address bit 4 ^= address bit 7 of the dense byte stream)."""
    raw = np.ascontiguousarray(box_vals).view(np.uint8).reshape(-1)
    assert raw.size % 256 == 0
    img = np.zeros(raw.size, dtype=np.uint8)
    for o in range(0, raw.size, 16):
        d = o ^ (((o >> 7) & 1) << 4)
        img[d:d + 16] = raw[o:o + 16]
    return img


SW128, SW32 = 1, 3       # descriptor layout types (128-byte / 32-byte swizzle)


def smem_desc(start_bytes: int, lbo_bytes: int, sbo_bytes: int, layout: int = SW128) -> int:
    """64-bit wgmma shared-memory descriptor (start address relative to the image; see csrc/tc_common.cuh::smem_desc)."""
    d = (start_bytes >> 4) & 0x3FFF
    d |= ((lbo_bytes >> 4) & 0x3FFF) << 16
    d |= ((sbo_bytes >> 4) & 0x3FFF) << 32
    d |= (layout & 3) << 62
    return d


def expected_tma_image(box_vals: np.ndarray) -> np.ndarray:
    """What a SWIZZLE_128B TMA box load leaves in shared memory: ``box_vals`` is the box as a uint16 array indexed
    [outer ..., inner] (dense, innermost last); the dense byte stream is cut into 128-byte rows and each row's 16-byte
    chunks are XOR-ed with (row index mod 8) -- the swizzle is a function of the shared-memory address bits only."""
    raw = np.ascontiguousarray(box_vals).view(np.uint8).reshape(-1)
    assert raw.size % 128 == 0
    rows = raw.size // 128
    img = np.zeros(raw.size, dtype=np.uint8)
    for r in range(rows):
        for c in range(8):
            o = sw128_offset(r, c * 16)
            img[o:o + 16] = raw[r * 128 + c * 16: r * 128 + (c + 1) * 16]
    return img
