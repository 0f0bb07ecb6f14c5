"""Address rehearsal of the stride-1 3x3 patch path (conv_tc.cu, tc_conv_patch_consumer), without a GPU.

The producer's TMA box {16-byte group, bw + 2, bh + 2, 8 groups} lands in shared memory as
[group][patch row][patch col][16 B].  The consumer reads tap (r, s), m64 half h and K step k through a no-swizzle K-major
descriptor
  start = (r * PW + s + half_off(h)) * 16 B + k * 2 * plane,  SBO = PW * 16 B,  LBO = plane,
  PW = bw + 2,  half_off(h) = 8 PW h (bw = 8) or 8 h (bw = 16),
whose canonical layout (PTX ISA, wgmma matrix descriptors) places element (row m, K index q) of the 64 x K operand at
  start + (m // 8) * SBO + (m % 8) * 16 B + (q // E) * LBO + (q % E) * elem,   E = 16 B / elem.
For every tile shape, tap, half, K step and element this must be the patch cell of the pixel that the epilogue stores
accumulator row m of half h to, shifted by (s, r), channel 2 E k + q of the K block."""
import itertools

import pytest

PLANE = 180 * 16                     # kPatchPlane


def epilogue_pixel(bw, h, m):
    """pixel (px, py) of accumulator row m of half h (tc_conv_epilogue's staging row = py * bw + px)"""
    if bw == 16:                     # col_halves
        row = ((m >> 3) << 4) + 8 * h + (m & 7)
    else:
        row = 64 * h + m
    return row % bw, row // bw


def desc_fields(start16, lbo16, sbo16):
    """desc_noswz of ptx.cuh, decoded back into byte quantities"""
    d = (start16 & 0x3FFF) | ((lbo16 & 0x3FFF) << 16) | ((sbo16 & 0x3FFF) << 32)
    assert d >> 62 == 0   # layout type 0: no swizzle
    return (d & 0x3FFF) * 16, ((d >> 16) & 0x3FFF) * 16, ((d >> 32) & 0x3FFF) * 16


@pytest.mark.parametrize("elem", [4, 2])   # tf32, bf16
@pytest.mark.parametrize("bw,bh", [(8, 16), (16, 8)])
def test_patch_descriptors_address_the_tap_window(bw, bh, elem):
    PW, PH = bw + 2, bh + 2
    assert PW * PH * 16 == PLANE
    row16 = PW
    half16 = 8 * row16 if bw == 8 else 8
    plane16 = PLANE // 16

    def tma_offset(group, y, x, byte):
        assert 0 <= y < PH and 0 <= x < PW
        return ((group * PH + y) * PW + x) * 16 + byte

    E = 16 // elem                 # K elements per core-matrix row
    KS = 2 * E                     # K per wgmma (8 tf32, 16 bf16)
    for r, s, h, k in itertools.product(range(3), range(3), range(2), range(4)):
        a16 = r * row16 + s + h * half16 + 2 * k * plane16
        start, lbo, sbo = desc_fields(a16, plane16, row16)
        for m in range(64):
            px, py = epilogue_pixel(bw, h, m)
            for q in range(KS):
                got = start + (m // 8) * sbo + (m % 8) * 16 + (q // E) * lbo + (q % E) * elem
                c = KS * k + q     # channel inside the 128-byte K block
                assert got == tma_offset(c // E, py + r, px + s, (c % E) * elem), (r, s, h, k, m, q)


@pytest.mark.parametrize("bw", [8, 16])
def test_epilogue_rows_cover_the_tile_once(bw):
    pix = {epilogue_pixel(bw, h, m) for h in range(2) for m in range(64)}
    assert pix == {(x, y) for x in range(bw) for y in range(128 // bw)}
