"""Level-1 post-filter slots on the inputs the checkasm-style tests leave to chance.

- CDEF fb: 8, 10 and 12 bit, every block size, edge combination and direction, pri-only / sec-only / both at the
  largest strengths, the smallest and largest damping, and saturated pixels beside missing edges; strengths and
  damping outside what dav1d passes are bad arguments.
- fgy / fguv (the frame kernel's apply arithmetic): every layout, row_num 0 and > 0, overlap on and off, odd widths, and
  the restricted-range clip with and without is_id.
- resize (the frame job's super-resolution kernel over one plane): widths that are not multiples of 4, with mx0 and dx
  at the ends of their ranges.
Each runs on the host emulator and on the GPU against the oracle.
"""
import numpy as np
import pytest

import refs
from test_cdef import oracle_cdef
from test_filmgrain import GH, GW, LAYOUTS, lib_ctx, lut_dtype, oracle_ctx, rand_fg_data

SIZES = [(8, 8), (4, 8), (4, 4)]


def cdef_block(rng, kind, bd, dt, n):
    if kind == 0:
        return np.full(n, bd, dt)
    if kind == 1:
        return rng.integers(0, bd + 1, n).astype(dt)
    return np.where(rng.integers(0, 2, n) == 1, bd, 0).astype(dt)


def check_cdef(new, chk, bpc, seed):
    rng = np.random.default_rng(seed)
    bd, b8, dt = (1 << bpc) - 1, bpc - 8, refs.pixel_dtype(bpc)
    n = 0
    for i, (w, h) in enumerate(SIZES):
        for edges in range(16):
            for d in range(8):
                for s in (1, 2, 3):
                    # saturated, random or 0 / max blocks; the neighbours are random, so a missing side read as a
                    # sample (rather than skipped) changes the result
                    src = cdef_block(rng, (edges + d + s) % 3, bd, dt, 16 * 10 + 16)
                    top = cdef_block(rng, 1, bd, dt, 16 * 2 + 16)
                    bot = cdef_block(rng, 1, bd, dt, 16 * 2 + 16)
                    left = cdef_block(rng, 1, bd, dt, 16)
                    pri = (15 << b8) if s & 2 else 0
                    sec = (4 << b8) if s & 1 else 0
                    for damp in (2 + b8, 6 + b8):
                        a, b = src.copy(), src.copy()
                        chk.fb[i](a[8:], 16 * a.itemsize, left, top[8:], bot[8:], pri, sec, d, damp, edges)
                        new.fb[i](b[8:], 16 * b.itemsize, left, top[8:], bot[8:], pri, sec, d, damp, edges)
                        assert np.array_equal(a, b), ("cdef fb", bpc, w, h, edges, d, pri, sec, damp)
                        n += 1
    return n


def check_cdef_rejects(lib, bpc):
    """b200_cdef_fb outside dav1d's damping 2 + b8 .. 6 + b8, pri <= 15 << b8, sec in {0, 1, 2, 4} << b8: -2, dst untouched"""
    b8, dt = bpc - 8, refs.pixel_dtype(bpc)
    left, edge = np.zeros(16, dt), np.zeros(16 * 2 + 16, dt)
    for pri, sec, damp in ((15 << b8, 0, 1 + b8), (0, 4 << b8, 7 + b8), (16 << b8, 0, 3 + b8), (-1, 1 << b8, 3 + b8),
                           (0, 3 << b8, 3 + b8), (0, 8 << b8, 3 + b8), (0, (2 << b8) + 1, 3 + b8), (0, -(1 << b8), 3 + b8)):
        dst = np.full(16 * 10 + 16, 7, dt)
        args = (dst[8:].ctypes.data, 16 * dst.itemsize, left.ctypes.data, edge[8:].ctypes.data, edge[8:].ctypes.data)
        assert lib.b200_cdef_fb(*args, pri, sec, 0, damp, 8, 8, 15, (1 << bpc) - 1) == -2, (bpc, pri, sec, damp)
        assert lib.b200_last_error().startswith(b"b200_cdef_fb: bad arguments")
        assert (dst == 7).all()


def check_fg(new, chk, bpc, seed):
    rng = np.random.default_rng(seed)
    bd, ldt, pdt = (1 << bpc) - 1, lut_dtype(bpc), refs.pixel_dtype(bpc)
    px, st = np.dtype(pdt).itemsize, 160
    n = 0
    for overlap in (0, 1):
        for clip in (0, 1):
            for row in (0, 7):
                for w in (127, 33):
                    d = rand_fg_data(rng, full=False)
                    d.overlap_flag, d.clip_to_restricted_range = overlap, clip
                    d.chroma_scaling_from_luma = int(w == 33)
                    bh = 32 if row else 17
                    lut = np.zeros((GH + 1, GW), ldt)
                    chk.generate_grain_y(lut, d)
                    scaling = rng.integers(0, 256, 4096).astype(np.uint8)
                    src = rng.integers(0, bd + 1, (32, st)).astype(pdt)
                    a, b = src.copy(), src.copy()
                    chk.fgy(a, src, st * px, d, w, scaling, lut, bh, row)
                    new.fgy(b, src, st * px, d, w, scaling, lut, bh, row)
                    assert np.array_equal(a, b), ("fgy", bpc, overlap, clip, row, w)
                    n += 1
                    for li, (sx, sy) in enumerate(LAYOUTS):
                        for uv, is_id in ((0, 0), (1, 1)):
                            ulut = np.zeros((GH + 1, GW), ldt)
                            chk.generate_grain_uv[li](ulut, lut, d, uv)
                            luma = rng.integers(0, bd + 1, (32, st)).astype(pdt)
                            csrc = rng.integers(0, bd + 1, (32, st)).astype(pdt)
                            a, b = csrc.copy(), csrc.copy()
                            args = (st * px, d, (w + sx) >> sx, scaling, ulut, (bh + sy) >> sy, row, luma, st * px, uv, is_id)
                            chk.fguv[li](a, csrc, *args)
                            new.fguv[li](b, csrc, *args)
                            assert np.array_equal(a, b), ("fguv", bpc, li, uv, is_id, overlap, clip, row, w)
                            n += 1
    return n


def check_resize(new, chk, bpc, seed):
    rng = np.random.default_rng(seed)
    bd, dt = (1 << bpc) - 1, refs.pixel_dtype(bpc)
    n = 0
    for dst_w in (1, 2, 3, 5, 67, 131, 250):
        for w_den in (9, 16):                       # the super-resolution denominators at the two ends (8 / 9 .. 8 / 16)
            src_w = max(1, (dst_w * 8 + w_den // 2) // w_den)
            exact = ((src_w << 14) + (dst_w >> 1)) // dst_w
            for dx in (exact, 1 << 13, 1 << 14):
                for mx0 in (0, 0x3fff):
                    h = 3
                    src = rng.integers(0, bd + 1, (h, 264)).astype(dt)
                    src[:, src_w - 1] = bd              # a saturated last column: the right-edge clamp reads it
                    a = rng.integers(0, bd + 1, (h, 264)).astype(dt)
                    b = a.copy()
                    chk.resize(a, a.strides[0], src, src.strides[0], dst_w, h, src_w, dx, mx0)
                    new.resize(b, b.strides[0], src, src.strides[0], dst_w, h, src_w, dx, mx0)
                    assert np.array_equal(a, b), ("resize", bpc, dst_w, src_w, dx, mx0)
                    n += 1
    return n


def run_all(lib, bpc, seed):
    from dav1d_b200.dsp import CdefDSPContext, MCDSPContext
    assert check_cdef(CdefDSPContext(bpc, lib=lib), oracle_cdef(bpc), bpc, seed) == 3 * 16 * 8 * 3 * 2
    check_cdef_rejects(lib, bpc)
    assert check_fg(lib_ctx(lib, bpc), oracle_ctx(bpc), bpc, seed + 1) == 16 * 7
    assert check_resize(MCDSPContext(bpc, lib=lib), refs.oracle_mc_ctx(bpc), bpc, seed + 2) == 7 * 2 * 3 * 2


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_level1_shared(bpc):
    run_all(refs.emu_lib(), bpc, 600 + bpc)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_level1_shared(bpc):
    from dav1d_b200 import get_lib
    run_all(get_lib(), bpc, 700 + bpc)
