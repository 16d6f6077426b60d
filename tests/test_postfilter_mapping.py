"""Edge cases of the CDEF and loop-restoration frame kernels' thread mappings, against the oracle.

CDEF: the direction search runs on 8 lanes per 8x8 block and the filter writes 4 adjacent columns of a pixel pair
per thread, so the cases cover luma widths ending at every residue mod 64 in steps of 4 (odd 4x4-unit widths and
heights included), images on which each of the 8 directions wins, and primary-only / secondary-only / unfiltered
blocks at the strength extremes with damping 3 and 6 at every bit depth.
Loop restoration: every sgr_idx, Wiener taps at the ends of their legal ranges, unit sizes 32 to 256 and frame widths
that end inside a 32-bit word of samples (the tiles' word staging, word copy and row stores).
Each case runs on the host emulator and on the GPU.
"""
import numpy as np
import pytest

import refs
from dav1d_b200 import synth
from test_cdef import make_cdef_frame, cdef_frame_lib, cdef_frame_oracle, frame_area_equal, oracle_cdef
from test_looprestoration import make_lr_frame, lr_frame_lib, lr_frame_oracle, picture_equal

CDEF_WIDTHS = [(8, 64 + 4 * k, 44, 1, 1) for k in range(1, 17)] + [(10, 100, 52, 1, 0), (12, 76, 36, 0, 0)]
# (y, uv) strength tables: pri + sec, pri only, sec only, neither, at the extremes (pri 15 / 1, sec 4 / 1)
STRENGTHS = ([63, 60, 3, 0, 4, 1, 62, 2], [60, 63, 0, 3, 1, 4, 2, 62])
CDEF_STRENGTH = [(bpc, damp, ssh, ssv) for bpc, ssh, ssv in ((8, 1, 1), (10, 1, 0), (12, 0, 0)) for damp in (3, 6)]


def cdef_case(bpc, W, H, ssh, ssv, seed, damping=None, strengths=None):
    S = make_cdef_frame(np.random.default_rng(seed), bpc, W, H, ssh, ssv)
    if damping is not None:
        S["damping"] = damping
    if strengths is not None:
        S["y_strength"], S["uv_strength"] = strengths
        S["masks"]["cdef_idx"] = np.random.default_rng(seed + 1).integers(0, 8, S["masks"]["cdef_idx"].shape).astype(np.int8)
    return S


def run_cdef(S, gpu):
    return cdef_frame_lib(S, *refs.lib_alloc(gpu))


def oriented_blocks(bpc):
    """8x8 images of straight edges at 32 angles plus noise: together they make every direction win"""
    rng = np.random.default_rng(600 + bpc)
    bd = (1 << bpc) - 1
    yy, xx = np.mgrid[0:8, 0:8]
    out = []
    for k in range(32):
        ang = np.pi * k / 32
        v = np.cos(ang) * xx + np.sin(ang) * yy
        img = np.where(np.sin(v * 1.7) > 0, bd * 3 // 4, bd // 4) + rng.integers(0, 1 + (bd >> 5), (8, 8))
        out.append(img.clip(0, bd).astype(refs.pixel_dtype(bpc)).reshape(-1))
    return out


def check_cdef_dir(bpc, lib):
    from dav1d_b200.dsp import CdefDSPContext
    new, chk = CdefDSPContext(bpc, lib=lib), oracle_cdef(bpc)
    won = set()
    for img in oriented_blocks(bpc):
        exp = chk.dir(img, 8 * img.itemsize)
        assert new.dir(img, 8 * img.itemsize) == exp
        won.add(exp[0])
    assert won == set(range(8))


def lr_case(bpc, W, H, ssh, ssv, us, seed, types=None, taps=None):
    S = make_lr_frame(np.random.default_rng(seed), bpc, W, H, ssh, ssv, 0, us, 7)
    u = S["lr_mask"]["lr"]
    if types is not None:
        u["type"] = np.resize(np.array(types, np.uint8), u["type"].shape)
        idx = np.clip(u["type"].astype(np.int32) - 3, 0, 15)
        s0 = np.array([p[0] for p in synth.SGR_PARAMS])[idx]; s1 = np.array([p[1] for p in synth.SGR_PARAMS])[idx]
        u["sgr_weights"][..., 0] = np.where(s0 > 0, u["sgr_weights"][..., 0], 0)
        u["sgr_weights"][..., 1] = np.where(s1 > 0, u["sgr_weights"][..., 1], 95)
    if taps is not None:
        u["filter_h"][...] = taps; u["filter_v"][...] = taps
        u["filter_h"][:, 1:, :, 0] = 0; u["filter_v"][:, 1:, :, 0] = 0
    return S


def run_lr(S, gpu):
    return lr_frame_lib(S, *refs.lib_alloc(gpu))


# every sgr_idx (types 3 .. 18) and Wiener with none mixed in, at 8 and 10 bit
LR_SGR = [(bpc, list(range(3 + i, 19 + i, 4))[:4]) for bpc in (8, 10) for i in range(4)]
WIENER_EXTREMES = [(-5, -23, -17), (10, 8, 46), (-5, 8, 46), (10, -23, -17)]
LR_UNITS = [(8, (5, 5)), (8, (6, 5)), (10, (7, 6)), (12, (8, 8)), (8, (8, 7))]
LR_WIDTHS = [129, 130, 131, 133, 134, 195]


def lr_sgr_frame(bpc, types):
    S = lr_case(bpc, 130, 57, 1, 1, (6, 5), 610 + types[0], types=[t for t in types] + [0, 2])
    return S


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", CDEF_WIDTHS)
def test_emu_cdef_widths(bpc, W, H, ssh, ssv):
    S = cdef_case(bpc, W, H, ssh, ssv, 620 + W)
    assert frame_area_equal(S, run_cdef(S, False), cdef_frame_oracle(S))


@pytest.mark.emu
@pytest.mark.parametrize("bpc,damp,ssh,ssv", CDEF_STRENGTH)
def test_emu_cdef_strengths(bpc, damp, ssh, ssv):
    S = cdef_case(bpc, 136, 72, ssh, ssv, 630 + bpc + damp, damping=damp, strengths=STRENGTHS)
    exp = cdef_frame_oracle(S)
    assert (exp != S["pic"]).mean() > 0.05
    assert frame_area_equal(S, run_cdef(S, False), exp)


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_cdef_dir_every_direction(bpc):
    check_cdef_dir(bpc, refs.emu_lib())


@pytest.mark.emu
@pytest.mark.parametrize("bpc,types", LR_SGR)
def test_emu_lr_sgr_idx(bpc, types):
    S = lr_sgr_frame(bpc, types)
    assert picture_equal(S, run_lr(S, False), lr_frame_oracle(S))


@pytest.mark.emu
@pytest.mark.parametrize("taps", WIENER_EXTREMES)
def test_emu_lr_wiener_extremes(taps):
    S = lr_case(8 if taps[0] < 0 else 12, 130, 57, 1, 1, (6, 5), 640 + taps[2], types=[2], taps=taps)
    assert picture_equal(S, run_lr(S, False), lr_frame_oracle(S))


@pytest.mark.emu
@pytest.mark.parametrize("bpc,us", LR_UNITS)
def test_emu_lr_unit_sizes(bpc, us):
    S = lr_case(bpc, 200, 76, 1, 1, us, 650 + us[0] + us[1])
    assert picture_equal(S, run_lr(S, False), lr_frame_oracle(S))


@pytest.mark.emu
@pytest.mark.parametrize("W", LR_WIDTHS)
def test_emu_lr_widths(W):
    S = lr_case(8 if W & 1 else 10, W, 40, 1, 1, (6, 6), 660 + W)
    assert picture_equal(S, run_lr(S, False), lr_frame_oracle(S))


@pytest.mark.gpu
def test_gpu_cdef_mapping():
    for case in CDEF_WIDTHS:
        S = cdef_case(*case, 620 + case[1])
        assert frame_area_equal(S, run_cdef(S, True), cdef_frame_oracle(S)), case
    for bpc, damp, ssh, ssv in CDEF_STRENGTH:
        S = cdef_case(bpc, 136, 72, ssh, ssv, 630 + bpc + damp, damping=damp, strengths=STRENGTHS)
        assert frame_area_equal(S, run_cdef(S, True), cdef_frame_oracle(S)), (bpc, damp)
    for bpc in (8, 10, 12):
        check_cdef_dir(bpc, None)


@pytest.mark.gpu
def test_gpu_lr_mapping():
    for bpc, types in LR_SGR:
        S = lr_sgr_frame(bpc, types)
        assert picture_equal(S, run_lr(S, True), lr_frame_oracle(S)), types
    for taps in WIENER_EXTREMES:
        S = lr_case(8 if taps[0] < 0 else 12, 130, 57, 1, 1, (6, 5), 640 + taps[2], types=[2], taps=taps)
        assert picture_equal(S, run_lr(S, True), lr_frame_oracle(S)), taps
    for bpc, us in LR_UNITS:
        S = lr_case(bpc, 200, 76, 1, 1, us, 650 + us[0] + us[1])
        assert picture_equal(S, run_lr(S, True), lr_frame_oracle(S)), us
    for W in LR_WIDTHS:
        S = lr_case(8 if W & 1 else 10, W, 40, 1, 1, (6, 6), 660 + W)
        assert picture_equal(S, run_lr(S, True), lr_frame_oracle(S)), W
    S = lr_case(8, 3840, 2160, 1, 1, (8, 7), 670)
    assert picture_equal(S, run_lr(S, True), lr_frame_oracle(S))
