"""Parity tests for the deblocking filter (Dav1dLoopFilterDSPContext + frame driver).

Level 1 follows the reference's tests/checkasm/loopfilter.c: four edge classes (random / long flat /
short flat / normal-or-hev, init_lpf_border :35-91), random sharpness LUT (:122-137), random masks
and levels per segment, 32 luma / 16 chroma segments per call (:194-203).
Frame level: a synthetic picture with random transform tilings; the frame-wide CUDA sweep must equal
dav1d's per-superblock-row driver (the REAL src/lf_apply_tmpl.c through oracle/_ref when present,
and the oracle restatement of it).
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, frame, synth


def clipp(v, bd):
    return max(0, min(bd, v))


def init_border(rng, buf, base, stride, E, Iv, bd):
    b8 = int(np.log2(bd + 1)) - 8
    F = 1 << b8; E <<= b8; Iv <<= b8
    ft = int(rng.integers(0, 4)); ed = int(rng.integers(0, (E + 2) * 4)) - 2 * (E + 2)
    r = lambda: int(rng.integers(0, bd + 1))
    if ft == 0:
        for i in range(-8, 8):
            buf[base + i * stride] = r()
        return
    n = 7 if ft == 1 else 4
    if ft == 1:
        buf[base - 8 * stride] = r(); buf[base + 7 * stride] = r()
    else:
        for i in range(4, 8):
            buf[base - (1 + i) * stride] = r(); buf[base + i * stride] = r()
    buf[base] = r(); buf[base - stride] = clipp(int(buf[base]) + ed, bd)
    for i in range(1, n):
        if ft == 3:
            buf[base - (1 + i) * stride] = clipp(int(buf[base - i * stride]) + int(rng.integers(0, 2 * (Iv + 1))) - (Iv + 1), bd)
            buf[base + i * stride] = clipp(int(buf[base + (i - 1) * stride]) + int(rng.integers(0, 2 * (Iv + 1))) - (Iv + 1), bd)
        else:
            buf[base - (1 + i) * stride] = clipp(int(buf[base - stride]) + int(rng.integers(0, 2 * (F + 1))) - (F + 1), bd)
            buf[base + i * stride] = clipp(int(buf[base]) + int(rng.integers(0, 2 * (F + 1))) - (F + 1), bd)


def ref_lf_tbl(bpc):
    from dav1d_b200 import dsp
    t = (C.c_void_p * 4)()
    (refs.ref().dav1d_loop_filter_dsp_init_8bpc if bpc == 8 else refs.ref().dav1d_loop_filter_dsp_init_16bpc)(t)
    w = dsp.wrap_dsp_table(t, [("f", 4)], {"f": (dsp.LF_PROTO, True)}, bpc > 8, (1 << bpc) - 1)["f"]
    return [[w[0], w[1]], [w[2], w[3]]]


def oracle_lf_tbl(bpc):
    o = refs.oracle(); bd = (1 << bpc) - 1
    P, S = C.c_void_p, C.c_ssize_t

    def mk(pc, d):
        return lambda dst, st, m, l, ls, lut, w: o.oracle_loop_filter_sb(pc, d, P(dst), S(st), P(m), P(l), S(ls), P(lut), bd)
    return [[mk(0, 0), mk(0, 1)], [mk(1, 0), mk(1, 1)]]


def run_lpf_checks(new, chk, bpc, seed, reps=6):
    rng = np.random.default_rng(seed)
    bd = (1 << bpc) - 1
    dt = refs.pixel_dtype(bpc)
    n = 0
    for rep in range(reps):
        for pc, dr, nb, lfidx in ((0, 0, 32, 0), (0, 1, 32, 1), (1, 0, 16, 2), (1, 1, 16, 2)):
            lut = _lib.FilterLUT()
            e, i, sh = synth.filter_lut(int(rng.integers(0, 8)))
            for k in range(64):
                lut.e[k], lut.i[k] = int(e[k]), int(i[k])
            lut.sharp[0], lut.sharp[1] = sh
            for st in range(3 if pc == 0 else 2):
                vmask = (C.c_uint32 * 4)(0, 0, 0, 0)
                l = np.zeros((64, 4), np.uint8)
                for j in range(nb):
                    idx = int(rng.integers(0, st + 2))
                    if idx:
                        vmask[idx - 1] |= 1 << j
                    if dr:
                        l[j][lfidx] = rng.integers(0, 64); l[j + 32][lfidx] = rng.integers(0, 64)
                    else:
                        l[2 * j][lfidx] = rng.integers(0, 64); l[2 * j + 1][lfidx] = rng.integers(0, 64)
                if dr:
                    w, b4s, off = nb * 4, 32, nb * 4 * 8
                else:
                    w, b4s, off = 16, 2, 8
                mem = np.zeros(128 * 16, dt)
                for k in range(4 * nb):
                    x = k >> 2
                    L = (l[32 + x][lfidx] or l[x][lfidx]) if dr else (l[2 * x + 1][lfidx] or l[2 * x][lfidx])
                    init_border(rng, mem, off + k * (1 if dr else 16), nb * 4 if dr else 1, int(lut.e[L]), int(lut.i[L]), bd)
                m1, m2 = mem.copy(), mem.copy()
                isz = mem.itemsize
                lp = l.ctypes.data + ((32 if dr else 1) * 4 + lfidx)
                chk[pc][dr](m1.ctypes.data + off * isz, w * isz, C.addressof(vmask), lp, b4s, C.addressof(lut), nb)
                new[pc][dr](m2.ctypes.data + off * isz, w * isz, C.addressof(vmask), lp, b4s, C.addressof(lut), nb)
                assert np.array_equal(m1, m2), ("lpf", bpc, pc, dr, st)
                assert not np.array_equal(m1, mem) or st == 0
                n += 1
    return n


# ------------------------------------------------------------------ frame level helpers
def lf_frame_oracle(S):
    pic = S["pic"].copy()
    refs.oracle().oracle_lf_frame(S["bd"], C.byref(frame.lf_frame(S, pic.ctypes.data, S["masks"].ctypes.data, S["level"].ctypes.data)))
    return pic


def lf_frame_reference(S, sb128=None):
    """dav1d's own driver; sb128 (default: S's) is the superblock walk order"""
    pic = S["pic"].copy()
    masks = S["masks"].copy()     # the real driver patches masks at tile edges in place
    fr = frame.lf_frame(S, pic.ctypes.data, masks.ctypes.data, S["level"].ctypes.data)
    if sb128 is not None:
        fr.sb128 = sb128
    (refs.ref().refdrv_lf_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_lf_frame_16bpc)(S["bd"], C.byref(fr))
    return pic


def lf_frame_buffers(S, alloc):
    """S's picture, masks and levels placed by `alloc` (keep the handles while the library uses them), and the
    B200LfFrame over them"""
    bufs = [alloc.upload(S[k]) for k in ("pic", "masks", "level")]
    return bufs, frame.lf_frame(S, *(ptr for _, ptr in bufs))


def lf_frame_lib(S, lib, alloc):
    """b200_lf_frame on S's picture, masks and levels placed by `alloc`"""
    bufs, fr = lf_frame_buffers(S, alloc)
    lib.check(lib.b200_lf_frame(S["bd"], C.byref(fr), None), "b200_lf_frame")
    alloc.sync()
    return alloc.download(bufs[0][0], S["pic"])


@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_lpf_vs_reference(bpc):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    assert run_lpf_checks(oracle_lf_tbl(bpc), ref_lf_tbl(bpc), bpc, seed=200 + bpc, reps=12) == 120


@pytest.mark.parametrize("bpc,W,H,ssh,ssv,sb128", [(8, 328, 200, 1, 1, 0), (10, 264, 136, 1, 0, 1), (12, 200, 264, 0, 0, 0),
                                                   (8, 640, 360, 1, 1, 1)])
def test_oracle_lf_frame_vs_reference_driver(bpc, W, H, ssh, ssv, sb128):
    """our restatement of the frame driver against dav1d's real dav1d_loopfilter_sbrow_cols/_rows"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = synth.make_lf_frame(np.random.default_rng(300 + bpc + W), bpc, W, H, ssh, ssv)
    S["sb128"] = sb128
    a, b = lf_frame_oracle(S), lf_frame_reference(S)
    assert np.array_equal(a, b)
    assert (a != S["pic"]).mean() > 0.004      # the filter really did something


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10])
def test_emu_lpf_level1(bpc):
    from dav1d_b200.dsp import LoopFilterDSPContext
    run_lpf_checks(LoopFilterDSPContext(bpc, lib=refs.emu_lib()).loop_filter_sb, oracle_lf_tbl(bpc), bpc, seed=210 + bpc, reps=2)


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 200, 136, 1, 1), (10, 136, 72, 0, 0)])
def test_emu_lf_frame(bpc, W, H, ssh, ssv):
    S = synth.make_lf_frame(np.random.default_rng(320 + bpc), bpc, W, H, ssh, ssv)
    assert np.array_equal(lf_frame_lib(S, *refs.lib_alloc(False)), lf_frame_oracle(S))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_lpf_level1(bpc):
    from dav1d_b200.dsp import LoopFilterDSPContext
    new = LoopFilterDSPContext(bpc).loop_filter_sb
    chk = ref_lf_tbl(bpc) if refs.have_ref() else oracle_lf_tbl(bpc)
    run_lpf_checks(new, chk, bpc, seed=220 + bpc, reps=8)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 1920, 1080, 1, 1), (10, 1280, 720, 1, 0), (12, 648, 360, 0, 0),
                                             (8, 3840, 2160, 1, 1)])
def test_gpu_lf_frame(bpc, W, H, ssh, ssv):
    S = synth.make_lf_frame(np.random.default_rng(330 + bpc + W), bpc, W, H, ssh, ssv)
    exp = lf_frame_reference(S) if refs.have_ref() else lf_frame_oracle(S)
    assert np.array_equal(exp, lf_frame_oracle(S))
    assert np.array_equal(lf_frame_lib(S, *refs.lib_alloc(True)), exp)
