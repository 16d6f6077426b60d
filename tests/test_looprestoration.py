"""Parity tests for loop restoration (Dav1dLoopRestorationDSPContext + frame driver).

Level 1 follows tests/checkasm/looprestoration.c: checkerboard-plus-noise input (init_tmp :41-54), random legal
Wiener taps (:73-83), SGR with dav1d_sgr_params[14 / 10 / 0] (:141-152), all 16 edge combinations, w = 256 /
h = 64 when HAVE_RIGHT / HAVE_BOTTOM else random <= 384 x 64.
Frame level: out-of-place CUDA restoration against dav1d's real dav1d_copy_lpf + dav1d_lr_sbrow (oracle/_ref)
and against the oracle restatement.
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import frame, synth


class LrParams(C.Union):
    class Sgr(C.Structure):
        _fields_ = [("s0", C.c_uint32), ("s1", C.c_uint32), ("w0", C.c_int16), ("w1", C.c_int16)]
    _fields_ = [("filter", (C.c_int16 * 8) * 2), ("sgr", Sgr)]


def aligned_params():
    raw = np.zeros(96, np.uint8)
    return raw, LrParams.from_address(raw.ctypes.data + (-raw.ctypes.data) % 32)


def init_tmp(rng, w, h, bd, dt):
    nm = bd >> 4
    xo, yo = int(rng.integers(0, 8)), int(rng.integers(0, 8))
    xs, ys = np.meshgrid(np.arange(w), np.arange(h))
    return ((np.where(((xs + xo) ^ (ys + yo)) & 8, bd, 0)) ^ rng.integers(0, nm + 1, (h, w))).astype(dt)


def ref_lr(bpc):
    from dav1d_b200 import dsp
    t = (C.c_void_p * 5)()
    (refs.ref().dav1d_loop_restoration_dsp_init_8bpc if bpc == 8 else refs.ref().dav1d_loop_restoration_dsp_init_16bpc)(t, bpc)
    w = dsp.wrap_dsp_table(t, [("wiener", 2), ("sgr", 3)], {"wiener": (dsp.LR_PROTO, True), "sgr": (dsp.LR_PROTO, True)},
                           bpc > 8, (1 << bpc) - 1)

    class Ctx:
        pass
    c = Ctx(); c._t = t; c.wiener, c.sgr = w["wiener"], w["sgr"]
    return c


def oracle_lr(bpc):
    o = refs.oracle(); bd = (1 << bpc) - 1
    P, S = C.c_void_p, C.c_ssize_t

    def a(x):
        return x.ctypes.data if isinstance(x, np.ndarray) else x

    class Ctx:
        pass
    c = Ctx()
    wf = lambda d, st, l, lpf, w, h, p, e: o.oracle_wiener(P(a(d)), S(st), P(a(l)), P(a(lpf)), w, h, P(p), e, bd)
    c.wiener = [wf, wf]

    def mk(mode):
        def f(d, st, l, lpf, w, h, p, e):
            pr = LrParams.from_address(p)
            o.oracle_sgr(mode, P(a(d)), S(st), P(a(l)), P(a(lpf)), w, h, C.c_uint(pr.sgr.s0), C.c_uint(pr.sgr.s1),
                         int(pr.sgr.w0), int(pr.sgr.w1), e, bd)
        return f
    c.sgr = [mk(0), mk(1), mk(2)]
    return c


def run_lr_checks(new, chk, bpc, seed, reps=2, edge_list=range(16)):
    rng = np.random.default_rng(seed)
    bd = (1 << bpc) - 1
    hbd = bpc > 8
    dt = refs.pixel_dtype(bpc)
    n = 0
    for _ in range(reps):
        for kind in range(5):
            raw, pr = aligned_params()
            if kind < 2:
                f = np.zeros((2, 8), np.int64)
                for a_ in range(2):
                    f[a_, 0] = f[a_, 6] = 0 if kind else int(rng.integers(0, 16)) - 5
                    f[a_, 1] = f[a_, 5] = int(rng.integers(0, 32)) - 23
                    f[a_, 2] = f[a_, 4] = int(rng.integers(0, 64)) - 17
                f[0, 3] = -(f[0, 0] + f[0, 1] + f[0, 2]) * 2 + (128 if hbd else 0)
                f[1, 3] = 128 - (f[1, 0] + f[1, 1] + f[1, 2]) * 2
                for a_ in range(2):
                    for b_ in range(8):
                        pr.filter[a_][b_] = int(f[a_, b_])
                fn_new, fn_chk = new.wiener[kind], chk.wiener[kind]
            else:
                s0, s1 = synth.SGR_PARAMS[[14, 10, 0][kind - 2]]
                pr.sgr.s0, pr.sgr.s1 = s0, s1
                w0 = (int(rng.integers(0, 128)) - 96) if s0 else 0
                pr.sgr.w0 = w0
                pr.sgr.w1 = ((160 - int(rng.integers(0, 128))) if s1 else 33) - w0
                fn_new, fn_chk = new.sgr[kind - 2], chk.sgr[kind - 2]
            base_w, base_h = 1 + int(rng.integers(0, 384)), 1 + int(rng.integers(0, 64))
            canvas = np.zeros((64 + 16, 384 + 64), dt); canvas[8:72, 28:28 + 388] = init_tmp(rng, 388, 64, bd, dt)
            hedge = np.zeros((8, 384 + 64), dt); hedge[:, 28:28 + 388] = init_tmp(rng, 388, 8, bd, dt)
            left = init_tmp(rng, 4, 64, bd, dt)
            for edges in edge_list:
                w = 256 if edges & 2 else base_w
                h = 64 if edges & 8 else base_h
                a, b = canvas.copy(), canvas.copy()
                fn_chk(a[8:, 32:], a.strides[0], left, hedge[:, 32:], w, h, C.addressof(pr), edges)
                fn_new(b[8:, 32:], b.strides[0], left, hedge[:, 32:], w, h, C.addressof(pr), edges)
                # the reference may write past w up to the unit alignment (src/looprestoration.h:57-63): compare w x h
                assert np.array_equal(a[8:8 + h, 32:32 + w], b[8:8 + h, 32:32 + w]), ("lr", bpc, kind, edges, w, h)
                assert np.array_equal(a[:8], b[:8]) and np.array_equal(a[8 + h:], b[8 + h:]) and np.array_equal(a[:, :32], b[:, :32])
                n += 1
    return n


# ------------------------------------------------------------------ frame level
def make_lr_frame(rng, bpc, W, H, ssh, ssv, sb128, us, rp):
    S = synth.make_lf_frame(rng, bpc, W, H, ssh, ssv)
    S["dbl"] = S["pic"]
    S["cdef"] = (S["pic"].astype(np.int32) ^ rng.integers(0, 4, S["pic"].shape)).clip(0, S["bd"]).astype(S["pic"].dtype)
    S["lr_mask"] = synth.make_lr_params(rng, W, H)
    S["sb128"], S["us"], S["rp"] = sb128, us, rp
    return S


def lr_frame_oracle(S):
    dst = np.zeros_like(S["cdef"])
    fr = frame.lr_frame(S, S["cdef"].ctypes.data, S["dbl"].ctypes.data, dst.ctypes.data, S["lr_mask"].ctypes.data)
    refs.oracle().oracle_lr_frame(S["bd"], C.byref(fr))
    return dst


def lr_frame_reference(S):
    c2 = S["cdef"].copy()
    fr = frame.lr_frame(S, c2.ctypes.data, S["dbl"].ctypes.data, None, S["lr_mask"].ctypes.data)
    (refs.ref().refdrv_lr_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_lr_frame_16bpc)(S["bd"], C.byref(fr))
    return c2


def lr_frame_lib(S, lib, alloc):
    """b200_lr_frame on S's CDEF and deblocked pictures and restoration units placed by `alloc`"""
    cdef, dbl, dst, lrm = alloc.upload(S["cdef"]), alloc.upload(S["dbl"]), alloc.zeros(S["cdef"].nbytes), alloc.upload(S["lr_mask"])
    lib.check(lib.b200_lr_frame(S["bd"], C.byref(frame.lr_frame(S, cdef[1], dbl[1], dst[1], lrm[1])), None), "b200_lr_frame")
    alloc.sync()
    return alloc.download(dst[0], S["cdef"])


def picture_equal(S, a, b):
    for pl in range(3):
        sh, sv = (S["ss_hor"], S["ss_ver"]) if pl else (0, 0)
        w, h = (S["W"] + sh) >> sh, (S["H"] + sv) >> sv
        o, st = S["off"][pl], S["stride"][pl]
        if not np.array_equal(a[o:o + st * h].reshape(h, st)[:, :w], b[o:o + st * h].reshape(h, st)[:, :w]):
            return False
    return True


FRAME_CASES = [(8, 328, 200, 1, 1, 0, (6, 6), 7), (8, 328, 200, 1, 1, 0, (7, 6), 7), (10, 264, 136, 1, 0, 1, (7, 7), 5),
               (12, 200, 264, 0, 0, 0, (8, 8), 7), (8, 644, 364, 1, 1, 1, (8, 7), 7), (8, 130, 57, 1, 1, 0, (6, 5), 7),
               (8, 97, 121, 1, 1, 0, (6, 6), 3)]


@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_lr_vs_reference(bpc):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    assert run_lr_checks(oracle_lr(bpc), ref_lr(bpc), bpc, seed=500 + bpc, reps=3) == 240


@pytest.mark.parametrize("case", FRAME_CASES)
def test_oracle_lr_frame_vs_reference_driver(case):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = make_lr_frame(np.random.default_rng(510 + case[1]), *case)
    a, b = lr_frame_oracle(S), lr_frame_reference(S)
    assert picture_equal(S, a, b)
    assert not picture_equal(S, a, S["cdef"])


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 12])
def test_emu_lr_level1(bpc):
    from dav1d_b200.dsp import LoopRestorationDSPContext
    run_lr_checks(LoopRestorationDSPContext(bpc, lib=refs.emu_lib()), oracle_lr(bpc), bpc, seed=520 + bpc, reps=1,
                  edge_list=(0, 5, 10, 15, 7, 12))


@pytest.mark.emu
@pytest.mark.parametrize("case", [FRAME_CASES[0], FRAME_CASES[2], FRAME_CASES[5]])
def test_emu_lr_frame(case):
    S = make_lr_frame(np.random.default_rng(530 + case[1]), *case)
    assert picture_equal(S, lr_frame_lib(S, *refs.lib_alloc(False)), lr_frame_oracle(S))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_lr_level1(bpc):
    from dav1d_b200.dsp import LoopRestorationDSPContext
    chk = ref_lr(bpc) if refs.have_ref() else oracle_lr(bpc)
    run_lr_checks(LoopRestorationDSPContext(bpc), chk, bpc, seed=540 + bpc, reps=2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FRAME_CASES + [(8, 1920, 1080, 1, 1, 0, (6, 6), 7), (10, 3840, 2160, 1, 1, 1, (8, 7), 7)])
def test_gpu_lr_frame(case):
    S = make_lr_frame(np.random.default_rng(550 + case[1]), *case)
    exp = lr_frame_reference(S) if refs.have_ref() else lr_frame_oracle(S)
    assert picture_equal(S, lr_frame_lib(S, *refs.lib_alloc(True)), exp)
