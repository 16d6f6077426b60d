"""Parity tests for CDEF (Dav1dCdefDSPContext + frame driver).

Level 1 follows tests/checkasm/cdef.c: 8 directions x 16 edge-flag combinations x {sec, pri, both},
under/overflow fills (init_tmp :42-53), random strengths / damping (:80-84); cdef_dir on 8x8 (:106-131).
Frame level: the out-of-place CUDA sweep against dav1d's real in-place dav1d_cdef_brow
(through oracle/_ref) and the oracle restatement.
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import frame, synth


def init_tmp(rng, n, bd, dt):
    ft = int(rng.integers(0, 8))
    if ft == 0:
        return rng.integers(0, 2, n).astype(dt)
    if ft == 1:
        return (bd - rng.integers(0, 2, n)).astype(dt)
    return rng.integers(0, bd + 1, n).astype(dt)


def ref_cdef(bpc):
    from dav1d_b200 import dsp
    t = (C.c_void_p * 4)()
    (refs.ref().dav1d_cdef_dsp_init_8bpc if bpc == 8 else refs.ref().dav1d_cdef_dsp_init_16bpc)(t)
    hbd = bpc > 8
    bd = [(1 << bpc) - 1] if hbd else []
    P, S, I = C.c_void_p, C.c_ssize_t, C.c_int
    dir_f = C.CFUNCTYPE(I, P, S, C.POINTER(C.c_uint), *([I] if hbd else []))(t[0])
    fbs = [C.CFUNCTYPE(None, P, S, P, P, P, I, I, I, I, I, *([I] if hbd else []))(t[1 + i]) for i in range(3)]

    class Ctx:
        pass
    c = Ctx(); c._t = t

    def dir_(img, st):
        v = C.c_uint(0)
        return dir_f(img.ctypes.data, st, C.byref(v), *bd), v.value
    c.dir = dir_
    c.fb = [(lambda d, st, l, tp, bt, pri, sec, dr, damp, e, _f=f:
             _f(d.ctypes.data, st, l.ctypes.data, tp.ctypes.data, bt.ctypes.data, pri, sec, dr, damp, e, *bd)) for f in fbs]
    return c


def oracle_cdef(bpc):
    o = refs.oracle(); bd = (1 << bpc) - 1
    P, S = C.c_void_p, C.c_ssize_t

    class Ctx:
        pass
    c = Ctx()

    def dir_(img, st):
        v = C.c_uint(0)
        return o.oracle_cdef_dir(P(img.ctypes.data), S(st), C.byref(v), bd), v.value
    c.dir = dir_
    dims = [(8, 8), (4, 8), (4, 4)]
    c.fb = [(lambda d, st, l, tp, bt, pri, sec, dr, damp, e, wh=wh:
             o.oracle_cdef_fb(P(d.ctypes.data), S(st), P(l.ctypes.data), P(tp.ctypes.data), P(bt.ctypes.data),
                              pri, sec, dr, damp, wh[0], wh[1], e, bd)) for wh in dims]
    return c


def run_cdef_checks(new, chk, bpc, seed, reps=1):
    rng = np.random.default_rng(seed)
    bd = (1 << bpc) - 1
    b8 = bpc - 8
    dt = refs.pixel_dtype(bpc)
    n = 0
    for _ in range(reps):
        for i, (w, h) in enumerate([(8, 8), (4, 8), (4, 4)]):
            for s in (1, 2, 3):
                for d in range(8):
                    for edges in range(16):
                        src = init_tmp(rng, 16 * 10 + 16, bd, dt)
                        top = init_tmp(rng, 16 * 2 + 16, bd, dt)
                        bot = init_tmp(rng, 16 * 2 + 16, bd, dt)
                        left = init_tmp(rng, 16, bd, dt)
                        pri = (1 + int(rng.integers(0, 15))) << b8 if s & 2 else 0
                        sec = 1 << (int(rng.integers(0, 3)) + b8) if s & 1 else 0
                        damp = 3 + int(rng.integers(0, 4)) + b8 - int(w == 4 or int(rng.integers(0, 2)))
                        a, b = src.copy(), src.copy()
                        chk.fb[i](a[8:], 16 * a.itemsize, left, top[8:], bot[8:], pri, sec, d, damp, edges)
                        new.fb[i](b[8:], 16 * b.itemsize, left, top[8:], bot[8:], pri, sec, d, damp, edges)
                        assert np.array_equal(a, b), ("cdef fb", bpc, w, h, s, d, edges, pri, sec, damp)
                        n += 1
        for k in range(24):
            img = init_tmp(rng, 64, bd, dt)
            if k % 3 == 0:   # structured content so that every direction can win
                yy, xx = np.mgrid[0:8, 0:8]
                ang = rng.random() * np.pi
                img = (np.clip(((np.cos(ang) * xx + np.sin(ang) * yy) * (bd / 10.0)) % bd, 0, bd)).astype(dt).reshape(-1)
            assert chk.dir(img, 8 * img.itemsize) == new.dir(img, 8 * img.itemsize), ("cdef dir", bpc, k)
            n += 1
    return n


def make_cdef_frame(rng, bpc, W, H, ssh, ssv):
    S = synth.make_lf_frame(rng, bpc, W, H, ssh, ssv, smooth=True)
    S["bw"], S["bh"] = S["w4"], S["h4"]
    S["damping"], S["y_strength"], S["uv_strength"] = synth.make_cdef_params(rng, S["bw"], S["bh"], S["sb128w"], S["masks"])
    return S


def cdef_frame_oracle(S):
    dst = S["pic"].copy()
    fr = frame.cdef_frame(S, S["pic"].ctypes.data, dst.ctypes.data, S["masks"].ctypes.data)
    refs.oracle().oracle_cdef_frame(S["bd"], C.byref(fr))
    return dst


def cdef_frame_reference(S):
    pic = S["pic"].copy()
    fr = frame.cdef_frame(S, pic.ctypes.data, None, S["masks"].ctypes.data)
    (refs.ref().refdrv_cdef_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_cdef_frame_16bpc)(S["bd"], C.byref(fr))
    return pic


def cdef_frame_lib(S, lib, alloc):
    """b200_cdef_frame on S's picture and masks placed by `alloc`"""
    src, dst, mask = alloc.upload(S["pic"]), alloc.zeros(S["pic"].nbytes), alloc.upload(S["masks"])
    lib.check(lib.b200_cdef_frame(S["bd"], C.byref(frame.cdef_frame(S, src[1], dst[1], mask[1])), None), "b200_cdef_frame")
    alloc.sync()
    return alloc.download(dst[0], S["pic"])


def frame_area_equal(S, a, b):
    """compare the bw x bh picture area of all planes (padding outside it is not defined output)"""
    for pl in range(3):
        sh, sv = (S["ss_hor"], S["ss_ver"]) if pl else (0, 0)
        w, h = (S["bw"] * 4) >> sh, (S["bh"] * 4) >> sv
        o, st = S["off"][pl], S["stride"][pl]
        va = a[o:o + st * h].reshape(h, st)[:, :w]
        vb = b[o:o + st * h].reshape(h, st)[:, :w]
        if not np.array_equal(va, vb):
            return False
    return True


@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_cdef_vs_reference(bpc):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    assert run_cdef_checks(oracle_cdef(bpc), ref_cdef(bpc), bpc, seed=400 + bpc, reps=2) > 2000


@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 328, 200, 1, 1), (10, 264, 136, 1, 0), (12, 200, 264, 0, 0), (8, 644, 364, 1, 1)])
def test_oracle_cdef_frame_vs_reference_driver(bpc, W, H, ssh, ssv):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = make_cdef_frame(np.random.default_rng(410 + bpc + W), bpc, W, H, ssh, ssv)
    a, b = cdef_frame_oracle(S), cdef_frame_reference(S)
    assert frame_area_equal(S, a, b)
    assert (a != S["pic"]).mean() > 0.05


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10])
def test_emu_cdef_level1(bpc):
    from dav1d_b200.dsp import CdefDSPContext
    run_cdef_checks(CdefDSPContext(bpc, lib=refs.emu_lib()), oracle_cdef(bpc), bpc, seed=420 + bpc)


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 136, 72, 1, 1), (10, 72, 72, 1, 0), (8, 72, 40, 0, 0), (8, 68, 44, 1, 1), (12, 140, 76, 1, 1),
                                                (12, 68, 36, 0, 0), (10, 204, 100, 1, 1)])
def test_emu_cdef_frame(bpc, W, H, ssh, ssv):
    S = make_cdef_frame(np.random.default_rng(430 + bpc + W), bpc, W, H, ssh, ssv)
    assert frame_area_equal(S, cdef_frame_lib(S, *refs.lib_alloc(False)), cdef_frame_oracle(S))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_cdef_level1(bpc):
    from dav1d_b200.dsp import CdefDSPContext
    chk = ref_cdef(bpc) if refs.have_ref() else oracle_cdef(bpc)
    run_cdef_checks(CdefDSPContext(bpc), chk, bpc, seed=440 + bpc)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 1920, 1080, 1, 1), (10, 1280, 720, 1, 0), (12, 648, 360, 0, 0), (8, 3840, 2160, 1, 1)])
def test_gpu_cdef_frame(bpc, W, H, ssh, ssv):
    S = make_cdef_frame(np.random.default_rng(450 + bpc + W), bpc, W, H, ssh, ssv)
    exp = cdef_frame_reference(S) if refs.have_ref() else cdef_frame_oracle(S)
    got = cdef_frame_lib(S, *refs.lib_alloc(True))
    assert frame_area_equal(S, got, exp)
    assert frame_area_equal(S, got, cdef_frame_oracle(S))
