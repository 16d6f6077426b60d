"""Parity tests for film grain (Dav1dFilmGrainDSPContext + dav1d_apply_grain).

Level 1 follows tests/checkasm/filmgrain.c: generate_grain_y/uv over grain_scale_shift, ar_coeff_shift
6..9, lag 0..3, random AR coefficients (:62-75, :112-133); fgy/fguv_32x32xn with random scaling points,
scaling_shift 8..11, clip flag, overlap on/off, random widths / heights / row numbers (:160-215, :280-340).
Frame level: dav1d's real dav1d_apply_grain (through oracle/_ref) against the oracle restatement and the
CUDA prep + apply kernels.
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, frame

GW, GH = 82, 73
LAYOUTS = [(1, 1), (1, 0), (0, 0)]          # table index -> (ss_hor, ss_ver): 420, 422, 444


def rand_fg_data(rng, full=True):
    d = _lib.FilmGrainData()
    d.seed = int(rng.integers(0, 1 << 16))
    d.grain_scale_shift = int(rng.integers(0, 4))
    d.ar_coeff_shift = int(rng.integers(6, 10))
    d.ar_coeff_lag = int(rng.integers(0, 4))
    for i in range(24):
        d.ar_coeffs_y[i] = int(rng.integers(-128, 128))
    for uv in range(2):
        for i in range(25):
            d.ar_coeffs_uv[uv][i] = int(rng.integers(-128, 128))
    d.num_y_points = int(rng.integers(0, 15)) if full else 2 + int(rng.integers(0, 13))

    def points(dst, n):
        pad = 0xff // n if n else 0
        for i in range(n):
            dst[i][0] = min(255, 0xff * i // n + int(rng.integers(0, max(pad, 1))))
            dst[i][1] = int(rng.integers(0, 256))
    points(d.y_points, d.num_y_points)
    d.chroma_scaling_from_luma = int(rng.integers(0, 2))
    for uv in range(2):
        d.num_uv_points[uv] = int(rng.integers(0, 11))
        points(d.uv_points[uv], d.num_uv_points[uv])
        d.uv_mult[uv] = int(rng.integers(-128, 128))
        d.uv_luma_mult[uv] = int(rng.integers(-128, 128))
        d.uv_offset[uv] = int(rng.integers(-256, 256))
    d.scaling_shift = int(rng.integers(8, 12))
    d.overlap_flag = int(rng.integers(0, 2))
    d.clip_to_restricted_range = int(rng.integers(0, 2))
    return d


def fg_ctx(init8, init16, bpc):
    """Bind a film grain function table (the reference's or ours: same prototypes)."""
    t = (C.c_void_p * 8)()
    (init8 if bpc == 8 else init16)(t)
    hbd = bpc > 8
    bd = [(1 << bpc) - 1] if hbd else []
    B = [C.c_int] if hbd else []
    P, S, I = C.c_void_p, C.c_ssize_t, C.c_int
    gy = C.CFUNCTYPE(None, P, P, *B)(t[0])
    guv = [C.CFUNCTYPE(None, P, P, P, C.c_ssize_t, *B)(t[1 + i]) for i in range(3)]
    fgy = C.CFUNCTYPE(None, P, P, S, P, C.c_size_t, P, P, I, I, *B)(t[4])
    fguv = [C.CFUNCTYPE(None, P, P, S, P, C.c_size_t, P, P, I, I, P, S, I, I, *B)(t[5 + i]) for i in range(3)]

    class Ctx:
        pass
    c = Ctx(); c._t = t
    c.generate_grain_y = lambda buf, d: gy(buf.ctypes.data, C.addressof(d), *bd)
    c.generate_grain_uv = [(lambda buf, by, d, uv, _f=f: _f(buf.ctypes.data, by.ctypes.data, C.addressof(d), uv, *bd)) for f in guv]
    c.fgy = lambda dst, src, st, d, pw, sc, lut, bh, row: fgy(dst.ctypes.data, src.ctypes.data, st, C.addressof(d), pw,
                                                               sc.ctypes.data, lut.ctypes.data, bh, row, *bd)
    c.fguv = [(lambda dst, src, st, d, pw, sc, lut, bh, row, luma, ls, uv, is_id, _f=f:
               _f(dst.ctypes.data, src.ctypes.data, st, C.addressof(d), pw, sc.ctypes.data, lut.ctypes.data, bh, row,
                  luma.ctypes.data, ls, uv, is_id, *bd)) for f in fguv]
    return c


def ref_ctx(bpc):
    r = refs.ref()
    return fg_ctx(r.dav1d_film_grain_dsp_init_8bpc, r.dav1d_film_grain_dsp_init_16bpc, bpc)


def oracle_ctx(bpc):
    o = refs.oracle(); bd = (1 << bpc) - 1
    P = C.c_void_p

    class Ctx:
        pass
    c = Ctx()
    c.generate_grain_y = lambda buf, d: o.oracle_fg_generate_grain(P(buf.ctypes.data), None, C.byref(d), -1, 0, 0, bd)
    c.generate_grain_uv = [(lambda buf, by, d, uv, sx=sx, sy=sy:
                            o.oracle_fg_generate_grain(P(buf.ctypes.data), P(by.ctypes.data), C.byref(d), uv, sx, sy, bd))
                           for sx, sy in LAYOUTS]
    c.fgy = lambda dst, src, st, d, pw, sc, lut, bh, row: o.oracle_fgy_32x32xn(
        P(dst.ctypes.data), P(src.ctypes.data), C.c_ssize_t(st), C.byref(d), C.c_size_t(pw), P(sc.ctypes.data),
        P(lut.ctypes.data), bh, row, bd)
    c.fguv = [(lambda dst, src, st, d, pw, sc, lut, bh, row, luma, ls, uv, is_id, sx=sx, sy=sy: o.oracle_fguv_32x32xn(
        P(dst.ctypes.data), P(src.ctypes.data), C.c_ssize_t(st), C.byref(d), C.c_size_t(pw), P(sc.ctypes.data),
        P(lut.ctypes.data), bh, row, P(luma.ctypes.data), C.c_ssize_t(ls), uv, is_id, sx, sy, bd)) for sx, sy in LAYOUTS]
    return c


def lib_ctx(lib, bpc):
    return fg_ctx(lib.b200_film_grain_dsp_init_8bpc, lib.b200_film_grain_dsp_init_16bpc, bpc)


def lut_dtype(bpc):
    return np.int8 if bpc == 8 else np.int16


def check_level1(ctx_a, ctx_b, bpc, iters, seed):
    """generate_grain_* and fg*_32x32xn of two tables against each other on checkasm-style inputs."""
    rng = np.random.default_rng(seed)
    bd = (1 << bpc) - 1
    ldt, pdt = lut_dtype(bpc), refs.pixel_dtype(bpc)
    px = np.dtype(pdt).itemsize
    n = 0
    for it in range(iters):
        d = rand_fg_data(rng, full=False)
        la = np.zeros((GH + 1, GW), ldt); lb = np.zeros_like(la)
        ctx_a.generate_grain_y(la, d); ctx_b.generate_grain_y(lb, d)
        assert np.array_equal(la[:GH], lb[:GH]), "generate_grain_y"
        for li, (sx, sy) in enumerate(LAYOUTS):
            cw, ch = (44 if sx else GW), (38 if sy else GH)
            for uv in range(2):
                ua = np.zeros((GH + 1, GW), ldt); ub = np.zeros_like(ua)
                ctx_a.generate_grain_uv[li](ua, la, d, uv); ctx_b.generate_grain_uv[li](ub, la, d, uv)
                assert np.array_equal(ua[:ch, :cw], ub[:ch, :cw]), ("generate_grain_uv", li, uv)
                n += 1
        # luma strips
        scaling = rng.integers(0, 256, 4096).astype(np.uint8)
        w = int(rng.integers(1, 129)) if it & 1 else 128
        bh = int(rng.integers(1, 33)) if it & 2 else 32
        row = int(rng.integers(0, 0x800)) if it & 4 else int(rng.integers(0, 3))
        st = 160
        src = rng.integers(0, bd + 1, (32, st)).astype(pdt)
        da = src.copy(); db = src.copy()
        ctx_a.fgy(da, src, st * px, d, w, scaling, la, bh, row); ctx_b.fgy(db, src, st * px, d, w, scaling, la, bh, row)
        assert np.array_equal(da, db), ("fgy", w, bh, row)
        for li, (sx, sy) in enumerate(LAYOUTS):
            for uv in range(2):
                is_id = int(rng.integers(0, 2))
                ulut = np.zeros((GH + 1, GW), ldt)
                ctx_a.generate_grain_uv[li](ulut, la, d, uv)
                cw = (w + sx) >> sx
                cbh = (bh + sy) >> sy
                luma = rng.integers(0, bd + 1, (32, st)).astype(pdt)
                csrc = rng.integers(0, bd + 1, (32, st)).astype(pdt)
                da = csrc.copy(); db = csrc.copy()
                ctx_a.fguv[li](da, csrc, st * px, d, cw, scaling, ulut, cbh, row, luma, st * px, uv, is_id)
                ctx_b.fguv[li](db, csrc, st * px, d, cw, scaling, ulut, cbh, row, luma, st * px, uv, is_id)
                assert np.array_equal(da, db), ("fguv", li, uv, w, bh, row)
                n += 1
    return n


@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_level1_vs_reference(bpc):
    if not refs.have_ref():
        pytest.skip("oracle/_ref not built")
    assert check_level1(ref_ctx(bpc), oracle_ctx(bpc), bpc, 16, 100 + bpc) > 0


# ---------------------------------------------------------------- whole picture
def make_fg_frame(rng, w, h, ss, bpc, d=None):
    sx, sy = ss
    bd = (1 << bpc) - 1
    pdt = refs.pixel_dtype(bpc)
    st0 = (w + 63) & ~63
    st1 = st0 >> sx if sx else st0
    st1 = (st1 + 31) & ~31
    ch = (h + sy) >> sy
    off = [0, st0 * (h + 1), st0 * (h + 1) + st1 * (ch + 1)]
    total = off[2] + st1 * (ch + 1)
    pic = rng.integers(0, bd + 1, total).astype(pdt)
    is_id = int(rng.integers(0, 2))
    fr = frame.fg_frame(dict(off=off, stride=[st0, st1, st1], W=w, H=h, ss_hor=sx, ss_ver=sy,
                             fg=d if d is not None else rand_fg_data(rng)), None, None)
    fr.is_id = is_id
    return fr, pic


class RefFg(C.Structure):
    _fields_ = [(n, t) for n, t in _lib.FgFrame._fields_ if n != "scratch"]


def run_ref_frame(fr, pic, bpc):
    out = np.zeros_like(pic)
    rf = RefFg()
    C.memmove(C.addressof(rf), C.addressof(fr), C.sizeof(RefFg))
    rf.in_ = pic.ctypes.data; rf.out = out.ctypes.data
    f = refs.ref().refdrv_fg_frame_8bpc if bpc == 8 else refs.ref().refdrv_fg_frame_16bpc
    f.restype = None
    f(C.c_int((1 << bpc) - 1), C.byref(rf))
    return out


def run_oracle_frame(fr, pic, bpc):
    out = np.zeros_like(pic)
    rf = RefFg()
    C.memmove(C.addressof(rf), C.addressof(fr), C.sizeof(RefFg))
    rf.in_ = pic.ctypes.data; rf.out = out.ctypes.data
    o = refs.oracle()
    o.oracle_fg_apply_frame.restype = None
    o.oracle_fg_apply_frame(C.c_int((1 << bpc) - 1), C.byref(rf))
    return out


def planes_equal(fr, a, b):
    for pl in range(3):
        sx = fr.ss_hor if pl else 0; sy = fr.ss_ver if pl else 0
        pw, ph = (fr.w + sx) >> sx, (fr.h + sy) >> sy
        st = fr.stride[pl]
        va = a[fr.plane_off[pl]: fr.plane_off[pl] + st * ph].reshape(ph, st)[:, :pw]
        vb = b[fr.plane_off[pl]: fr.plane_off[pl] + st * ph].reshape(ph, st)[:, :pw]
        if not np.array_equal(va, vb):
            ys, xs = np.nonzero(va != vb)
            return False, (pl, int(ys[0]), int(xs[0]), int(va[ys[0], xs[0]]), int(vb[ys[0], xs[0]]), len(ys))
    return True, None


FRAME_CASES = [(176, 144, (1, 1), 8), (97, 67, (1, 1), 8), (130, 70, (1, 0), 8), (96, 40, (0, 0), 8),
               (176, 144, (1, 1), 10), (99, 65, (1, 1), 10), (130, 33, (1, 0), 12), (70, 96, (0, 0), 12)]


@pytest.mark.parametrize("w,h,ss,bpc", FRAME_CASES)
def test_oracle_frame_vs_reference(w, h, ss, bpc):
    if not refs.have_ref():
        pytest.skip("oracle/_ref not built")
    rng = np.random.default_rng(w * 7 + h + bpc)
    for it in range(4):
        fr, pic = make_fg_frame(rng, w, h, ss, bpc)
        a = run_ref_frame(fr, pic, bpc)
        b = run_oracle_frame(fr, pic, bpc)
        ok, where = planes_equal(fr, a, b)
        assert ok, where


def run_lib_frame(lib, fr, pic, bpc, alloc):
    """alloc(nbytes) -> (device/host pointer owner, address); copies are the caller's (emu: plain numpy)."""
    raise NotImplementedError


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_level1_vs_oracle(bpc):
    lib = refs.emu_lib()
    assert check_level1(oracle_ctx(bpc), lib_ctx(lib, bpc), bpc, 6, 300 + bpc) > 0


@pytest.mark.emu
@pytest.mark.parametrize("w,h,ss,bpc", FRAME_CASES)
def test_emu_frame_vs_oracle(w, h, ss, bpc):
    lib = refs.emu_lib()
    rng = np.random.default_rng(w * 11 + h + bpc)
    for it in range(2):
        fr, pic = make_fg_frame(rng, w, h, ss, bpc)
        ref_out = run_oracle_frame(fr, pic, bpc)
        out = np.zeros_like(pic)
        scratch = np.zeros(256 * 1024, np.uint8)
        fr.in_ = pic.ctypes.data; fr.out = out.ctypes.data; fr.scratch = scratch.ctypes.data
        assert lib.b200_fg_apply_frame((1 << bpc) - 1, C.byref(fr), None) == 0, lib.b200_last_error()
        ok, where = planes_equal(fr, ref_out, out)
        assert ok, where


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_level1_vs_oracle(bpc):
    lib = _lib.get_lib()
    assert check_level1(oracle_ctx(bpc), lib_ctx(lib, bpc), bpc, 6, 500 + bpc) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,ss,bpc", FRAME_CASES + [(3840, 2160, (1, 1), 10), (1920, 1080, (1, 1), 8)])
def test_gpu_frame_vs_oracle(w, h, ss, bpc):
    import torch
    lib = _lib.get_lib()
    rng = np.random.default_rng(w * 13 + h + bpc)
    fr, pic = make_fg_frame(rng, w, h, ss, bpc)
    ref_out = run_oracle_frame(fr, pic, bpc)
    tdt = torch.uint8 if bpc == 8 else torch.int16
    d_in = torch.from_numpy(pic.view(np.uint8 if bpc == 8 else np.int16)).cuda()
    d_out = torch.zeros_like(d_in)
    scratch = torch.zeros(256 * 1024, dtype=torch.uint8, device="cuda")
    fr.in_ = d_in.data_ptr(); fr.out = d_out.data_ptr(); fr.scratch = scratch.data_ptr()
    assert lib.b200_fg_apply_frame((1 << bpc) - 1, C.byref(fr), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().view(pic.dtype)
    ok, where = planes_equal(fr, ref_out, out)
    assert ok, where
