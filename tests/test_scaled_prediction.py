"""Scaled prediction and super-resolution upscaling at frame scale, against dav1d's own C functions.

`b200_mc_scaled_batch` runs every prediction from a reference of another size, and `b200_resize_frame` upscales
every plane of a super-resolution frame. The Level-1 checks of test_mc.py call them one block (or one strip) at a
time on exactly the window the block reads, so the kernels' edge clamping never changes a value there, only the
frame's own plane geometry is used, and the resize grid-stride loop never wraps. Here:

- whole batches of scaled records, with 2 to 8 references of their own sizes (1/16 to 2 times the frame), strides
  and plane offsets (`B200McFrame.ref_geom`, `scaled_mask`), all three ops (put, prep, put into the OBMC pixel
  scratch) and windows on every side of and across every edge of the reference, against what dav1d's mc() does for
  a scaled reference (reference src/recon_tmpl.c:991-1046: emu_edge into a 320-sample buffer, then
  mc_scaled / mct_scaled);
- whole three-plane pictures through the resize stage with the parameters dav1d derives
  (reference src/decode.c:3530-3540), against dav1d's resize run once per plane over all its rows;
- full-size super-resolution and scaled-reference streams through the hooked decoder on the H100, byte for byte
  against stock dav1d.

The C side is the reference build (oracle/_ref) where it exists and the oracle's restatement otherwise.
"""
import ctypes as C

import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, obu, stream
from test_stream import _check

EMU_W = 320                        # dav1d's emu_edge scratch is 320 samples wide (t->scratch.emu_edge)
EMU_ROWS = ((127 * 2048 + 1023) >> 10) + 1 + 7    # the tallest window a 128-row block at step 2048 reads
STEPS = (64, 511, 512, 1024, 2048)
SIZES = (2, 4, 8, 16, 32, 64, 128)
LAYOUTS = {"420": (1, 1), "422": (1, 0), "444": (0, 0), "400": (1, 0)}


def checker(bpc):
    return refs.ref_mc_ctx(bpc) if refs.have_ref() else refs.oracle_mc_ctx(bpc)


def _align(v, a):
    return (v + a - 1) // a * a


def picture_geom(rng, w, h, layout):
    """Plane geometry of a picture of w x h, laid out as the hooks lay out dav1d's pictures: planes back to back,
    rows rounded up to 128, 128-aligned strides (plus 64 bytes where dav1d adds them) and some extra padding of
    the picture's own."""
    ss_hor, ss_ver = LAYOUTS[layout]
    rows = _align(h, 128)
    s0 = _align(w, 128) + int(rng.choice([0, 32, 64, 96]))
    s1 = s0 if layout == "400" else (s0 >> ss_hor) + int(rng.choice([0, 16, 32]))
    off = [0, s0 * rows, s0 * rows + s1 * (rows >> ss_ver)]
    return dict(off=off, stride=[s0, s1, s1],
                w=[w] + [(w + ss_hor) >> ss_hor] * 2, h=[h] + [(h + ss_ver) >> ss_ver] * 2,
                total=off[1] if layout == "400" else off[2] + s1 * (rows >> ss_ver))


def _cdiv(a, b):
    """C integer division (truncates toward zero)"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def resize_params(in_w, out_w):
    """The super-resolution step and start phase for upscaling in_w samples to out_w, as dav1d computes them
    (reference src/decode.c scale_fac / get_upscale_x0): returns (dx, mx0)."""
    dx = ((in_w << 14) + (out_w >> 1)) // out_w
    err = out_w * dx - (in_w << 14)
    x0 = _cdiv(-((out_w - in_w) << 13) + (out_w >> 1), out_w) + 128 - _cdiv(err, 2)
    return dx, x0 & 0x3fff


def scale_mv(val, scale):
    """dav1d's scale_mv (reference src/recon_tmpl.c:996-999)"""
    tmp = val * scale + (scale - 0x4000) * 8
    return (1 if tmp >= 0 else -1) * ((abs(tmp) + 128) >> 8) + 32


def _window_pos(rng, extent, size):
    """a window start for `extent` samples against a plane of `size`: wholly before / after it, across either edge,
    or inside it (8-tap filters read 3 before and 4 after)"""
    kind = int(rng.integers(0, 5))
    if kind == 0:
        return -(extent + 4 + int(rng.integers(0, 40)))
    if kind == 1:
        return size + 3 + int(rng.integers(0, 40))
    if kind == 2:
        return int(rng.integers(-extent - 3, 3))
    if kind == 3:
        return int(rng.integers(size - extent - 3, size + 3))
    return int(rng.integers(3, max(4, size - extent - 3)))


def make_scaled_batch(rng, bpc, layout, W, H, n_rec):
    """A batch of B200McScaledBlock records as the hooks emit them (b200_hooks_tmpl.c emit_mc, scaled branch), plus a
    share of arbitrary records at the extreme steps and phases. Returns host-side state."""
    bd = (1 << bpc) - 1
    dt = refs.pixel_dtype(bpc)
    ss_hor, ss_ver = LAYOUTS[layout]
    n_planes = 1 if layout == "400" else 3
    frame = picture_geom(rng, W, H, layout)
    n_refs = int(rng.integers(2, 9))
    # reference 0 has the frame's size (the frame geometry, scaled_mask bit clear); the others their own size from
    # W/16 to 2W (odd sizes included), the extremes drawn more often
    ref_sz, geoms, mask = [(W, H)], [frame], 0
    for k in range(1, n_refs):
        def draw(n):
            lo, hi = -(-n // 16), 2 * n
            return int(rng.choice([lo, hi, int(rng.integers(lo, hi + 1)), int(rng.integers(lo, hi + 1))]))
        rw, rh = draw(W), draw(H)
        ref_sz.append((rw, rh))
        geoms.append(picture_geom(rng, rw, rh, layout))
        mask |= 1 << k
    pics = [rng.integers(0, bd + 1, g["total"]).astype(dt) for g in geoms]
    # where the records may write: put records tile the frame planes without overlapping (they run concurrently)
    taken = [np.zeros((frame["h"][p], frame["w"][p]), bool) for p in range(3)]
    recs = (_lib.McScaledBlock * n_rec)()
    n_tmp = n_px = 0
    for i in range(n_rec):
        r = recs[i]
        pl = int(rng.integers(0, n_planes))
        pw, ph = frame["w"][pl], frame["h"][pl]
        w, h = int(rng.choice(SIZES)), int(rng.choice(SIZES))
        if w > 4 * h or h > 4 * w:
            h = w
        op = int(rng.choice([0, 0, 1, 2]))
        if op == 1 and w < 4:
            op = 0
        x0 = y0 = None
        if op == 0:
            for _ in range(24):
                if w > pw or h > ph:
                    break
                cx, cy = w * int(rng.integers(0, pw // w)), h * int(rng.integers(0, ph // h))
                if not taken[pl][cy:cy + h, cx:cx + w].any():
                    taken[pl][cy:cy + h, cx:cx + w] = True
                    x0, y0 = cx, cy
                    break
            if x0 is None:
                op = 1 if w >= 4 else 2
        if op == 0:
            r.dst_off = frame["off"][pl] + y0 * frame["stride"][pl] + x0
        elif op == 1:
            r.dst_off = n_tmp
            n_tmp += w * h + int(rng.integers(1, 24))          # gaps stay at their sentinel
        else:
            r.dst_off = n_px
            n_px += w * h + int(rng.integers(1, 24))
        k = int(rng.integers(0, n_refs))
        rpw, rph = geoms[k]["w"][pl], geoms[k]["h"][pl]
        if rng.integers(0, 10) < 7:
            # the hook's arithmetic: a block at (x0, y0) of the plane, a motion vector in 1/8 luma sample units (1/16 for
            # subsampled chroma), the reference's scale and step (reference src/decode.c:3473-3480)
            bx = x0 if x0 is not None else int(rng.integers(0, pw))
            by = y0 if y0 is not None else int(rng.integers(0, ph))
            reach = int(rng.choice([64, 1024, 8 * W]))
            mvx, mvy = (int(np.clip(rng.integers(-reach, reach + 1), -(1 << 14), (1 << 14) - 1)) for _ in range(2))
            sx = ((ref_sz[k][0] << 14) + (W >> 1)) // W
            sy = ((ref_sz[k][1] << 14) + (H >> 1)) // H
            pos_x = scale_mv((bx << 4) + mvx * (1 << (1 - (ss_hor if pl else 0))), sx)
            pos_y = scale_mv((by << 4) + mvy * (1 << (1 - (ss_ver if pl else 0))), sy)
            dx, dy = (sx + 8) >> 4, (sy + 8) >> 4
            src_x, mx, src_y, my = pos_x >> 10, pos_x & 0x3ff, pos_y >> 10, pos_y & 0x3ff
        else:
            dx, dy = (int(rng.choice(STEPS)) if rng.integers(0, 4) else int(rng.integers(1, 2049)) for _ in range(2))
            mx, my = (int(rng.choice([0, 1023, int(rng.integers(0, 1024))])) for _ in range(2))
            src_x = _window_pos(rng, ((mx + (w - 1) * dx) >> 10) + 1, rpw)
            src_y = _window_pos(rng, ((my + (h - 1) * dy) >> 10) + 1, rph)
        r.src_x, r.src_y, r.mx, r.my, r.dx, r.dy = src_x, src_y, mx, my, dx, dy
        r.w, r.h, r.filter2d, r.op, r.plane, r.ref = w, h, int(rng.integers(0, 10)), op, pl, k
    return dict(bpc=bpc, bd=bd, dt=dt, frame=frame, geoms=geoms, mask=mask, pics=pics, recs=recs, n=n_rec,
                dst=rng.integers(0, bd + 1, frame["total"]).astype(dt),
                tmp=rng.integers(-(1 << 15), 1 << 15, max(1, n_tmp)).astype(np.int16),
                px_tmp=rng.integers(0, bd + 1, max(1, n_px)).astype(dt))


def scaled_batch_reference(B, ctx):
    """What dav1d's mc() does for each record of a scaled reference: emu_edge of the window into a 320-sample-wide
    buffer, then mc_scaled / mct_scaled on it. Always going through emu_edge is what dav1d computes when the window
    lies inside the plane too."""
    out = {k: B[k].copy() for k in ("dst", "tmp", "px_tmp")}
    dt = B["dt"]
    isz = np.dtype(dt).itemsize
    ebuf = np.zeros((EMU_ROWS + 1, EMU_W), dt)
    eptr = ebuf.ctypes.data + (EMU_W * 3 + 3) * isz
    for i in range(B["n"]):
        r = B["recs"][i]
        pl, w, h = r.plane, r.w, r.h
        g = B["geoms"][r.ref] if (B["mask"] >> r.ref) & 1 else B["frame"]
        left, top = r.src_x, r.src_y
        right = ((r.mx + (w - 1) * r.dx) >> 10) + 1 + left
        bottom = ((r.my + (h - 1) * r.dy) >> 10) + 1 + top
        ctx.emu_edge(right - left + 7, bottom - top + 7, g["w"][pl], g["h"][pl], left - 3, top - 3,
                     ebuf, EMU_W * isz, B["pics"][r.ref].ctypes.data + g["off"][pl] * isz, g["stride"][pl] * isz)
        if r.op == 1:
            ctx.mct_scaled[r.filter2d](out["tmp"].ctypes.data + r.dst_off * 2, eptr, EMU_W * isz, w, h, r.mx, r.my, r.dx, r.dy)
        else:
            d, ds = (out["dst"], B["frame"]["stride"][pl]) if r.op == 0 else (out["px_tmp"], w)
            ctx.mc_scaled[r.filter2d](d.ctypes.data + r.dst_off * isz, ds * isz, eptr, EMU_W * isz, w, h, r.mx, r.my, r.dx, r.dy)
    return out


def run_scaled_batch(B, lib, alloc):
    dev = {k: alloc.upload(B[k]) for k in ("dst", "tmp", "px_tmp")}
    pics = [alloc.upload(p) for p in B["pics"]]
    fr = _lib.McFrame()
    f = B["frame"]
    for p in range(3):
        fr.ref_plane_off[p], fr.ref_stride[p], fr.ref_w[p], fr.ref_h[p] = f["off"][p], f["stride"][p], f["w"][p], f["h"][p]
        fr.dst_stride[p] = f["stride"][p]
    for k, (g, pic) in enumerate(zip(B["geoms"], pics)):
        fr.ref[k] = pic[1]
        if (B["mask"] >> k) & 1:
            for p in range(3):
                rg = fr.ref_geom[k]
                rg.plane_off[p], rg.stride[p], rg.w[p], rg.h[p] = g["off"][p], g["stride"][p], g["w"][p], g["h"][p]
    fr.scaled_mask = B["mask"]
    fr.dst, fr.tmp, fr.px_tmp = dev["dst"][1], dev["tmp"][1], dev["px_tmp"][1]
    recs = alloc.upload(np.frombuffer(B["recs"], np.uint8))
    lib.check(lib.b200_mc_scaled_batch(B["bd"], C.byref(fr), recs[1], B["n"], None), "b200_mc_scaled_batch")
    alloc.sync()
    return {k: alloc.download(v[0], B[k]) for k, v in dev.items()}


def compare(B, exp, got):
    for k in ("dst", "tmp", "px_tmp"):
        if not np.array_equal(exp[k], got[k]):
            bad = np.nonzero(exp[k] != got[k])[0]
            raise AssertionError("%s: %d of %d samples differ, first at %d" % (k, len(bad), exp[k].size, bad[0]))
    ops = np.bincount([B["recs"][i].op for i in range(B["n"])], minlength=3)
    assert ops.min() > 0, ops


# ------------------------------------------------------------------ 1. b200_mc_scaled_batch
SCALED_EMU = [(bpc, lay) for bpc in (8, 10, 12) for lay in ("420", "422", "444", "400")]


@pytest.mark.emu
@pytest.mark.parametrize("bpc,layout", SCALED_EMU)
def test_emu_scaled_batch(bpc, layout):
    B = make_scaled_batch(np.random.default_rng(1100 + 10 * bpc + list(LAYOUTS).index(layout)), bpc, layout, 200, 136, 300)
    exp = scaled_batch_reference(B, checker(bpc))
    compare(B, exp, run_scaled_batch(B, *refs.lib_alloc(False)))


def test_oracle_scaled_batch_matches_reference():
    """the oracle's emu_edge / mc_scaled / mct_scaled give dav1d's bytes on a whole batch, so a run that has only the
    oracle still checks the kernel against dav1d"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    for bpc, layout in ((8, "420"), (12, "444")):
        B = make_scaled_batch(np.random.default_rng(1190 + bpc), bpc, layout, 200, 136, 300)
        a, b = scaled_batch_reference(B, refs.ref_mc_ctx(bpc)), scaled_batch_reference(B, refs.oracle_mc_ctx(bpc))
        for k in a:
            assert np.array_equal(a[k], b[k]), (bpc, layout, k)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,layout,W,H,n", [(8, "420", 1920, 1080, 3000), (10, "420", 3840, 2160, 5000),
                                              (12, "444", 1280, 720, 2500), (10, "422", 1280, 720, 2500)])
def test_gpu_scaled_batch(bpc, layout, W, H, n):
    B = make_scaled_batch(np.random.default_rng(1200 + W + bpc), bpc, layout, W, H, n)
    exp = scaled_batch_reference(B, checker(bpc))
    compare(B, exp, run_scaled_batch(B, *refs.lib_alloc(True)))


# ------------------------------------------------------------------ 2. b200_resize_frame
SENTINEL = {8: 0xa5, 10: 0x3a5, 12: 0xa5a}


def make_resize_frame(rng, bpc, layout, out_w, H, den):
    """A super-resolution frame coded at (out_w * 8 + den / 2) / den, upscaled to out_w, with the parameters the hook
    takes from dav1d (b200_hooks_tmpl.c: src_w = (4 * bw + ss) >> ss may be wider than the coded width; step and start
    phase from the coded and upscaled widths of each plane). Source and destination are three planes in one
    allocation each, with strides wider than the rows; the destination holds a sentinel."""
    bd = (1 << bpc) - 1
    dt = refs.pixel_dtype(bpc)
    ss_hor, ss_ver = LAYOUTS[layout]
    coded = (out_w * 8 + den // 2) // den
    bw = ((coded + 7) >> 3) << 1                       # f->bw, in 4-sample units
    fr = _lib.ResizeFrame()
    fr.n_planes = 1 if layout == "400" else 3
    soff = doff = 0
    for p in range(fr.n_planes):
        sh, sv = (ss_hor, ss_ver) if p else (0, 0)
        fr.src_w[p] = (4 * bw + sh) >> sh
        fr.dst_w[p] = (out_w + sh) >> sh
        fr.h[p] = (H + sv) >> sv
        fr.dx[p], fr.mx0[p] = resize_params((coded + sh) >> sh, fr.dst_w[p])
        fr.src_stride[p] = fr.src_w[p] + int(rng.integers(1, 64))
        fr.dst_stride[p] = fr.dst_w[p] + int(rng.integers(1, 64))
        fr.src_plane_off[p], fr.dst_plane_off[p] = soff, doff
        soff += fr.src_stride[p] * fr.h[p] + int(rng.integers(0, 256))
        doff += fr.dst_stride[p] * fr.h[p] + int(rng.integers(0, 256))
    return dict(bd=bd, dt=dt, fr=fr, src=rng.integers(0, bd + 1, soff).astype(dt), dst=np.full(doff, SENTINEL[bpc], dt))


def resize_reference(R, ctx):
    fr, isz = R["fr"], np.dtype(R["dt"]).itemsize
    dst = R["dst"].copy()
    for p in range(fr.n_planes):
        ctx.resize(dst.ctypes.data + fr.dst_plane_off[p] * isz, fr.dst_stride[p] * isz,
                   R["src"].ctypes.data + fr.src_plane_off[p] * isz, fr.src_stride[p] * isz,
                   fr.dst_w[p], fr.h[p], fr.src_w[p], fr.dx[p], fr.mx0[p])
    return dst


def run_resize(R, lib, alloc):
    src, dst = alloc.upload(R["src"]), alloc.upload(R["dst"])
    fr = _lib.ResizeFrame.from_buffer_copy(R["fr"])
    fr.src, fr.dst = src[1], dst[1]
    lib.check(lib.b200_resize_frame(R["bd"], C.byref(fr), None), "b200_resize_frame")
    alloc.sync()
    return alloc.download(dst[0], R["dst"])


def check_resize(R, exp, got):
    fr = R["fr"]
    inside = np.zeros(R["dst"].size, bool)
    for p in range(fr.n_planes):
        rows = fr.dst_plane_off[p] + np.arange(fr.h[p])[:, None] * fr.dst_stride[p]
        inside[(rows + np.arange(fr.dst_w[p])[None, :]).ravel()] = True
    assert np.all(got[~inside] == R["dst"][~inside]), "samples outside dst_w x h of a plane changed"
    for p in range(fr.n_planes):
        o, s = fr.dst_plane_off[p], fr.dst_stride[p]
        e = exp[o:o + s * fr.h[p]].reshape(fr.h[p], s)[:, :fr.dst_w[p]]
        g = got[o:o + s * fr.h[p]].reshape(fr.h[p], s)[:, :fr.dst_w[p]]
        if not np.array_equal(e, g):
            y, x = np.argwhere(e != g)[0]
            raise AssertionError("plane %d: %d of %d samples differ, first at (%d, %d)" % (p, int((e != g).sum()), e.size, x, y))


# the largest plane of the second case has 640 x 480 = 307 200 samples: more than one pass of the grid-stride loop
RESIZE_EMU = [(10, "420", 203, 67, 9), (8, "400", 640, 480, 16), (12, "444", 97, 40, 13)]
# every denominator 9 ... 16 once, odd target widths
RESIZE_GPU = [(8, "420", 1921, 1080, 9), (10, "420", 3839, 2160, 10), (10, "420", 7679, 4320, 16), (12, "444", 1919, 1080, 13),
              (10, "422", 1281, 721, 11), (10, "400", 1921, 1081, 12), (8, "420", 1279, 720, 14), (12, "420", 2561, 1441, 15)]


@pytest.mark.emu
@pytest.mark.parametrize("bpc,layout,out_w,H,den", RESIZE_EMU)
def test_emu_resize_frame(bpc, layout, out_w, H, den):
    R = make_resize_frame(np.random.default_rng(1300 + out_w), bpc, layout, out_w, H, den)
    exp = resize_reference(R, checker(bpc))
    check_resize(R, exp, run_resize(R, *refs.lib_alloc(False)))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,layout,out_w,H,den", RESIZE_GPU)
def test_gpu_resize_frame(bpc, layout, out_w, H, den):
    R = make_resize_frame(np.random.default_rng(1400 + out_w), bpc, layout, out_w, H, den)
    exp = resize_reference(R, checker(bpc))
    check_resize(R, exp, run_resize(R, *refs.lib_alloc(True)))


def _resize_arguments(lib):
    buf = np.zeros(4096, np.uint8)

    def frame(**kw):
        fr = _lib.ResizeFrame()
        fr.src = fr.dst = buf.ctypes.data
        fr.n_planes = 3
        for p in range(3):
            fr.src_stride[p] = fr.dst_stride[p] = fr.src_w[p] = fr.dst_w[p] = 16
            fr.h[p] = 4
            fr.dx[p], fr.mx0[p] = resize_params(12, 16)
            fr.src_plane_off[p] = fr.dst_plane_off[p] = 64 * p
        for k, v in kw.items():
            if isinstance(v, tuple):
                getattr(fr, k)[v[0]] = v[1]
            else:
                setattr(fr, k, v)
        return fr

    bad = [dict(n_planes=4), dict(n_planes=7), dict(src=None), dict(dst=None), dict(dst_w=(0, 0)), dict(src_w=(1, 0)),
           dict(h=(2, 0)), dict(dst_w=(2, -5)), dict(n_planes=1, h=(0, -1))]
    for kw in bad:
        assert lib.b200_mc_resize(None, 0, None, 0, 0, 1, 1, 1, 0, 255) == -2      # leaves another function's message
        assert lib.b200_resize_frame(255, C.byref(frame(**kw)), None) == -2, kw
        assert lib.b200_last_error().decode().startswith("b200_resize_frame"), (kw, lib.b200_last_error())
    assert lib.b200_resize_frame(255, C.byref(frame(n_planes=0, src=None, dst=None)), None) == 0
    assert not buf.any()


@pytest.mark.emu
def test_resize_frame_arguments_emu():
    _resize_arguments(refs.emu_lib())


@pytest.mark.gpu
def test_resize_frame_arguments_gpu():
    from dav1d_b200 import get_lib
    _resize_arguments(get_lib())


# ------------------------------------------------------------------ 3. full-size streams on the H100
@pytest.fixture(scope="module")
def gpu_decoder():
    d = stream.HookedDecoder()
    yield d
    d.release()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,kw", [(1920, 1080, dict(bpc=8, film_grain=1)), (3840, 2160, dict(bpc=10, log2_cols=2)),
                                    (1280, 720, dict(bpc=12, layout="444")), (1280, 720, dict(bpc=10, layout="400"))])
def test_gpu_super_resolution_streams(gpu_decoder, w, h, kw):
    """key and inter frames with super-resolution: each frame draws its own denominator, so inter frames also predict
    from references of another coded width"""
    tus = obu.inter_stream(1500 + w + kw["bpc"], w, h, n_frames=4, super_res=1, **kw)
    _check(gpu_decoder, tus, 4, apply_grain=1)
    assert gpu_decoder.last_stats["scaled"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,sizes,kw", [(1920, 1080, [(960, 540), (1920, 1080), (1440, 816)], dict(bpc=8, motion_modes=1)),
                                          (3840, 2160, [(1920, 1080), (3840, 2160), (2880, 1632)], dict(bpc=10)),
                                          (1280, 720, [(640, 360), (1280, 720)], dict(bpc=12, layout="444", motion_modes=2))])
def test_gpu_scaled_reference_streams(gpu_decoder, w, h, sizes, kw):
    """inter frames coded at changing sizes at full frame size: their predictions are B200McScaledBlock records against
    references of other sizes (every frame within the factor of 2 down and 16 up AV1 allows)"""
    tus = obu.inter_stream(1600 + w + kw["bpc"], w, h, n_frames=len(sizes) + 2, sizes=sizes, **kw)
    _check(gpu_decoder, tus, len(sizes) + 2, apply_grain=1)
    assert gpu_decoder.last_stats["scaled"] >= 1000, gpu_decoder.last_stats["scaled"]
