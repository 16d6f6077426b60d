"""Parity tests for motion compensation (Dav1dMCDSPContext), modelled on the reference's
tests/checkasm/mc.c: check_mc :58-110, check_mct :124-167 (worst-case corner pattern :114-122),
check_mc_scaled :169-275, check_avg/w_avg/mask/w_mask :289-447 (inputs are real mct outputs,
init_tmp :278-287), check_blend* :449-560, check_warp8x8{,t} :562-640, check_emuedge :680-719,
check_resize :727-770.

`run_mc_checks(new, chk, ...)` drives any two objects exposing the Dav1dMCDSPContext members:
the reference C path (oracle/_ref), the oracle restatement (oracle/mc.c), the CUDA kernels
through the Level-1 table, or the same CUDA sources on the host emulator.
"""
import numpy as np
import pytest

import refs
from test_scaled_prediction import resize_params

PAD = 8


def h_next(h):   # mc_h_next, reference tests/checkasm/mc.c:43-56
    if h in (4, 8, 16):
        return (h * 3) >> 1
    if h in (6, 12, 24):
        return (h & (h - 1)) * 2
    return h * 2


def mct_input(rng, bdmax, dt):
    """generate_mct_input: worst case in the top-left corner, random elsewhere"""
    pattern = np.array([-1, 0, -1, 0, 0, -1, 0, -1])
    sign = -int(rng.integers(0, 2))
    buf = rng.integers(0, bdmax + 1, (135, 135)).astype(np.int64)
    corner = (pattern[None, :8] ^ pattern[:8, None] ^ sign) & bdmax
    xs, ys = np.meshgrid(np.arange(135), np.arange(135))
    m = (xs | ys) < 8
    buf[m] = np.broadcast_to(np.pad(corner, ((0, 127), (0, 127))), (135, 135))[m]
    return buf.astype(dt)


def padded(h, w, dt, rng, bdmax, fill_random=True):
    c = rng.integers(0, bdmax + 1, (h + 2 * PAD, w + 2 * PAD)).astype(dt) if fill_random \
        else np.zeros((h + 2 * PAD, w + 2 * PAD), dt)
    return c


def run_mc_checks(new, chk, bpc, seed, light=False, scaled=False, sections=None):
    rng = np.random.default_rng(seed)
    bd = (1 << bpc) - 1
    dt = refs.pixel_dtype(bpc)
    isz = np.dtype(dt).itemsize
    n = 0
    want = lambda s: sections is None or s in sections
    filters = [0, 5, 7, 9] if light else range(10)

    # ---- mc / mct ----
    if want("mc"):
        for f in filters:
            w = 2
            while w <= 128:
                for mxy in range(4):
                    h = 2 if w <= 32 else w // 4
                    hmax = max(min(w * 4, 128), 32)
                    while h <= hmax:
                        mx = int(rng.integers(1, 16)) if mxy & 1 else 0
                        my = int(rng.integers(1, 16)) if mxy & 2 else 0
                        src = rng.integers(0, bd + 1, (135, 135)).astype(dt)
                        sp = src[3:, 3:]
                        c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                        chk.mc[f](c1[PAD:, PAD:], c1.strides[0], sp, src.strides[0], w, h, mx, my)
                        new.mc[f](c2[PAD:, PAD:], c2.strides[0], sp, src.strides[0], w, h, mx, my)
                        assert np.array_equal(c1, c2), ("mc", bpc, f, w, h, mx, my)
                        n += 1
                        if w >= 4 and h >= 4 and (h & (h - 1)) == 0 and h <= w * 4 and w <= h * 4:
                            src = mct_input(rng, bd, dt)
                            sp = src[3:, 3:]
                            t1 = np.zeros(w * h + 16, np.int16); t2 = t1.copy()
                            chk.mct[f](t1, sp, src.strides[0], w, h, mx, my)
                            new.mct[f](t2, sp, src.strides[0], w, h, mx, my)
                            assert np.array_equal(t1, t2), ("mct", bpc, f, w, h, mx, my)
                            n += 1
                        h = h_next(h) if not light else h * 2
                w <<= 1

    # ---- scaled (only where both sides implement it) ----
    if scaled and want("scaled") and new.mc_scaled[0] is not None:
        for f in filters:
            for w in (2, 4, 8, 16, 32, 64, 128):
                for p in range(3):
                    h = int(rng.choice([4, 8, 16, 32, 64, 128]))
                    if w > h * 8 or h > w * 8:
                        continue
                    mx, my = int(rng.integers(0, 1024)), int(rng.integers(0, 1024))
                    dx = int(rng.integers(1, 2049))
                    dy = [int(rng.integers(1, 2049)), 1024, 2048][p]
                    src = rng.integers(0, bd + 1, (263 + 8, 263 + 8)).astype(dt)
                    sp = src[3:, 3:]
                    c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                    chk.mc_scaled[f](c1[PAD:, PAD:], c1.strides[0], sp, src.strides[0], w, h, mx, my, dx, dy)
                    new.mc_scaled[f](c2[PAD:, PAD:], c2.strides[0], sp, src.strides[0], w, h, mx, my, dx, dy)
                    assert np.array_equal(c1, c2), ("mc_scaled", bpc, f, w, h)
                    n += 1
                    if w >= 4:
                        t1 = np.zeros(w * h, np.int16); t2 = t1.copy()
                        chk.mct_scaled[f](t1, sp, src.strides[0], w, h, mx, my, dx, dy)
                        new.mct_scaled[f](t2, sp, src.strides[0], w, h, mx, my, dx, dy)
                        assert np.array_equal(t1, t2), ("mct_scaled", bpc, f, w, h)
                        n += 1

    # ---- compound: inputs are real prep outputs of the worst-case pattern (init_tmp) ----
    def init_tmp():
        out = []
        for _ in range(2):
            src = mct_input(rng, bd, dt)
            t = np.zeros(128 * 128, np.int16)
            chk.mct[5](t, src[3:, 3:], src.strides[0], 128, 128, 8, 8)
            out.append(t)
        return out

    if want("comp"):
        w = 4
        while w <= 128:
            h = max(w // 4, 4)
            while h <= min(w * 4, 128):
                t = init_tmp()
                # the functions read tmp densely with pitch w: take the first w*h entries
                a, b = t[0][:w * h].copy(), t[1][:w * h].copy()
                c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                chk.avg(c1[PAD:, PAD:], c1.strides[0], a, b, w, h)
                new.avg(c2[PAD:, PAD:], c2.strides[0], a, b, w, h)
                assert np.array_equal(c1, c2), ("avg", bpc, w, h)
                wt = int(rng.integers(1, 16))
                chk.w_avg(c1[PAD:, PAD:], c1.strides[0], a, b, w, h, wt)
                new.w_avg(c2[PAD:, PAD:], c2.strides[0], a, b, w, h, wt)
                assert np.array_equal(c1, c2), ("w_avg", bpc, w, h, wt)
                m = rng.integers(0, 65, w * h).astype(np.uint8)
                chk.mask(c1[PAD:, PAD:], c1.strides[0], a, b, w, h, m)
                new.mask(c2[PAD:, PAD:], c2.strides[0], a, b, w, h, m)
                assert np.array_equal(c1, c2), ("mask", bpc, w, h)
                n += 3
                for lay in range(3):
                    sign = int(rng.integers(0, 2))
                    m1 = np.full(w * h, 0xAA, np.uint8); m2 = m1.copy()
                    chk.w_mask[lay](c1[PAD:, PAD:], c1.strides[0], a, b, w, h, m1, sign)
                    new.w_mask[lay](c2[PAD:, PAD:], c2.strides[0], a, b, w, h, m2, sign)
                    assert np.array_equal(c1, c2), ("w_mask dst", bpc, lay, w, h)
                    assert np.array_equal(m1, m2), ("w_mask mask", bpc, lay, w, h)
                    n += 1
                h <<= 1
            w <<= 1

    # ---- blends ----
    if want("blend"):
        w = 4
        while w <= 32:
            h = max(w // 2, 4)
            while h <= min(w * 2, 32):
                tmp = rng.integers(0, bd + 1, 32 * 32).astype(dt)
                mask = rng.integers(0, 65, 32 * 32).astype(np.uint8)
                c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                chk.blend(c1[PAD:, PAD:], c1.strides[0], tmp, w, h, mask)
                new.blend(c2[PAD:, PAD:], c2.strides[0], tmp, w, h, mask)
                assert np.array_equal(c1, c2), ("blend", bpc, w, h)
                n += 1
                h <<= 1
            w <<= 1
        for w in (2, 4, 8, 16, 32):
            h = 2
            while h <= (128 if w >= 8 else w * 8):
                tmp = rng.integers(0, bd + 1, 32 * 128).astype(dt)
                c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                chk.blend_v(c1[PAD:, PAD:], c1.strides[0], tmp, w, h)
                new.blend_v(c2[PAD:, PAD:], c2.strides[0], tmp, w, h)
                assert np.array_equal(c1, c2), ("blend_v", bpc, w, h)
                n += 1
                h <<= 1
        for w in (2, 4, 8, 16, 32, 64, 128):
            for h in (2, 4, 8, 16, 32):
                tmp = rng.integers(0, bd + 1, 128 * 32).astype(dt)
                c1 = padded(h, w, dt, rng, bd); c2 = c1.copy()
                chk.blend_h(c1[PAD:, PAD:], c1.strides[0], tmp, w, h)
                new.blend_h(c2[PAD:, PAD:], c2.strides[0], tmp, w, h)
                assert np.array_equal(c1, c2), ("blend_h", bpc, w, h)
                n += 1

    # ---- warp ----
    if want("warp"):
        for it in range(6 if light else 40):
            src = rng.integers(0, bd + 1, (15, 15)).astype(dt)
            sp = src[3:, 3:]
            abcd = ((rng.integers(0, 1 << 16, 4) & 0x1fff) - 0xa00).astype(np.int16)
            mx = int((rng.integers(0, 1 << 16) & 0x1fff) - 0xa00)
            my = int((rng.integers(0, 1 << 16) & 0x1fff) - 0xa00)
            c1 = padded(8, 8, dt, rng, bd); c2 = c1.copy()
            chk.warp8x8(c1[PAD:, PAD:], c1.strides[0], sp, src.strides[0], abcd, mx, my)
            new.warp8x8(c2[PAD:, PAD:], c2.strides[0], sp, src.strides[0], abcd, mx, my)
            assert np.array_equal(c1, c2), ("warp8x8", bpc)
            t1 = np.zeros(64, np.int16); t2 = t1.copy()
            chk.warp8x8t(t1, 8, sp, src.strides[0], abcd, mx, my)
            new.warp8x8t(t2, 8, sp, src.strides[0], abcd, mx, my)
            assert np.array_equal(t1, t2), ("warp8x8t", bpc)
            n += 2

    # ---- emu_edge ----
    if want("emu"):
        src = rng.integers(0, bd + 1, (160, 160)).astype(dt)

        def rnd_off(bdim, edge2):   # edge2: bit0 = HAVE_<first> (left/top), bit1 = HAVE_<second>
            idim = 160 if edge2 else 1 + int(rng.integers(0, bdim - 2))
            if edge2 == 3:
                pos = int(rng.integers(0, idim - bdim + 1))
            elif edge2 == 1:
                pos = (idim - bdim) + 1 + int(rng.integers(0, bdim - 1))
            elif edge2 == 2:
                pos = -(1 + int(rng.integers(0, bdim - 1)))
            else:
                pos = -(1 + int(rng.integers(0, bdim - idim - 1)))
            return pos, idim
        w = 4
        while w <= 128:
            h = max(w // 4, 4)
            while h <= min(w * 4, 128):
                for edge in range(0xf):
                    bw, bh = w + int(rng.integers(0, 8)), h + int(rng.integers(0, 8))
                    x, iw = rnd_off(bw, ((edge >> 2) & 1) | (((edge >> 3) & 1) << 1))
                    y, ih = rnd_off(bh, (edge & 1) | (((edge >> 1) & 1) << 1))
                    d1 = np.zeros((135, 192), dt); d2 = d1.copy()
                    chk.emu_edge(bw, bh, iw, ih, x, y, d1, 192 * isz, src, 160 * isz)
                    new.emu_edge(bw, bh, iw, ih, x, y, d2, 192 * isz, src, 160 * isz)
                    assert np.array_equal(d1, d2), ("emu_edge", bpc, bw, bh, iw, ih, x, y)
                    n += 1
                    if light and edge > 4:
                        break
                h <<= 1
            w <<= 1

    # ---- resize ----
    if want("resize"):
        for it in range(2 if light else 6):
            src_w = 16 + int(rng.integers(0, 512 - 16 + 1))
            w_den = 9 + int(rng.integers(0, 8))
            dst_w = w_den * src_w >> 3
            dx, mx0 = resize_params(src_w, dst_w)
            hh = 8 if light else 64
            src = rng.integers(0, bd + 1, (hh, 512)).astype(dt)
            c1 = padded(hh, dst_w, dt, rng, bd); c2 = c1.copy()
            chk.resize(c1[PAD:, PAD:], c1.strides[0], src, src.strides[0], dst_w, hh, src_w, dx, mx0)
            new.resize(c2[PAD:, PAD:], c2.strides[0], src, src.strides[0], dst_w, hh, src_w, dx, mx0)
            assert np.array_equal(c1, c2), ("resize", bpc, dst_w, src_w)
            n += 1
    return n


# ------------------------------------------------------------------ oracle pinning (CPU)
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_mc_vs_reference(bpc):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    n = run_mc_checks(refs.oracle_mc_ctx(bpc), refs.ref_mc_ctx(bpc), bpc, seed=40 + bpc, scaled=True)
    assert n > 2000


# ------------------------------------------------------------------ host emulator (debug harness)
@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_mc(bpc):
    from dav1d_b200.dsp import MCDSPContext
    new = MCDSPContext(bpc, lib=refs.emu_lib())
    run_mc_checks(new, refs.oracle_mc_ctx(bpc), bpc, seed=50 + bpc, light=True, scaled=True)


# ------------------------------------------------------------------ GPU parity (Level-1 table)
@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_mc_level1(bpc):
    from dav1d_b200.dsp import MCDSPContext
    new = MCDSPContext(bpc)
    chk = refs.ref_mc_ctx(bpc) if refs.have_ref() else refs.oracle_mc_ctx(bpc)
    n = run_mc_checks(new, chk, bpc, seed=60 + bpc, scaled=True)
    assert n > 1500
    run_mc_checks(new, refs.oracle_mc_ctx(bpc), bpc, seed=70 + bpc, light=True)


# ------------------------------------------------------------------ Level-2 (batched) parity
def make_mc_frame(rng, bpc, W=192, H=128, n_pred=220):
    """A small synthetic inter frame: one reference picture (3 planes, 4:2:0), put/prep blocks with
    motion vectors that also point outside the picture (-> clamped loads = emu_edge), compound
    combines over the prep outputs, blends and 8x8 warps. Returns host-side numpy state."""
    from dav1d_b200 import _lib
    bd = (1 << bpc) - 1
    dt = refs.pixel_dtype(bpc)
    pw, ph = [W, W // 2, W // 2], [H, H // 2, H // 2]
    stride = [W + 32, W // 2 + 16, W // 2 + 16]
    off = [0, stride[0] * H, stride[0] * H + stride[1] * ph[1]]
    total = off[2] + stride[2] * ph[2]
    refpic = rng.integers(0, bd + 1, total).astype(dt)
    dst = rng.integers(0, bd + 1, total).astype(dt)
    sizes = [(w, h) for w in (4, 8, 16, 32, 64, 128) for h in (4, 8, 16, 32, 64, 128) if w <= 4 * h and h <= 4 * w]
    blocks = (_lib.McBlock * n_pred)()
    comp, tmp_off = [], 0
    put_rects = []
    for i in range(n_pred):
        pl = int(rng.integers(0, 3))
        w, h = sizes[int(rng.integers(0, len(sizes)))]
        w, h = min(w, pw[pl]), min(h, ph[pl])
        b = blocks[i]
        b.w, b.h, b.plane, b.ref = w, h, pl, 0
        b.mx, b.my = int(rng.integers(0, 16)), int(rng.integers(0, 16))
        if rng.integers(0, 4) == 0:
            b.mx = 0
        if rng.integers(0, 4) == 0:
            b.my = 0
        b.filter2d = int(rng.integers(0, 10))
        b.src_x = int(rng.integers(-w - 12, pw[pl] + 12))
        b.src_y = int(rng.integers(-h - 12, ph[pl] + 12))
        b.op = int(rng.integers(0, 2))
        if b.op:
            b.dst_off = tmp_off
            comp.append((tmp_off, w, h, pl))
            tmp_off += w * h
        else:
            x0 = int(rng.integers(0, pw[pl] - w + 1)); y0 = int(rng.integers(0, ph[pl] - h + 1))
            b.dst_off = off[pl] + y0 * stride[pl] + x0
    # pair up prep outputs of equal size for the compound ops
    cblocks = []
    by_size = {}
    for t in comp:
        by_size.setdefault(t[1:], []).append(t[0])
    mask_off = 0
    for (w, h, pl), offs in by_size.items():
        for k in range(0, len(offs) - 1, 2):
            cb = _lib.CompBlock()
            cb.tmp1_off, cb.tmp2_off, cb.w, cb.h, cb.plane = offs[k], offs[k + 1], w, h, pl
            cb.op = int(rng.integers(0, 6))
            if cb.op == 5 and (h & 1):
                cb.op = 0
            cb.param = int(rng.integers(1, 16)) if cb.op == 1 else int(rng.integers(0, 2))
            cb.mask_off = mask_off
            mask_off += w * h
            x0 = int(rng.integers(0, pw[pl] - w + 1)); y0 = int(rng.integers(0, ph[pl] - h + 1))
            cb.dst_off = off[pl] + y0 * stride[pl] + x0
            cblocks.append(cb)
    carr = (_lib.CompBlock * max(1, len(cblocks)))(*cblocks)
    mask = rng.integers(0, 65, max(1, mask_off)).astype(np.uint8)
    # blends
    nb = 40
    bl = (_lib.BlendBlock * nb)()
    px_tmp = rng.integers(0, bd + 1, nb * 32 * 32).astype(dt)
    bmask_off = mask_off
    for i in range(nb):
        pl = int(rng.integers(0, 3))
        w, h = int(rng.choice([4, 8, 16, 32])), int(rng.choice([4, 8, 16, 32]))
        bl[i].w, bl[i].h, bl[i].op, bl[i].plane = w, h, int(rng.integers(0, 3)), pl
        bl[i].tmp_off = i * 32 * 32
        bl[i].mask_off = bmask_off
        bmask_off += w * h
        x0 = int(rng.integers(0, pw[pl] - w + 1)); y0 = int(rng.integers(0, ph[pl] - h + 1))
        bl[i].dst_off = off[pl] + y0 * stride[pl] + x0
    mask = np.concatenate([mask, rng.integers(0, 65, bmask_off - mask_off).astype(np.uint8)])
    # warps
    nw = 50
    wb = (_lib.WarpBlock * nw)()
    wtmp0 = tmp_off
    for i in range(nw):
        pl = int(rng.integers(0, 3))
        wb[i].plane, wb[i].ref, wb[i].op = pl, 0, int(rng.integers(0, 2))
        wb[i].src_x = int(rng.integers(-10, pw[pl] + 4)); wb[i].src_y = int(rng.integers(-10, ph[pl] + 4))
        wb[i].mx = int((rng.integers(0, 1 << 16) & 0x1fff) - 0xa00); wb[i].my = int((rng.integers(0, 1 << 16) & 0x1fff) - 0xa00)
        for k in range(4):
            wb[i].abcd[k] = int((rng.integers(0, 1 << 16) & 0x1fff) - 0xa00)
        if wb[i].op:
            wb[i].dst_off, wb[i].tmp_stride = tmp_off, 8
            tmp_off += 64
        else:
            x0 = int(rng.integers(0, pw[pl] - 8 + 1)); y0 = int(rng.integers(0, ph[pl] - 8 + 1))
            wb[i].dst_off = off[pl] + y0 * stride[pl] + x0
    tmp = np.zeros(tmp_off + 64, np.int16)
    return dict(bd=bd, dt=dt, refpic=refpic, dst=dst, tmp=tmp, mask=mask, px_tmp=px_tmp, blocks=blocks, n_pred=n_pred,
                carr=carr, n_comp=len(cblocks), bl=bl, nb=nb, wb=wb, nw=nw, pw=pw, ph=ph, stride=stride, off=off)


def mc_frame_struct(S, ptrs):
    from dav1d_b200 import _lib
    fr = _lib.McFrame()
    fr.ref[0] = ptrs["refpic"]
    for p in range(3):
        fr.ref_plane_off[p] = S["off"][p]; fr.ref_stride[p] = S["stride"][p]
        fr.ref_w[p] = S["pw"][p]; fr.ref_h[p] = S["ph"][p]; fr.dst_stride[p] = S["stride"][p]
    fr.dst, fr.tmp, fr.mask, fr.px_tmp = ptrs["dst"], ptrs["tmp"], ptrs["mask"], ptrs["px_tmp"]
    return fr


def run_mc_frame_oracle(S):
    import ctypes as C
    o = refs.oracle()
    st = {k: S[k].copy() for k in ("refpic", "dst", "tmp", "mask", "px_tmp")}
    fr = mc_frame_struct(S, {k: v.ctypes.data for k, v in st.items()})
    # prediction -> compound -> blend -> warp, each stage complete before the next (as the device does)
    o.oracle_mc_batch(S["bd"], C.byref(fr), S["blocks"], S["n_pred"])
    o.oracle_mc_comp_batch(S["bd"], C.byref(fr), S["carr"], S["n_comp"])
    o.oracle_mc_blend_batch(S["bd"], C.byref(fr), S["bl"], S["nb"])
    o.oracle_mc_warp_batch(S["bd"], C.byref(fr), S["wb"], S["nw"])
    return st


def dedupe_writes(S):
    """Blocks of one batch run concurrently on the device, so destination rectangles inside one
    stage must not overlap: drop later blocks that would overlap an earlier one."""
    def run(arr, n, wh):
        keep, used = [], {0: [], 1: [], 2: []}
        for i in range(n):
            b = arr[i]
            pl = b.plane
            rel = b.dst_off - S["off"][pl]
            y0, x0 = divmod(rel, S["stride"][pl])
            w, h = wh(b)
            r = (x0, y0, x0 + w, y0 + h)
            if any(not (r[2] <= q[0] or q[2] <= r[0] or r[3] <= q[1] or q[3] <= r[1]) for q in used[pl]):
                continue
            used[pl].append(r); keep.append(i)
        return keep
    import ctypes as C
    from dav1d_b200 import _lib
    kp = [i for i in range(S["n_pred"]) if S["blocks"][i].op == 1] + \
        run(S["blocks"], S["n_pred"], lambda b: (b.w, b.h) if b.op == 0 else (0, 0))
    kp = sorted(set(kp))
    # prediction blocks with op 0 that overlap were dropped by `run`; rebuild arrays
    put_keep = set(run(S["blocks"], S["n_pred"], lambda b: (b.w, b.h)))
    idx = [i for i in range(S["n_pred"]) if S["blocks"][i].op == 1 or i in put_keep]
    nbk = (_lib.McBlock * len(idx))(*[S["blocks"][i] for i in idx])
    S["blocks"], S["n_pred"] = nbk, len(idx)
    for key, nkey, cls in (("carr", "n_comp", _lib.CompBlock), ("bl", "nb", _lib.BlendBlock)):
        k = run(S[key], S[nkey], lambda b: (b.w, b.h))
        S[key] = (cls * max(1, len(k)))(*[S[key][i] for i in k]); S[nkey] = len(k)
    k = [i for i in range(S["nw"]) if S["wb"][i].op == 1] + run(S["wb"], S["nw"], lambda b: (8, 8) if b.op == 0 else (0, 0))
    putk = set(run(S["wb"], S["nw"], lambda b: (8, 8)))
    k = [i for i in range(S["nw"]) if S["wb"][i].op == 1 or i in putk]
    S["wb"] = (_lib.WarpBlock * len(k))(*[S["wb"][i] for i in k]); S["nw"] = len(k)
    return S


def run_mc_frame_lib(S, lib, alloc):
    import ctypes as C
    dev = {k: alloc.upload(S[k]) for k in ("refpic", "dst", "tmp", "mask", "px_tmp")}
    fr = mc_frame_struct(S, {k: v[1] for k, v in dev.items()})

    def up(arr, n, cls):
        return alloc.upload(np.frombuffer(arr, np.uint8)[:max(1, n) * C.sizeof(cls)])
    d_b = up(S["blocks"], S["n_pred"], type(S["blocks"][0]))
    d_c = up(S["carr"], S["n_comp"], type(S["carr"][0]))
    d_l = up(S["bl"], S["nb"], type(S["bl"][0]))
    d_w = up(S["wb"], S["nw"], type(S["wb"][0]))
    lib.check(lib.b200_mc_batch(S["bd"], C.byref(fr), d_b[1], S["n_pred"], None), "mc_batch")
    lib.check(lib.b200_mc_comp_batch(S["bd"], C.byref(fr), d_c[1], S["n_comp"], None), "comp")
    lib.check(lib.b200_mc_blend_batch(S["bd"], C.byref(fr), d_l[1], S["nb"], None), "blend")
    lib.check(lib.b200_mc_warp_batch(S["bd"], C.byref(fr), d_w[1], S["nw"], None), "warp")
    alloc.sync()
    return {k: alloc.download(v[0], S[k]) for k, v in dev.items()}


def compare_mc_frame(exp, got):
    for k in ("dst", "tmp", "mask"):
        assert np.array_equal(exp[k], got[k]), "mc frame mismatch in " + k


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10])
def test_emu_mc_frame(bpc):
    rng = np.random.default_rng(90 + bpc)
    S = dedupe_writes(make_mc_frame(rng, bpc, n_pred=60))
    exp = run_mc_frame_oracle(S)
    compare_mc_frame(exp, run_mc_frame_lib(S, *refs.lib_alloc(False)))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_mc_frame(bpc):
    rng = np.random.default_rng(95 + bpc)
    S = dedupe_writes(make_mc_frame(rng, bpc, W=320, H=192, n_pred=900))
    exp = run_mc_frame_oracle(S)
    compare_mc_frame(exp, run_mc_frame_lib(S, *refs.lib_alloc(True)))
