"""Synthetic frame records for tests and bench.py.

No AV1 stream or encoder exists in this environment (SURVEY.md §7 hard part 7), so the "host
side" that dav1d's entropy decoder would play is synthesised at the RECORD level: random block
tilings, transform sizes, filter levels, masks ... in exactly the layouts dav1d's pass 1 leaves
in memory (Av1Filter bit masks, level[4] per 4x4, ...). Everything here is seeded and pure numpy.
"""
import numpy as np

# byte-identical to dav1d's Av1Filter (reference src/lf_mask.h:51-57), 1348 bytes
AV1FILTER_DT = np.dtype([("filter_y", "<u2", (2, 32, 3, 2)), ("filter_uv", "<u2", (2, 32, 2, 2)),
                         ("cdef_idx", "i1", (4,)), ("noskip_mask", "<u2", (16, 2))])
assert AV1FILTER_DT.itemsize == 1348


def random_tiling(rng, w4, h4, max_log=4, min_log=0, p_split=0.55, order=None):
    """Random block tiling of a w4 x h4 grid of 4x4 units. Returns int arrays (h4, w4):
    bx, by (origin of the block covering each unit) and lw, lh (log2 of block width/height in units).
    `order`: a list that receives the blocks (x, y, lw, lh) in decode order (superblock raster, partition recursion)."""
    bx = np.zeros((h4, w4), np.int32); by = np.zeros((h4, w4), np.int32)
    lw = np.zeros((h4, w4), np.int8); lh = np.zeros((h4, w4), np.int8)
    S = 1 << max_log

    def fill(x, y, lwv, lhv):
        x1, y1 = min(w4, x + (1 << lwv)), min(h4, y + (1 << lhv))
        bx[y:y1, x:x1] = x; by[y:y1, x:x1] = y; lw[y:y1, x:x1] = lwv; lh[y:y1, x:x1] = lhv
        if order is not None:
            order.append((x, y, lwv, lhv))

    def rec(x, y, lwv, lhv):
        if x >= w4 or y >= h4:
            return
        can_w, can_h = lwv > min_log, lhv > min_log
        if (can_w or can_h) and rng.random() < p_split:
            mode = rng.integers(0, 3)
            if mode == 0 and can_w and can_h:
                for dy in (0, 1):
                    for dx in (0, 1):
                        rec(x + (dx << (lwv - 1)), y + (dy << (lhv - 1)), lwv - 1, lhv - 1)
                return
            if (mode == 1 or not can_h) and can_w and lwv >= lhv:       # keep aspect within 1:2 .. 2:1 .. 4:1
                rec(x, y, lwv - 1, lhv); rec(x + (1 << (lwv - 1)), y, lwv - 1, lhv)
                return
            if can_h and lhv >= lwv:
                rec(x, y, lwv, lhv - 1); rec(x, y + (1 << (lhv - 1)), lwv, lhv - 1)
                return
        fill(x, y, lwv, lhv)

    for y in range(0, h4, S):
        for x in range(0, w4, S):
            rec(x, y, max_log, max_log)
    return bx, by, lw, lh


def _pack_bits(flags, axis_units, halves_len):
    """flags: bool [n_sb_a, units_a(<=32), ...]; pack `axis_units` along axis 1 into 2 uint16 halves."""
    n = flags.shape[1]
    out = []
    for h in range(2):
        lo, hi = h * halves_len, min(n, (h + 1) * halves_len)
        if lo >= hi:
            out.append(np.zeros(flags.shape[:1] + flags.shape[2:], np.uint16))
            continue
        w = (1 << np.arange(hi - lo)).astype(np.uint32)
        shape = [1] * flags.ndim; shape[1] = hi - lo
        out.append((flags[:, lo:hi] * w.reshape(shape)).sum(axis=1).astype(np.uint16))
    return out


def build_lf_masks(w4, h4, til_y, til_uv, ss_hor, ss_ver):
    """Av1Filter[] (one per 128x128 area, row-major sb128h x sb128w) from a luma tiling and a chroma
    tiling (chroma tiling in chroma 4x4 units). Edge filter size = min(size class of the two
    transform blocks that meet, capped: luma 4/8/16 -> 0/1/2, chroma 4/6 -> 0/1), as
    dav1d_create_lf_mask_* does (reference src/lf_mask.c)."""
    sb128w, sb128h = (w4 + 31) // 32, (h4 + 31) // 32
    masks = np.zeros(sb128h * sb128w, AV1FILTER_DT)

    def edges(til, cap):
        bx, by, lw, lh = til
        hh, ww = bx.shape
        xs = np.arange(ww)[None, :]; ys = np.arange(hh)[:, None]
        cw, ch = np.minimum(lw, cap), np.minimum(lh, cap)
        col = np.full((hh, ww), -1, np.int8)
        is_l = (bx == xs) & (xs > 0)
        col[:, 1:] = np.where(is_l[:, 1:], np.minimum(cw[:, 1:], cw[:, :-1]), -1)
        row = np.full((hh, ww), -1, np.int8)
        is_t = (by == ys) & (ys > 0)
        row[1:, :] = np.where(is_t[1:, :], np.minimum(ch[1:, :], ch[:-1, :]), -1)
        return col, row

    def put(field, col, row, ux, uy, ncls):
        # ux / uy: units per 128x128 area in x / y; pad to whole areas
        hh, ww = col.shape
        H, W = sb128h * uy, sb128w * ux
        for d, cls_map in ((0, col), (1, row)):
            full = np.full((H, W), -1, np.int8); full[:hh, :ww] = cls_map
            t = full.reshape(sb128h, uy, sb128w, ux)           # [sby, yi, sbx, xi]
            for k in range(ncls):
                f = (t == k)
                if d == 0:   # col edges: index [xi][k][half(yi)] bit yi
                    a = f.transpose(0, 1, 2, 3)                # [sby, yi, sbx, xi]
                    halves = _pack_bits(a, uy, 16 * uy // 32)
                    for h in range(2):
                        masks[field][:, 0, :ux, k, h] = halves[h].reshape(sb128h * sb128w, ux)
                else:        # row edges: index [yi][k][half(xi)] bit xi
                    a = f.transpose(0, 3, 2, 1)                # [sby, xi, sbx, yi]
                    halves = _pack_bits(a, ux, 16 * ux // 32)
                    for h in range(2):
                        masks[field][:, 1, :uy, k, h] = halves[h].reshape(sb128h * sb128w, uy)

    cy, ry = edges(til_y, 2)
    put("filter_y", cy, ry, 32, 32, 3)
    if til_uv is not None:
        cu, ru = edges(til_uv, 1)
        put("filter_uv", cu, ru, 32 >> ss_hor, 32 >> ss_ver, 2)
    return masks


def filter_lut(sharp):
    """Av1FilterLUT from the frame's sharpness (dav1d_calc_eih, reference src/lf_mask.c:385-...;
    same formula as tests/checkasm/loopfilter.c:122-137)."""
    e = np.zeros(64, np.uint8); i = np.zeros(64, np.uint8)
    for level in range(64):
        limit = level
        if sharp > 0:
            limit >>= (sharp + 3) >> 2
            limit = min(limit, 9 - sharp)
        limit = max(limit, 1)
        i[level] = limit
        e[level] = 2 * (level + 2) + limit
    return e, i, [(sharp + 3) >> 2, (9 - sharp) if sharp else 0xff]


def make_lf_frame(rng, bpc, W, H, ss_hor=1, ss_ver=1, sharp=None, smooth=True):
    """Picture + deblocking records for one frame. Returns a dict of numpy arrays / ints."""
    bd = (1 << bpc) - 1
    dt = np.uint8 if bpc == 8 else np.uint16
    w4, h4 = (W + 3) // 4, (H + 3) // 4
    cw4, ch4 = (w4 + ss_hor) >> ss_hor, (h4 + ss_ver) >> ss_ver
    sb128w = (w4 + 31) // 32
    b4_stride = (w4 + 31) & ~31
    # planes: stride padded like dav1d's allocator (reference src/picture.c:46-78)
    aw, ah = (W + 127) & ~127, (H + 127) & ~127
    stride = [aw + 64, (aw >> ss_hor) + 64, (aw >> ss_hor) + 64]
    rows = [ah, ah >> ss_ver, ah >> ss_ver]
    off = [0, stride[0] * rows[0], stride[0] * rows[0] + stride[1] * rows[1]]
    total = off[2] + stride[2] * rows[2]
    if smooth:   # low-amplitude texture so that the flat / narrow decisions all occur
        base = rng.integers(0, bd + 1, total // 64 + 2)
        pic = (np.repeat(base, 64)[:total] + rng.integers(-3 << (bpc - 8), (3 << (bpc - 8)) + 1, total)).clip(0, bd).astype(dt)
    else:
        pic = rng.integers(0, bd + 1, total).astype(dt)
    til_y = random_tiling(rng, w4, h4)
    til_uv = random_tiling(rng, cw4, ch4, max_log=3)
    masks = build_lf_masks(w4, h4, til_y, til_uv, ss_hor, ss_ver)
    # levels per block (0 sometimes, to exercise the neighbour fallback and the L == 0 skip)
    level = np.zeros((h4 + 32) * b4_stride * 4, np.uint8).reshape(-1, 4)
    lv = level.reshape(h4 + 32, b4_stride, 4)

    def per_block(til, hh, ww):
        bx, by, _, _ = til
        key = by.astype(np.int64) * 65536 + bx
        uniq, inv = np.unique(key, return_inverse=True)
        vals = rng.integers(0, 64, len(uniq)).astype(np.uint8)
        vals[rng.random(len(uniq)) < 0.15] = 0
        return vals[inv].reshape(hh, ww)
    lv[:h4, :w4, 0] = per_block(til_y, h4, w4)
    lv[:h4, :w4, 1] = per_block(til_y, h4, w4)
    lv[:ch4, :cw4, 2] = per_block(til_uv, ch4, cw4)
    lv[:ch4, :cw4, 3] = per_block(til_uv, ch4, cw4)
    e, i, sh = filter_lut(int(rng.integers(0, 8)) if sharp is None else sharp)
    return dict(bpc=bpc, bd=bd, W=W, H=H, w4=w4, h4=h4, sb128w=sb128w, b4_stride=b4_stride, ss_hor=ss_hor,
                ss_ver=ss_ver, stride=stride, off=off, rows=rows, pic=pic, masks=masks, level=level,
                lut_e=e, lut_i=i, lut_sharp=sh, til_y=til_y, til_uv=til_uv)


def make_cdef_params(rng, bw, bh, sb128w, masks, p_unset=0.1, p_noskip=0.8):
    """Fill cdef_idx / noskip_mask of an Av1Filter array in place and draw the frame header strengths
    (frame_hdr->cdef, reference include/dav1d/headers.h). Returns (damping, y_strength[8], uv_strength[8])."""
    sb128h = (bh + 31) // 32
    idx = rng.integers(0, 8, (sb128h * sb128w, 4)).astype(np.int8)
    idx[rng.random(idx.shape) < p_unset] = -1
    masks["cdef_idx"] = idx
    ns = rng.random((sb128h * sb128w, 16, 16)) < p_noskip          # [sb][8x8 row][8x8 col]
    bits = np.zeros((sb128h * sb128w, 16, 2), np.uint16)
    for h in range(2):
        w = (3 << (2 * np.arange(8))).astype(np.uint32)
        bits[:, :, h] = (ns[:, :, h * 8:(h + 1) * 8] * w[None, None, :]).sum(axis=2).astype(np.uint16)
    masks["noskip_mask"] = bits
    y = rng.integers(0, 64, 8); uv = rng.integers(0, 64, 8)
    y[rng.random(8) < 0.2] = 0; uv[rng.random(8) < 0.2] = 0
    y[0] &= 3                     # one entry with secondary-only luma
    uv[1] &= ~3                   # one with primary-only chroma
    return int(rng.integers(3, 7)), [int(v) for v in y], [int(v) for v in uv]


# byte-identical to dav1d's Av1Restoration (reference src/lf_mask.h:42-62): lr[3 planes][4 units] x 9 bytes
LR_UNIT_DT = np.dtype([("type", "u1"), ("filter_h", "i1", (3,)), ("filter_v", "i1", (3,)), ("sgr_weights", "i1", (2,))])
AV1RESTORATION_DT = np.dtype([("lr", LR_UNIT_DT, (3, 4))])
assert AV1RESTORATION_DT.itemsize == 108
SGR_PARAMS = [(140, 3236), (112, 2158), (93, 1618), (80, 1438), (70, 1295), (58, 1177), (47, 1079), (37, 996),
              (30, 925), (25, 863), (0, 2589), (0, 1618), (0, 1177), (0, 925), (56, 0), (22, 0)]


def make_lr_params(rng, W, H, p_none=0.25):
    """Random legal loop-restoration units in dav1d's lr_mask layout. type: 0 none, 2 Wiener,
    3 + sgr_idx self-guided (reference src/lr_apply_tmpl.c:53-84)."""
    sb128w, sb128h = (W + 127) >> 7, (H + 127) >> 7
    m = np.zeros(sb128h * sb128w, AV1RESTORATION_DT)
    u = m["lr"]
    n = u["type"].shape
    kind = rng.random(n)
    typ = np.where(kind < p_none, 0, np.where(kind < p_none + (1 - p_none) / 2, 2, 3 + rng.integers(0, 16, n))).astype(np.uint8)
    u["type"] = typ
    u["filter_h"][..., 0] = rng.integers(-5, 11, n); u["filter_h"][..., 1] = rng.integers(-23, 9, n); u["filter_h"][..., 2] = rng.integers(-17, 47, n)
    u["filter_v"][..., 0] = rng.integers(-5, 11, n); u["filter_v"][..., 1] = rng.integers(-23, 9, n); u["filter_v"][..., 2] = rng.integers(-17, 47, n)
    u["filter_h"][:, 1:, :, 0] = 0; u["filter_v"][:, 1:, :, 0] = 0          # chroma uses the 5-tap form
    idx = np.clip(typ.astype(np.int32) - 3, 0, 15)
    s0 = np.array([p[0] for p in SGR_PARAMS])[idx]; s1 = np.array([p[1] for p in SGR_PARAMS])[idx]
    u["sgr_weights"][..., 0] = np.where(s0 > 0, rng.integers(-96, 32, n), 0)
    u["sgr_weights"][..., 1] = np.where(s1 > 0, rng.integers(-32, 96, n), 95)
    return m


# ------------------------------------------------------------------------------------------
# whole inter frame (BASELINE configs 2-4): prediction + residual + post-filter records
# ------------------------------------------------------------------------------------------
import os as _os
from . import levels as _L

MC_BLOCK_DT = np.dtype([("dst_off", "<u4"), ("src_x", "<i4"), ("src_y", "<i4"), ("w", "u1"), ("h", "u1"), ("mx", "u1"),
                        ("my", "u1"), ("filter2d", "u1"), ("op", "u1"), ("plane", "u1"), ("ref", "u1")])
COMP_BLOCK_DT = np.dtype([("dst_off", "<u4"), ("tmp1_off", "<u4"), ("tmp2_off", "<u4"), ("mask_off", "<u4"), ("w", "u1"),
                          ("h", "u1"), ("op", "u1"), ("param", "u1"), ("plane", "u1"), ("pad", "u1", (3,))])
COMP_FUSED_DT = np.dtype([("dst_off", "<u4"), ("mask_off", "<u4"), ("src_x", "<i4", (2,)), ("src_y", "<i4", (2,)), ("w", "u1"), ("h", "u1"),
                          ("mx", "u1", (2,)), ("my", "u1", (2,)), ("ref", "u1", (2,)), ("filter2d", "u1"), ("op", "u1"), ("param", "u1"),
                          ("plane", "u1"), ("pad", "u1", (4,))])
assert COMP_FUSED_DT.itemsize == 40
ITX_BLOCK_DT = np.dtype([("dst_off", "<u4"), ("coef_off", "<u4"), ("eob", "<i2"), ("txtp", "u1"), ("plane", "u1")])
assert MC_BLOCK_DT.itemsize == 20 and COMP_BLOCK_DT.itemsize == 24 and ITX_BLOCK_DT.itemsize == 12
BLEND_BLOCK_DT = np.dtype([("dst_off", "<u4"), ("tmp_off", "<u4"), ("mask_off", "<u4"), ("w", "u1"), ("h", "u1"), ("op", "u1"), ("plane", "u1")])
WARP_BLOCK_DT = np.dtype([("dst_off", "<u4"), ("src_x", "<i4"), ("src_y", "<i4"), ("mx", "<i4"), ("my", "<i4"), ("abcd", "<i2", (4,)),
                          ("tmp_stride", "<u2"), ("op", "u1"), ("plane", "u1"), ("ref", "u1"), ("pad", "u1", (3,))])
assert BLEND_BLOCK_DT.itemsize == 16 and WARP_BLOCK_DT.itemsize == 36
TX_FROM_WH = {(_L.TX_W[t], _L.TX_H[t]): t for t in range(19)}
_scans = None


def scan_table(tx):
    """dav1d_scans[tx] (committed copy generated from the reference, tests/golden/make_golden.py)."""
    global _scans
    if _scans is None:
        _scans = np.load(_os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "data", "scans.npz"))
    return _scans["tx%d" % tx].astype(np.int64)


def smooth_picture(rng, total, bd, dt):
    """low-pass filtered noise so that sub-pel interpolation is non-trivial"""
    base = rng.integers(0, bd + 1, total // 16 + 2).astype(np.int32)
    up = np.repeat(base, 16)[:total]
    up = (up + np.roll(up, 5) + np.roll(up, 11) + np.roll(up, 23)) // 4
    return (up + rng.integers(-6, 7, total)).clip(0, bd).astype(dt)


def make_film_grain(rng, full=True):
    """random Dav1dFilmGrainData in the ranges of tests/checkasm/filmgrain.c (:62-75, :160-215)"""
    from . import _lib
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


def make_inter_frame(rng, bpc, W, H, ss_hor=1, ss_ver=1, n_refs=2, p_compound=0.3, p_skip=0.25, min_log=1, max_log=4,
                     film_grain=False, p_intra=0.0, p_obmc=0.0, p_warp=0.0, p_ii=0.0):
    """Synthetic inter frame: every block is predicted from `n_refs` reference pictures (single or
    compound), carries a residual (unless skipped) and the frame has deblock / CDEF / LR parameters.
    p_obmc / p_warp / p_ii: share of the single-reference blocks of 8x8 luma samples and more that use overlapped block
    motion compensation (predictions with the neighbours' motion blended over the top rows / left columns: B200McBlock op 2
    + B200BlendBlock, what obmc() does, reference src/recon_tmpl.c:1052-1113), an affine warp (B200WarpBlock per 8x8,
    warp_affine :1115-1165) or an inter-intra blend (B200_INTRA_MODE_II + RESID records, :1601-1626, 1737-1777).
    p_intra > 0: that share of the blocks is intra coded instead (what real inter frames contain): B200IntraTx records
    (S["intra_tx"], wavefront order among themselves) + S["done_init"], the done map in which every cell of an inter block
    is final before the intra kernel starts (include/b200av1.h, B200IntraFrame.done_init)."""
    bd = (1 << bpc) - 1
    dt = np.uint8 if bpc == 8 else np.uint16
    cdt = np.int16 if bpc == 8 else np.int32
    S = make_lf_frame(rng, bpc, W, H, ss_hor, ss_ver)          # geometry + placeholder masks (rebuilt below)
    stride, off = S["stride"], S["off"]
    total = len(S["pic"])
    w4, h4 = S["w4"], S["h4"]
    ssh, ssv = [0, ss_hor, ss_hor], [0, ss_ver, ss_ver]
    refs = [smooth_picture(rng, total, bd, dt) for _ in range(n_refs)]
    decode_order = []
    bx, by, lw, lh = random_tiling(rng, w4, h4, max_log=max_log, min_log=min_log, order=decode_order)
    if p_intra > 0 or p_ii > 0:
        blocks = [b for b in decode_order if b[0] < w4 and b[1] < h4]      # intra blocks need their neighbours first: decode order
    else:
        key = by.astype(np.int64) * 65536 + bx
        _, first = np.unique(key, return_index=True)
        blocks = [(int(bx.flat[i]), int(by.flat[i]), int(lw.flat[i]), int(lh.flat[i])) for i in first]
    intra_recs = []
    pw4 = [w4, (w4 + ss_hor) >> ss_hor, (w4 + ss_hor) >> ss_hor]; ph4 = [h4, (h4 + ss_ver) >> ss_ver, (h4 + ss_ver) >> ss_ver]
    edge_filter = int(rng.integers(0, 2)) if p_intra > 0 else 0
    warp, blend, blend2 = [], [], []
    px_tmp_off = 0

    def add_intra(pl, x, y, tlw, tlh, mode, angle, skip):
        """one intra transform block of plane pl at (x, y) [plane 4-sample units] (cf. make_intra_frame.add)"""
        r = np.zeros(1, INTRA_TX_DT)[0]
        r["dst_off"] = off[pl] + y * 4 * stride[pl] + x * 4
        r["x4"], r["y4"], r["xend4"], r["yend4"] = x, y, pw4[pl], ph4[pl]
        if pl == 0:
            r["max_w"], r["max_h"] = 4 * w4 - 4 * x, 4 * h4 - 4 * y
        else:
            r["max_w"] = (4 * w4 + ss_hor - 4 * (x << ss_hor)) >> ss_hor
            r["max_h"] = (4 * h4 + ss_ver - 4 * (y << ss_ver)) >> ss_ver
        r["angle_flags"] = edge_filter << 10
        r["tx"] = TX_FROM_WH[(4 << tlw, 4 << tlh)]
        r["mode"], r["angle"], r["plane"] = mode, angle, pl
        r["flags"] = (1 if x > 0 else 0) | (2 if y > 0 else 0)        # top-right / bottom-left never used: always a valid choice
        r["eob"] = -1 if skip else 0                                  # residual filled in below
        intra_recs.append(r)
        return r

    pred, comp, comp2 = [], [], []
    pred_single, cfused, cfused2 = [], [], []  # the same predictions for the fused compound kernel
    itx = {t: [] for t in range(19)}          # tx -> list of (dst_off, plane, txtp)
    tmp_off, mask_off = 0, 0
    # transform tilings for the deblocking masks (tx granularity)
    ty = [np.zeros((h4, w4), np.int32), np.zeros((h4, w4), np.int32), np.zeros((h4, w4), np.int8), np.zeros((h4, w4), np.int8)]
    cw4, ch4 = (w4 + ss_hor) >> ss_hor, (h4 + ss_ver) >> ss_ver
    tuv = [np.zeros((ch4, cw4), np.int32), np.zeros((ch4, cw4), np.int32), np.zeros((ch4, cw4), np.int8), np.zeros((ch4, cw4), np.int8)]
    skip_map = np.zeros((h4, w4), bool)

    def paint(t, x, y, lwv, lhv, hh, ww):
        x1, y1 = min(ww, x + (1 << lwv)), min(hh, y + (1 << lhv))
        if x < ww and y < hh:
            t[0][y:y1, x:x1] = x; t[1][y:y1, x:x1] = y; t[2][y:y1, x:x1] = lwv; t[3][y:y1, x:x1] = lhv

    for (x4, y4, lwv, lhv) in blocks:
        bw, bh = 4 << lwv, 4 << lhv
        if p_intra > 0 and rng.random() < p_intra:
            # ---- an intra block inside the inter frame: predicted from its reconstructed neighbours at transform-block
            # granularity (the neighbours may be inter blocks: final before the intra kernel starts)
            skip = rng.random() < p_skip
            skip_map[y4:y4 + (1 << lhv), x4:x4 + (1 << lwv)] = skip
            cwb, chb = min(1 << lwv, w4 - x4), min(1 << lhv, h4 - y4)
            m = int(rng.integers(0, 13)); ang = int(rng.integers(-3, 4)) if 1 <= m <= 8 else 0
            tlw, tlh = min(lwv, 4), min(lhv, 4)
            if rng.random() < 0.4 and tlw > 0 and tlh > 0:
                tlw -= 1; tlh -= 1
            for yy in range(0, chb, 1 << tlh):
                for xx in range(0, cwb, 1 << tlw):
                    paint(ty, x4 + xx, y4 + yy, tlw, tlh, h4, w4)
                    add_intra(0, x4 + xx, y4 + yy, tlw, tlh, m, ang, skip)
            clw, clh = max(lwv - ss_hor, 0), max(lhv - ss_ver, 0)
            cx4, cy4 = x4 >> ss_hor, y4 >> ss_ver
            ccw, cch = (cwb + ss_hor) >> ss_hor, (chb + ss_ver) >> ss_ver
            um = int(rng.integers(0, 13)); uang = int(rng.integers(-3, 4)) if 1 <= um <= 8 else 0
            ctl, cth = min(clw, 3), min(clh, 3)
            for pl in (1, 2):
                for yy in range(0, cch, 1 << cth):
                    for xx in range(0, ccw, 1 << ctl):
                        if pl == 1:
                            paint(tuv, cx4 + xx, cy4 + yy, ctl, cth, ch4, cw4)
                        add_intra(pl, cx4 + xx, cy4 + yy, ctl, cth, um, uang, skip)
            continue
        compound = rng.random() < p_compound
        motion = None
        inside = x4 + (1 << lwv) <= w4 and y4 + (1 << lhv) <= h4
        if not compound and inside and min(bw, bh) >= 8 and (p_obmc or p_warp or p_ii):
            u = rng.random()
            if u < p_warp:
                motion = "warp"
            elif u < p_warp + p_obmc:
                motion = "obmc"
            elif u < p_warp + p_obmc + p_ii and max(bw, bh) <= 32 and max(bw, bh) <= 2 * min(bw, bh):
                motion = "ii"
        mv = [(int(rng.integers(-512, 513)), int(rng.integers(-512, 513))) for _ in range(2)]   # 1/8 luma pixels
        if rng.random() < 0.05:
            mv[0] = (mv[0][0] & ~7, mv[0][1] & ~7)                                              # integer-pel sometimes
        f2d = int(rng.integers(0, 10))
        rf = [int(rng.integers(0, n_refs)), int(rng.integers(0, n_refs))]
        cop = int(rng.choice([0, 0, 0, 0, 0, 1, 1, 1, 2, 5])) if compound else -1   # avg 50 / w_avg 30 / wedge 10 / seg 10
        cparam = int(rng.integers(1, 16)) if cop == 1 else int(rng.integers(0, 2))
        luma_mask_off = None
        for pl in range(3):
            w, h = bw >> ssh[pl], bh >> ssv[pl]
            px, py = (x4 * 4) >> ssh[pl], (y4 * 4) >> ssv[pl]
            dst_off = off[pl] + py * stride[pl] + px
            n = 2 if compound else 1
            offs, srcs = [], []
            for k in range(n):
                mvx, mvy = mv[k]
                if pl == 0 or not ss_hor:
                    sx, mx = px + (mvx >> 3), (mvx & 7) << 1
                else:
                    sx, mx = px + (mvx >> 4), mvx & 15
                if pl == 0 or not ss_ver:
                    sy, my = py + (mvy >> 3), (mvy & 7) << 1
                else:
                    sy, my = py + (mvy >> 4), mvy & 15
                srcs.append((sx, sy, mx, my))
                if compound:
                    pred.append((tmp_off, sx, sy, w, h, mx, my, f2d, 1, pl, rf[k])); offs.append(tmp_off); tmp_off += w * h
                elif motion == "warp" and min(w, h) >= 8:
                    # one record per 8x8 of the block; the matrix of the block is shared, the per-8x8 positions / phases are
                    # what warp_affine derives from it (here: drawn, the kernel does not care where they come from)
                    abcd = [int(v) for v in rng.integers(-2048, 2049, 4)]
                    for yy in range(0, h, 8):
                        for xx in range(0, w, 8):
                            warp.append((dst_off + yy * stride[pl] + xx, sx + xx + int(rng.integers(-2, 3)), sy + yy + int(rng.integers(-2, 3)),
                                         int(rng.integers(0, 1 << 16)) & ~0x3f, int(rng.integers(0, 1 << 16)) & ~0x3f, abcd, 0, 0, pl, rf[k], (0, 0, 0)))
                else:
                    pred.append((dst_off, sx, sy, w, h, mx, my, f2d, 0, pl, rf[k]))
                    pred_single.append(pred[-1])
            if motion == "obmc":
                # predictions with the motion of the block above over the top rows (3/4 of half the block height are computed,
                # blend_h blends them) and of the block to the left over the left columns (blend_v)
                def lap(wl, hl):
                    nonlocal px_tmp_off
                    mvx, mvy = int(rng.integers(-512, 513)), int(rng.integers(-512, 513))
                    sxl, mxl = (px + (mvx >> 3), (mvx & 7) << 1) if (pl == 0 or not ss_hor) else (px + (mvx >> 4), mvx & 15)
                    syl, myl = (py + (mvy >> 3), (mvy & 7) << 1) if (pl == 0 or not ss_ver) else (py + (mvy >> 4), mvy & 15)
                    rec = (px_tmp_off, sxl, syl, wl, hl, mxl, myl, int(rng.integers(0, 10)), 2, pl, int(rng.integers(0, n_refs)))
                    pred.append(rec); pred_single.append(rec)
                    o = px_tmp_off; px_tmp_off += wl * hl
                    return o
                h_mul, v_mul = 4 >> ssh[pl], 4 >> ssv[pl]
                if y4 > 0:
                    oh4 = min(1 << lhv, 16) >> 1
                    o = lap(w, ((oh4 * 3 + 3) >> 2) * v_mul)
                    blend.append((dst_off, o, 0, w, v_mul * oh4, 2, pl))
                if x4 > 0:
                    ow4 = min(1 << lwv, 16) >> 1
                    o = lap(h_mul * ow4, h)
                    blend2.append((dst_off, o, 0, h_mul * ow4, h, 1, pl))
            if motion == "ii":
                r = add_intra(pl, (x4 * 4 >> ssh[pl]) >> 2, (y4 * 4 >> ssv[pl]) >> 2, 0, 0, 15, int(rng.choice([0, 1, 2, 9])), True)
                r["tx"] = TX_FROM_WH[(w, h)]
                r["luma_off"] = mask_off; mask_off += w * h
                intra_recs[-1] = r
            if compound:
                def fused(moff, op_, par):
                    return (dst_off, moff, (srcs[0][0], srcs[1][0]), (srcs[0][1], srcs[1][1]), w, h, (srcs[0][2], srcs[1][2]),
                            (srcs[0][3], srcs[1][3]), (rf[0], rf[1]), f2d, op_, par, pl, (0, 0, 0, 0))
                if cop == 5:           # segment mask: luma derives it (w_mask), chroma consumes it (mask)
                    if pl == 0:
                        lay = 3 + (ss_hor + ss_ver)           # w_mask_444 / 422 / 420
                        luma_mask_off = mask_off
                        comp.append((dst_off, offs[0], offs[1], mask_off, w, h, lay, cparam, pl, (0, 0, 0)))
                        cfused.append(fused(mask_off, lay, cparam))
                        mask_off += w * h
                    else:
                        comp2.append((dst_off, offs[0], offs[1], luma_mask_off, w, h, 2, 0, pl, (0, 0, 0)))
                        cfused2.append(fused(luma_mask_off, 2, 0))
                elif cop == 2:         # wedge: explicit mask from the host
                    comp.append((dst_off, offs[0], offs[1], mask_off, w, h, 2, 0, pl, (0, 0, 0)))
                    cfused.append(fused(mask_off, 2, 0)); mask_off += w * h
                else:
                    comp.append((dst_off, offs[0], offs[1], 0, w, h, cop, cparam, pl, (0, 0, 0)))
                    cfused.append(fused(0, cop, cparam))
        # residual: transform tiling of the block (var-tx split depth <= 1), capped at 64
        skip = rng.random() < p_skip
        skip_map[y4:y4 + (1 << lhv), x4:x4 + (1 << lwv)] = skip
        if motion == "ii":
            # the residual of an inter-intra block goes through the intra machine as RESID records (after the blend); the II
            # records just appended say whether any follow
            for r in intra_recs[-3:]:
                r["cfl_alpha"] = 0 if skip else 1
        tlw, tlh = min(lwv, 4), min(lhv, 4)
        if rng.random() < 0.3 and tlw > 0 and tlh > 0:
            tlw -= 1; tlh -= 1
        for yy in range(y4, y4 + (1 << lhv), 1 << tlh):
            for xx in range(x4, x4 + (1 << lwv), 1 << tlw):
                paint(ty, xx, yy, tlw, tlh, h4, w4)
                if not skip and xx < w4 and yy < h4:
                    tx = TX_FROM_WH[(4 << tlw, 4 << tlh)]
                    if motion == "ii":
                        add_intra(0, xx, yy, tlw, tlh, 16, 0, False)
                    else:
                        itx[tx].append((off[0] + yy * 4 * stride[0] + xx * 4, 0))
        # chroma: one transform per block, capped at 32 (64x64 luma -> 32x32 chroma)
        clw, clh = max(lwv - ss_hor, 0), max(lhv - ss_ver, 0)
        cx4, cy4 = x4 >> ss_hor, y4 >> ss_ver
        ctl, cth = min(clw, 3), min(clh, 3)
        for yy in range(cy4, cy4 + (1 << clh), 1 << cth):
            for xx in range(cx4, cx4 + (1 << clw), 1 << ctl):
                paint(tuv, xx, yy, ctl, cth, ch4, cw4)
                if not skip and xx < cw4 and yy < ch4:
                    tx = TX_FROM_WH[(4 << ctl, 4 << cth)]
                    for pl in (1, 2):
                        if motion == "ii":
                            add_intra(pl, xx, yy, ctl, cth, 16, 0, False)
                        else:
                            itx[tx].append((off[pl] + yy * 4 * stride[pl] + xx * 4, pl))

    # ---- coefficient stream (vectorised per transform size) ----
    coef_chunks, itx_arrays, coef_off = [], {}, 0
    for tx in range(19):
        lst = itx[tx]
        if not lst:
            itx_arrays[tx] = np.zeros(0, ITX_BLOCK_DT)
            continue
        n = len(lst)
        sw, sh = _L.tx_coef_dims(tx)
        ncf = sw * sh
        legal = [tp for tp in range(10) if _L.itx_defined(tx, tp)]          # 2-D transform classes only
        txtp = rng.choice(legal, n, p=None if len(legal) == 1 else [0.55] + [0.45 / (len(legal) - 1)] * (len(legal) - 1))
        scan = scan_table(tx)
        inv = np.empty(ncf, np.int64); inv[scan] = np.arange(ncf)          # coefficient index -> scan position
        eob = np.minimum((rng.exponential(ncf / 10.0, n)).astype(np.int64), ncf - 1)
        eob[rng.random(n) < 0.25] = 0                                        # dc-only blocks
        amp = (bd + 1) / 2.0
        pos = inv[None, :]
        mag = rng.laplace(0.0, amp * 0.35, (n, ncf)) / (1.0 + pos / 6.0)
        c = np.rint(mag).astype(np.int64)
        c[pos > eob[:, None]] = 0
        c[np.arange(n), scan[eob]] = np.where(c[np.arange(n), scan[eob]] == 0, 1, c[np.arange(n), scan[eob]])
        arr = np.zeros(n, ITX_BLOCK_DT)
        arr["dst_off"] = [d for d, _ in lst]; arr["plane"] = [p for _, p in lst]
        arr["coef_off"] = coef_off + np.arange(n) * ncf
        arr["eob"] = eob; arr["txtp"] = txtp
        itx_arrays[tx] = arr
        coef_chunks.append(c.astype(cdt).reshape(-1))
        coef_off += n * ncf
    intra_extra = {}
    if intra_recs:
        tx = np.array(intra_recs, INTRA_TX_DT)
        for t in range(19):
            sel = np.nonzero((tx["tx"] == t) & (tx["eob"] >= 0))[0]
            if not len(sel):
                continue
            k = len(sel)
            sw, sh = _L.tx_coef_dims(t)
            ncf = sw * sh
            legal = [tp for tp in range(10) if _L.itx_defined(t, tp)]
            txtp = rng.choice(legal, k, p=None if len(legal) == 1 else [0.55] + [0.45 / (len(legal) - 1)] * (len(legal) - 1))
            scan = scan_table(t)
            inv = np.empty(ncf, np.int64); inv[scan] = np.arange(ncf)
            eob = np.minimum((rng.exponential(ncf / 10.0, k)).astype(np.int64), ncf - 1)
            eob[rng.random(k) < 0.25] = 0
            pos = inv[None, :]
            c = np.rint(rng.laplace(0.0, (bd + 1) / 2.0 * 0.25, (k, ncf)) / (1.0 + pos / 6.0)).astype(np.int64)
            c[pos > eob[:, None]] = 0
            c[np.arange(k), scan[eob]] = np.where(c[np.arange(k), scan[eob]] == 0, 1, c[np.arange(k), scan[eob]])
            tx["coef_off"][sel] = coef_off + np.arange(k) * ncf
            tx["eob"][sel] = eob; tx["txtp"][sel] = txtp
            coef_chunks.append(c.astype(cdt).reshape(-1))
            coef_off += k * ncf
        # wavefront numbers among the intra records (cells of inter blocks are final from the start: depth 0)
        wave_map = [np.zeros((ph4[p], pw4[p]), np.int32) for p in range(3)]
        covered = [np.zeros((ph4[p], pw4[p]), bool) for p in range(3)]
        wave = np.zeros(len(tx), np.int64)
        for i in range(len(tx)):
            r = tx[i]
            pl, x, y = int(r["plane"]), int(r["x4"]), int(r["y4"])
            tw, th = _L.TX_W[r["tx"]] // 4, _L.TX_H[r["tx"]] // 4
            wm = wave_map[pl]
            dep = 0
            if r["mode"] == 16:                        # RESID: after the II record that predicted these cells
                wave[i] = int(wm[y:y + th, x:x + tw].max()) + 1
                wm[y:y + th, x:x + tw] = wave[i]
                continue
            if x > 0:
                dep = max(dep, int(wm[y:y + min(th, ph4[pl] - y), x - 1].max()))
            if y > 0:
                dep = max(dep, int(wm[y - 1, x:x + min(tw, pw4[pl] - x)].max()))
            if x > 0 and y > 0:
                dep = max(dep, int(wm[y - 1, x - 1]))
            wave[i] = dep + 1
            wm[y:y + th, x:x + tw] = dep + 1
            covered[pl][y:y + th, x:x + tw] = True
        # done map image (b200_intra_scratch_bytes layout): 256 zero bytes, then one byte per 4x4 cell of plane 0, 1, 2,
        # each map padded to a multiple of 256 bytes; 1 = final before the kernel starts (not covered by an intra record)
        parts = [np.zeros(256, np.uint8)]
        for p in range(3):
            mcell = (~covered[p]).astype(np.uint8).reshape(-1)
            parts.append(np.concatenate([mcell, np.zeros((-len(mcell)) % 256, np.uint8)]))
        intra_extra = dict(intra_tx=tx[np.argsort(wave, kind="stable")].copy(), intra_tx_decode_order=tx, intra_waves=int(wave.max()),
                           done_init=np.concatenate(parts))
    coefs = np.concatenate(coef_chunks) if coef_chunks else np.zeros(1, cdt)

    def to_arr(lst, dtp):
        a = np.zeros(len(lst), dtp)
        for i, rec in enumerate(lst):
            a[i] = rec
        return a
    def by_area(a):
        """records bucketed by block area, largest first (what a record emitter would do with one list per size class):
        the warps of a CTA then work on blocks of the same size and the long blocks start first"""
        if not len(a):
            return a
        return a[np.argsort(-(a["w"].astype(np.int64) * a["h"]), kind="stable")]
    S.update(refs=refs, pred=by_area(to_arr(pred, MC_BLOCK_DT)), comp=by_area(to_arr(comp, COMP_BLOCK_DT)),
             comp2=by_area(to_arr(comp2, COMP_BLOCK_DT)), pred_single=by_area(to_arr(pred_single, MC_BLOCK_DT)),
             cfused=by_area(to_arr(cfused, COMP_FUSED_DT)), cfused2=by_area(to_arr(cfused2, COMP_FUSED_DT)),
             itx=itx_arrays, coefs=coefs, tmp_len=tmp_off + 64, mask=rng.integers(0, 65, max(1, mask_off)).astype(np.uint8))
    if warp or blend or blend2:
        S.update(warp=to_arr(warp, WARP_BLOCK_DT), blend=by_area(to_arr(blend, BLEND_BLOCK_DT)), blend2=by_area(to_arr(blend2, BLEND_BLOCK_DT)),
                 px_tmp_len=px_tmp_off + 64)
    S.update(intra_extra)
    S["pic"] = np.zeros(total, dt)                     # the picture being reconstructed
    # post-filter records from the transform tilings
    S["masks"] = build_lf_masks(w4, h4, tuple(ty), tuple(tuv), ss_hor, ss_ver)
    S["til_y"], S["til_uv"] = tuple(ty), tuple(tuv)
    S["bw"], S["bh"] = w4, h4
    S["damping"], S["y_strength"], S["uv_strength"] = make_cdef_params(rng, w4, h4, S["sb128w"], S["masks"])
    # noskip_mask from the real skip flags (reference src/decode.c:1946-1955)
    sb128h = (h4 + 31) // 32
    ns8 = np.zeros((sb128h * 16, S["sb128w"] * 16), bool)
    nsk = ~skip_map
    hh, ww = (h4 + 1) // 2, (w4 + 1) // 2
    pad = np.zeros((hh * 2, ww * 2), bool); pad[:h4, :w4] = nsk
    ns8[:hh, :ww] = pad.reshape(hh, 2, ww, 2).any(axis=(1, 3))
    t = ns8.reshape(sb128h, 16, S["sb128w"], 16).transpose(0, 2, 1, 3).reshape(-1, 16, 16)
    bits = np.zeros((t.shape[0], 16, 2), np.uint16)
    wgt = (3 << (2 * np.arange(8))).astype(np.uint32)
    for h in range(2):
        bits[:, :, h] = (t[:, :, h * 8:(h + 1) * 8] * wgt[None, None, :]).sum(axis=2).astype(np.uint16)
    S["masks"]["noskip_mask"] = bits
    S["lr_mask"] = make_lr_params(rng, W, H)
    S["us"] = (6, 6 - (1 if ss_hor else 0))
    S["rp"], S["sb128"] = 7, 0
    if film_grain:
        d = make_film_grain(rng, full=False)
        d.overlap_flag = 1
        S["fg"] = d
    return S


# ---------------------------------------------------------------------------------------------------------
# intra frames: transform-block records for b200_intra_frame (include/b200av1.h, B200IntraTx)
INTRA_TX_DT = np.dtype([("dst_off", "<u4"), ("coef_off", "<u4"), ("luma_off", "<u4"), ("eob", "<i2"), ("x4", "<u2"), ("y4", "<u2"),
                        ("xend4", "<u2"), ("yend4", "<u2"), ("max_w", "<i2"), ("max_h", "<i2"), ("angle_flags", "<u2"),
                        ("tx", "u1"), ("txtp", "u1"), ("mode", "u1"), ("angle", "i1"), ("plane", "u1"), ("flags", "u1"),
                        ("cfl_alpha", "i1"), ("cfl_w_pad", "u1"), ("cfl_h_pad", "u1"), ("pad", "u1", (3,))])
assert INTRA_TX_DT.itemsize == 40
INTRA_SB_DT = np.dtype([("first", "<u4"), ("count", "<u4"), ("sx", "<u2"), ("sy", "<u2")])
_SMOOTH_MODES = (9, 10, 11)
MODE_FILTER, MODE_CFL = 13, 14


def ordered_tiling(rng, w4, h4, max_log=4, min_log=1, p_split=0.6):
    """Blocks (x4, y4, lw, lh) in decode order: superblock raster, recursive partition order inside."""
    out = []
    S = 1 << max_log

    def rec(x, y, lwv, lhv):
        if x >= w4 or y >= h4:
            return
        can_w, can_h = lwv > min_log, lhv > min_log
        if (can_w or can_h) and rng.random() < p_split:
            mode = rng.integers(0, 3)
            if mode == 0 and can_w and can_h:
                for dy in (0, 1):
                    for dx in (0, 1):
                        rec(x + (dx << (lwv - 1)), y + (dy << (lhv - 1)), lwv - 1, lhv - 1)
                return
            if (mode == 1 or not can_h) and can_w and lwv >= lhv:
                rec(x, y, lwv - 1, lhv); rec(x + (1 << (lwv - 1)), y, lwv - 1, lhv)
                return
            if can_h and lhv >= lwv:
                rec(x, y, lwv, lhv - 1); rec(x, y + (1 << (lhv - 1)), lwv, lhv - 1)
                return
        out.append((x, y, lwv, lhv))
    for y in range(0, h4, S):
        for x in range(0, w4, S):
            rec(x, y, max_log, max_log)
    return out


MODE_RESID, MODE_IBC = 16, 18


def make_intra_frame(rng, bpc, W, H, ss_hor=1, ss_ver=1, p_skip=0.2, p_cfl=0.25, p_ibc=0.0):
    """Synthetic intra-only frame (BASELINE configs[1]): every block intra predicted (all 13 modes with angle deltas,
    filter-intra, CFL) at transform-block granularity + residual, deblocking parameters. W, H multiples of 8
    (dav1d's f->bw / f->bh are even). Availability of the top-right / bottom-left neighbours follows decode order
    geometrically (a superset of the bitstream rule; what matters to the kernels is that it is consistent).
    p_ibc: that share of the blocks below the first superblock row is an intra block copy instead (B200_INTRA_MODE_IBC, one
    record per plane + RESID records): copied, with dav1d's bilinear put, from anywhere in the superblock rows above — whole
    luma samples, hence half-sample phases in sub-sampled chroma for odd vectors (reference src/recon_tmpl.c:1583-1596)."""
    assert W % 8 == 0 and H % 8 == 0
    bd = (1 << bpc) - 1
    dt = np.uint8 if bpc == 8 else np.uint16
    cdt = np.int16 if bpc == 8 else np.int32
    S = make_lf_frame(rng, bpc, W, H, ss_hor, ss_ver)
    stride, off = S["stride"], S["off"]
    w4, h4 = S["w4"], S["h4"]
    ssh, ssv = [0, ss_hor, ss_hor], [0, ss_ver, ss_ver]
    pw4 = [w4, w4 >> ss_hor, w4 >> ss_hor]; ph4 = [h4, h4 >> ss_ver, h4 >> ss_ver]
    edge_filter = int(rng.integers(0, 2))
    order = [np.full((ph4[p], pw4[p]), -1, np.int64) for p in range(3)]       # owning record (decode order) per 4x4 cell
    ymode = np.zeros((h4, w4), np.int8); uvmode = np.zeros((h4, w4), np.int8)
    ty = [np.zeros((h4, w4), np.int32), np.zeros((h4, w4), np.int32), np.zeros((h4, w4), np.int8), np.zeros((h4, w4), np.int8)]
    cw4, ch4 = (w4 + ss_hor) >> ss_hor, (h4 + ss_ver) >> ss_ver
    tuv = [np.zeros((ch4, cw4), np.int32), np.zeros((ch4, cw4), np.int32), np.zeros((ch4, cw4), np.int8), np.zeros((ch4, cw4), np.int8)]
    recs = []

    def paint(t, x, y, lwv, lhv, hh, ww):
        x1, y1 = min(ww, x + (1 << lwv)), min(hh, y + (1 << lhv))
        t[0][y:y1, x:x1] = x; t[1][y:y1, x:x1] = y; t[2][y:y1, x:x1] = lwv; t[3][y:y1, x:x1] = lhv

    def is_sm(m):
        return 512 if m in _SMOOTH_MODES else 0

    def add(pl, x, y, tlw, tlh, mode, angle, sm, skip, bx4, by4, cfl=None):
        """one transform block of plane pl at (x, y) [plane 4-sample units]"""
        tw, th = 1 << tlw, 1 << tlh
        idx = len(recs)
        om = order[pl]
        fl = (1 if x > 0 else 0) | (2 if y > 0 else 0)
        if cfl is None or cfl[0] == 0:
            if y > 0 and x + tw < pw4[pl] and 0 <= om[y - 1, x + tw]:
                fl |= 4
            if x > 0 and y + th < ph4[pl] and 0 <= om[y + th, x - 1]:
                fl |= 8
        om[y:y + th, x:x + tw] = idx
        r = np.zeros(1, INTRA_TX_DT)[0]
        r["dst_off"] = off[pl] + y * 4 * stride[pl] + x * 4
        r["x4"], r["y4"], r["xend4"], r["yend4"] = x, y, pw4[pl], ph4[pl]
        if pl == 0:
            r["max_w"], r["max_h"] = 4 * w4 - 4 * x, 4 * h4 - 4 * y
        else:
            r["max_w"] = (4 * w4 + ss_hor - 4 * (x << ss_hor)) >> ss_hor
            r["max_h"] = (4 * h4 + ss_ver - 4 * (y << ss_ver)) >> ss_ver
        r["angle_flags"] = sm | (edge_filter << 10)
        r["tx"] = TX_FROM_WH[(4 * tw, 4 * th)]
        r["mode"], r["angle"], r["plane"], r["flags"] = mode, angle, pl, fl
        r["eob"] = -1 if skip else 0           # residual filled in below
        if cfl is not None:
            r["cfl_alpha"], r["cfl_w_pad"], r["cfl_h_pad"] = cfl
            r["luma_off"] = off[0] + (by4 & ~ss_ver) * 4 * stride[0] + (bx4 & ~ss_hor) * 4
        recs.append(r)

    def add_ibc(pl, x, y, tw, th, sx, sy, mx, my, resid):
        """an IBC record of plane pl: block at (x, y), tw x th [4-sample units], source sample position (sx, sy) + phase"""
        r = np.zeros(1, INTRA_TX_DT)[0]
        r["dst_off"] = off[pl] + y * 4 * stride[pl] + x * 4
        r["x4"], r["y4"], r["xend4"], r["yend4"] = x, y, pw4[pl], ph4[pl]
        r["tx"] = TX_FROM_WH[(4 * tw, 4 * th)]
        r["mode"], r["plane"], r["eob"] = MODE_IBC, pl, -1
        r["luma_off"] = (sy << 16) | sx
        r["cfl_w_pad"], r["cfl_h_pad"], r["cfl_alpha"] = mx, my, 1 if resid else 0
        order[pl][y:y + th, x:x + tw] = len(recs)
        recs.append(r)

    for (x4, y4, lwv, lhv) in ordered_tiling(rng, w4, h4):
        bw4, bh4 = 1 << lwv, 1 << lhv
        cw, chh = min(bw4, w4 - x4), min(bh4, h4 - y4)                         # clipped block size (w4, h4 in :1188)
        skip = rng.random() < p_skip
        small = bw4 <= 8 and bh4 <= 8
        if p_ibc and y4 >= 16 and cw == bw4 and chh == bh4 and rng.random() < p_ibc:
            # ---- intra block copy from the superblock rows above (all of them are reconstructed: superblock raster order)
            sx = int(rng.integers(0, 4 * w4 - 4 * bw4 + 1)); sy = int(rng.integers(0, (y4 >> 4) * 64 - 4 * bh4 + 1))
            dx, dy = sx - 4 * x4, sy - 4 * y4                                   # the (whole-sample) luma vector
            add_ibc(0, x4, y4, bw4, bh4, sx, sy, 0, 0, not skip)
            ymode[y4:y4 + bh4, x4:x4 + bw4] = 0; uvmode[y4:y4 + bh4, x4:x4 + bw4] = 0
            tlw, tlh = min(lwv, 4), min(lhv, 4)
            if rng.random() < 0.5 and tlw > 0 and tlh > 0:
                tlw -= 1; tlh -= 1
            for yy in range(0, bh4, 1 << tlh):
                for xx in range(0, bw4, 1 << tlw):
                    paint(ty, x4 + xx, y4 + yy, tlw, tlh, h4, w4)
                    if not skip:
                        add(0, x4 + xx, y4 + yy, tlw, tlh, MODE_RESID, 0, 0, False, x4, y4)
            clw, clh = lwv - ss_hor, lhv - ss_ver
            cx4, cy4 = x4 >> ss_hor, y4 >> ss_ver
            ctl, cth = min(clw, 3), min(clh, 3)
            for pl in (1, 2):
                # chroma: mv >> (3 + ss) whole samples, (mv & 15) the phase of the bilinear filter (mc(), :948-956)
                csx = (cx4 * 4 + (dx >> 1)) if ss_hor else sx; csy = (cy4 * 4 + (dy >> 1)) if ss_ver else sy
                add_ibc(pl, cx4, cy4, 1 << clw, 1 << clh, csx, csy, (dx & 1) * 8 if ss_hor else 0, (dy & 1) * 8 if ss_ver else 0, not skip)
                for yy in range(0, 1 << clh, 1 << cth):
                    for xx in range(0, 1 << clw, 1 << ctl):
                        if pl == 1:
                            paint(tuv, cx4 + xx, cy4 + yy, ctl, cth, ch4, cw4)
                        if not skip:
                            add(pl, cx4 + xx, cy4 + yy, ctl, cth, MODE_RESID, 0, 0, False, x4, y4)
            continue
        # ---- luma
        m = int(rng.integers(0, 13))
        ang = int(rng.integers(-3, 4)) if 1 <= m <= 8 else 0
        if m == 0 and small and rng.random() < 0.4:
            m, ang = MODE_FILTER, int(rng.integers(0, 5))
        sm = (is_sm(ymode[y4 - 1, x4]) if y4 > 0 else 0) | (is_sm(ymode[y4, x4 - 1]) if x4 > 0 else 0)
        ymode[y4:y4 + chh, x4:x4 + cw] = 0 if m == MODE_FILTER else m          # filter-intra blocks store DC_PRED
        tlw, tlh = min(lwv, 4), min(lhv, 4)
        for _ in range(int(rng.integers(0, 3))):                               # tx split depth 0..2
            if tlw >= tlh and tlw > 0:
                tlw -= 1
                if tlh > tlw + 2:
                    tlh -= 1
            elif tlh > 0:
                tlh -= 1
            if tlw > tlh + 2:
                tlw = tlh + 2
            if tlh > tlw + 2:
                tlh = tlw + 2
        for yy in range(0, chh, 1 << tlh):
            for xx in range(0, cw, 1 << tlw):
                paint(ty, x4 + xx, y4 + yy, tlw, tlh, h4, w4)
                add(0, x4 + xx, y4 + yy, tlw, tlh, m, ang, sm, skip, x4, y4)
        # ---- chroma (every block is at least 8x8 luma, so every block carries chroma)
        clw, clh = lwv - ss_hor, lhv - ss_ver
        cx4, cy4 = x4 >> ss_hor, y4 >> ss_ver
        ccw, cch = (cw + ss_hor) >> ss_hor, (chh + ss_ver) >> ss_ver
        um = int(rng.integers(0, 13))
        uang = int(rng.integers(-3, 4)) if 1 <= um <= 8 else 0
        cfl = None
        if small and rng.random() < p_cfl:
            um, uang = MODE_CFL, 0
        smu = (is_sm(uvmode[y4 - 1, x4]) if y4 > 0 else 0) | (is_sm(uvmode[y4, x4 - 1]) if x4 > 0 else 0)
        uvmode[y4:y4 + chh, x4:x4 + cw] = 0 if um == MODE_CFL else um
        ctl, cth = min(clw, 3), min(clh, 3)
        for pl in (1, 2):
            if um == MODE_CFL:
                fr = ((ccw << ss_hor) + (1 << tlw) - 1) & ~((1 << tlw) - 1)
                fb = ((cch << ss_ver) + (1 << tlh) - 1) & ~((1 << tlh) - 1)
                alpha = int(rng.integers(-16, 17)) if rng.random() < 0.85 else 0
                cfl = (alpha, (1 << clw) - (fr >> ss_hor), (1 << clh) - (fb >> ss_ver))
            for yy in range(0, cch, 1 << cth):
                for xx in range(0, ccw, 1 << ctl):
                    if pl == 1:
                        paint(tuv, cx4 + xx, cy4 + yy, ctl, cth, ch4, cw4)
                    add(pl, cx4 + xx, cy4 + yy, ctl, cth, um, uang, smu, skip, x4, y4, cfl)

    tx = np.array(recs, INTRA_TX_DT)
    n = len(tx)
    # ---- residuals (same generator as the inter frames)
    coef_off = 0
    chunks = []
    for t in range(19):
        sel = np.nonzero((tx["tx"] == t) & (tx["eob"] >= 0))[0]
        if not len(sel):
            continue
        k = len(sel)
        sw, sh = _L.tx_coef_dims(t)
        ncf = sw * sh
        legal = [tp for tp in range(10) if _L.itx_defined(t, tp)]
        txtp = rng.choice(legal, k, p=None if len(legal) == 1 else [0.55] + [0.45 / (len(legal) - 1)] * (len(legal) - 1))
        scan = scan_table(t)
        inv = np.empty(ncf, np.int64); inv[scan] = np.arange(ncf)
        eob = np.minimum((rng.exponential(ncf / 10.0, k)).astype(np.int64), ncf - 1)
        eob[rng.random(k) < 0.25] = 0
        amp = (bd + 1) / 2.0
        pos = inv[None, :]
        c = np.rint(rng.laplace(0.0, amp * 0.25, (k, ncf)) / (1.0 + pos / 6.0)).astype(np.int64)
        c[pos > eob[:, None]] = 0
        c[np.arange(k), scan[eob]] = np.where(c[np.arange(k), scan[eob]] == 0, 1, c[np.arange(k), scan[eob]])
        tx["coef_off"][sel] = coef_off + np.arange(k) * ncf
        tx["eob"][sel] = eob; tx["txtp"][sel] = txtp
        chunks.append(c.astype(cdt).reshape(-1))
        coef_off += k * ncf
    coefs = np.concatenate(chunks) if chunks else np.zeros(1, cdt)

    # ---- wavefront numbers: 1 + the latest wave among the cells the device waits for (same cells as intra.cu)
    wave_map = [np.zeros((ph4[p], pw4[p]), np.int32) for p in range(3)]
    wave = np.zeros(n, np.int64)
    for i in range(n):
        r = tx[i]
        pl, x, y = int(r["plane"]), int(r["x4"]), int(r["y4"])
        tw, th = _L.TX_W[r["tx"]] // 4, _L.TX_H[r["tx"]] // 4
        wm = wave_map[pl]
        fl = int(r["flags"])
        dep = 0
        if r["mode"] == MODE_RESID:                     # after the record that predicted these cells
            wave[i] = int(wm[y:y + th, x:x + tw].max()) + 1
            wm[y:y + th, x:x + tw] = wave[i]
            continue
        if r["mode"] == MODE_IBC:                       # after every cell its source rectangle touches
            sx, sy = int(r["luma_off"]) & 0xffff, int(r["luma_off"]) >> 16
            x1 = min((sx + 4 * tw - 1 + (1 if r["cfl_w_pad"] else 0)) >> 2, pw4[pl] - 1)
            y1 = min((sy + 4 * th - 1 + (1 if r["cfl_h_pad"] else 0)) >> 2, ph4[pl] - 1)
            wave[i] = int(wm[min(sy >> 2, ph4[pl] - 1):y1 + 1, min(sx >> 2, pw4[pl] - 1):x1 + 1].max()) + 1
            wm[y:y + th, x:x + tw] = wave[i]
            continue
        if fl & 1:
            nrow = min(th, ph4[pl] - y) + (min(th, ph4[pl] - y - th) if (fl & 8) and y + th < ph4[pl] else 0)
            dep = max(dep, int(wm[y:y + nrow, x - 1].max()))
        if fl & 2:
            ncol = min(tw, pw4[pl] - x) + (min(tw, pw4[pl] - x - tw) if (fl & 4) and x + tw < pw4[pl] else 0)
            dep = max(dep, int(wm[y - 1, x:x + ncol].max()))
        if (fl & 3) == 3:
            dep = max(dep, int(wm[y - 1, x - 1]))
        if r["mode"] == MODE_CFL and r["cfl_alpha"] != 0:
            lx, ly = x << ss_hor, y << ss_ver
            lw_ = min((tw - int(r["cfl_w_pad"])) << ss_hor, w4 - lx); lh_ = min((th - int(r["cfl_h_pad"])) << ss_ver, h4 - ly)
            dep = max(dep, int(wave_map[0][ly:ly + lh_, lx:lx + lw_].max()))
        wave[i] = dep + 1
        wm[y:y + th, x:x + tw] = dep + 1
    sorted_idx = np.argsort(wave, kind="stable")
    # superblock-granular schedule: records grouped by 64x64 superblock (decode order inside), superblocks in
    # wavefront order sx + 2*sy (left / top-left / top / top-right neighbours always earlier)
    sbw_n, sbh_n = (w4 + 15) // 16, (h4 + 15) // 16
    shx = np.array([4, 4 - ss_hor, 4 - ss_hor])[tx["plane"]]; shy = np.array([4, 4 - ss_ver, 4 - ss_ver])[tx["plane"]]
    rsx = (tx["x4"].astype(np.int64) >> shx); rsy = (tx["y4"].astype(np.int64) >> shy)
    sb_of = rsy * sbw_n + rsx
    order_sb = sorted(range(sbw_n * sbh_n), key=lambda k: ((k % sbw_n) + 2 * (k // sbw_n), k // sbw_n))
    by_sb = np.argsort(sb_of, kind="stable")                      # keeps decode order inside a superblock
    counts = np.bincount(sb_of, minlength=sbw_n * sbh_n)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    sb_recs = np.zeros(len(order_sb), INTRA_SB_DT)
    pieces, pos = [], 0
    for t, k in enumerate(order_sb):
        pieces.append(by_sb[starts[k]:starts[k] + counts[k]])
        sb_recs[t] = (pos, counts[k], k % sbw_n, k // sbw_n)
        pos += counts[k]
    tx_sb = tx[np.concatenate(pieces)].copy() if pieces else tx.copy()
    S.update(intra_tx=tx[sorted_idx].copy(), intra_tx_decode_order=tx, intra_waves=int(wave.max()), coefs=coefs,
             intra_tx_sb=tx_sb, intra_sb=sb_recs, intra_sb_grid=(sbw_n, sbh_n),
             refs=[], pred=np.zeros(0, MC_BLOCK_DT), comp=np.zeros(0, COMP_BLOCK_DT), comp2=np.zeros(0, COMP_BLOCK_DT),
             itx={t: np.zeros(0, ITX_BLOCK_DT) for t in range(19)}, tmp_len=64, mask=np.zeros(1, np.uint8))
    S["pic"] = np.zeros(len(S["pic"]), dt)
    S["masks"] = build_lf_masks(w4, h4, tuple(ty), tuple(tuv), ss_hor, ss_ver)
    S["til_y"], S["til_uv"] = tuple(ty), tuple(tuv)
    S["bw"], S["bh"] = w4, h4
    S["damping"], S["y_strength"], S["uv_strength"] = make_cdef_params(rng, w4, h4, S["sb128w"], S["masks"])
    S["lr_mask"] = make_lr_params(rng, W, H)
    S["us"] = (6, 6 - (1 if ss_hor else 0))
    S["rp"], S["sb128"] = 7, 0
    return S


# ---------------------------------------------------------------------------------------------------------
COEF_BLOCK_DT = np.dtype([("dense_off", "<u4"), ("compact_off", "<u4"), ("eob", "<i2"), ("tx", "u1"), ("tx_class", "u1")])
# TxClass per TxfmType (reference src/tables.c dav1d_tx_type_class): 0 2-D, 1 H_* (TX_CLASS_H), 2 V_* (TX_CLASS_V)
TX_CLASS = np.array([0] * 10 + [2, 1, 2, 1, 2, 1] + [0], np.int64)


def class_scan(tx, cls):
    """coefficient index of scan position k for a block of TxClass cls, as decode_coefs walks it (reference
    src/recon_tmpl.c:458-467, 548-576): dav1d_scans[tx] (2-D), k (H), x * sh + y with x = k % sw, y = k / sw (V)"""
    if cls == 0:
        return scan_table(tx)
    sw, sh = _L.tx_coef_dims(tx)
    k = np.arange(sw * sh, dtype=np.int64)
    return k if cls == 1 else (k % sw) * sh + k // sw


def compact_coefs(S):
    """What a record emitter would ship instead of the dense coefficient plane: per coded transform block the
    coefficients 0 .. eob in the scan order of its class, plus one B200CoefBlock record each (include/b200av1.h). Returns
    (compact stream, records)."""
    dense = S["coefs"]
    recs, chunks, pos = [], [], 0
    groups = [(tx, S["itx"][tx]["coef_off"].astype(np.int64), S["itx"][tx]["eob"].astype(np.int64), TX_CLASS[S["itx"][tx]["txtp"]])
              for tx in range(19) if len(S["itx"][tx])]
    it = S.get("intra_tx")
    if it is not None and len(it):
        for tx in range(19):
            sel = (it["tx"] == tx) & (it["eob"] >= 0)
            if sel.any():
                groups.append((tx, it["coef_off"][sel].astype(np.int64), it["eob"][sel].astype(np.int64), TX_CLASS[it["txtp"][sel]]))
    for tx, offs, eobs, cls in groups:
        scans = np.stack([class_scan(tx, c) for c in range(3)])
        n = len(offs)
        cnt = eobs + 1
        # gather dense[off + scan[k]] for k <= eob, block after block
        k = np.arange(int(cnt.max()))[None, :]
        valid = k < cnt[:, None]
        idx = offs[:, None] + scans[cls[:, None], np.minimum(k, scans.shape[1] - 1)]
        chunks.append(dense[idx[valid]])
        a = np.zeros(n, COEF_BLOCK_DT)
        a["dense_off"] = offs
        a["compact_off"] = pos + np.concatenate([[0], np.cumsum(cnt)[:-1]])
        a["eob"] = eobs; a["tx"] = tx; a["tx_class"] = cls
        recs.append(a)
        pos += int(cnt.sum())
    if not recs:
        return np.zeros(1, dense.dtype), np.zeros(0, COEF_BLOCK_DT)
    return np.concatenate(chunks).astype(dense.dtype), np.concatenate(recs)
