"""Unscaled inter prediction at frame scale, against dav1d's own mc().

The Level-1 checks of test_mc.py call the prediction kernels one block at a time on exactly the window the block
reads, and test_mc.py's frame test has one reference, 4:2:0 only and word-aligned pitches. Here whole batches go
through every unscaled stage the frame job runs:

- `b200_mc_batch` (put / prep / put into the OBMC pixel scratch), with the records emit_mc / emit_obmc of
  integration/dav1d/b200_hooks_tmpl.c make: every AV1 block size in every layout, the 2x2 / 2x4 / 4x2 chroma of
  sub-8x8 blocks, OBMC neighbour heights 2 ... 24, all ten filters, phases of 0 on either axis, 1 to 8 references
  and windows before, after, across and inside every edge, and on the lines of the kernel's interior predicate;
- `b200_mc_comp_batch`, stage `comp` then `comp2`, on the prep outputs of the same batch: all six ops, the w_avg
  weights dav1d derives, w_mask 4:4:4 / 4:2:2 / 4:2:0 with either sign, and chroma records reading the mask
  their luma block wrote;
- `b200_mc_comp_fused_batch` on the same compound blocks, which must give the bytes of prep + compound;
- `b200_mc_blend_batch`: blend_h, then blend_v (they overlap in the top-left corner of a block), and blend;
- `b200_mc_warp_batch`: shears inside dav1d's validity bounds, reaching both ends of the warp filter table.

Expected values are what dav1d's mc() does for an unscaled reference (reference src/recon_tmpl.c:938-988):
emu_edge into a 192-wide buffer when the block's footprint leaves the plane, then mc[] / mct[], and the same for
warp_affine (:1115-1165). The C side is the reference build (oracle/_ref) where it exists, the oracle otherwise;
the oracle's coverage counters (oracle_mc_counts) and the interior / clamped split restated below are held to
floors, so that a change to the record generator cannot quietly drop an edge. Whole buffers are compared: dst,
tmp, mask and px_tmp, including the samples around and between the blocks.
"""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import refs
from dav1d_b200 import _lib
from test_mc import mct_input
from test_scaled_prediction import LAYOUTS, _align, _emu_dev, _torch_dev, _torch_host, _torch_sync, _window_pos, checker, \
    picture_geom

EMU_W = 192                       # dav1d's emu_edge scratch (t->scratch.emu_edge) is 192 samples wide
COUNTS = ("put_clip_lo", "put_clip_hi", "prep_max_8", "prep_max_10", "prep_max_12", "wmask_38", "wmask_64",
          "h_4tap", "h_8tap", "v_4tap", "v_8tap", "h_identity", "v_identity")
# AV1 block sizes in luma samples (reference src/tables.c dav1d_block_dimensions)
BLOCK_SIZES = [(128, 128), (128, 64), (64, 128), (64, 64), (64, 32), (64, 16), (32, 64), (32, 32), (32, 16), (32, 8),
               (16, 64), (16, 32), (16, 16), (16, 8), (16, 4), (8, 32), (8, 16), (8, 8), (8, 4), (4, 16), (4, 8), (4, 4)]
COMP_SIZES = [s for s in BLOCK_SIZES if min(s) >= 8]     # compound, OBMC and wedge blocks are 8x8 or larger
JNT_WEIGHTS = (3, 4, 5, 7, 9, 11, 12, 13)       # every f->jnt_weights value (quant_dist_lookup_table, src/decode.c)
W_MASK_OP = {"420": 5, "422": 4, "444": 3, "400": 3}    # B200_COMP_W_MASK_444 + chr_layout_idx
# compound shapes outside the hooks' set: item counts that are not a multiple of 32 in the fused kernel
ODD_COMP_SHAPES = [(4, 4), (8, 6), (16, 12), (32, 24), (4, 12)]


def plane_shapes(layout, pl):
    """(w, h) of every prediction emit_mc makes on a plane of `layout`: each block size, and for sub-sampled chroma
    the widened 4-sample chroma of 4-wide / 4-tall blocks as well as the 2-sample sub-8x8 quarters"""
    if pl == 0:
        return list(BLOCK_SIZES)
    sh, sv = LAYOUTS[layout]
    out = set()
    for bw, bh in BLOCK_SIZES:
        bw4, bh4 = bw // 4, bh // 4
        h_mul, v_mul = 4 >> sh, 4 >> sv
        out.add(((bw4 << (bw4 == sh)) * h_mul, (bh4 << (bh4 == sv)) * v_mul))
        if bw4 == sh or bh4 == sv:
            out.add((bw4 * h_mul, bh4 * v_mul))
    return sorted(out)


def frame_geom(rng, kind, W, H, layout, bpc):
    """"hooks": the hooks' picture layout; "tight": pitches only as wide as the words the kernels load need;
    "odd": plane 0 an unaligned pitch, plane 1 an unaligned offset, plane 2 both (nothing can take the interior path)"""
    if kind == "hooks":
        return picture_geom(rng, W, H, layout)
    ppw = 4 if bpc == 8 else 2
    sh, sv = LAYOUTS[layout]
    w, h = [W] + [(W + sh) >> sh] * 2, [H] + [(H + sv) >> sv] * 2
    n = 1 if layout == "400" else 3
    off, stride, o = [], [], 0
    for p in range(3):
        if kind == "tight":
            s = _align(w[p], ppw)
        else:
            s = w[p] + int(rng.integers(0, 6))
            if p == 1:
                s = _align(s, ppw)
            elif s % ppw == 0:
                s += 1
            if p and o % ppw == 0:
                o += 1
        if p < n:
            off.append(o); stride.append(s)
            o += s * h[p]
        else:
            off.append(off[0]); stride.append(stride[0])
    return dict(off=off, stride=stride, w=w, h=h, total=o + 8)


def plane_view(pic, g, p):
    isz = pic.itemsize
    return np.lib.stride_tricks.as_strided(pic[g["off"][p]:], shape=(g["h"][p], g["w"][p]), strides=(g["stride"][p] * isz, isz))


def fill_picture(rng, g, n_planes, bd, dt):
    """noise, with rectangles of checkasm's worst-case corner pattern and flat areas at 0 and bitdepth_max, some of
    them on the plane's edges"""
    pic = rng.integers(0, bd + 1, g["total"]).astype(dt)
    for p in range(n_planes):
        v = plane_view(pic, g, p)
        ph, pw = v.shape
        for _ in range(max(6, pw * ph // 1200)):
            rh, rw = int(rng.integers(4, 48)), int(rng.integers(4, 48))
            y, x = int(rng.integers(-rh // 2, ph)), int(rng.integers(-rw // 2, pw))
            ys, xs = slice(max(0, y), min(ph, y + rh)), slice(max(0, x), min(pw, x + rw))
            kind = int(rng.integers(0, 4))
            if kind <= 1:
                corner = mct_input(rng, bd, dt)[:8, :8]
                sub = v[ys, xs]
                sub[...] = np.tile(corner, (sub.shape[0] // 8 + 1, sub.shape[1] // 8 + 1))[:sub.shape[0], :sub.shape[1]]
            else:
                v[ys, xs] = 0 if kind == 2 else bd
    return pic


def interior(g, pl, src_x, src_y, w, h, bpc):
    """mc_pred_setup's interior predicate (the base pointers of the test's pictures are word-aligned)"""
    ppw, isz = (4, 1) if bpc == 8 else (2, 2)
    rs, rw, rh = g["stride"][pl], g["w"][pl], g["h"][pl]
    gx, gy, nc, nr = src_x - 3, src_y - 3, w + 7, h + 7
    aligned = rs % ppw == 0 and (g["off"][pl] * isz) % 4 == 0
    pos = gx >= 0 and gy >= 0 and gx + nc <= rw and gy + nr <= rh
    return aligned and pos and word_bound(gx, nc, ppw) <= rs, pos


def word_bound(gx, nc, ppw):
    return (gx & ~(ppw - 1)) + ((nc + (gx & (ppw - 1)) + ppw - 1) & ~(ppw - 1)) + ppw


class Batch:
    """Records of every unscaled stage over one frame, as the hooks make them, and the buffers they work on."""

    def __init__(self, rng, bpc, layout, W, H, geom, n_refs):
        self.rng, self.bpc, self.layout = rng, bpc, layout
        self.bd, self.dt = (1 << bpc) - 1, refs.pixel_dtype(bpc)
        self.ppw = 4 if bpc == 8 else 2
        self.n_planes = 1 if layout == "400" else 3
        self.geom = geom
        self.g = frame_geom(rng, geom, W, H, layout, bpc)
        self.pics = [fill_picture(rng, self.g, self.n_planes, self.bd, self.dt) for _ in range(n_refs)]
        self.taken = [np.zeros((self.g["h"][p], self.g["w"][p]), bool) for p in range(self.n_planes)]
        self.pred, self.comp, self.comp2, self.blend, self.blend2, self.warp = [], [], [], [], [], []
        self.fused, self.fused2 = [], []
        self.n_tmp = self.n_px = self.n_wmask = 0
        self.n_single = [0, 0, 0]
        self.mask = []                         # chunks of the initial mask buffer
        self.n_mask = 0
        self.stats = dict(interior=np.zeros(3, int), clamped=np.zeros(3, int), pos_inside=np.zeros(3, int), gx0=0, gx_end=0,
                          gy0=0, gy_end=0, wb_hit=0, wb_miss=0, mixed_pairs=0, warp_lo=999, warp_hi=-999)

    # ---- placement: records of one stage run concurrently, so the ones that write dst must not overlap
    def place(self, pl, w, h, tries=24, align=None, first=0):
        """a free w x h area at a multiple of `align` (default: the block's own size), `first` steps from the top / left"""
        t = self.taken[pl]
        ph, pw = t.shape
        ax, ay = (w, h) if align is None else align
        if w + first * ax > pw or h + first * ay > ph:
            return None
        for _ in range(tries):
            x = ax * int(self.rng.integers(first, (pw - w) // ax + 1))
            y = ay * int(self.rng.integers(first, (ph - h) // ay + 1))
            if not t[y:y + h, x:x + w].any():
                t[y:y + h, x:x + w] = True
                return x, y
        return None

    def dst_off(self, pl, x, y):
        return self.g["off"][pl] + y * self.g["stride"][pl] + x

    def tmp_alloc(self, n):
        o = self.n_tmp + int(self.rng.choice([0, 1, 2, 3, 7]))      # odd offsets too: both sides of mc_comp_kernel's `vec`
        self.n_tmp = o + n
        return o

    def px_alloc(self, n):
        o = self.n_px + int(self.rng.integers(0, 5))
        self.n_px = o + n
        return o

    def mask_alloc(self, data):
        o = self.n_mask + int(self.rng.integers(0, 3)) * 64
        if o > self.n_mask:
            self.mask.append(self.rng.integers(0, 256, o - self.n_mask).astype(np.uint8))
        self.mask.append(data)
        self.n_mask = o + data.size
        return o

    def wedge_mask(self, n):
        m = self.rng.integers(0, 65, n)
        m[self.rng.random(n) < 0.5] = 0
        m[self.rng.random(n) < 0.3] = 64
        return m.astype(np.uint8)

    # ---- one prediction: a motion vector turned into src_x / mx as emit_mc does it
    def window(self, pl, x0, w, h, y0, inside=False):
        """src_x, src_y for a block at (x0, y0) of plane pl: one of the interior predicate's lines, or a window before,
        after, across or inside an edge (`inside`: a window wholly inside the plane, where there is room)"""
        rng, g = self.rng, self.g
        rw, rh, rs, ppw = g["w"][pl], g["h"][pl], g["stride"][pl], self.ppw
        nc, nr = w + 7, h + 7
        if inside and rw >= nc and rh >= nr:
            return int(rng.integers(0, rw - nc + 1)) + 3, int(rng.integers(0, rh - nr + 1)) + 3
        kind = int(rng.integers(0, 14))
        sx = None
        if kind == 0:
            sx = 3                                              # gx = 0
        elif kind == 1:
            sx = rw - nc + 3                                    # gx + w + 7 = rw
        elif kind in (2, 3):
            # the word bound hit exactly (kind 2) or missed by one word (kind 3) with gx + w + 7 <= rw
            e = min(rs - ppw if kind == 2 else rs, rw)
            if e - nc >= 0 and _align(e, ppw) + ppw == rs + (kind == 3) * ppw:
                sx = e - nc + 3
        if sx is None:
            sx = _window_pos(rng, w, rw)
        ky = int(rng.integers(0, 10))
        sy = 3 if ky == 0 else rh - nr + 3 if ky == 1 else _window_pos(rng, h, rh)
        return sx, sy

    def mv_to_src(self, pl, x0, y0, sx, sy, zero_x, zero_y):
        """the hook's arithmetic: a motion vector (1/8 luma sample units; 1/16 for sub-sampled chroma) from the block at
        (x0, y0) towards (sx, sy), in the AV1 range, turned into src_x / mx"""
        sh, sv = LAYOUTS[self.layout] if pl else (0, 0)
        fx = 0 if zero_x else int(self.rng.integers(1, (15 >> (1 - sh)) + 1))
        fy = 0 if zero_y else int(self.rng.integers(1, (15 >> (1 - sv)) + 1))
        mvx = int(np.clip(((sx - x0) << (3 + sh)) + fx, -(1 << 14), (1 << 14) - 1))
        mvy = int(np.clip(((sy - y0) << (3 + sv)) + fy, -(1 << 14), (1 << 14) - 1))
        return (x0 + (mvx >> (3 + sh)), (mvx & (15 >> (1 - sh))) << (1 - sh),
                y0 + (mvy >> (3 + sv)), (mvy & (15 >> (1 - sv))) << (1 - sv))

    def pred_rec(self, op, pl, w, h, x0, y0, dst_off, ref=None, f2d=None, inside=False):
        rng = self.rng
        sx, sy = self.window(pl, x0, w, h, y0, inside)
        phase = int(rng.integers(0, 6))                         # 0: both axes without phase, 1: x, 2: y, else both phased
        src_x, mx, src_y, my = self.mv_to_src(pl, x0, y0, sx, sy, phase in (0, 1), phase in (0, 2))
        r = _lib.McBlock()
        r.dst_off, r.src_x, r.src_y, r.w, r.h, r.mx, r.my = dst_off, src_x, src_y, w, h, mx, my
        r.filter2d = int(rng.integers(0, 10)) if f2d is None else f2d
        r.op, r.plane = op, pl
        r.ref = int(rng.integers(0, len(self.pics))) if ref is None else ref
        self.pred.append(r)
        return r, self.note(r)

    def note(self, r):
        s, g, pl = self.stats, self.g, r.plane
        inside, pos = interior(g, pl, r.src_x, r.src_y, r.w, r.h, self.bpc)
        s["interior" if inside else "clamped"][pl] += 1
        s["pos_inside"][pl] += pos
        gx, gy = r.src_x - 3, r.src_y - 3
        s["gx0"] += gx == 0
        s["gx_end"] += gx + r.w + 7 == g["w"][pl]
        s["gy0"] += gy == 0
        s["gy_end"] += gy + r.h + 7 == g["h"][pl]
        if pos and g["stride"][pl] % self.ppw == 0:
            b = word_bound(gx, r.w + 7, self.ppw)
            s["wb_hit"] += b == g["stride"][pl]
            s["wb_miss"] += b == g["stride"][pl] + self.ppw
        return inside

    # ---- blocks
    def single(self, pl):
        shapes = plane_shapes(self.layout, pl)
        w, h = shapes[self.n_single[pl] % len(shapes)]          # every shape in turn
        self.n_single[pl] += 1
        p = self.place(pl, w, h)
        if p is not None:
            self.pred_rec(0, pl, w, h, p[0], p[1], self.dst_off(pl, *p))
        elif w >= 4 and h >= 4:
            x0, y0 = self.anywhere(pl)
            self.pred_rec(1, pl, w, h, x0, y0, self.tmp_alloc(w * h))
        else:
            x0, y0 = self.anywhere(pl)
            self.pred_rec(2, pl, w, h, x0, y0, self.px_alloc(w * h))

    def anywhere(self, pl):
        return int(self.rng.integers(0, self.g["w"][pl])), int(self.rng.integers(0, self.g["h"][pl]))

    def obmc(self, pl, size=None, inner=None):
        """a block's own prediction, then emit_obmc: predictions with the motion of the blocks above into the pixel
        scratch + blend_h (stage blend), with that of the blocks to the left + blend_v (stage blend2)"""
        rng = self.rng
        sh, sv = LAYOUTS[self.layout] if pl else (0, 0)
        h_mul, v_mul = 4 >> sh, 4 >> sv
        bw4, bh4 = (v // 4 for v in (size or COMP_SIZES[int(rng.integers(0, len(COMP_SIZES)))]))
        bw, bh = bw4 * h_mul, bh4 * v_mul
        # any 8x8 position but the first row and column: the block has neighbours above and to the left
        inner = int(rng.integers(0, 4)) > 0 if inner is None else inner
        p = self.place(pl, bw, bh, align=(2 * h_mul, 2 * v_mul), first=int(inner))
        if p is None:
            return
        x0, y0 = p
        base = self.dst_off(pl, x0, y0)
        f2d = int(rng.integers(0, 10))
        self.pred_rec(0, pl, bw, bh, x0, y0, base, f2d=f2d)
        stride = self.g["stride"][pl]
        if y0 > 0 and (not pl or bw4 * h_mul + bh4 * v_mul >= 16):
            x, i = 0, 0
            while x < bw4 and i < 4:
                step4 = int(rng.choice([2, 4, 8, 16]))
                if x:
                    step4 = min(step4, bw4 - x)
                ow4, oh4 = min(step4, bw4), min(bh4, 16) >> 1
                ph = ((oh4 * 3 + 3) >> 2) * v_mul
                o = self.px_alloc(ow4 * h_mul * ph)
                self.pred_rec(2, pl, ow4 * h_mul, ph, x0 + x * h_mul, y0, o)
                self.blend.append(self.blend_rec(base + x * h_mul, o, 0, h_mul * ow4, v_mul * oh4, 2, pl))
                x += step4; i += 1
        if x0 > 0:
            y, i = 0, 0
            while y < bh4 and i < 4:
                step4 = int(rng.choice([2, 4, 8, 16]))
                if y:
                    step4 = min(step4, bh4 - y)
                ow4, oh4 = min(bw4, 16) >> 1, min(step4, bh4)
                o = self.px_alloc(ow4 * h_mul * oh4 * v_mul)
                self.pred_rec(2, pl, ow4 * h_mul, oh4 * v_mul, x0, y0 + y * v_mul, o)
                self.blend2.append(self.blend_rec(base + y * v_mul * stride, o, 0, h_mul * ow4, v_mul * oh4, 1, pl))
                y += step4; i += 1

    @staticmethod
    def blend_rec(dst_off, tmp_off, mask_off, w, h, op, pl):
        b = _lib.BlendBlock()
        b.dst_off, b.tmp_off, b.mask_off, b.w, b.h, b.op, b.plane = dst_off, tmp_off, mask_off, w, h, op, pl
        return b

    def masked_blend(self, pl):
        """blend with a mask (the inter-intra form of the blend stage) over pixels of the scratch"""
        w, h = (int(v) for v in self.rng.choice([2, 4, 8, 16, 32], 2))
        p = self.place(pl, w, h)
        if p is not None:
            o = self.px_alloc(w * h)
            self.blend.append(self.blend_rec(self.dst_off(pl, *p), o, self.mask_alloc(self.wedge_mask(w * h)), w, h, 0, pl))

    def compound(self, shape=None, op=None, kind=None, size=None):
        """a compound block as the hooks emit it: per plane two prep records, then avg / w_avg / mask / w_mask; a
        difference-weighted block's chroma reads the mask its luma w_mask writes (stage comp2)"""
        rng = self.rng
        sh, sv = LAYOUTS[self.layout]
        if shape is None:
            bw, bh = size or COMP_SIZES[int(rng.integers(0, len(COMP_SIZES)))]
            planes = range(self.n_planes)
            kind = int(rng.integers(0, 4)) if kind is None else kind     # avg, w_avg, wedge, difference-weighted
        else:
            bw, bh = shape
            planes, kind = [0], 3
        sign = int(rng.integers(0, 2))
        f2d = int(rng.integers(0, 10))
        luma_mask = None
        refs2 = [int(rng.integers(0, len(self.pics))) for _ in range(2)]
        for pl in planes:
            pw, ph = (bw >> sh, bh >> sv) if pl else (bw, bh)
            pos = self.place(pl, pw, ph)
            if pos is None:
                continue
            x0, y0 = pos
            # one prediction of some pairs inside the plane: the fused kernel's interior dispatch needs both
            into = int(rng.integers(0, 3))
            recs, ins = zip(*[self.pred_rec(1, pl, pw, ph, x0, y0, self.tmp_alloc(pw * ph), ref=refs2[i], f2d=f2d, inside=into == i + 1)
                              for i in range(2)])
            self.stats["mixed_pairs"] += ins[0] != ins[1]
            cb = _lib.CompBlock()
            cb.dst_off, cb.w, cb.h, cb.plane = self.dst_off(pl, x0, y0), pw, ph, pl
            first = recs
            stage = self.comp
            if kind == 0:
                cb.op = 0
            elif kind == 1:
                cb.op, cb.param = 1, int(rng.choice(JNT_WEIGHTS))
            else:
                first = [recs[sign], recs[1 - sign]]
                if kind == 2:
                    cb.op, cb.mask_off = 2, self.mask_alloc(self.wedge_mask(pw * ph))
                elif pl == 0:
                    cb.op = W_MASK_OP[self.layout] if op is None else op
                    cb.param = sign
                    mw, mh = (pw >> (cb.op >= 4), ph >> (cb.op == 5))
                    cb.mask_off = luma_mask = self.mask_alloc(rng.integers(0, 256, mw * mh).astype(np.uint8))
                elif luma_mask is not None:
                    cb.op, cb.mask_off = 2, luma_mask
                    stage = self.comp2
                else:
                    continue
            cb.tmp1_off, cb.tmp2_off = first[0].dst_off, first[1].dst_off
            stage.append(cb)
            fb = _lib.CompFusedBlock()
            fb.dst_off, fb.mask_off, fb.w, fb.h = cb.dst_off, cb.mask_off, pw, ph
            for i, r in enumerate(first):
                fb.src_x[i], fb.src_y[i], fb.mx[i], fb.my[i], fb.ref[i] = r.src_x, r.src_y, r.mx, r.my, r.ref
            fb.filter2d, fb.op, fb.param, fb.plane = f2d, cb.op, cb.param, pl
            (self.fused2 if stage is self.comp2 else self.fused).append(fb)

    def extreme_compound(self, f2d=None):
        """a w_mask block whose two predictions read checkasm's worst-case pattern and its inverse, lined up with
        their windows: the largest and smallest prep values of the bit depth meet, so the mask saturates at 64"""
        rng = self.rng
        w, h = (int(v) for v in rng.choice([8, 16, 32], 2))
        pl = int(rng.integers(0, self.n_planes))
        rw, rh = self.g["w"][pl], self.g["h"][pl]
        pos = self.place(pl, w, h)
        if pos is None or rw < w + 7 or rh < h + 7:
            return
        corner = mct_input(rng, self.bd, self.dt)[:8, :8]
        f2d = int(rng.integers(3, 6)) if f2d is None else f2d             # sharp horizontally
        op, sign = int(rng.integers(3, 6)), int(rng.integers(0, 2))
        recs = []
        for i in range(2):
            k = int(rng.integers(0, len(self.pics)))
            gx, gy = int(rng.integers(0, rw - w - 6)), int(rng.integers(0, rh - h - 6))
            v = plane_view(self.pics[k], self.g, pl)[gy:gy + h + 7, gx:gx + w + 7]
            pat = corner if i == 0 else self.bd - corner
            v[...] = np.tile(pat, ((h + 7) // 8 + 1, (w + 7) // 8 + 1))[:h + 7, :w + 7]
            r = _lib.McBlock()
            r.dst_off, r.src_x, r.src_y, r.w, r.h, r.mx, r.my = self.tmp_alloc(w * h), gx + 3, gy + 3, w, h, 8, 8
            r.filter2d, r.op, r.plane, r.ref = f2d, 1, pl, k
            self.pred.append(r)
            self.note(r)
            recs.append(r)
        cb = _lib.CompBlock()
        cb.dst_off, cb.w, cb.h, cb.plane, cb.op, cb.param = self.dst_off(pl, *pos), w, h, pl, op, sign
        cb.tmp1_off, cb.tmp2_off = recs[0].dst_off, recs[1].dst_off
        cb.mask_off = self.mask_alloc(rng.integers(0, 256, (w >> (op >= 4)) * (h >> (op == 5))).astype(np.uint8))
        self.comp.append(cb)
        fb = _lib.CompFusedBlock()
        fb.dst_off, fb.mask_off, fb.w, fb.h = cb.dst_off, cb.mask_off, w, h
        for i, r in enumerate(recs):
            fb.src_x[i], fb.src_y[i], fb.mx[i], fb.my[i], fb.ref[i] = r.src_x, r.src_y, r.mx, r.my, r.ref
        fb.filter2d, fb.op, fb.param, fb.plane = f2d, op, sign, pl
        self.fused.append(fb)

    def warp_block(self, pl, op, extreme=False):
        """emit_warp: one record per 8x8 of a block, mx / my from the 16.16 position and the shear as the hook derives
        them (so they can be negative); shears inside dav1d's bounds 4|a| + 7|b| < 0x10000, 4|c| + 4|d| < 0x10000,
        some at their extremes so that the filter index reaches 0 ... 2 and 190 ... 192"""
        rng = self.rng
        bw, bh = (int(v) for v in rng.choice([8, 16, 32], 2))
        if op == 0:
            p = self.place(pl, bw, bh)
            if p is None:
                return
            base, pitch = self.dst_off(pl, *p), self.g["stride"][pl]
        else:
            base, pitch = self.tmp_alloc(bw * bh), bw
        extreme = extreme or rng.integers(0, 3) == 0
        if extreme:
            b = int(rng.integers(8960, 9344) // 64 * 64)
            a = int(rng.integers(0, (0x10000 - 7 * abs(b)) // 4) // 64 * 64)
        else:
            b = int(rng.integers(-2000, 2000) // 64 * 64)
            a = int(rng.integers(-(0x10000 - 7 * abs(b)) // 4 + 64, (0x10000 - 7 * abs(b)) // 4) // 64 * 64)
        d = int(rng.integers(-15000, 15000) // 64 * 64)
        c = int(rng.integers(-(0x10000 - 4 * abs(d)) // 4 + 64, (0x10000 - 4 * abs(d)) // 4) // 64 * 64)
        assert 4 * abs(a) + 7 * abs(b) < 0x10000 and 4 * abs(c) + 4 * abs(d) < 0x10000
        ref = int(rng.integers(0, len(self.pics)))
        rw, rh = self.g["w"][pl], self.g["h"][pl]
        for y in range(0, bh, 8):
            for x in range(0, bw, 8):
                sx, sy = _window_pos(rng, 8, rw), _window_pos(rng, 8, rh)
                fx = (0, 0xffff)[len(self.warp) % 2] if extreme else int(rng.integers(0, 0x10000))
                fy = int(rng.integers(0, 0x10000))
                r = _lib.WarpBlock()
                r.dst_off = base + y * pitch + x
                r.src_x, r.src_y = sx, sy
                r.mx = (fx - a * 4 - b * 7) & ~0x3f           # two's complement, as in C
                r.my = (fy - c * 4 - d * 4) & ~0x3f
                r.abcd[0], r.abcd[1], r.abcd[2], r.abcd[3] = a, b, c, d
                r.tmp_stride, r.op, r.plane, r.ref = pitch, op, pl, ref
                idx = [64 + ((r.mx + yy * b + xx * a + 512) >> 10) for yy in (0, 14) for xx in (0, 7)]
                self.stats["warp_lo"] = min(self.stats["warp_lo"], *idx)
                self.stats["warp_hi"] = max(self.stats["warp_hi"], *idx)
                self.warp.append(r)

    def finish(self):
        rng = self.rng
        self.tmp = rng.integers(-(1 << 15), 1 << 15, self.n_tmp + 8).astype(np.int16)
        self.px_tmp = rng.integers(0, self.bd + 1, self.n_px + 8).astype(self.dt)
        self.mask_buf = np.concatenate(self.mask + [rng.integers(0, 256, 64).astype(np.uint8)])
        self.dst = rng.integers(0, self.bd + 1, self.g["total"]).astype(self.dt)
        # the pixel scratch the blend stages read is written by op-2 records; blend (with a mask) reads what is there
        return self


def make_batch(rng, bpc, layout, W, H, n_blocks, geom, n_refs):
    B = Batch(rng, bpc, layout, W, H, geom, n_refs)
    # first, while the planes are empty: warps at the ends of the filter table, an OBMC block of every size on every
    # plane (neighbour heights 2 ... 24), a compound block of each kind and worst-case pairs with the sharp filter
    for op in (0, 1):
        B.warp_block(0, op, extreme=True)
    for pl in range(B.n_planes):
        for size in sorted(COMP_SIZES, key=lambda s: (s[1] < 64, s[0] * s[1])):      # 64 tall first: the tallest neighbours
            B.obmc(pl, size, inner=True)
    for kind in range(4):
        B.compound(kind=kind, size=(16, 16))
    for _ in range(4):
        B.extreme_compound(f2d=5)
    for _ in range(n_blocks):
        k = int(rng.integers(0, 20))
        pl = int(rng.integers(0, B.n_planes))
        if k < 8:
            B.single(pl)
        elif k < 12:
            B.compound()
        elif k < 14:
            # w_mask of every layout on luma-only blocks (4:2:2 / 4:2:0 masks whatever the picture's layout), at the
            # hooks' shapes and at shapes whose fused item count is not a multiple of 32; and worst-case pairs
            op = 3 + B.n_wmask % 3
            B.n_wmask += 1
            if k == 12:
                B.compound(shape=ODD_COMP_SHAPES[int(rng.integers(0, len(ODD_COMP_SHAPES)))], op=op)
            elif rng.integers(0, 2):
                B.compound(shape=COMP_SIZES[int(rng.integers(0, len(COMP_SIZES)))], op=op)
            else:
                B.extreme_compound()
        elif k < 18:
            B.obmc(pl)
        elif k < 19:
            B.masked_blend(pl)
        else:
            B.warp_block(pl, int(rng.integers(0, 2)))
    return B.finish()


# ------------------------------------------------------------------ expected values: dav1d's mc() / warp_affine()
def predict(B, ctx, out):
    """mc() for an unscaled reference (reference src/recon_tmpl.c:938-988)"""
    g, isz = B.g, np.dtype(B.dt).itemsize
    ebuf = np.zeros((136, EMU_W), B.dt)
    for r in B.pred:
        pl, w, h, mx, my = r.plane, r.w, r.h, r.mx, r.my
        iw, ih, rs = g["w"][pl], g["h"][pl], g["stride"][pl]
        base = B.pics[r.ref].ctypes.data + g["off"][pl] * isz
        fx, fy = int(mx != 0), int(my != 0)
        dx, dy = r.src_x, r.src_y
        if dx < fx * 3 or dy < fy * 3 or dx + w + fx * 4 > iw or dy + h + fy * 4 > ih:
            ctx.emu_edge(w + fx * 7, h + fy * 7, iw, ih, dx - fx * 3, dy - fy * 3, ebuf, EMU_W * isz, base, rs * isz)
            src, ss = ebuf.ctypes.data + (EMU_W * fy * 3 + fx * 3) * isz, EMU_W * isz
        else:
            src, ss = base + (dy * rs + dx) * isz, rs * isz
        if r.op == 1:
            ctx.mct[r.filter2d](out["tmp"].ctypes.data + r.dst_off * 2, src, ss, w, h, mx, my)
        elif r.op == 2:
            ctx.mc[r.filter2d](out["px_tmp"].ctypes.data + r.dst_off * isz, w * isz, src, ss, w, h, mx, my)
        else:
            ctx.mc[r.filter2d](out["dst"].ctypes.data + r.dst_off * isz, rs * isz, src, ss, w, h, mx, my)


def combine(B, ctx, out, stages):
    isz = np.dtype(B.dt).itemsize
    t = out["tmp"].ctypes.data
    for stage in stages:
        for b in stage:
            d, ds = out["dst"].ctypes.data + b.dst_off * isz, B.g["stride"][b.plane] * isz
            t1, t2, m = t + b.tmp1_off * 2, t + b.tmp2_off * 2, out["mask"].ctypes.data + b.mask_off
            if b.op == 0:
                ctx.avg(d, ds, t1, t2, b.w, b.h)
            elif b.op == 1:
                ctx.w_avg(d, ds, t1, t2, b.w, b.h, b.param)
            elif b.op == 2:
                ctx.mask(d, ds, t1, t2, b.w, b.h, m)
            else:
                ctx.w_mask[b.op - 3](d, ds, t1, t2, b.w, b.h, m, b.param)


def blends(B, ctx, out):
    isz = np.dtype(B.dt).itemsize
    for stage in (B.blend, B.blend2):
        for b in stage:
            d, ds = out["dst"].ctypes.data + b.dst_off * isz, B.g["stride"][b.plane] * isz
            t = out["px_tmp"].ctypes.data + b.tmp_off * isz
            if b.op == 0:
                ctx.blend(d, ds, t, b.w, b.h, out["mask"].ctypes.data + b.mask_off)
            elif b.op == 1:
                ctx.blend_v(d, ds, t, b.w, b.h)
            else:
                ctx.blend_h(d, ds, t, b.w, b.h)


def warps(B, ctx, out):
    """warp_affine (reference src/recon_tmpl.c:1115-1165): emu_edge of the 15x15 window when it leaves the plane"""
    g, isz = B.g, np.dtype(B.dt).itemsize
    ebuf = np.zeros((15, 32), B.dt)
    for r in B.warp:
        pl = r.plane
        iw, ih, rs = g["w"][pl], g["h"][pl], g["stride"][pl]
        base = B.pics[r.ref].ctypes.data + g["off"][pl] * isz
        dx, dy = r.src_x, r.src_y
        if dx < 3 or dx + 8 + 4 > iw or dy < 3 or dy + 8 + 4 > ih:
            ctx.emu_edge(15, 15, iw, ih, dx - 3, dy - 3, ebuf, 32 * isz, base, rs * isz)
            src, ss = ebuf.ctypes.data + (32 * 3 + 3) * isz, 32 * isz
        else:
            src, ss = base + (dy * rs + dx) * isz, rs * isz
        abcd = np.array(list(r.abcd), np.int16)
        if r.op:
            ctx.warp8x8t(out["tmp"].ctypes.data + r.dst_off * 2, r.tmp_stride, src, ss, abcd, r.mx, r.my)
        else:
            ctx.warp8x8(out["dst"].ctypes.data + r.dst_off * isz, rs * isz, src, ss, abcd, r.mx, r.my)


def reference(B, ctx):
    """every stage in the frame job's order: prediction, comp, comp2, blend, blend2, warp; and the fused form of the
    compound stages (comp / comp2 on the untouched dst and mask, with the same prep outputs)"""
    out = dict(dst=B.dst.copy(), tmp=B.tmp.copy(), mask=B.mask_buf.copy(), px_tmp=B.px_tmp.copy())
    predict(B, ctx, out)
    fused = dict(dst=B.dst.copy(), tmp=out["tmp"].copy(), mask=B.mask_buf.copy())
    combine(B, ctx, out, (B.comp, B.comp2))
    blends(B, ctx, out)
    warps(B, ctx, out)
    combine(B, ctx, fused, (B.comp, B.comp2))
    return out, dict(dst=fused["dst"], mask=fused["mask"])


def counted_reference(B):
    """the expected buffers, and the oracle's counters over them; where the reference build exists the oracle's
    buffers must equal dav1d's too"""
    o = refs.oracle()
    o.oracle_mc_counts(None)
    exp = reference(B, refs.oracle_mc_ctx(B.bpc))
    out = np.zeros(len(COUNTS), np.int64)
    assert o.oracle_mc_counts(C.c_void_p(out.ctypes.data)) == len(COUNTS)
    if refs.have_ref():
        ref = reference(B, refs.ref_mc_ctx(B.bpc))
        for a, b in zip(exp, ref):
            for k in a:
                assert np.array_equal(a[k], b[k]), "oracle differs from dav1d in " + k
        exp = ref
    return exp, dict(zip(COUNTS, map(int, out)))


# ------------------------------------------------------------------ the kernels
def _records(recs, cls, to_dev):
    if not recs:
        return None, 0
    arr = (cls * len(recs))(*recs)
    return to_dev(np.frombuffer(bytes(arr), np.uint8).copy()), len(recs)


def run(B, lib, to_dev, from_dev, sync, fused=False):
    """the stages on the library: the separate prediction / compound / blend / warp stages, or (fused) only the two
    fused compound stages"""
    names = ("dst", "mask") if fused else ("dst", "tmp", "mask", "px_tmp")
    init = dict(dst=B.dst, tmp=B.tmp, mask=B.mask_buf, px_tmp=B.px_tmp)
    dev = {k: to_dev(init[k]) for k in names}
    pics = [to_dev(p) for p in B.pics]
    fr = _lib.McFrame()
    g = B.g
    for p in range(3):
        fr.ref_plane_off[p], fr.ref_stride[p], fr.ref_w[p], fr.ref_h[p] = g["off"][p], g["stride"][p], g["w"][p], g["h"][p]
        fr.dst_stride[p] = g["stride"][p]
    for k, pic in enumerate(pics):
        assert pic[1] % 4 == 0
        fr.ref[k] = pic[1]
    fr.dst, fr.mask = dev["dst"][1], dev["mask"][1]
    if not fused:
        fr.tmp, fr.px_tmp = dev["tmp"][1], dev["px_tmp"][1]
    bd = B.bd
    if fused:
        stages = [(lib.b200_mc_comp_fused_batch, B.fused, _lib.CompFusedBlock), (lib.b200_mc_comp_fused_batch, B.fused2, _lib.CompFusedBlock)]
    else:
        stages = [(lib.b200_mc_batch, B.pred, _lib.McBlock), (lib.b200_mc_comp_batch, B.comp, _lib.CompBlock),
                  (lib.b200_mc_comp_batch, B.comp2, _lib.CompBlock), (lib.b200_mc_blend_batch, B.blend, _lib.BlendBlock),
                  (lib.b200_mc_blend_batch, B.blend2, _lib.BlendBlock), (lib.b200_mc_warp_batch, B.warp, _lib.WarpBlock)]
    for fn, recs, cls in stages:
        d, n = _records(recs, cls, to_dev)
        if n:
            lib.check(fn(bd, C.byref(fr), d[1], n, None), fn.__name__)
    sync()
    return {k: from_dev(v, init[k]) for k, v in dev.items()}


def compare(exp, got, what):
    for k in got:
        if not np.array_equal(exp[k], got[k]):
            bad = np.nonzero(exp[k] != got[k])[0]
            raise AssertionError("%s %s: %d of %d samples differ, first at %d" % (what, k, len(bad), exp[k].size, bad[0]))


def check_coverage(B, counts, floors):
    """the oracle's counters and the interior / clamped split reach their floors"""
    s = B.stats
    for p in range(B.n_planes):
        if B.geom == "odd":
            assert s["interior"][p] == 0, s
            assert s["pos_inside"][p] >= floors["split"], ("plane %d: too few inside-the-plane records on unaligned geometry" % p, s)
        else:
            assert min(s["interior"][p], s["clamped"][p]) >= floors["split"], ("plane %d" % p, s)
    for k in ("gx0", "gx_end", "gy0", "gy_end"):
        assert s[k] > 0, (k, s)
    if B.geom == "tight":
        assert s["wb_hit"] > 0 and s["wb_miss"] > 0, s
    if B.geom != "odd":
        assert s["mixed_pairs"] > 0, s
    if B.warp:
        assert s["warp_lo"] <= 2 and s["warp_hi"] >= 190, s
    for k, floor in COUNT_FLOORS.items():
        assert counts[k] >= floor, (k, counts)
    assert counts["prep_max_%d" % B.bpc] >= PREP_MAX[B.bpc], counts
    assert {r.op for r in B.pred} == {0, 1, 2} and {b.op for b in B.comp + B.comp2} == set(range(6)), \
        ("an op is missing", {r.op for r in B.pred}, {b.op for b in B.comp + B.comp2})
    assert {r.filter2d for r in B.pred} == set(range(10))
    assert {b.op for b in B.blend} == {0, 2} and B.blend2 and {r.op for r in B.warp} == {0, 1}
    hs = {r.h for r in B.pred if r.op == 2}
    assert {4, 8, 12, 24} | ({2, 6} if B.layout == "420" else set()) <= hs, ("OBMC neighbour heights", sorted(hs))
    for p in range(B.n_planes):
        assert set(plane_shapes(B.layout, p)) <= {(r.w, r.h) for r in B.pred if r.plane == p}, "plane %d: a block shape is missing" % p


# the prep value before the bias that checkasm's worst-case pattern gives under the sharp filter on both axes at the
# half-sample phase, per bit depth: the worst-case compound pairs reach it
PREP_MAX = {8: 9212, 10: 36956, 12: 36983}
# least count of each oracle counter in every case (outputs, or predictions for the tap counts)
COUNT_FLOORS = dict(put_clip_lo=30, put_clip_hi=30, wmask_38=300, wmask_64=16, h_4tap=10, h_8tap=100, v_4tap=10, v_8tap=100,
                    h_identity=50, v_identity=50)


def _case(bpc, layout, W, H, n, geom, n_refs, seed, lib, to_dev, from_dev, sync, split_floor):
    rng = np.random.default_rng(seed)
    B = make_batch(rng, bpc, layout, W, H, n, geom, n_refs)
    (exp, exp_fused), counts = counted_reference(B)
    compare(exp, run(B, lib, to_dev, from_dev, sync), "stages")
    compare(exp_fused, run(B, lib, to_dev, from_dev, sync, fused=True), "fused")
    check_coverage(B, counts, dict(split=split_floor))
    return B, counts


# every bit depth x layout on the emulator at odd sizes (chroma planes of rounded-up size), each geometry in turn
EMU_CASES = [(bpc, lay) + ((201, 137), (135, 73))[i % 2] + (("hooks", "tight", "odd")[i % 3], (1, 8, 3, 5)[i % 4])
             for i, (bpc, lay) in enumerate((b, l) for b in (8, 10, 12) for l in ("420", "422", "444", "400"))]


@pytest.mark.emu
@pytest.mark.parametrize("bpc,layout,W,H,geom,n_refs", EMU_CASES)
def test_emu_inter_prediction(bpc, layout, W, H, geom, n_refs):
    keep = []
    _case(bpc, layout, W, H, 400, geom, n_refs, 2000 + 10 * bpc + list(LAYOUTS).index(layout), refs.emu_lib(),
          _emu_dev(keep), lambda v, like: v[0], lambda: None, split_floor=5)


GPU_CASES = [(8, "420", 1920, 1080, "hooks", 8, 14000), (10, "420", 3840, 2160, "tight", 7, 14000),
             (10, "422", 1920, 1080, "odd", 4, 14000), (12, "444", 1280, 720, "tight", 2, 14000),
             (8, "400", 1280, 720, "hooks", 1, 27000)]


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,layout,W,H,geom,n_refs,n", GPU_CASES)
def test_gpu_inter_prediction(bpc, layout, W, H, geom, n_refs, n):
    from dav1d_b200 import get_lib
    B, _ = _case(bpc, layout, W, H, n, geom, n_refs, 2100 + W + bpc, get_lib(), _torch_dev, _torch_host, _torch_sync,
                 split_floor=200)
    assert len(B.pred) + len(B.comp) + len(B.comp2) + len(B.blend) + len(B.blend2) + len(B.warp) >= 20000


# ------------------------------------------------------------------ reads past the reference picture (emulator only)
_GUARD_CHILD = r'''
import ctypes as C, mmap, sys
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import refs
import test_inter_prediction as T
from dav1d_b200 import _lib

libc = C.CDLL(None, use_errno=True)
libc.mmap.restype = C.c_void_p
libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
PAGE = mmap.PAGESIZE
lib = refs.emu_lib()
for bpc in (8, 10):
    B = T.guard_batch(bpc)
    exp = T.guard_expected(B)
    isz = np.dtype(B.dt).itemsize
    bases = []
    for k, (pic, pl) in enumerate(zip(B.pics, B.guard_plane)):
        # reference k: the last row of plane `pl` ends where a PROT_NONE page begins
        end = (B.g["off"][pl] + B.g["stride"][pl] * B.g["h"][pl]) * isz
        n = (end + PAGE - 1) // PAGE * PAGE
        m = libc.mmap(None, n + PAGE, mmap.PROT_READ | mmap.PROT_WRITE, mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, -1, 0)
        assert m not in (None, C.c_void_p(-1).value)
        assert libc.mprotect(m + n, PAGE, 0) == 0             # PROT_NONE
        base = m + n - end
        C.memmove(base, pic.ctypes.data, end)
        bases.append(base)
    keep = []
    def to_dev(a):
        c = a.copy(); keep.append(c)
        return (c, c.ctypes.data)
    dst, tmp = to_dev(B.dst), to_dev(B.tmp)
    fr = _lib.McFrame()
    for p in range(3):
        fr.ref_plane_off[p], fr.ref_stride[p], fr.ref_w[p], fr.ref_h[p] = B.g["off"][p], B.g["stride"][p], B.g["w"][p], B.g["h"][p]
        fr.dst_stride[p] = B.g["stride"][p]
    for k, b in enumerate(bases):
        fr.ref[k] = b
    fr.dst, fr.tmp = dst[1], tmp[1]
    recs, n = T._records(B.pred, _lib.McBlock, to_dev)
    lib.check(lib.b200_mc_batch(B.bd, C.byref(fr), recs[1], n, None), "b200_mc_batch")
    assert np.array_equal(dst[0], exp["dst"]) and np.array_equal(tmp[0], exp["tmp"]), "wrong bytes at bpc %d" % bpc
print("ok")
'''


def guard_batch(bpc):
    """records on the right and bottom edges of each plane of a tight 4:2:0 picture whose widths are whole words:
    the interior ones read up to the last word of the last row's pitch"""
    rng = np.random.default_rng(2300 + bpc)
    B = Batch(rng, bpc, "420", 200, 120, "tight", 3)
    B.guard_plane = [0, 1, 2]              # reference k guards the end of plane k
    g = B.g
    for pl in range(3):
        rw, rh = g["w"][pl], g["h"][pl]
        for w in (2, 4, 8, 16, 32, 64):
            for h in (2, 4, 8, 16, 32):
                for kx in range(3):
                    for ky in range(2):
                        # gx + w + 7: at the plane's end (word bound one word past the pitch: clamped), one word less
                        # (word bound exactly at the pitch: interior), two words less; the last row, or any row
                        gx = rw - (w + 7) - kx * B.ppw
                        gy = rh - (h + 7) if ky == 0 else int(rng.integers(0, rh - h - 7))
                        r = _lib.McBlock()
                        r.dst_off = B.tmp_alloc(w * h)
                        r.src_x, r.src_y, r.w, r.h = gx + 3, gy + 3, w, h
                        r.mx, r.my = int(rng.integers(0, 16)), int(rng.integers(0, 16))
                        r.filter2d, r.op, r.plane, r.ref = int(rng.integers(0, 10)), 1, pl, pl
                        B.pred.append(r)
                        B.note(r)
    B.finish()
    assert all(B.stats["interior"]) and B.stats["wb_hit"] > 0, B.stats
    return B


def guard_expected(B):
    out = dict(dst=B.dst.copy(), tmp=B.tmp.copy(), mask=B.mask_buf.copy(), px_tmp=B.px_tmp.copy())
    predict(B, checker(B.bpc), out)
    return out


@pytest.mark.emu
def test_emu_interior_reads_stay_inside_the_reference():
    """The interior path loads whole words, up to one word past a block's last tap: only the word bound of
    mc_pred_setup keeps that inside the pitch, and no value comparison sees an over-read that stays inside the
    allocation. Each reference here ends its plane's last row exactly at an inaccessible page (emulator, subprocess)."""
    refs.emu_lib()
    here = os.path.dirname(os.path.abspath(__file__))
    code = _GUARD_CHILD.format(root=os.path.dirname(here), tests=here)
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], capture_output=True, text=True, timeout=600)
    if r.returncode < 0:
        raise AssertionError("kernel read outside the reference picture (signal %d)" % -r.returncode)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
