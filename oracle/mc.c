/*
 * oracle/mc.c — TEST INFRASTRUCTURE (see oracle_common.h).
 *
 * Plain-C restatement of dav1d's motion-compensation DSP functions (reference src/mc_tmpl.c):
 *   put/prep 8-tap + bilinear   :129-187, 246-305, 434-489, 533-586  (filter choice :115-123)
 *   put/prep scaled              :189-244, 307-358, 491-531, 588-626
 *   avg / w_avg / mask / w_mask  :628-681, 724-781
 *   blend / blend_v / blend_h    :683-722
 *   warp_affine_8x8{,t}          :799-866
 *   emu_edge / resize            :868-944
 * One body serves 8 bpc and 10/12 bpc: `bdmax` (255/1023/4095) selects pixel width,
 * intermediate_bits (4/4/2) and PREP_BIAS (0/8192/8192) as in :39-49.
 * All strides are in BYTES like the reference's function pointers.
 */
#include "oracle_common.h"
#include "tables_gen.h"

typedef struct { int hbd, bdmax, ibits, bias; } BdInfo;
static inline BdInfo bdinfo(int bdmax) {
    BdInfo b;
    b.hbd = bdmax > 255; b.bdmax = bdmax;
    b.ibits = !b.hbd ? 4 : 14 - (o_ulog2((unsigned)bdmax) + 1);
    b.bias = b.hbd ? 8192 : 0;
    return b;
}
static inline int PX(const void *p, int hbd, ptrdiff_t i) {
    return hbd ? ((const uint16_t *)p)[i] : ((const uint8_t *)p)[i];
}
static inline void SPX(void *p, int hbd, ptrdiff_t i, int v) {
    if (hbd) ((uint16_t *)p)[i] = (uint16_t)v; else ((uint8_t *)p)[i] = (uint8_t)v;
}
#define PSTRIDE(bytes, hbd) ((hbd) ? (bytes) / 2 : (bytes))

/* Coverage counters for the tests (oracle_mc_counts) over the unscaled put / prep and w_mask: they only observe.
 * PREP_MAX_* hold the largest |prep| value before the bias is removed, per bit depth (8 / 10 / 12); the tap counts
 * are per prediction and axis: a 4-tap or 8-tap set (w or h <= 4 selects the 4-tap one), or no phase on the axis. */
enum { MC_PUT_CLIP_LO, MC_PUT_CLIP_HI, MC_PREP_MAX_8, MC_PREP_MAX_10, MC_PREP_MAX_12, MC_WMASK_38, MC_WMASK_64,
       MC_H_4TAP, MC_H_8TAP, MC_V_4TAP, MC_V_8TAP, MC_H_IDENTITY, MC_V_IDENTITY, MC_N_COUNTS };
static long mc_counts[MC_N_COUNTS];

/* copies the counters to out[MC_N_COUNTS] and resets them; returns MC_N_COUNTS */
ORACLE_API int oracle_mc_counts(long *out)
{
    if (out) memcpy(out, mc_counts, sizeof(mc_counts));
    memset(mc_counts, 0, sizeof(mc_counts));
    return MC_N_COUNTS;
}
/* a put output: counted when the clip changes it */
static inline int put_clip(int v, int bdmax)
{
    if (v < 0) mc_counts[MC_PUT_CLIP_LO]++;
    else if (v > bdmax) mc_counts[MC_PUT_CLIP_HI]++;
    return o_clip(v, 0, bdmax);
}
/* a prep output before the bias is removed */
static inline int prep_out(int v, BdInfo b)
{
    long *const m = &mc_counts[MC_PREP_MAX_8 + (b.bdmax > 255) + (b.bdmax > 1023)];
    if (o_abs(v) > *m) *m = o_abs(v);
    return v - b.bias;
}
static void count_taps(int mx, int my, int w, int h, int bilin)
{
    if (!mx) mc_counts[MC_H_IDENTITY]++; else if (!bilin) mc_counts[w > 4 ? MC_H_8TAP : MC_H_4TAP]++;
    if (!my) mc_counts[MC_V_IDENTITY]++; else if (!bilin) mc_counts[h > 4 ? MC_V_8TAP : MC_V_4TAP]++;
}

/* enum Filter2d -> (horizontal, vertical) Dav1dFilterMode; reference src/levels.h:184-196,
 * src/mc_tmpl.c:406-414 */
static const uint8_t f2d_h[9] = { 0, 0, 0, 2, 2, 2, 1, 1, 1 };
static const uint8_t f2d_v[9] = { 0, 1, 2, 0, 1, 2, 0, 1, 2 };

static const int8_t *h_filter(int f2d, int mx, int w) {
    if (!mx) return NULL;
    const int t = f2d_h[f2d];
    return w > 4 ? b200_mc_subpel_filters[t][mx - 1] : b200_mc_subpel_filters[3 + (t & 1)][mx - 1];
}
static const int8_t *v_filter(int f2d, int my, int h) {
    if (!my) return NULL;
    const int t = f2d_v[f2d];
    return h > 4 ? b200_mc_subpel_filters[t][my - 1] : b200_mc_subpel_filters[3 + (t & 1)][my - 1];
}

static inline int tap8_px(const void *src, int hbd, ptrdiff_t x, const int8_t *f, ptrdiff_t st) {
    int s = 0;
    for (int k = 0; k < 8; k++) s += f[k] * PX(src, hbd, x + (k - 3) * st);
    return s;
}
static inline int tap8_mid(const int16_t *m, ptrdiff_t x, const int8_t *f, ptrdiff_t st) {
    int s = 0;
    for (int k = 0; k < 8; k++) s += f[k] * m[x + (k - 3) * st];
    return s;
}
#define RND(v, sh) (((v) + ((1 << (sh)) >> 1)) >> (sh))

/* put (op = 0, out = pixels with out_stride bytes) or prep (op = 1, out = int16, dense w) */
static void mc_8tap(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride,
                    int w, int h, int mx, int my, int f2d, int bdmax)
{
    const BdInfo b = bdinfo(bdmax);
    const int hbd = b.hbd, ib = b.ibits;
    const ptrdiff_t ss = PSTRIDE(src_stride, hbd), ds = op ? w : PSTRIDE(out_stride, hbd);
    const int8_t *fh = h_filter(f2d, mx, w), *fv = v_filter(f2d, my, h);
    int16_t *tmp = (int16_t *)out;
    static __thread int16_t mid[128 * 135];
    count_taps(mx, my, w, h, 0);

    if (fh && fv) {
        for (int y = 0; y < h + 7; y++)
            for (int x = 0; x < w; x++)
                mid[y * 128 + x] = (int16_t)RND(tap8_px(src, hbd, (y - 3) * ss + x, fh, 1), 6 - ib);
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int s = tap8_mid(mid + (y + 3) * 128, x, fv, 128);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(RND(s, 6), b);
                else SPX(out, hbd, y * ds + x, put_clip(RND(s, 6 + ib), bdmax));
            }
    } else if (fh) {
        const int irnd = 32 + ((1 << (6 - ib)) >> 1);
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int s = tap8_px(src, hbd, y * ss + x, fh, 1);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(RND(s, 6 - ib), b);
                else SPX(out, hbd, y * ds + x, put_clip((s + irnd) >> 6, bdmax));
            }
    } else if (fv) {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int s = tap8_px(src, hbd, y * ss + x, fv, ss);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(RND(s, 6 - ib), b);
                else SPX(out, hbd, y * ds + x, put_clip(RND(s, 6), bdmax));
            }
    } else {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int p = PX(src, hbd, y * ss + x);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(p << ib, b);
                else SPX(out, hbd, y * ds + x, p);
            }
    }
}

static void mc_bilin(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride,
                     int w, int h, int mx, int my, int bdmax)
{
    const BdInfo b = bdinfo(bdmax);
    const int hbd = b.hbd, ib = b.ibits;
    const ptrdiff_t ss = PSTRIDE(src_stride, hbd), ds = op ? w : PSTRIDE(out_stride, hbd);
    int16_t *tmp = (int16_t *)out;
    static __thread int16_t mid[128 * 129];
    count_taps(mx, my, w, h, 1);
#define BIL(a, bb, m) (16 * (a) + (m) * ((bb) - (a)))
    if (mx && my) {
        for (int y = 0; y < h + 1; y++)
            for (int x = 0; x < w; x++)
                mid[y * 128 + x] = (int16_t)RND(BIL(PX(src, hbd, y * ss + x), PX(src, hbd, y * ss + x + 1), mx), 4 - ib);
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int s = BIL(mid[y * 128 + x], mid[(y + 1) * 128 + x], my);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(RND(s, 4), b);
                else SPX(out, hbd, y * ds + x, put_clip(RND(s, 4 + ib), bdmax));
            }
    } else if (mx) {
        const int irnd = (1 << ib) >> 1;
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int px = RND(BIL(PX(src, hbd, y * ss + x), PX(src, hbd, y * ss + x + 1), mx), 4 - ib);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(px, b);
                else SPX(out, hbd, y * ds + x, put_clip((px + irnd) >> ib, bdmax));
            }
    } else if (my) {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int s = BIL(PX(src, hbd, y * ss + x), PX(src, hbd, (y + 1) * ss + x), my);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(RND(s, 4 - ib), b);
                else SPX(out, hbd, y * ds + x, put_clip(RND(s, 4), bdmax));
            }
    } else {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int p = PX(src, hbd, y * ss + x);
                if (op) tmp[y * ds + x] = (int16_t)prep_out(p << ib, b);
                else SPX(out, hbd, y * ds + x, p);
            }
    }
}

/* c->mc[filter2d] / c->mct[filter2d] (filter2d 0..8 = 8-tap pairs, 9 = bilinear) */
ORACLE_API void oracle_mc_put(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
                              int w, int h, int mx, int my, int filter2d, int bdmax) {
    if (filter2d == 9) mc_bilin(0, dst, dst_stride, src, src_stride, w, h, mx, my, bdmax);
    else mc_8tap(0, dst, dst_stride, src, src_stride, w, h, mx, my, filter2d, bdmax);
}
ORACLE_API void oracle_mc_prep(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h,
                               int mx, int my, int filter2d, int bdmax) {
    if (filter2d == 9) mc_bilin(1, tmp, 0, src, src_stride, w, h, mx, my, bdmax);
    else mc_8tap(1, tmp, 0, src, src_stride, w, h, mx, my, filter2d, bdmax);
}

/* ---- scaled references: reference src/mc_tmpl.c:189-244, 307-358, 491-531, 588-626 ---- */
static void mc_scaled(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride,
                      int w, int h, int mx, int my, int dx, int dy, int f2d, int bdmax)
{
    const BdInfo b = bdinfo(bdmax);
    const int hbd = b.hbd, ib = b.ibits;
    const ptrdiff_t ss = PSTRIDE(src_stride, hbd), ds = op ? w : PSTRIDE(out_stride, hbd);
    int16_t *tmp = (int16_t *)out;
    if (f2d == 9) {
        int16_t mid[2][128];
        int in_y = -2;
        ptrdiff_t srow = 0;
        for (int yy = 0; yy < h; yy++) {
            const int y = my >> 10, dmy = my & 0x3ff;
            const int16_t *m1 = mid[y & 1], *m2 = mid[(y + 1) & 1];
            while (in_y < y) {
                int imx = mx, ioff = 0;
                int16_t *mp = mid[in_y & 1];
                for (int x = 0; x < w; x++) {
                    mp[x] = (int16_t)RND(BIL(PX(src, hbd, srow + ioff), PX(src, hbd, srow + ioff + 1), imx >> 6), 4 - ib);
                    imx += dx; ioff += imx >> 10; imx &= 0x3ff;
                }
                srow += ss; in_y++;
            }
            for (int x = 0; x < w; x++) {
                const int s = BIL(m1[x], m2[x], dmy >> 6);
                if (op) tmp[yy * ds + x] = (int16_t)(RND(s, 4) - b.bias);
                else SPX(out, hbd, yy * ds + x, o_clip(RND(s, 4 + ib), 0, bdmax));
            }
            my += dy;
        }
        return;
    }
    int16_t mid[8][128];
    int order[8];
    for (int i = 0; i < 8; i++) order[i] = i;
    int in_y = -8;
    ptrdiff_t srow = -3 * ss;
    const int irnd = (1 << ib) >> 1;
    for (int yy = 0; yy < h; yy++) {
        const int src_y = my >> 10;
        const int8_t *fv = v_filter(f2d, (my & 0x3ff) >> 6, h);
        while (in_y < src_y) {
            int imx = mx, ioff = 0;
            const int first = order[0];
            for (int i = 0; i < 7; i++) order[i] = order[i + 1];
            order[7] = first;
            int16_t *mp = mid[first];
            for (int x = 0; x < w; x++) {
                const int8_t *fh = h_filter(f2d, imx >> 6, w);
                mp[x] = fh ? (int16_t)RND(tap8_px(src, hbd, srow + ioff, fh, 1), 6 - ib)
                           : (int16_t)(PX(src, hbd, srow + ioff) << ib);
                imx += dx; ioff += imx >> 10; imx &= 0x3ff;
            }
            srow += ss; in_y++;
        }
        for (int x = 0; x < w; x++) {
            int s = 0;
            if (fv) for (int k = 0; k < 8; k++) s += fv[k] * mid[order[k]][x];
            if (op) tmp[yy * ds + x] = (int16_t)((fv ? RND(s, 6) : mid[order[3]][x]) - b.bias);
            else SPX(out, hbd, yy * ds + x,
                     o_clip(fv ? RND(s, 6 + ib) : (mid[order[3]][x] + irnd) >> ib, 0, bdmax));
        }
        my += dy;
    }
}
ORACLE_API void oracle_mc_put_scaled(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
                                     int w, int h, int mx, int my, int dx, int dy, int filter2d, int bdmax) {
    mc_scaled(0, dst, dst_stride, src, src_stride, w, h, mx, my, dx, dy, filter2d, bdmax);
}
ORACLE_API void oracle_mc_prep_scaled(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h,
                                      int mx, int my, int dx, int dy, int filter2d, int bdmax) {
    mc_scaled(1, tmp, 0, src, src_stride, w, h, mx, my, dx, dy, filter2d, bdmax);
}

/* ---- compound ---- */
ORACLE_API void oracle_avg(void *dst, ptrdiff_t dst_stride, const int16_t *t1, const int16_t *t2,
                           int w, int h, int bdmax) {
    const BdInfo b = bdinfo(bdmax);
    const ptrdiff_t ds = PSTRIDE(dst_stride, b.hbd);
    const int sh = b.ibits + 1, rnd = (1 << b.ibits) + b.bias * 2;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            SPX(dst, b.hbd, y * ds + x, o_clip((t1[y * w + x] + t2[y * w + x] + rnd) >> sh, 0, bdmax));
}
ORACLE_API void oracle_w_avg(void *dst, ptrdiff_t dst_stride, const int16_t *t1, const int16_t *t2,
                             int w, int h, int weight, int bdmax) {
    const BdInfo b = bdinfo(bdmax);
    const ptrdiff_t ds = PSTRIDE(dst_stride, b.hbd);
    const int sh = b.ibits + 4, rnd = (8 << b.ibits) + b.bias * 16;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            SPX(dst, b.hbd, y * ds + x,
                o_clip((t1[y * w + x] * weight + t2[y * w + x] * (16 - weight) + rnd) >> sh, 0, bdmax));
}
ORACLE_API void oracle_mask(void *dst, ptrdiff_t dst_stride, const int16_t *t1, const int16_t *t2,
                            int w, int h, const uint8_t *mask, int bdmax) {
    const BdInfo b = bdinfo(bdmax);
    const ptrdiff_t ds = PSTRIDE(dst_stride, b.hbd);
    const int sh = b.ibits + 6, rnd = (32 << b.ibits) + b.bias * 64;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int m = mask[y * w + x];
            SPX(dst, b.hbd, y * ds + x, o_clip((t1[y * w + x] * m + t2[y * w + x] * (64 - m) + rnd) >> sh, 0, bdmax));
        }
}
/* layout: 0 = 4:4:4, 1 = 4:2:2, 2 = 4:2:0 (index of c->w_mask[]) */
ORACLE_API void oracle_w_mask(void *dst, ptrdiff_t dst_stride, const int16_t *t1, const int16_t *t2,
                              int w, int h, uint8_t *mask, int sign, int layout, int bdmax) {
    const BdInfo b = bdinfo(bdmax);
    const ptrdiff_t ds = PSTRIDE(dst_stride, b.hbd);
    const int ss_hor = layout > 0, ss_ver = layout == 2;
    const int bitdepth = o_ulog2((unsigned)bdmax) + 1;
    const int sh = b.ibits + 6, rnd = (32 << b.ibits) + b.bias * 64;
    const int mask_sh = bitdepth + b.ibits - 4, mask_rnd = 1 << (mask_sh - 5);
    for (int y = 0; y < h; y++) {
        uint8_t *mrow = mask + (ss_ver ? (y >> 1) : y) * (w >> ss_hor);
        for (int x = 0; x < w; x++) {
            const int d = t1[y * w + x] - t2[y * w + x];
            const int m = o_min(38 + ((o_abs(d) + mask_rnd) >> mask_sh), 64);
            mc_counts[MC_WMASK_38] += m == 38; mc_counts[MC_WMASK_64] += m == 64;
            SPX(dst, b.hbd, y * ds + x, o_clip((d * m + t2[y * w + x] * 64 + rnd) >> sh, 0, bdmax));
            if (!ss_hor) { mrow[x] = (uint8_t)m; continue; }
            x++;
            const int d2 = t1[y * w + x] - t2[y * w + x];
            const int n = o_min(38 + ((o_abs(d2) + mask_rnd) >> mask_sh), 64);
            mc_counts[MC_WMASK_38] += n == 38; mc_counts[MC_WMASK_64] += n == 64;
            SPX(dst, b.hbd, y * ds + x, o_clip((d2 * n + t2[y * w + x] * 64 + rnd) >> sh, 0, bdmax));
            if (ss_ver && (y & 1)) mrow[x >> 1] = (uint8_t)((m + n + mrow[x >> 1] + 2 - sign) >> 2);
            else if (ss_ver)       mrow[x >> 1] = (uint8_t)(m + n);
            else                   mrow[x >> 1] = (uint8_t)((m + n + 1 - sign) >> 1);
        }
    }
}

/* ---- OBMC / inter-intra blends ---- */
#define BLEND(a, bb, m) ((((a) * (64 - (m)) + (bb) * (m)) + 32) >> 6)
ORACLE_API void oracle_blend(void *dst, ptrdiff_t dst_stride, const void *tmp, int w, int h,
                             const uint8_t *mask, int bdmax) {
    const int hbd = bdmax > 255; const ptrdiff_t ds = PSTRIDE(dst_stride, hbd);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            SPX(dst, hbd, y * ds + x, BLEND(PX(dst, hbd, y * ds + x), PX(tmp, hbd, y * w + x), mask[y * w + x]));
}
ORACLE_API void oracle_blend_v(void *dst, ptrdiff_t dst_stride, const void *tmp, int w, int h, int bdmax) {
    const int hbd = bdmax > 255; const ptrdiff_t ds = PSTRIDE(dst_stride, hbd);
    const uint8_t *mask = &b200_obmc_masks[w];
    for (int y = 0; y < h; y++)
        for (int x = 0; x < (w * 3) >> 2; x++)
            SPX(dst, hbd, y * ds + x, BLEND(PX(dst, hbd, y * ds + x), PX(tmp, hbd, y * w + x), mask[x]));
}
ORACLE_API void oracle_blend_h(void *dst, ptrdiff_t dst_stride, const void *tmp, int w, int h, int bdmax) {
    const int hbd = bdmax > 255; const ptrdiff_t ds = PSTRIDE(dst_stride, hbd);
    const uint8_t *mask = &b200_obmc_masks[h];
    for (int y = 0; y < (h * 3) >> 2; y++)
        for (int x = 0; x < w; x++)
            SPX(dst, hbd, y * ds + x, BLEND(PX(dst, hbd, y * ds + x), PX(tmp, hbd, y * w + x), mask[y]));
}

/* ---- 8x8 affine warp; op 0: pixels (out_stride bytes), op 1: int16 (out_stride elements) ---- */
ORACLE_API void oracle_warp8x8(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride,
                               const int16_t *abcd, int mx, int my, int bdmax) {
    const BdInfo b = bdinfo(bdmax);
    const int hbd = b.hbd, ib = b.ibits;
    const ptrdiff_t ss = PSTRIDE(src_stride, hbd), ds = op ? out_stride : PSTRIDE(out_stride, hbd);
    int16_t mid[15 * 8];
    for (int y = 0; y < 15; y++, mx += abcd[1])
        for (int x = 0, tmx = mx; x < 8; x++, tmx += abcd[0]) {
            const int8_t *f = b200_mc_warp_filter[64 + ((tmx + 512) >> 10)];
            mid[y * 8 + x] = (int16_t)RND(tap8_px(src, hbd, (y - 3) * ss + x, f, 1), 7 - ib);
        }
    for (int y = 0; y < 8; y++, my += abcd[3])
        for (int x = 0, tmy = my; x < 8; x++, tmy += abcd[2]) {
            const int8_t *f = b200_mc_warp_filter[64 + ((tmy + 512) >> 10)];
            const int s = tap8_mid(mid + (y + 3) * 8, x, f, 8);
            if (op) ((int16_t *)out)[y * ds + x] = (int16_t)(RND(s, 7) - b.bias);
            else SPX(out, hbd, y * ds + x, o_clip(RND(s, 7 + ib), 0, bdmax));
        }
}

/* ---- edge emulation: replicate-pad a bw x bh window at (x, y) of an iw x ih plane ---- */
ORACLE_API void oracle_emu_edge(intptr_t bw, intptr_t bh, intptr_t iw, intptr_t ih, intptr_t x, intptr_t y,
                                void *dst, ptrdiff_t dst_stride, const void *ref, ptrdiff_t ref_stride, int bdmax) {
    const int hbd = bdmax > 255;
    const ptrdiff_t ds = PSTRIDE(dst_stride, hbd), rs = PSTRIDE(ref_stride, hbd);
    for (intptr_t j = 0; j < bh; j++) {
        const intptr_t sy = o_clip((int)(y + j), 0, (int)ih - 1);
        for (intptr_t i = 0; i < bw; i++) {
            const intptr_t sx = o_clip((int)(x + i), 0, (int)iw - 1);
            SPX(dst, hbd, j * ds + i, PX(ref, hbd, sy * rs + sx));
        }
    }
}

/* ---- super-resolution horizontal resample ---- */
ORACLE_API void oracle_resize(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
                              int dst_w, int h, int src_w, int dx, int mx0, int bdmax) {
    const int hbd = bdmax > 255;
    const ptrdiff_t ds = PSTRIDE(dst_stride, hbd), ss = PSTRIDE(src_stride, hbd);
    for (int y = 0; y < h; y++) {
        int mx = mx0, src_x = -1;
        for (int x = 0; x < dst_w; x++) {
            const int8_t *F = b200_resize_filter[mx >> 8];
            int s = 0;
            for (int k = 0; k < 8; k++) s += F[k] * PX(src, hbd, y * ss + o_clip(src_x - 3 + k, 0, src_w - 1));
            SPX(dst, hbd, y * ds + x, o_clip((-s + 64) >> 7, 0, bdmax));
            mx += dx; src_x += mx >> 14; mx &= 0x3fff;
        }
    }
}

/* ---- batched forms over the records the CUDA kernels consume (layouts restate
 * B200McFrame / B200McBlock / B200CompBlock / B200BlendBlock / B200WarpBlock of include/b200av1.h).
 * Prediction follows dav1d's own route for blocks that leave the picture: emu_edge into a
 * scratch window, then the regular mc function (reference src/recon_tmpl.c:956-988). */
typedef struct {
    const void *ref[8]; uint32_t ref_plane_off[3]; int32_t ref_stride[3], ref_w[3], ref_h[3];
    void *dst; int32_t dst_stride[3]; int16_t *tmp; uint8_t *mask; const void *px_tmp;
} OracleMcFrame;
typedef struct { uint32_t dst_off; int32_t src_x, src_y; uint8_t w, h, mx, my, filter2d, op, plane, ref; } OracleMcBlock;
typedef struct { uint32_t dst_off, tmp1_off, tmp2_off, mask_off; uint8_t w, h, op, param, plane, pad[3]; } OracleCompBlock;
typedef struct { uint32_t dst_off, tmp_off, mask_off; uint8_t w, h, op, plane; } OracleBlendBlock;
typedef struct { uint32_t dst_off; int32_t src_x, src_y, mx, my; int16_t abcd[4]; uint16_t tmp_stride; uint8_t op, plane, ref, pad; } OracleWarpBlock;

ORACLE_API void oracle_mc_batch(int bdmax, const OracleMcFrame *f, const OracleMcBlock *b, int n) {
    const int hbd = bdmax > 255; const size_t px = hbd ? 2 : 1;
    static __thread uint8_t win[135 * 135 * 2];
    for (int i = 0; i < n; i++, b++) {
        const int pl = b->plane;
        const uint8_t *ref = (const uint8_t *)f->ref[b->ref] + (size_t)f->ref_plane_off[pl] * px;
        oracle_emu_edge(b->w + 7, b->h + 7, f->ref_w[pl], f->ref_h[pl], b->src_x - 3, b->src_y - 3, win,
                        135 * (ptrdiff_t)px, ref, f->ref_stride[pl] * (ptrdiff_t)px, bdmax);
        const uint8_t *src = win + (3 * 135 + 3) * px;
        if (b->op == 2)       /* put into the pixel scratch (pitch w): the overlapped predictions of obmc(), src/recon_tmpl.c:1052-1113 */
            oracle_mc_put((uint8_t *)f->px_tmp + (size_t)b->dst_off * px, b->w * (ptrdiff_t)px, src, 135 * (ptrdiff_t)px, b->w, b->h,
                          b->mx, b->my, b->filter2d, bdmax);
        else if (b->op) oracle_mc_prep(f->tmp + b->dst_off, src, 135 * (ptrdiff_t)px, b->w, b->h, b->mx, b->my, b->filter2d, bdmax);
        else oracle_mc_put((uint8_t *)f->dst + (size_t)b->dst_off * px, f->dst_stride[pl] * (ptrdiff_t)px, src,
                           135 * (ptrdiff_t)px, b->w, b->h, b->mx, b->my, b->filter2d, bdmax);
    }
}
ORACLE_API void oracle_mc_comp_batch(int bdmax, const OracleMcFrame *f, const OracleCompBlock *b, int n) {
    const size_t px = bdmax > 255 ? 2 : 1;
    for (int i = 0; i < n; i++, b++) {
        void *dst = (uint8_t *)f->dst + (size_t)b->dst_off * px;
        const ptrdiff_t ds = f->dst_stride[b->plane] * (ptrdiff_t)px;
        const int16_t *t1 = f->tmp + b->tmp1_off, *t2 = f->tmp + b->tmp2_off;
        if (b->op == 0) oracle_avg(dst, ds, t1, t2, b->w, b->h, bdmax);
        else if (b->op == 1) oracle_w_avg(dst, ds, t1, t2, b->w, b->h, b->param, bdmax);
        else if (b->op == 2) oracle_mask(dst, ds, t1, t2, b->w, b->h, f->mask + b->mask_off, bdmax);
        else oracle_w_mask(dst, ds, t1, t2, b->w, b->h, f->mask + b->mask_off, b->param, b->op - 3, bdmax);
    }
}
ORACLE_API void oracle_mc_blend_batch(int bdmax, const OracleMcFrame *f, const OracleBlendBlock *b, int n) {
    const size_t px = bdmax > 255 ? 2 : 1;
    for (int i = 0; i < n; i++, b++) {
        void *dst = (uint8_t *)f->dst + (size_t)b->dst_off * px;
        const ptrdiff_t ds = f->dst_stride[b->plane] * (ptrdiff_t)px;
        const void *tmp = (const uint8_t *)f->px_tmp + (size_t)b->tmp_off * px;
        if (b->op == 0) oracle_blend(dst, ds, tmp, b->w, b->h, f->mask + b->mask_off, bdmax);
        else if (b->op == 1) oracle_blend_v(dst, ds, tmp, b->w, b->h, bdmax);
        else oracle_blend_h(dst, ds, tmp, b->w, b->h, bdmax);
    }
}
ORACLE_API void oracle_mc_warp_batch(int bdmax, const OracleMcFrame *f, const OracleWarpBlock *b, int n) {
    const int hbd = bdmax > 255; const size_t px = hbd ? 2 : 1;
    uint8_t win[15 * 15 * 2];
    for (int i = 0; i < n; i++, b++) {
        const int pl = b->plane;
        const uint8_t *ref = (const uint8_t *)f->ref[b->ref] + (size_t)f->ref_plane_off[pl] * px;
        oracle_emu_edge(15, 15, f->ref_w[pl], f->ref_h[pl], b->src_x - 3, b->src_y - 3, win, 15 * (ptrdiff_t)px,
                        ref, f->ref_stride[pl] * (ptrdiff_t)px, bdmax);
        const uint8_t *src = win + (3 * 15 + 3) * px;
        if (b->op) oracle_warp8x8(1, f->tmp + b->dst_off, b->tmp_stride, src, 15 * (ptrdiff_t)px, b->abcd, b->mx, b->my, bdmax);
        else oracle_warp8x8(0, (uint8_t *)f->dst + (size_t)b->dst_off * px, f->dst_stride[pl] * (ptrdiff_t)px, src,
                            15 * (ptrdiff_t)px, b->abcd, b->mx, b->my, bdmax);
    }
}
