/*
 * oracle/looprestoration.c — TEST INFRASTRUCTURE (see oracle_common.h).
 *
 * Plain-C restatement of dav1d's loop-restoration filters, written as direct 2-D formulas over
 * a virtual padded source instead of the reference's rolling row buffers:
 *   wiener_c (7-tap separable)            reference src/looprestoration_tmpl.c:44-386
 *   sgr_3x3_c / sgr_5x5_c / sgr_mix_c     reference src/looprestoration_tmpl.c:419-1327
 * Virtual source S(x, y), x in [-3, w+2], y in [-3, h+2]  (reference :265-277, 363-372, 704-...):
 *   rows 0..h-1   the unit itself (pre-LR samples); left of it `left[y][4+x]`, right of it the
 *                 picture, or edge replication when LR_HAVE_LEFT / LR_HAVE_RIGHT are clear
 *   rows < 0      lpf[0..1] (row -3 repeats lpf[0]) with LR_HAVE_TOP, else row 0 repeated
 *   rows >= h     lpf[6..7] (row h+2 repeats lpf[7]) when the bottom is used, else row h-1 repeated;
 *                 the reference's short-stripe exits skip the bottom rows for tiny / odd h, which
 *                 `use_bottom` below reproduces.
 */
#include "oracle_common.h"
#include "tables_gen.h"
#include <stdlib.h>

/* Branch counters for the tests (oracle_lr_counts): per plane class (0 luma, 1 chroma), the restoration units of
 * oracle_lr_frame by filter (one per unit and stripe), the stripes by their edges and unit row, and the samples that took
 * a clip or clamp. The filters count into the class of the plane oracle_lr_frame is restoring (luma for direct calls).
 * They only observe. */
enum { LR_NONE, LR_WIENER, LR_SGR5, LR_SGR3, LR_SGR_MIX, LR_EXT_H, LR_PULLED_UP, LR_HOR_CLIP_LO, LR_HOR_CLIP_HI,
       LR_OUT_CLIP_LO, LR_OUT_CLIP_HI, LR_Z0, LR_Z255, LR_SGR_BIG, LR_TOP, LR_NO_TOP, LR_BOT, LR_NO_BOT, LR_BOT_CLAMP, LR_N };
static long lr_counts[2][LR_N];
static int lr_cls;

/* copies the counters to out[2][LR_N] (plane class, counter) and resets them; returns LR_N */
ORACLE_API int oracle_lr_counts(long *out)
{
    if (out) memcpy(out, lr_counts, sizeof(lr_counts));
    memset(lr_counts, 0, sizeof(lr_counts));
    return LR_N;
}

typedef struct {
    const void *p, *left, *lpf;
    ptrdiff_t ps;
    int w, h, edges, hbd, use_bottom;
} LrSrc;

static inline int PXv(const void *p, int hbd, ptrdiff_t i) {
    return hbd ? ((const uint16_t *)p)[i] : ((const uint8_t *)p)[i];
}

static int lr_S(const LrSrc *s, int x, int y) {
    const ptrdiff_t rb = s->ps * (s->hbd ? 2 : 1);          /* row pitch in bytes */
    const void *row; int from_unit = 0;
    if (y < 0 && (s->edges & 4)) {
        row = (const uint8_t *)s->lpf + (ptrdiff_t)((y < -2 ? -2 : y) + 2) * rb;
    } else if (y >= s->h && s->use_bottom) {
        row = (const uint8_t *)s->lpf + (ptrdiff_t)(6 + (y - s->h > 1 ? 1 : y - s->h)) * rb;
    } else {
        y = y < 0 ? 0 : y >= s->h ? s->h - 1 : y;
        row = (const uint8_t *)s->p + (ptrdiff_t)y * rb; from_unit = 1;
    }
    if (x < 0) {
        if (!(s->edges & 1)) return PXv(row, s->hbd, 0);
        if (from_unit && s->left) return PXv(s->left, s->hbd, (ptrdiff_t)y * 4 + 4 + x);
        return PXv(row, s->hbd, x);
    }
    if (x >= s->w && !(s->edges & 2)) return PXv(row, s->hbd, s->w - 1);
    return PXv(row, s->hbd, x);
}

static void st_px(void *p, int hbd, ptrdiff_t i, int v) {
    if (hbd) ((uint16_t *)p)[i] = (uint16_t)v; else ((uint8_t *)p)[i] = (uint8_t)v;
}

/* filter[2][8] as built by lr_stripe (reference src/lr_apply_tmpl.c:55-72) */
ORACLE_API void oracle_wiener(void *p, ptrdiff_t stride_bytes, const void *left, const void *lpf, int w, int h,
                              const int16_t filter[2][8], int edges, int bdmax)
{
    const int hbd = bdmax > 255, bitdepth = o_ulog2((unsigned)bdmax) + 1;
    LrSrc s = { p, left, lpf, hbd ? stride_bytes / 2 : stride_bytes, w, h, edges, hbd, 0 };
    s.use_bottom = (edges & 8) && h > ((edges & 4) ? 3 : 5);
    const int rbh = 3 + (bitdepth == 12) * 2, rbv = 11 - (bitdepth == 12) * 2;
    const int clip_limit = 1 << (bitdepth + 1 + 7 - rbh);
    const int round_offset = 1 << (bitdepth + (rbv - 1));
    /* horizontally filtered rows -3 .. h+2 */
    uint16_t *hor = malloc(sizeof(uint16_t) * (size_t)(h + 6) * w);
    for (int y = -3; y < h + 3; y++)
        for (int x = 0; x < w; x++) {
            int sum = 1 << (bitdepth + 6);
            if (!hbd) sum += lr_S(&s, x, y) * 128;
            for (int i = 0; i < 7; i++) sum += lr_S(&s, x + i - 3, y) * filter[0][i];
            const int v = (sum + (1 << (rbh - 1))) >> rbh;
            lr_counts[lr_cls][LR_HOR_CLIP_LO] += v < 0;
            lr_counts[lr_cls][LR_HOR_CLIP_HI] += v > clip_limit - 1;
            hor[(size_t)(y + 3) * w + x] = (uint16_t)o_clip(v, 0, clip_limit - 1);
        }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int sum = -round_offset;
            for (int k = 0; k < 7; k++) sum += hor[(size_t)(y + k) * w + x] * filter[1][k];
            const int v = (sum + (1 << (rbv - 1))) >> rbv;
            lr_counts[lr_cls][LR_OUT_CLIP_LO] += v < 0;
            lr_counts[lr_cls][LR_OUT_CLIP_HI] += v > bdmax;
            st_px(p, hbd, y * s.ps + x, o_clip(v, 0, bdmax));
        }
    free(hor);
}

/* a/b planes for box size n (9 or 25): arrays indexed [(y + 1) * (w + 2) + (x + 1)], x in [-1, w], y in [-1, h] */
static void sgr_ab(const LrSrc *s, int r, unsigned strength, int bdmax, int32_t *A, int32_t *B)
{
    const int b8 = (o_ulog2((unsigned)bdmax) + 1) - 8;
    const int n = (2 * r + 1) * (2 * r + 1), one_by_x = r == 2 ? 164 : 455;
    const int w = s->w, h = s->h;
    for (int y = -1; y <= h; y++)
        for (int x = -1; x <= w; x++) {
            int sum = 0, sumsq = 0;
            for (int dy = -r; dy <= r; dy++)
                for (int dx = -r; dx <= r; dx++) {
                    const int v = lr_S(s, x + dx, y + dy);
                    sum += v; sumsq += v * v;
                }
            const int a = (sumsq + ((1 << (2 * b8)) >> 1)) >> (2 * b8);
            const int b = (sum + ((1 << b8) >> 1)) >> b8;
            const unsigned p = (unsigned)o_max(a * n - b * b, 0);
            const unsigned z = (p * strength + (1 << 19)) >> 20;
            const unsigned xx = b200_sgr_x_by_x[z < 255 ? z : 255];
            lr_counts[lr_cls][LR_Z0] += z == 0;
            lr_counts[lr_cls][LR_Z255] += z >= 255;
            lr_counts[lr_cls][LR_SGR_BIG] += xx * (unsigned)sum * (unsigned)one_by_x >= 0x80000000u;   /* past the int32 range */
            A[(y + 1) * (w + 2) + x + 1] = (int32_t)((xx * (unsigned)sum * (unsigned)one_by_x + (1 << 11)) >> 12);
            B[(y + 1) * (w + 2) + x + 1] = (int32_t)xx;
        }
}

/* mode 0: 5x5, 1: 3x3, 2: mix  (index of c->sgr[]); s0/s1/w0/w1 as in LooprestorationParams.sgr */
ORACLE_API void oracle_sgr(int mode, void *p, ptrdiff_t stride_bytes, const void *left, const void *lpf, int w, int h,
                           unsigned s0, unsigned s1, int w0, int w1, int edges, int bdmax)
{
    const int hbd = bdmax > 255;
    LrSrc s = { p, left, lpf, hbd ? stride_bytes / 2 : stride_bytes, w, h, edges, hbd, 0 };
    if (mode == 1) s.use_bottom = (edges & 8) && h > 2;
    else s.use_bottom = (edges & 8) && !(h & 1) && h > ((edges & 4) ? 2 : 4);
    const size_t n = (size_t)(w + 2) * (h + 2);
    int32_t *A5 = malloc(4 * n), *B5 = malloc(4 * n), *A3 = malloc(4 * n), *B3 = malloc(4 * n);
    if (mode != 1) sgr_ab(&s, 2, s0, bdmax, A5, B5);
    if (mode != 0) sgr_ab(&s, 1, s1, bdmax, A3, B3);
    uint8_t *out = malloc((size_t)w * h * 2);
#define AT(P, x, y) P[((y) + 1) * (w + 2) + (x) + 1]
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int src = lr_S(&s, x, y);
            int t5 = 0, t3 = 0;
            if (mode != 1) {
                if (!(y & 1)) {
                    const int a = (AT(B5, x, y - 1) + AT(B5, x, y + 1)) * 6 +
                                  (AT(B5, x - 1, y - 1) + AT(B5, x - 1, y + 1) + AT(B5, x + 1, y - 1) + AT(B5, x + 1, y + 1)) * 5;
                    const int b = (AT(A5, x, y - 1) + AT(A5, x, y + 1)) * 6 +
                                  (AT(A5, x - 1, y - 1) + AT(A5, x - 1, y + 1) + AT(A5, x + 1, y - 1) + AT(A5, x + 1, y + 1)) * 5;
                    t5 = (b - a * src + (1 << 8)) >> 9;
                } else {
                    const int a = AT(B5, x, y) * 6 + (AT(B5, x - 1, y) + AT(B5, x + 1, y)) * 5;
                    const int b = AT(A5, x, y) * 6 + (AT(A5, x - 1, y) + AT(A5, x + 1, y)) * 5;
                    t5 = (b - a * src + (1 << 7)) >> 8;
                }
            }
            if (mode != 0) {
#define EIGHT(P) ((AT(P, x, y) + AT(P, x - 1, y) + AT(P, x + 1, y) + AT(P, x, y - 1) + AT(P, x, y + 1)) * 4 + \
                  (AT(P, x - 1, y - 1) + AT(P, x - 1, y + 1) + AT(P, x + 1, y - 1) + AT(P, x + 1, y + 1)) * 3)
                const int a = EIGHT(B3), b = EIGHT(A3);
                t3 = (b - a * src + (1 << 8)) >> 9;
            }
            const int v = mode == 0 ? w0 * t5 : mode == 1 ? w1 * t3 : w0 * t5 + w1 * t3;
            const int o = src + ((v + (1 << 10)) >> 11);
            lr_counts[lr_cls][LR_OUT_CLIP_LO] += o < 0;
            lr_counts[lr_cls][LR_OUT_CLIP_HI] += o > bdmax;
            st_px(out, hbd, (ptrdiff_t)y * w + x, o_clip(o, 0, bdmax));
        }
    for (int y = 0; y < h; y++)
        memcpy((uint8_t *)p + (ptrdiff_t)y * stride_bytes, out + (size_t)y * w * (hbd ? 2 : 1), (size_t)w * (hbd ? 2 : 1));
    free(out); free(A5); free(B5); free(A3); free(B3);
}

/* ---- whole frame, out of place -----------------------------------------------------------
 * cdef  : picture after CDEF (source of every row inside a stripe)
 * dbl   : picture after deblocking, before CDEF (source of the 2 rows above / below each 64-row
 *         stripe boundary: what dav1d_copy_lpf saves into lr_lpf_line, src/lf_apply_tmpl.c:40-101)
 * dst   : restored picture; units with type NONE are copied through.
 * Unit lookup follows lr_sbrow (reference src/lr_apply_tmpl.c:107-166). */
typedef struct { uint8_t type; int8_t filter_h[3], filter_v[3], sgr_weights[2]; } OracleLrUnit;   /* Av1RestorationUnit */
typedef struct { OracleLrUnit lr[3][4]; } OracleAv1Restoration;                                  /* Av1Restoration */
typedef struct {           /* restates B200LrFrame (include/b200av1.h) */
    const void *cdef, *dbl; void *dst;
    uint32_t plane_off[3]; int32_t stride[3];
    int32_t w, h;              /* picture size in luma pixels */
    int32_t ss_hor, ss_ver, sb128, sr_sb128w;
    int32_t unit_size_log2[2]; /* frame_hdr->restoration.unit_size[y, uv] */
    int32_t restore_planes;    /* bit p set: plane p has a frame-level restoration type */
    const OracleAv1Restoration *lr_mask;
} OracleLrFrame;

ORACLE_API void oracle_lr_frame(int bdmax, const OracleLrFrame *f)
{
    const int hbd = bdmax > 255; const size_t px = hbd ? 2 : 1;
    for (int pl = 0; pl < 3; pl++) {
        const int ssh = pl ? f->ss_hor : 0, ssv = pl ? f->ss_ver : 0;
        const int w = (f->w + ssh) >> ssh, h = (f->h + ssv) >> ssv;
        const ptrdiff_t st = f->stride[pl], sb = st * (ptrdiff_t)px;
        const uint8_t *C = (const uint8_t *)f->cdef + (size_t)f->plane_off[pl] * px;
        const uint8_t *D = (const uint8_t *)f->dbl + (size_t)f->plane_off[pl] * px;
        uint8_t *O = (uint8_t *)f->dst + (size_t)f->plane_off[pl] * px;
        for (int y = 0; y < h; y++) memcpy(O + y * sb, C + y * sb, (size_t)w * px);
        if (!(f->restore_planes & (1 << pl))) continue;
        const int us_log2 = f->unit_size_log2[!!pl], unit = 1 << us_log2, half = unit >> 1, max_unit = unit + half;
        const int shift_hor = 7 - ssh;
        long *const cnt = lr_counts[lr_cls = !!pl];
        uint8_t *lpf = malloc((size_t)8 * sb), *left = malloc(64 * 4 * px), *work = malloc((size_t)64 * sb);
        for (int y0 = 0, k = 0; y0 < h; k++) {
            const int y1 = o_min(h, ((64 * (k + 1) - 8) >> ssv));
            const int sh_ = y1 - y0;
            /* superblock row this stripe belongs to and its restoration-unit row */
            const int sby = ((y0 << ssv) + (y0 ? 8 : 0)) >> (6 + f->sb128);
            const int row_y = (sby << (6 + f->sb128)) >> ssv;
            int aligned = row_y & ~(unit - 1);
            if (aligned && aligned + half > h) { aligned -= unit; cnt[LR_PULLED_UP]++; }
            aligned <<= ssv;
            const int sb_idx = (aligned >> 7) * f->sr_sb128w, unit_idx = ((aligned >> 6) & 1) << 1;
            int edges = (y0 > 0 ? 4 : 0) | (y1 < h ? 8 : 0);
            cnt[y0 > 0 ? LR_TOP : LR_NO_TOP]++;
            cnt[y1 < h ? LR_BOT : LR_NO_BOT]++;
            cnt[LR_BOT_CLAMP] += y1 < h && y1 + 1 > h - 1;
            /* rows above / below the stripe from the deblocked picture (8-row lpf layout: 0,1 above, 6,7 below) */
            for (int i = 0; i < 2; i++) {
                memcpy(lpf + i * sb, D + (ptrdiff_t)o_max(y0 - 2 + i, 0) * sb, (size_t)sb);
                memcpy(lpf + (6 + i) * sb, D + (ptrdiff_t)o_min(y1 + i, h - 1) * sb, (size_t)sb);
            }
            for (int x = 0; x < w;) {
                const int last = !(x + max_unit <= w);
                const int uw = last ? w - x : unit;
                const OracleLrUnit *u = &f->lr_mask[sb_idx + (x >> shift_hor)].lr[pl][unit_idx + ((x >> (shift_hor - 1)) & 1)];
                const int s0 = u->type >= 3 && b200_sgr_params[u->type - 3][0], s1 = u->type >= 3 && b200_sgr_params[u->type - 3][1];
                cnt[!u->type ? LR_NONE : u->type == 2 ? LR_WIENER : s0 && s1 ? LR_SGR_MIX : s0 ? LR_SGR5 : LR_SGR3]++;
                cnt[LR_EXT_H] += uw > unit;
                if (u->type) {
                    const int e = edges | (x > 0 ? 1 : 0) | (last ? 0 : 2);
                    /* working copy of the stripe rows of this unit plus its right neighbourhood, pre-LR */
                    for (int y = 0; y < sh_; y++) {
                        memcpy(work + y * sb, C + (ptrdiff_t)(y0 + y) * sb, (size_t)sb);
                        if (x > 0) memcpy(left + (size_t)y * 4 * px, C + (ptrdiff_t)(y0 + y) * sb + (size_t)(x - 4) * px, 4 * px);
                    }
                    if (u->type == 2) {
                        int16_t filt[2][8];
                        for (int i = 0; i < 3; i++) {
                            filt[0][i] = filt[0][6 - i] = u->filter_h[i];
                            filt[1][i] = filt[1][6 - i] = u->filter_v[i];
                        }
                        filt[0][3] = (int16_t)(-(filt[0][0] + filt[0][1] + filt[0][2]) * 2 + (hbd ? 128 : 0));
                        filt[1][3] = (int16_t)(128 - (filt[1][0] + filt[1][1] + filt[1][2]) * 2);
                        filt[0][7] = filt[1][7] = 0;
                        oracle_wiener(work + (size_t)x * px, sb, x > 0 ? left : NULL, lpf + (size_t)x * px, uw, sh_, filt, e, bdmax);
                    } else {
                        const int idx = u->type - 3;
                        const unsigned s0 = b200_sgr_params[idx][0], s1 = b200_sgr_params[idx][1];
                        const int w0 = u->sgr_weights[0], w1 = 128 - (u->sgr_weights[0] + u->sgr_weights[1]);
                        oracle_sgr(!!s0 + !!s1 * 2 - 1, work + (size_t)x * px, sb, x > 0 ? left : NULL, lpf + (size_t)x * px,
                                   uw, sh_, s0, s1, w0, w1, e, bdmax);
                    }
                    for (int y = 0; y < sh_; y++)
                        memcpy(O + (ptrdiff_t)(y0 + y) * sb + (size_t)x * px, work + y * sb + (size_t)x * px, (size_t)uw * px);
                }
                x += uw;
            }
            y0 = y1;
        }
        free(lpf); free(left); free(work);
    }
    lr_cls = 0;
}
