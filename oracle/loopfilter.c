/*
 * oracle/loopfilter.c — TEST INFRASTRUCTURE (see oracle_common.h).
 *
 * Plain-C restatement of dav1d's deblocking filter:
 *   loop_filter (one 4-line edge segment)      reference src/loopfilter_tmpl.c:37-161
 *   loop_filter_{h,v}_sb128{y,uv}              reference src/loopfilter_tmpl.c:163-245
 *   frame driver: mask assembly + plane loops  reference src/lf_apply_tmpl.c:176-311, 403-466
 * The frame driver walks superblock rows in the reference's order (all column edges of an
 * sbrow, then its row edges), which is what the frame-wide two-pass CUDA sweep must equal.
 */
#include "oracle_common.h"

static inline int PX(const void *p, int hbd, ptrdiff_t i) {
    return hbd ? ((const uint16_t *)p)[i] : ((const uint8_t *)p)[i];
}
static inline void SPX(void *p, int hbd, ptrdiff_t i, int v) {
    if (hbd) ((uint16_t *)p)[i] = (uint16_t)v; else ((uint8_t *)p)[i] = (uint8_t)v;
}

/* Branch counters for the tests (oracle_lf_branch_counts): per plane class (0 luma, 1 chroma) and direction
 * (0 column edges, 1 row edges), the number of edge lines that took each branch of lf_segment. They only observe. */
enum { LF_FM_FAIL, LF_NARROW_HEV, LF_NARROW, LF_FLAT6, LF_FLAT8, LF_FLAT8_OF16, LF_FLAT16, LF_NARROW_CLIP, LF_N_BRANCHES };
static long lf_counts[2][2][LF_N_BRANCHES];

/* copies the counters to out[2][2][LF_N_BRANCHES] (plane class, direction, branch) and resets them; returns the branch count */
ORACLE_API int oracle_lf_branch_counts(long *out)
{
    if (out) memcpy(out, lf_counts, sizeof(lf_counts));
    memset(lf_counts, 0, sizeof(lf_counts));
    return LF_N_BRANCHES;
}

/* dst: pixel index base; sa = step between the 4 lines, sb = step across the edge (pixels) */
static void lf_segment(void *pic, ptrdiff_t base, int E, int I, int H, ptrdiff_t sa, ptrdiff_t sb,
                       int wd, int bdmax, long *cnt)
{
    const int hbd = bdmax > 255;
    const int b8 = (o_ulog2((unsigned)bdmax) + 1) - 8;
    const int F = 1 << b8;
    E <<= b8; I <<= b8; H <<= b8;
    for (int i = 0; i < 4; i++, base += sa) {
        int p[7], q[7];   /* p[k] = sample k+1 before the edge, q[k] = sample k after it */
        for (int k = 0; k < 7; k++) { p[k] = 0; q[k] = 0; }
        const int np = wd >= 16 ? 7 : wd >= 8 ? 4 : wd == 6 ? 3 : 2;
        for (int k = 0; k < np; k++) {
            p[k] = PX(pic, hbd, base - (k + 1) * sb);
            q[k] = PX(pic, hbd, base + k * sb);
        }
        int fm = o_abs(p[1] - p[0]) <= I && o_abs(q[1] - q[0]) <= I &&
                 o_abs(p[0] - q[0]) * 2 + (o_abs(p[1] - q[1]) >> 1) <= E;
        if (wd > 4) fm &= o_abs(p[2] - p[1]) <= I && o_abs(q[2] - q[1]) <= I;
        if (wd > 6) fm &= o_abs(p[3] - p[2]) <= I && o_abs(q[3] - q[2]) <= I;
        if (!fm) { cnt[LF_FM_FAIL]++; continue; }

        int flat8out = 0, flat8in = 0;
        if (wd >= 16)
            flat8out = o_abs(p[6] - p[0]) <= F && o_abs(p[5] - p[0]) <= F && o_abs(p[4] - p[0]) <= F &&
                       o_abs(q[4] - q[0]) <= F && o_abs(q[5] - q[0]) <= F && o_abs(q[6] - q[0]) <= F;
        if (wd >= 6)
            flat8in = o_abs(p[2] - p[0]) <= F && o_abs(p[1] - p[0]) <= F &&
                      o_abs(q[1] - q[0]) <= F && o_abs(q[2] - q[0]) <= F;
        if (wd >= 8)
            flat8in &= o_abs(p[3] - p[0]) <= F && o_abs(q[3] - q[0]) <= F;

        if (wd >= 16 && (flat8out & flat8in)) {
            cnt[LF_FLAT16]++;
            /* 13-tap smoothing: out(k) = (sum of a 13-wide window with replicated ends + 8) >> 4 */
            int s[14];   /* s[0..6] = p6..p0, s[7..13] = q0..q6 */
            for (int k = 0; k < 7; k++) { s[k] = p[6 - k]; s[7 + k] = q[k]; }
            for (int o = 1; o <= 12; o++) {            /* output position o: p5 (o=1) .. q5 (o=12) */
                int sum = 8;
                for (int t = -6; t <= 6; t++) {
                    int idx = o + t;
                    if (idx < 0) idx = 0; else if (idx > 13) idx = 13;
                    /* centre-weighted window: taps at -1, 0, +1 ... the reference's sums weight the
                     * centre sample and its two neighbours twice */
                    sum += s[idx];
                }
                /* the reference window has 16 terms: the 13 above plus s[o-1], s[o], s[o+1] once more */
                sum += s[o - 1 < 0 ? 0 : o - 1] + s[o] + s[o + 1 > 13 ? 13 : o + 1];
                const ptrdiff_t pos = o < 7 ? base - (7 - o) * sb : base + (o - 7) * sb;
                SPX(pic, hbd, pos, sum >> 4);
            }
        } else if (wd >= 8 && flat8in) {
            cnt[wd == 8 ? LF_FLAT8 : LF_FLAT8_OF16]++;
            const int p3 = p[3], p2 = p[2], p1 = p[1], p0 = p[0], q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
            SPX(pic, hbd, base - 3 * sb, (p3 + p3 + p3 + 2 * p2 + p1 + p0 + q0 + 4) >> 3);
            SPX(pic, hbd, base - 2 * sb, (p3 + p3 + p2 + 2 * p1 + p0 + q0 + q1 + 4) >> 3);
            SPX(pic, hbd, base - 1 * sb, (p3 + p2 + p1 + 2 * p0 + q0 + q1 + q2 + 4) >> 3);
            SPX(pic, hbd, base + 0 * sb, (p2 + p1 + p0 + 2 * q0 + q1 + q2 + q3 + 4) >> 3);
            SPX(pic, hbd, base + 1 * sb, (p1 + p0 + q0 + 2 * q1 + q2 + q3 + q3 + 4) >> 3);
            SPX(pic, hbd, base + 2 * sb, (p0 + q0 + q1 + 2 * q2 + q3 + q3 + q3 + 4) >> 3);
        } else if (wd == 6 && flat8in) {
            cnt[LF_FLAT6]++;
            const int p2 = p[2], p1 = p[1], p0 = p[0], q0 = q[0], q1 = q[1], q2 = q[2];
            SPX(pic, hbd, base - 2 * sb, (p2 + 2 * p2 + 2 * p1 + 2 * p0 + q0 + 4) >> 3);
            SPX(pic, hbd, base - 1 * sb, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
            SPX(pic, hbd, base + 0 * sb, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
            SPX(pic, hbd, base + 1 * sb, (p0 + 2 * q0 + 2 * q1 + 2 * q2 + q2 + 4) >> 3);
        } else {
            const int lo = -128 * (1 << b8), hi = 128 * (1 << b8) - 1;
            const int hev = o_abs(p[1] - p[0]) > H || o_abs(q[1] - q[0]) > H;
            int f = hev ? o_clip(p[1] - q[1], lo, hi) : 0;
            f = o_clip(3 * (q[0] - p[0]) + f, lo, hi);
            const int f1 = o_min(f + 4, hi) >> 3, f2 = o_min(f + 3, hi) >> 3;
            SPX(pic, hbd, base - sb, o_clip(p[0] + f2, 0, bdmax));
            SPX(pic, hbd, base, o_clip(q[0] - f1, 0, bdmax));
            int clipped = p[0] + f2 < 0 || p[0] + f2 > bdmax || q[0] - f1 < 0 || q[0] - f1 > bdmax;
            if (!hev) {
                const int g = (f1 + 1) >> 1;
                SPX(pic, hbd, base - 2 * sb, o_clip(p[1] + g, 0, bdmax));
                SPX(pic, hbd, base + sb, o_clip(q[1] - g, 0, bdmax));
                clipped |= p[1] + g < 0 || p[1] + g > bdmax || q[1] - g < 0 || q[1] - g > bdmax;
            }
            cnt[hev ? LF_NARROW_HEV : LF_NARROW]++;
            cnt[LF_NARROW_CLIP] += clipped;
        }
    }
}

typedef struct { uint8_t e[64], i[64]; uint64_t sharp[2]; } OracleFilterLUT;   /* Av1FilterLUT */

/* c->loop_filter_sb[plane_class][dir]: plane_class 0 luma / 1 chroma, dir 0 = column edges ("h"),
 * 1 = row edges ("v"). dst points at the first pixel after the edge of segment 0. */
ORACLE_API void oracle_loop_filter_sb(int plane_class, int dir, void *dst, ptrdiff_t stride_bytes,
                                      const uint32_t *mask, const uint8_t (*l)[4], ptrdiff_t b4_stride,
                                      const OracleFilterLUT *lut, int bdmax)
{
    const int hbd = bdmax > 255;
    const ptrdiff_t ps = hbd ? stride_bytes / 2 : stride_bytes;
    const unsigned vm = mask[0] | mask[1] | (plane_class ? 0 : mask[2]);
    ptrdiff_t base = 0;
    for (unsigned bit = 1; vm & ~(bit - 1); bit <<= 1, base += dir ? 4 : 4 * ps, l += dir ? 1 : b4_stride) {
        if (!(vm & bit)) continue;
        const int L = l[0][0] ? l[0][0] : (dir ? l[-b4_stride][0] : l[-1][0]);
        if (!L) continue;
        int wd;
        if (plane_class) wd = 4 + 2 * !!(mask[1] & bit);
        else wd = 4 << ((mask[2] & bit) ? 2 : !!(mask[1] & bit));
        long *const cnt = lf_counts[!!plane_class][!!dir];
        if (dir) lf_segment(dst, base, lut->e[L], lut->i[L], L >> 4, 1, ps, wd, bdmax, cnt);
        else     lf_segment(dst, base, lut->e[L], lut->i[L], L >> 4, ps, 1, wd, bdmax, cnt);
    }
}

/* ---- whole frame, reference order ------------------------------------------------------- */
typedef struct {           /* layout of dav1d's Av1Filter, reference src/lf_mask.h:51-57 */
    uint16_t filter_y[2][32][3][2];
    uint16_t filter_uv[2][32][2][2];
    int8_t cdef_idx[4];
    uint16_t noskip_mask[16][2];
} OracleAv1Filter;

typedef struct {           /* restates B200LfFrame (include/b200av1.h) */
    void *pic;
    uint32_t plane_off[3];
    int32_t stride[3];     /* pixels */
    int32_t w4, h4;        /* picture size in luma 4-px units (f->w4, f->h4) */
    int32_t sb128w;
    int32_t b4_stride;
    int32_t ss_hor, ss_ver;
    int32_t sb128;         /* sequence uses 128x128 superblocks (only changes the walk order) */
    int32_t filter_y, filter_uv;   /* frame-level enables (level_y[0]|level_y[1]; level_u|level_v) */
    const OracleAv1Filter *mask;
    const uint8_t (*level)[4];
    OracleFilterLUT lut;
} OracleLfFrame;

ORACLE_API void oracle_lf_frame(int bdmax, const OracleLfFrame *f)
{
    const int hbd = bdmax > 255;
    const size_t px = hbd ? 2 : 1;
    const int is_sb64 = !f->sb128, sbsz = 32 >> is_sb64;
    const int sbh = (f->h4 + sbsz - 1) / sbsz;
    const int ss_hor = f->ss_hor, ss_ver = f->ss_ver;
    uint8_t *const pl[3] = { (uint8_t *)f->pic + f->plane_off[0] * px, (uint8_t *)f->pic + f->plane_off[1] * px,
                             (uint8_t *)f->pic + f->plane_off[2] * px };
    if (!f->filter_y) return;
    for (int sby = 0; sby < sbh; sby++) {
        const int starty4 = (sby & is_sb64) << 4;
        const int endy4 = starty4 + o_min(f->h4 - sby * sbsz, sbsz);
        const int uv_endy4 = (endy4 + ss_ver) >> ss_ver;
        const OracleAv1Filter *lflvl = f->mask + (sby >> is_sb64) * f->sb128w;
        uint8_t *py = pl[0] + (size_t)sby * sbsz * 4 * f->stride[0] * px;
        uint8_t *pu = pl[1] + (size_t)(sby * sbsz * 4 >> ss_ver) * f->stride[1] * px;
        uint8_t *pv = pl[2] + (size_t)(sby * sbsz * 4 >> ss_ver) * f->stride[2] * px;
        for (int pass = 0; pass < 2; pass++) {          /* 0: column edges, 1: row edges */
            /* ---- luma ---- */
            const uint8_t (*lvl)[4] = f->level + (ptrdiff_t)f->b4_stride * sby * sbsz;
            for (int x = 0; x < f->sb128w; x++, lvl += 32) {
                const int w = o_min(32, f->w4 - x * 32);
                uint8_t *d = py + (size_t)x * 128 * px;
                if (!pass) {
                    for (int xi = 0; xi < w; xi++) {
                        if (!x && !xi) continue;
                        uint32_t m[3];
                        for (int k = 0; k < 3; k++) {
                            const uint16_t *h = lflvl[x].filter_y[0][xi][k];
                            m[k] = !starty4 ? (h[0] | (endy4 > 16 ? (uint32_t)h[1] << 16 : 0)) : h[1];
                        }
                        oracle_loop_filter_sb(0, 0, d + (size_t)xi * 4 * px, f->stride[0] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lvl[xi][0], f->b4_stride, &f->lut, bdmax);
                    }
                } else {
                    const uint8_t (*lr)[4] = lvl;
                    uint8_t *dr = d;
                    for (int y = starty4; y < endy4; y++, dr += (size_t)4 * f->stride[0] * px, lr += f->b4_stride) {
                        if (!sby && !y) continue;
                        uint32_t m[3];
                        for (int k = 0; k < 3; k++) {
                            const uint16_t *h = lflvl[x].filter_y[1][y][k];
                            m[k] = h[0] | ((uint32_t)h[1] << 16);
                        }
                        oracle_loop_filter_sb(0, 1, dr, f->stride[0] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lr[0][1], f->b4_stride, &f->lut, bdmax);
                    }
                }
            }
            if (!f->filter_uv) continue;
            /* ---- chroma ---- */
            lvl = f->level + (ptrdiff_t)f->b4_stride * (sby * sbsz >> ss_ver);
            for (int x = 0; x < f->sb128w; x++, lvl += 32 >> ss_hor) {
                const int w = (o_min(32, f->w4 - x * 32) + ss_hor) >> ss_hor;
                const size_t uv_off = (size_t)x * (128 >> ss_hor) * px;
                if (!pass) {
                    for (int xi = 0; xi < w; xi++) {
                        if (!x && !xi) continue;
                        uint32_t m[2];
                        for (int k = 0; k < 2; k++) {
                            const uint16_t *h = lflvl[x].filter_uv[0][xi][k];
                            if (!starty4) m[k] = h[0] | (uv_endy4 > (16 >> ss_ver) ? (uint32_t)h[1] << (16 >> ss_ver) : 0);
                            else m[k] = h[1];
                        }
                        oracle_loop_filter_sb(1, 0, pu + uv_off + (size_t)xi * 4 * px, f->stride[1] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lvl[xi][2], f->b4_stride, &f->lut, bdmax);
                        oracle_loop_filter_sb(1, 0, pv + uv_off + (size_t)xi * 4 * px, f->stride[2] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lvl[xi][3], f->b4_stride, &f->lut, bdmax);
                    }
                } else {
                    const uint8_t (*lr)[4] = lvl;
                    size_t off = 0;
                    for (int y = starty4 >> ss_ver; y < uv_endy4; y++, off += (size_t)4 * f->stride[1] * px, lr += f->b4_stride) {
                        if (!sby && !y) continue;
                        uint32_t m[2];
                        for (int k = 0; k < 2; k++) {
                            const uint16_t *h = lflvl[x].filter_uv[1][y][k];
                            m[k] = h[0] | ((uint32_t)h[1] << (16 >> ss_hor));
                        }
                        oracle_loop_filter_sb(1, 1, pu + uv_off + off, f->stride[1] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lr[0][2], f->b4_stride, &f->lut, bdmax);
                        oracle_loop_filter_sb(1, 1, pv + uv_off + off, f->stride[2] * (ptrdiff_t)px, m,
                                              (const uint8_t (*)[4])&lr[0][3], f->b4_stride, &f->lut, bdmax);
                    }
                }
            }
        }
    }
}
