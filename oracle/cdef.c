/*
 * oracle/cdef.c — TEST INFRASTRUCTURE (see oracle_common.h).
 *
 * Plain-C restatement of dav1d's constrained directional enhancement filter:
 *   cdef_find_dir_c                    reference src/cdef_tmpl.c:239-305
 *   cdef_filter_block_c + padding      reference src/cdef_tmpl.c:37-216
 *   frame driver dav1d_cdef_brow       reference src/cdef_apply_tmpl.c:91-308
 * The frame function is written OUT OF PLACE (src picture -> dst picture): CDEF reads only
 * pre-CDEF samples (the reference keeps line/column backups to achieve that in place), so the
 * result is the same picture dav1d produces.
 */
#include "oracle_common.h"

static inline int PX(const void *p, int hbd, ptrdiff_t i) {
    return hbd ? ((const uint16_t *)p)[i] : ((const uint8_t *)p)[i];
}
static inline void SPX(void *p, int hbd, ptrdiff_t i, int v) {
    if (hbd) ((uint16_t *)p)[i] = (uint16_t)v; else ((uint8_t *)p)[i] = (uint8_t)v;
}

/* taps of direction d, k = 0 (near) / 1 (far): (dy, dx); reference src/tables.c:400-413 */
static const int8_t cdef_dir_off[8][2][2] = {
    { { -1, 1 }, { -2, 2 } }, { { 0, 1 }, { -1, 2 } }, { { 0, 1 }, { 0, 2 } }, { { 0, 1 }, { 1, 2 } },
    { { 1, 1 }, { 2, 2 } },   { { 1, 0 }, { 2, 1 } },  { { 1, 0 }, { 2, 0 } }, { { 1, 0 }, { 2, -1 } },
};

/* Branch counters for the tests (oracle_cdef_counts): per plane class (0 luma, 1 chroma), 8x8 blocks (4x4 / 4x8 in
 * subsampled chroma) of oracle_cdef_frame by the way they were filtered, plus pixels and taps. They only observe. */
enum { CD_SKIP_IDX, CD_SKIP_NOSKIP, CD_SKIP_ZERO, CD_PRI_SEC, CD_PRI, CD_SEC, CD_ADJ_ZERO, CD_ADJ_FULL, CD_SHIFT_CLAMP,
       CD_DIR0, CD_EDGE_L = CD_DIR0 + 8, CD_EDGE_R, CD_EDGE_T, CD_EDGE_B, CD_CLAMP_PX, CD_TAP_DROPPED, CD_N };
static long cd_counts[2][CD_N];

/* copies the counters to out[2][CD_N] (plane class, counter) and resets them; returns CD_N */
ORACLE_API int oracle_cdef_counts(long *out)
{
    if (out) memcpy(out, cd_counts, sizeof(cd_counts));
    memset(cd_counts, 0, sizeof(cd_counts));
    return CD_N;
}

static inline int constrain(int diff, int threshold, int shift) {
    const int adiff = o_abs(diff);
    const int v = o_min(adiff, o_max(0, threshold - (adiff >> shift)));
    return diff < 0 ? -v : v;
}

ORACLE_API int oracle_cdef_dir(const void *img, ptrdiff_t stride_bytes, unsigned *var, int bdmax)
{
    const int hbd = bdmax > 255;
    const ptrdiff_t ps = hbd ? stride_bytes / 2 : stride_bytes;
    const int b8 = (o_ulog2((unsigned)bdmax) + 1) - 8;
    int hv[2][8] = { { 0 } }, diag[2][15] = { { 0 } }, alt[4][11] = { { 0 } };
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) {
            const int px = (PX(img, hbd, y * ps + x) >> b8) - 128;
            diag[0][y + x] += px;          alt[0][y + (x >> 1)] += px;
            hv[0][y] += px;                alt[1][3 + y - (x >> 1)] += px;
            diag[1][7 + y - x] += px;      alt[2][3 - (y >> 1) + x] += px;
            hv[1][x] += px;                alt[3][(y >> 1) + x] += px;
        }
    unsigned cost[8] = { 0 };
    for (int n = 0; n < 8; n++) {
        cost[2] += hv[0][n] * hv[0][n];
        cost[6] += hv[1][n] * hv[1][n];
    }
    cost[2] *= 105; cost[6] *= 105;
    static const uint16_t div_table[7] = { 840, 420, 280, 210, 168, 140, 120 };
    for (int n = 0; n < 7; n++) {
        const int d = div_table[n];
        cost[0] += (diag[0][n] * diag[0][n] + diag[0][14 - n] * diag[0][14 - n]) * d;
        cost[4] += (diag[1][n] * diag[1][n] + diag[1][14 - n] * diag[1][14 - n]) * d;
    }
    cost[0] += diag[0][7] * diag[0][7] * 105;
    cost[4] += diag[1][7] * diag[1][7] * 105;
    for (int n = 0; n < 4; n++) {
        unsigned *c = &cost[n * 2 + 1];
        for (int m = 0; m < 5; m++) *c += alt[n][3 + m] * alt[n][3 + m];
        *c *= 105;
        for (int m = 0; m < 3; m++) {
            const int d = div_table[2 * m + 1];
            *c += (alt[n][m] * alt[n][m] + alt[n][10 - m] * alt[n][10 - m]) * d;
        }
    }
    int best = 0; unsigned bc = cost[0];
    for (int n = 1; n < 8; n++) if (cost[n] > bc) { bc = cost[n]; best = n; }
    *var = (bc - cost[best ^ 4]) >> 10;
    return best;
}

/* filter one w x h block. `get(ctx, x, y, &v)` returns 0 when sample (x, y) (block-relative,
 * -2 .. w+1 / h+1) is unavailable, else 1 with the PRE-CDEF value in v. */
typedef int (*sample_fn)(const void *ctx, int x, int y, int *v);

static void cdef_block(void *dst, ptrdiff_t ps, int hbd, sample_fn get, const void *ctx, int pri, int sec,
                       int dir, int damping, int w, int h, int bdmax, long *cnt)
{
    static long unused[CD_N];
    if (!cnt) cnt = unused;
    const int b8 = (o_ulog2((unsigned)bdmax) + 1) - 8;
    const int pri_tap0 = 4 - ((pri >> b8) & 1);
    const int pri_shift = pri ? o_max(0, damping - o_ulog2((unsigned)pri)) : 0;
    const int sec_shift = sec ? damping - o_ulog2((unsigned)sec) : 0;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int px; get(ctx, x, y, &px);
            int sum = 0, mx = px, mn = px;
            for (int k = 0; k < 2; k++) {
                if (pri) {
                    const int tap = k ? ((pri_tap0 & 3) | 2) : pri_tap0;
                    for (int s = -1; s <= 1; s += 2) {
                        int p;
                        if (!get(ctx, x + s * cdef_dir_off[dir][k][1], y + s * cdef_dir_off[dir][k][0], &p)) continue;
                        const int c = constrain(p - px, pri, pri_shift);
                        cnt[CD_TAP_DROPPED] += p != px && !c;
                        sum += tap * c;
                        mn = o_min(mn, p); mx = o_max(mx, p);
                    }
                }
                if (sec) {
                    const int tap = 2 - k;
                    for (int j = 0; j < 2; j++) {
                        const int d2 = (dir + (j ? 6 : 2)) & 7;       /* dir + 2, dir - 2 */
                        for (int s = -1; s <= 1; s += 2) {
                            int p;
                            if (!get(ctx, x + s * cdef_dir_off[d2][k][1], y + s * cdef_dir_off[d2][k][0], &p)) continue;
                            const int c = constrain(p - px, sec, sec_shift);
                            cnt[CD_TAP_DROPPED] += p != px && !c;
                            sum += tap * c;
                            mn = o_min(mn, p); mx = o_max(mx, p);
                        }
                    }
                }
            }
            int v = px + ((sum - (sum < 0) + 8) >> 4);
            if (pri && sec) {                          /* only the combined filter clamps (:165) */
                cnt[CD_CLAMP_PX] += v < mn || v > mx;
                v = o_clip(v, mn, mx);
            }
            SPX(dst, hbd, y * ps + x, v);
        }
}

/* ---- Level-1 form: dst / left / top / bottom + edge flags, like decl_cdef_fn ---- */
typedef struct { const void *dst, *left, *top, *bottom; ptrdiff_t ps; int w, h, edges, hbd; uint8_t copy[8 * 8 * 2]; } L1Ctx;
static int l1_get(const void *c_, int x, int y, int *v) {
    const L1Ctx *c = c_;
    if ((x < 0 && !(c->edges & 1)) || (x >= c->w && !(c->edges & 2)) ||
        (y < 0 && !(c->edges & 4)) || (y >= c->h && !(c->edges & 8))) return 0;
    if (y < 0) *v = PX(c->top, c->hbd, (y + 2) * c->ps + x);
    else if (y >= c->h) *v = PX(c->bottom, c->hbd, (y - c->h) * c->ps + x);
    else if (x < 0) *v = PX(c->left, c->hbd, y * 2 + (2 + x));
    else if (x < c->w) *v = PX(c->copy, c->hbd, y * c->w + x);      /* pre-filter copy of the block */
    else *v = PX(c->dst, c->hbd, y * c->ps + x);
    return 1;
}
ORACLE_API void oracle_cdef_fb(void *dst, ptrdiff_t stride_bytes, const void *left, const void *top,
                               const void *bottom, int pri, int sec, int dir, int damping, int w, int h,
                               int edges, int bdmax)
{
    L1Ctx c;
    c.hbd = bdmax > 255; c.ps = c.hbd ? stride_bytes / 2 : stride_bytes;
    c.dst = dst; c.left = left; c.top = top; c.bottom = bottom; c.w = w; c.h = h; c.edges = edges;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) SPX(c.copy, c.hbd, y * w + x, PX(dst, c.hbd, y * c.ps + x));
    cdef_block(dst, c.ps, c.hbd, l1_get, &c, pri, sec, dir, damping, w, h, bdmax, NULL);
}

/* ---- whole frame, out of place ---- */
typedef struct {           /* Av1Filter, reference src/lf_mask.h:51-57 */
    uint16_t filter_y[2][32][3][2]; uint16_t filter_uv[2][32][2][2]; int8_t cdef_idx[4]; uint16_t noskip_mask[16][2];
} OracleAv1Filter;
typedef struct {           /* restates B200CdefFrame (include/b200av1.h) */
    const void *src; void *dst;
    uint32_t plane_off[3]; int32_t stride[3];
    int32_t bw, bh;            /* f->bw, f->bh: frame size in 4-px units */
    int32_t sb128w, ss_hor, ss_ver;
    int32_t damping;           /* frame_hdr->cdef.damping */
    int32_t y_strength[8], uv_strength[8];
    const OracleAv1Filter *mask;
} OracleCdefFrame;

typedef struct { const uint8_t *base; ptrdiff_t ps; int hbd, x0, y0, xmin, xmax, ymin, ymax; } FrCtx;
static int fr_get(const void *c_, int x, int y, int *v) {
    const FrCtx *c = c_;
    const int ax = c->x0 + x, ay = c->y0 + y;
    if (ax < c->xmin || ax >= c->xmax || ay < c->ymin || ay >= c->ymax) return 0;
    *v = PX(c->base, c->hbd, ay * c->ps + ax);
    return 1;
}
static int adjust_strength(int strength, unsigned var) {
    if (!var) return 0;
    const int i = (var >> 6) ? o_min(o_ulog2(var >> 6), 12) : 0;
    return (strength * (4 + i) + 8) >> 4;
}

ORACLE_API void oracle_cdef_frame(int bdmax, const OracleCdefFrame *f)
{
    const int hbd = bdmax > 255; const size_t px = hbd ? 2 : 1;
    const int b8 = (o_ulog2((unsigned)bdmax) + 1) - 8;
    const int ss_hor = f->ss_hor, ss_ver = f->ss_ver;
    static const uint8_t uv_dirs[2][8] = { { 0, 1, 2, 3, 4, 5, 6, 7 }, { 7, 0, 2, 4, 5, 6, 6, 6 } };
    const uint8_t *uv_dir = uv_dirs[ss_hor && !ss_ver];
    const int damping = f->damping + b8;
    for (int by = 0; by < f->bh; by += 2)
        for (int bx = 0; bx < f->bw; bx += 2) {
            /* blocks that end up unfiltered pass through unchanged */
            for (int pl = 0; pl < 3; pl++) {
                const int sh = pl ? ss_hor : 0, sv = pl ? ss_ver : 0;
                for (int y = 0; y < (8 >> sv); y++) {
                    const size_t o = ((size_t)f->plane_off[pl] + (size_t)((by * 4 >> sv) + y) * f->stride[pl] + (bx * 4 >> sh)) * px;
                    memcpy((uint8_t *)f->dst + o, (const uint8_t *)f->src + o, (size_t)(8 >> sh) * px);
                }
            }
            const OracleAv1Filter *m = &f->mask[(by >> 5) * f->sb128w + (bx >> 5)];
            const int cdef_idx = m->cdef_idx[((by & 16) >> 3) + ((bx & 16) >> 4)];
            const uint16_t *nr = m->noskip_mask[(by & 30) >> 1];
            const unsigned noskip = (unsigned)nr[1] << 16 | nr[0];
            const int skip = cdef_idx == -1 ? CD_SKIP_IDX : !f->y_strength[cdef_idx] && !f->uv_strength[cdef_idx] ? CD_SKIP_ZERO :
                             !(noskip & (3U << (bx & 30))) ? CD_SKIP_NOSKIP : -1;
            if (skip >= 0) { cd_counts[0][skip]++; cd_counts[1][skip] += 2; continue; }
            const int y_lvl = f->y_strength[cdef_idx], uv_lvl = f->uv_strength[cdef_idx];
            const int y_pri = (y_lvl >> 2) << b8;
            int y_sec = y_lvl & 3; y_sec += y_sec == 3; y_sec <<= b8;
            const int uv_pri = (uv_lvl >> 2) << b8;
            int uv_sec = uv_lvl & 3; uv_sec += uv_sec == 3; uv_sec <<= b8;
            /* edges: src/cdef_apply_tmpl.c:101,125,142-143,171-173 */
            const int have_l = bx > 0, have_r = bx + 2 < f->bw, have_t = by > 0, have_b = by + 2 < f->bh;
            int dir = 0; unsigned var = 0;
            const uint8_t *ysrc = (const uint8_t *)f->src + (size_t)f->plane_off[0] * px;
            if (y_pri || uv_pri)
                dir = oracle_cdef_dir(ysrc + ((size_t)by * 4 * f->stride[0] + bx * 4) * px, f->stride[0] * (ptrdiff_t)px, &var, bdmax);
            for (int pl = 0; pl < 3; pl++) {
                const int sh = pl ? ss_hor : 0, sv = pl ? ss_ver : 0;
                const int w = 8 >> sh, h = 8 >> sv;
                int pri, sec, d, damp;
                long *const cnt = cd_counts[!!pl];
                if (!pl) {
                    if (y_pri) {
                        pri = adjust_strength(y_pri, var); sec = y_sec; d = dir;
                        cnt[CD_ADJ_ZERO] += !pri;
                        cnt[CD_ADJ_FULL] += pri == y_pri;
                        if (!pri && !sec) continue;
                    }
                    else if (y_sec) { pri = 0; sec = y_sec; d = 0; }
                    else continue;
                    damp = damping;
                } else {
                    if (!uv_lvl) continue;
                    pri = uv_pri; sec = uv_sec; d = uv_pri ? uv_dir[dir] : 0; damp = damping - 1;
                }
                cnt[pri && sec ? CD_PRI_SEC : pri ? CD_PRI : CD_SEC]++;
                if (pri) { cnt[CD_DIR0 + d]++; cnt[CD_SHIFT_CLAMP] += damp < o_ulog2((unsigned)pri); }
                cnt[CD_EDGE_L] += !have_l; cnt[CD_EDGE_R] += !have_r; cnt[CD_EDGE_T] += !have_t; cnt[CD_EDGE_B] += !have_b;
                FrCtx c;
                c.base = (const uint8_t *)f->src + (size_t)f->plane_off[pl] * px; c.ps = f->stride[pl]; c.hbd = hbd;
                c.x0 = bx * 4 >> sh; c.y0 = by * 4 >> sv;
                c.xmin = c.x0 - 2 * have_l; c.xmax = c.x0 + w + 2 * have_r;
                c.ymin = c.y0 - 2 * have_t; c.ymax = c.y0 + h + 2 * have_b;
                uint8_t *d8 = (uint8_t *)f->dst + ((size_t)f->plane_off[pl] + (size_t)c.y0 * f->stride[pl] + c.x0) * px;
                cdef_block(d8, f->stride[pl], hbd, fr_get, &c, pri, sec, d, damp, w, h, bdmax, cnt);
            }
        }
}
