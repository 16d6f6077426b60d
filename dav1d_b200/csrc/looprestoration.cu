// Loop restoration (dav1d Dav1dLoopRestorationDSPContext; reference src/looprestoration_tmpl.c,
// driver src/lr_apply_tmpl.c, stripe-border rows src/lf_apply_tmpl.c:40-174).
//
// Frame-wide and out of place. A CTA of 256 threads restores one tile (<= 64 x 32) that lies inside one 64-row stripe
// and one restoration unit, or, where a plane's units are 32 wide (4:2:0 / 4:2:2 chroma), the U and the V tile at the
// same place on 128 threads each:
//   1. the tile plus a 3-sample halo of the *virtual source* is staged in shared memory: rows inside
//      the stripe come from the post-CDEF picture, the two rows above / below the stripe from the
//      post-deblock picture (third row repeated), columns are clamped at the picture edges — the same
//      samples dav1d assembles from lr_lpf_line / pre_lr_border / edge replication;
//   2. Wiener: 7-tap rows into a shared uint16 tile, then 7-tap columns;
//      self-guided: 3x3 / 5x5 box sums -> (a, b) surfaces in shared memory -> weighted neighbourhood
//      sums -> output (5x5 at half vertical rate, exactly like sgr_finish_filter2).
// The Level-1 entry points run the same tile code over a host-assembled window.
#include "host_util.h"
// the tables live in global memory: x_by_x is copied into shared memory per CTA, the sgr parameters are read once per tile
#define B200_TBL __device__
#include "tables_gen.h"

namespace b200 {

constexpr int kTW = 64, kTH = 32, kSH = kTH + 6;

struct LrTileParams {
    int type;             // 0 none, 1 wiener, 2 sgr
    int fh[7], fv[7];     // wiener taps (fh[3] without the 8-bit +128 split: added from the centre sample)
    unsigned s0, s1; int w0, w1;   // sgr
    ptrdiff_t out; int st;   // lr_frame_kernel: the tile's first output sample (in samples from B200LrFrame::dst), pitch
};

// the shared layout of one tile at most TW wide; a 32-wide one is half the size of a 64-wide one, so a U / V pair of
// them overlays one 64-wide tile
template <int TW> struct LrShared {
    static constexpr int SW = TW + 6;
    LrTileParams P;       // lr_frame_kernel: the tile's parameters (at the tile's own base: one address register per half)
    uint16_t src[kSH][SW + 2];
    union {
        uint16_t hor[kSH][TW];
        struct {
            int A3[kTH + 2][TW + 2]; uint16_t B3[kTH + 2][TW + 2];
            int A5[kTH / 2 + 2][TW + 2]; uint16_t B5[kTH / 2 + 2][TW + 2];
        } s;
    } u;
};
constexpr size_t kLrSmem = sizeof(LrShared<kTW>) > 2 * sizeof(LrShared<32>) ? sizeof(LrShared<kTW>) : 2 * sizeof(LrShared<32>);

// b200_sgr_x_by_x as 64 words in shared memory: the self-guided passes index it per lane, which a constant-bank load
// would serialise into one replay per distinct index; a shared byte table costs at most a 2-way bank conflict
B200_DEV void lr_stage_x_by_x(unsigned *tbl)
{
    const int i = threadIdx.x;
    if (i < 64)
        tbl[i] = (unsigned)b200_sgr_x_by_x[4 * i] | (unsigned)b200_sgr_x_by_x[4 * i + 1] << 8 |
                 (unsigned)b200_sgr_x_by_x[4 * i + 2] << 16 | (unsigned)b200_sgr_x_by_x[4 * i + 3] << 24;
}

// The two compute passes of a staged tile on threads tid = 0 .. nt - 1; the caller puts one barrier between them, so
// both tiles of a pair (and every tile type) run one barrier schedule.
// pass 1: Wiener rows into u.hor, or the self-guided (a, b) surfaces
template <bool HBD, int TW>
B200_DEV void lr_tile_pass1(LrShared<TW> &sm, const LrTileParams &P, const unsigned *tbl, int tw, int th, int bdmax,
                            int tid, int nt)
{
    const int bitdepth = HBD ? 32 - __clz(bdmax) : 8;
    const uint8_t *x_by_x = (const uint8_t *)tbl;
    if (P.type == 1) {
        const int rbh = 3 + (bitdepth == 12) * 2;
        const int clip_limit = 1 << (bitdepth + 1 + 7 - rbh);
        // horizontal: 4 consecutive outputs per thread share their 10 source samples
        for (int i = tid; i < (th + 6) * (TW / 4); i += nt) {
            const int y = i / (TW / 4), x = (i - y * (TW / 4)) * 4;
            if (x >= tw) continue;
            int v[10];
#pragma unroll
            for (int k = 0; k < 10; k++) v[k] = sm.src[y][x + k];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                int sum = 1 << (bitdepth + 6);
                if (!HBD) sum += v[j + 3] * 128;
#pragma unroll
                for (int k = 0; k < 7; k++) sum += v[j + k] * P.fh[k];
                sm.u.hor[y][x + j] = (uint16_t)iclip((sum + (1 << (rbh - 1))) >> rbh, 0, clip_limit - 1);
            }
        }
        return;
    }
    // ---- self-guided ----
    const int b8 = bitdepth - 8;
    constexpr int NS = (TW + 2 + 3) / 4;
    if (P.s1) {      // 3x3 surfaces at rows -1 .. th, cols -1 .. tw
        // 4 consecutive surface points per thread: 3 x 6 source samples -> column sums -> sliding 3-wide sums
        for (int i = tid; i < (th + 2) * NS; i += nt) {
            const int yy = i / NS, xx = (i - yy * NS) * 4;           // surface index; source centre (xx + 2, yy + 2)
            if (xx >= tw + 2) continue;
            int cs[6], cq[6];
#pragma unroll
            for (int k = 0; k < 6; k++) {
                const int v0 = sm.src[yy + 1][xx + 1 + k], v1 = sm.src[yy + 2][xx + 1 + k], v2 = sm.src[yy + 3][xx + 1 + k];
                cs[k] = v0 + v1 + v2; cq[k] = v0 * v0 + v1 * v1 + v2 * v2;
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (xx + k >= tw + 2) break;
                const int sum = cs[k] + cs[k + 1] + cs[k + 2], sq = cq[k] + cq[k + 1] + cq[k + 2];
                const int a = (sq + ((1 << (2 * b8)) >> 1)) >> (2 * b8);
                const int b = (sum + ((1 << b8) >> 1)) >> b8;
                const unsigned p = (unsigned)imax(a * 9 - b * b, 0);
                const unsigned z = (p * P.s1 + (1u << 19)) >> 20;
                const unsigned x = x_by_x[z < 255u ? z : 255u];
                sm.u.s.A3[yy][xx + k] = (int)((x * (unsigned)sum * 455u + (1u << 11)) >> 12);
                sm.u.s.B3[yy][xx + k] = (uint16_t)x;
            }
        }
    }
    if (P.s0) {      // 5x5 surfaces at odd rows -1, 1, 3, ... (index j <-> row 2j - 1)
        const int nrow = (th + 1) / 2 + 1;
        for (int i = tid; i < nrow * NS; i += nt) {
            const int j = i / NS, xx = (i - j * NS) * 4;
            if (xx >= tw + 2) continue;
            const int cy = 2 * j - 1 + 3;                            // source row index of the centre
            int cs[8], cq[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                int su = 0, sq = 0;
#pragma unroll
                for (int dy = -2; dy <= 2; dy++) { const int v = sm.src[cy + dy][xx + k]; su += v; sq += v * v; }
                cs[k] = su; cq[k] = sq;
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (xx + k >= tw + 2) break;
                const int sum = cs[k] + cs[k + 1] + cs[k + 2] + cs[k + 3] + cs[k + 4];
                const int sq = cq[k] + cq[k + 1] + cq[k + 2] + cq[k + 3] + cq[k + 4];
                const int a = (sq + ((1 << (2 * b8)) >> 1)) >> (2 * b8);
                const int b = (sum + ((1 << b8) >> 1)) >> b8;
                const unsigned p = (unsigned)imax(a * 25 - b * b, 0);
                const unsigned z = (p * P.s0 + (1u << 19)) >> 20;
                const unsigned x = x_by_x[z < 255u ? z : 255u];
                sm.u.s.A5[j][xx + k] = (int)((x * (unsigned)sum * 164u + (1u << 11)) >> 12);
                sm.u.s.B5[j][xx + k] = (uint16_t)x;
            }
        }
    }
}

// pass 2: Wiener columns, or the self-guided output; tw x th outputs
template <bool HBD, int TW, class Store>
B200_DEV void lr_tile_pass2(LrShared<TW> &sm, const LrTileParams &P, int tw, int th, int bdmax, int tid, int nt, Store store)
{
    const int bitdepth = HBD ? 32 - __clz(bdmax) : 8;
    if (P.type == 1) {
        const int rbv = 11 - (bitdepth == 12) * 2;
        // vertical: 4 consecutive rows per thread share their 10 intermediate samples
        const int round_offset = 1 << (bitdepth + (rbv - 1));
        for (int i = tid; i < ((th + 3) / 4) * TW; i += nt) {
            const int yq = i / TW, x = i - yq * TW, y = yq * 4;
            if (x >= tw) continue;
            int v[10];
#pragma unroll
            for (int k = 0; k < 10; k++) v[k] = y + k < th + 6 ? (int)sm.u.hor[y + k][x] : 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (y + j >= th) break;
                int sum = -round_offset;
#pragma unroll
                for (int k = 0; k < 7; k++) sum += v[j + k] * P.fv[k];
                store(x, y + j, iclip((sum + (1 << (rbv - 1))) >> rbv, 0, bdmax));
            }
        }
        return;
    }
    // 4 consecutive pixels of a row per thread: the neighbourhood sums are built from per-column partial sums
    for (int i = tid; i < th * (TW / 4); i += nt) {
        const int y = i / (TW / 4), x = (i - y * (TW / 4)) * 4;
        if (x >= tw) continue;
        int t5a[4] = { 0, 0, 0, 0 }, t5b[4] = { 0, 0, 0, 0 }, t3a[4] = { 0, 0, 0, 0 }, t3b[4] = { 0, 0, 0, 0 };
        if (P.s0) {
            int ca[6], cb[6];
            if (!(y & 1)) {
                const int j0 = y >> 1, j1 = j0 + 1;                   // rows y - 1 and y + 1
#pragma unroll
                for (int k = 0; k < 6; k++) { ca[k] = (int)sm.u.s.B5[j0][x + k] + sm.u.s.B5[j1][x + k]; cb[k] = sm.u.s.A5[j0][x + k] + sm.u.s.A5[j1][x + k]; }
            } else {
                const int j = (y + 1) >> 1;                           // row y
#pragma unroll
                for (int k = 0; k < 6; k++) { ca[k] = sm.u.s.B5[j][x + k]; cb[k] = sm.u.s.A5[j][x + k]; }
            }
#pragma unroll
            for (int k = 0; k < 4; k++) { t5a[k] = ca[k + 1] * 6 + (ca[k] + ca[k + 2]) * 5; t5b[k] = cb[k + 1] * 6 + (cb[k] + cb[k + 2]) * 5; }
        }
        if (P.s1) {
            const int ys = y + 1;
            int ma[6], va[6], mb[6], vb[6];
#pragma unroll
            for (int k = 0; k < 6; k++) {
                ma[k] = sm.u.s.B3[ys][x + k]; va[k] = (int)sm.u.s.B3[ys - 1][x + k] + sm.u.s.B3[ys + 1][x + k];
                mb[k] = sm.u.s.A3[ys][x + k]; vb[k] = sm.u.s.A3[ys - 1][x + k] + sm.u.s.A3[ys + 1][x + k];
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                t3a[k] = (ma[k + 1] + ma[k] + ma[k + 2] + va[k + 1]) * 4 + (va[k] + va[k + 2]) * 3;
                t3b[k] = (mb[k + 1] + mb[k] + mb[k + 2] + vb[k + 1]) * 4 + (vb[k] + vb[k + 2]) * 3;
            }
        }
        int out[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int src = sm.src[y + 3][x + k + 3];
            int t5 = 0, t3 = 0;
            if (P.s0) t5 = !(y & 1) ? (t5b[k] - t5a[k] * src + (1 << 8)) >> 9 : (t5b[k] - t5a[k] * src + (1 << 7)) >> 8;
            if (P.s1) t3 = (t3b[k] - t3a[k] * src + (1 << 8)) >> 9;
            const int v = P.w0 * t5 + P.w1 * t3;     // the unused term is zero (w0 = 0 without s0; t3 = 0 without s1)
            out[k] = iclip(src + ((v + (1 << 10)) >> 11), 0, bdmax);
        }
        store.row4(x, y, out, imin(4, tw - x));
    }
}

// where lr_tile_pass2 writes: sample (x, y) of the tile, or 4 consecutive samples of a row of which the first n are inside
template <class pixel> struct LrStore {
    pixel *o; ptrdiff_t st;   // tile origin and row pitch
    B200_DEV void operator()(int x, int y, int v) const { o[y * st + x] = (pixel)v; }
    B200_DEV void row4(int x, int y, const int (&v)[4], int n) const {
        pixel *p = o + y * st + x;
        if (n == 4 && !((uintptr_t)p & (4 * sizeof(pixel) - 1))) {
            if (sizeof(pixel) == 1) *(unsigned *)p = (unsigned)v[0] | (unsigned)v[1] << 8 | (unsigned)v[2] << 16 | (unsigned)v[3] << 24;
            else *(uint2 *)p = make_uint2((unsigned)v[0] | (unsigned)v[1] << 16, (unsigned)v[2] | (unsigned)v[3] << 16);
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) if (k < n) p[k] = (pixel)v[k];
        }
    }
};

B200_DEV void lr_unit_params(const B200RestorationUnit &u, bool hbd, LrTileParams &P)
{
    P.type = u.type == 0 ? 0 : (u.type == 2 ? 1 : 2);
    P.s0 = P.s1 = 0; P.w0 = P.w1 = 0;
    if (u.type == 2) {                    // reference src/lr_apply_tmpl.c:55-72
#pragma unroll
        for (int i = 0; i < 3; i++) { P.fh[i] = P.fh[6 - i] = u.filter_h[i]; P.fv[i] = P.fv[6 - i] = u.filter_v[i]; }
        P.fh[3] = -(P.fh[0] + P.fh[1] + P.fh[2]) * 2 + (hbd ? 128 : 0);
        P.fv[3] = 128 - (P.fv[0] + P.fv[1] + P.fv[2]) * 2;
    } else if (u.type >= 3) {             // :73-84
        const int idx = u.type - 3;
        P.s0 = b200_sgr_params[idx][0]; P.s1 = b200_sgr_params[idx][1];
        P.w0 = u.sgr_weights[0]; P.w1 = 128 - (u.sgr_weights[0] + u.sgr_weights[1]);
        if (!P.s0) P.w0 = 0;              // sgr_3x3 ignores w0; keeps the fused formula exact
        if (!P.s1) P.w1 = 0;              // sgr_5x5 ignores w1
    }
}

// flattened tile list: plane p owns CTAs base[p] .. , nx[p] tiles per row; nx_recip = ceil(2^32 / nx):
// local / nx == mulhi(local, nx_recip) while local * nx < 2^32. pair: the chroma tiles are 32 wide and run as U / V
// pairs, so plane 1's CTAs restore both chroma planes and plane 2's range is empty.
struct LrGrid { int base[3], nx[3]; unsigned nx_recip[3]; int ty0[3]; int pair; };

// One tile of plane pl on threads tid = 0 .. NT - 1 (all 256 of the CTA, or one half of a U / V pair). Both halves of
// a pair have the same geometry, so they leave together or run the same two barriers whatever their unit types: one
// after the parameters and the staged source, one between the two compute passes (an unrestored tile is copied out
// of the staged source in the first pass).
template <bool HBD, int TW, int NT>
B200_DEV void lr_frame_tile(const B200LrFrame &f, const LrGrid &lg, int bdmax, int rp, int pl, int local, int tid,
                            LrShared<TW> &sm, const unsigned *tbl)
{
    typedef typename Bd<HBD>::pixel pixel;
    const int ssh = pl ? f.ss_hor : 0, ssv = pl ? f.ss_ver : 0;
    const int w = (f.w + ssh) >> ssh, h = (f.h + ssv) >> ssv;
    const int us_log2 = f.unit_size_log2[pl ? 1 : 0], unit = 1 << us_log2, half = unit >> 1;
    const int tw_full = unit < TW ? unit : TW;
    const int nxp = lg.nx[rp];
    const int tyl = nxp > 1 ? (int)__umulhi((unsigned)local, lg.nx_recip[rp]) : local, txi = local - tyl * nxp;
    const int tyi = tyl + lg.ty0[rp];                     // first tile row of this launch (a band, or 0 for the frame)
    const int x0 = txi * tw_full;
    // a 64-row luma stripe is 2 tiles tall; a vertically subsampled stripe (32 rows) is 1
    const int k = ssv ? tyi : tyi >> 1, ty = ssv ? 0 : tyi & 1;
    const int y0s = k ? (64 * k - 8) >> ssv : 0;
    const int y1s = imin(h, (64 * (k + 1) - 8) >> ssv);
    const int ty0 = y0s + ty * kTH;
    if (x0 >= w || y0s >= h || ty0 >= y1s) return;
    const int tw = imin(tw_full, w - x0), th = imin(kTH, y1s - ty0);
    const pixel *C = (const pixel *)f.cdef + f.plane_off[pl];
    const pixel *D = (const pixel *)f.dbl + f.plane_off[pl];
    const int st = f.stride[pl];

    const bool have_top = y0s > 0, have_bot = y1s < h;
    constexpr int PPW = HBD ? 2 : 4;                                 // samples per 32-bit word
    // interior tiles are staged from aligned words over picture columns x0-4 .. x0+tw+3 (one more column on each
    // side than needed)
    const bool interior = x0 >= 4 && x0 + tw + 4 <= w && !(tw & 3) && !(x0 & 3) && !(st & (PPW - 1)) &&
                          !(((uintptr_t)C | (uintptr_t)D | (uintptr_t)((pixel *)f.dst + f.plane_off[pl])) & 3);
    const int NW = (tw + 8) / PPW;
    const unsigned magic = recip16(NW);                   // exact i / NW for i < 38 * 36

    // The unit lookup and the tap / weight set-up are per-tile work: the tile's thread 0 starts them, the loads of the
    // interior staging are issued by every thread while its lr_mask load is in flight, and the tile reads the
    // parameters and the staged source after the first barrier.
    B200RestorationUnit u;
    u.type = 0;
    if (tid == 0 && (f.restore_planes & (1 << pl))) {
        // unit lookup: reference src/lr_apply_tmpl.c:107-148
        int n_full = 0;
        { const int max_unit = unit + half; if (w >= max_unit) n_full = (w - max_unit) / unit + 1; }
        const int ux = imin(x0 >> us_log2, n_full), xu = ux << us_log2;
        const int sby = ((y0s << ssv) + (y0s ? 8 : 0)) >> (6 + f.sb128);
        const int row_y = (sby << (6 + f.sb128)) >> ssv;
        int aligned = row_y & ~(unit - 1);
        if (aligned && aligned + half > h) aligned -= unit;
        aligned <<= ssv;
        const int sb_idx = (aligned >> 7) * f.sr_sb128w, unit_idx = ((aligned >> 6) & 1) << 1;
        const int shift_hor = 7 - ssh;
        u = f.lr_mask[sb_idx + (xu >> shift_hor)].lr[pl][unit_idx + ((xu >> (shift_hor - 1)) & 1)];
    }
    constexpr int NI = ((kSH * (TW + 8)) / PPW + NT - 1) / NT;    // words per thread: 3 (8-bit) or 6
    unsigned wv[NI];
    if (interior) {
#pragma unroll
        for (int n = 0; n < NI; n++) {
            const int i = tid + n * NT;
            const int yy = (int)((i * magic) >> 16), g = i - yy * NW;
            if (yy >= th + 6) break;
            int Y = ty0 - 3 + yy;
            const pixel *base = C;
            if (Y < y0s) {
                if (have_top) { base = D; Y = imax(Y, y0s - 2); } else Y = y0s;
            } else if (Y >= y1s) {
                if (have_bot) { base = D; Y = imin(imin(Y, y1s + 1), h - 1); } else Y = y1s - 1;
            }
            wv[n] = *(const unsigned *)(base + (ptrdiff_t)Y * st + x0 - 4 + g * PPW);
        }
    }
    // stage the virtual source: rows ty0-3 .. ty0+th+2, cols x0-3 .. x0+tw+2
    if (interior) {
#pragma unroll
        for (int n = 0; n < NI; n++) {
            const int i = tid + n * NT;
            const int yy = (int)((i * magic) >> 16), g = i - yy * NW;
            if (yy >= th + 6) break;
            const int c0 = g * PPW - 1;                              // tile column of the word's first sample
#pragma unroll
            for (int k = 0; k < PPW; k++) {
                const int c = c0 + k;
                if (c >= 0 && c < tw + 6) sm.src[yy][c] = (uint16_t)(HBD ? (wv[n] >> (16 * k)) & 0xffff : (wv[n] >> (8 * k)) & 0xff);
            }
        }
    } else
    for (int i = tid; i < (th + 6) * LrShared<TW>::SW; i += NT) {
        const int yy = i / LrShared<TW>::SW, xx = i - yy * LrShared<TW>::SW;
        if (xx >= tw + 6) continue;
        int Y = ty0 - 3 + yy;
        const int X = iclip(x0 - 3 + xx, 0, w - 1);
        const pixel *base = C;
        if (Y < y0s) {
            if (have_top) { base = D; Y = imax(Y, y0s - 2); } else Y = y0s;
        } else if (Y >= y1s) {
            if (have_bot) { base = D; Y = imin(imin(Y, y1s + 1), h - 1); } else Y = y1s - 1;
        }
        sm.src[yy][xx] = base[(ptrdiff_t)Y * st + X];
    }
    if (tid == 0) {
        LrTileParams P;
        lr_unit_params(u, HBD, P);
        P.out = f.plane_off[pl] + (ptrdiff_t)ty0 * st + x0; P.st = st;
        sm.P = P;
    }
    __syncthreads();
    const LrTileParams &P = sm.P;
    // (the output origin and pitch are read from shared memory where they are used: kept in registers across the
    // passes, they cost registers the passes need)
    if (P.type == 0) {
        // an unrestored tile is the staged tile copied out, 4 samples of a row per thread
        const LrStore<pixel> store{ (pixel *)f.dst + P.out, P.st };
        for (int i = tid; i < th * (TW / 4); i += NT) {
            const int y = i / (TW / 4), x = (i - y * (TW / 4)) * 4;
            if (x >= tw) continue;
            const int v[4] = { sm.src[y + 3][x + 3], sm.src[y + 3][x + 4], sm.src[y + 3][x + 5], sm.src[y + 3][x + 6] };
            store.row4(x, y, v, imin(4, tw - x));
        }
    } else
        lr_tile_pass1<HBD>(sm, P, tbl, tw, th, bdmax, tid, NT);
    __syncthreads();
    if (P.type) lr_tile_pass2<HBD>(sm, P, tw, th, bdmax, tid, NT, LrStore<pixel>{ (pixel *)f.dst + P.out, P.st });
}

template <bool HBD>
#ifndef B200_LR_MINB
#define B200_LR_MINB 6
#endif
__global__ void __launch_bounds__(256, B200_LR_MINB) lr_frame_kernel(const __grid_constant__ B200LrFrame f, const __grid_constant__ LrGrid lg, int bdmax)
{
    B200_PDL_ENTRY();
    __shared__ __align__(16) unsigned char smem[kLrSmem];
    __shared__ unsigned tbl[64];
    lr_stage_x_by_x(tbl);                                 // read after the tile's first barrier
    const int bid = blockIdx.x;
    const int pl = bid >= lg.base[2] ? 2 : bid >= lg.base[1] ? 1 : 0;
    if (pl && lg.pair) {
        const int hf = threadIdx.x >> 7;                  // threads 0-127: U, 128-255: V
        lr_frame_tile<HBD, 32, 128>(f, lg, bdmax, 1, 1 + hf, bid - lg.base[1], threadIdx.x & 127,
                                    ((LrShared<32> *)smem)[hf], tbl);
    } else
        lr_frame_tile<HBD, kTW, 256>(f, lg, bdmax, pl, pl, bid - lg.base[pl], threadIdx.x, *(LrShared<kTW> *)smem, tbl);
}

// Level 1: window = host-assembled (w + 6) x (h + 6) virtual source; out = dense w x h
template <bool HBD>
__global__ void __launch_bounds__(256) lr_window_kernel(const typename Bd<HBD>::pixel *win, typename Bd<HBD>::pixel *out,
                                                        int w, int h, LrTileParams P, int bdmax)
{
    __shared__ LrShared<kTW> sm;
    __shared__ unsigned tbl[64];
    lr_stage_x_by_x(tbl);
    const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const int tw = imin(kTW, w - x0), th = imin(kTH, h - y0);
    for (int i = threadIdx.x; i < (th + 6) * LrShared<kTW>::SW; i += blockDim.x) {
        const int yy = i / LrShared<kTW>::SW, xx = i - yy * LrShared<kTW>::SW;
        if (xx >= tw + 6) continue;
        sm.src[yy][xx] = win[(size_t)(y0 + yy) * (w + 6) + x0 + xx];
    }
    __syncthreads();
    lr_tile_pass1<HBD>(sm, P, tbl, tw, th, bdmax, (int)threadIdx.x, (int)blockDim.x);
    __syncthreads();
    lr_tile_pass2<HBD>(sm, P, tw, th, bdmax, (int)threadIdx.x, (int)blockDim.x, LrStore<typename Bd<HBD>::pixel>{ out + (size_t)y0 * w + x0, w });
}

// tile rows [r0, r1) of the sweep, counted in half stripes: tile row r is rows 32 r - 8 .. 32 r + 23 of the luma plane
// (the first one starts at row 0); a vertically subsampled plane has one tile per stripe, so it runs its stripes
// [r0 / 2, r1 / 2) — callers that cut a frame into bands pass r0, r1 odd: a chroma stripe runs with the band that completes it.
int lr_frame_rows(int bdmax, const B200LrFrame *f, int r0, int r1, cudaStream_t stream)
{
    if (int r = check_bdmax(bdmax, "b200_lr_frame")) return r;
    for (int i = 0; i < 2; i++)
        if (f->unit_size_log2[i] < 5 || f->unit_size_log2[i] > 8) { b200_set_error("b200_lr_frame: bad unit size"); return -2; }
    const int n_stripes = (f->h + 8 + 63) / 64;
    r0 = imax(r0, 0); r1 = imin(r1, 2 * n_stripes);
    // (A register-only path for Wiener tiles — rolling ring as in mc.cu, dp4a horizontal pass, no staging — was no faster
    // than this staged form, and slower with all rows loaded up front at lower occupancy. Dropped.)
    LrGrid lg;
    lg.pair = f->unit_size_log2[1] == 5;                  // 32-wide chroma tiles: U / V pairs in plane 1's range
    int total = 0;
    for (int p = 0; p < 3; p++) {
        const int ssh = p ? f->ss_hor : 0, ssv = p ? f->ss_ver : 0;
        const int w = (f->w + ssh) >> ssh;
        const int unit = 1 << f->unit_size_log2[p ? 1 : 0], tw_full = unit < kTW ? unit : kTW;
        lg.nx[p] = (w + tw_full - 1) / tw_full;
        lg.nx_recip[p] = lg.nx[p] > 1 ? (unsigned)(((1ull << 32) + lg.nx[p] - 1) / lg.nx[p]) : 0u;
        lg.base[p] = total;
        const int a = ssv ? r0 >> 1 : r0, b = ssv ? r1 >> 1 : r1;
        lg.ty0[p] = a;
        if (p < 2 || !lg.pair) total += lg.nx[p] * imax(b - a, 0);
    }
    if (!total) return 0;
    return launch_hbd(bdmax, Launch::pdl, dim3(total), dim3(256), 0, stream,
                      [&](auto hbd) { return std::make_tuple(lr_frame_kernel<hbd>, *f, lg, bdmax); });
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_lr_frame(int bdmax, const B200LrFrame *f, void *stream)
{
    return b200::lr_frame_rows(bdmax, f, 0, 1 << 30, (cudaStream_t)stream);
}

int b200_lr_filter(int kind, void *dst, ptrdiff_t stride, const void *left, const void *lpf, int w, int h,
                   const void *params, int edges, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_lr_filter")) return r;
    if (kind < 0 || kind > 3 || w < 1 || w > 384 || h < 1 || h > 64) { b200_set_error("b200_lr_filter: bad arguments"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    // which short-stripe exits of the C reference skip the bottom rows (see oracle/looprestoration.c header)
    int use_bottom;
    if (kind == 0) use_bottom = (edges & 8) && h > ((edges & 4) ? 3 : 5);
    else if (kind == 2) use_bottom = (edges & 8) && h > 2;
    else use_bottom = (edges & 8) && !(h & 1) && h > ((edges & 4) ? 2 : 4);
    // assemble the virtual source window (pure data movement; all arithmetic happens on the device)
    uint8_t *win = (uint8_t *)L.host((size_t)(w + 6) * (h + 6) * px);
    if (!win) return -1;
    for (int y = -3; y < h + 3; y++) {
        const uint8_t *row; int from_unit = 0, yy = y;
        if (y < 0 && (edges & 4)) row = (const uint8_t *)lpf + (ptrdiff_t)((y < -2 ? -2 : y) + 2) * stride;
        else if (y >= h && use_bottom) row = (const uint8_t *)lpf + (ptrdiff_t)(6 + (y - h > 1 ? 1 : y - h)) * stride;
        else { yy = y < 0 ? 0 : y >= h ? h - 1 : y; row = (const uint8_t *)dst + (ptrdiff_t)yy * stride; from_unit = 1; }
        for (int x = -3; x < w + 3; x++) {
            const uint8_t *sp;
            if (x < 0) {
                if (!(edges & 1)) sp = row;
                else if (from_unit && left) sp = (const uint8_t *)left + ((size_t)yy * 4 + 4 + x) * px;
                else sp = row + (ptrdiff_t)x * (ptrdiff_t)px;
            } else if (x >= w && !(edges & 2)) sp = row + (size_t)(w - 1) * px;
            else sp = row + (size_t)x * px;
            memcpy(win + ((size_t)(y + 3) * (w + 6) + (x + 3)) * px, sp, px);
        }
    }
    LrTileParams P;
    memset(&P, 0, sizeof(P));
    if (kind == 0) {
        const int16_t (*flt)[8] = (const int16_t (*)[8])params;
        P.type = 1;
        for (int i = 0; i < 7; i++) { P.fh[i] = flt[0][i]; P.fv[i] = flt[1][i]; }
    } else {
        const uint32_t *sp = (const uint32_t *)params;
        const int16_t *wp = (const int16_t *)(sp + 2);
        P.type = 2;
        P.s0 = kind == 2 ? 0 : sp[0]; P.s1 = kind == 1 ? 0 : sp[1];
        P.w0 = kind == 2 ? 0 : wp[0]; P.w1 = kind == 1 ? 0 : wp[1];
        if (kind == 1) P.w0 = wp[0];   // sgr_5x5 weights its single term with w0
    }
    void *in, *out;
    if (!(in = L.upload(0, win, (size_t)(w + 6) * (h + 6) * px)) || !(out = L.dev(1, (size_t)w * h * px))) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3((w + kTW - 1) / kTW, (h + kTH - 1) / kTH), dim3(256), 0, 0, [&](auto hbd) {
            typedef typename Bd<hbd>::pixel pixel;
            return std::make_tuple(lr_window_kernel<hbd>, (const pixel *)in, (pixel *)out, w, h, P, bdmax);
        }))
        return r;
    return L.download_rect(1, dst, stride, w, h, px);
}

}  // extern "C"

namespace {
template <int K> void lr8(uint8_t *d, ptrdiff_t s, const void *l, const uint8_t *lpf, int w, int h, const void *p, int e) {
    if (b200_lr_filter(K, d, s, l, lpf, w, h, p, e, 255)) die("looprestoration");
}
template <int K> void lr16(uint16_t *d, ptrdiff_t s, const void *l, const uint16_t *lpf, int w, int h, const void *p, int e, int bd) {
    if (b200_lr_filter(K, d, s, l, lpf, w, h, p, e, bd)) die("looprestoration");
}
}
extern "C" {
void b200_loop_restoration_dsp_init_8bpc(B200LoopRestorationDSPContext *c, int bpc) {
    (void)bpc;
    c->wiener[0] = c->wiener[1] = (void *)lr8<0>;
    c->sgr[0] = (void *)lr8<1>; c->sgr[1] = (void *)lr8<2>; c->sgr[2] = (void *)lr8<3>;
}
void b200_loop_restoration_dsp_init_16bpc(B200LoopRestorationDSPContext *c, int bpc) {
    (void)bpc;
    c->wiener[0] = c->wiener[1] = (void *)lr16<0>;
    c->sgr[0] = (void *)lr16<1>; c->sgr[1] = (void *)lr16<2>; c->sgr[2] = (void *)lr16<3>;
}
}
