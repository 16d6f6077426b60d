// Motion compensation (dav1d Dav1dMCDSPContext, reference src/mc_tmpl.c).
//
//   mc_pred_kernel   put / prep, 8-tap pairs + bilinear (:129-187, 246-305, 434-489, 533-586)
//                    one CTA per prediction block; a lane owns one output column of an
//                    8-row strip, keeps the 15 horizontally-filtered rows it needs in
//                    registers and runs the vertical filter from them (no shared memory,
//                    no int16 `mid` round trip). Source coordinates are clamped to the
//                    reference plane = dav1d's emu_edge (:868-916) folded into the loads.
//   mc_comp_kernel   avg / w_avg / mask / w_mask{444,422,420} (:628-681, 724-781)
//   mc_blend_kernel  blend / blend_v / blend_h (:683-722)
//   mc_warp_kernel   warp_affine_8x8 / 8x8t (:799-866), one warp per 8x8 block
//   resize_frame_kernel  super-resolution upscaling of whole planes (:918-944)
//   emu_edge_kernel  (:868-916) for the Level-1 table only: the prediction kernels fold emu_edge into their loads
// Integer only; bit-exact with the reference C path.
#include "host_util.h"
#define B200_TBL __constant__
#include "tables_gen.h"

namespace b200 {

// enum Filter2d -> horizontal / vertical Dav1dFilterMode (reference src/levels.h:184-196)
__constant__ uint8_t c_f2d_h[9] = { 0, 0, 0, 2, 2, 2, 1, 1, 1 };
__constant__ uint8_t c_f2d_v[9] = { 0, 1, 2, 0, 1, 2, 0, 1, 2 };

template <bool HBD> B200_DEV int inter_bits(int bdmax) {
    if (!HBD) return 4;
    return 14 - (32 - __clz(bdmax));   // 4 for 10-bit, 2 for 12-bit
}

#define RND_SH(v, sh) (((v) + ((1 << (sh)) >> 1)) >> (sh))

constexpr int kMcWarps = 4;

// sum of 4 unsigned bytes of `px` times 4 signed bytes of `taps`, plus acc
B200_DEV int dp4a_us(unsigned px, int taps, int acc) {
#ifdef B200_EMU
    return __dp4a_us(px, taps, acc);
#else
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(px), "r"(taps), "r"(acc));
    return d;
#endif
}

// two unsigned halfwords of `px` times signed bytes {0,1} (HI = false) or {2,3} (HI = true) of `taps`, plus acc
template <bool HI> B200_DEV int dp2a_us(unsigned px, int taps, int acc) {
#ifdef B200_EMU
    const int t0 = (int8_t)(taps >> (HI ? 16 : 0)), t1 = (int8_t)(taps >> (HI ? 24 : 8));
    return acc + (int)(px & 0xffff) * t0 + (int)(px >> 16) * t1;
#else
    int d;
    if (HI) asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(px), "r"(taps), "r"(acc));
    else asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(px), "r"(taps), "r"(acc));
    return d;
#endif
}

#ifndef B200_MC_MINB
#define B200_MC_MINB 5
#endif
#ifndef B200_MC_S1
#define B200_MC_S1 0
#endif

// filter taps of one prediction (registers): 8-tap / 4-tap sets or the bilinear pair, and the base shift
struct McTaps { int fh[8], fv[8]; int fsh; bool has_h, has_v; };
B200_DEV void mc_taps(McTaps &t, int filter2d, int mx, int my, int w, int h)
{
    const bool bilin = filter2d == 9;
    t.has_h = mx != 0; t.has_v = my != 0; t.fsh = bilin ? 4 : 6;
#pragma unroll
    for (int k = 0; k < 8; k++) t.fh[k] = t.fv[k] = 0;
    // an axis without a fractional phase gets the identity filter (1 << fsh at the centre tap): every block then runs the
    // same horizontal + vertical code, and the result is the reference's "no filter on this axis" arithmetic exactly
    // (sum = px << fsh, so each rounding shift of the filtered form reduces to the shift of the unfiltered form)
    t.fh[3] = t.fv[3] = 1 << t.fsh;
    if (bilin) {
        t.fh[3] = 16 - mx; t.fh[4] = mx; t.fv[3] = 16 - my; t.fv[4] = my;
    } else {
        // 4-tap sets for w <= 4 / h <= 4 (reference src/mc_tmpl.c:115-123)
        if (t.has_h) {
            const int f = c_f2d_h[filter2d];
            const int idx = w > 4 ? f : 3 + (f & 1);
#pragma unroll
            for (int k = 0; k < 8; k++) t.fh[k] = b200_mc_subpel_filters[idx][mx - 1][k];
        }
        if (t.has_v) {
            const int f = c_f2d_v[filter2d];
            const int idx = h > 4 ? f : 3 + (f & 1);
#pragma unroll
            for (int k = 0; k < 8; k++) t.fv[k] = b200_mc_subpel_filters[idx][my - 1][k];
        }
    }
}

// ---- put / prep, register-column form ------------------------------------------------------------------
// One warp per prediction block; a lane owns an ITEM = one output column x R consecutive rows. It walks the R + 7 source
// rows of its column from top to bottom: each row is filtered horizontally straight from the reference picture (three
// aligned 32-bit words, realigned with funnel shifts, 2 dp4a — 10/12-bit: five words, 4 dp2a) and its value is
// scattered into the 8 running vertical sums it contributes to (a ring of 8 accumulators: row r feeds outputs r-7 .. r);
// the sum of output r-7 is complete after row r and is rounded and stored at once. No shared memory, no barriers, no
// int16 tile: neighbouring lanes read the same words (L1 hits), a row store is one contiguous segment per warp, and the
// code is ONE loop body of 8 rows for every block shape and filter (an axis without a fractional phase runs the identity
// filter), a couple of hundred instructions.
// History: an earlier form staged a window in shared memory and made two passes over an int16 tile (more instructions).
// A first register form kept all R + 7 row values in registers, fully unrolled per item height and per filter case: fewer
// instructions but so much straight-line code that instruction-cache misses became the top stall. The rolling ring keeps
// the instruction count and fits the instruction cache.
template <bool HBD> struct McSrc {
    typedef typename Bd<HBD>::pixel pixel;
    const pixel *ref; int rs, rw, rh;
};

struct McOut {             // where an item's outputs go: pixels (put) or int16 (prep)
    void *px; int ds; int16_t *tmp; int tw; bool is_prep;
};

// per-prediction constants of an item computation
template <bool HBD> struct McPred {
    McSrc<HBD> S;
    int fv[8];               // vertical taps
    int fh_lo, fh_hi;        // horizontal taps packed as signed bytes (dp4a / dp2a operands)
    int gx, gy;              // reference sample of output (0, 0)'s first tap
    int fsh, hsh, hrnd;      // base shift; horizontal pass: (sum + hrnd) >> hsh = RND_SH(sum, fsh - intermediate_bits)
    bool interior;
};

template <bool HBD>
B200_DEV void mc_pred_setup(McPred<HBD> &P, const B200McFrame &fr, int ref, int pl, int filter2d, int mx, int my, int w, int h,
                            int sx, int sy, int ib)
{
    typedef typename Bd<HBD>::pixel pixel;
    P.S.ref = (const pixel *)fr.ref[ref] + fr.ref_plane_off[pl];
    P.S.rs = fr.ref_stride[pl]; P.S.rw = fr.ref_w[pl]; P.S.rh = fr.ref_h[pl];
    McTaps t;
    mc_taps(t, filter2d, mx, my, w, h);
#pragma unroll
    for (int k = 0; k < 8; k++) P.fv[k] = t.fv[k];
    P.fh_lo = (t.fh[0] & 0xff) | (t.fh[1] & 0xff) << 8 | (t.fh[2] & 0xff) << 16 | (t.fh[3] & 0xff) << 24;
    P.fh_hi = (t.fh[4] & 0xff) | (t.fh[5] & 0xff) << 8 | (t.fh[6] & 0xff) << 16 | (t.fh[7] & 0xff) << 24;
    P.gx = sx - 3; P.gy = sy - 3;
    P.fsh = t.fsh; P.hsh = t.fsh - ib; P.hrnd = (1 << P.hsh) >> 1;
    // is every sample (and every aligned word) the block's items read inside the reference plane? The window is always the
    // 8-tap one (w + 7) x (h + 7): samples under the zero taps of an identity / 4-tap / bilinear filter are read, not used
    constexpr int PPW = HBD ? 2 : 4;
    const int nc = w + 7, nr = h + 7;
    bool in = !(P.S.rs & (PPW - 1)) && !(((uintptr_t)P.S.ref) & 3) && P.gx >= 0 && P.gy >= 0 && P.gx + nc <= P.S.rw && P.gy + nr <= P.S.rh;
    // the realigning loads read whole words: from the word holding the first tap to one word past the one holding the last
    // tap; all of it must lie inside the row's pitch (the bottom row has nothing behind it to run into)
    if (in) in = (P.gx & ~(PPW - 1)) + ((nc + (P.gx & (PPW - 1)) + PPW - 1) & ~(PPW - 1)) + PPW <= P.S.rs;
    P.interior = in;
}

// the aligned words (or, outside the plane interior, the clamped samples packed the same way) of window row `row` that
// the horizontal filter of column b0 needs: loaded for a whole group of rows before any of them is filtered, so that a
// lane has 8 rows of loads in flight (the row-at-a-time form stalled mostly on outstanding global loads)
template <bool HBD> struct McRowWords { unsigned w[HBD ? 5 : 3]; };

template <bool HBD, bool INTERIOR>
B200_DEV void mc_load_row(McRowWords<HBD> &W, const McPred<HBD> &P, const unsigned char *ip, const int rsb, const int row, const int b0)
{
    typedef typename Bd<HBD>::pixel pixel;
    if constexpr (INTERIOR) {
        const unsigned *wp = (const unsigned *)(ip + (ptrdiff_t)row * rsb);
#pragma unroll
        for (int k = 0; k < (HBD ? 5 : 3); k++) W.w[k] = wp[k];
    } else {
        // per-sample loads clamped to the plane = dav1d's emu_edge (reference src/mc_tmpl.c:868-916) folded in
        const pixel *rp = P.S.ref + (ptrdiff_t)iclip(P.gy + row, 0, P.S.rh - 1) * P.S.rs;
        unsigned p[8];
#pragma unroll
        for (int k = 0; k < 8; k++) p[k] = rp[iclip(b0 + k, 0, P.S.rw - 1)];
        if constexpr (!HBD) { W.w[0] = p[0] | p[1] << 8 | p[2] << 16 | p[3] << 24; W.w[1] = p[4] | p[5] << 8 | p[6] << 16 | p[7] << 24; W.w[2] = 0; }
        else { W.w[0] = p[0] | p[1] << 16; W.w[1] = p[2] | p[3] << 16; W.w[2] = p[4] | p[5] << 16; W.w[3] = p[6] | p[7] << 16; W.w[4] = 0; }
    }
}

// horizontal filter of one loaded row: realign (al = bit offset of the first tap inside the first word; 0 for the packed
// samples of the clamped form), 2 dp4a / 4 dp2a, rounding shift
template <bool HBD>
B200_DEV int mc_hfilter(const McRowWords<HBD> &W, const McPred<HBD> &P, const unsigned al)
{
    if constexpr (!HBD) {
        const unsigned lo = __funnelshift_r(W.w[0], W.w[1], al), hi = __funnelshift_r(W.w[1], W.w[2], al);
        return dp4a_us(hi, P.fh_hi, dp4a_us(lo, P.fh_lo, P.hrnd)) >> P.hsh;
    } else {
        const unsigned a0 = __funnelshift_r(W.w[0], W.w[1], al), a1 = __funnelshift_r(W.w[1], W.w[2], al);
        const unsigned a2 = __funnelshift_r(W.w[2], W.w[3], al), a3 = __funnelshift_r(W.w[3], W.w[4], al);
        int acc = dp2a_us<false>(a0, P.fh_lo, P.hrnd);
        acc = dp2a_us<true>(a1, P.fh_lo, acc);
        acc = dp2a_us<false>(a2, P.fh_hi, acc);
        acc = dp2a_us<true>(a3, P.fh_hi, acc);
        return acc >> P.hsh;
    }
}

// The rolling vertical filter of NP predictions in lockstep (1: put / prep, 2: compound). emit(j, v[NP]) receives the
// complete vertical sums of output row y0 + j, j = 0 .. R - 1 in order. Window row r (r = 0 .. R + 6) feeds output j = r - k
// with tap k; output j lives in accumulator j & 7 until row j + 7 has been added. Rows are processed in groups whose
// loads are all issued first: the 7 rows before the first output, then RG = min(R, 8) rows per group.
template <bool HBD, bool INTERIOR, int NP, int RG, class Emit>
B200_DEV void mc_item_roll(const McPred<HBD> (&P)[NP], const int x, const int y0, const int R, Emit emit)
{
    constexpr int PX = HBD ? 2 : 1, PPW = HBD ? 2 : 4;
    const unsigned char *ip[NP]; int rsb[NP], b0[NP]; unsigned al[NP];
    int acc[NP][8];
#pragma unroll
    for (int n = 0; n < NP; n++) {
        rsb[n] = P[n].S.rs * PX;
        b0[n] = P[n].gx + x;
        ip[n] = (const unsigned char *)P[n].S.ref + (ptrdiff_t)(P[n].gy + y0) * rsb[n] + (b0[n] & ~(PPW - 1)) * PX;
        al[n] = INTERIOR ? (b0[n] & (PPW - 1)) * (HBD ? 16 : 8) : 0;
    }
    {   // rows 0 .. 6: no output completes yet
        McRowWords<HBD> W[NP][7];
#pragma unroll
        for (int r = 0; r < 7; r++)
#pragma unroll
            for (int n = 0; n < NP; n++) mc_load_row<HBD, INTERIOR>(W[n][r], P[n], ip[n], rsb[n], INTERIOR ? r : y0 + r, b0[n]);
#pragma unroll
        for (int r = 0; r < 7; r++)
#pragma unroll
            for (int n = 0; n < NP; n++) {
                const int m = mc_hfilter<HBD>(W[n][r], P[n], al[n]);
                acc[n][r] = P[n].fv[0] * m;
#pragma unroll
                for (int k = 1; k <= r; k++) acc[n][r - k] += P[n].fv[k] * m;
            }
    }
    // rows 7 .. R + 6, RG per trip (R is a multiple of RG): row 7 + 8 g + i completes output 8 g + i, held in accumulator i
    for (int rb = 7; rb < R + 7; rb += RG) {
        McRowWords<HBD> W[NP][RG];
#pragma unroll
        for (int i = 0; i < RG; i++)
#pragma unroll
            for (int n = 0; n < NP; n++) mc_load_row<HBD, INTERIOR>(W[n][i], P[n], ip[n], rsb[n], INTERIOR ? rb + i : y0 + rb + i, b0[n]);
#pragma unroll
        for (int i = 0; i < RG; i++) {
            int v[NP];
#pragma unroll
            for (int n = 0; n < NP; n++) {
                const int m = mc_hfilter<HBD>(W[n][i], P[n], al[n]);
#pragma unroll
                for (int k = 1; k < 8; k++) acc[n][(7 + i - k) & 7] += P[n].fv[k] * m;
                v[n] = acc[n][i];                                  // output rb + i - 7: all eight taps are in
                acc[n][(7 + i) & 7] = P[n].fv[0] * m;              // output rb + i starts in the slot output rb + i - 8 left long ago
            }
            emit(rb + i - 7, v);
        }
    }
}

// run-time item height -> group size (R is a power of two)
template <bool HBD, bool INTERIOR, int NP, class Emit>
B200_DEV void mc_item_roll_any(const McPred<HBD> (&P)[NP], const int x, const int y0, const int R, Emit emit)
{
    if (R >= 8) mc_item_roll<HBD, INTERIOR, NP, 8>(P, x, y0, R, emit);
    else if (R == 4) mc_item_roll<HBD, INTERIOR, NP, 4>(P, x, y0, R, emit);
    else if (R == 2) mc_item_roll<HBD, INTERIOR, NP, 2>(P, x, y0, R, emit);
    else mc_item_roll<HBD, INTERIOR, NP, 1>(P, x, y0, R, emit);
}

// final rounding of one output (reference src/mc_tmpl.c: put / prep after the second pass)
B200_DEV int mc_finish(const int v, const int fsh, const int ib, const int bias, const int bdmax, const bool is_prep)
{
    return is_prep ? RND_SH(v, fsh) - bias : iclip(RND_SH(v, fsh + ib), 0, bdmax);
}

// rows of an item: as many as still give every lane an item (an item costs ~20 instructions per source row, R + 7 of
// them, + ~5 per output; idle lanes cost the same as busy ones), a power of two that divides the height
B200_DEV int mc_item_rows(int w, int h)
{
    int R = imin(32, imax(1, (w * h) >> 5));
    R = 1 << (31 - __clz(R));
    while (h & (R - 1)) R >>= 1;        // whole items only (h is 2^k, or 12 / 24 for OBMC neighbour predictions)
    return R;
}

template <bool HBD, bool INTERIOR>
B200_DEV void mc_block_items(const McPred<HBD> (&P)[1], const int lane, const int w, const int h, const int ib, const int bias,
                             const int bdmax, const McOut &o)
{
    typedef typename Bd<HBD>::pixel pixel;
    const int R = mc_item_rows(w, h);
    const int items = w * (h / R);
    const unsigned magic_w = recip16(w);                               // exact it / w: w is 2^k, 12 or 24 and it < 8192
    for (int it = lane; it < items; it += 32) {
        const int g = (int)(((unsigned)it * magic_w) >> 16), x = it - g * w, y0 = g * R;
        mc_item_roll_any<HBD, INTERIOR, 1>(P, x, y0, R, [&](const int j, const int (&v)[1]) {
            const int out = mc_finish(v[0], P[0].fsh, ib, bias, bdmax, o.is_prep);
            if (o.is_prep) o.tmp[(y0 + j) * o.tw + x] = (int16_t)out;
            else ((pixel *)o.px)[(ptrdiff_t)(y0 + j) * o.ds + x] = (pixel)out;
        });
    }
}

template <bool HBD>
__global__ void __launch_bounds__(kMcWarps * 32, B200_MC_MINB)
mc_pred_kernel(const B200McBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bi = blockIdx.x * kMcWarps + warp;
    if (bi >= n_blocks) return;
    const B200McBlock b = blocks[bi];
    const int w = b.w, h = b.h, pl = b.plane;
    const int ib = inter_bits<HBD>(bdmax);
    const int bias = HBD ? 8192 : 0;
    McPred<HBD> P[1];
    mc_pred_setup<HBD>(P[0], fr, b.ref, pl, b.filter2d, b.mx, b.my, w, h, b.src_x, b.src_y, ib);
    // op 2: "put" into the dense pixel scratch (pitch w) that the blend stages read (OBMC neighbour predictions)
    McOut o;
    o.is_prep = b.op == 1;
    o.px = (b.op == 2 ? (pixel *)fr.px_tmp : (pixel *)fr.dst) + b.dst_off;
    o.ds = b.op == 2 ? w : fr.dst_stride[pl];
    o.tmp = fr.tmp + b.dst_off; o.tw = w;
    if (P[0].interior) mc_block_items<HBD, true>(P, lane, w, h, ib, bias, bdmax, o);
    else mc_block_items<HBD, false>(P, lane, w, h, ib, bias, bdmax, o);
}

// ---- fused compound prediction -----------------------------------------------------------------------
// Both predictions of a compound block and their combination in one pass: the two rolling filters run in lockstep, so
// the two int16-precision values of an output row are complete together and are combined on the spot (avg / w_avg /
// mask / w_mask, reference src/mc_tmpl.c:628-781) — no int16 round trip through mc.tmp (2 x 2 bytes written and read
// back per sample) and no separate compound launch. Same arithmetic as prep + compound: bit-identical.
// w_mask sums the mask over horizontal pairs (neighbouring lanes: one shuffle) and, for 4:2:0, row pairs (same lane,
// consecutive outputs).
template <bool HBD, bool INTERIOR>
B200_DEV void mc_comp_fused_items(const McPred<HBD> (&P)[2], const int lane, const B200CompFusedBlock &b, const int ib,
                                  const int bias, const int bdmax, typename Bd<HBD>::pixel *dpx, const int ds, uint8_t *mask)
{
    typedef typename Bd<HBD>::pixel pixel;
    const int w = b.w, h = b.h, op = b.op;
    int R = mc_item_rows(w, h);
    if (op == B200_COMP_W_MASK_420 && R < 2) R = 2;       // row pairs stay inside an item (h is even)
    const int items = w * (h / R);
    const unsigned magic_w = recip16(w);
    const int bitdepth = 32 - __clz(bdmax);
    const int ss_hor = op >= B200_COMP_W_MASK_422, ss_ver = op == B200_COMP_W_MASK_420;
    const int sign = b.param, wt = b.param;
    const int shc = ib + 6, rnd = (32 << ib) + bias * 64;
    const int mask_sh = bitdepth + ib - 4, mask_rnd = 1 << (mask_sh - 5);
    const int mw = ss_hor ? w >> 1 : w;                                // pitch of an emitted mask
    for (int it0 = 0; it0 < items; it0 += 32) {
        const bool active = it0 + lane < items;
        const int it = active ? it0 + lane : items - 1;               // idle lanes of the last round redo the last item (w_mask shuffles need the whole warp)
        const int g = (int)(((unsigned)it * magic_w) >> 16), x = it - g * w, y0 = g * R;
        int m_prev = 0;
        mc_item_roll_any<HBD, INTERIOR, 2>(P, x, y0, R, [&](const int j, const int (&v)[2]) {
            const int a = mc_finish(v[0], P[0].fsh, ib, bias, bdmax, true), c = mc_finish(v[1], P[1].fsh, ib, bias, bdmax, true);
            const int y = y0 + j;
            if (op <= B200_COMP_MASK) {
                int o;
                if (op == B200_COMP_AVG) o = (a + c + (1 << ib) + bias * 2) >> (ib + 1);
                else if (op == B200_COMP_W_AVG) o = (a * wt + c * (16 - wt) + (8 << ib) + bias * 16) >> (ib + 4);
                else { const int m = mask[y * w + x]; o = (a * m + c * (64 - m) + (32 << ib) + bias * 64) >> (ib + 6); }
                if (active) dpx[(ptrdiff_t)y * ds + x] = (pixel)iclip(o, 0, bdmax);
            } else {
                // w_mask: derive the blend mask from |tmp1 - tmp2|, blend, emit the (sub-sampled) mask
                const int d = a - c;
                int m = imin(38 + ((iabs(d) + mask_rnd) >> mask_sh), 64);
                if (active) dpx[(ptrdiff_t)y * ds + x] = (pixel)iclip((d * m + c * 64 + rnd) >> shc, 0, bdmax);
                if (!ss_hor) {
                    if (active) mask[y * w + x] = (uint8_t)m;
                } else {
                    m += __shfl_xor_sync(0xffffffffu, m, 1);           // x and x ^ 1 are neighbouring lanes (w is even)
                    if (ss_ver) {
                        if (j & 1) { if (active && !(x & 1)) mask[(y >> 1) * mw + (x >> 1)] = (uint8_t)((m_prev + m + 2 - sign) >> 2); }
                        else m_prev = m;
                    } else if (active && !(x & 1)) mask[y * mw + (x >> 1)] = (uint8_t)((m + 1 - sign) >> 1);
                }
            }
        });
    }
}

template <bool HBD>
__global__ void __launch_bounds__(kMcWarps * 32, 4)          // two rings + two tap sets: 128 registers, no spills
mc_comp_fused_kernel(const B200CompFusedBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bi = blockIdx.x * kMcWarps + warp;
    if (bi >= n_blocks) return;
    const B200CompFusedBlock b = blocks[bi];
    const int w = b.w, h = b.h, pl = b.plane;
    const int ib = inter_bits<HBD>(bdmax);
    const int bias = HBD ? 8192 : 0;
    McPred<HBD> P[2];
#pragma unroll
    for (int r = 0; r < 2; r++) mc_pred_setup<HBD>(P[r], fr, b.ref[r], pl, b.filter2d, b.mx[r], b.my[r], w, h, b.src_x[r], b.src_y[r], ib);
    pixel *const dpx = (pixel *)fr.dst + b.dst_off;
    const int ds = fr.dst_stride[pl];
    uint8_t *const mask = fr.mask + b.mask_off;
    if (P[0].interior && P[1].interior) mc_comp_fused_items<HBD, true>(P, lane, b, ib, bias, bdmax, dpx, ds, mask);
    else mc_comp_fused_items<HBD, false>(P, lane, b, ib, bias, bdmax, dpx, ds, mask);
}

// ---- scaled references -----------------------------------------------------------------------------
// One CTA per block, one thread per output sample: column x reads the source at (mx + x*dx) >> 10 with the
// filter phase ((mx + x*dx) & 1023) >> 6, row y at (my + y*dy) >> 10 likewise (closed form of the reference's
// running imx / ioff, src/mc_tmpl.c:213-222); the 8 horizontally filtered rows a sample needs are computed on the
// fly (scaled prediction is rare: super-resolution / reference scaling only). Clamped loads = emu_edge.
template <bool HBD>
__global__ void __launch_bounds__(256)
mc_scaled_kernel(const B200McScaledBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const B200McScaledBlock b = blocks[blockIdx.x];
    const int w = b.w, h = b.h, pl = b.plane;
    // a reference of another size brings its own plane geometry
    const bool own = (fr.scaled_mask >> b.ref) & 1;
    const pixel *__restrict__ ref = (const pixel *)fr.ref[b.ref] + (own ? fr.ref_geom[b.ref].plane_off[pl] : fr.ref_plane_off[pl]);
    const int rs = own ? fr.ref_geom[b.ref].stride[pl] : fr.ref_stride[pl];
    const int rw1 = (own ? fr.ref_geom[b.ref].w[pl] : fr.ref_w[pl]) - 1, rh1 = (own ? fr.ref_geom[b.ref].h[pl] : fr.ref_h[pl]) - 1;
    const int ib = inter_bits<HBD>(bdmax);
    const int bias = HBD ? 8192 : 0;
    const bool bilin = b.filter2d == 9, is_prep = b.op == 1;
    const int th = bilin ? 0 : c_f2d_h[b.filter2d], tv = bilin ? 0 : c_f2d_v[b.filter2d];
    const int hidx = w > 4 ? th : 3 + (th & 1), vidx = h > 4 ? tv : 3 + (tv & 1);
    pixel *const dpx = b.op == 2 ? (pixel *)fr.px_tmp : (pixel *)fr.dst;      // op 2: the overlapped predictions of OBMC
    const int ds = b.op == 2 ? w : fr.dst_stride[pl];
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int y = i / w, x = i - y * w;
        const int px = b.mx + x * b.dx, py = b.my + y * b.dy;
        const int sx = b.src_x + (px >> 10), sy = b.src_y + (py >> 10);
        int out;
        if (bilin) {
            const int fx = (px & 0x3ff) >> 6, fy = (py & 0x3ff) >> 6;
            int m[2];
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const pixel *row = ref + (ptrdiff_t)iclip(sy + r, 0, rh1) * rs;
                const int p0 = row[iclip(sx, 0, rw1)], p1 = row[iclip(sx + 1, 0, rw1)];
                m[r] = RND_SH(16 * p0 + fx * (p1 - p0), 4 - ib);
            }
            const int s = 16 * m[0] + fy * (m[1] - m[0]);
            out = is_prep ? RND_SH(s, 4) - bias : iclip(RND_SH(s, 4 + ib), 0, bdmax);
        } else {
            const int fx = (px & 0x3ff) >> 6, fy = (py & 0x3ff) >> 6;
            int mid[8];
#pragma unroll
            for (int r = 0; r < 8; r++) {
                if (!fy && r != 3) { mid[r] = 0; continue; }
                const pixel *row = ref + (ptrdiff_t)iclip(sy + r - 3, 0, rh1) * rs;
                if (fx) {
                    int sacc = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) sacc += b200_mc_subpel_filters[hidx][fx - 1][k] * (int)row[iclip(sx + k - 3, 0, rw1)];
                    mid[r] = RND_SH(sacc, 6 - ib);
                } else {
                    mid[r] = (int)row[iclip(sx, 0, rw1)] << ib;
                }
            }
            if (fy) {
                int sacc = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) sacc += b200_mc_subpel_filters[vidx][fy - 1][k] * mid[k];
                out = is_prep ? RND_SH(sacc, 6) - bias : iclip(RND_SH(sacc, 6 + ib), 0, bdmax);
            } else {
                out = is_prep ? mid[3] - bias : iclip((mid[3] + ((1 << ib) >> 1)) >> ib, 0, bdmax);
            }
        }
        if (is_prep) fr.tmp[b.dst_off + y * w + x] = (int16_t)out;
        else dpx[b.dst_off + (ptrdiff_t)y * ds + x] = (pixel)out;
    }
}

// ---------------------------------------------------------------------------------------
template <bool HBD>
__global__ void __launch_bounds__(128)
mc_comp_kernel(const B200CompBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const B200CompBlock b = blocks[blockIdx.x];
    const int w = b.w, h = b.h, op = b.op;
    const int ib = inter_bits<HBD>(bdmax);
    const int bias = HBD ? 8192 : 0;
    const int16_t *__restrict__ t1 = fr.tmp + b.tmp1_off;
    const int16_t *__restrict__ t2 = fr.tmp + b.tmp2_off;
    pixel *const dst = (pixel *)fr.dst + b.dst_off;
    const int ds = fr.dst_stride[b.plane];
    uint8_t *const mask = fr.mask + b.mask_off;

    if (op <= B200_COMP_MASK) {
        // two horizontally adjacent samples per thread: one 32-bit load per int16 source when the block is 2-aligned
        const int qw = w >> 1, qsh = 31 - __clz(qw);
        const bool pow2 = (qw & (qw - 1)) == 0;
        const bool vec = !((b.tmp1_off | b.tmp2_off) & 1u);
        const bool vst = !((b.dst_off | (unsigned)ds) & 1u);
        const int wt = b.param;
        for (int i = threadIdx.x; i < qw * h; i += blockDim.x) {
            const int y = pow2 ? i >> qsh : i / qw, x = (i - y * qw) * 2;
            int a[2], c[2], v[2];
            if (vec) {
                const unsigned ua = *(const unsigned *)(t1 + 2 * i), uc = *(const unsigned *)(t2 + 2 * i);
                a[0] = (int16_t)(ua & 0xffff); a[1] = (int)ua >> 16; c[0] = (int16_t)(uc & 0xffff); c[1] = (int)uc >> 16;
            } else {
                a[0] = t1[2 * i]; a[1] = t1[2 * i + 1]; c[0] = t2[2 * i]; c[1] = t2[2 * i + 1];
            }
#pragma unroll
            for (int k = 0; k < 2; k++) {
                if (op == B200_COMP_AVG) {
                    v[k] = (a[k] + c[k] + (1 << ib) + bias * 2) >> (ib + 1);
                } else if (op == B200_COMP_W_AVG) {
                    v[k] = (a[k] * wt + c[k] * (16 - wt) + (8 << ib) + bias * 16) >> (ib + 4);
                } else {
                    const int m = mask[2 * i + k];
                    v[k] = (a[k] * m + c[k] * (64 - m) + (32 << ib) + bias * 64) >> (ib + 6);
                }
                v[k] = iclip(v[k], 0, bdmax);
            }
            pixel *o = dst + (ptrdiff_t)y * ds + x;
            if (vst) {
                if (HBD) *(unsigned *)o = (unsigned)v[0] | (unsigned)v[1] << 16;
                else *(uint16_t *)o = (uint16_t)(v[0] | v[1] << 8);
            } else { o[0] = (pixel)v[0]; o[1] = (pixel)v[1]; }
        }
        return;
    }
    // w_mask: derive the blend mask from |tmp1 - tmp2|, blend, and emit the (sub-sampled) mask
    const int ss_hor = op != B200_COMP_W_MASK_444, ss_ver = op == B200_COMP_W_MASK_420;
    const int sign = b.param;
    const int bitdepth = 32 - __clz(bdmax);
    const int sh = ib + 6, rnd = (32 << ib) + bias * 64;
    const int mask_sh = bitdepth + ib - 4, mask_rnd = 1 << (mask_sh - 5);
    const int qw = w >> 1, qh = ss_ver ? h >> 1 : h;       // work items: 2 px wide, 1 or 2 rows tall
    for (int i = threadIdx.x; i < qw * qh; i += blockDim.x) {
        const int qy = i / qw, qx = i - qy * qw;
        const int x = qx * 2;
        int msum = 0;
        for (int r = 0; r <= ss_ver; r++) {
            const int y = ss_ver ? qy * 2 + r : qy;
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const int idx = y * w + x + k;
                const int c = t2[idx], d = t1[idx] - c;
                const int m = imin(38 + ((iabs(d) + mask_rnd) >> mask_sh), 64);
                dst[(ptrdiff_t)y * ds + x + k] = (pixel)iclip((d * m + c * 64 + rnd) >> sh, 0, bdmax);
                if (!ss_hor) mask[idx] = (uint8_t)m;
                msum += m;
            }
        }
        if (ss_ver)      mask[qy * qw + qx] = (uint8_t)((msum + 2 - sign) >> 2);
        else if (ss_hor) mask[qy * qw + qx] = (uint8_t)((msum + 1 - sign) >> 1);
    }
}

template <bool HBD>
__global__ void __launch_bounds__(128)
mc_blend_kernel(const B200BlendBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const B200BlendBlock b = blocks[blockIdx.x];
    const int w = b.w, h = b.h, op = b.op;
    pixel *const dst = (pixel *)fr.dst + b.dst_off;
    const pixel *__restrict__ tmp = (const pixel *)fr.px_tmp + b.tmp_off;
    const int ds = fr.dst_stride[b.plane];
    const int bw = op == B200_BLEND_V ? (w * 3) >> 2 : w;
    const int bh = op == B200_BLEND_H ? (h * 3) >> 2 : h;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
        const int y = i / bw, x = i - y * bw;
        int m;
        if (op == B200_BLEND) m = fr.mask[b.mask_off + y * w + x];
        else if (op == B200_BLEND_V) m = b200_obmc_masks[w + x];
        else m = b200_obmc_masks[h + y];
        pixel *p = dst + (ptrdiff_t)y * ds + x;
        *p = (pixel)(((int)*p * (64 - m) + (int)tmp[y * w + x] * m + 32) >> 6);
    }
}

// one warp per 8x8 block; the 15x8 horizontally filtered rows go through shared memory
constexpr int kWarpWarps = 4;
template <bool HBD>
__global__ void __launch_bounds__(kWarpWarps * 32)
mc_warp_kernel(const B200WarpBlock *__restrict__ blocks, int n_blocks, const __grid_constant__ B200McFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    __shared__ int mid[kWarpWarps][15 * 8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bi = blockIdx.x * kWarpWarps + warp;
    const bool valid = bi < n_blocks;
    B200WarpBlock b;
    if (valid) b = blocks[bi]; else { b = blocks[0]; }
    const int pl = b.plane;
    const pixel *__restrict__ ref = (const pixel *)fr.ref[b.ref] + fr.ref_plane_off[pl];
    const int rs = fr.ref_stride[pl], rw1 = fr.ref_w[pl] - 1, rh1 = fr.ref_h[pl] - 1;
    const int ib = inter_bits<HBD>(bdmax);
    const int bias = HBD ? 8192 : 0;
    if (valid) {
        for (int i = lane; i < 15 * 8; i += 32) {
            const int y = i >> 3, x = i & 7;
            const int tmx = b.mx + y * b.abcd[1] + x * b.abcd[0];
            const int8_t *f = b200_mc_warp_filter[64 + ((tmx + 512) >> 10)];
            const pixel *row = ref + (ptrdiff_t)iclip(b.src_y + y - 3, 0, rh1) * rs;
            int s = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) s += f[k] * (int)row[iclip(b.src_x + x + k - 3, 0, rw1)];
            mid[warp][i] = RND_SH(s, 7 - ib);
        }
    }
    __syncwarp();
    if (valid) {
        for (int i = lane; i < 64; i += 32) {
            const int y = i >> 3, x = i & 7;
            const int tmy = b.my + y * b.abcd[3] + x * b.abcd[2];
            const int8_t *f = b200_mc_warp_filter[64 + ((tmy + 512) >> 10)];
            int s = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) s += f[k] * mid[warp][(y + k) * 8 + x];
            if (b.op) fr.tmp[b.dst_off + y * b.tmp_stride + x] = (int16_t)(RND_SH(s, 7) - bias);
            else ((pixel *)fr.dst)[b.dst_off + (ptrdiff_t)y * fr.dst_stride[pl] + x] =
                     (pixel)iclip(RND_SH(s, 7 + ib), 0, bdmax);
        }
    }
}

template <bool HBD>
__global__ void emu_edge_kernel(int bw, int bh, int iw, int ih, int x0, int y0,
                                typename Bd<HBD>::pixel *dst, const typename Bd<HBD>::pixel *ref)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < bw * bh; i += gridDim.x * blockDim.x) {
        const int y = i / bw, x = i - y * bw;
        dst[i] = ref[iclip(y0 + y, 0, ih - 1) * iw + iclip(x0 + x, 0, iw - 1)];
    }
}

// whole planes, strided (the frame job's super-resolution stage): one thread per output sample, grid.y = plane.
// The x position recurrence (mx += dx; src_x += mx >> 14; mx &= 0x3fff) has the closed form below.
template <bool HBD>
__global__ void __launch_bounds__(256) resize_frame_kernel(const __grid_constant__ B200ResizeFrame fr, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int pl = blockIdx.y;
    const int dst_w = fr.dst_w[pl], src_w = fr.src_w[pl], h = fr.h[pl], dx = fr.dx[pl], mx0 = fr.mx0[pl];
    const pixel *const src = (const pixel *)fr.src + fr.src_plane_off[pl];
    pixel *const dst = (pixel *)fr.dst + fr.dst_plane_off[pl];
    const int ss = fr.src_stride[pl], ds = fr.dst_stride[pl];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < dst_w * h; i += gridDim.x * blockDim.x) {
        const int y = i / dst_w, x = i - y * dst_w;
        const long long pos = (long long)mx0 + (long long)x * dx;
        const int src_x = -1 + (int)(pos >> 14), mx = (int)(pos & 0x3fff);
        const int8_t *F = b200_resize_filter[mx >> 8];
        const pixel *const row = src + (ptrdiff_t)y * ss;
        int s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s += F[k] * (int)row[iclip(src_x - 3 + k, 0, src_w - 1)];
        dst[(ptrdiff_t)y * ds + x] = (pixel)iclip((-s + 64) >> 7, 0, bdmax);
    }
}

}  // namespace b200

// =======================================================================================
using namespace b200;

// one prediction stage of a frame: records [0, n), `per_cta` of them per CTA of `threads` threads
template <class Rec, class Kern>
static int mc_stage(const char *who, int bdmax, const B200McFrame *frame, const Rec *d_blocks, int n, int per_cta, int threads,
                    void *stream, Kern kern)
{
    if (int r = check_bdmax(bdmax, who)) return r;
    if (n <= 0) return 0;
    return launch_hbd(bdmax, Launch::pdl, dim3((n + per_cta - 1) / per_cta), dim3(threads), 0, (cudaStream_t)stream,
                      [&](auto hbd) { return std::make_tuple(kern(hbd), d_blocks, n, *frame, bdmax); });
}

extern "C" {

int b200_mc_batch(int bitdepth_max, const B200McFrame *frame, const B200McBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_batch", bitdepth_max, frame, d_blocks, n, kMcWarps, kMcWarps * 32, stream, [](auto hbd) { return mc_pred_kernel<hbd>; });
}
int b200_mc_scaled_batch(int bitdepth_max, const B200McFrame *frame, const B200McScaledBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_scaled_batch", bitdepth_max, frame, d_blocks, n, 1, 256, stream, [](auto hbd) { return mc_scaled_kernel<hbd>; });
}
int b200_mc_comp_fused_batch(int bitdepth_max, const B200McFrame *frame, const B200CompFusedBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_comp_fused_batch", bitdepth_max, frame, d_blocks, n, kMcWarps, kMcWarps * 32, stream, [](auto hbd) { return mc_comp_fused_kernel<hbd>; });
}
int b200_mc_comp_batch(int bitdepth_max, const B200McFrame *frame, const B200CompBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_comp_batch", bitdepth_max, frame, d_blocks, n, 1, 128, stream, [](auto hbd) { return mc_comp_kernel<hbd>; });
}
int b200_mc_blend_batch(int bitdepth_max, const B200McFrame *frame, const B200BlendBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_blend_batch", bitdepth_max, frame, d_blocks, n, 1, 128, stream, [](auto hbd) { return mc_blend_kernel<hbd>; });
}
int b200_mc_warp_batch(int bitdepth_max, const B200McFrame *frame, const B200WarpBlock *d_blocks, int n, void *stream) {
    return mc_stage("b200_mc_warp_batch", bitdepth_max, frame, d_blocks, n, kWarpWarps, kWarpWarps * 32, stream, [](auto hbd) { return mc_warp_kernel<hbd>; });
}

}  // extern "C"

// ---- Level 1: host pointers -------------------------------------------------------------
enum { REF, DST, TMP, MASK, DESC };   // Level1 scratch slots

static int mc_l1(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride, int w, int h,
                 int mx, int my, int f2d, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc")) return r;
    if (f2d < 0 || f2d > 9 || w < 2 || w > 128 || (w & (w - 1)) || h < 2 || h > 128 || mx < 0 || mx > 15 || my < 0 || my > 15) {
        b200_set_error("b200_mc: bad arguments (w=%d h=%d mx=%d my=%d filter=%d)", w, h, mx, my, f2d);
        return -2;
    }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    // the window the reference reads: 3 before / 4 after for 8-tap, 0 / 1 for bilinear, only on filtered axes
    const int bl = f2d == 9 ? 0 : 3, al = f2d == 9 ? 1 : 4;
    const int x0 = mx ? bl : 0, x1 = mx ? al : 0, y0 = my ? bl : 0, y1 = my ? al : 0;
    const int ww = w + x0 + x1, wh = h + y0 + y1;
    B200McBlock b;
    memset(&b, 0, sizeof(b));
    b.dst_off = 0; b.src_x = x0; b.src_y = y0; b.w = (uint8_t)w; b.h = (uint8_t)h; b.mx = (uint8_t)mx; b.my = (uint8_t)my;
    b.filter2d = (uint8_t)f2d; b.op = (uint8_t)op;
    void *ref, *dst, *desc;
    if (!(ref = L.upload_rect(REF, (const uint8_t *)src - (ptrdiff_t)y0 * src_stride - (ptrdiff_t)x0 * (ptrdiff_t)px, src_stride, ww, wh, px)) ||
        !(dst = L.dev(DST, (size_t)w * h * 2)) || !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    B200McFrame fr;
    memset(&fr, 0, sizeof(fr));
    fr.ref[0] = ref; fr.ref_stride[0] = ww; fr.ref_w[0] = ww; fr.ref_h[0] = wh;
    fr.dst = dst; fr.dst_stride[0] = w; fr.tmp = (int16_t *)dst;
    if (int r = b200_mc_batch(bdmax, &fr, (const B200McBlock *)desc, 1, 0)) return r;
    return op ? L.download_rect(DST, out, (ptrdiff_t)w * 2, w, h, 2) : L.download_rect(DST, out, out_stride, w, h, px);
}

static int mc_scaled_l1(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride, int w, int h,
                        int mx, int my, int dx, int dy, int f2d, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_scaled")) return r;
    if (f2d < 0 || f2d > 9 || w < 2 || w > 128 || h < 2 || h > 128 || mx < 0 || mx > 1023 || my < 0 || my > 1023 ||
        dx < 1 || dx > 2048 || dy < 1 || dy > 2048) {
        b200_set_error("b200_mc_scaled: bad arguments (w=%d h=%d mx=%d my=%d dx=%d dy=%d filter=%d)", w, h, mx, my, dx, dy, f2d);
        return -2;
    }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    // the window the reference reads (8-tap: 3 before / 4 after the integer position; bilinear: 0 / 1)
    const int bl = f2d == 9 ? 0 : 3, al = f2d == 9 ? 1 : 4;
    const int ww = ((mx + (w - 1) * dx) >> 10) + 1 + bl + al, wh = ((my + (h - 1) * dy) >> 10) + 1 + bl + al;
    B200McScaledBlock b;
    memset(&b, 0, sizeof(b));
    b.src_x = bl; b.src_y = bl; b.w = (uint8_t)w; b.h = (uint8_t)h; b.mx = (uint16_t)mx; b.my = (uint16_t)my;
    b.dx = (uint16_t)dx; b.dy = (uint16_t)dy; b.filter2d = (uint8_t)f2d; b.op = (uint8_t)op;
    void *ref, *dst, *desc;
    if (!(ref = L.upload_rect(REF, (const uint8_t *)src - (ptrdiff_t)bl * src_stride - (ptrdiff_t)bl * (ptrdiff_t)px, src_stride, ww, wh, px)) ||
        !(dst = L.dev(DST, (size_t)w * h * 2)) || !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    B200McFrame fr;
    memset(&fr, 0, sizeof(fr));
    fr.ref[0] = ref; fr.ref_stride[0] = ww; fr.ref_w[0] = ww; fr.ref_h[0] = wh;
    fr.dst = dst; fr.dst_stride[0] = w; fr.tmp = (int16_t *)dst;
    if (int r = b200_mc_scaled_batch(bdmax, &fr, (const B200McScaledBlock *)desc, 1, 0)) return r;
    return op ? L.download_rect(DST, out, (ptrdiff_t)w * 2, w, h, 2) : L.download_rect(DST, out, out_stride, w, h, px);
}

extern "C" {

int b200_mc_put_scaled(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int w, int h,
                       int mx, int my, int dx, int dy, int filter2d, int bitdepth_max) {
    return mc_scaled_l1(0, dst, dst_stride, src, src_stride, w, h, mx, my, dx, dy, filter2d, bitdepth_max);
}
int b200_mc_prep_scaled(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h, int mx, int my,
                        int dx, int dy, int filter2d, int bitdepth_max) {
    return mc_scaled_l1(1, tmp, 0, src, src_stride, w, h, mx, my, dx, dy, filter2d, bitdepth_max);
}

int b200_mc_put(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int w, int h,
                int mx, int my, int filter2d, int bitdepth_max) {
    return mc_l1(0, dst, dst_stride, src, src_stride, w, h, mx, my, filter2d, bitdepth_max);
}
int b200_mc_prep(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h, int mx, int my,
                 int filter2d, int bitdepth_max) {
    return mc_l1(1, tmp, 0, src, src_stride, w, h, mx, my, filter2d, bitdepth_max);
}

int b200_mc_comp(void *dst, ptrdiff_t dst_stride, const int16_t *tmp1, const int16_t *tmp2, int w, int h,
                 int op, int param, uint8_t *mask, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_comp")) return r;
    if (op < 0 || op > B200_COMP_W_MASK_420 || w < 4 || w > 128 || h < 4 || h > 128 || (w & 1) || (op == B200_COMP_W_MASK_420 && (h & 1))) {
        b200_set_error("b200_mc_comp: bad arguments (op=%d w=%d h=%d)", op, w, h);
        return -2;
    }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1, n = (size_t)w * h;
    B200CompBlock b;
    memset(&b, 0, sizeof(b));
    b.tmp1_off = 0; b.tmp2_off = (uint32_t)n; b.w = (uint8_t)w; b.h = (uint8_t)h; b.op = (uint8_t)op; b.param = (uint8_t)param;
    int16_t *both = (int16_t *)L.host(n * 4);     // tmp1 and tmp2 back to back
    if (!both) return -1;
    memcpy(both, tmp1, n * 2);
    memcpy(both + n, tmp2, n * 2);
    void *tmp, *out, *m, *desc;
    if (!(tmp = L.upload(TMP, both, n * 4)) || !(out = L.dev(DST, n * 2)) ||
        !(m = op == B200_COMP_MASK ? L.upload(MASK, mask, n) : L.dev(MASK, n)) || !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    B200McFrame fr;
    memset(&fr, 0, sizeof(fr));
    fr.dst = out; fr.dst_stride[0] = w; fr.tmp = (int16_t *)tmp; fr.mask = (uint8_t *)m;
    if (int r = b200_mc_comp_batch(bdmax, &fr, (const B200CompBlock *)desc, 1, 0)) return r;
    if (op >= B200_COMP_W_MASK_444 && L.download(MASK, mask, (size_t)(w >> (op != B200_COMP_W_MASK_444)) * (h >> (op == B200_COMP_W_MASK_420))))
        return -1;
    return L.download_rect(DST, dst, dst_stride, w, h, px);
}

int b200_mc_blend(void *dst, ptrdiff_t dst_stride, const void *tmp, int w, int h, int op, const uint8_t *mask, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_blend")) return r;
    if (op < 0 || op > B200_BLEND_H || w < 1 || w > 128 || h < 1 || h > 128) { b200_set_error("b200_mc_blend: bad arguments"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1, n = (size_t)w * h;
    B200BlendBlock b;
    memset(&b, 0, sizeof(b));
    b.w = (uint8_t)w; b.h = (uint8_t)h; b.op = (uint8_t)op;
    void *out, *t, *m = nullptr, *desc;
    if (!(out = L.upload_rect(DST, dst, dst_stride, w, h, px)) || !(t = L.upload(TMP, tmp, n * px)) ||
        (op == B200_BLEND && !(m = L.upload(MASK, mask, n))) || !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    B200McFrame fr;
    memset(&fr, 0, sizeof(fr));
    fr.dst = out; fr.dst_stride[0] = w; fr.px_tmp = t; fr.mask = (uint8_t *)m;
    if (int r = b200_mc_blend_batch(bdmax, &fr, (const B200BlendBlock *)desc, 1, 0)) return r;
    return L.download_rect(DST, dst, dst_stride, w, h, px);
}

int b200_mc_warp8x8(int op, void *out, ptrdiff_t out_stride, const void *src, ptrdiff_t src_stride,
                    const int16_t *abcd, int mx, int my, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_warp8x8")) return r;
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    B200WarpBlock b;
    memset(&b, 0, sizeof(b));
    b.src_x = 3; b.src_y = 3; b.mx = mx; b.my = my; b.op = (uint8_t)op; b.tmp_stride = 8;
    memcpy(b.abcd, abcd, 8);
    void *ref, *dst, *desc;
    if (!(ref = L.upload_rect(REF, (const uint8_t *)src - 3 * src_stride - 3 * (ptrdiff_t)px, src_stride, 15, 15, px)) ||
        !(dst = L.dev(DST, 64 * 2)) || !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    B200McFrame fr;
    memset(&fr, 0, sizeof(fr));
    fr.ref[0] = ref; fr.ref_stride[0] = 15; fr.ref_w[0] = 15; fr.ref_h[0] = 15;
    fr.dst = dst; fr.dst_stride[0] = 8; fr.tmp = (int16_t *)dst;
    if (int r = b200_mc_warp_batch(bdmax, &fr, (const B200WarpBlock *)desc, 1, 0)) return r;
    return op ? L.download_rect(DST, out, out_stride * 2, 8, 8, 2) : L.download_rect(DST, out, out_stride, 8, 8, px);
}

int b200_mc_emu_edge(intptr_t bw, intptr_t bh, intptr_t iw, intptr_t ih, intptr_t x, intptr_t y, void *dst,
                     ptrdiff_t dst_stride, const void *ref, ptrdiff_t ref_stride, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_emu_edge")) return r;
    if (bw < 1 || bh < 1 || iw < 1 || ih < 1 || bw * bh > (1 << 22) || iw * ih > (1 << 26)) { b200_set_error("b200_mc_emu_edge: bad geometry"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    // only the part of the plane the window can touch is shipped: rows/cols clamp(x..x+bw-1)
    const int cx0 = iclip((int)x, 0, (int)iw - 1), cx1 = iclip((int)(x + bw - 1), 0, (int)iw - 1);
    const int cy0 = iclip((int)y, 0, (int)ih - 1), cy1 = iclip((int)(y + bh - 1), 0, (int)ih - 1);
    const int sw = cx1 - cx0 + 1, shh = cy1 - cy0 + 1;
    void *s, *d;
    if (!(s = L.upload_rect(REF, (const uint8_t *)ref + (ptrdiff_t)cy0 * ref_stride + (ptrdiff_t)cx0 * (ptrdiff_t)px, ref_stride, sw, shh, px)) ||
        !(d = L.dev(DST, (size_t)bw * bh * px)))
        return -1;
    const int n = (int)(bw * bh), grid = imin((n + 255) / 256, 1184);
    if (int r = launch_hbd(bdmax, Launch::plain, dim3(grid), dim3(256), 0, 0, [&](auto hbd) {
            typedef typename Bd<hbd>::pixel pixel;
            return std::make_tuple(emu_edge_kernel<hbd>, (int)bw, (int)bh, sw, shh, (int)x - cx0, (int)y - cy0, (pixel *)d, (const pixel *)s);
        }))
        return r;
    return L.download_rect(DST, dst, dst_stride, (int)bw, (int)bh, px);
}

int b200_resize_frame(int bitdepth_max, const B200ResizeFrame *fr, void *stream)
{
    if (int r = check_bdmax(bitdepth_max, "b200_resize_frame")) return r;
    if (fr->n_planes <= 0) return 0;
    if (fr->n_planes > 3 || !fr->src || !fr->dst) { b200_set_error("b200_resize_frame: bad arguments"); return -2; }
    int most = 0;
    for (int p = 0; p < fr->n_planes; p++) {
        if (fr->dst_w[p] < 1 || fr->src_w[p] < 1 || fr->h[p] < 1) { b200_set_error("b200_resize_frame: bad geometry"); return -2; }
        most = imax(most, fr->dst_w[p] * fr->h[p]);
    }
    const dim3 grid(imin((most + 255) / 256, 8 * kSmCount), fr->n_planes);
    return launch_hbd(bitdepth_max, Launch::pdl, grid, dim3(256), 0, (cudaStream_t)stream,
                      [&](auto hbd) { return std::make_tuple(resize_frame_kernel<hbd>, *fr, bitdepth_max); });
}

int b200_mc_resize(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int dst_w, int h,
                   int src_w, int dx, int mx, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_mc_resize")) return r;
    if (dst_w < 1 || h < 1 || src_w < 1 || (size_t)dst_w * h > (1u << 26)) { b200_set_error("b200_mc_resize: bad geometry"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    B200ResizeFrame fr;
    memset(&fr, 0, sizeof(fr));
    if (!(fr.src = L.upload_rect(REF, src, src_stride, src_w, h, px)) || !(fr.dst = L.dev(DST, (size_t)dst_w * h * px))) return -1;
    fr.n_planes = 1;
    fr.src_stride[0] = fr.src_w[0] = src_w; fr.dst_stride[0] = fr.dst_w[0] = dst_w; fr.h[0] = h;
    fr.dx[0] = dx; fr.mx0[0] = mx;
    // the frame entry point launches with PDL; on stream 0 after the staging copies that orders like a plain launch (as mc_l1)
    if (int r = b200_resize_frame(bdmax, &fr, 0)) return r;
    return L.download_rect(DST, dst, dst_stride, dst_w, h, px);
}

}  // extern "C"

// ---- Level-1 table: thunks with dav1d's exact signatures (reference src/mc.h:38-114) ---------
namespace {
#define DIE_IF(x, what) do { if (x) die(what); } while (0)
template <int F> void put8(uint8_t *d, ptrdiff_t ds, const uint8_t *s, ptrdiff_t ss, int w, int h, int mx, int my) { DIE_IF(b200_mc_put(d, ds, s, ss, w, h, mx, my, F, 255), "mc"); }
template <int F> void put16(uint16_t *d, ptrdiff_t ds, const uint16_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int bd) { DIE_IF(b200_mc_put(d, ds, s, ss, w, h, mx, my, F, bd), "mc"); }
template <int F> void prep8(int16_t *t, const uint8_t *s, ptrdiff_t ss, int w, int h, int mx, int my) { DIE_IF(b200_mc_prep(t, s, ss, w, h, mx, my, F, 255), "mct"); }
template <int F> void prep16(int16_t *t, const uint16_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int bd) { DIE_IF(b200_mc_prep(t, s, ss, w, h, mx, my, F, bd), "mct"); }
template <int F> void puts8(uint8_t *d, ptrdiff_t ds, const uint8_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int dx, int dy) { DIE_IF(b200_mc_put_scaled(d, ds, s, ss, w, h, mx, my, dx, dy, F, 255), "mc_scaled"); }
template <int F> void puts16(uint16_t *d, ptrdiff_t ds, const uint16_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int dx, int dy, int bd) { DIE_IF(b200_mc_put_scaled(d, ds, s, ss, w, h, mx, my, dx, dy, F, bd), "mc_scaled"); }
template <int F> void preps8(int16_t *t, const uint8_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int dx, int dy) { DIE_IF(b200_mc_prep_scaled(t, s, ss, w, h, mx, my, dx, dy, F, 255), "mct_scaled"); }
template <int F> void preps16(int16_t *t, const uint16_t *s, ptrdiff_t ss, int w, int h, int mx, int my, int dx, int dy, int bd) { DIE_IF(b200_mc_prep_scaled(t, s, ss, w, h, mx, my, dx, dy, F, bd), "mct_scaled"); }
void avg8(uint8_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_AVG, 0, nullptr, 255), "avg"); }
void avg16(uint16_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, int bd) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_AVG, 0, nullptr, bd), "avg"); }
void wavg8(uint8_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, int wt) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_W_AVG, wt, nullptr, 255), "w_avg"); }
void wavg16(uint16_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, int wt, int bd) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_W_AVG, wt, nullptr, bd), "w_avg"); }
void mask8(uint8_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, const uint8_t *m) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_MASK, 0, (uint8_t *)m, 255), "mask"); }
void mask16(uint16_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, const uint8_t *m, int bd) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_MASK, 0, (uint8_t *)m, bd), "mask"); }
template <int L> void wmask8(uint8_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, uint8_t *m, int sign) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_W_MASK_444 + L, sign, m, 255), "w_mask"); }
template <int L> void wmask16(uint16_t *d, ptrdiff_t ds, const int16_t *a, const int16_t *b, int w, int h, uint8_t *m, int sign, int bd) { DIE_IF(b200_mc_comp(d, ds, a, b, w, h, B200_COMP_W_MASK_444 + L, sign, m, bd), "w_mask"); }
template <int BD> void blend_t(void *d, ptrdiff_t ds, const void *t, int w, int h, const uint8_t *m) { DIE_IF(b200_mc_blend(d, ds, t, w, h, B200_BLEND, m, BD), "blend"); }
template <int BD> void blendv_t(void *d, ptrdiff_t ds, const void *t, int w, int h) { DIE_IF(b200_mc_blend(d, ds, t, w, h, B200_BLEND_V, nullptr, BD), "blend_v"); }
template <int BD> void blendh_t(void *d, ptrdiff_t ds, const void *t, int w, int h) { DIE_IF(b200_mc_blend(d, ds, t, w, h, B200_BLEND_H, nullptr, BD), "blend_h"); }
void warp8(uint8_t *d, ptrdiff_t ds, const uint8_t *s, ptrdiff_t ss, const int16_t *abcd, int mx, int my) { DIE_IF(b200_mc_warp8x8(0, d, ds, s, ss, abcd, mx, my, 255), "warp8x8"); }
void warp16(uint16_t *d, ptrdiff_t ds, const uint16_t *s, ptrdiff_t ss, const int16_t *abcd, int mx, int my, int bd) { DIE_IF(b200_mc_warp8x8(0, d, ds, s, ss, abcd, mx, my, bd), "warp8x8"); }
void warpt8(int16_t *t, ptrdiff_t ts, const uint8_t *s, ptrdiff_t ss, const int16_t *abcd, int mx, int my) { DIE_IF(b200_mc_warp8x8(1, t, ts, s, ss, abcd, mx, my, 255), "warp8x8t"); }
void warpt16(int16_t *t, ptrdiff_t ts, const uint16_t *s, ptrdiff_t ss, const int16_t *abcd, int mx, int my, int bd) { DIE_IF(b200_mc_warp8x8(1, t, ts, s, ss, abcd, mx, my, bd), "warp8x8t"); }
template <int BD> void emu_t(intptr_t bw, intptr_t bh, intptr_t iw, intptr_t ih, intptr_t x, intptr_t y, void *d, ptrdiff_t ds, const void *r, ptrdiff_t rs) { DIE_IF(b200_mc_emu_edge(bw, bh, iw, ih, x, y, d, ds, r, rs, BD), "emu_edge"); }
void resize8(uint8_t *d, ptrdiff_t ds, const uint8_t *s, ptrdiff_t ss, int dw, int h, int sw, int dx, int mx) { DIE_IF(b200_mc_resize(d, ds, s, ss, dw, h, sw, dx, mx, 255), "resize"); }
void resize16(uint16_t *d, ptrdiff_t ds, const uint16_t *s, ptrdiff_t ss, int dw, int h, int sw, int dx, int mx, int bd) { DIE_IF(b200_mc_resize(d, ds, s, ss, dw, h, sw, dx, mx, bd), "resize"); }

template <int... F> void fill_mc8(B200MCDSPContext *c, std::integer_sequence<int, F...>) {
    ((c->mc[F] = (void *)put8<F>, c->mct[F] = (void *)prep8<F>, c->mc_scaled[F] = (void *)puts8<F>, c->mct_scaled[F] = (void *)preps8<F>), ...);
}
template <int... F> void fill_mc16(B200MCDSPContext *c, std::integer_sequence<int, F...>) {
    ((c->mc[F] = (void *)put16<F>, c->mct[F] = (void *)prep16<F>, c->mc_scaled[F] = (void *)puts16<F>, c->mct_scaled[F] = (void *)preps16<F>), ...);
}
}  // namespace

extern "C" {
void b200_mc_dsp_init_8bpc(B200MCDSPContext *c) {
    fill_mc8(c, std::make_integer_sequence<int, B200_N_2D_FILTERS>{});
    c->avg = (void *)avg8; c->w_avg = (void *)wavg8; c->mask = (void *)mask8;
    c->w_mask[0] = (void *)wmask8<0>; c->w_mask[1] = (void *)wmask8<1>; c->w_mask[2] = (void *)wmask8<2>;
    c->blend = (void *)blend_t<255>; c->blend_v = (void *)blendv_t<255>; c->blend_h = (void *)blendh_t<255>;
    c->warp8x8 = (void *)warp8; c->warp8x8t = (void *)warpt8; c->emu_edge = (void *)emu_t<255>; c->resize = (void *)resize8;
}
void b200_mc_dsp_init_16bpc(B200MCDSPContext *c) {
    fill_mc16(c, std::make_integer_sequence<int, B200_N_2D_FILTERS>{});
    c->avg = (void *)avg16; c->w_avg = (void *)wavg16; c->mask = (void *)mask16;
    c->w_mask[0] = (void *)wmask16<0>; c->w_mask[1] = (void *)wmask16<1>; c->w_mask[2] = (void *)wmask16<2>;
    // blend*/emu_edge carry no bitdepth argument in dav1d: pixel width is all that matters (any hbd max works)
    c->blend = (void *)blend_t<1023>; c->blend_v = (void *)blendv_t<1023>; c->blend_h = (void *)blendh_t<1023>;
    c->warp8x8 = (void *)warp16; c->warp8x8t = (void *)warpt16; c->emu_edge = (void *)emu_t<1023>; c->resize = (void *)resize16;
}
}
