// The per-CTA work of the inverse transform + add, shared by the batched itx kernels (itx.cu) and the fused
// intra reconstruction kernel (intra.cu). See itx.cu for the decomposition.
#pragma once
#include "itx_1d.cuh"
#ifndef B200_TBL
#define B200_TBL __constant__
#endif
#include "tables_gen.h"
#include "../../include/b200av1.h"

namespace b200 {

// per TxfmType slot: 1-D type of the row pass (first) and of the column pass (second).
// Slot X_Y = X vertical, Y horizontal (reference src/levels.h:81-83, src/itx_tmpl.c:232-262).
static __constant__ uint8_t c_tx_first[16]  = { 0, 0, 1, 1, 0, 2, 2, 2, 1, 3, 3, 0, 3, 1, 3, 2 };
static __constant__ uint8_t c_tx_second[16] = { 0, 1, 0, 1, 2, 0, 2, 1, 2, 3, 0, 3, 1, 3, 2, 3 };
// per TxfmType slot: dav1d_tx_type_class (reference src/tables.c): 0 2-D (scan of the size), 1 H_*, 2 V_*; WHT_WHT is 2-D
static __constant__ uint8_t c_tx_class[16] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 1, 2, 1, 2, 1 };

constexpr int kItxWarps = 4;

template <int W, int H> struct ItxGeom {
    static constexpr int SW = W < 32 ? W : 32;
    static constexpr int SH = H < 32 ? H : 32;
    static constexpr int L = SH > SW ? SH : SW;          // lanes per block
    static constexpr int NB = 32 / L;                     // blocks per warp
    static constexpr int P = W + 1;                       // tile pitch (words)
    static constexpr int SLOT = SH * P;                   // words per block tile
    static constexpr int LW = W == 4 ? 0 : W == 8 ? 1 : W == 16 ? 2 : W == 32 ? 3 : 4;
    static constexpr int LSW = SW == 4 ? 2 : SW == 8 ? 3 : SW == 16 ? 4 : 5;    // log2 of the coded region's size
    static constexpr int LSH = SH == 4 ? 2 : SH == 8 ? 3 : SH == 16 ? 4 : 5;
    static constexpr bool RECT2 = (W * 2 == H) || (H * 2 == W);
    // 64-wide blocks are shared by a pair of warps: one warp runs the row pass (32 coefficient rows), then each warp
    // takes 32 of the 64 picture columns of the column pass
    static constexpr bool PAIR = W == 64;
    static constexpr int BPC = PAIR ? kItxWarps / 2 : kItxWarps * NB;   // blocks per CTA
};

// Out-of-line passes shared by every block size with the same row length W / column length H. Used by the intra
// reconstruction kernels, whose code size (every size x type inlined: 48 K instructions) thrashes the instruction cache
// once several CTAs share an SM; the batched itx kernels keep the fully inlined form.
template <int W, bool HBD>
__device__ __noinline__ void itx_row_pass_shared(const typename Bd<HBD>::coef *cfy, int sh_stride, int *trow, int rect2,
                                                 int shift, int t_first, int row_lo, int row_hi, int col_lo, int col_hi)
{
    constexpr int SW = W < 32 ? W : 32;
    int c[W];
#pragma unroll
    for (int x = 0; x < W; x++) {
        if (x < SW) {
            const int v = (int)cfy[x * sh_stride];
            c[x] = rect2 ? (int)((unsigned)v * 181u + 128u) >> 8 : v;
        } else {
            c[x] = 0;
        }
    }
    tx1d_apply<W>(c, t_first, row_lo, row_hi);
    const int rnd = (1 << shift) >> 1;
#pragma unroll
    for (int x = 0; x < W; x++) trow[x] = iclip((c[x] + rnd) >> shift, col_lo, col_hi);
}

// resid != nullptr: the residual column ((c + 8) >> 4, before the add) goes to the int16 tile `resid` (pitch `stride`)
// instead of being added to the picture column: the warp-per-block intra kernel transforms a block's coefficients
// while it is still waiting for the neighbours its prediction needs
template <int H, bool HBD>
__device__ __noinline__ void itx_col_pass_shared(const int *tcol, int pitch, typename Bd<HBD>::pixel *dcol, int stride,
                                                 int t_second, int col_lo, int col_hi, int bitdepth_max, int16_t *resid = nullptr)
{
    typedef typename Bd<HBD>::pixel pixel;
    constexpr int SH = H < 32 ? H : 32;
    int c[H];
#pragma unroll
    for (int y = 0; y < H; y++) c[y] = y < SH ? tcol[y * pitch] : 0;
    tx1d_apply<H>(c, t_second, col_lo, col_hi);
    if (resid) {
        // high bit depth: saturated, as in itx_add_warp's DC and WHT paths (|residual| >= 2^15 clips the 12-bit sum exactly
        // like the full value; 12-bit IDTX with 32-sample columns reaches (131071 * 4 + 8) >> 4 = 32768). The 8-bit column
        // clip keeps the residual within (32767 * 4 + 8) >> 4 = 8192.
#pragma unroll
        for (int y = 0; y < H; y++) {
            if constexpr (HBD) resid[y * stride] = (int16_t)iclip((c[y] + 8) >> 4, -32768, 32767);
            else resid[y * stride] = (int16_t)((c[y] + 8) >> 4);
        }
        return;
    }
#pragma unroll
    for (int y = 0; y < H; y++)
        dcol[(ptrdiff_t)y * stride] = (pixel)iclip((int)dcol[(ptrdiff_t)y * stride] + ((c[y] + 8) >> 4), 0, bitdepth_max);
}

// the work of one CTA (`cta` = its index among the CTAs of this transform size); smem: kItxWarps * NB * SLOT words
// COMPACT: `coefs` is the compact coefficient stream (per block the coefficients 0 .. eob in the scan order of its class,
// include/b200av1.h B200CoefBlock) and block bi's first value is coefs[coffs[bi]]; blk.coef_off is not read. `scan` =
// dav1d_scans[TX]. The block's coefficients are scattered into its own tile before pass 1, which then reads them from there.
template <int W, int H, int TX, int SHIFT, bool HBD, bool SHARED = false, bool COMPACT = false>
B200_DEV void itx_add_body(const int cta, int *const smem, const B200ItxBlock *__restrict__ blocks, int n_blocks,
                           typename Bd<HBD>::coef *__restrict__ coefs, typename Bd<HBD>::pixel *__restrict__ pic,
                           int stride0, int stride1, int stride2, int bitdepth_max, int zero_coefs,
                           const uint32_t *__restrict__ coffs = nullptr, const uint16_t *__restrict__ scan = nullptr)
{
    static_assert(!(SHARED && COMPACT), "the intra kernels read the dense coefficient plane");
    typedef ItxGeom<W, H> G;
    typedef typename Bd<HBD>::pixel pixel;
    typedef typename Bd<HBD>::coef coef;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = lane / G::L, li = lane % G::L;
    const int half = G::PAIR ? warp & 1 : 0;                       // which 32 columns of a 64-wide block
    const int slot = G::PAIR ? warp >> 1 : warp * G::NB + grp;     // block slot inside the CTA
    const int bi = cta * G::BPC + slot;
    const bool valid = bi < n_blocks;
    int *const t = smem + slot * G::SLOT;

    B200ItxBlock blk;
    blk.dst_off = 0; blk.coef_off = 0; blk.eob = 0; blk.txtp = 0; blk.plane = 0;
    if (valid) blk = blocks[bi];
    const int txtp = blk.txtp;
    const int eob = blk.eob;
    uint32_t coff = blk.coef_off;
    if constexpr (COMPACT) coff = valid ? coffs[bi] : 0;
    coef *const cf = coefs + coff;
    const int stride = blk.plane == 0 ? stride0 : blk.plane == 1 ? stride1 : stride2;
    pixel *const dst = pic + blk.dst_off;

    constexpr int rnd = (1 << SHIFT) >> 1;
    const bool is_wht = (W == 4 && H == 4) && txtp == B200_WHT_WHT;
    const bool dc_only = !is_wht && eob < (txtp == 0 ? 1 : 0);

    int row_lo, col_lo;
    if (HBD) {
        row_lo = (int)((unsigned)~bitdepth_max << 7);
        col_lo = (int)((unsigned)~bitdepth_max << 5);
    } else {
        row_lo = col_lo = -32768;
    }
    const int row_hi = ~row_lo, col_hi = ~col_lo;

    const int t_first = is_wht ? 0 : c_tx_first[txtp & 15];
    const int t_second = is_wht ? 0 : c_tx_second[txtp & 15];

    // rows past this bound are zero by definition (reference src/itx_tmpl.c:86-105)
    const auto last_row = [&]() {
        if (t_second == TX1D_IDENTITY && t_first != TX1D_IDENTITY) return imin(G::SH - 1, eob);
        if (t_first == TX1D_IDENTITY && t_second != TX1D_IDENTITY) return eob >> (G::LW + 2);
        return (int)b200_lnz_col[b200_lnz_col_off[TX] + eob];
    };

    int dc = 0;
    if constexpr (COMPACT) {
        if (valid && dc_only) dc = (int)cf[0];
        // Stage the coded region in the tile, coefficient (y, x) at t[y * P + x]: lane y of pass 1 then reads its row from
        // where it writes it back (no lane reads another's row), and the odd pitch keeps those reads conflict-free. The rows
        // pass 1 reads are cleared, then the block's group scatters cf[0 .. eob] through the scan of its class, the mapping
        // of coef_expand_kernel (coef.cu). A dc-only block reads cf[0] (scan position 0 is coefficient 0) and stages nothing.
        const bool stage = valid && !dc_only && half == 0;
        if (stage && li < G::SH && li <= (is_wht ? G::SH - 1 : last_row())) {
#pragma unroll
            for (int x = 0; x < G::SW; x++) t[li * G::P + x] = 0;
        }
        __syncwarp();
        if (stage) {
            const int cls = is_wht ? 0 : c_tx_class[txtp & 15];
            for (int k = li; k <= eob; k += G::L) {
                int y, x;
                if (cls == 0) {
                    const int d = scan[k];
                    y = d & (G::SH - 1); x = d >> G::LSH;
                } else if (cls == 1) {
                    y = k & (G::SH - 1); x = k >> G::LSH;
                } else {
                    y = k >> G::LSW; x = k & (G::SW - 1);
                }
                t[y * G::P + x] = (int)cf[k];
            }
        }
        __syncwarp();
    }

    // ---------------- pass 1: one lane per coefficient row ----------------
    if (valid && !dc_only && li < G::SH && half == 0) {
        const int y = li;
        int c[W];
        if (is_wht) {
            if constexpr (W == 4 && H == 4) {
#pragma unroll
                for (int x = 0; x < 4; x++) c[x] = (COMPACT ? t[y * G::P + x] : (int)cf[y + x * 4]) >> 2;
                iwht4(c);
#pragma unroll
                for (int x = 0; x < 4; x++) t[y * G::P + x] = c[x];
            }
        } else {
            const int last = last_row();
            if (SHARED && y <= last) {
                itx_row_pass_shared<W, HBD>(cf + y, G::SH, t + y * G::P, G::RECT2, SHIFT, t_first, row_lo, row_hi, col_lo, col_hi);
            } else if (y <= last) {
#pragma unroll
                for (int x = 0; x < W; x++) {
                    if (x < G::SW) {
                        const int v = COMPACT ? t[y * G::P + x] : (int)cf[y + x * G::SH];
                        c[x] = G::RECT2 ? (int)((unsigned)v * 181u + 128u) >> 8 : v;
                    } else {
                        c[x] = 0;
                    }
                }
                tx1d_apply<W>(c, t_first, row_lo, row_hi);
#pragma unroll
                for (int x = 0; x < W; x++)
                    t[y * G::P + x] = iclip((c[x] + rnd) >> SHIFT, col_lo, col_hi);
            } else {
#pragma unroll
                for (int x = 0; x < W; x++) t[y * G::P + x] = 0;
            }
        }
        if (!COMPACT && zero_coefs) {          // (the compact stream is read-only)
#pragma unroll
            for (int x = 0; x < G::SW; x++) cf[y + x * G::SH] = 0;
        }
    }
    if (!COMPACT && valid && dc_only) dc = (int)cf[0];
    if (G::PAIR) __syncthreads(); else __syncwarp();               // (every thread of the CTA runs this function)
    if (!COMPACT && valid && dc_only && zero_coefs && li == 0 && half == 0) cf[0] = 0;

    // ---------------- pass 2: one lane per picture column ----------------
    if (valid) {
        if (dc_only) {
            if (G::RECT2) dc = (dc * 181 + 128) >> 8;
            dc = (dc * 181 + 128) >> 8;
            dc = (dc + rnd) >> SHIFT;
            dc = (dc * 181 + 128 + 2048) >> 12;
            // read-modify-write in load batches: the stores of one row must not serialise the loads of the next
            constexpr int CH = H < 16 ? H : 16;
            for (int x = li + half * 32; x < W; x += G::PAIR ? 64 : G::L) {
                for (int y0 = 0; y0 < H; y0 += CH) {
                    int v[CH];
#pragma unroll
                    for (int y = 0; y < CH; y++) v[y] = dst[(ptrdiff_t)(y0 + y) * stride + x];
#pragma unroll
                    for (int y = 0; y < CH; y++) dst[(ptrdiff_t)(y0 + y) * stride + x] = (pixel)iclip(v[y] + dc, 0, bitdepth_max);
                }
            }
        } else {
            for (int x = li + half * 32; x < W; x += G::PAIR ? 64 : G::L) {
                if (SHARED && !is_wht) {
                    itx_col_pass_shared<H, HBD>(t + x, G::P, dst + x, stride, t_second, col_lo, col_hi, bitdepth_max);
                    continue;
                }
                int c[H];
#pragma unroll
                for (int y = 0; y < H; y++) c[y] = y < G::SH ? t[y * G::P + x] : 0;
                if (is_wht) {
                    if constexpr (W == 4 && H == 4) {
                        iwht4(c);
#pragma unroll
                        for (int y = 0; y < 4; y++) {
                            pixel *p = dst + (ptrdiff_t)y * stride + x;
                            *p = (pixel)iclip((int)*p + c[y], 0, bitdepth_max);
                        }
                    }
                } else {
                    // The picture column is read in batches of up to 16 rows whose loads are all issued before the
                    // first store of the batch (a store may alias the next load, so row-by-row read-modify-write
                    // would serialise on memory latency); for H <= 16 the batch is issued before the transform so
                    // that the loads fly while the butterflies run.
                    if constexpr (H <= 8) {
                        // short columns: plain row-by-row read-modify-write (other warps hide the latency, and the
                        // extra registers of a batch would cost occupancy in the 8x8 / 4x4 bulk)
                        tx1d_apply<H>(c, t_second, col_lo, col_hi);
#pragma unroll
                        for (int y = 0; y < H; y++) {
                            pixel *p = dst + (ptrdiff_t)y * stride + x;
                            *p = (pixel)iclip((int)*p + ((c[y] + 8) >> 4), 0, bitdepth_max);
                        }
                    } else {
                        constexpr int CH = 16;
                        int pv[CH];
                        if (H <= 16) {
#pragma unroll
                            for (int y = 0; y < CH; y++) pv[y] = dst[(ptrdiff_t)y * stride + x];
                        }
                        tx1d_apply<H>(c, t_second, col_lo, col_hi);
#pragma unroll
                        for (int y0 = 0; y0 < H; y0 += CH) {
                            if (H > 16) {
#pragma unroll
                                for (int y = 0; y < CH; y++) pv[y] = dst[(ptrdiff_t)(y0 + y) * stride + x];
                            }
#pragma unroll
                            for (int y = 0; y < CH; y++)
                                dst[(ptrdiff_t)(y0 + y) * stride + x] = (pixel)iclip(pv[y] + ((c[y0 + y] + 8) >> 4), 0, bitdepth_max);
                        }
                    }
                }
            }
        }
    }
}

// One transform block by ONE warp (the warp-per-block intra kernel): the same two passes as itx_add_body — lane = coefficient
// row, padded tile `t` (>= SH * (W + 1) words), lane = picture column (64-wide blocks: two rounds) — through the out-of-line
// 1-D passes, so that all block sizes of a kernel share one copy of each butterfly network.
// resid != nullptr: nothing is added; the W x H residual goes to the dense int16 tile `resid` (pitch W).
template <int W, int H, int TX, int SHIFT, bool HBD>
B200_DEV void itx_add_warp(int *const t, typename Bd<HBD>::coef *const cf, typename Bd<HBD>::pixel *const dst, const int stride,
                           const int eob, const int txtp, const int bitdepth_max, int16_t *const resid = nullptr)
{
    typedef ItxGeom<W, H> G;
    typedef typename Bd<HBD>::pixel pixel;
    const int lane = threadIdx.x & 31;
    constexpr int rnd = (1 << SHIFT) >> 1;
    const bool is_wht = (W == 4 && H == 4) && txtp == B200_WHT_WHT;
    const bool dc_only = !is_wht && eob < (txtp == 0 ? 1 : 0);
    int row_lo, col_lo;
    if (HBD) { row_lo = (int)((unsigned)~bitdepth_max << 7); col_lo = (int)((unsigned)~bitdepth_max << 5); }
    else row_lo = col_lo = -32768;
    const int row_hi = ~row_lo, col_hi = ~col_lo;
    const int t_first = is_wht ? 0 : c_tx_first[txtp & 15];
    const int t_second = is_wht ? 0 : c_tx_second[txtp & 15];
    if (dc_only) {
        int dc = (int)cf[0];
        if (G::RECT2) dc = (dc * 181 + 128) >> 8;
        dc = (dc * 181 + 128) >> 8;
        dc = (dc + rnd) >> SHIFT;
        dc = (dc * 181 + 128 + 2048) >> 12;
        if (resid) {
            // (saturated: |residual| >= 2^15 clips the 12-bit sum exactly like the full value)
            for (int i = lane; i < W * H; i += 32) resid[i] = (int16_t)iclip(dc, -32768, 32767);
            __syncwarp();
            return;
        }
        for (int i = lane; i < W * H; i += 32) {
            pixel *p = dst + (ptrdiff_t)(i / W) * stride + (i % W);
            *p = (pixel)iclip((int)*p + dc, 0, bitdepth_max);
        }
        return;
    }
    if (lane < G::SH) {
        const int y = lane;
        if (is_wht) {
            if constexpr (W == 4 && H == 4) {
                int c[4];
#pragma unroll
                for (int x = 0; x < 4; x++) c[x] = (int)cf[y + x * 4] >> 2;
                iwht4(c);
#pragma unroll
                for (int x = 0; x < 4; x++) t[y * G::P + x] = c[x];
            }
        } else {
            int last;       // rows past this bound are zero by definition (reference src/itx_tmpl.c:86-105)
            if (t_second == TX1D_IDENTITY && t_first != TX1D_IDENTITY) last = imin(G::SH - 1, eob);
            else if (t_first == TX1D_IDENTITY && t_second != TX1D_IDENTITY) last = eob >> (G::LW + 2);
            else last = b200_lnz_col[b200_lnz_col_off[TX] + eob];
            if (y <= last) itx_row_pass_shared<W, HBD>(cf + y, G::SH, t + y * G::P, G::RECT2, SHIFT, t_first, row_lo, row_hi, col_lo, col_hi);
            else {
#pragma unroll
                for (int x = 0; x < W; x++) t[y * G::P + x] = 0;
            }
        }
    }
    __syncwarp();
    for (int x = lane; x < W; x += 32) {
        if (is_wht) {
            if constexpr (W == 4 && H == 4) {
                int c[4];
#pragma unroll
                for (int y = 0; y < 4; y++) c[y] = t[y * G::P + x];
                iwht4(c);
#pragma unroll
                for (int y = 0; y < 4; y++) {
                    if (resid) { resid[y * W + x] = (int16_t)iclip(c[y], -32768, 32767); continue; }
                    pixel *p = dst + (ptrdiff_t)y * stride + x;
                    *p = (pixel)iclip((int)*p + c[y], 0, bitdepth_max);
                }
            }
        } else {
            itx_col_pass_shared<H, HBD>(t + x, G::P, dst + x, stride, t_second, col_lo, col_hi, bitdepth_max, resid ? resid + x : nullptr);
        }
    }
    __syncwarp();
}

// transform size -> width / height in 4-sample units
static __constant__ uint8_t c_tx_w4[B200_N_RECT_TX_SIZES] = { 1, 2, 4, 8, 16, 1, 2, 2, 4, 4, 8, 8, 16, 1, 4, 2, 8, 4, 16 };
static __constant__ uint8_t c_tx_h4[B200_N_RECT_TX_SIZES] = { 1, 2, 4, 8, 16, 2, 1, 4, 2, 8, 4, 16, 8, 4, 1, 8, 2, 16, 4 };

}  // namespace b200
