// Batched inverse transform + add (dav1d Dav1dInvTxfmDSPContext, reference src/itx_tmpl.c:43-203).
//
// Work decomposition (all sizes 4x4 .. 64x64, all 16 transform types + WHT):
//   * a transform block of w x h is owned by a group of L = max(min(h,32), min(w,32)) lanes
//     (32/L blocks per warp, 4 warps per CTA);
//   * pass 1: lane y holds coefficient row y (length w) in registers, runs the horizontal
//     1-D transform, applies the inter-pass rounding/clip and parks the row in a padded
//     shared-memory tile (pitch w+1 words: conflict-free both ways);
//   * pass 2: lane x pulls column x (length h) back into registers, runs the vertical 1-D
//     transform and does the read-modify-write of the picture column, so that consecutive
//     lanes touch consecutive pixels of a row (coalesced).
// Integer only, bit-exact with the reference C path for every input (including coefficient
// garbage: rows beyond the eob-derived bound are treated as zero exactly like the reference).
#include "itx_body.cuh"
#include "host_util.h"
#include "launch_count.h"
#define B200_SCAN_TBL __device__
#include "scan_gen.h"

namespace b200 {

template <int W, int H, int TX, int SHIFT, bool HBD>
__global__ void __launch_bounds__(kItxWarps * 32)
itx_add_kernel(const B200ItxBlock *__restrict__ blocks, int n_blocks,
               typename Bd<HBD>::coef *__restrict__ coefs, typename Bd<HBD>::pixel *__restrict__ pic,
               int stride0, int stride1, int stride2, int bitdepth_max, int zero_coefs)
{
    B200_PDL_ENTRY();
    typedef ItxGeom<W, H> G;
    __shared__ int tile[ItxGeom<W, H>::BPC * G::SLOT];
    itx_add_body<W, H, TX, SHIFT, HBD>(blockIdx.x, tile, blocks, n_blocks, coefs, pic, stride0, stride1, stride2,
                                       bitdepth_max, zero_coefs);
}

// ---- all transform sizes of a frame in two launches (one per register class), CTAs dealt largest size first ---
struct ItxGroups {
    const B200ItxBlock *blocks[B200_N_RECT_TX_SIZES];
    const uint32_t *coffs[B200_N_RECT_TX_SIZES];          // compact form: per block the offset of its coefficients
    int n[B200_N_RECT_TX_SIZES];
    int cta_begin[B200_N_RECT_TX_SIZES], cta_end[B200_N_RECT_TX_SIZES];
};

// Two register classes, one launch each: sizes with a 64-point dimension (long butterflies, up to ~170 live
// registers, 33 KB tile) and everything else (<= 64 registers, 17 KB tile, 8 CTAs per SM).
#ifndef B200_ITX_SMALL_MINB
#define B200_ITX_SMALL_MINB 7
#endif
template <bool BIG> struct ItxClass {
    static constexpr int kMinCtas = BIG ? 3 : B200_ITX_SMALL_MINB;
    static constexpr int kTileWords = kItxWarps * (BIG ? ItxGeom<64, 64>::NB * ItxGeom<64, 64>::SLOT
                                                       : ItxGeom<32, 32>::NB * ItxGeom<32, 32>::SLOT);
};

// COMPACT: `coefs` is the compact coefficient stream, g.coffs[tx] the blocks' offsets into it (itx_add_body)
template <bool HBD, bool BIG, bool COMPACT>
__global__ void __launch_bounds__(kItxWarps * 32, ItxClass<BIG>::kMinCtas)
itx_add_grouped_kernel(const __grid_constant__ ItxGroups g, typename Bd<HBD>::coef *__restrict__ coefs, typename Bd<HBD>::pixel *__restrict__ pic,
                       int stride0, int stride1, int stride2, int bitdepth_max, int zero_coefs)
{
    B200_PDL_ENTRY();
    __shared__ int tile[ItxClass<BIG>::kTileWords];
    const int c = blockIdx.x;
#define X(TX, W, H, SH) \
    if constexpr ((W == 64 || H == 64) == BIG) { \
        if (c < g.cta_end[TX]) { \
            itx_add_body<W, H, TX, SH, HBD, false, COMPACT>(c - g.cta_begin[TX], tile, g.blocks[TX], g.n[TX], coefs, pic, stride0, \
                                                            stride1, stride2, bitdepth_max, zero_coefs, g.coffs[TX], \
                                                            b200_scan + b200_scan_off[TX]); \
            return; \
        } \
    }
    B200_ITX_SIZES(X)
#undef X
}

int launch_itx_grouped(const void *const *blocks, const int32_t *n, void *coefs, void *pic, const int32_t *st,
                       int bdmax, int zero, cudaStream_t stream, const uint32_t *const *coffs)
{
    for (int big = 1; big >= 0; big--) {
        ItxGroups g;
        int total = 0;
#define X(TX, W, H, SH) { \
            const int per_cta = ItxGeom<W, H>::BPC; \
            const int mine = ((W == 64 || H == 64) ? 1 : 0) == big; \
            const int ctas = (mine && n[TX] > 0) ? (n[TX] + per_cta - 1) / per_cta : 0; \
            g.blocks[TX] = (const B200ItxBlock *)blocks[TX]; g.n[TX] = n[TX] > 0 ? n[TX] : 0; \
            g.coffs[TX] = coffs ? coffs[TX] : nullptr; \
            g.cta_begin[TX] = total; total += ctas; g.cta_end[TX] = total; }
        B200_ITX_SIZES(X)
#undef X
        if (!total) continue;
        if (int r = launch_hbd(bdmax, Launch::pdl, dim3(total), dim3(kItxWarps * 32), 0, stream, [&](auto hbd) {
                typedef Bd<hbd> B;
                auto kern = coffs ? (big ? itx_add_grouped_kernel<hbd, true, true> : itx_add_grouped_kernel<hbd, false, true>)
                                  : (big ? itx_add_grouped_kernel<hbd, true, false> : itx_add_grouped_kernel<hbd, false, false>);
                return std::make_tuple(kern, g, (typename B::coef *)coefs, (typename B::pixel *)pic, st[0], st[1], st[2], bdmax, zero);
            }))
            return r;
    }
    return 0;
}

// one transform size: n blocks of the batch, BPC of them per CTA
int launch_itx(int tx, const B200ItxBlock *blocks, int n, void *coefs, void *pic, const int32_t *st, int bdmax, int zero,
               cudaStream_t stream)
{
    switch (tx) {
#define X(TX, W, H, SH) \
    case TX: \
        return launch_hbd(bdmax, Launch::plain, dim3((n + ItxGeom<W, H>::BPC - 1) / ItxGeom<W, H>::BPC), dim3(kItxWarps * 32), 0, stream, \
                          [&](auto hbd) { \
                              typedef Bd<hbd> B; \
                              return std::make_tuple(itx_add_kernel<W, H, TX, SH, hbd>, blocks, n, (typename B::coef *)coefs, \
                                                     (typename B::pixel *)pic, st[0], st[1], st[2], bdmax, zero); \
                          });
    B200_ITX_SIZES(X)
#undef X
    }
    b200_set_error("bad transform size %d", tx);
    return -2;
}

}  // namespace b200
