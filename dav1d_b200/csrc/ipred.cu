// Intra prediction (dav1d Dav1dIntraPredDSPContext; reference src/ipred_tmpl.c:39-675).
// One CTA per block: the edge array is copied into shared memory as ints, directional modes first
// build their filtered / upsampled edge there, then every thread produces pixels of the block with
// consecutive threads on consecutive columns. Filter-intra walks its 4x2 units along anti-diagonals
// (each unit depends on its left / top / top-left neighbours only). Integer, bit-exact.
#include "ipred_body.cuh"

namespace b200 {

template <bool HBD>
__global__ void __launch_bounds__(kIpT) ipred_kernel(const B200IpredBlock *__restrict__ blocks, int n, const __grid_constant__ B200IpredFrame f, int bdmax)
{
    typedef typename Bd<HBD>::pixel pixel;
    __shared__ IpShared S;
    const B200IpredBlock b = blocks[blockIdx.x];
    const int w = b.w, h = b.h, tid = threadIdx.x;
    pixel *const dst = (pixel *)f.dst + b.dst_off;
    const int st = f.dst_stride[b.plane];
    int *const tl = S.edge + 128;

    if (b.op == B200_IPRED_OP_PAL_PRED) {
        const pixel *pal = (const pixel *)f.edge + b.edge_off;
        const uint8_t *idx = f.pal_idx + b.ac_off;
        for (int i = tid; i < (w * h) >> 1; i += kIpT) {
            const int y = i / (w >> 1), x = (i - y * (w >> 1)) * 2, v = idx[i];
            dst[(ptrdiff_t)y * st + x] = pal[v & 7];
            dst[(ptrdiff_t)y * st + x + 1] = pal[v >> 4];
        }
        return;
    }
    if (b.op == B200_IPRED_OP_CFL_AC) {
        // dst_off addresses the luma block inside the picture (plane 0)
        ipred_cfl_ac_body<HBD>(S, (const pixel *)f.dst + b.dst_off, f.dst_stride[0], f.ss_hor, f.ss_ver, w, h,
                               b.angle & 0xff, (b.angle >> 8) & 0xff, f.ac + b.ac_off);
        return;
    }

    // ---- edge array to shared memory: tl[-(w+h) .. w+h] ----
    {
        const pixel *e = (const pixel *)f.edge + b.edge_off;
        for (int i = tid - (w + h); i <= w + h; i += kIpT) tl[i] = e[i];
    }
    __syncthreads();
    if (b.op == B200_IPRED_OP_CFL_PRED) {
        ipred_cfl_pred_body<HBD>(S, dst, st, w, h, b.mode, b.alpha, f.ac + b.ac_off, bdmax);
        return;
    }
    ipred_pred_body<HBD>(S, dst, st, w, h, b.mode, b.angle, b.max_w, b.max_h, bdmax);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_ipred_batch(int bdmax, const B200IpredFrame *f, const B200IpredBlock *d_blocks, int n, void *stream)
{
    if (int r = check_bdmax(bdmax, "b200_ipred_batch")) return r;
    if (n <= 0) return 0;
    return launch_hbd(bdmax, Launch::plain, dim3(n), dim3(kIpT), 0, (cudaStream_t)stream,
                      [&](auto hbd) { return std::make_tuple(ipred_kernel<hbd>, d_blocks, n, *f, bdmax); });
}

}

// ---- Level 1 -------------------------------------------------------------------------------
namespace {
enum { DST, EDGE, AC, IDX, DESC };   // Level1 scratch slots

// the one-record batch of f / b, then the w x h pixels it wrote into the rectangle at dst
int ipred_l1(Level1 &L, B200IpredFrame &f, const B200IpredBlock &b, void *dst, ptrdiff_t stride, int bdmax)
{
    const void *desc = L.upload(DESC, &b, sizeof(b));
    if (!desc) return -1;
    if (int r = b200_ipred_batch(bdmax, &f, (const B200IpredBlock *)desc, 1, 0)) return r;
    return L.download_rect(DST, dst, stride, b.w, b.h, bdmax > 255 ? 2 : 1);
}

int ipred_pred_l1(int op, int mode, void *dst, ptrdiff_t stride, const void *topleft, int w, int h, int angle, int max_w,
                  int max_h, const int16_t *ac, int alpha, int bdmax)
{
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    B200IpredFrame f;
    memset(&f, 0, sizeof(f));
    f.dst_stride[0] = w;
    // the edge window [-(w+h), w+h] around topleft
    if (!(f.edge = L.upload(EDGE, (const uint8_t *)topleft - (ptrdiff_t)(w + h) * (ptrdiff_t)px, (size_t)(2 * (w + h) + 1) * px)) ||
        !(f.dst = L.dev(DST, (size_t)w * h * px)) || (op == B200_IPRED_OP_CFL_PRED && !(f.ac = (int16_t *)L.upload(AC, ac, (size_t)w * h * 2))))
        return -1;
    B200IpredBlock b;
    memset(&b, 0, sizeof(b));
    b.edge_off = (uint32_t)(w + h); b.w = (uint8_t)w; b.h = (uint8_t)h; b.mode = (uint8_t)mode; b.op = (uint8_t)op;
    b.angle = (int16_t)angle; b.max_w = max_w; b.max_h = max_h; b.alpha = (int8_t)alpha;
    return ipred_l1(L, f, b, dst, stride, bdmax);
}
}  // namespace

extern "C" {

int b200_ipred(int mode, void *dst, ptrdiff_t stride, const void *topleft, int w, int h, int angle, int max_w, int max_h, int bdmax)
{
    if (mode < 0 || mode > 13 || w < 4 || w > 64 || h < 4 || h > 64 || (mode == 13 && (w > 32 || h > 32))) { b200_set_error("b200_ipred: bad arguments"); return -2; }
    return ipred_pred_l1(B200_IPRED_OP_PRED, mode, dst, stride, topleft, w, h, angle, max_w, max_h, nullptr, 0, bdmax);
}
int b200_cfl_pred(int mode, void *dst, ptrdiff_t stride, const void *topleft, int w, int h, const int16_t *ac, int alpha, int bdmax)
{
    if (!(mode == 0 || mode == 3 || mode == 4 || mode == 5) || w < 4 || w > 32 || h < 4 || h > 32) { b200_set_error("b200_cfl_pred: bad arguments"); return -2; }
    return ipred_pred_l1(B200_IPRED_OP_CFL_PRED, mode, dst, stride, topleft, w, h, 0, 0, 0, ac, alpha, bdmax);
}
int b200_cfl_ac(int16_t *ac, const void *ypx, ptrdiff_t stride, int w_pad, int h_pad, int cw, int ch, int ss_hor, int ss_ver, int bdmax)
{
    if (cw < 4 || cw > 32 || ch < 4 || ch > 32) { b200_set_error("b200_cfl_ac: bad arguments"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    const int lw = (cw - 4 * w_pad) << ss_hor, lh = (ch - 4 * h_pad) << ss_ver;   // luma samples actually read
    B200IpredFrame f;
    memset(&f, 0, sizeof(f));
    f.dst_stride[0] = lw; f.ss_hor = ss_hor; f.ss_ver = ss_ver;
    B200IpredBlock b;
    memset(&b, 0, sizeof(b));
    b.w = (uint8_t)cw; b.h = (uint8_t)ch; b.op = B200_IPRED_OP_CFL_AC; b.angle = (int16_t)(w_pad | (h_pad << 8));
    const void *desc;
    if (!(f.dst = L.upload_rect(DST, ypx, stride, lw, lh, px)) || !(f.ac = (int16_t *)L.dev(AC, (size_t)cw * ch * 2)) ||
        !(desc = L.upload(DESC, &b, sizeof(b))))
        return -1;
    if (int r = b200_ipred_batch(bdmax, &f, (const B200IpredBlock *)desc, 1, 0)) return r;
    return L.download_rect(AC, ac, (ptrdiff_t)cw * 2, cw, ch, 2);
}
int b200_pal_pred(void *dst, ptrdiff_t stride, const void *pal, const uint8_t *idx, int w, int h, int bdmax)
{
    if (w < 4 || w > 64 || h < 4 || h > 64) { b200_set_error("b200_pal_pred: bad arguments"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    B200IpredFrame f;
    memset(&f, 0, sizeof(f));
    f.dst_stride[0] = w;
    if (!(f.edge = L.upload(EDGE, pal, 8 * px)) || !(f.pal_idx = (const uint8_t *)L.upload(IDX, idx, (size_t)w * h / 2)) ||
        !(f.dst = L.dev(DST, (size_t)w * h * px)))
        return -1;
    B200IpredBlock b;
    memset(&b, 0, sizeof(b));
    b.w = (uint8_t)w; b.h = (uint8_t)h; b.op = B200_IPRED_OP_PAL_PRED;
    return ipred_l1(L, f, b, dst, stride, bdmax);
}

}  // extern "C"

namespace {
template <int M> void ip8(uint8_t *d, ptrdiff_t s, const uint8_t *tl, int w, int h, int a, int mw, int mh) { if (b200_ipred(M, d, s, tl, w, h, a, mw, mh, 255)) die("intra_pred"); }
template <int M> void ip16(uint16_t *d, ptrdiff_t s, const uint16_t *tl, int w, int h, int a, int mw, int mh, int bd) { if (b200_ipred(M, d, s, tl, w, h, a, mw, mh, bd)) die("intra_pred"); }
template <int M> void cp8(uint8_t *d, ptrdiff_t s, const uint8_t *tl, int w, int h, const int16_t *ac, int al) { if (b200_cfl_pred(M, d, s, tl, w, h, ac, al, 255)) die("cfl_pred"); }
template <int M> void cp16(uint16_t *d, ptrdiff_t s, const uint16_t *tl, int w, int h, const int16_t *ac, int al, int bd) { if (b200_cfl_pred(M, d, s, tl, w, h, ac, al, bd)) die("cfl_pred"); }
template <int BD, int SH, int SV> void ca(int16_t *ac, const void *y, ptrdiff_t s, int wp, int hp, int cw, int ch) { if (b200_cfl_ac(ac, y, s, wp, hp, cw, ch, SH, SV, BD)) die("cfl_ac"); }
template <int BD> void pp(void *d, ptrdiff_t s, const void *pal, const uint8_t *idx, int w, int h) { if (b200_pal_pred(d, s, pal, idx, w, h, BD)) die("pal_pred"); }
template <int... M> void fill_ip8(B200IntraPredDSPContext *c, std::integer_sequence<int, M...>) { ((c->intra_pred[M] = (void *)ip8<M>), ...); }
template <int... M> void fill_ip16(B200IntraPredDSPContext *c, std::integer_sequence<int, M...>) { ((c->intra_pred[M] = (void *)ip16<M>), ...); }
}
extern "C" {
void b200_intra_pred_dsp_init_8bpc(B200IntraPredDSPContext *c) {
    memset(c, 0, sizeof(*c));
    fill_ip8(c, std::make_integer_sequence<int, 14>{});
    c->cfl_ac[0] = (void *)ca<255, 1, 1>; c->cfl_ac[1] = (void *)ca<255, 1, 0>; c->cfl_ac[2] = (void *)ca<255, 0, 0>;
    c->cfl_pred[0] = (void *)cp8<0>; c->cfl_pred[3] = (void *)cp8<3>; c->cfl_pred[4] = (void *)cp8<4>; c->cfl_pred[5] = (void *)cp8<5>;
    c->pal_pred = (void *)pp<255>;
}
void b200_intra_pred_dsp_init_16bpc(B200IntraPredDSPContext *c) {
    memset(c, 0, sizeof(*c));
    fill_ip16(c, std::make_integer_sequence<int, 14>{});
    // cfl_ac / pal_pred carry no bit-depth argument in dav1d; only the pixel width matters
    c->cfl_ac[0] = (void *)ca<1023, 1, 1>; c->cfl_ac[1] = (void *)ca<1023, 1, 0>; c->cfl_ac[2] = (void *)ca<1023, 0, 0>;
    c->cfl_pred[0] = (void *)cp16<0>; c->cfl_pred[3] = (void *)cp16<3>; c->cfl_pred[4] = (void *)cp16<4>; c->cfl_pred[5] = (void *)cp16<5>;
    c->pal_pred = (void *)pp<1023>;
}
}
