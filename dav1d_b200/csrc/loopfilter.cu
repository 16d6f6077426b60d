// Deblocking filter (dav1d Dav1dLoopFilterDSPContext; reference src/loopfilter_tmpl.c:37-245,
// frame driver src/lf_apply_tmpl.c:176-466).
//
// Within one direction every edge segment is independent (a width-wd filter reads <= wd/2 and
// writes < wd/2 samples per side, and wd is bounded by the transform size on both sides), so a
// picture is deblocked by two flat sweeps instead of dav1d's per-superblock-row calls:
//   lf_cols_kernel  all column (vertical) edges: thread = (edge x4, unit row y4), 4 lines each; threadIdx.x
//                   walks consecutive edges of one line so a warp touches one contiguous row span
//   lf_rows_kernel  all row (horizontal) edges: thread = (pixel column, edge y4); threadIdx.x walks
//                   consecutive pixel columns, every tap is a coalesced row access
// Masks and levels are consumed in dav1d's own layout (Av1Filter bit masks, level[4] per 4x4).
#include "host_util.h"

namespace b200 {

// sample accessor for one line across one edge: index i = offset from the first sample after the edge (-8 .. 7).
// (A register-window accessor fed by aligned word loads was tried for the column edges and was slower.)
template <bool HBD> struct LfMem {            // straight from the picture, sb = step across the edge
    typename Bd<HBD>::pixel *p; ptrdiff_t sb;
    B200_DEV int get(int i) const { return p[i * sb]; }
    B200_DEV void set(int i, int v) { p[i * sb] = (typename Bd<HBD>::pixel)v; }
};
template <bool HBD, class Acc>
B200_DEV void lf_line_acc(Acc &px, int E, int I, int H, int wd, int bdmax)
{
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    const int F = 1 << b8;
    E <<= b8; I <<= b8; H <<= b8;
    const int p1 = px.get(-2), p0 = px.get(-1), q0 = px.get(0), q1 = px.get(1);
    int fm = iabs(p1 - p0) <= I && iabs(q1 - q0) <= I && iabs(p0 - q0) * 2 + (iabs(p1 - q1) >> 1) <= E;
    int p2 = 0, q2 = 0, p3 = 0, q3 = 0;
    if (wd > 4) {
        p2 = px.get(-3); q2 = px.get(2);
        fm &= iabs(p2 - p1) <= I && iabs(q2 - q1) <= I;
        if (wd > 6) {
            p3 = px.get(-4); q3 = px.get(3);
            fm &= iabs(p3 - p2) <= I && iabs(q3 - q2) <= I;
        }
    }
    if (!fm) return;
    int flat8in = 0;
    if (wd >= 6) flat8in = iabs(p2 - p0) <= F && iabs(p1 - p0) <= F && iabs(q1 - q0) <= F && iabs(q2 - q0) <= F;
    if (wd >= 8) flat8in &= iabs(p3 - p0) <= F && iabs(q3 - q0) <= F;
    if (wd >= 16) {
        const int p6 = px.get(-7), p5 = px.get(-6), p4 = px.get(-5), q4 = px.get(4), q5 = px.get(5), q6 = px.get(6);
        const int flat8out = iabs(p6 - p0) <= F && iabs(p5 - p0) <= F && iabs(p4 - p0) <= F &&
                             iabs(q4 - q0) <= F && iabs(q5 - q0) <= F && iabs(q6 - q0) <= F;
        if (flat8out & flat8in) {
            // sliding 16-term window over p6*6 p6 p5 .. q5 q6 q6*6 (reference :95-118)
            int s = p6 * 7 + p5 * 2 + p4 * 2 + p3 + p2 + p1 + p0 + q0 + 8;
            px.set(-6, (s >> 4)); s += -2 * p6 + p3 + q1;
            px.set(-5, (s >> 4)); s += -p6 - p5 + p2 + q2;
            px.set(-4, (s >> 4)); s += -p6 - p4 + p1 + q3;
            px.set(-3, (s >> 4)); s += -p6 - p3 + p0 + q4;
            px.set(-2, (s >> 4)); s += -p6 - p2 + q0 + q5;
            px.set(-1, (s >> 4)); s += -p6 - p1 + q1 + q6;
            px.set(0, (s >> 4)); s += -p5 - p0 + q2 + q6;
            px.set(1, (s >> 4)); s += -p4 - q0 + q3 + q6;
            px.set(2, (s >> 4)); s += -p3 - q1 + q4 + q6;
            px.set(3, (s >> 4)); s += -p2 - q2 + q5 + q6;
            px.set(4, (s >> 4)); s += -p1 - q3 + q6 + q6;
            px.set(5, (s >> 4));
            return;
        }
    }
    if (wd >= 8 && flat8in) {
        px.set(-3, ((p3 + p3 + p3 + 2 * p2 + p1 + p0 + q0 + 4) >> 3));
        px.set(-2, ((p3 + p3 + p2 + 2 * p1 + p0 + q0 + q1 + 4) >> 3));
        px.set(-1, ((p3 + p2 + p1 + 2 * p0 + q0 + q1 + q2 + 4) >> 3));
        px.set(0, ((p2 + p1 + p0 + 2 * q0 + q1 + q2 + q3 + 4) >> 3));
        px.set(1, ((p1 + p0 + q0 + 2 * q1 + q2 + q3 + q3 + 4) >> 3));
        px.set(2, ((p0 + q0 + q1 + 2 * q2 + q3 + q3 + q3 + 4) >> 3));
    } else if (wd == 6 && flat8in) {
        px.set(-2, ((p2 + 2 * p2 + 2 * p1 + 2 * p0 + q0 + 4) >> 3));
        px.set(-1, ((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3));
        px.set(0, ((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3));
        px.set(1, ((p0 + 2 * q0 + 2 * q1 + 2 * q2 + q2 + 4) >> 3));
    } else {
        const int lo = -128 * (1 << b8), hi = 128 * (1 << b8) - 1;
        const bool hev = iabs(p1 - p0) > H || iabs(q1 - q0) > H;
        int f = hev ? iclip(p1 - q1, lo, hi) : 0;
        f = iclip(3 * (q0 - p0) + f, lo, hi);
        const int f1 = imin(f + 4, hi) >> 3, f2 = imin(f + 3, hi) >> 3;
        px.set(-1, iclip(p0 + f2, 0, bdmax));
        px.set(0, iclip(q0 - f1, 0, bdmax));
        if (!hev) {
            const int g = (f1 + 1) >> 1;
            px.set(-2, iclip(p1 + g, 0, bdmax));
            px.set(1, iclip(q1 - g, 0, bdmax));
        }
    }
}

template <bool HBD>
B200_DEV void lf_line(typename Bd<HBD>::pixel *p, ptrdiff_t sb, int E, int I, int H, int wd, int bdmax)
{
    LfMem<HBD> m{ p, sb };
    lf_line_acc<HBD>(m, E, I, H, wd, bdmax);
}

// decode the filter width of unit `a` (index along the edge direction inside the 128x128 area) for
// the line of units `b` (index across it); returns 0 when no edge is filtered there
B200_DEV int lf_width(const B200Av1Filter &m, int plane, int dir, int b, int a, int ss_a)
{
    if (plane == 0) {
        const int half = a >> 4, bit = a & 15;
        if ((m.filter_y[dir][b][2][half] >> bit) & 1) return 16;
        if ((m.filter_y[dir][b][1][half] >> bit) & 1) return 8;
        if ((m.filter_y[dir][b][0][half] >> bit) & 1) return 4;
        return 0;
    }
    const int hs = 16 >> ss_a;                       // units per 16-bit half along the edge direction
    const int half = a >= hs, bit = a - half * hs;
    if ((m.filter_uv[dir][b][1][half] >> bit) & 1) return 6;
    if ((m.filter_uv[dir][b][0][half] >> bit) & 1) return 4;
    return 0;
}

// grid: (ceil(units_x / 32), ceil(units_y / 8), 3 planes); block (32, 8); a thread owns the 4 lines of one 4x4 unit
// edge: mask decoding and level look-up are per unit, and the 4 lines give the memory system independent loads
template <bool HBD>
__global__ void __launch_bounds__(256) lf_cols_kernel(const __grid_constant__ B200LfFrame f, int bdmax, int ya4, int yb4)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int plane = blockIdx.z;
    if (plane ? !f.filter_uv : !f.filter_y) return;
    const int ssh = plane ? f.ss_hor : 0, ssv = plane ? f.ss_ver : 0;
    const int x4 = blockIdx.x * 32 + threadIdx.x;            // 4-px unit (plane units)
    const int y4 = (ya4 >> ssv) + blockIdx.y * 8 + threadIdx.y;     // rows [ya4, yb4) in luma units: one band (or the frame)
    const int pw4 = (f.w4 + ssh) >> ssh, ph4 = imin((f.h4 + ssv) >> ssv, (yb4 + ssv) >> ssv);
    if (x4 >= pw4 || x4 == 0 || y4 >= ph4) return;
    // 32 >> ss units per 128x128 area: shifts, not divisions (a run-time divisor costs ~20 instructions per thread)
    const int sbx = x4 >> (5 - ssh), xi = x4 & ((32 >> ssh) - 1);
    const int sby = y4 >> (5 - ssv), yi = y4 & ((32 >> ssv) - 1);
    const B200Av1Filter &m = f.mask[sby * f.sb128w + sbx];
    const int wd = lf_width(m, plane, 0, xi, yi, ssv);
    if (!wd) return;
    const uint8_t (*l)[4] = f.level + (ptrdiff_t)y4 * f.b4_stride + x4;
    const int c = plane == 0 ? 0 : plane + 1;
    const int L = l[0][c] ? l[0][c] : l[-1][c];
    if (!L) return;
    const int E = f.lut.e[L], I = f.lut.i[L];
    pixel *p = (pixel *)f.pic + f.plane_off[plane] + (ptrdiff_t)(y4 * 4) * f.stride[plane] + x4 * 4;
#pragma unroll 1
    for (int k = 0; k < 4; k++, p += f.stride[plane]) lf_line<HBD>(p, 1, E, I, L >> 4, wd, bdmax);
}

// grid: (ceil(width_px / 128), ceil(units_y / 2), 3); block (128, 2)
template <bool HBD>
__global__ void __launch_bounds__(256) lf_rows_kernel(const __grid_constant__ B200LfFrame f, int bdmax, int ya4, int yb4)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int plane = blockIdx.z;
    if (plane ? !f.filter_uv : !f.filter_y) return;
    const int ssh = plane ? f.ss_hor : 0, ssv = plane ? f.ss_ver : 0;
    const int x = blockIdx.x * 128 + threadIdx.x;
    const int y4 = (ya4 >> ssv) + blockIdx.y * 2 + threadIdx.y;
    const int pw4 = (f.w4 + ssh) >> ssh, ph4 = imin((f.h4 + ssv) >> ssv, (yb4 + ssv) >> ssv);
    if (x >= pw4 * 4 || y4 >= ph4 || y4 == 0) return;
    const int x4 = x >> 2, sbx = x4 >> (5 - ssh), xi = x4 & ((32 >> ssh) - 1);
    const int sby = y4 >> (5 - ssv), yi = y4 & ((32 >> ssv) - 1);
    const B200Av1Filter &m = f.mask[sby * f.sb128w + sbx];
    const int wd = lf_width(m, plane, 1, yi, xi, ssh);
    if (!wd) return;
    const uint8_t (*l)[4] = f.level + (ptrdiff_t)y4 * f.b4_stride + x4;
    const int c = plane == 0 ? 1 : plane + 1;
    const int L = l[0][c] ? l[0][c] : l[-f.b4_stride][c];
    if (!L) return;
    pixel *p = (pixel *)f.pic + f.plane_off[plane] + (ptrdiff_t)(y4 * 4) * f.stride[plane] + x;
    lf_line<HBD>(p, f.stride[plane], f.lut.e[L], f.lut.i[L], L >> 4, wd, bdmax);
}

// Level-1 form: one call of loop_filter_sb = up to 32 segments along one line of units
struct LfSbArgs {
    uint32_t mask[3];
    uint8_t cur[32], prev[32];
    B200FilterLUT lut;
    int plane_class, dir, n_units, stride;
};
template <bool HBD>
__global__ void lf_sb_kernel(typename Bd<HBD>::pixel *dst, LfSbArgs a, int bdmax)
{
    const int line = blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= a.n_units * 4) return;
    const int u = line >> 2;
    int wd = 0;
    if (a.plane_class) wd = (a.mask[1] >> u) & 1 ? 6 : ((a.mask[0] >> u) & 1 ? 4 : 0);
    else wd = (a.mask[2] >> u) & 1 ? 16 : ((a.mask[1] >> u) & 1 ? 8 : ((a.mask[0] >> u) & 1 ? 4 : 0));
    if (!wd) return;
    const int L = a.cur[u] ? a.cur[u] : a.prev[u];
    if (!L) return;
    // dense window: dir 0 -> 16 px wide rows, edge at column 8; dir 1 -> 16 rows, edge at row 8
    typename Bd<HBD>::pixel *p = a.dir ? dst + 8 * a.stride + line : dst + (ptrdiff_t)line * a.stride + 8;
    lf_line<HBD>(p, a.dir ? a.stride : 1, a.lut.e[L], a.lut.i[L], L >> 4, wd, bdmax);
}

// rows [ya4, yb4) (luma 4-px units; even, so that subsampled chroma rows split at the same place) of both sweeps:
// the column edges of those rows, then the row edges at ya4 .. yb4 - 1. Run band after band from the top this is the
// whole-frame order: a row-edge filter at y touches rows y - 7 .. y + 6 only, all of them column-filtered already.
int lf_frame_rows(int bdmax, const B200LfFrame *f, int ya4, int yb4, cudaStream_t stream)
{
    if (int r = check_bdmax(bdmax, "b200_lf_frame")) return r;
    if (!f->filter_y) return 0;   // dav1d skips deblocking entirely when both luma levels are 0 (src/recon_tmpl.c:1988)
    ya4 = imax(ya4, 0); yb4 = imin(yb4, f->h4);
    if (yb4 <= ya4) return 0;
    if ((ya4 & 1) || ((yb4 & 1) && yb4 != f->h4)) { b200_set_error("b200_lf_frame: odd band boundary"); return -2; }
    const int w4 = f->w4, n4 = yb4 - ya4;
    if (int r = launch_hbd(bdmax, Launch::pdl, dim3((w4 + 31) / 32, (n4 + 7) / 8, 3), dim3(32, 8), 0, stream,
                           [&](auto hbd) { return std::make_tuple(lf_cols_kernel<hbd>, *f, bdmax, ya4, yb4); }))
        return r;
    return launch_hbd(bdmax, Launch::pdl, dim3((w4 * 4 + 127) / 128, (n4 + 1) / 2, 3), dim3(128, 2), 0, stream,
                      [&](auto hbd) { return std::make_tuple(lf_rows_kernel<hbd>, *f, bdmax, ya4, yb4); });
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_lf_frame(int bdmax, const B200LfFrame *f, void *stream)
{
    return b200::lf_frame_rows(bdmax, f, 0, f->h4, (cudaStream_t)stream);
}

int b200_loop_filter_sb(int plane_class, int dir, void *dst, ptrdiff_t stride, const uint32_t *mask,
                        const uint8_t (*lvl)[4], ptrdiff_t lvl_stride, const B200FilterLUT *lut, int w, int bdmax)
{
    (void)w;   // like the C reference, the extent comes from the highest set mask bit
    if (int r = check_bdmax(bdmax, "b200_loop_filter_sb")) return r;
    const uint32_t vm = mask[0] | mask[1] | (plane_class ? 0 : mask[2]);
    if (!vm) return 0;
    int n_units = 32 - __builtin_clz(vm);
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    LfSbArgs a;
    memset(&a, 0, sizeof(a));
    a.mask[0] = mask[0]; a.mask[1] = mask[1]; a.mask[2] = plane_class ? 0 : mask[2];
    a.lut = *lut; a.plane_class = plane_class; a.dir = dir; a.n_units = n_units;
    for (int u = 0; u < n_units; u++) {
        const uint8_t (*l)[4] = lvl + (dir ? u : u * lvl_stride);
        a.cur[u] = l[0][0];
        a.prev[u] = dir ? l[-lvl_stride][0] : l[-1][0];
    }
    const int lines = n_units * 4;
    int ww, wh; uint8_t *org;
    if (dir) { ww = lines; wh = 16; org = (uint8_t *)dst - 8 * stride; }
    else { ww = 16; wh = lines; org = (uint8_t *)dst - 8 * (ptrdiff_t)px; }
    a.stride = ww;
    void *win = L.upload_rect(0, org, stride, ww, wh, px);
    if (!win) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3((lines + 127) / 128), dim3(128), 0, 0,
                           [&](auto hbd) { return std::make_tuple(lf_sb_kernel<hbd>, (typename Bd<hbd>::pixel *)win, a, bdmax); }))
        return r;
    return L.download_rect(0, org, stride, ww, wh, px);
}

}  // extern "C"

namespace {
template <int PC, int DIR> void lf8(uint8_t *d, ptrdiff_t s, const uint32_t *m, const uint8_t (*l)[4], ptrdiff_t ls, const B200FilterLUT *lut, int w) {
    if (b200_loop_filter_sb(PC, DIR, d, s, m, l, ls, lut, w, 255)) die("loop_filter_sb");
}
template <int PC, int DIR> void lf16(uint16_t *d, ptrdiff_t s, const uint32_t *m, const uint8_t (*l)[4], ptrdiff_t ls, const B200FilterLUT *lut, int w, int bd) {
    if (b200_loop_filter_sb(PC, DIR, d, s, m, l, ls, lut, w, bd)) die("loop_filter_sb");
}
}
extern "C" {
void b200_loop_filter_dsp_init_8bpc(B200LoopFilterDSPContext *c) {
    c->loop_filter_sb[0][0] = (void *)lf8<0, 0>; c->loop_filter_sb[0][1] = (void *)lf8<0, 1>;
    c->loop_filter_sb[1][0] = (void *)lf8<1, 0>; c->loop_filter_sb[1][1] = (void *)lf8<1, 1>;
}
void b200_loop_filter_dsp_init_16bpc(B200LoopFilterDSPContext *c) {
    c->loop_filter_sb[0][0] = (void *)lf16<0, 0>; c->loop_filter_sb[0][1] = (void *)lf16<0, 1>;
    c->loop_filter_sb[1][0] = (void *)lf16<1, 0>; c->loop_filter_sb[1][1] = (void *)lf16<1, 1>;
}
}
