// Film grain (dav1d Dav1dFilmGrainDSPContext; reference src/filmgrain_tmpl.c:50-402,
// driver src/fg_apply_tmpl.c:41-240).
//
//   fg_prep_kernel   one CTA per picture: (1) the raw grain fields (16-bit LFSR -> Gaussian table), one thread
//                    per LUT row after an LFSR jump-ahead (GF(2) matrix powers); (2) the raster-order AR
//                    filter as a skewed wavefront in shared memory, one thread per LUT row, row y trailing
//                    row y-1 by lag+1 columns; (3) scaling LUTs (closed form of the `d += delta`
//                    recurrence) and (4) the per-row block-offset chains.
//   fg_apply_kernel  one thread per 4 consecutive pixels: LUT samples of their own 32x32 block blended with
//                    the left / top / top-left blocks' samples inside the 2-sample overlap, scaled by
//                    scaling[] of the (luma-mixed) sample value, clipped.
#include "host_util.h"
#define B200_TBL __constant__
#include "tables_gen.h"

namespace b200 {

constexpr int GW = B200_GRAIN_WIDTH, GH = B200_GRAIN_HEIGHT;
constexpr int kMaxBlocksX = 512;           // 16384 / 32

// scratch layout (bytes): 3 LUTs of (GH+1)*GW int16, 3 scaling tables of 4096 bytes, offsets[rows][kMaxBlocksX]
struct FgScratch {
    int16_t lut[3][(GH + 1) * GW];
    uint8_t scaling[3][4096];
    uint8_t offsets[(B200_FG_SCRATCH_BYTES - 3 * (GH + 1) * GW * 2 - 3 * 4096)];
};
static_assert(sizeof(FgScratch) <= B200_FG_SCRATCH_BYTES, "scratch layout");

B200_HD int fg_rnd(int bits, unsigned *state) {
    const int r = (int)*state;
    const unsigned bit = ((r >> 0) ^ (r >> 1) ^ (r >> 3) ^ (r >> 12)) & 1;
    *state = (r >> 1) | (bit << 15);
    return (*state >> (16 - bits)) & ((1 << bits) - 1);
}
B200_HD int fg_round2(int x, int sh) { return (x + ((1 << sh) >> 1)) >> sh; }

// ---- grain LUT generation, parallel ------------------------------------------------------------------------
// The reference fills a LUT from ONE 16-bit LFSR in raster order and then runs the auto-regressive filter in raster
// order (reference src/filmgrain_tmpl.c:50-160). Both are parallelised without changing a bit:
//   * the LFSR step is linear over GF(2): state_{n+k} = A^k state_n. The images of the 16 basis states under A^(2^b)
//     are built once per launch (16 threads per squaring), every LUT row then jumps straight to its first state
//     (row y starts after y * width draws) and fills its own 82 / 44 entries: one thread per row, all planes at once;
//   * the AR filter of pixel (x, y) needs the filtered (x + lag, y - 1): rows run as a skewed wavefront, row y trailing
//     row y - 1 by lag + 1 columns, in SHARED memory (one barrier + <= 24 multiply-adds per step); luma first, then both
//     chroma planes side by side (they read the filtered luma grain).
// (The LFSR chain on one thread and the wavefront in global memory, the first form, was several times slower.)
struct FgJump { uint16_t t[14][16]; };      // t[b][i] = A^(2^b) e_i ; 2^13 > 73 * 82 draws

B200_DEV unsigned fg_lfsr_step(unsigned r) { return (r >> 1) | ((((r >> 0) ^ (r >> 1) ^ (r >> 3) ^ (r >> 12)) & 1u) << 15); }

// called by the whole CTA
B200_DEV void fg_build_jump(FgJump &J)
{
    const int i = threadIdx.x;
    if (i < 16) J.t[0][i] = (uint16_t)fg_lfsr_step(1u << i);
    __syncthreads();
    for (int b = 1; b < 14; b++) {
        if (i < 16) {
            const unsigned v = J.t[b - 1][i];
            unsigned r = 0;
#pragma unroll
            for (int k = 0; k < 16; k++) if ((v >> k) & 1) r ^= J.t[b - 1][k];
            J.t[b][i] = (uint16_t)r;
        }
        __syncthreads();
    }
}

B200_DEV unsigned fg_lfsr_advance(const FgJump &J, unsigned s, int n)
{
    for (int b = 0; n; b++, n >>= 1) {
        if (!(n & 1)) continue;
        unsigned r = 0;
#pragma unroll
        for (int k = 0; k < 16; k++) if ((s >> k) & 1) r ^= J.t[b][k];
        s = r;
    }
    return s;
}

// one LUT row of raw grain (thread-level): row y of plane uv (< 0: luma)
B200_DEV void fg_fill_row(int16_t *buf, const FgJump &J, const B200FilmGrainData &d, int uv, int cw, int y, int shift)
{
    unsigned seed = fg_lfsr_advance(J, d.seed ^ (uv < 0 ? 0u : uv ? 0x49d8u : 0xb524u), y * cw);
    for (int x = 0; x < cw; x++) buf[y * GW + x] = (int16_t)fg_round2(b200_gaussian_sequence[fg_rnd(11, &seed)], shift);
}

// one wavefront step of the AR filter for LUT row y (thread-level); the caller separates steps with barriers
B200_DEV void fg_ar_step(int16_t *buf, const int16_t *buf_y, const B200FilmGrainData &d, int uv, int subx, int suby,
                         int cw, int ch, int y, int t, int gmin, int gmax)
{
    const int lag = d.ar_coeff_lag;
    const int x = t - (lag + 1) * (y - 3) + 3;
    if (y >= ch || x < 3 || x >= cw - 3) return;
    const int8_t *coeff = uv < 0 ? d.ar_coeffs_y : d.ar_coeffs_uv[uv];
    int sum = 0;
    for (int dy = -lag; dy <= 0; dy++)
        for (int dx = -lag; dx <= lag; dx++) {
            if (!dx && !dy) {
                if (uv >= 0 && d.num_y_points) {
                    int luma = 0;
                    const int lx = ((x - 3) << subx) + 3, ly = ((y - 3) << suby) + 3;
                    for (int i = 0; i <= suby; i++)
                        for (int j = 0; j <= subx; j++) luma += buf_y[(ly + i) * GW + lx + j];
                    sum += fg_round2(luma, subx + suby) * *coeff;
                }
                break;
            }
            sum += *(coeff++) * buf[(y + dy) * GW + x + dx];
        }
    buf[y * GW + x] = (int16_t)iclip(buf[y * GW + x] + fg_round2(sum, (int)d.ar_coeff_shift), gmin, gmax);
}

B200_DEV int fg_ar_steps(const B200FilmGrainData &d, int cw, int ch) { return (cw - 6) + (d.ar_coeff_lag + 1) * (ch - 3 - 1); }

// grain LUT of one plane; buf / buf_y are int16 working copies (pitch GW) in shared or global memory. Called by a whole
// CTA of >= 73 threads (Level 1: one plane per launch).
B200_DEV void fg_generate(int16_t *buf, const int16_t *buf_y, const B200FilmGrainData &d, int uv, int subx, int suby, int b8, FgJump &J)
{
    const int cw = uv >= 0 && subx ? 44 : GW, ch = uv >= 0 && suby ? 38 : GH;
    const int shift = 4 - b8 + d.grain_scale_shift;
    const int gmin = -(128 << b8), gmax = (128 << b8) - 1;
    fg_build_jump(J);
    if ((int)threadIdx.x < ch) fg_fill_row(buf, J, d, uv, cw, threadIdx.x, shift);
    __syncthreads();
    const int steps = fg_ar_steps(d, cw, ch);
    for (int t = 0; t < steps; t++) {
        fg_ar_step(buf, buf_y, d, uv, subx, suby, cw, ch, threadIdx.x + 3, t, gmin, gmax);
        __syncthreads();
    }
}

B200_DEV void fg_scaling(int bitdepth, const uint8_t (*points)[2], int num, uint8_t *scaling)
{
    const int shift_x = bitdepth - 8, size = 1 << bitdepth, tid = threadIdx.x, nt = blockDim.x;
    if (!num) { for (int i = tid; i < size; i += nt) scaling[i] = 0; __syncthreads(); return; }
    // phase 1: entries at multiples of (1 << shift_x), plus the flat head / tail
    for (int i = tid; i < size; i += nt) {
        const int v = i >> shift_x;
        if (v < points[0][0]) scaling[i] = points[0][1];
        else if (v >= points[num - 1][0]) scaling[i] = points[num - 1][1];
        else if (!(i & ((1 << shift_x) - 1))) {
            int k = 0;
            while (k < num - 2 && v >= points[k + 1][0]) k++;
            const int bx = points[k][0], by = points[k][1], dx = points[k + 1][0] - bx, dy = points[k + 1][1] - by;
            const int delta = dy * ((0x10000 + (dx >> 1)) / dx);
            scaling[i] = (uint8_t)(by + ((0x8000 + (v - bx) * delta) >> 16));
        }
    }
    __syncthreads();
    if (shift_x) {   // phase 2: linear fill between the coarse entries (reference :83-96)
        const int pad = 1 << shift_x, rnd = pad >> 1;
        for (int i = tid; i < size; i += nt) {
            const int v = i >> shift_x, n = i & (pad - 1);
            if (n && v >= points[0][0] && v < points[num - 1][0]) {
                const int base = i - n;
                const int range = (int)scaling[base + pad] - (int)scaling[base];
                scaling[i] = (uint8_t)(scaling[base] + ((rnd + n * range) >> shift_x));
            }
        }
        __syncthreads();
    }
}

constexpr int kFgPrepThreads = 256;
__global__ void __launch_bounds__(kFgPrepThreads) fg_prep_kernel(const __grid_constant__ B200FgFrame f, int bdmax)
{
    FgScratch *S = (FgScratch *)f.scratch;
    const B200FilmGrainData &d = f.data;
    const int bitdepth = 32 - __clz(bdmax), b8 = bitdepth - 8;
    const int tid = threadIdx.x;
    __shared__ FgJump J;
    __shared__ int16_t sbuf[3][(GH + 1) * GW];
    const bool has_uv[2] = { d.num_uv_points[0] || d.chroma_scaling_from_luma, d.num_uv_points[1] || d.chroma_scaling_from_luma };
    const int cw = f.ss_hor ? 44 : GW, ch = f.ss_ver ? 38 : GH;
    const int shift = 4 - b8 + d.grain_scale_shift;
    const int gmin = -(128 << b8), gmax = (128 << b8) - 1;
    fg_build_jump(J);
    // raw grain: one thread per LUT row, the three planes side by side (threads 0.., 80.., 160..)
    {
        const int pl = tid < 80 ? 0 : tid < 160 ? 1 : 2, y = tid - 80 * pl;
        if (pl == 0) { if (y < GH) fg_fill_row(sbuf[0], J, d, -1, GW, y, shift); }
        else if (has_uv[pl - 1] && y < ch) fg_fill_row(sbuf[pl], J, d, pl - 1, cw, y, shift);
    }
    __syncthreads();
    // AR filter: luma, then the two chroma planes together
    for (int t = 0, n = fg_ar_steps(d, GW, GH); t < n; t++) {
        if (tid < 80) fg_ar_step(sbuf[0], nullptr, d, -1, 0, 0, GW, GH, tid + 3, t, gmin, gmax);
        __syncthreads();
    }
    if (has_uv[0] || has_uv[1]) {
        for (int t = 0, n = fg_ar_steps(d, cw, ch); t < n; t++) {
            const int pl = tid < 80 ? 0 : tid < 160 ? 1 : 2;
            if (pl && has_uv[pl - 1]) fg_ar_step(sbuf[pl], sbuf[0], d, pl - 1, f.ss_hor, f.ss_ver, cw, ch, tid - 80 * pl + 3, t, gmin, gmax);
            __syncthreads();
        }
    }
    for (int pl = 0; pl < 3; pl++)
        if (pl == 0 || has_uv[pl - 1])
            for (int i = tid; i < GH * GW; i += kFgPrepThreads) S->lut[pl][i] = sbuf[pl][i];
    if (d.num_y_points || d.chroma_scaling_from_luma) fg_scaling(bitdepth, d.y_points, d.num_y_points, S->scaling[0]);
    for (int uv = 0; uv < 2; uv++)
        if (d.num_uv_points[uv]) fg_scaling(bitdepth, d.uv_points[uv], d.num_uv_points[uv], S->scaling[1 + uv]);
    // block offsets: row r, k-th draw of the row's LFSR (reference :190-214)
    const int rows = (f.h + 31) / 32, nbx = (f.w + 31) / 32;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) {
        unsigned s = d.seed;
        s ^= (unsigned)(((r * 37 + 178) & 0xFF) << 8);
        s ^= (unsigned)((r * 173 + 105) & 0xFF);
        for (int k = 0; k < nbx; k++) S->offsets[r * kMaxBlocksX + k] = (uint8_t)fg_rnd(8, &s);
    }
}

B200_DEV int fg_sample(const int16_t *lut, int randval, int subx, int suby, int x, int y) {
    const int offx = 3 + (2 >> subx) * (3 + (randval >> 4)), offy = 3 + (2 >> suby) * (3 + (randval & 0xF));
    return lut[(offy + y) * GW + offx + x];
}

// grain of pixel (x, y) of a strip (plane units); off_cur / off_prev: this strip's / the previous strip's offsets
B200_DEV int fg_pixel_grain(const B200FilmGrainData &d, const int16_t *lut, const uint8_t *off_cur, const uint8_t *off_prev,
                            int b8, int row, int x, int y, int pw, int bh, int sx, int sy)
{
    const int gmin = -(128 << b8), gmax = (128 << b8) - 1;
    const int bs = 32 >> sx, bsy = 32 >> sy, bi = x >> (5 - sx), xin = x & (bs - 1);
    const int bw = imin(bs, pw - bi * bs);
    const bool xov = d.overlap_flag && bi && xin < imin(2 >> sx, bw);
    const bool yov = d.overlap_flag && row > 0 && y < imin(2 >> sy, bh);
    // blend weights (reference :221, :313-316): [sub][position] -> {old, new}
    const int wx0 = sx ? 23 : (xin ? 17 : 27), wx1 = sx ? 22 : (xin ? 27 : 17);
    const int wy0 = sy ? 23 : (y ? 17 : 27), wy1 = sy ? 22 : (y ? 27 : 17);
    int g = fg_sample(lut, off_cur[bi], sx, sy, xin, y);
    if (xov) {
        const int old = fg_sample(lut, off_cur[bi - 1], sx, sy, xin + bs, y);
        g = iclip(fg_round2(old * wx0 + g * wx1, 5), gmin, gmax);
    }
    if (yov) {
        int top = fg_sample(lut, off_prev[bi], sx, sy, xin, y + bsy);
        if (xov) {
            const int old = fg_sample(lut, off_prev[bi - 1], sx, sy, xin + bs, y + bsy);
            top = iclip(fg_round2(old * wx0 + top * wx1, 5), gmin, gmax);
        }
        g = iclip(fg_round2(top * wy0 + g * wy1, 5), gmin, gmax);
    }
    return g;
}

// Writes out[k] = sample s[k] of plane pl (0: luma) with grain value g[k] applied, k < n <= N (reference :181-226,
// :292-352). The scaling index is s[k] for luma; for chroma it is the co-located luma sample luma(k, 0), averaged with its
// right neighbour luma(k, 1) when subsampled horizontally, and unless chroma scaling comes from luma combined with s[k].
// luma(k, j) is the caller's load, so the caller decides how a missing right neighbour (odd widths) is replicated.
template <int N, class pixel, class Luma>
B200_DEV void fg_apply_samples(const B200FilmGrainData &d, const uint8_t *scaling, int pl, int is_id, int sx, int b8, int bdmax,
                               int n, const int (&s)[N], const int (&g)[N], Luma luma, pixel *out)
{
    int mn, mx;
    if (d.clip_to_restricted_range) { mn = 16 << b8; mx = (pl && !is_id ? 240 : 235) << b8; }
    else { mn = 0; mx = bdmax; }
    int val[N];
#pragma unroll
    for (int k = 0; k < N; k++) val[k] = s[k];
    if (pl) {
#pragma unroll
        for (int k = 0; k < N; k++) {
            if (k >= n) break;
            int avg = luma(k, 0);
            if (sx) avg = (avg + luma(k, 1) + 1) >> 1;
            val[k] = avg;
            if (!d.chroma_scaling_from_luma) {
                const int combined = avg * d.uv_luma_mult[pl - 1] + s[k] * d.uv_mult[pl - 1];
                val[k] = iclip((combined >> 6) + d.uv_offset[pl - 1] * (1 << b8), 0, bdmax);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
        if (k >= n) break;
        const int noise = fg_round2((int)scaling[val[k]] * g[k], d.scaling_shift);
        out[k] = (pixel)iclip(s[k] + noise, mn, mx);
    }
}

// grid: (ceil(w / 128), ceil(h / 8), 3 planes); block (32, 8); a thread owns 4 consecutive samples of one row
// (always inside one 32-wide grain block: 4 divides the block width of every layout)
template <bool HBD>
__global__ void __launch_bounds__(256) fg_apply_kernel(const __grid_constant__ B200FgFrame f, int bdmax)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const int pl = blockIdx.z;
    const B200FilmGrainData &d = f.data;
    const int sx = pl ? f.ss_hor : 0, sy = pl ? f.ss_ver : 0;
    const int pw = (f.w + sx) >> sx, ph = (f.h + sy) >> sy;
    const int x0 = (blockIdx.x * 32 + threadIdx.x) * 4, yp = blockIdx.y * 8 + threadIdx.y;
    if (x0 >= pw || yp >= ph) return;
    const int nx = imin(4, pw - x0);
    const pixel *in = (const pixel *)f.in + f.plane_off[pl] + (ptrdiff_t)yp * f.stride[pl] + x0;
    pixel *out = (pixel *)f.out + f.plane_off[pl] + (ptrdiff_t)yp * f.stride[pl] + x0;
    int s[4];
#pragma unroll
    for (int k = 0; k < 4; k++) s[k] = k < nx ? (int)in[k] : 0;
    const bool grained = pl ? (d.chroma_scaling_from_luma || d.num_uv_points[pl - 1]) : d.num_y_points != 0;
    if (!grained) {
#pragma unroll
        for (int k = 0; k < 4; k++) if (k < nx) out[k] = (pixel)s[k];
        return;
    }
    const FgScratch *S = (const FgScratch *)f.scratch;
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    const int srows = 32 >> sy, bs = 32 >> sx;        // strip height / block width in plane samples
    const int row = yp >> (5 - sy), y = yp & (srows - 1);
    const int bh_l = imin(f.h - row * 32, 32), bh = (bh_l + sy) >> sy;
    const uint8_t *off_cur = &S->offsets[row * kMaxBlocksX], *off_prev = &S->offsets[(row ? row - 1 : 0) * kMaxBlocksX];
    const int bi = x0 >> (5 - sx), xin0 = x0 & (bs - 1);
    int g[4];
    const bool any_ov = d.overlap_flag && ((bi && xin0 < (2 >> sx)) || (row > 0 && y < imin(2 >> sy, bh)));
    if (any_ov) {
#pragma unroll
        for (int k = 0; k < 4; k++) g[k] = k < nx ? fg_pixel_grain(d, S->lut[pl], off_cur, off_prev, b8, row, x0 + k, y, pw, bh, sx, sy) : 0;
    } else {      // the common case: 4 consecutive samples of this block's window into the grain LUT
        const int rv = off_cur[bi];
        const int offx = 3 + (2 >> sx) * (3 + (rv >> 4)), offy = 3 + (2 >> sy) * (3 + (rv & 0xF));
        const int16_t *gp = S->lut[pl] + (offy + y) * GW + offx + xin0;
#pragma unroll
        for (int k = 0; k < 4; k++) g[k] = gp[k];
    }
    const uint8_t *scaling = S->scaling[0];
    if (pl && !d.chroma_scaling_from_luma) scaling = S->scaling[pl];
    fg_apply_samples(d, scaling, pl, f.is_id, sx, b8, bdmax, nx, s, g, [&](int k, int j) {
        const pixel *luma = (const pixel *)f.in + f.plane_off[0] + (ptrdiff_t)(yp << sy) * f.stride[0];
        const int lx = (x0 + k) << sx;
        return j ? (int)luma[imin(lx + 1, f.w - 1)] : (int)luma[lx];   // odd widths: replicate the last column (:196-203)
    }, out);
}

// ---- Level-1 kernels ----
__global__ void __launch_bounds__(128) fg_gen_l1_kernel(int16_t *buf, const int16_t *buf_y, B200FilmGrainData d, int uv, int subx, int suby, int bdmax)
{
    __shared__ FgJump J;
    fg_generate(buf, buf_y, d, uv, subx, suby, (32 - __clz(bdmax)) - 8, J);
}

template <bool HBD>
__global__ void fg_strip_l1_kernel(typename Bd<HBD>::pixel *dst, const typename Bd<HBD>::pixel *src, const typename Bd<HBD>::pixel *luma,
                                   B200FilmGrainData d, int pw, int lw, const uint8_t *scaling, const int16_t *lut, int bh, int row_num,
                                   int uv, int is_id, int sx, int sy, int bdmax)
{
    __shared__ uint8_t off[2][kMaxBlocksX];
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    if (threadIdx.x < 2) {
        const int r = row_num - threadIdx.x;
        unsigned s = d.seed;
        s ^= (unsigned)(((r * 37 + 178) & 0xFF) << 8);
        s ^= (unsigned)((r * 173 + 105) & 0xFF);
        const int nbx = (pw + (32 >> sx) - 1) / (32 >> sx);
        for (int k = 0; k < nbx; k++) off[threadIdx.x][k] = (uint8_t)fg_rnd(8, &s);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < pw * bh; i += blockDim.x) {
        const int y = i / pw, x = i - y * pw;
        const int g = fg_pixel_grain(d, lut, off[0], off[1], b8, row_num, x, y, pw, bh, sx, sy);
        // dav1d pads an odd-width luma row, so the right neighbour of the last column is always there
        const int lx = (y << sy) * lw + (x << sx);
        const int s[1] = { src[i] }, gr[1] = { g };
        fg_apply_samples(d, scaling, uv + 1, is_id, sx, b8, bdmax, 1, s, gr, [&](int, int j) { return (int)luma[lx + j]; }, dst + i);
    }
}

}  // namespace b200

using namespace b200;

extern "C" {

static int fg_check(int bdmax, const B200FgFrame *f, const char *who)
{
    if (int r = check_bdmax(bdmax, who)) return r;
    const int rows = (f->h + 31) / 32, nbx = (f->w + 31) / 32;
    if (nbx > kMaxBlocksX || (size_t)rows * kMaxBlocksX > sizeof(((FgScratch *)0)->offsets)) { b200_set_error("%s: picture too large", who); return -2; }
    return 0;
}

int b200_fg_prep(int bdmax, const B200FgFrame *f, void *stream)
{
    if (int r = fg_check(bdmax, f, "b200_fg_prep")) return r;
    B200_LAUNCH(fg_prep_kernel, dim3(1), dim3(kFgPrepThreads), 0, (cudaStream_t)stream, *f, bdmax);
    b200_count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int b200_fg_apply(int bdmax, const B200FgFrame *f, void *stream)
{
    if (int r = fg_check(bdmax, f, "b200_fg_apply")) return r;
    return launch_hbd(bdmax, Launch::pdl, dim3((f->w + 127) / 128, (f->h + 7) / 8, 3), dim3(32, 8), 0, (cudaStream_t)stream,
                      [&](auto hbd) { return std::make_tuple(fg_apply_kernel<hbd>, *f, bdmax); });
}

int b200_fg_apply_frame(int bdmax, const B200FgFrame *f, void *stream)
{
    int r = b200_fg_prep(bdmax, f, stream);
    return r ? r : b200_fg_apply(bdmax, f, stream);
}

// a grain LUT of 8-bit (int8) or high bit-depth (int16) entries, widened to the (GH + 1) x GW int16 the kernels read
static void widen_lut(int16_t *dst, const void *lut, bool hbd)
{
    for (int i = 0; i < GH * GW; i++) dst[i] = hbd ? ((const int16_t *)lut)[i] : ((const int8_t *)lut)[i];
    memset(dst + GH * GW, 0, GW * sizeof(int16_t));
}

int b200_fg_generate_grain(void *buf, const void *buf_y, const B200FilmGrainData *data, int uv, int ss_hor, int ss_ver, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_fg_generate_grain")) return r;
    Level1 L;
    const bool hbd = bdmax > 255;
    const size_t n = (GH + 1) * GW;
    int16_t *lut = (int16_t *)L.host(n * 2);
    void *d_buf, *d_y;
    if (!lut || !(d_buf = L.dev(0, n * 2))) return -1;
    if (uv >= 0) widen_lut(lut, buf_y, hbd);
    if (!(d_y = uv >= 0 ? L.upload(1, lut, n * 2) : L.dev(1, n * 2))) return -1;
    const int cw = uv >= 0 && ss_hor ? 44 : GW, ch = uv >= 0 && ss_ver ? 38 : GH;
    B200_LAUNCH(fg_gen_l1_kernel, dim3(1), dim3(128), 0, (cudaStream_t)0, (int16_t *)d_buf, (const int16_t *)d_y, *data, uv, ss_hor, ss_ver, bdmax);
    b200_count_launch();
    B200_CUDA_OK(cudaGetLastError());
    int16_t grain[(GH + 1) * GW];
    if (L.download_rect(0, grain, 0, 1, 1, sizeof(grain))) return -1;
    for (int y = 0; y < ch; y++)
        for (int x = 0; x < cw; x++) {
            if (hbd) ((int16_t *)buf)[y * GW + x] = grain[y * GW + x];
            else ((int8_t *)buf)[y * GW + x] = (int8_t)grain[y * GW + x];
        }
    return 0;
}

static int fg_strip_l1(void *dst_row, const void *src_row, ptrdiff_t stride, const B200FilmGrainData *data, size_t pw_,
                       const uint8_t *scaling, const void *grain_lut, int bh, int row_num, const void *luma_row,
                       ptrdiff_t luma_stride, int uv, int is_id, int sx, int sy, int bdmax)
{
    if (int r = check_bdmax(bdmax, "fg strip")) return r;
    const int pw = (int)pw_;
    if (pw < 1 || pw > 16384 || bh < 1 || bh > 32) { b200_set_error("fg strip: bad geometry"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    enum { SRC, DST, LUMA, SCAL, LUT };
    void *src, *dst, *luma = nullptr, *scal, *lut;
    if (!(src = L.upload_rect(SRC, src_row, stride, pw, bh, px)) || !(dst = L.dev(DST, (size_t)pw * bh * px))) return -1;
    int lw = 0;
    if (uv >= 0) {
        lw = pw << sx;
        if (!(luma = L.upload_rect(LUMA, luma_row, luma_stride, lw, ((bh - 1) << sy) + 1, px))) return -1;
    }
    const size_t lut_bytes = (GH + 1) * GW * 2;
    int16_t *lut16 = (int16_t *)L.host(lut_bytes);
    if (!lut16) return -1;
    widen_lut(lut16, grain_lut, bdmax > 255);
    if (!(lut = L.upload(LUT, lut16, lut_bytes)) || !(scal = L.upload(SCAL, scaling, bdmax > 255 ? 4096 : 256))) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3(1), dim3(256), 0, 0, [&](auto hbd) {
            typedef typename Bd<hbd>::pixel pixel;
            return std::make_tuple(fg_strip_l1_kernel<hbd>, (pixel *)dst, (const pixel *)src, (const pixel *)luma, *data, pw, lw,
                                   (const uint8_t *)scal, (const int16_t *)lut, bh, row_num, uv, is_id, sx, sy, bdmax);
        }))
        return r;
    return L.download_rect(DST, dst_row, stride, pw, bh, px);
}

int b200_fgy_32x32xn(void *dst_row, const void *src_row, ptrdiff_t stride, const B200FilmGrainData *data, size_t pw,
                     const uint8_t *scaling, const void *grain_lut, int bh, int row_num, int bdmax)
{
    return fg_strip_l1(dst_row, src_row, stride, data, pw, scaling, grain_lut, bh, row_num, nullptr, 0, -1, 0, 0, 0, bdmax);
}
int b200_fguv_32x32xn(void *dst_row, const void *src_row, ptrdiff_t stride, const B200FilmGrainData *data, size_t pw,
                      const uint8_t *scaling, const void *grain_lut, int bh, int row_num, const void *luma_row,
                      ptrdiff_t luma_stride, int uv_pl, int is_id, int ss_hor, int ss_ver, int bdmax)
{
    return fg_strip_l1(dst_row, src_row, stride, data, pw, scaling, grain_lut, bh, row_num, luma_row, luma_stride, uv_pl, is_id, ss_hor, ss_ver, bdmax);
}

}  // extern "C"

namespace {
template <int BD> void ggy(void *buf, const B200FilmGrainData *d) { if (b200_fg_generate_grain(buf, nullptr, d, -1, 0, 0, BD)) die("generate_grain_y"); }
void ggy16(void *buf, const B200FilmGrainData *d, int bd) { if (b200_fg_generate_grain(buf, nullptr, d, -1, 0, 0, bd)) die("generate_grain_y"); }
template <int SX, int SY> void gguv8(void *buf, const void *by, const B200FilmGrainData *d, intptr_t uv) { if (b200_fg_generate_grain(buf, by, d, (int)uv, SX, SY, 255)) die("generate_grain_uv"); }
template <int SX, int SY> void gguv16(void *buf, const void *by, const B200FilmGrainData *d, intptr_t uv, int bd) { if (b200_fg_generate_grain(buf, by, d, (int)uv, SX, SY, bd)) die("generate_grain_uv"); }
void fgy8(uint8_t *d, const uint8_t *s, ptrdiff_t st, const B200FilmGrainData *fd, size_t pw, const uint8_t *sc, const void *lut, int bh, int row) { if (b200_fgy_32x32xn(d, s, st, fd, pw, sc, lut, bh, row, 255)) die("fgy_32x32xn"); }
void fgy16(uint16_t *d, const uint16_t *s, ptrdiff_t st, const B200FilmGrainData *fd, size_t pw, const uint8_t *sc, const void *lut, int bh, int row, int bd) { if (b200_fgy_32x32xn(d, s, st, fd, pw, sc, lut, bh, row, bd)) die("fgy_32x32xn"); }
template <int SX, int SY> void fguv8(uint8_t *d, const uint8_t *s, ptrdiff_t st, const B200FilmGrainData *fd, size_t pw, const uint8_t *sc, const void *lut, int bh, int row, const uint8_t *l, ptrdiff_t ls, int uv, int is_id) { if (b200_fguv_32x32xn(d, s, st, fd, pw, sc, lut, bh, row, l, ls, uv, is_id, SX, SY, 255)) die("fguv_32x32xn"); }
template <int SX, int SY> void fguv16(uint16_t *d, const uint16_t *s, ptrdiff_t st, const B200FilmGrainData *fd, size_t pw, const uint8_t *sc, const void *lut, int bh, int row, const uint16_t *l, ptrdiff_t ls, int uv, int is_id, int bd) { if (b200_fguv_32x32xn(d, s, st, fd, pw, sc, lut, bh, row, l, ls, uv, is_id, SX, SY, bd)) die("fguv_32x32xn"); }
}
extern "C" {
void b200_film_grain_dsp_init_8bpc(B200FilmGrainDSPContext *c) {
    c->generate_grain_y = (void *)ggy<255>;
    c->generate_grain_uv[0] = (void *)gguv8<1, 1>; c->generate_grain_uv[1] = (void *)gguv8<1, 0>; c->generate_grain_uv[2] = (void *)gguv8<0, 0>;
    c->fgy_32x32xn = (void *)fgy8;
    c->fguv_32x32xn[0] = (void *)fguv8<1, 1>; c->fguv_32x32xn[1] = (void *)fguv8<1, 0>; c->fguv_32x32xn[2] = (void *)fguv8<0, 0>;
}
void b200_film_grain_dsp_init_16bpc(B200FilmGrainDSPContext *c) {
    c->generate_grain_y = (void *)ggy16;
    c->generate_grain_uv[0] = (void *)gguv16<1, 1>; c->generate_grain_uv[1] = (void *)gguv16<1, 0>; c->generate_grain_uv[2] = (void *)gguv16<0, 0>;
    c->fgy_32x32xn = (void *)fgy16;
    c->fguv_32x32xn[0] = (void *)fguv16<1, 1>; c->fguv_32x32xn[1] = (void *)fguv16<1, 0>; c->fguv_32x32xn[2] = (void *)fguv16<0, 0>;
}
}
