// CDEF (dav1d Dav1dCdefDSPContext; reference src/cdef_tmpl.c:37-305, driver src/cdef_apply_tmpl.c).
//
// Frame-wide and out of place: one warp owns one 8x8 luma block and its chroma blocks. The warp
// finds the block's direction/variance from the (pre-CDEF) luma samples, derives the strengths
// exactly like dav1d_cdef_brow, then every lane filters its pixels reading taps straight from the
// source picture; taps outside the block's available rectangle (picture edges) are skipped, which is
// what the reference's INT16_MIN padding achieves. Unfiltered blocks are copied through.
#include "host_util.h"

namespace b200 {

// taps of direction d: [k = near/far][dy, dx]  (reference src/tables.c:400-413, stride 12 removed)
__constant__ int8_t c_cdef_off[8][2][2] = {
    { { -1, 1 }, { -2, 2 } }, { { 0, 1 }, { -1, 2 } }, { { 0, 1 }, { 0, 2 } }, { { 0, 1 }, { 1, 2 } },
    { { 1, 1 }, { 2, 2 } },   { { 1, 0 }, { 2, 1 } },  { { 1, 0 }, { 2, 0 } }, { { 1, 0 }, { 2, -1 } },
};
__constant__ uint16_t c_cdef_div[7] = { 840, 420, 280, 210, 168, 140, 120 };
__constant__ uint8_t c_uv_dir422[8] = { 7, 0, 2, 4, 5, 6, 6, 6 };

B200_DEV int cdef_constrain(int diff, int threshold, int shift) {
    const int adiff = iabs(diff);
    const int v = imin(adiff, imax(0, threshold - (adiff >> shift)));
    return diff < 0 ? -v : v;
}

struct CdefRect { int xmin, xmax, ymin, ymax; };   // available samples: [xmin, xmax) x [ymin, ymax)

template <bool HBD>
B200_DEV int cdef_pixel(const typename Bd<HBD>::pixel *__restrict__ plane, int stride, int ax, int ay,
                        const CdefRect &r, int pri, int sec, int dir, int pri_shift, int sec_shift, int pri_tap0)
{
    const int px = plane[(ptrdiff_t)ay * stride + ax];
    int sum = 0, mx = px, mn = px;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        if (pri) {
            const int tap = k ? ((pri_tap0 & 3) | 2) : pri_tap0;
            const int dy = c_cdef_off[dir][k][0], dx = c_cdef_off[dir][k][1];
#pragma unroll
            for (int s = -1; s <= 1; s += 2) {
                const int x = ax + s * dx, y = ay + s * dy;
                if (x < r.xmin || x >= r.xmax || y < r.ymin || y >= r.ymax) continue;
                const int p = plane[(ptrdiff_t)y * stride + x];
                sum += tap * cdef_constrain(p - px, pri, pri_shift);
                mn = imin(mn, p); mx = imax(mx, p);
            }
        }
        if (sec) {
            const int tap = 2 - k;
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int d2 = (dir + (j ? 6 : 2)) & 7;
                const int dy = c_cdef_off[d2][k][0], dx = c_cdef_off[d2][k][1];
#pragma unroll
                for (int s = -1; s <= 1; s += 2) {
                    const int x = ax + s * dx, y = ay + s * dy;
                    if (x < r.xmin || x >= r.xmax || y < r.ymin || y >= r.ymax) continue;
                    const int p = plane[(ptrdiff_t)y * stride + x];
                    sum += tap * cdef_constrain(p - px, sec, sec_shift);
                    mn = imin(mn, p); mx = imax(mx, p);
                }
            }
        }
    }
    int v = px + ((sum - (sum < 0) + 8) >> 4);
    if (pri && sec) v = iclip(v, mn, mx);
    return v;
}

// direction search over an 8x8 block held in shared memory as (px >> (bitdepth-8)) - 128;
// lanes 0..7 each own one direction's cost. Returns dir in all lanes, *var likewise.
B200_DEV int cdef_find_dir(const int *v, int lane, unsigned *var)
{
    unsigned cost = 0;
    if (lane < 8) {
        int sums[15];
#pragma unroll
        for (int i = 0; i < 15; i++) sums[i] = 0;
        for (int i = 0; i < 64; i++) {
            const int y = i >> 3, x = i & 7, p = v[i];
            int idx;
            switch (lane) {
            case 0: idx = y + x; break;
            case 1: idx = y + (x >> 1); break;
            case 2: idx = y; break;
            case 3: idx = 3 + y - (x >> 1); break;
            case 4: idx = 7 + y - x; break;
            case 5: idx = 3 - (y >> 1) + x; break;
            case 6: idx = x; break;
            default: idx = (y >> 1) + x; break;
            }
#pragma unroll
            for (int k = 0; k < 15; k++) if (k == idx) sums[k] += p;
        }
        if (lane == 2 || lane == 6) {
#pragma unroll
            for (int n = 0; n < 8; n++) cost += sums[n] * sums[n];
            cost *= 105;
        } else if (lane == 0 || lane == 4) {
#pragma unroll
            for (int n = 0; n < 7; n++) cost += (sums[n] * sums[n] + sums[14 - n] * sums[14 - n]) * c_cdef_div[n];
            cost += sums[7] * sums[7] * 105;
        } else {
#pragma unroll
            for (int m = 0; m < 5; m++) cost += sums[3 + m] * sums[3 + m];
            cost *= 105;
#pragma unroll
            for (int m = 0; m < 3; m++) cost += (sums[m] * sums[m] + sums[10 - m] * sums[10 - m]) * c_cdef_div[2 * m + 1];
        }
    }
    unsigned c[8];
#pragma unroll
    for (int n = 0; n < 8; n++) c[n] = __shfl_sync(0xffffffffu, cost, n);
    int best = 0; unsigned bc = c[0];
#pragma unroll
    for (int n = 1; n < 8; n++) if (c[n] > bc) { bc = c[n]; best = n; }
    unsigned opp = c[0];
#pragma unroll
    for (int n = 1; n < 8; n++) if (n == (best ^ 4)) opp = c[n];
    if ((best ^ 4) == 0) opp = c[0];
    *var = (bc - opp) >> 10;
    return best;
}

B200_DEV int cdef_adjust_strength(int strength, unsigned var) {
    if (!var) return 0;
    const int i = (var >> 6) ? imin(ulog2(var >> 6), 12) : 0;
    return (strength * (4 + i) + 8) >> 4;
}

// ---- frame kernel ---------------------------------------------------------------------------------
// One CTA filters a 64x32 luma tile (half a 64x64 superblock: cdef_idx is uniform) and the matching chroma
// tiles. The pre-CDEF samples are staged once in shared memory as 32-bit words holding the vertical pair
// (p[y][x], p[y+1][x]) in its two int16 halves, samples outside the picture replaced by a sentinel, so
// that a thread filters two vertically adjacent pixels at once with the 16x2 SIMD integer instructions
// (VIADD.16x2 / VIMNMX.S16x2[.RELU]) and every tap is a single conflict-free LDS.32.
//
// constrain(diff) = sign(diff) * min(|diff|, max(0, thr - (|diff| >> shift))) is accumulated as
//   P = relu(min(diff, t)), N = relu(min(-diff, t)), t = thr - (|diff| >> shift)   (sum = sum(P) - sum(N)),
// which needs no sign restore. The sentinel (-16384) keeps diff inside int16 and makes t <= 0 for every
// legal damping, so out-of-picture taps contribute nothing and are ignored by the signed max / unsigned min.
constexpr int kCdefTW = 64, kCdefTH = 32, kCdefPitch = kCdefTW + 8, kCdefRows = kCdefTH + 3;
constexpr int kCdefThreads = 256;
constexpr unsigned kCdefSentinel = 0xC000u;

struct CdefBlockInfo { int16_t y_pri, y_sec, uv_pri, uv_sec; int8_t y_dir, uv_dir, inside, pad;
                       uint8_t y_pri_shift, y_sec_shift, uv_pri_shift, uv_sec_shift; };   // constrain shifts, computed once per block

struct CdefShared {
    uint32_t tile[3][kCdefRows * kCdefPitch];   // pair rows -2 .. TH, columns -4 .. TW+3
    CdefBlockInfo info[32];
    int16_t off[8][2];                          // word offset of direction d, tap k (filled per plane pitch: constant pitch)
};

template <int D> B200_DEV unsigned cdef_dir_cost(const int (&v)[8][8])
{
    constexpr int NB = (D == 2 || D == 6) ? 8 : (D == 0 || D == 4) ? 15 : 11;
    int sums[NB];
#pragma unroll
    for (int i = 0; i < NB; i++) sums[i] = 0;
#pragma unroll
    for (int y = 0; y < 8; y++)
#pragma unroll
        for (int x = 0; x < 8; x++) {
            constexpr int dummy = 0; (void)dummy;
            const int idx = D == 0 ? y + x : D == 1 ? y + (x >> 1) : D == 2 ? y : D == 3 ? 3 + y - (x >> 1)
                          : D == 4 ? 7 + y - x : D == 5 ? 3 - (y >> 1) + x : D == 6 ? x : (y >> 1) + x;
            sums[idx] += v[y][x];
        }
    unsigned cost = 0;
    if (D == 2 || D == 6) {
#pragma unroll
        for (int n = 0; n < 8; n++) cost += sums[n] * sums[n];
        cost *= 105;
    } else if (D == 0 || D == 4) {
#pragma unroll
        for (int n = 0; n < 7; n++) cost += (sums[n] * sums[n] + sums[14 - n] * sums[14 - n]) * c_cdef_div[n];
        cost += sums[7] * sums[7] * 105;
    } else {
#pragma unroll
        for (int m = 0; m < 5; m++) cost += sums[3 + m] * sums[3 + m];
        cost *= 105;
#pragma unroll
        for (int m = 0; m < 3; m++) cost += (sums[m] * sums[m] + sums[10 - m] * sums[10 - m]) * c_cdef_div[2 * m + 1];
    }
    return cost;
}

// one tap pair (+off / -off) on two packed pixels
B200_DEV void cdef_tap2(const uint32_t *t, int idx, int off, unsigned negpx, unsigned thr1, int shift, unsigned smask, int tap,
                        unsigned &sumP, unsigned &sumN, unsigned &mx, unsigned &mn)
{
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const unsigned p = t[idx + (s ? -off : off)];
        const unsigned diff = __vadd2(p, negpx);
        const unsigned ndiff = __vadd2(~diff, 0x00010001u);
        const unsigned adiff = __vmaxs2(diff, ndiff);
        const unsigned th = __vadd2(thr1, ~((adiff >> shift) & smask));
        sumP += tap * __vimin_s16x2_relu(diff, th);
        sumN += tap * __vimin_s16x2_relu(ndiff, th);
        mx = __vmaxs2(mx, p);
        mn = __vminu2(mn, p);
    }
}

template <bool HBD>
#ifndef B200_CDEF_MINB
#define B200_CDEF_MINB 4
#endif
__global__ void __launch_bounds__(kCdefThreads, B200_CDEF_MINB) cdef_frame_kernel(const __grid_constant__ B200CdefFrame f, int bdmax, int tile_row0)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    __shared__ CdefShared S;
    const int tid = threadIdx.x;
    const int bx0 = blockIdx.x * 16, by0 = (tile_row0 + blockIdx.y) * 8;      // tile origin, 4-px units
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    const pixel *const src = (const pixel *)f.src;
    pixel *const dst = (pixel *)f.dst;

    // ---- stage the three planes (4 samples of two consecutive rows per thread and step)
#pragma unroll 1
    for (int pl = 0; pl < 3; pl++) {
        const int sh = pl ? f.ss_hor : 0, sv = pl ? f.ss_ver : 0;
        const int tw = kCdefTW >> sh, th = kCdefTH >> sv;
        const int availw = ((f.bw + 1) >> 1) * 8 >> sh, availh = ((f.bh + 1) >> 1) * 8 >> sv;
        const int x0 = bx0 * 4 >> sh, y0 = by0 * 4 >> sv;
        const int groups = (tw + 8) >> 2, rows = th + 3;
        const pixel *sp = src + f.plane_off[pl];
        const int st = f.stride[pl];
        const unsigned magic = recip16(groups);            // exact i / groups for i < 36 * 18
        for (int i = tid; i < groups * rows; i += kCdefThreads) {
            const int r = (int)((i * magic) >> 16), g = i - r * groups;
            const int x = x0 - 4 + g * 4, y = y0 - 2 + r;
            uint4 w;
            w.x = w.y = w.z = w.w = kCdefSentinel * 0x00010001u;
            if (x >= 0 && x < availw) {
                const bool ha = y >= 0 && y < availh, hb = y + 1 >= 0 && y + 1 < availh;
                if (HBD) {
                    uint2 qa, qb;
                    qa.x = qa.y = qb.x = qb.y = kCdefSentinel * 0x00010001u;
                    if (ha) qa = *(const uint2 *)(sp + (ptrdiff_t)y * st + x);
                    if (hb) qb = *(const uint2 *)(sp + (ptrdiff_t)(y + 1) * st + x);
                    // (a0 a1 | a2 a3) x (b0 b1 | b2 b3) -> (a0 b0) (a1 b1) (a2 b2) (a3 b3): one byte permute each
                    w.x = __byte_perm(qa.x, qb.x, 0x5410); w.y = __byte_perm(qa.x, qb.x, 0x7632);
                    w.z = __byte_perm(qa.y, qb.y, 0x5410); w.w = __byte_perm(qa.y, qb.y, 0x7632);
                } else {
                    const unsigned sent4 = 0;         // per-byte sentinel impossible: handled after the permutes
                    unsigned qa = sent4, qb = sent4;
                    if (ha) qa = *(const unsigned *)(sp + (ptrdiff_t)y * st + x);
                    if (hb) qb = *(const unsigned *)(sp + (ptrdiff_t)(y + 1) * st + x);
                    // bytes a_k, b_k -> halfwords (a_k | b_k << 16): two byte permutes per word
                    const unsigned t01 = __byte_perm(qa, qb, 0x5140), t23 = __byte_perm(qa, qb, 0x7362);   // a0 b0 a1 b1 | a2 b2 a3 b3
                    w.x = __byte_perm(t01, 0, 0x4140); w.y = __byte_perm(t01, 0, 0x4342);
                    w.z = __byte_perm(t23, 0, 0x4140); w.w = __byte_perm(t23, 0, 0x4342);
                    if (!ha) { w.x = (w.x & 0xffff0000u) | kCdefSentinel; w.y = (w.y & 0xffff0000u) | kCdefSentinel; w.z = (w.z & 0xffff0000u) | kCdefSentinel; w.w = (w.w & 0xffff0000u) | kCdefSentinel; }
                    if (!hb) { w.x = (w.x & 0xffffu) | kCdefSentinel << 16; w.y = (w.y & 0xffffu) | kCdefSentinel << 16; w.z = (w.z & 0xffffu) | kCdefSentinel << 16; w.w = (w.w & 0xffffu) | kCdefSentinel << 16; }
                }
            }
            *(uint4 *)&S.tile[pl][r * kCdefPitch + g * 4] = w;
        }
    }
    if (tid < 16) {
        const int d = tid >> 1, k = tid & 1;
        S.off[d][k] = (int16_t)(c_cdef_off[d][k][0] * kCdefPitch + c_cdef_off[d][k][1]);
    }
    __syncthreads();

    // ---- per-8x8 parameters: one thread per block (direction search over all 8 directions)
    if (tid < 32) {
        const int bxi = tid & 7, byi = tid >> 3;
        const int bx = bx0 + bxi * 2, by = by0 + byi * 2;
        CdefBlockInfo bi; bi.y_pri = bi.y_sec = bi.uv_pri = bi.uv_sec = 0; bi.y_dir = bi.uv_dir = 0; bi.pad = 0;
        bi.inside = bx < f.bw && by < f.bh;
        if (bi.inside) {
            int y_lvl = 0, uv_lvl = 0;
            const B200Av1Filter &m = f.mask[(by >> 5) * f.sb128w + (bx >> 5)];
            const int cdef_idx = m.cdef_idx[((by & 16) >> 3) + ((bx & 16) >> 4)];
            const uint16_t *nr = m.noskip_mask[(by & 30) >> 1];
            const unsigned noskip = (unsigned)nr[1] << 16 | nr[0];
            if (cdef_idx != -1 && (noskip & (3u << (bx & 30)))) { y_lvl = f.y_strength[cdef_idx]; uv_lvl = f.uv_strength[cdef_idx]; }
            const int y_pri = (y_lvl >> 2) << b8;
            int y_sec = y_lvl & 3; y_sec += y_sec == 3; y_sec <<= b8;
            const int uv_pri = (uv_lvl >> 2) << b8;
            int uv_sec = uv_lvl & 3; uv_sec += uv_sec == 3; uv_sec <<= b8;
            int dir = 0; unsigned var = 0;
            if (y_pri || uv_pri) {
                int v[8][8];
                const uint32_t *t = &S.tile[0][(2 + byi * 8) * kCdefPitch + 4 + bxi * 8];
#pragma unroll
                for (int y = 0; y < 8; y += 2)
#pragma unroll
                    for (int x = 0; x < 8; x++) {
                        const unsigned w = t[y * kCdefPitch + x];
                        v[y][x] = (int)((w & 0xffff) >> b8) - 128;
                        v[y + 1][x] = (int)((w >> 16) >> b8) - 128;
                    }
                unsigned c[8];
                c[0] = cdef_dir_cost<0>(v); c[1] = cdef_dir_cost<1>(v); c[2] = cdef_dir_cost<2>(v); c[3] = cdef_dir_cost<3>(v);
                c[4] = cdef_dir_cost<4>(v); c[5] = cdef_dir_cost<5>(v); c[6] = cdef_dir_cost<6>(v); c[7] = cdef_dir_cost<7>(v);
                unsigned bc = c[0];
#pragma unroll
                for (int n = 1; n < 8; n++) if (c[n] > bc) { bc = c[n]; dir = n; }
                unsigned opp = 0;
#pragma unroll
                for (int n = 0; n < 8; n++) if (n == (dir ^ 4)) opp = c[n];
                var = (bc - opp) >> 10;
            }
            if (y_pri) { bi.y_pri = (int16_t)cdef_adjust_strength(y_pri, var); bi.y_sec = (int16_t)y_sec; bi.y_dir = (int8_t)dir; }
            else bi.y_sec = (int16_t)y_sec;
            if (uv_lvl) {
                bi.uv_pri = (int16_t)uv_pri; bi.uv_sec = (int16_t)uv_sec;
                bi.uv_dir = (int8_t)(uv_pri ? ((f.ss_hor && !f.ss_ver) ? c_uv_dir422[dir] : dir) : 0);
            }
        }
        {   // shift = max(0, damping - ulog2(strength)) per class (luma damping, chroma damping - 1)
            const int dl = f.damping + b8, dc = dl - 1;
            bi.y_pri_shift = (uint8_t)(bi.y_pri ? imax(0, dl - ulog2(bi.y_pri)) : 0);
            bi.y_sec_shift = (uint8_t)(bi.y_sec ? dl - ulog2(bi.y_sec) : 0);
            bi.uv_pri_shift = (uint8_t)(bi.uv_pri ? imax(0, dc - ulog2(bi.uv_pri)) : 0);
            bi.uv_sec_shift = (uint8_t)(bi.uv_sec ? dc - ulog2(bi.uv_sec) : 0);
        }
        S.info[tid] = bi;
    }
    __syncthreads();

    // ---- filter: one thread per vertical pixel pair
#pragma unroll 1
    for (int pl = 0; pl < 3; pl++) {
        const int sh = pl ? f.ss_hor : 0, sv = pl ? f.ss_ver : 0;
        const int tw = kCdefTW >> sh, th = kCdefTH >> sv;
        const int x0 = bx0 * 4 >> sh, y0 = by0 * 4 >> sv;
        pixel *dp = dst + f.plane_off[pl];
        const int st = f.stride[pl];
        const uint32_t *t = S.tile[pl];
        const int twl = 6 - sh;                                   // tw = 64 >> sh is a power of two
        for (int i = tid; i < tw * (th >> 1); i += kCdefThreads) {
            const int yp = i >> twl, x = i & (tw - 1), y = yp * 2;
            const CdefBlockInfo bi = S.info[(y >> (3 - sv)) * 8 + (x >> (3 - sh))];
            if (!bi.inside) continue;
            const int idx = (y + 2) * kCdefPitch + x + 4;
            const unsigned px2 = t[idx];
            int o0 = px2 & 0xffff, o1 = px2 >> 16;
            const int pri = pl ? bi.uv_pri : bi.y_pri, sec = pl ? bi.uv_sec : bi.y_sec, dir = pl ? bi.uv_dir : bi.y_dir;
            if (pri | sec) {
                const unsigned negpx = __vadd2(~px2, 0x00010001u);
                unsigned sumP = 0, sumN = 0, mx = px2, mn = px2;
                if (pri) {
                    const int shift = pl ? bi.uv_pri_shift : bi.y_pri_shift;
                    const unsigned thr1 = (unsigned)(pri + 1) * 0x00010001u, smask = (0xffffu >> shift) * 0x00010001u;
                    const int tap0 = 4 - ((pri >> b8) & 1);
                    cdef_tap2(t, idx, S.off[dir][0], negpx, thr1, shift, smask, tap0, sumP, sumN, mx, mn);
                    cdef_tap2(t, idx, S.off[dir][1], negpx, thr1, shift, smask, (tap0 & 3) | 2, sumP, sumN, mx, mn);
                }
                if (sec) {
                    const int shift = pl ? bi.uv_sec_shift : bi.y_sec_shift;
                    const unsigned thr1 = (unsigned)(sec + 1) * 0x00010001u, smask = (0xffffu >> shift) * 0x00010001u;
                    const int d2 = (dir + 2) & 7, d6 = (dir + 6) & 7;
                    cdef_tap2(t, idx, S.off[d2][0], negpx, thr1, shift, smask, 2, sumP, sumN, mx, mn);
                    cdef_tap2(t, idx, S.off[d6][0], negpx, thr1, shift, smask, 2, sumP, sumN, mx, mn);
                    cdef_tap2(t, idx, S.off[d2][1], negpx, thr1, shift, smask, 1, sumP, sumN, mx, mn);
                    cdef_tap2(t, idx, S.off[d6][1], negpx, thr1, shift, smask, 1, sumP, sumN, mx, mn);
                }
                const int s0 = (int)(sumP & 0xffff) - (int)(sumN & 0xffff), s1 = (int)(sumP >> 16) - (int)(sumN >> 16);
                o0 += (s0 - (s0 < 0) + 8) >> 4;
                o1 += (s1 - (s1 < 0) + 8) >> 4;
                if (pri && sec) {
                    o0 = iclip(o0, (int)(mn & 0xffff), (int)(mx & 0xffff));
                    o1 = iclip(o1, (int)(mn >> 16), (int)(mx >> 16));
                }
            }
            pixel *o = dp + (ptrdiff_t)(y0 + y) * st + x0 + x;
            o[0] = (pixel)o0;
            o[st] = (pixel)o1;
        }
    }
}

// Level-1 kernels ---------------------------------------------------------------------------
template <bool HBD>
__global__ void cdef_fb_kernel(const typename Bd<HBD>::pixel *win, typename Bd<HBD>::pixel *out, int w, int h,
                               int pri, int sec, int dir, int damping, int edges, int bdmax)
{
    // win: dense (w+4) x (h+4) window, block at (2,2)
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    CdefRect r;
    r.xmin = (edges & B200_CDEF_HAVE_LEFT) ? 0 : 2; r.xmax = w + 2 + ((edges & B200_CDEF_HAVE_RIGHT) ? 2 : 0);
    r.ymin = (edges & B200_CDEF_HAVE_TOP) ? 0 : 2;  r.ymax = h + 2 + ((edges & B200_CDEF_HAVE_BOTTOM) ? 2 : 0);
    const int pri_tap0 = 4 - ((pri >> b8) & 1);
    const int pri_shift = pri ? imax(0, damping - ulog2(pri)) : 0;
    const int sec_shift = sec ? damping - ulog2(sec) : 0;
    for (int i = threadIdx.x; i < w * h; i += blockDim.x)
        out[i] = (typename Bd<HBD>::pixel)cdef_pixel<HBD>(win, w + 4, 2 + (i % w), 2 + (i / w), r, pri, sec, dir,
                                                          pri_shift, sec_shift, pri_tap0);
}

template <bool HBD>
__global__ void cdef_dir_kernel(const typename Bd<HBD>::pixel *img, int *out, int bdmax)
{
    __shared__ int v[64];
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    for (int i = threadIdx.x; i < 64; i += 32) v[i] = ((int)img[i] >> b8) - 128;
    __syncwarp();
    unsigned var;
    const int d = cdef_find_dir(v, threadIdx.x, &var);
    if (threadIdx.x == 0) { out[0] = d; out[1] = (int)var; }
}

}  // namespace b200

using namespace b200;

namespace b200 {
// tile rows [t0, t1) of the sweep: a tile row is 32 luma rows (16 subsampled chroma rows) and reads 2 rows beyond each side
int cdef_frame_rows(int bdmax, const B200CdefFrame *f, int t0, int t1, cudaStream_t stream)
{
    if (int r = check_bdmax(bdmax, "b200_cdef_frame")) return r;
    const size_t px = bdmax > 255 ? 2 : 1;
    for (int pl = 0; pl < 3; pl++)   // the tile loader reads 4 samples at a time
        if ((f->stride[pl] & 3) || (f->plane_off[pl] & 3) || ((uintptr_t)f->src * 1 % (4 * px))) { b200_set_error("b200_cdef_frame: planes must be 4-sample aligned"); return -2; }
    t0 = imax(t0, 0); t1 = imin(t1, (f->bh + 7) / 8);
    if (t1 <= t0) return 0;
    return launch_hbd(bdmax, Launch::pdl, dim3((f->bw + 15) / 16, t1 - t0), dim3(kCdefThreads), 0, stream,
                      [&](auto hbd) { return std::make_tuple(cdef_frame_kernel<hbd>, *f, bdmax, t0); });
}
}  // namespace b200

extern "C" {

int b200_cdef_frame(int bdmax, const B200CdefFrame *f, void *stream)
{
    return b200::cdef_frame_rows(bdmax, f, 0, (f->bh + 7) / 8, (cudaStream_t)stream);
}

int b200_cdef_dir(const void *img, ptrdiff_t stride, unsigned *var, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_cdef_dir")) return r;
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    void *in, *out;
    if (!(in = L.upload_rect(0, img, stride, 8, 8, px)) || !(out = L.dev(1, 8))) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3(1), dim3(32), 0, 0, [&](auto hbd) {
            return std::make_tuple(cdef_dir_kernel<hbd>, (const typename Bd<hbd>::pixel *)in, (int *)out, bdmax);
        }))
        return r;
    int res[2];
    if (L.download_rect(1, res, 0, 1, 1, sizeof(res))) return -1;
    *var = (unsigned)res[1];
    return res[0];   // 0..7
}

int b200_cdef_fb(void *dst, ptrdiff_t stride, const void *left, const void *top, const void *bottom, int pri,
                 int sec, int dir, int damping, int w, int h, int edges, int bdmax)
{
    if (int r = check_bdmax(bdmax, "b200_cdef_fb")) return r;
    if (!((w == 4 || w == 8) && (h == 4 || h == 8)) || dir < 0 || dir > 7 || (!pri && !sec)) { b200_set_error("b200_cdef_fb: bad arguments"); return -2; }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    const int ww = w + 4;
    uint8_t win[12 * 12 * 2];
    memset(win, 0, sizeof(win));
    auto put = [&](int wx, int wy, const void *p) { memcpy(win + ((size_t)wy * ww + wx) * px, p, px); };
    const int xs = (edges & B200_CDEF_HAVE_LEFT) ? -2 : 0, xe = w + ((edges & B200_CDEF_HAVE_RIGHT) ? 2 : 0);
    for (int y = 0; y < h; y++) {
        for (int x = 0; x < xe; x++) put(2 + x, 2 + y, (const uint8_t *)dst + (ptrdiff_t)y * stride + (ptrdiff_t)x * (ptrdiff_t)px);
        if (edges & B200_CDEF_HAVE_LEFT) for (int x = -2; x < 0; x++) put(2 + x, 2 + y, (const uint8_t *)left + (size_t)(y * 2 + 2 + x) * px);
    }
    if (edges & B200_CDEF_HAVE_TOP)
        for (int y = -2; y < 0; y++) for (int x = xs; x < xe; x++)
            put(2 + x, 2 + y, (const uint8_t *)top + (ptrdiff_t)(y + 2) * stride + (ptrdiff_t)x * (ptrdiff_t)px);
    if (edges & B200_CDEF_HAVE_BOTTOM)
        for (int y = 0; y < 2; y++) for (int x = xs; x < xe; x++)
            put(2 + x, 2 + h + y, (const uint8_t *)bottom + (ptrdiff_t)y * stride + (ptrdiff_t)x * (ptrdiff_t)px);
    void *in, *out;
    if (!(in = L.upload(0, win, (size_t)ww * (h + 4) * px)) || !(out = L.dev(1, 64 * 2))) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3(1), dim3(64), 0, 0, [&](auto hbd) {
            typedef typename Bd<hbd>::pixel pixel;
            return std::make_tuple(cdef_fb_kernel<hbd>, (const pixel *)in, (pixel *)out, w, h, pri, sec, dir, damping, edges, bdmax);
        }))
        return r;
    return L.download_rect(1, dst, stride, w, h, px);
}

}  // extern "C"

namespace {
int dir8(const uint8_t *img, ptrdiff_t st, unsigned *var) { int r = b200_cdef_dir(img, st, var, 255); if (r < 0) die("cdef.dir"); return r; }
int dir16(const uint16_t *img, ptrdiff_t st, unsigned *var, int bd) { int r = b200_cdef_dir(img, st, var, bd); if (r < 0) die("cdef.dir"); return r; }
template <int W, int H> void fb8(uint8_t *d, ptrdiff_t st, const void *l, const uint8_t *t, const uint8_t *b, int pri, int sec, int dir, int damp, int edges) {
    if (b200_cdef_fb(d, st, l, t, b, pri, sec, dir, damp, W, H, edges, 255)) die("cdef.fb");
}
template <int W, int H> void fb16(uint16_t *d, ptrdiff_t st, const void *l, const uint16_t *t, const uint16_t *b, int pri, int sec, int dir, int damp, int edges, int bd) {
    if (b200_cdef_fb(d, st, l, t, b, pri, sec, dir, damp, W, H, edges, bd)) die("cdef.fb");
}
}
extern "C" {
void b200_cdef_dsp_init_8bpc(B200CdefDSPContext *c) {
    c->dir = (void *)dir8; c->fb[0] = (void *)fb8<8, 8>; c->fb[1] = (void *)fb8<4, 8>; c->fb[2] = (void *)fb8<4, 4>;
}
void b200_cdef_dsp_init_16bpc(B200CdefDSPContext *c) {
    c->dir = (void *)dir16; c->fb[0] = (void *)fb16<8, 8>; c->fb[1] = (void *)fb16<4, 8>; c->fb[2] = (void *)fb16<4, 4>;
}
}
