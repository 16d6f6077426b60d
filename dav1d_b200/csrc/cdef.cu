// CDEF (dav1d Dav1dCdefDSPContext; reference src/cdef_tmpl.c:37-305, driver src/cdef_apply_tmpl.c).
//
// Frame-wide and out of place: one CTA owns a 64x32 luma tile and its chroma tiles, staged once in shared
// memory as vertical pixel pairs with a sentinel for samples outside the picture (see the frame kernel).
// Eight lanes per 8x8 block find its direction / variance from the (pre-CDEF) luma samples and derive the
// strengths exactly like dav1d_cdef_brow; the filter then reads every tap from the tile. Unfiltered blocks
// are copied through. The Level-1 slots run the same code: cdef.dir the same cdef_dir8, cdef.fb the same
// cdef_filter4 / cdef_store2 on a tile holding one block, the sentinel in every sample the edges flags mark
// unavailable (the reference's INT16_MIN padding).
#include "host_util.h"

namespace b200 {

// taps of direction d: [k = near/far][dy, dx]  (reference src/tables.c:400-413, stride 12 removed)
__constant__ int8_t c_cdef_off[8][2][2] = {
    { { -1, 1 }, { -2, 2 } }, { { 0, 1 }, { -1, 2 } }, { { 0, 1 }, { 0, 2 } }, { { 0, 1 }, { 1, 2 } },
    { { 1, 1 }, { 2, 2 } },   { { 1, 0 }, { 2, 1 } },  { { 1, 0 }, { 2, 0 } }, { { 1, 0 }, { 2, -1 } },
};
__constant__ uint16_t c_cdef_div[7] = { 840, 420, 280, 210, 168, 140, 120 };
__constant__ uint8_t c_uv_dir422[8] = { 7, 0, 2, 4, 5, 6, 6, 6 };

// Direction search (cdef_find_dir_c) of one 8x8 block by an aligned group of 8 lanes of one warp; lane y supplies row y
// as v[x] = (px >> (bitdepth - 8)) - 128. bins is the block's zeroed 8 x 16 int scratch in shared memory: bins[d * 16 + n]
// collects the sum along line n of direction d. The slanted lines are accumulated with shared-memory integer atomics
// (the order does not change a sum), the row sums (d = 2) and column sums (d = 6) are formed in registers. Lane d then
// evaluates direction d's cost as sum_n w(d, n) * s(d, n)^2, which equals the reference's grouped form modulo 2^32, and the
// argmax (first index on ties), the opposite cost and var are reduced over the 8 lanes. Returns dir in all 8 lanes, *var likewise.
B200_HD constexpr unsigned cdef_w04(int n) { return n < 7 ? 840u / (n + 1) : n == 7 ? 105u : 840u / (15 - n); }
B200_HD constexpr unsigned cdef_wodd(int n) { return n < 3 ? 420u / (n + 1) : n < 8 ? 105u : n < 11 ? 420u / (11 - n) : 0u; }
B200_DEV int cdef_dir8(const int (&v)[8], int y, int *bins, unsigned *var)
{
    int rs = 0;
#pragma unroll
    for (int x = 0; x < 8; x++) rs += v[x];
    bins[2 * 16 + y] = rs;
    int c[8];                                      // column sums: reduce-scatter over the 8 lanes, lane y ends with column y
#pragma unroll
    for (int x = 0; x < 8; x++) c[x] = v[x];
#pragma unroll
    for (int h = 4; h; h >>= 1)
#pragma unroll
        for (int k = 0; k < h; k++) {
            const bool hi = y & h;
            const int send = hi ? c[k] : c[k + h], keep = hi ? c[k + h] : c[k];
            c[k] = keep + __shfl_xor_sync(0xffffffffu, send, h, 8);
        }
    bins[6 * 16 + y] = c[0];
#pragma unroll
    for (int x = 0; x < 8; x++) {
        atomicAdd(&bins[0 * 16 + y + x], v[x]);
        atomicAdd(&bins[4 * 16 + 7 + y - x], v[x]);
        atomicAdd(&bins[5 * 16 + 3 - (y >> 1) + x], v[x]);
        atomicAdd(&bins[7 * 16 + (y >> 1) + x], v[x]);
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int q = v[2 * j] + v[2 * j + 1];
        atomicAdd(&bins[1 * 16 + y + j], q);
        atomicAdd(&bins[3 * 16 + 3 + y - j], q);
    }
    __syncwarp();
    const int d = y;
    unsigned cost = 0;
#pragma unroll
    for (int n = 0; n < 15; n++) {
        const int s = bins[d * 16 + n];
        const unsigned w = (d & 1) ? cdef_wodd(n) : (d & 2) ? (n < 8 ? 105u : 0u) : cdef_w04(n);
        cost += (unsigned)(s * s) * w;
    }
    unsigned bc = cost;
    int best = d;
#pragma unroll
    for (int m = 1; m < 8; m <<= 1) {
        const unsigned oc = __shfl_xor_sync(0xffffffffu, bc, m, 8);
        const int ob = __shfl_xor_sync(0xffffffffu, best, m, 8);
        if (oc > bc || (oc == bc && ob < best)) { bc = oc; best = ob; }
    }
    const unsigned opp = __shfl_sync(0xffffffffu, cost, best ^ 4, 8);
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
// which needs no sign restore. The sentinel (-16384) keeps diff inside int16 and makes t <= 0 for the strengths
// and damping dav1d derives (damping 2 + b8 .. 6 + b8, pri <= 15 << b8, sec in {0, 1, 2, 4} << b8), so
// out-of-picture taps contribute nothing and are ignored by the signed max / unsigned min.
constexpr int kCdefTW = 64, kCdefTH = 32, kCdefPitch = kCdefTW + 8, kCdefRows = kCdefTH + 3;
constexpr int kCdefThreads = 256;
constexpr unsigned kCdefSentinel = 0xC000u;

struct CdefBlockInfo { int16_t y_pri, y_sec, uv_pri, uv_sec; int8_t y_dir, uv_dir, inside, pad;
                       uint8_t y_pri_shift, y_sec_shift, uv_pri_shift, uv_sec_shift; };   // constrain shifts, computed once per block

constexpr int kCdefBins = 8 * 16 + 8;           // per-block direction-search scratch (ints); the pad staggers the blocks' banks

struct CdefShared {
    uint32_t tile[3][kCdefRows * kCdefPitch];   // pair rows -2 .. TH, columns -4 .. TW+3
    int bins[32][kCdefBins];
    CdefBlockInfo info[32];
    int16_t off[8][2];                          // word offset of direction d, tap k (filled per plane pitch: constant pitch)
};

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

// 8-bit: the low bytes of four packed pairs' halves as one row word (sel 0x0040 / 0x0062 picks the low / high halves)
B200_DEV unsigned cdef_row8(const unsigned (&o)[4], unsigned sel) {
    return __byte_perm(__byte_perm(o[0], o[1], sel), __byte_perm(o[2], o[3], sel), 0x5410);
}

// The filter of one item: o[] are the 4 packed pairs at word idx of a staged tile t (pitch kCdefPitch, off[d][k] the word
// offset of tap k of direction d), filtered in place with the block's strengths (pri | sec != 0), direction and
// constrain shifts.
B200_DEV void cdef_filter4(const uint32_t *t, int idx, const int16_t (&off)[8][2], int pri, int sec, int dir,
                           int pshift, int sshift, int b8, unsigned (&o)[4])
{
    const unsigned pthr1 = (unsigned)(pri + 1) * 0x00010001u, psmask = (0xffffu >> pshift) * 0x00010001u;
    const unsigned sthr1 = (unsigned)(sec + 1) * 0x00010001u, ssmask = (0xffffu >> sshift) * 0x00010001u;
    const int tap0 = 4 - ((pri >> b8) & 1);
    const int d2 = (dir + 2) & 7, d6 = (dir + 6) & 7;
    const int op0 = off[dir][0], op1 = off[dir][1];
    const int os20 = off[d2][0], os60 = off[d6][0], os21 = off[d2][1], os61 = off[d6][1];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const unsigned px2 = o[c];
        const unsigned negpx = __vadd2(~px2, 0x00010001u);
        unsigned mn = px2, mx = px2, sumN = 0, sumP = 0;
        if (pri) {
            cdef_tap2(t, idx + c, op0, negpx, pthr1, pshift, psmask, tap0, sumP, sumN, mx, mn);
            cdef_tap2(t, idx + c, op1, negpx, pthr1, pshift, psmask, (tap0 & 3) | 2, sumP, sumN, mx, mn);
        }
        if (sec) {
            cdef_tap2(t, idx + c, os20, negpx, sthr1, sshift, ssmask, 2, sumP, sumN, mx, mn);
            cdef_tap2(t, idx + c, os60, negpx, sthr1, sshift, ssmask, 2, sumP, sumN, mx, mn);
            cdef_tap2(t, idx + c, os21, negpx, sthr1, sshift, ssmask, 1, sumP, sumN, mx, mn);
            cdef_tap2(t, idx + c, os61, negpx, sthr1, sshift, ssmask, 1, sumP, sumN, mx, mn);
        }
        const int s0 = (int)(sumP & 0xffff) - (int)(sumN & 0xffff), s1 = (int)(sumP >> 16) - (int)(sumN >> 16);
        int o0 = (int)(px2 & 0xffff) + ((s0 - (s0 < 0) + 8) >> 4);
        int o1 = (int)(px2 >> 16) + ((s1 - (s1 < 0) + 8) >> 4);
        if (pri && sec) {
            o0 = iclip(o0, (int)(mn & 0xffff), (int)(mx & 0xffff));
            o1 = iclip(o1, (int)(mn >> 16), (int)(mx >> 16));
        }
        o[c] = (unsigned)o0 | (unsigned)o1 << 16;
    }
}

// an item's two rows of 4 pixels: row y at op, row y + 1 at op + st
template <bool HBD>
B200_DEV void cdef_store2(typename Bd<HBD>::pixel *op, int st, const unsigned (&o)[4])
{
    if (HBD) {
        *(uint2 *)op = make_uint2(__byte_perm(o[0], o[1], 0x5410), __byte_perm(o[2], o[3], 0x5410));
        *(uint2 *)(op + st) = make_uint2(__byte_perm(o[0], o[1], 0x7632), __byte_perm(o[2], o[3], 0x7632));
    } else {
        *(unsigned *)op = cdef_row8(o, 0x0040);
        *(unsigned *)(op + st) = cdef_row8(o, 0x0062);
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
    const int ssh = f.ss_hor, ssv = f.ss_ver;

    // the 8 lanes of 8x8 block b = tid / 8 look up its strengths; the loads are in flight during the staging
    const int blk = tid >> 3, brow = tid & 7, bxi = blk & 7, byi = blk >> 3;
    const int bx = bx0 + bxi * 2, by = by0 + byi * 2;
    const bool inside = bx < f.bw && by < f.bh;
    int y_lvl = 0, uv_lvl = 0;
    if (inside) {
        const B200Av1Filter &m = f.mask[(by >> 5) * f.sb128w + (bx >> 5)];
        const int cdef_idx = m.cdef_idx[((by & 16) >> 3) + ((bx & 16) >> 4)];
        const uint16_t *nr = m.noskip_mask[(by & 30) >> 1];
        const unsigned noskip = (unsigned)nr[1] << 16 | nr[0];
        if (cdef_idx != -1 && (noskip & (3u << (bx & 30)))) { y_lvl = f.y_strength[cdef_idx]; uv_lvl = f.uv_strength[cdef_idx]; }
    }

    // ---- stage the three planes: one flat list of items (4 samples of two consecutive rows); a thread issues the
    // loads of up to 4 items before it stores any of them, so a 4:2:0 tile is staged with all its loads in flight
    {
        const int cw = kCdefTW >> ssh, ch = kCdefTH >> ssv;
        const int g0 = (kCdefTW + 8) >> 2, n0 = g0 * (kCdefTH + 3);
        const int gc = (cw + 8) >> 2, nc = gc * (ch + 3);
        const unsigned magic0 = recip16(g0), magicc = recip16(gc);   // exact i / groups for i < 36 * 18
        const int total = n0 + 2 * nc;
        for (int base = 0; base < total; base += 4 * kCdefThreads) {
            unsigned qa[4][HBD ? 2 : 1], qb[4][HBD ? 2 : 1];
            int dsti[4]; bool ha[4], hb[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                int i = base + u * kCdefThreads + tid, pl = 0;
                if (i >= n0) { i -= n0; pl = 1; if (i >= nc) { i -= nc; pl = 2; } }
                const int sh = pl ? ssh : 0, sv = pl ? ssv : 0, groups = pl ? gc : g0;
                const int r = (int)((i * (pl ? magicc : magic0)) >> 16), g = i - r * groups;
                const int availw = ((f.bw + 1) >> 1) * 8 >> sh, availh = ((f.bh + 1) >> 1) * 8 >> sv;
                const int x = (bx0 * 4 >> sh) - 4 + g * 4, y = (by0 * 4 >> sv) - 2 + r;
                const bool ok = base + u * kCdefThreads + tid < total && x >= 0 && x < availw;
                dsti[u] = base + u * kCdefThreads + tid < total ? pl * (kCdefRows * kCdefPitch) + r * kCdefPitch + g * 4 : -1;
                ha[u] = ok && y >= 0 && y < availh;
                hb[u] = ok && y + 1 >= 0 && y + 1 < availh;
                const pixel *sp = src + f.plane_off[pl] + x;
                const int st = f.stride[pl];
#pragma unroll
                for (int k = 0; k < (HBD ? 2 : 1); k++) qa[u][k] = qb[u][k] = HBD ? kCdefSentinel * 0x00010001u : 0u;
                if (HBD) {
                    if (ha[u]) { const uint2 q = *(const uint2 *)(sp + (ptrdiff_t)y * st); qa[u][0] = q.x; qa[u][HBD] = q.y; }
                    if (hb[u]) { const uint2 q = *(const uint2 *)(sp + (ptrdiff_t)(y + 1) * st); qb[u][0] = q.x; qb[u][HBD] = q.y; }
                } else {
                    if (ha[u]) qa[u][0] = *(const unsigned *)(sp + (ptrdiff_t)y * st);
                    if (hb[u]) qb[u][0] = *(const unsigned *)(sp + (ptrdiff_t)(y + 1) * st);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (dsti[u] < 0) continue;
                uint4 w;
                if (HBD) {
                    // (a0 a1 | a2 a3) x (b0 b1 | b2 b3) -> (a0 b0) (a1 b1) (a2 b2) (a3 b3): one byte permute each
                    w.x = __byte_perm(qa[u][0], qb[u][0], 0x5410); w.y = __byte_perm(qa[u][0], qb[u][0], 0x7632);
                    w.z = __byte_perm(qa[u][HBD], qb[u][HBD], 0x5410); w.w = __byte_perm(qa[u][HBD], qb[u][HBD], 0x7632);
                } else {
                    // bytes a_k, b_k -> halfwords (a_k | b_k << 16): two byte permutes per word; the sentinel replaces
                    // missing rows afterwards (a per-byte sentinel is impossible)
                    const unsigned t01 = __byte_perm(qa[u][0], qb[u][0], 0x5140), t23 = __byte_perm(qa[u][0], qb[u][0], 0x7362);
                    w.x = __byte_perm(t01, 0, 0x4140); w.y = __byte_perm(t01, 0, 0x4342);
                    w.z = __byte_perm(t23, 0, 0x4140); w.w = __byte_perm(t23, 0, 0x4342);
                    if (!ha[u]) { w.x = (w.x & 0xffff0000u) | kCdefSentinel; w.y = (w.y & 0xffff0000u) | kCdefSentinel; w.z = (w.z & 0xffff0000u) | kCdefSentinel; w.w = (w.w & 0xffff0000u) | kCdefSentinel; }
                    if (!hb[u]) { w.x = (w.x & 0xffffu) | kCdefSentinel << 16; w.y = (w.y & 0xffffu) | kCdefSentinel << 16; w.z = (w.z & 0xffffu) | kCdefSentinel << 16; w.w = (w.w & 0xffffu) | kCdefSentinel << 16; }
                }
                *(uint4 *)&S.tile[0][dsti[u]] = w;
            }
        }
    }
    for (int i = tid; i < 32 * kCdefBins / 4; i += kCdefThreads) ((uint4 *)S.bins)[i] = make_uint4(0, 0, 0, 0);
    if (tid < 16) {
        const int d = tid >> 1, k = tid & 1;
        S.off[d][k] = (int16_t)(c_cdef_off[d][k][0] * kCdefPitch + c_cdef_off[d][k][1]);
    }
    __syncthreads();

    // ---- per-8x8 parameters: 8 lanes per block, lane y supplies the block's row y to the direction search
    {
        const uint32_t *t = &S.tile[0][(2 + byi * 8 + brow) * kCdefPitch + 4 + bxi * 8];
        const uint4 w0 = *(const uint4 *)t, w1 = *(const uint4 *)(t + 4);
        const unsigned wr[8] = { w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w };
        int v[8];
#pragma unroll
        for (int x = 0; x < 8; x++) v[x] = (int)((wr[x] & 0xffff) >> b8) - 128;
        unsigned var;
        const int dir = cdef_dir8(v, brow, S.bins[blk], &var);
        if (brow == 0) {
            CdefBlockInfo bi; bi.y_pri = bi.y_sec = bi.uv_pri = bi.uv_sec = 0; bi.y_dir = bi.uv_dir = 0; bi.pad = 0;
            bi.inside = inside;
            const int y_pri = (y_lvl >> 2) << b8;
            int y_sec = y_lvl & 3; y_sec += y_sec == 3; y_sec <<= b8;
            const int uv_pri = (uv_lvl >> 2) << b8;
            int uv_sec = uv_lvl & 3; uv_sec += uv_sec == 3; uv_sec <<= b8;
            if (y_pri) { bi.y_pri = (int16_t)cdef_adjust_strength(y_pri, var); bi.y_sec = (int16_t)y_sec; bi.y_dir = (int8_t)dir; }
            else bi.y_sec = (int16_t)y_sec;
            if (uv_lvl) {
                bi.uv_pri = (int16_t)uv_pri; bi.uv_sec = (int16_t)uv_sec;
                bi.uv_dir = (int8_t)(uv_pri ? ((ssh && !ssv) ? c_uv_dir422[dir] : dir) : 0);
            }
            // shift = max(0, damping - ulog2(strength)) per class (luma damping, chroma damping - 1)
            const int dl = f.damping + b8, dc = dl - 1;
            bi.y_pri_shift = (uint8_t)(bi.y_pri ? imax(0, dl - ulog2(bi.y_pri)) : 0);
            bi.y_sec_shift = (uint8_t)(bi.y_sec ? dl - ulog2(bi.y_sec) : 0);
            bi.uv_pri_shift = (uint8_t)(bi.uv_pri ? imax(0, dc - ulog2(bi.uv_pri)) : 0);
            bi.uv_sec_shift = (uint8_t)(bi.uv_sec ? dc - ulog2(bi.uv_sec) : 0);
            S.info[blk] = bi;
        }
    }
    __syncthreads();

    // ---- filter: a thread takes 4 adjacent columns of one vertical pixel pair (a group never straddles an 8x8 block, so
    // the block's parameters and tap offsets are decoded once) and writes each of the two rows with one store.
    // Items: the luma tile's 16 x 16 groups, then each chroma plane's (16 >> ss_hor) x (16 >> ss_ver).
    const int cgl = 4 - ssh, nc = 1 << (cgl + 4 - ssv);
    for (int i = tid; i < 256 + 2 * nc; i += kCdefThreads) {
        int pl = 0, li = i;
        if (li >= 256) { li -= 256; pl = 1; if (li >= nc) { li -= nc; pl = 2; } }
        const int sh = pl ? ssh : 0, sv = pl ? ssv : 0, gl = pl ? cgl : 4;
        const int y = (li >> gl) * 2, x = (li & ((1 << gl) - 1)) * 4;
        const CdefBlockInfo bi = S.info[(y >> (3 - sv)) * 8 + (x >> (3 - sh))];
        if (!bi.inside) continue;
        const uint32_t *t = S.tile[pl];
        const int idx = (y + 2) * kCdefPitch + x + 4;
        const uint4 pw = *(const uint4 *)&t[idx];
        unsigned o[4] = { pw.x, pw.y, pw.z, pw.w };              // (row y | row y + 1 << 16) per column
        const int pri = pl ? bi.uv_pri : bi.y_pri, sec = pl ? bi.uv_sec : bi.y_sec, dir = pl ? bi.uv_dir : bi.y_dir;
        if (pri | sec)
            cdef_filter4(t, idx, S.off, pri, sec, dir, pl ? bi.uv_pri_shift : bi.y_pri_shift,
                         pl ? bi.uv_sec_shift : bi.y_sec_shift, b8, o);
        const int st = f.stride[pl];
        cdef_store2<HBD>(dst + f.plane_off[pl] + (ptrdiff_t)((by0 * 4 >> sv) + y) * st + (bx0 * 4 >> sh) + x, st, o);
    }
}

// Level-1 kernels ---------------------------------------------------------------------------
// One w x h block (cdef.fb) on the frame kernel's filter: win is the block's dense (w+4) x (h+4) window with the block at
// (2, 2) and kCdefSentinel in every sample the edges flags mark unavailable. Its rows are staged as pair words at the
// frame tile's pitch with the block at the tile's origin, so the same tap offsets apply; out is the dense w x h result.
template <bool HBD>
__global__ void cdef_block_kernel(const uint16_t *win, typename Bd<HBD>::pixel *out, int w, int h, int pri, int sec,
                                  int dir, int damping, int bdmax)
{
    __shared__ uint32_t tile[(8 + 3) * kCdefPitch];
    __shared__ int16_t off[8][2];
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    const int ww = w + 4;
    for (int i = threadIdx.x; i < (h + 3) * ww; i += blockDim.x) {
        const int r = i / ww, c = i - r * ww;
        tile[r * kCdefPitch + 2 + c] = win[r * ww + c] | (unsigned)win[(r + 1) * ww + c] << 16;
    }
    if (threadIdx.x < 16) {
        const int d = threadIdx.x >> 1, k = threadIdx.x & 1;
        off[d][k] = (int16_t)(c_cdef_off[d][k][0] * kCdefPitch + c_cdef_off[d][k][1]);
    }
    __syncthreads();
    const int i = threadIdx.x, gw = w >> 2;
    if (i >= gw * (h >> 1)) return;
    const int y = i / gw * 2, x = i % gw * 4, idx = (y + 2) * kCdefPitch + x + 4;
    unsigned o[4] = { tile[idx], tile[idx + 1], tile[idx + 2], tile[idx + 3] };
    cdef_filter4(tile, idx, off, pri, sec, dir, pri ? imax(0, damping - ulog2(pri)) : 0, sec ? damping - ulog2(sec) : 0,
                 b8, o);
    cdef_store2<HBD>(out + y * w + x, w, o);
}

template <bool HBD>
__global__ void cdef_dir_kernel(const typename Bd<HBD>::pixel *img, int *out, int bdmax)
{
    // the four 8-lane groups of the warp each search the same block
    __shared__ int bins[4][8 * 16];
    const int b8 = HBD ? (32 - __clz(bdmax)) - 8 : 0;
    const int g = threadIdx.x >> 3, y = threadIdx.x & 7;
    for (int i = y; i < 8 * 16; i += 8) bins[g][i] = 0;
    int v[8];
#pragma unroll
    for (int x = 0; x < 8; x++) v[x] = ((int)img[y * 8 + x] >> b8) - 128;
    __syncwarp();
    unsigned var;
    const int d = cdef_dir8(v, y, bins[g], &var);
    if (threadIdx.x == 0) { out[0] = d; out[1] = (int)var; }
}

}  // namespace b200

using namespace b200;

namespace b200 {
// tile rows [t0, t1) of the sweep: a tile row is 32 luma rows (16 subsampled chroma rows) and reads 2 rows beyond each side;
// the tile loader reads and the filter writes 4 samples at a time
int cdef_frame_rows(int bdmax, const B200CdefFrame *f, int t0, int t1, cudaStream_t stream)
{
    if (int r = check_bdmax(bdmax, "b200_cdef_frame")) return r;
    const size_t px = bdmax > 255 ? 2 : 1;
    for (int pl = 0; pl < 3; pl++)
        if ((f->stride[pl] & 3) || (f->plane_off[pl] & 3) || ((uintptr_t)f->src % (4 * px)) || ((uintptr_t)f->dst % (4 * px))) { b200_set_error("b200_cdef_frame: planes must be 4-sample aligned"); return -2; }
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
    // the strengths and damping for which the sentinel silences the unavailable taps (kCdefSentinel): what dav1d
    // passes, luma damping 3 + b8 .. 6 + b8 and chroma one less
    const int b8 = ulog2(bdmax) - 7;
    const bool sec_ok = sec == 0 || sec == 1 << b8 || sec == 2 << b8 || sec == 4 << b8;
    if (!((w == 4 || w == 8) && (h == 4 || h == 8)) || dir < 0 || dir > 7 || (!pri && !sec) || pri < 0 || pri > 15 << b8 ||
        !sec_ok || damping < 2 + b8 || damping > 6 + b8) {
        b200_set_error("b200_cdef_fb: bad arguments (w=%d h=%d pri=%d sec=%d dir=%d damping=%d)", w, h, pri, sec, dir, damping);
        return -2;
    }
    Level1 L;
    const size_t px = bdmax > 255 ? 2 : 1;
    const int ww = w + 4;
    uint16_t win[12 * 12];
    for (uint16_t &v : win) v = kCdefSentinel;
    auto put = [&](int wx, int wy, const void *p) { win[wy * ww + wx] = px == 2 ? *(const uint16_t *)p : *(const uint8_t *)p; };
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
    if (!(in = L.upload(0, win, (size_t)ww * (h + 4) * sizeof(win[0]))) || !(out = L.dev(1, 64 * 2))) return -1;
    if (int r = launch_hbd(bdmax, Launch::plain, dim3(1), dim3(64), 0, 0, [&](auto hbd) {
            return std::make_tuple(cdef_block_kernel<hbd>, (const uint16_t *)in, (typename Bd<hbd>::pixel *)out, w, h, pri,
                                   sec, dir, damping, bdmax);
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
