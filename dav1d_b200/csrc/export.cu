// Export of a decoded picture from its device copy into caller-owned device memory (B200ExportJob, B200TensorJob,
// include/b200av1.h):
//   export_planes_kernel  Y / U / V cropped to the visible size, tightly packed
//   export_rgb_kernel     planar R / G / B at the stream's bit depth (nearest chroma sample, integer matrix)
//   export_tensor_kernel  R / G / B resized (bilinear, chroma upsampling included), normalised, as fp32 / fp16 / bf16 in
//                         CHW or HWC order: what a model takes, in one pass
//   export_tensor_aa_kernel  the same with antialiasing (triangle filter) on reduced axes, or bicubic (plain or
//                         antialiased): a separable pass over shared-memory tiles, sharing export_tensor_kernel's epilogue
// Memory bound: a thread owns a run of horizontally adjacent output samples (8 bytes: 8 samples at 8 bit, 4 above), read
// and written with one 8-byte access where the run is complete and the rows are aligned; the RGB kernel of a vertically
// sub-sampled picture takes two rows per thread, so that each chroma sample is read once for its 2 x 2 luma quad. The
// tensor kernel's thread owns 4 adjacent output pixels, written per channel with one 16-byte (fp32) or 8-byte store.
#include "common.cuh"
#include "host_util.h"
#include <cmath>
#ifndef B200_EMU
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#else
// Host build of these sources (tests/emu): the rounding intrinsics of the tensor export with the same results. Each fp32
// operation is rounded on its own (the volatile store keeps the compiler from contracting a multiply and an add into an
// FMA), and g++'s _Float16 / __bf16 conversions round to nearest even like __float2half_rn / __float2bfloat16_rn. The
// library is built with --use_fast_math, whose -ftz=true makes a subnormal operand or result of these operations a zero
// of the same sign on the GPU: emu_ftz does the same here.
typedef _Float16 __half;
typedef __bf16 __nv_bfloat16;
static inline float emu_ftz(float v) { return std::fabs(v) < 1.17549435e-38f ? std::copysign(0.0f, v) : v; }
static inline float __fmul_rn(float a, float b) { volatile float r = emu_ftz(a) * emu_ftz(b); return emu_ftz(r); }
static inline float __fadd_rn(float a, float b) { volatile float r = emu_ftz(a) + emu_ftz(b); return emu_ftz(r); }
static inline float __fsub_rn(float a, float b) { volatile float r = emu_ftz(a) - emu_ftz(b); return emu_ftz(r); }
static inline float __fdiv_rn(float a, float b) { volatile float r = emu_ftz(a) / emu_ftz(b); return emu_ftz(r); }
static inline __half __float2half_rn(float v) { return (__half)v; }
static inline __nv_bfloat16 __float2bfloat16_rn(float v) { return (__nv_bfloat16)v; }
static inline unsigned short __half_as_ushort(__half h) { unsigned short u; memcpy(&u, &h, 2); return u; }
static inline unsigned short __bfloat16_as_ushort(__nv_bfloat16 h) { unsigned short u; memcpy(&u, &h, 2); return u; }
static inline int __float2int_rn(float v) { return (int)lrintf(v); }     // the default rounding mode: to nearest even
#endif

namespace b200 {

// n <= N samples at p into v; one access of N samples when all of them are there and p is aligned to that size
template <class pixel, int N>
B200_DEV void load_run(const pixel *p, int n, pixel (&v)[N])
{
    constexpr int B = N * sizeof(pixel);
    static_assert(B == 4 || B == 8, "run size");
    if (n == N && !((uintptr_t)p & (B - 1))) {
        if constexpr (B == 8) { const uint2 u = *(const uint2 *)p; memcpy(v, &u, 8); }
        else { const uint32_t u = *(const uint32_t *)p; memcpy(v, &u, 4); }
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) if (i < n) v[i] = p[i];
    }
}
template <class pixel, int N>
B200_DEV void store_run(pixel *p, int n, const pixel (&v)[N])
{
    constexpr int B = N * sizeof(pixel);
    static_assert(B == 8 || B == 16, "run size");
    if (n == N && !((uintptr_t)p & (B - 1))) {
        if constexpr (B == 16) { uint4 u; memcpy(&u, v, 16); *(uint4 *)p = u; }
        else { uint2 u; memcpy(&u, v, 8); *(uint2 *)p = u; }
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) if (i < n) p[i] = v[i];
    }
}

// grid (runs of the widest plane / 32, rows / 8, planes), block (32, 8)
template <bool HBD>
__global__ void __launch_bounds__(256) export_planes_kernel(const __grid_constant__ B200ExportJob j)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    constexpr int N = 8 / sizeof(pixel);
    const int pl = blockIdx.z;
    const int w = pl ? (j.w + j.ss_hor) >> j.ss_hor : j.w, h = pl ? (j.h + j.ss_ver) >> j.ss_ver : j.h;
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * N, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x0 >= w || y >= h) return;
    const int n = imin(N, w - x0);
    pixel v[N];
    load_run(((const pixel *)j.src) + j.plane_off[pl] + (ptrdiff_t)y * j.stride[pl] + x0, n, v);
    store_run(((pixel *)j.dst[pl]) + (ptrdiff_t)y * j.dst_pitch[pl] + x0, n, v);
}

// grid (runs / 32, row groups / 8), block (32, 8); a row group is 2 rows when chroma is vertically sub-sampled, else 1
template <bool HBD, int SSH>
__global__ void __launch_bounds__(256) export_rgb_kernel(const __grid_constant__ B200ExportJob j)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    constexpr int N = 8 / sizeof(pixel), CN = N >> SSH;
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * N, y0 = (blockIdx.y * blockDim.y + threadIdx.y) << j.ss_ver;
    if (x0 >= j.w || y0 >= j.h) return;
    const int n = imin(N, j.w - x0), rows = j.ss_ver && y0 + 1 < j.h ? 2 : 1;
    const int bdmax = j.bitdepth_max, s = bdmax == 4095 ? 4 : bdmax == 1023 ? 2 : 0;
    const int yoff = j.full_range ? 0 : 16 << s, coff = 128 << s;
    pixel u[CN] = {}, v[CN] = {};
    if (j.mono) {
#pragma unroll
        for (int i = 0; i < CN; i++) u[i] = v[i] = (pixel)coff;
    } else {
        const int cn = (n + SSH) >> SSH;
        const ptrdiff_t c = (ptrdiff_t)(y0 >> j.ss_ver) * j.stride[1] + (x0 >> SSH);
        load_run(((const pixel *)j.src) + j.plane_off[1] + c, cn, u);
        load_run(((const pixel *)j.src) + j.plane_off[2] + c, cn, v);
    }
    for (int r = 0; r < rows; r++) {
        pixel yv[N] = {}, ro[N], go[N], bo[N];
        load_run(((const pixel *)j.src) + j.plane_off[0] + (ptrdiff_t)(y0 + r) * j.stride[0] + x0, n, yv);
#pragma unroll
        for (int i = 0; i < N; i++) {
            const int Y = yv[i], U = u[i >> SSH], V = v[i >> SSH];
            if (j.identity) {
                ro[i] = (pixel)V; go[i] = (pixel)Y; bo[i] = (pixel)U;
            } else {
                const int yy = j.cy * (Y - yoff) + 8192, cb = U - coff, cr = V - coff;
                ro[i] = (pixel)iclip((yy + j.rv * cr) >> 14, 0, bdmax);
                go[i] = (pixel)iclip((yy - j.gu * cb - j.gv * cr) >> 14, 0, bdmax);
                bo[i] = (pixel)iclip((yy + j.bu * cb) >> 14, 0, bdmax);
            }
        }
        const ptrdiff_t y = y0 + r;
        store_run(((pixel *)j.dst[0]) + y * j.dst_pitch[0] + x0, n, ro);
        store_run(((pixel *)j.dst[1]) + y * j.dst_pitch[1] + x0, n, go);
        store_run(((pixel *)j.dst[2]) + y * j.dst_pitch[2] + x0, n, bo);
    }
}

// One axis of one plane's sampling positions (B200TensorJob): q, r = floor quotient and remainder of the position numerator
// by OUT. The numerator grows by a constant from one output index to the next, so after one int64 division for the first
// index every later one costs an add and a compare.
struct TapAxis {
    int q, r, dq, dr, out;
    // output index x, stepping by `step` indices; IN = luma length, s = the plane's sub-sampling, k = its siting
    B200_DEV TapAxis(int x, int step, int in, int out_, int s, int k) : out(out_)
    {
        const int64_t num = ((int64_t)(2 * x + 1) * in - (int64_t)(1 + k) * out) * (128 >> s);
        int64_t q64 = num / out, r64 = num % out;
        if (r64 < 0) { r64 += out; q64--; }
        q = (int)q64; r = (int)r64;
        const int d = 2 * step * in * (128 >> s);
        dq = d / out; dr = d % out;
    }
    B200_DEV void next() { q += dq; r += dr; if (r >= out) { r -= out; q++; } }
    // the two taps (i0, i1) and weight f of the current index on a plane of n samples
    B200_DEV void taps(int n, int &i0, int &i1, int &f) const
    {
        const int pos = imax(q, 0);
        i0 = imin(pos >> 8, n - 1); i1 = imin(i0 + 1, n - 1); f = pos & 255;
    }
};

// Q of one output pixel: the bilinear sample with 2 fractional bits
template <class pixel>
B200_DEV int tensor_sample(const pixel *r0, const pixel *r1, int x0, int x1, int fx, int fy)
{
    const int a = __ldg(r0 + x0) * (256 - fx) + __ldg(r0 + x1) * fx, b = __ldg(r1 + x0) * (256 - fx) + __ldg(r1 + x1) * fx;
    return (a * (256 - fy) + b * fy + (1 << 13)) >> 14;
}

// the taps of a run of 4 output columns on one plane
struct RunTaps { int x0[4], x1[4], f[4]; };
B200_DEV void run_taps(RunTaps &t, int x, int in, int out, int n, int s, int k)
{
    TapAxis a(x, 1, in, out, s, k);
#pragma unroll
    for (int i = 0; i < 4; i++) { a.taps(n, t.x0[i], t.x1[i], t.f[i]); a.next(); }
}

template <class pixel>
B200_DEV void run_samples(int (&q)[4], const pixel *plane, int stride, const TapAxis &ay, int n_rows, const RunTaps &t)
{
    int y0, y1, fy;
    ay.taps(n_rows, y0, y1, fy);
    const pixel *const r0 = plane + (ptrdiff_t)y0 * stride, *const r1 = plane + (ptrdiff_t)y1 * stride;
#pragma unroll
    for (int i = 0; i < 4; i++) q[i] = tensor_sample(r0, r1, t.x0[i], t.x1[i], t.f[i], fy);
}

template <int DT> struct TensorElem { typedef uint16_t type; };
template <> struct TensorElem<B200_TENSOR_F32> { typedef float type; };

// v: the matrix's integer R, or with a tone map the float T
template <int DT, class V>
B200_DEV typename TensorElem<DT>::type tensor_value(V v, float scale, float bias)
{
    const float f = __fadd_rn(__fmul_rn((float)v, scale), bias);
    if constexpr (DT == B200_TENSOR_F16) return __half_as_ushort(__float2half_rn(f));
    else if constexpr (DT == B200_TENSOR_BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(f));
    else return f;
}

// The stores of tensor_store: output pixel i of the run at x goes to x + i, or with MIRROR (B200TensorJob.flip) to
// out_w - 1 - x - i. A mirrored run of 4 is the reversed run at out_w - 4 - x, stored like any other; a ragged one (n < 4,
// the row's right end) lands at the row's left end one value at a time.
template <bool MIRROR, bool HWC, class E>
B200_DEV void store_pixels(const B200TensorJob &j, E *row, int x, int n, const E (&o)[3][4])
{
    if (MIRROR && n < 4) {
#pragma unroll
        for (int i = 0; i < 4; i++)
            if (i < n) {
                const int64_t at = j.out_w - 1 - x - i;
#pragma unroll
                for (int c = 0; c < 3; c++) row[HWC ? 3 * at + c : c * j.pitch_c + at] = o[c][i];
            }
        return;
    }
    const int px = MIRROR ? j.out_w - 4 - x : x;
    if constexpr (HWC) {
        // the run is 12 contiguous values: R G B of pixel 0, then of pixel 1, ...
        E v[3][4];
#pragma unroll
        for (int e = 0; e < 12; e++) v[e >> 2][e & 3] = o[e % 3][MIRROR ? 3 - e / 3 : e / 3];
#pragma unroll
        for (int r = 0; r < 3; r++) store_run(row + 3 * px + 4 * r, imin(4, 3 * n - 4 * r), v[r]);
    } else {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            if constexpr (MIRROR) {
                const E v[4] = {o[c][3], o[c][2], o[c][1], o[c][0]};
                store_run(row + c * j.pitch_c + px, n, v);
            } else {
                store_run(row + c * j.pitch_c + px, n, o[c]);
            }
        }
    }
}

// The HDR to SDR stage of a tone-mapped job (B200ToneMap, include/b200av1.h): curve, gamut matrix, clip and OETF of the
// matrix's R, G, B (each 0 .. 4 * bdmax) into T, on the same scale
B200_DEV void tone_map(const B200ToneMap &t, const int (&rgb)[3], float (&T)[3])
{
    float L[3];
#pragma unroll
    for (int c = 0; c < 3; c++) L[c] = __ldg(t.curve + rgb[c]);
    const float top = (float)(1 << t.oetf_bits);
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const float g = __fadd_rn(__fadd_rn(__fmul_rn(t.m[3 * r], L[0]), __fmul_rn(t.m[3 * r + 1], L[1])), __fmul_rn(t.m[3 * r + 2], L[2]));
        T[r] = __ldg(t.oetf + __float2int_rn(__fmul_rn(fminf(fmaxf(g, 0.0f), 1.0f), top)));
    }
}

// ---- colour jitter (B200ColorJitter, include/b200av1.h): torchvision's float32 operations, each rounded on its own ----
enum { kJitBrightness = 0, kJitContrast = 1, kJitSaturation = 2, kJitHue = 3 };
B200_DEV float unit_clip(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }
B200_DEV float jitter_gray(const float (&x)[3])
{
    return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, x[0]), __fmul_rn(0.587f, x[1])), __fmul_rn(0.114f, x[2]));
}
// clip(a * x_c + a1 * g) per channel: torchvision's _blend
B200_DEV void jitter_blend(float (&x)[3], float a, float a1, float g)
{
#pragma unroll
    for (int c = 0; c < 3; c++) x[c] = unit_clip(__fadd_rn(__fmul_rn(a, x[c]), __fmul_rn(a1, g)));
}
// _rgb2hsv, h = remainder(h + hue, 1), _hsv2rgb
B200_DEV void jitter_hue(float (&x)[3], float hue)
{
    const float r = x[0], g = x[1], b = x[2];
    const float maxc = fmaxf(fmaxf(r, g), b), minc = fminf(fminf(r, g), b);
    const bool eqc = maxc == minc;
    const float cr = __fsub_rn(maxc, minc), d = eqc ? 1.0f : cr;
    const float s = __fdiv_rn(cr, eqc ? 1.0f : maxc);
    const float rc = __fdiv_rn(__fsub_rn(maxc, r), d), gc = __fdiv_rn(__fsub_rn(maxc, g), d), bc = __fdiv_rn(__fsub_rn(maxc, b), d);
    float h = maxc == r ? __fsub_rn(bc, gc) : maxc == g ? __fsub_rn(__fadd_rn(2.0f, rc), bc) : __fsub_rn(__fadd_rn(4.0f, gc), rc);
    h = __fadd_rn(__fdiv_rn(h, 6.0f), 1.0f);           // in [5/6, 11/6]: fmod(h, 1) is exact
    if (h >= 1.0f) h = __fsub_rn(h, 1.0f);
    h = __fadd_rn(h, hue);                             // in [-1/2, 3/2]: torch.remainder(h, 1)
    if (h >= 1.0f) h = __fsub_rn(h, 1.0f);
    if (h < 0.0f) h = __fadd_rn(h, 1.0f);
    const float h6 = __fmul_rn(h, 6.0f), fi = floorf(h6), f = __fsub_rn(h6, fi);
    const float p = unit_clip(__fmul_rn(maxc, __fsub_rn(1.0f, s)));
    const float q = unit_clip(__fmul_rn(maxc, __fsub_rn(1.0f, __fmul_rn(s, f))));
    const float t = unit_clip(__fmul_rn(maxc, __fsub_rn(1.0f, __fmul_rn(s, __fsub_rn(1.0f, f)))));
    switch ((int)fi % 6) {
    case 0: x[0] = maxc; x[1] = t; x[2] = p; break;
    case 1: x[0] = q; x[1] = maxc; x[2] = p; break;
    case 2: x[0] = p; x[1] = maxc; x[2] = t; break;
    case 3: x[0] = p; x[1] = q; x[2] = maxc; break;
    case 4: x[0] = t; x[1] = p; x[2] = maxc; break;
    default: x[0] = maxc; x[1] = p; x[2] = q; break;
    }
}
// the enabled operations in t.order on x (in [0, 1]); PRE: only those before contrast, whose gray the contrast pass sums.
// m = the contrast mean M
template <bool PRE>
B200_DEV void color_jitter(const B200ColorJitter &t, float m, float (&x)[3])
{
#pragma unroll 1
    for (int k = 0; k < 4; k++) {
        const int op = t.order[k];
        if (!((t.enabled >> op) & 1)) continue;
        if (op == kJitContrast) {
            if (PRE) return;
            jitter_blend(x, t.contrast, t.contrast1, m);
        } else if (op == kJitBrightness) {
#pragma unroll
            for (int c = 0; c < 3; c++) x[c] = unit_clip(__fmul_rn(t.brightness, x[c]));
        } else if (op == kJitSaturation) {
            jitter_blend(x, t.saturation, t.saturation1, jitter_gray(x));
        } else {
            jitter_hue(x, t.hue);
        }
    }
    if (!PRE && t.grayscale) x[0] = x[1] = x[2] = jitter_gray(x);
}
// M of a jittered job from the contrast pass's sum S at t.acc: f32(f64(S) / (f64(OW * OH) * 2^24))
B200_DEV float contrast_mean(const B200ColorJitter &t, const B200TensorJob &j)
{
    if (!((t.enabled >> kJitContrast) & 1)) return 0.0f;
    return (float)((double)*t.acc / ((double)j.out_w * (double)j.out_h * 16777216.0));
}

// The epilogues of the tensor kernels (kernel template parameter EPI): plain, tone-mapped (B200ToneMap), colour-jittered
// (B200ColorJitter, the tone map a runtime branch: tone.curve NULL is none) and the contrast pass of jittered jobs, which
// stores nothing and adds rint(gray * 2^24) of each output pixel before contrast into its thread's sum
enum { kEpiPlain = 0, kEpiTone = 1, kEpiJitter = 2, kEpiContrast = 3 };
// what the jittered epilogues take besides the job: the jitter t, the contrast mean M, unit = f32(1 / (4 * bdmax)) (both
// worked out once per thread) and, in the contrast pass, the thread's sum: at most 16 pixels (export_tensor_kernel's 4 x 4;
// the tile kernel's epilogue gives a thread one run of 4) of at most 2^24 each, so 32 bits hold it
struct JitterArgs { const B200ColorJitter *t; float mean, unit; uint32_t *sum; };

// The epilogue of both tensor kernels: Q of a run of n (<= 4) output pixels at (x, y), per plane, through the matrix, the
// clip, (kEpiTone: the tone map tm; kEpiJitter: tm when it has a curve, then the jitter ja.t with contrast mean ja.mean) scale /
// bias and rounding into the destination (yoff, coff, qmax as include/b200av1.h defines them for the job); MIRROR =
// j.flip and EPI, parameters of the kernels: jobs with and without a flip, tone map or jitter take kernels of their own.
// kEpiContrast adds to *ja.sum instead of storing.
template <int DT, bool HWC, bool MIRROR, int EPI>
B200_DEV void tensor_store(const B200TensorJob &j, const B200ToneMap *tm, int x, int y, int n, const int (&qy)[4], const int (&qu)[4],
                           const int (&qv)[4], int yoff, int coff, int qmax, const JitterArgs &ja = {})
{
    typedef typename TensorElem<DT>::type E;
    E o[3][4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int rgb[3];
        if (j.identity) {
            rgb[0] = qv[i]; rgb[1] = qy[i]; rgb[2] = qu[i];
        } else {
            const int yy = j.cy * (qy[i] - yoff) + 8192, cb = j.mono ? 0 : qu[i] - coff, cr = j.mono ? 0 : qv[i] - coff;
            rgb[0] = iclip((yy + j.rv * cr) >> 14, 0, qmax);
            rgb[1] = iclip((yy - j.gu * cb - j.gv * cr) >> 14, 0, qmax);
            rgb[2] = iclip((yy + j.bu * cb) >> 14, 0, qmax);
        }
        if constexpr (EPI >= kEpiJitter) {
            float J[3];
            if (tm->curve) {
                tone_map(*tm, rgb, J);
#pragma unroll
                for (int c = 0; c < 3; c++) J[c] = __fmul_rn(J[c], ja.unit);
            } else {
#pragma unroll
                for (int c = 0; c < 3; c++) J[c] = __fmul_rn((float)rgb[c], ja.unit);
            }
            if constexpr (EPI == kEpiContrast) {
                color_jitter<true>(*ja.t, 0.0f, J);
                if (i < n) *ja.sum += (uint32_t)__float2int_rn(__fmul_rn(jitter_gray(J), 16777216.0f));
            } else {
                color_jitter<false>(*ja.t, ja.mean, J);
#pragma unroll
                for (int c = 0; c < 3; c++) o[c][i] = tensor_value<DT>(J[c], j.scale[c], j.bias[c]);
            }
        } else if constexpr (EPI == kEpiTone) {
            float T[3];
            tone_map(*tm, rgb, T);
#pragma unroll
            for (int c = 0; c < 3; c++) o[c][i] = tensor_value<DT>(T[c], j.scale[c], j.bias[c]);
        } else {
#pragma unroll
            for (int c = 0; c < 3; c++) o[c][i] = tensor_value<DT>(rgb[c], j.scale[c], j.bias[c]);
        }
    }
    if constexpr (EPI != kEpiContrast) {
        E *const row = (E *)j.dst + y * j.pitch_y;
        store_pixels<MIRROR, HWC>(j, row, x, n, o);
    }
}

// The jobs of one launch travel in the kernel's parameter block (no staging copy): B200_TENSOR_BATCH_MAX of them fit the
// classic 4 KB limit. A one-job launch takes the N = 1 form: its job's fields are then read at fixed parameter offsets, as
// operands of the instructions that use them; indexed by blockIdx.z they are separate loads, which made the prologue of a
// small one-picture export up to a quarter slower. Tone-mapped jobs (kEpiTone) carry their B200ToneMap beside them, and
// jittered ones (kEpiJitter, and their contrast pass) a tone map (curve NULL: none) and their B200ColorJitter; both always
// take the batched form.
template <int N, int B> struct TensorBatch { B200TensorJob job[N]; };
template <int N> struct TensorBatch<N, kEpiTone> { B200TensorJob job[N]; B200ToneMap tone[N]; };
template <int N> struct TensorBatch<N, kEpiJitter> { B200TensorJob job[N]; B200ToneMap tone[N]; B200ColorJitter jit[N]; };
// the batch an epilogue's kernels take: the contrast pass reads the jittered jobs' own
constexpr int batch_of(int epi) { return epi == kEpiContrast ? kEpiJitter : epi; }
static_assert(sizeof(TensorBatch<B200_TENSOR_BATCH_MAX, kEpiPlain>) <= 4096, "the jobs of one launch must fit a 4 KB kernel parameter block");
static_assert(sizeof(TensorBatch<B200_TENSOR_TONE_BATCH_MAX, kEpiTone>) <= 4096,
              "the tone-mapped jobs of one launch must fit a 4 KB kernel parameter block");
static_assert(sizeof(TensorBatch<B200_TENSOR_JITTER_BATCH_MAX, kEpiJitter>) + sizeof(int) <= 4096,
              "the jittered jobs of one launch must fit a 4 KB kernel parameter block");
template <int N, int B>
B200_DEV const B200ToneMap *tone_of(const TensorBatch<N, B> &b)
{
    if constexpr (B != kEpiPlain) return &b.tone[N == 1 ? 0 : blockIdx.z];
    else return nullptr;
}
template <int N, int B>
B200_DEV const B200ColorJitter *jitter_of(const TensorBatch<N, B> &b)
{
    if constexpr (B == kEpiJitter) return &b.jit[blockIdx.z];
    else return nullptr;
}
// __launch_bounds__'s minimum of resident CTAs per SM: 0 (none) for every form but the contrast pass, where 2 keeps
// ptxas from choosing a register budget that spills (64 registers and a 48-byte stack frame in the 10/12-bit cubic one)
template <int EPI> constexpr int kMinBlocks = EPI == kEpiContrast ? 2 : 0;
// the JitterArgs of the epilogue EPI for job j of b (the contrast pass reads no M: it is summing it)
template <int EPI, int N, int B>
B200_DEV JitterArgs jitter_args(const TensorBatch<N, B> &b, const B200TensorJob &j, uint32_t *sum)
{
    if constexpr (EPI == kEpiJitter || EPI == kEpiContrast) {
        const B200ColorJitter &t = *jitter_of(b);
        return {&t, EPI == kEpiJitter ? contrast_mean(t, j) : 0.0f, __fdiv_rn(1.0f, (float)(4 * j.bitdepth_max)), sum};
    } else {
        return {nullptr, 0.0f, 0.0f, sum};
    }
}

// The contrast pass's end: the sums of a warp's threads added into the job's S with one 64-bit integer atomic add, so
// that S does not depend on the order of the adds. Every thread of the warp calls it, at the kernel's end
B200_DEV void contrast_add(const B200ColorJitter &t, uint64_t sum)
{
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (threadIdx.x == 0 && sum) atomicAdd((unsigned long long *)t.acc, (unsigned long long)sum);
}

// grid (1), block (32): zeroes S of the n jittered jobs with contrast, before their contrast pass
template <int N>
__global__ void __launch_bounds__(32) contrast_zero_kernel(const __grid_constant__ TensorBatch<N, kEpiJitter> b, int n)
{
    B200_PDL_ENTRY();
    const int i = threadIdx.x;
    if (i < n && ((b.jit[i].enabled >> kJitContrast) & 1)) *b.jit[i].acc = 0;
}

// grid (runs of 4 output columns / 32, output rows / (8 * kTensorRows), jobs), block (32, 8): x / y cover the largest
// output of the launch, z selects the job. A thread converts its run of 4 columns on kTensorRows rows 8 apart, so the
// column taps are worked out once for all of them
constexpr int kTensorRows = 4;
template <bool HBD, int DT, bool HWC, int N, bool MIRROR, int EPI>
__global__ void __launch_bounds__(256, kMinBlocks<EPI>) export_tensor_kernel(const __grid_constant__ TensorBatch<N, batch_of(EPI)> b)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    const B200TensorJob &j = b.job[N == 1 ? 0 : blockIdx.z];
    if constexpr (EPI == kEpiContrast)
        if (!((jitter_of(b)->enabled >> kJitContrast) & 1)) return;
    uint32_t sum = 0;
    const JitterArgs ja = jitter_args<EPI>(b, j, &sum);
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y0 = blockIdx.y * 8 * kTensorRows + threadIdx.y;
    // the contrast pass keeps every lane to its one contrast_add at the end: a lane outside the output skips the rows
    if (x >= j.out_w || y0 >= j.out_h)
        if constexpr (EPI != kEpiContrast) return;
    const int n = imin(4, j.out_w - x);
    const int cw = (j.w + j.ss_hor) >> j.ss_hor, ch = (j.h + j.ss_ver) >> j.ss_ver;
    const int kx = j.ss_hor ? j.siting_x : 0, ky = j.ss_ver ? j.siting_y : 0;
    const int bdmax = j.bitdepth_max, s = bdmax == 4095 ? 4 : bdmax == 1023 ? 2 : 0, qmax = 4 * bdmax;
    const int yoff = j.full_range ? 0 : 64 << s, coff = 512 << s;
    const pixel *const src = (const pixel *)j.src;
    RunTaps lt, ct;
    run_taps(lt, x, j.w, j.out_w, j.w, 0, 0);
    if (!j.mono) run_taps(ct, x, j.w, j.out_w, cw, j.ss_hor, kx);
    TapAxis lrow(y0, 8, j.h, j.out_h, 0, 0), crow(y0, 8, j.h, j.out_h, j.ss_ver, ky);
    for (int k = 0; k < kTensorRows; k++, lrow.next(), crow.next()) {
        const int y = y0 + 8 * k;
        if (y >= j.out_h) break;
        if constexpr (EPI == kEpiContrast)
            if (x >= j.out_w) break;
        int qy[4], qu[4] = {}, qv[4] = {};
        run_samples(qy, src + j.plane_off[0], j.stride[0], lrow, j.h, lt);
        if (!j.mono) {
            run_samples(qu, src + j.plane_off[1], j.stride[1], crow, ch, ct);
            run_samples(qv, src + j.plane_off[2], j.stride[2], crow, ch, ct);
        }
        tensor_store<DT, HWC, MIRROR, EPI>(j, tone_of(b), x, y, n, qy, qu, qv, yoff, coff, qmax, ja);
    }
    if constexpr (EPI == kEpiContrast) contrast_add(*jitter_of(b), sum);
}

// ---- antialiased reduction (B200TensorJob.antialias = 1, include/b200av1.h) ----
// floor(num / den) for den > 0 and a quotient below 2^26, without the int64 division routine (a call, whose call sites
// spill): two float estimates, then the remainder brought into [0, den). Exact whatever the float rounding.
B200_DEV int64_t floor_div(int64_t num, int64_t den)
{
    const float rd = 1.0f / (float)den;
    int64_t q = (int64_t)((float)num * rd);
    q += (int64_t)((float)(num - q * den) * rd);
    int64_t r = num - q * den;
    while (r < 0) { q--; r += den; }
    while (r >= den) { q++; r -= den; }
    return q;
}

// One output sample on one axis of one plane: its taps [jlo, jhi] and their weights (1/2^14). A reduced axis (sigma > 256)
// takes the triangle's taps with cumulative rounding, any other the bilinear taps i0 = jlo, i1 = jhi as weights.
struct AaAxis {
    int64_t P, T;
    int sigma, jlo, jhi, f;
    B200_DEV AaAxis(int x, int in, int out, int n, int s, int k)
    {
        P = floor_div(((int64_t)(2 * x + 1) * in - (int64_t)(1 + k) * out) * (128 >> s), out);
        sigma = (int)floor_div((int64_t)in << (8 - s), out);
        if (sigma <= 256) {
            const int pos = (int)(P > 0 ? P : 0);
            jlo = imin(pos >> 8, n - 1); jhi = imin(jlo + 1, n - 1); f = pos & 255; T = 0;
        } else {
            // t_j > 0 <=> P - sigma < 256 j < P + sigma (arithmetic shifts floor)
            jlo = (int)(((P - sigma) >> 8) + 1); jhi = (int)((P + sigma - 1) >> 8);
            jlo = imax(jlo, 0); jhi = imin(jhi, n - 1); f = 0;
            T = cum(jhi);
        }
    }
    // C_j: the sum of t_i over jlo <= i <= j, an arithmetic series on each side of P
    B200_DEV int64_t cum(int j) const
    {
        const int64_t m = P >> 8;                // t_i = sigma - P + 256 i for i <= m, sigma + P - 256 i above
        int64_t c = 0, a = jlo, e = j < m ? j : m;
        if (e >= a) c += (e - a + 1) * (sigma - P) + 128 * (e - a + 1) * (a + e);
        a = jlo > m + 1 ? jlo : m + 1;
        if (j >= a) c += (j - a + 1) * (sigma + P) - 128 * (j - a + 1) * (a + j);
        return c;
    }
    B200_DEV int64_t rounded(int j) const { return floor_div(cum(j) * 32768 + T, 2 * T); }
    B200_DEV int weight(int j) const
    {
        if (j < jlo || j > jhi) return 0;
        if (sigma <= 256) return (j == jlo ? (256 - f) * 64 : 0) + (j == jhi ? f * 64 : 0);
        return (int)(rounded(j) - (j > jlo ? rounded(j - 1) : 0));
    }
};

// ---- bicubic (B200TensorJob.interpolation = B200_TENSOR_BICUBIC, include/b200av1.h) ----
// 4 * 256^3 * K(u / 256): the Keys cubic with a = a4 / 4 at u / 256 samples, exact in int32 for 0 <= u
B200_DEV int keys(int u, int a4)
{
    if (u < 256) return ((a4 + 8) * u - (a4 + 12) * 256) * u * u + (1 << 26);
    if (u < 512) return a4 * ((((u - 1280) * u + 524288) * u) - (1 << 26));
    return 0;
}

// One output sample on one axis of one plane: its taps [jlo, jhi] (within [0, n - 1]) and their t_j. Plain (aa = 0): the
// four taps around P, folded onto the edge (plain_weight); antialiased: every tap with u_j < 512, the weights being the
// cumulative rounding over them (cubic_weights)
struct CubicAxis {
    int64_t P;
    int sg, a4, jlo, jhi;                            // sg = sigma'
    B200_DEV CubicAxis(int x, int in, int out, int n, int s, int k, bool aa)
    {
        P = floor_div(((int64_t)(2 * x + 1) * in - (int64_t)(1 + k) * out) * (128 >> s), out);
        if (aa) {
            sg = imax((int)floor_div((int64_t)in << (8 - s), out), 256); a4 = -2;
            // u_j < 512 <=> P - 2 sg < 256 j < P + 2 sg
            jlo = imax((int)(((P - 2 * sg) >> 8) + 1), 0); jhi = imin((int)((P + 2 * sg - 1) >> 8), n - 1);
        } else {
            sg = 256; a4 = -3;
            const int m = (int)(P >> 8);
            jlo = imax(m - 1, 0); jhi = imin(m + 2, n - 1);
        }
    }
    B200_DEV int t(int j) const
    {
        int64_t d = 256 * (int64_t)j - P;
        d = d < 0 ? -d : d;
        if (d >= 2 * sg) return 0;
        return keys(sg == 256 ? (int)d : (int)floor_div(d << 8, sg), a4);
    }
    // plain bicubic: the weight of tap j, the sum of the rounded weights of the unclamped taps m - 1 .. m + 2 that clamp to j
    B200_DEV int plain_weight(int j, int n) const
    {
        const int m = (int)(P >> 8);
        int c = 0, r0 = 0, w = 0;
        for (int i = m - 1; i <= m + 2; i++) {
            c += t(i);
            const int r = (c + (1 << 11)) >> 12;
            if (iclip(i, 0, n - 1) == j) w += r - r0;
            r0 = r;
        }
        return w;
    }
    // antialiased bicubic, called by a whole warp: T, the sum of t_j over the taps
    B200_DEV int64_t total(int lane) const
    {
        int64_t T = 0;
        for (int i = jlo + lane; i <= jhi; i += 32) T += t(i);
        for (int o = 16; o; o >>= 1) T += __shfl_xor_sync(0xffffffffu, T, o);
        return T;
    }
    // antialiased bicubic, called by a whole warp: the weight of tap j0 + lane (0 outside [jlo, jhi]). C and R hold C_j and
    // R_j of tap j0 - 1 (0 and 0 before jlo) and are advanced to tap j0 + 31, so consecutive calls walk the taps in runs of 32
    B200_DEV int scan_weight(int j0, int lane, int64_t T, int64_t &C, int64_t &R) const
    {
        const int jj = j0 + lane;
        int64_t c = jj >= jlo && jj <= jhi ? t(jj) : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t v = __shfl_up_sync(0xffffffffu, c, o);
            if (lane >= o) c += v;
        }
        c += C;
        const int64_t r = floor_div(c * 32768 + T, 2 * T);
        int64_t rp = __shfl_up_sync(0xffffffffu, r, 1);
        if (lane == 0) rp = R;
        C = __shfl_sync(0xffffffffu, c, 31); R = __shfl_sync(0xffffffffu, r, 31);
        return (int)(r - rp);
    }
};

// the tensor kernels' filters: export_tensor_kernel's bilinear, export_tensor_aa_kernel's triangle and cubic
enum { kBilinear = 0, kTriangle = 1, kCubic = 2 };
template <int F>
B200_DEV auto filter_axis(const B200TensorJob &j, int x, int in, int out, int n, int s, int k)
{
    if constexpr (F == kCubic) return CubicAxis(x, in, out, n, s, k, j.antialias);
    else return AaAxis(x, in, out, n, s, k);
}

// A CTA owns kAaCols output columns x th output rows of one job (th = 1 .. kAaRowsMax, chosen per launch so that a single
// picture still fills the GPU). Per plane it walks the tile's source rows in chunks of kAaChunk: the horizontal sums H' of
// the chunk (a warp per row, a lane per column; the column weights sit in shared memory, kAaTaps at a time) go to shared
// memory, then each thread adds wy * H' into the vertical sums of its output pixels. Shared memory does not depend on the
// reduction factor; source samples are read straight from global memory, each source row once per tile.
// F = kTriangle: the antialiased bilinear definition; kCubic: both bicubic ones, job.antialias choosing the weight rule
// in the weight fills alone. The antialiased cubic weights are cumulative sums: a warp owns a column (or an output row)
// and scans its taps 32 at a time, carrying C_j and R_j in shared memory across tap windows (row chunks).
constexpr int kAaCols = 32, kAaRowsMax = 32, kAaChunk = 32, kAaTaps = 64;
template <bool HBD, int DT, bool HWC, int N, bool MIRROR, int F, int EPI>
__global__ void __launch_bounds__(256, kMinBlocks<EPI>) export_tensor_aa_kernel(const __grid_constant__ TensorBatch<N, batch_of(EPI)> b, int th)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    __shared__ int wx[kAaCols][kAaTaps + 1];         // column weights of the current tap window
    __shared__ int hs[kAaChunk][kAaCols + 1];        // H' of the current row chunk
    __shared__ int wy[kAaRowsMax][kAaChunk];         // row weights of the current row chunk
    __shared__ int qs[3][kAaRowsMax][kAaCols];       // Q of the tile
    __shared__ int cjlo[kAaCols], cnt[kAaCols];
    const B200TensorJob &j = b.job[N == 1 ? 0 : blockIdx.z];
    if constexpr (EPI == kEpiContrast)
        if (!((jitter_of(b)->enabled >> kJitContrast) & 1)) return;
    const int x0 = blockIdx.x * kAaCols, y0 = blockIdx.y * th;
    if (x0 >= j.out_w || y0 >= j.out_h) return;        // the whole CTA
    const int lane = threadIdx.x, warp = threadIdx.y, tid = warp * 32 + lane;
    const int rows = imin(th, j.out_h - y0);
    for (int p = 0; p < (j.mono ? 1 : 3); p++) {
        const int sh = p ? j.ss_hor : 0, sv = p ? j.ss_ver : 0;
        const int kx = sh ? j.siting_x : 0, ky = sv ? j.siting_y : 0;
        const int pw = (j.w + sh) >> sh, ph = (j.h + sv) >> sv;
        const pixel *const plane = (const pixel *)j.src + j.plane_off[p];
        const int stride = j.stride[p];
        // this lane's column, and the tile's source rows [r_lo, r_hi]
        const bool col_in = x0 + lane < j.out_w;
        const auto cx = filter_axis<F>(j, col_in ? x0 + lane : x0, j.w, j.out_w, pw, sh, kx);
        const int ntaps = col_in ? cx.jhi - cx.jlo + 1 : 0;
        int windows = ntaps;                          // tap windows of the widest column
        for (int o = 16; o; o >>= 1) windows = imax(windows, __shfl_xor_sync(0xffffffffu, windows, o));
        windows = (windows + kAaTaps - 1) / kAaTaps;
        const int r_lo = filter_axis<F>(j, y0, j.h, j.out_h, ph, sv, ky).jlo;
        const int r_hi = filter_axis<F>(j, y0 + rows - 1, j.h, j.out_h, ph, sv, ky).jhi;
        __syncthreads();                              // the previous plane is done with the shared arrays
        if (warp == 0) { cjlo[lane] = cx.jlo; cnt[lane] = ntaps; }
        // antialiased cubic: T, and C_j / R_j of the last tap weighted so far, of every column (row), each kept by the warp
        // that owns the column (row): columns and rows warp + 8 q
        __shared__ int64_t cubic_T[2][kAaCols], cubic_C[2][kAaCols], cubic_R[2][kAaCols];
        const auto col_axis = [&](int c) { return CubicAxis(x0 + c, j.w, j.out_w, pw, sh, kx, true); };
        const auto row_axis = [&](int t) { return CubicAxis(y0 + t, j.h, j.out_h, ph, sv, ky, true); };
        if constexpr (F == kCubic) {
            if (j.antialias)
                for (int q = 0; q < kAaCols / 8; q++) {
                    const int c = warp + 8 * q;
                    if (x0 + c < j.out_w) cubic_T[0][c] = col_axis(c).total(lane);
                    if (c < rows) cubic_T[1][c] = row_axis(c).total(lane);
                    cubic_C[1][c] = cubic_R[1][c] = 0;
                }
        }
        const auto fill_wx = [&](int w0) {            // the weights of taps w0 .. w0 + kAaTaps - 1 of every column
            if constexpr (F == kCubic) {
                if (j.antialias) {
                    for (int q = 0; q < kAaCols / 8; q++) {
                        const int c = warp + 8 * q;
                        if (x0 + c >= j.out_w) {
                            wx[c][lane] = wx[c][lane + 32] = 0;
                            continue;
                        }
                        const CubicAxis a = col_axis(c);
                        int64_t C = w0 ? cubic_C[0][c] : 0, R = w0 ? cubic_R[0][c] : 0;
                        for (int i = 0; i < kAaTaps; i += 32) wx[c][i + lane] = a.scan_weight(a.jlo + w0 + i, lane, cubic_T[0][c], C, R);
                        if (lane == 0) { cubic_C[0][c] = C; cubic_R[0][c] = R; }
                    }
                    return;
                }
            }
            for (int e = tid; e < kAaCols * kAaTaps; e += 256) {
                const int c = e / kAaTaps, i = e % kAaTaps;
                const bool in = x0 + c < j.out_w && w0 + i < cnt[c];
                if constexpr (F == kCubic)
                    wx[c][i] = in ? CubicAxis(x0 + c, j.w, j.out_w, pw, sh, kx, false).plain_weight(cjlo[c] + w0 + i, pw) : 0;
                else
                    wx[c][i] = in ? AaAxis(x0 + c, j.w, j.out_w, pw, sh, kx).weight(cjlo[c] + w0 + i) : 0;
            }
        };
        __syncthreads();
        if (windows == 1) fill_wx(0);
        int acc[kAaRowsMax / 8] = {};                 // V of output rows warp + 8 k, column lane
        for (int r0 = r_lo; r0 <= r_hi; r0 += kAaChunk) {
            const int nr = imin(kAaChunk, r_hi - r0 + 1);
            int h[kAaChunk / 8] = {};
            for (int w0 = 0; w0 < windows * kAaTaps; w0 += kAaTaps) {
                if (windows > 1) { __syncthreads(); fill_wx(w0); }
                __syncthreads();
                const int m = imin(kAaTaps, ntaps - w0);
                const pixel *const src = plane + cx.jlo + w0;
#pragma unroll
                for (int k = 0; k < kAaChunk / 8; k++) {
                    const int r = warp + 8 * k;
                    if (r < nr) {
                        const pixel *const row = src + (ptrdiff_t)(r0 + r) * stride;
                        int sum = 0;
                        for (int i = 0; i < m; i++) sum += wx[lane][i] * (int)__ldg(row + i);
                        h[k] += sum;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < kAaChunk / 8; k++) {
                if constexpr (F == kCubic) hs[warp + 8 * k][lane] = iclip((h[k] + (1 << 9)) >> 10, 0, 16 * j.bitdepth_max);
                else hs[warp + 8 * k][lane] = (h[k] + (1 << 8)) >> 9;
            }
            if (F == kCubic && j.antialias) {
                for (int t = warp; t < rows; t += 8) {
                    int64_t C = cubic_C[1][t], R = cubic_R[1][t];
                    wy[t][lane] = row_axis(t).scan_weight(r0, lane, cubic_T[1][t], C, R);
                    if (lane == 0) { cubic_C[1][t] = C; cubic_R[1][t] = R; }
                }
            } else {
                for (int e = tid; e < rows * kAaChunk; e += 256) {
                    const int t = e / kAaChunk, r = e % kAaChunk;
                    if constexpr (F == kCubic)
                        wy[t][r] = r < nr ? CubicAxis(y0 + t, j.h, j.out_h, ph, sv, ky, false).plain_weight(r0 + r, ph) : 0;
                    else
                        wy[t][r] = r < nr ? AaAxis(y0 + t, j.h, j.out_h, ph, sv, ky).weight(r0 + r) : 0;
                }
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < kAaRowsMax / 8; k++) {
                const int t = warp + 8 * k;
                if (t < rows) {
                    int v = 0;
                    for (int r = 0; r < nr; r++) v += wy[t][r] * hs[r][lane];
                    acc[k] += v;
                }
            }
            __syncthreads();                          // hs and wy are rewritten by the next chunk
        }
#pragma unroll
        for (int k = 0; k < kAaRowsMax / 8; k++) {
            if (warp + 8 * k >= rows) continue;
            if constexpr (F == kCubic) qs[p][warp + 8 * k][lane] = iclip((acc[k] + (1 << 15)) >> 16, 0, 4 * j.bitdepth_max);
            else qs[p][warp + 8 * k][lane] = (acc[k] + (1 << 16)) >> 17;
        }
    }
    __syncthreads();
    const int bdmax = j.bitdepth_max, s = bdmax == 4095 ? 4 : bdmax == 1023 ? 2 : 0;
    const int yoff = j.full_range ? 0 : 64 << s, coff = 512 << s;
    // the epilogue: a thread per run of 4 columns of one row (the jitter's arguments taken here, not held through the loops)
    uint32_t sum = 0;
    const JitterArgs ja = jitter_args<EPI>(b, j, &sum);
    for (int e = tid; e < rows * (kAaCols / 4); e += 256) {
        const int t = e / (kAaCols / 4), c = 4 * (e % (kAaCols / 4)), x = x0 + c;
        if (x >= j.out_w) continue;
        int qy[4], qu[4] = {}, qv[4] = {};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            qy[i] = qs[0][t][c + i];
            if (!j.mono) { qu[i] = qs[1][t][c + i]; qv[i] = qs[2][t][c + i]; }
        }
        tensor_store<DT, HWC, MIRROR, EPI>(j, tone_of(b), x, y0 + t, imin(4, j.out_w - x), qy, qu, qv, yoff, coff, 4 * bdmax,
                                           ja);
    }
    if constexpr (EPI == kEpiContrast) contrast_add(*jitter_of(b), sum);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_export_picture(const B200ExportJob *job, void *stream)
{
    if (!job) { b200_set_error("b200_export_picture: no job"); return -2; }
    const B200ExportJob &j = *job;
    if (int r = check_bdmax(j.bitdepth_max, "b200_export_picture")) return r;
    const int rgb = j.format == B200_EXPORT_RGB, npl = j.mono ? 1 : 3;
    if ((j.format != B200_EXPORT_PLANES && !rgb) || j.w < 1 || j.h < 1 || (unsigned)j.ss_hor > 1 || (unsigned)j.ss_ver > 1 || !j.src) {
        b200_set_error("b200_export_picture: bad arguments (format %d, %d x %d)", j.format, j.w, j.h);
        return -2;
    }
    if (rgb && j.identity && (j.mono || j.ss_hor || j.ss_ver)) { b200_set_error("b200_export_picture: identity matrix needs 4:4:4"); return -2; }
    for (int p = 0; p < (rgb ? 3 : npl); p++)
        if (!j.dst[p] || j.dst_pitch[p] < (p && !rgb ? (j.w + j.ss_hor) >> j.ss_hor : j.w)) {
            b200_set_error("b200_export_picture: bad destination %d", p);
            return -2;
        }
    const int run = j.bitdepth_max > 255 ? 4 : 8, runs = (j.w + run - 1) / run;
    const dim3 block(32, 8);
    if (!rgb)
        return launch_hbd(j.bitdepth_max, Launch::pdl, dim3((runs + 31) / 32, (j.h + 7) / 8, npl), block, 0, (cudaStream_t)stream,
                          [&](auto hbd) { return std::make_tuple(export_planes_kernel<hbd>, j); });
    const int groups = (j.h + j.ss_ver) >> j.ss_ver;
    return launch_hbd(j.bitdepth_max, Launch::pdl, dim3((runs + 31) / 32, (groups + 7) / 8), block, 0, (cudaStream_t)stream,
                      [&](auto hbd) { return std::make_tuple(j.ss_hor ? export_rgb_kernel<hbd, 1> : export_rgb_kernel<hbd, 0>, j); });
}

// every field of one tensor job, checked as it arrives from outside the library: 0, or -2 with the error set
static int check_tensor_job(const B200TensorJob &j, const char *who)
{
    if (int r = check_bdmax(j.bitdepth_max, who)) return r;
    const auto in_range = [](int v, int lo, int hi) { return v >= lo && v <= hi; };
    if (!j.src || !in_range(j.w, 1, 65536) || !in_range(j.h, 1, 65536) || !in_range(j.out_w, 1, 65536) || !in_range(j.out_h, 1, 65536) ||
        !in_range(j.ss_hor, 0, 1) || !in_range(j.ss_ver, 0, 1) || !in_range(j.siting_x, 0, 1) || !in_range(j.siting_y, 0, 1) ||
        !in_range(j.dtype, B200_TENSOR_F32, B200_TENSOR_BF16) || !in_range(j.layout, B200_TENSOR_CHW, B200_TENSOR_HWC) ||
        !in_range(j.antialias, 0, 1) || !in_range(j.flip, 0, 1) || !in_range(j.interpolation, B200_TENSOR_BILINEAR, B200_TENSOR_BICUBIC)) {
        b200_set_error("%s: bad arguments (%d x %d -> %d x %d, dtype %d, layout %d, antialias %d, flip %d, interpolation %d)", who,
                       j.w, j.h, j.out_w, j.out_h, j.dtype, j.layout, j.antialias, j.flip, j.interpolation);
        return -2;
    }
    if (j.identity && (j.mono || j.ss_hor || j.ss_ver)) { b200_set_error("%s: identity matrix needs 4:4:4", who); return -2; }
    for (int p = 0; p < (j.mono ? 1 : 3); p++)
        if (j.stride[p] < (p ? (j.w + j.ss_hor) >> j.ss_hor : j.w)) {
            b200_set_error("%s: stride of plane %d too small", who, p);
            return -2;
        }
    // the addresses of the last element of every channel must fit int64 with room to spare
    const int64_t esize = j.dtype == B200_TENSOR_F32 ? 4 : 2, row = j.layout == B200_TENSOR_HWC ? 3 * (int64_t)j.out_w : j.out_w;
    const int64_t lim = ((int64_t)1 << 52) / esize;
    const bool pitch_ok = j.pitch_y >= row && j.pitch_y <= lim / j.out_h;
    if (!j.dst || ((uintptr_t)j.dst % esize) || !pitch_ok ||
        (j.layout == B200_TENSOR_CHW && (j.pitch_c < (j.out_h - 1) * j.pitch_y + row || j.pitch_c > lim / 3))) {
        b200_set_error("%s: bad destination (pitches %lld, %lld)", who, (long long)j.pitch_c, (long long)j.pitch_y);
        return -2;
    }
    return 0;
}

// the kernel a job takes: the bilinear export_tensor_kernel, the tile kernel's triangle (antialias = 1 with a reduced luma
// axis: sigma > 256, include/b200av1.h) or its cubic (bicubic, plain or antialiased, whatever the scale)
static int tensor_job_kind(const B200TensorJob &j)
{
    if (j.interpolation == B200_TENSOR_BICUBIC) return kCubic;
    const bool reduced = (int64_t)j.w * 256 / j.out_w > 256 || (int64_t)j.h * 256 / j.out_h > 256;
    return j.antialias && reduced ? kTriangle : kBilinear;
}

// the tile kernel's launch: the tallest tile (th output rows) whose grid still has kAaMinCtas CTAs, the SM count of an
// H100 SXM, so that a single picture reduced to a small output still spreads over the whole GPU
constexpr int kAaMinCtas = 132;
template <int N, int F, int E>
static int launch_tensor_aa_jobs(const TensorBatch<N, batch_of(E)> &b, int n, int out_w, int out_h, cudaStream_t stream)
{
    const B200TensorJob &j = b.job[0];
    const int xt = (out_w + kAaCols - 1) / kAaCols;
    int th = kAaRowsMax;
    while (th > 1 && (int64_t)xt * ((out_h + th - 1) / th) * n < kAaMinCtas) th >>= 1;
    const dim3 grid(xt, (out_h + th - 1) / th, n);
    return launch_hbd(j.bitdepth_max, Launch::pdl, grid, dim3(32, 8), 0, stream, [&](auto hbd) {
        constexpr bool H = decltype(hbd)::value;
        if constexpr (E == kEpiContrast) {          // S depends on none of dtype, layout and flip
            return std::make_tuple(export_tensor_aa_kernel<H, B200_TENSOR_F32, false, N, false, F, E>, b, th);
        } else {
            void (*const k[2][3][2])(TensorBatch<N, E>, int) = {
                {{export_tensor_aa_kernel<H, B200_TENSOR_F32, false, N, false, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_F32, true, N, false, F, E>},
                 {export_tensor_aa_kernel<H, B200_TENSOR_F16, false, N, false, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_F16, true, N, false, F, E>},
                 {export_tensor_aa_kernel<H, B200_TENSOR_BF16, false, N, false, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_BF16, true, N, false, F, E>}},
                {{export_tensor_aa_kernel<H, B200_TENSOR_F32, false, N, true, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_F32, true, N, true, F, E>},
                 {export_tensor_aa_kernel<H, B200_TENSOR_F16, false, N, true, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_F16, true, N, true, F, E>},
                 {export_tensor_aa_kernel<H, B200_TENSOR_BF16, false, N, true, F, E>, export_tensor_aa_kernel<H, B200_TENSOR_BF16, true, N, true, F, E>}}};
            return std::make_tuple(k[j.flip][j.dtype][j.layout], b, th);
        }
    });
}

// one launch of the epilogue E for the n jobs of b, all of one bit-depth class, dtype, layout, kernel kind and flip
template <int N, int E>
static int launch_tensor_kind(const TensorBatch<N, batch_of(E)> &b, int n, int kind, cudaStream_t stream)
{
    int out_w = 0, out_h = 0;
    for (int i = 0; i < n; i++) { out_w = imax(out_w, b.job[i].out_w); out_h = imax(out_h, b.job[i].out_h); }
    if (kind == kTriangle) return launch_tensor_aa_jobs<N, kTriangle, E>(b, n, out_w, out_h, stream);
    if (kind == kCubic) return launch_tensor_aa_jobs<N, kCubic, E>(b, n, out_w, out_h, stream);
    const B200TensorJob &j = b.job[0];
    const int runs = (out_w + 3) / 4;
    const dim3 grid((runs + 31) / 32, (out_h + 8 * kTensorRows - 1) / (8 * kTensorRows), n);
    return launch_hbd(j.bitdepth_max, Launch::pdl, grid, dim3(32, 8), 0, stream, [&](auto hbd) {
        constexpr bool H = decltype(hbd)::value;
        if constexpr (E == kEpiContrast) {
            return std::make_tuple(export_tensor_kernel<H, B200_TENSOR_F32, false, N, false, E>, b);
        } else {
            void (*const k[2][3][2])(TensorBatch<N, E>) = {
                {{export_tensor_kernel<H, B200_TENSOR_F32, false, N, false, E>, export_tensor_kernel<H, B200_TENSOR_F32, true, N, false, E>},
                 {export_tensor_kernel<H, B200_TENSOR_F16, false, N, false, E>, export_tensor_kernel<H, B200_TENSOR_F16, true, N, false, E>},
                 {export_tensor_kernel<H, B200_TENSOR_BF16, false, N, false, E>, export_tensor_kernel<H, B200_TENSOR_BF16, true, N, false, E>}},
                {{export_tensor_kernel<H, B200_TENSOR_F32, false, N, true, E>, export_tensor_kernel<H, B200_TENSOR_F32, true, N, true, E>},
                 {export_tensor_kernel<H, B200_TENSOR_F16, false, N, true, E>, export_tensor_kernel<H, B200_TENSOR_F16, true, N, true, E>},
                 {export_tensor_kernel<H, B200_TENSOR_BF16, false, N, true, E>, export_tensor_kernel<H, B200_TENSOR_BF16, true, N, true, E>}}};
            return std::make_tuple(k[j.flip][j.dtype][j.layout], b);
        }
    });
}

// the launches of the n (1 .. N) jobs at `jobs`, all of one bit-depth class, dtype, layout, kernel kind and flip, with
// (E = kEpiTone) the tone maps at `tones`, or (kEpiJitter) the optional tone maps at `tones` and the jitters at `jits`.
// Jittered jobs with contrast first take their contrast pass: S zeroed, then summed by the kernel's sampling code; the
// export's B200_PDL_ENTRY waits for it before reading S.
template <int N, int E>
static int launch_tensor_jobs(const B200TensorJob *const *jobs, const B200ToneMap *const *tones, const B200ColorJitter *const *jits,
                              int n, int kind, cudaStream_t stream)
{
    TensorBatch<N, E> b{};
    bool contrast = false;
    for (int i = 0; i < n; i++) {
        b.job[i] = *jobs[i];
        if constexpr (E != kEpiPlain) if (tones[i]) b.tone[i] = *tones[i];
        if constexpr (E == kEpiJitter) {
            b.jit[i] = *jits[i];
            contrast |= (jits[i]->enabled >> kJitContrast) & 1;
        }
    }
    if constexpr (E == kEpiJitter) {
        if (contrast) {
            if (int r = launch_hbd(b.job[0].bitdepth_max, Launch::pdl, dim3(1), dim3(32), 0, stream,
                                   [&](auto) { return std::make_tuple(contrast_zero_kernel<N>, b, n); }))
                return r;
            if (int r = launch_tensor_kind<N, kEpiContrast>(b, n, kind, stream)) return r;
        }
    }
    return launch_tensor_kind<N, E>(b, n, kind, stream);
}
// the tone-mapped and jittered forms are batched forms only: the N = 1 specialisation would double their build time for
// a prologue
static int launch_tensor_group(const B200TensorJob *const *jobs, const B200ToneMap *const *tones, const B200ColorJitter *const *jits,
                               int n, int kind, int epi, cudaStream_t stream)
{
    if (epi == kEpiJitter) return launch_tensor_jobs<B200_TENSOR_JITTER_BATCH_MAX, kEpiJitter>(jobs, tones, jits, n, kind, stream);
    if (epi == kEpiTone) return launch_tensor_jobs<B200_TENSOR_TONE_BATCH_MAX, kEpiTone>(jobs, tones, jits, n, kind, stream);
    return n == 1 ? launch_tensor_jobs<1, kEpiPlain>(jobs, tones, jits, n, kind, stream)
                  : launch_tensor_jobs<B200_TENSOR_BATCH_MAX, kEpiPlain>(jobs, tones, jits, n, kind, stream);
}

extern "C" int b200_export_tensor(const B200TensorJob *job, void *stream)
{
    return b200_export_tensor_batch(job, 1, stream);
}

extern "C" int b200_export_tensor_batch(const B200TensorJob *jobs, int n, void *stream)
{
    return b200_export_tensor_tone_batch(jobs, nullptr, n, stream);
}

extern "C" int b200_export_tensor_tone_batch(const B200TensorJob *jobs, const B200ToneMap *const *tones, int n, void *stream)
{
    return b200_export_tensor_jitter_batch(jobs, tones, nullptr, n, stream);
}

// a job's tone map, checked as it arrives from outside the library: 0, or -2 with the error set
static int check_tone_map(const B200ToneMap &t, const B200TensorJob &j, int i, const char *who)
{
    bool finite = true;
    for (int k = 0; k < 9; k++) finite &= std::isfinite(t.m[k]);
    if (!t.curve || !t.oetf || t.curve_len != 4 * j.bitdepth_max + 1 || t.oetf_bits < 8 || t.oetf_bits > 16 || !finite) {
        b200_set_error("%s: bad tone map of job %d (curve_len %d for bitdepth_max %d, oetf_bits %d)", who, i,
                       t.curve_len, j.bitdepth_max, t.oetf_bits);
        return -2;
    }
    return 0;
}

// a job's colour jitter, checked as it arrives from outside the library: 0, or -2 with the error set
static int check_jitter(const B200ColorJitter &t, int i, const char *who)
{
    const float f[6] = {t.brightness, t.contrast, t.saturation, t.hue, t.contrast1, t.saturation1};
    bool finite = true;
    for (float v : f) finite &= std::isfinite(v);
    int seen = 0;
    for (int k = 0; k < 4; k++) seen |= (unsigned)t.order[k] < 4 ? 1 << t.order[k] : 16;
    const bool contrast = (t.enabled >> kJitContrast) & 1;
    if (!finite || t.brightness < 0 || t.contrast < 0 || t.saturation < 0 || !(t.hue >= -0.5f && t.hue <= 0.5f) || seen != 15 ||
        (t.enabled & ~15) || (unsigned)t.grayscale > 1 || (contrast && (!t.acc || ((uintptr_t)t.acc & 7)))) {
        b200_set_error("%s: bad colour jitter of job %d (factors %g %g %g %g, order %d %d %d %d, enabled %#x, grayscale %d, acc %p)",
                       who, i, t.brightness, t.contrast, t.saturation, t.hue, t.order[0], t.order[1], t.order[2], t.order[3],
                       t.enabled, t.grayscale, (const void *)t.acc);
        return -2;
    }
    return 0;
}

extern "C" int b200_export_tensor_jitter_batch(const B200TensorJob *jobs, const B200ToneMap *const *tones,
                                               const B200ColorJitter *const *jits, int n, void *stream)
{
    const char *const who = jits ? "b200_export_tensor_jitter_batch" : tones ? "b200_export_tensor_tone_batch"
                                                                      : n == 1 ? "b200_export_tensor" : "b200_export_tensor_batch";
    if (!jobs || n < 1) { b200_set_error("%s: no jobs (%d)", who, n); return -2; }
    for (int i = 0; i < n; i++) {
        if (int r = check_tensor_job(jobs[i], who)) return r;
        if (jobs[i].dtype != jobs[0].dtype || jobs[i].layout != jobs[0].layout) {
            b200_set_error("%s: job %d has another dtype or layout than job 0", who, i);
            return -2;
        }
        if (tones && tones[i])
            if (int r = check_tone_map(*tones[i], jobs[i], i, who)) return r;
        if (jits && jits[i])
            if (int r = check_jitter(*jits[i], i, who)) return r;
    }
    // one launch per bit-depth class, kernel kind (bilinear, triangle, cubic), flip and epilogue (plain, tone-mapped,
    // jittered with or without a tone map) and per B200_TENSOR_BATCH_MAX (tone-mapped: B200_TENSOR_TONE_BATCH_MAX,
    // jittered: B200_TENSOR_JITTER_BATCH_MAX) jobs of it, jobs in their order
    for (int group = 0; group < 36; group++) {
        const int hbd = group & 1, kind = (group >> 1) % 3, flip = (group / 6) & 1, epi = group / 12;
        const int cap = epi == kEpiJitter ? B200_TENSOR_JITTER_BATCH_MAX : epi == kEpiTone ? B200_TENSOR_TONE_BATCH_MAX : B200_TENSOR_BATCH_MAX;
        const B200TensorJob *part[B200_TENSOR_BATCH_MAX];
        const B200ToneMap *tpart[B200_TENSOR_BATCH_MAX];
        const B200ColorJitter *jpart[B200_TENSOR_BATCH_MAX];
        int m = 0;
        for (int i = 0; i < n; i++) {
            const B200ToneMap *const t = tones ? tones[i] : nullptr;
            const B200ColorJitter *const c = jits ? jits[i] : nullptr;
            const int e = c ? kEpiJitter : t ? kEpiTone : kEpiPlain;
            if ((jobs[i].bitdepth_max > 255) != hbd || tensor_job_kind(jobs[i]) != kind || jobs[i].flip != flip || e != epi) continue;
            part[m] = &jobs[i]; tpart[m] = t; jpart[m++] = c;
            if (m == cap) {
                if (int r = launch_tensor_group(part, tpart, jpart, m, kind, epi, (cudaStream_t)stream)) return r;
                m = 0;
            }
        }
        if (m)
            if (int r = launch_tensor_group(part, tpart, jpart, m, kind, epi, (cudaStream_t)stream)) return r;
    }
    return 0;
}
