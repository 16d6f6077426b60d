// Export of a decoded picture from its device copy into caller-owned device memory (B200ExportJob, B200TensorJob,
// include/b200av1.h):
//   export_planes_kernel  Y / U / V cropped to the visible size, tightly packed
//   export_rgb_kernel     planar R / G / B at the stream's bit depth (nearest chroma sample, integer matrix)
//   export_tensor_kernel  R / G / B resized (bilinear, chroma upsampling included), normalised, as fp32 / fp16 / bf16 in
//                         CHW or HWC order: what a model takes, in one pass
// Memory bound: a thread owns a run of horizontally adjacent output samples (8 bytes: 8 samples at 8 bit, 4 above), read
// and written with one 8-byte access where the run is complete and the rows are aligned; the RGB kernel of a vertically
// sub-sampled picture takes two rows per thread, so that each chroma sample is read once for its 2 x 2 luma quad. The
// tensor kernel's thread owns 4 adjacent output pixels, written per channel with one 16-byte (fp32) or 8-byte store.
#include "common.cuh"
#include "host_util.h"
#ifndef B200_EMU
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#else
// Host build of these sources (tests/emu): the rounding intrinsics of the tensor export with the same results. Each fp32
// operation is rounded on its own (the volatile store keeps the compiler from contracting a multiply and an add into an
// FMA), and g++'s _Float16 / __bf16 conversions round to nearest even like __float2half_rn / __float2bfloat16_rn.
typedef _Float16 __half;
typedef __bf16 __nv_bfloat16;
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline __half __float2half_rn(float v) { return (__half)v; }
static inline __nv_bfloat16 __float2bfloat16_rn(float v) { return (__nv_bfloat16)v; }
static inline unsigned short __half_as_ushort(__half h) { unsigned short u; memcpy(&u, &h, 2); return u; }
static inline unsigned short __bfloat16_as_ushort(__nv_bfloat16 h) { unsigned short u; memcpy(&u, &h, 2); return u; }
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

template <int DT>
B200_DEV typename TensorElem<DT>::type tensor_value(int v, float scale, float bias)
{
    const float f = __fadd_rn(__fmul_rn((float)v, scale), bias);
    if constexpr (DT == B200_TENSOR_F16) return __half_as_ushort(__float2half_rn(f));
    else if constexpr (DT == B200_TENSOR_BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(f));
    else return f;
}

// The jobs of one launch travel in the kernel's parameter block (no staging copy): B200_TENSOR_BATCH_MAX of them fit the
// classic 4 KB limit. A one-job launch takes the N = 1 form: its job's fields are then read at fixed parameter offsets, as
// operands of the instructions that use them; indexed by blockIdx.z they are separate loads, which made the prologue of a
// small one-picture export up to a quarter slower.
template <int N> struct TensorBatch { B200TensorJob job[N]; };
static_assert(sizeof(TensorBatch<B200_TENSOR_BATCH_MAX>) <= 4096, "the jobs of one launch must fit a 4 KB kernel parameter block");

// grid (runs of 4 output columns / 32, output rows / (8 * kTensorRows), jobs), block (32, 8): x / y cover the largest
// output of the launch, z selects the job. A thread converts its run of 4 columns on kTensorRows rows 8 apart, so the
// column taps are worked out once for all of them
constexpr int kTensorRows = 4;
template <bool HBD, int DT, bool HWC, int N>
__global__ void __launch_bounds__(256) export_tensor_kernel(const __grid_constant__ TensorBatch<N> b)
{
    B200_PDL_ENTRY();
    typedef typename Bd<HBD>::pixel pixel;
    typedef typename TensorElem<DT>::type E;
    const B200TensorJob &j = b.job[N == 1 ? 0 : blockIdx.z];
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y0 = blockIdx.y * 8 * kTensorRows + threadIdx.y;
    if (x >= j.out_w || y0 >= j.out_h) return;
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
        int qy[4], qu[4] = {}, qv[4] = {};
        run_samples(qy, src + j.plane_off[0], j.stride[0], lrow, j.h, lt);
        if (!j.mono) {
            run_samples(qu, src + j.plane_off[1], j.stride[1], crow, ch, ct);
            run_samples(qv, src + j.plane_off[2], j.stride[2], crow, ch, ct);
        }
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
#pragma unroll
            for (int c = 0; c < 3; c++) o[c][i] = tensor_value<DT>(rgb[c], j.scale[c], j.bias[c]);
        }
        E *const row = (E *)j.dst + y * j.pitch_y;
        if constexpr (HWC) {
            // the run is 12 contiguous values: R G B of pixel 0, then of pixel 1, ...
            E v[3][4];
#pragma unroll
            for (int e = 0; e < 12; e++) v[e >> 2][e & 3] = o[e % 3][e / 3];
#pragma unroll
            for (int r = 0; r < 3; r++) store_run(row + 3 * x + 4 * r, imin(4, 3 * n - 4 * r), v[r]);
        } else {
#pragma unroll
            for (int c = 0; c < 3; c++) store_run(row + c * j.pitch_c + x, n, o[c]);
        }
    }
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
        !in_range(j.dtype, B200_TENSOR_F32, B200_TENSOR_BF16) || !in_range(j.layout, B200_TENSOR_CHW, B200_TENSOR_HWC)) {
        b200_set_error("%s: bad arguments (%d x %d -> %d x %d, dtype %d, layout %d)", who, j.w, j.h, j.out_w, j.out_h,
                       j.dtype, j.layout);
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

// one launch for the n (1 .. N) jobs at `jobs`, all of one bit-depth class, dtype and layout
template <int N>
static int launch_tensor_jobs(const B200TensorJob *const *jobs, int n, cudaStream_t stream)
{
    TensorBatch<N> b{};
    int out_w = 0, out_h = 0;
    for (int i = 0; i < n; i++) {
        b.job[i] = *jobs[i];
        out_w = imax(out_w, jobs[i]->out_w); out_h = imax(out_h, jobs[i]->out_h);
    }
    const B200TensorJob &j = b.job[0];
    const int runs = (out_w + 3) / 4;
    const dim3 grid((runs + 31) / 32, (out_h + 8 * kTensorRows - 1) / (8 * kTensorRows), n);
    return launch_hbd(j.bitdepth_max, Launch::pdl, grid, dim3(32, 8), 0, stream, [&](auto hbd) {
        constexpr bool H = decltype(hbd)::value;
        void (*const k[3][2])(TensorBatch<N>) = {
            {export_tensor_kernel<H, B200_TENSOR_F32, false, N>, export_tensor_kernel<H, B200_TENSOR_F32, true, N>},
            {export_tensor_kernel<H, B200_TENSOR_F16, false, N>, export_tensor_kernel<H, B200_TENSOR_F16, true, N>},
            {export_tensor_kernel<H, B200_TENSOR_BF16, false, N>, export_tensor_kernel<H, B200_TENSOR_BF16, true, N>}};
        return std::make_tuple(k[j.dtype][j.layout], b);
    });
}
static int launch_tensor_jobs(const B200TensorJob *const *jobs, int n, cudaStream_t stream)
{
    return n == 1 ? launch_tensor_jobs<1>(jobs, n, stream) : launch_tensor_jobs<B200_TENSOR_BATCH_MAX>(jobs, n, stream);
}

extern "C" int b200_export_tensor(const B200TensorJob *job, void *stream)
{
    return b200_export_tensor_batch(job, 1, stream);
}

extern "C" int b200_export_tensor_batch(const B200TensorJob *jobs, int n, void *stream)
{
    if (!jobs || n < 1) { b200_set_error("b200_export_tensor_batch: no jobs (%d)", n); return -2; }
    for (int i = 0; i < n; i++) {
        if (int r = check_tensor_job(jobs[i], n == 1 ? "b200_export_tensor" : "b200_export_tensor_batch")) return r;
        if (jobs[i].dtype != jobs[0].dtype || jobs[i].layout != jobs[0].layout) {
            b200_set_error("b200_export_tensor_batch: job %d has another dtype or layout than job 0", i);
            return -2;
        }
    }
    // one launch per bit-depth class present and per B200_TENSOR_BATCH_MAX jobs of it, jobs in their order
    for (int hbd = 0; hbd < 2; hbd++) {
        const B200TensorJob *part[B200_TENSOR_BATCH_MAX];
        int m = 0;
        for (int i = 0; i < n; i++) {
            if ((jobs[i].bitdepth_max > 255) != hbd) continue;
            part[m++] = &jobs[i];
            if (m == B200_TENSOR_BATCH_MAX) {
                if (int r = launch_tensor_jobs(part, m, (cudaStream_t)stream)) return r;
                m = 0;
            }
        }
        if (m)
            if (int r = launch_tensor_jobs(part, m, (cudaStream_t)stream)) return r;
    }
    return 0;
}
