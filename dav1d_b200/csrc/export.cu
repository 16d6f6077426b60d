// Export of a decoded picture from its device copy into caller-owned device memory (B200ExportJob, include/b200av1.h):
//   export_planes_kernel  Y / U / V cropped to the visible size, tightly packed
//   export_rgb_kernel     planar R / G / B at the stream's bit depth (nearest chroma sample, integer matrix)
// Memory bound: a thread owns a run of horizontally adjacent output samples (8 bytes: 8 samples at 8 bit, 4 above), read
// and written with one 8-byte access where the run is complete and the rows are aligned; the RGB kernel of a vertically
// sub-sampled picture takes two rows per thread, so that each chroma sample is read once for its 2 x 2 luma quad.
#include "common.cuh"
#include "host_util.h"

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
    static_assert(B == 8, "run size");
    if (n == N && !((uintptr_t)p & (B - 1))) {
        uint2 u;
        memcpy(&u, v, 8);
        *(uint2 *)p = u;
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
