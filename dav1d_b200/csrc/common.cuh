// Shared device/host helpers for the sm_90a kernels of the AV1 reconstruction back end.
#pragma once
#ifndef B200_EMU
#include <cuda_runtime.h>
#include <stdlib.h>
#define B200_LAUNCH(kern, grid, block, smem, stream, ...) \
    kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
// Programmatic dependent launch for the kernels of a frame job: the next kernel's CTAs may become resident while the
// previous kernel's last wave drains (they park in b200_pdl_entry() until it has completed and its writes are visible), so
// the launch latency and the ramp-up of every stage overlap the tail of the stage before it. A frame is a chain of a dozen
// dependent launches (a band of a frame another dozen), each paying launch latency + drain.
// Every kernel launched this way calls B200_PDL_ENTRY() before anything else (every thread, before any return).
// It pays on ONE chain of kernels (whole-frame jobs); when several chains share the GPU (banded frames:
// reconstruction and post-filter chains, two frames in flight) the parked CTAs take the slots the other chain's kernels
// would have used, so the pipeline turns it off there (b200_set_pdl).
bool b200_pdl_enabled();         // capi.cu: b200_set_pdl() / B200_NO_PDL
template <class... KArgs, class... Args>
inline void b200_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args &&...args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = b200_pdl_enabled() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#define B200_LAUNCH_PDL(kern, grid, block, smem, stream, ...) b200_launch_pdl(kern, grid, block, smem, stream, __VA_ARGS__)
#define B200_PDL_ENTRY() do { asm volatile("griddepcontrol.launch_dependents;"); asm volatile("griddepcontrol.wait;" ::: "memory"); } while (0)
#else
#define B200_LAUNCH_PDL B200_LAUNCH
#define B200_PDL_ENTRY() do { } while (0)
#endif
#include <stdint.h>
#include <stddef.h>

#define B200_DEV __device__ __forceinline__
#define B200_HD __host__ __device__ __forceinline__

namespace b200 {

// SMs of the target GPU (H100 SXM): the size of the persistent and capped grids
constexpr int kSmCount = 132;

B200_HD int imin(int a, int b) { return a < b ? a : b; }
B200_HD int imax(int a, int b) { return a > b ? a : b; }
// min / max form (lo <= hi everywhere): sm_90a fuses the producing add into VIADDMNMX, so add + clamp is two instructions
// instead of four (ISETP + predicated VIMNMX sequence); iclip is a large share of the transform kernel's instructions
B200_HD int iclip(int v, int lo, int hi) { return imax(lo, imin(v, hi)); }
B200_HD int iabs(int v) { return v < 0 ? -v : v; }
B200_HD int ulog2(unsigned v) {
#if defined(__CUDA_ARCH__)
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}

// ceil(65536 / d) for d < 64: the multiplier of the "exact i / d for small i" trick ((i * m) >> 16) that the tile loops use
// to split a flat work-item index. A constant-memory lookup instead of a 20-instruction unsigned division executed by
// every thread (a few percent of the instructions of the LR, CDEF and prediction kernels).
#ifndef B200_EMU
static __constant__ uint32_t c_recip16[64] = { 0, 65536, 32768, 21846, 16384, 13108, 10923, 9363, 8192, 7282, 6554, 5958, 5462, 5042, 4682, 4370, 4096, 3856, 3641, 3450, 3277, 3121, 2979, 2850, 2731, 2622, 2521, 2428, 2341, 2260, 2185, 2115, 2048, 1986, 1928, 1873, 1821, 1772, 1725, 1681, 1639, 1599, 1561, 1525, 1490, 1457, 1425, 1395, 1366, 1338, 1311, 1286, 1261, 1237, 1214, 1192, 1171, 1150, 1130, 1111, 1093, 1075, 1058, 1041 };
#else
static const uint32_t c_recip16[64] = { 0, 65536, 32768, 21846, 16384, 13108, 10923, 9363, 8192, 7282, 6554, 5958, 5462, 5042, 4682, 4370, 4096, 3856, 3641, 3450, 3277, 3121, 2979, 2850, 2731, 2622, 2521, 2428, 2341, 2260, 2185, 2115, 2048, 1986, 1928, 1873, 1821, 1772, 1725, 1681, 1639, 1599, 1561, 1525, 1490, 1457, 1425, 1395, 1366, 1338, 1311, 1286, 1261, 1237, 1214, 1192, 1171, 1150, 1130, 1111, 1093, 1075, 1058, 1041 };
#endif
B200_DEV unsigned recip16(int d) { return d < 64 ? (unsigned)c_recip16[d] : (d & (d - 1)) ? (65536u + d - 1) / d : 65536u >> (31 - __clz(d)); }

// transform size tx -> (w, h, inter-pass shift), largest first: reference src/itx_tmpl.c:160-178
#define B200_ITX_SIZES(X) \
    X(4, 64, 64, 2) X(11, 32, 64, 1) X(12, 64, 32, 1) X(17, 16, 64, 2) X(18, 64, 16, 2) X(3, 32, 32, 2) X(9, 16, 32, 1) \
    X(10, 32, 16, 1) X(15, 8, 32, 2) X(16, 32, 8, 2) X(2, 16, 16, 2) X(7, 8, 16, 1) X(8, 16, 8, 1) X(13, 4, 16, 1) \
    X(14, 16, 4, 1) X(1, 8, 8, 1) X(5, 4, 8, 0) X(6, 8, 4, 0) X(0, 4, 4, 0)

// pixel / coefficient types per bit-depth class (reference include/common/bitdepth.h:42-86)
template <bool HBD> struct Bd;
template <> struct Bd<false> { typedef uint8_t pixel; typedef int16_t coef; };
template <> struct Bd<true> { typedef uint16_t pixel; typedef int32_t coef; };

}  // namespace b200

// error plumbing for the C ABI (capi.cu)
void b200_set_error(const char *fmt, ...);
#define B200_CUDA_OK(expr)                                                                   \
    do {                                                                                     \
        cudaError_t e_ = (expr);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            b200_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
            return -1;                                                                       \
        }                                                                                    \
    } while (0)
