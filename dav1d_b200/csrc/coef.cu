// Coefficient stream expansion. The host emitter ships, per coded transform block, only the eob + 1 coefficients
// that can be non-zero, in scan order (what dav1d's decode_coefs walks, reference src/recon_tmpl.c:318-730, before
// it scatters them into the dense frame_thread.cf plane, src/decode.c:2852-2863). This kernel rebuilds the dense
// min(w,32) x min(h,32) blocks the transform kernels read: dense[scan[k]] = compact[k]. The dense buffer is zeroed
// first by the caller (b200_frame_run). One warp per block. Cuts the host->device traffic of a frame ~3x.
#include "host_util.h"
#define B200_SCAN_TBL __device__
#include "scan_gen.h"
#include "launch_count.h"

namespace b200 {

template <class coef>
__global__ void __launch_bounds__(128) coef_expand_kernel(const B200CoefBlock *__restrict__ recs, int n,
                                                          const coef *__restrict__ compact, coef *__restrict__ dense)
{
    B200_PDL_ENTRY();
    const int wi = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (wi >= n) return;
    const B200CoefBlock r = recs[wi];
    const uint16_t *scan = b200_scan + b200_scan_off[r.tx];
    const coef *src = compact + r.compact_off;
    coef *dst = dense + r.dense_off;
    for (int k = lane; k <= r.eob; k += 32) dst[scan[k]] = src[k];
}

}  // namespace b200

extern "C" {

int b200_coef_expand(int bitdepth_max, const B200CoefBlock *d_blocks, int n_blocks, const void *d_compact, void *d_dense,
                     void *stream)
{
    if (int r = b200::check_bdmax(bitdepth_max, "b200_coef_expand")) return r;
    if (n_blocks <= 0) return 0;
    return b200::launch_hbd(bitdepth_max, b200::Launch::pdl, dim3((n_blocks + 3) / 4), dim3(128), 0, (cudaStream_t)stream, [&](auto hbd) {
        typedef typename b200::Bd<hbd>::coef coef;
        return std::make_tuple(b200::coef_expand_kernel<coef>, d_blocks, n_blocks, (const coef *)d_compact, (coef *)d_dense);
    });
}

}
