// Coefficient stream expansion. The host emitter ships, per coded transform block, only the eob + 1 coefficients
// that can be non-zero, in scan order (what dav1d's decode_coefs walks, reference src/recon_tmpl.c:318-730, before
// it scatters them into the dense frame_thread.cf plane, src/decode.c:2852-2863). This kernel rebuilds the dense
// min(w,32) x min(h,32) blocks the transform kernels read: dense[scan[k]] = compact[k], where the scan is the one of
// the block's transform class (src/recon_tmpl.c:458-467, 548-576): dav1d_scans[tx] for the 2-D types, k for H_*,
// (k % sw) * sh + k / sw for V_*. The dense buffer is zeroed first by the caller (b200_frame_run). One warp per block.
// Cuts the host->device traffic of a frame ~3x.
#include "host_util.h"
#define B200_SCAN_TBL __device__
#include "scan_gen.h"
#include "launch_count.h"

namespace b200 {

// log2 of min(w, 32) / min(h, 32) per transform size
static __constant__ uint8_t c_coef_lw[B200_N_RECT_TX_SIZES] = { 2, 3, 4, 5, 5, 2, 3, 3, 4, 4, 5, 5, 5, 2, 4, 3, 5, 4, 5 };
static __constant__ uint8_t c_coef_lh[B200_N_RECT_TX_SIZES] = { 2, 3, 4, 5, 5, 3, 2, 4, 3, 5, 4, 5, 5, 4, 2, 5, 3, 5, 4 };

template <class coef>
__global__ void __launch_bounds__(128) coef_expand_kernel(const B200CoefBlock *__restrict__ recs, int n,
                                                          const coef *__restrict__ compact, coef *__restrict__ dense)
{
    B200_PDL_ENTRY();
    const int wi = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (wi >= n) return;
    const B200CoefBlock r = recs[wi];
    const coef *src = compact + r.compact_off;
    coef *dst = dense + r.dense_off;
    if (r.tx_class == 0) {
        const uint16_t *scan = b200_scan + b200_scan_off[r.tx];
        for (int k = lane; k <= r.eob; k += 32) dst[scan[k]] = src[k];
    } else if (r.tx_class == 1) {
        for (int k = lane; k <= r.eob; k += 32) dst[k] = src[k];
    } else {
        const int lw = c_coef_lw[r.tx], lh = c_coef_lh[r.tx];
        for (int k = lane; k <= r.eob; k += 32) dst[((k & ((1 << lw) - 1)) << lh) | (k >> lw)] = src[k];
    }
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
