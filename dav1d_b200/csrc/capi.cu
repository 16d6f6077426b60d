// C ABI of the back end (include/b200av1.h): error plumbing, the Level-1 drop-in function
// tables (record -> launch -> sync shims with dav1d's exact signatures) and the Level-2
// batched entry points. No CPU fallback anywhere: every path ends in a kernel launch.
#include "common.cuh"
#include "../../include/b200av1.h"
#include "host_util.h"
#include <atomic>
#include <mutex>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <utility>

namespace b200 {   // itx.cu
int launch_itx(int tx, const B200ItxBlock *blocks, int n, void *coefs, void *pic, const int32_t *st, int bdmax, int zero,
               cudaStream_t stream);
}

static thread_local char g_err[512];
static std::atomic<uint64_t> g_launches{0};

void b200_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void b200_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
static std::atomic<int> g_pdl{-1};
bool b200_pdl_enabled() {
    int v = g_pdl.load(std::memory_order_relaxed);
    if (v < 0) { v = getenv("B200_NO_PDL") ? 0 : 1; g_pdl.store(v, std::memory_order_relaxed); }
    return v != 0;
}

extern "C" {

int b200_version(void) { return 100; }
const char *b200_last_error(void) { return g_err; }
uint64_t b200_launch_count(void) { return g_launches.load(); }
void b200_set_pdl(int on) { g_pdl.store(on ? 1 : 0, std::memory_order_relaxed); }

void *b200_dev_alloc(size_t bytes) {
    void *p = nullptr;
    const cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
    if (e != cudaSuccess) { b200_set_error("b200_dev_alloc(%zu): %s", bytes, cudaGetErrorString(e)); return nullptr; }
    return p;
}
void b200_dev_free(void *p) { if (p) cudaFree(p); }
void *b200_host_alloc(size_t bytes) {
    void *p = nullptr;
    const cudaError_t e = cudaMallocHost(&p, bytes ? bytes : 1);
    if (e != cudaSuccess) { b200_set_error("b200_host_alloc(%zu): %s", bytes, cudaGetErrorString(e)); return nullptr; }
    return p;
}
void b200_host_free(void *p) { if (p) cudaFreeHost(p); }
void *b200_stream_create(void) {
    cudaStream_t s = nullptr;
    const cudaError_t e = cudaStreamCreate(&s);
    if (e != cudaSuccess) { b200_set_error("b200_stream_create: %s", cudaGetErrorString(e)); return nullptr; }
#ifdef B200_EMU
    if (!s) return (void *)(uintptr_t)1;      // the host emulator has no stream objects; NULL means failure to callers
#endif
    return (void *)s;
}
void b200_stream_destroy(void *stream) { if (stream) cudaStreamDestroy((cudaStream_t)stream); }
int b200_dev_memset(void *p, int value, size_t bytes, void *stream) {
    B200_CUDA_OK(cudaMemsetAsync(p, value, bytes, (cudaStream_t)stream));
    return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------
namespace {
// width and height of transform size tx (0 <= tx < 19)
void tx_size(int tx, int *w, int *h) {
#define X(TX, W, H, SH) if (tx == TX) { *w = W; *h = H; }
    B200_ITX_SIZES(X)
#undef X
}

// is (tx, txtp) a slot dav1d defines? (reference src/itx_tmpl.c:220-288)
bool itx_defined(int tx, int txtp) {
    if (tx < 0 || tx >= 19 || txtp < 0 || txtp > 16) return false;
    if (txtp == 16) return tx == 0;
    int w, h;
    tx_size(tx, &w, &h);
    const int mx = w > h ? w : h, mn = w < h ? w : h;
    if (mx == 64) return txtp == 0;
    if (mx == 32) return txtp == 0 || txtp == 9;
    if (mx == 16 && mn == 16) return txtp <= 11;
    return true;
}

using b200::die;
using b200::Level1;
enum { BLOCKS, COEF, PIC };   // Level1 scratch slots
}  // namespace

extern "C" {

int b200_itx_add_batch(int bitdepth_max, int tx, const B200ItxBlock *d_blocks, int n_blocks,
                       void *d_coef, void *d_pic, const int32_t stride_px[3], int zero_coefs,
                       void *stream)
{
    if (tx < 0 || tx >= 19) { b200_set_error("b200_itx_add_batch: bad tx %d", tx); return -2; }
    if (int r = b200::check_bdmax(bitdepth_max, "b200_itx_add_batch")) return r;
    if (n_blocks <= 0) return 0;
    return b200::launch_itx(tx, d_blocks, n_blocks, d_coef, d_pic, stride_px, bitdepth_max, zero_coefs, (cudaStream_t)stream);
}

int b200_itx_add_frame(int bitdepth_max, const void *const d_blocks[19], const int32_t n_blocks[19], void *d_coef,
                       void *d_pic, const int32_t stride_px[3], int zero_coefs, void *stream)
{
    if (int r = b200::check_bdmax(bitdepth_max, "b200_itx_add_frame")) return r;
    return b200::launch_itx_grouped(d_blocks, n_blocks, d_coef, d_pic, stride_px, bitdepth_max, zero_coefs, (cudaStream_t)stream);
}

int b200_itx_add_batch_host(int bitdepth_max, int tx, const B200ItxBlock *blocks, int n_blocks,
                            void *coef, size_t coef_bytes, void *pic, size_t pic_bytes,
                            const int32_t stride_px[3], int zero_coefs)
{
    Level1 L;
    if (n_blocks <= 0) return 0;
    void *d_blocks, *d_coef, *d_pic;
    if (!(d_blocks = L.upload(BLOCKS, blocks, (size_t)n_blocks * sizeof(B200ItxBlock))) || !(d_coef = L.upload(COEF, coef, coef_bytes)) ||
        !(d_pic = L.upload(PIC, pic, pic_bytes)))
        return -1;
    if (int r = b200_itx_add_batch(bitdepth_max, tx, (const B200ItxBlock *)d_blocks, n_blocks, d_coef, d_pic, stride_px, zero_coefs, 0))
        return r;
    if (L.download(PIC, pic, pic_bytes) || (zero_coefs && L.download(COEF, coef, coef_bytes))) return -1;
    return L.sync();
}

// Level-1 single call, host pointers, arbitrary (possibly negative) byte stride.
int b200_inv_txfm_add(void *dst, ptrdiff_t dst_stride, void *coeff, int eob, int tx, int txtp,
                      int bitdepth_max)
{
    if (!itx_defined(tx, txtp)) { b200_set_error("b200_inv_txfm_add: undefined (tx=%d, txtp=%d)", tx, txtp); return -2; }
    if (eob < 0) { b200_set_error("b200_inv_txfm_add: eob < 0"); return -2; }
    Level1 L;
    const bool hbd = bitdepth_max > 255;
    int w, h;
    tx_size(tx, &w, &h);
    const int sw = w < 32 ? w : 32, sh = h < 32 ? h : 32;
    const size_t px = hbd ? 2 : 1, coef_bytes = (size_t)sw * sh * (hbd ? 4 : 2);
    B200ItxBlock b;
    b.dst_off = 0; b.coef_off = 0; b.eob = (int16_t)eob; b.txtp = (uint8_t)txtp; b.plane = 0;
    const int32_t st[3] = { w, w, w };
    void *d_blocks, *d_coef, *d_pic;
    if (!(d_blocks = L.upload(BLOCKS, &b, sizeof(b))) || !(d_coef = L.upload(COEF, coeff, coef_bytes)) ||
        !(d_pic = L.upload_rect(PIC, dst, dst_stride, w, h, px)))
        return -1;
    if (int r = b200_itx_add_batch(bitdepth_max, tx, (const B200ItxBlock *)d_blocks, 1, d_coef, d_pic, st, 1, 0)) return r;
    if (L.download(COEF, coeff, coef_bytes)) return -1;
    return L.download_rect(PIC, dst, dst_stride, w, h, px);
}

}  // extern "C"

// ---- Level-1 function tables: one thunk per (tx, txtp) slot, dav1d signatures -------------
namespace {
template <int TX, int TXTP>
void itx_thunk8(uint8_t *dst, ptrdiff_t stride, int16_t *coeff, int eob) {
    if (b200_inv_txfm_add(dst, stride, coeff, eob, TX, TXTP, 255)) die("itxfm_add (8 bpc)");
}
template <int TX, int TXTP>
void itx_thunk16(uint16_t *dst, ptrdiff_t stride, int32_t *coeff, int eob, int bitdepth_max) {
    if (b200_inv_txfm_add(dst, stride, coeff, eob, TX, TXTP, bitdepth_max)) die("itxfm_add (16 bpc)");
}
template <int TX, int... TP>
void fill_row(B200InvTxfmDSPContext8 *c8, B200InvTxfmDSPContext16 *c16, std::integer_sequence<int, TP...>) {
    if (c8)  { ((c8->itxfm_add[TX][TP]  = itx_defined(TX, TP) ? itx_thunk8<TX, TP>  : nullptr), ...); }
    if (c16) { ((c16->itxfm_add[TX][TP] = itx_defined(TX, TP) ? itx_thunk16<TX, TP> : nullptr), ...); }
}
template <int... TX>
void fill_all(B200InvTxfmDSPContext8 *c8, B200InvTxfmDSPContext16 *c16, std::integer_sequence<int, TX...>) {
    (fill_row<TX>(c8, c16, std::make_integer_sequence<int, B200_N_TX_TYPES_PLUS_LL>{}), ...);
}
}  // namespace

extern "C" {
void b200_itx_dsp_init_8bpc(B200InvTxfmDSPContext8 *c, int bpc) {
    (void)bpc;
    fill_all(c, nullptr, std::make_integer_sequence<int, B200_N_RECT_TX_SIZES>{});
}
void b200_itx_dsp_init_16bpc(B200InvTxfmDSPContext16 *c, int bpc) {
    (void)bpc;
    fill_all(nullptr, c, std::make_integer_sequence<int, B200_N_RECT_TX_SIZES>{});
}
}
