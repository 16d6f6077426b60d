// Host-side helpers shared by the C-ABI translation units: the bit-depth check and the launch of a kernel's
// high / low bit-depth instantiation (every entry point), and the staging of the host-pointer (Level-1) calls.
#pragma once
#include "common.cuh"
#include "launch_count.h"
#include "../../include/b200av1.h"
#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <tuple>
#include <type_traits>

namespace b200 {

// bitdepth_max arrives from outside the library: 255, 1023 or 4095, anything else is a bad argument (-2)
inline int check_bdmax(int bdmax, const char *who) {
    if (bdmax == 255 || bdmax == 1023 || bdmax == 4095) return 0;
    b200_set_error("%s: bad bitdepth_max %d", who, bdmax);
    return -2;
}

// Whether a kernel is launched with programmatic dependent launch is part of its contract: a kernel launched with
// Launch::pdl calls B200_PDL_ENTRY() first (common.cuh).
enum class Launch { plain, pdl };

// Launches the high (bdmax > 255) or low bit-depth instantiation of a kernel, counts the launch and checks its error.
// pick(std::bool_constant<HBD>) returns std::make_tuple(kernel<HBD>, args...), so that the pixel-typed casts of the
// arguments stay at the call site.
template <class Pick>
int launch_hbd(int bdmax, Launch mode, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Pick &&pick)
{
    auto go = [&](auto &&kernel_and_args) {
        std::apply([&](auto kern, auto... args) {
            if (mode == Launch::pdl) B200_LAUNCH_PDL(kern, grid, block, smem, stream, args...);
            else B200_LAUNCH(kern, grid, block, smem, stream, args...);
        }, kernel_and_args);
    };
    if (bdmax > 255) go(pick(std::true_type()));
    else go(pick(std::false_type()));
    b200_count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// row-range forms of the frame-wide sweeps (a band of a frame job, frame.cu; the b200_*_frame entry points pass the whole range)
int lf_frame_rows(int bdmax, const B200LfFrame *f, int ya4, int yb4, cudaStream_t stream);
int cdef_frame_rows(int bdmax, const B200CdefFrame *f, int t0, int t1, cudaStream_t stream);
int lr_frame_rows(int bdmax, const B200LrFrame *f, int r0, int r1, cudaStream_t stream);
// band-sliced intra (intra.cu): the n records at d_tx of the band starting at luma row y0 (the band at y0 = 0 initialises the
// done map, records on a later band's first row read the row above from `edge`); and the copy of the rows above luma row
// y1 into `edge` at the end of a band's reconstruction
int intra_band(int bdmax, const B200IntraFrame *f, const B200IntraTx *d_tx, int n, int y0, const void *edge, cudaStream_t stream);
int intra_edge_save(int bdmax, const B200IntraFrame *f, int y1, void *edge, cudaStream_t stream);
// all transform sizes of a frame (itx.cu, b200_itx_add_frame). coffs != nullptr: the compact form, `coefs` is the compact
// coefficient stream and coffs[tx][i] the offset of block i's coefficients in it (B200FrameJob.d_itx_coff)
int launch_itx_grouped(const void *const *blocks, const int32_t *n, void *coefs, void *pic, const int32_t *st,
                       int bdmax, int zero, cudaStream_t stream, const uint32_t *const *coffs = nullptr);

[[noreturn]] inline void die(const char *what) {
    fprintf(stderr, "b200av1: %s failed: %s\n", what, b200_last_error());
    abort();
}

// One Level-1 call: a dav1d DSP call made through host pointers and run as a one-record batch on stream 0. All such
// calls stage their data through one grow-only host buffer and one set of grow-only device scratch slots, so the
// object holds the lock that serialises them for its whole lifetime. The host buffer is pageable memory: an upload
// from it has been consumed when cudaMemcpyAsync returns, so one call may reuse it for several uploads.
class Level1 {
public:
    enum { kSlots = 5 };
    Level1() : lk_(state().mu) {}

    // device scratch slot `s`, grown to at least n bytes; nullptr (error set) when the allocation fails
    void *dev(int s, size_t n) {
        Slot &d = state().dev[s];
        if (n > d.cap || !d.p) {
            if (d.p) cudaFree(d.p);
            d.p = nullptr; d.cap = 0;
            const size_t want = n + (n >> 2) + 4096;
            if (!ok(cudaMalloc(&d.p, want), "scratch")) { d.p = nullptr; return nullptr; }
            d.cap = want;
        }
        return d.p;
    }
    // n bytes of host memory (a record, or an array) into slot s
    void *upload(int s, const void *src, size_t n) {
        void *d = dev(s, n);
        if (d && n && !ok(cudaMemcpyAsync(d, src, n, cudaMemcpyHostToDevice, 0), "upload")) return nullptr;
        return d;
    }
    // the w x h rectangle of `px`-byte pixels at pic (byte stride, possibly negative), densely into slot s
    void *upload_rect(int s, const void *pic, ptrdiff_t stride, int w, int h, size_t px) {
        uint8_t *buf = (uint8_t *)host((size_t)w * h * px);
        if (!buf) return nullptr;
        for (int y = 0; y < h; y++)
            memcpy(buf + (size_t)y * w * px, (const uint8_t *)pic + (ptrdiff_t)y * stride, (size_t)w * px);
        return upload(s, buf, (size_t)w * h * px);
    }
    // n bytes of slot s into host memory: complete once the next download_rect() or sync() has returned
    int download(int s, void *dst, size_t n) {
        return !n || ok(cudaMemcpyAsync(dst, state().dev[s].p, n, cudaMemcpyDeviceToHost, 0), "download") ? 0 : -1;
    }
    int sync() { return ok(cudaStreamSynchronize(0), "sync") ? 0 : -1; }
    // the dense w x h rectangle in slot s into the rectangle at pic, once everything enqueued so far has completed
    int download_rect(int s, void *pic, ptrdiff_t stride, int w, int h, size_t px) {
        uint8_t *buf = (uint8_t *)host((size_t)w * h * px);
        if (!buf || download(s, buf, (size_t)w * h * px) || sync()) return -1;
        for (int y = 0; y < h; y++)
            memcpy((uint8_t *)pic + (ptrdiff_t)y * stride, buf + (size_t)y * w * px, (size_t)w * px);
        return 0;
    }
    // the host staging buffer, at least n bytes, for a window a family assembles itself (the *_rect calls reuse it)
    void *host(size_t n) {
        State &st = state();
        if (n > st.host_cap) {
            free(st.host);
            st.host = malloc(n);
            st.host_cap = st.host ? n : 0;
            if (!st.host) { b200_set_error("level-1 staging (%zu bytes): out of memory", n); return nullptr; }
        }
        return st.host;
    }

private:
    struct Slot { void *p = nullptr; size_t cap = 0; };
    struct State { std::mutex mu; Slot dev[kSlots]; void *host = nullptr; size_t host_cap = 0; };
    static State &state() { static State s; return s; }
    static bool ok(cudaError_t e, const char *what) {
        if (e == cudaSuccess) return true;
        b200_set_error("level-1 %s: %s", what, cudaGetErrorString(e));
        return false;
    }
    std::lock_guard<std::mutex> lk_;
};

}  // namespace b200

#ifndef B200_EMU
#include <map>
// A side stream + fork/join events per (caller stream, slot): lets a stage that is latency bound on few CTAs run
// beside the next stage instead of in front of it. fork(): side waits for everything enqueued on `main` so far;
// join(): `main` waits for everything enqueued on the side stream.
struct SideStream {
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool fork(cudaStream_t main) {
        return cudaEventRecord(ev_fork, main) == cudaSuccess && cudaStreamWaitEvent(side, ev_fork, 0) == cudaSuccess;
    }
    bool join(cudaStream_t main) {
        return cudaEventRecord(ev_join, side) == cudaSuccess && cudaStreamWaitEvent(main, ev_join, 0) == cudaSuccess;
    }
};
inline SideStream *side_stream_for(cudaStream_t main, int slot)
{
    static std::map<std::pair<cudaStream_t, int>, SideStream> pool;
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    auto key = std::make_pair(main, slot);
    auto it = pool.find(key);
    if (it != pool.end()) return &it->second;
    SideStream s;
    if (cudaStreamCreateWithFlags(&s.side, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&s.ev_fork, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&s.ev_join, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    return &(pool[key] = s);
}
#endif
