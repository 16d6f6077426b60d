/*
 * integration/dav1d/b200_hooks.h — state shared by the dav1d `f->bd_fn` record emitters
 * (b200_hooks_tmpl.c, compiled at BITDEPTH 8 and 16) and the back-end loader (b200_hooks.c).
 *
 * This directory is the reference-side half of the drop-in (INTEGRATION.md): it is compiled against dav1d's
 * internal headers where they lie under $(REF) and linked with dav1d's own objects into ONE library whose
 * decode.c was compiled with the f->bd_fn targets renamed (-Ddav1d_recon_b_intra_8bpc=b200hook_recon_b_intra_8bpc
 * ..., reference src/decode.c:3418-3442) — no reference source is modified or copied.
 */
#ifndef B200_HOOKS_H
#define B200_HOOKS_H
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/b200av1.h"

/* libb200av1.so entry points, resolved once with dlopen/dlsym (b200hook_set_backend) */
typedef struct B200Backend {
    void *handle;
    const char *(*last_error)(void);
    void *(*dev_alloc)(size_t);
    void (*dev_free)(void *);
    void *(*host_alloc)(size_t);
    void (*host_free)(void *);
    void *(*stream_create)(void);
    void (*stream_destroy)(void *);
    size_t (*intra_scratch_bytes)(const B200IntraFrame *);
    int (*frame_run_host)(const B200FrameJob *, const B200Xfer *, int, const B200Xfer *, int, void *);
    int (*frame_submit_host)(const B200FrameJob *, const B200Xfer *, int, const B200Xfer *, int, void *);
    int (*frame_wait)(void *);
    int (*copy_async)(void *, const void *, size_t, void *);
    void *(*event_create)(void);
    void (*event_destroy)(void *);
    int (*event_record)(void *, void *);
    int (*stream_wait_event)(void *, void *);
    int (*struct_size)(int);
    int (*event_sync)(void *);
    int (*export_picture)(const B200ExportJob *, void *);
    int (*export_tensor_jitter_batch)(const B200TensorJob *, const B200ToneMap *const *, const B200ColorJitter *const *, int, void *);
} B200Backend;
const B200Backend *b200hook_backend(void);   /* NULL (after logging) when no back end is loaded: the decode fails */

/* a device buffer paired with its pinned host staging copy, grown on demand */
typedef struct HookBuf { void *host, *dev; size_t cap; } HookBuf;
int b200hook_buf_reserve(HookBuf *b, size_t bytes, int need_host, int keep);
void b200hook_buf_free(HookBuf *b);

/* Inter records are appended per TILE: a tile is reconstructed by one thread at a time, so its lists need no lock, and the
 * tile threads of a frame no longer serialise on the frame's mutex once per block (with 8 threads on a 16-tile 4K frame that
 * mutex made pass 2 effectively single threaded). Plain host memory, grown by doubling, kept across frames; the lists of all
 * tiles are concatenated into the pinned upload buffers when the frame completes (the order of the records inside a stage does
 * not matter: blocks do not overlap). */
enum { B200L_PRED, B200L_COMP, B200L_COMP2, B200L_WARP, B200L_BLEND, B200L_BLEND2, B200L_SCALED, B200L_ITX, B200L_COUNT = B200L_ITX + 19 };
typedef struct HookList { uint8_t *data; int n, cap; } HookList;
typedef struct HookTile { HookList l[B200L_COUNT]; } HookTile;

/* per frame context (dav1d's n_fc frames in flight): the records of the frame being reconstructed */
typedef struct HookFrame {
    const void *key;               /* the Dav1dFrameContext this slot serves */
    pthread_mutex_t lock;
    int cap_tx;                    /* capacity of tx.host in B200IntraTx records (n_tx below: slots are taken atomically) */
    size_t cap_coef;               /* capacity of coef.host in elements (n_coef below) */
    int tile_sbrows_done;          /* completed pass-2 tile superblock rows of the current frame */
    HookBuf tx, tx_sorted, coef, mask, level, lr_mask, pic[3], scratch;
    /* inter frames: prediction / compound / transform records (B200McBlock, B200CompBlock x 2 stages, B200ItxBlock
     * per transform size), the int16 scratch of the compound predictions (device only), the mask buffer (dav1d's
     * wedge tables at its head, difference-weighted masks behind them) and the initial done map of the intra kernel
     * (cells of inter blocks are "done" before it starts) */
    HookBuf pred, comp, comp2, itx[19], tmp16, cmask, done_init;
    HookBuf pal;                             /* palettes + packed index maps of palette blocks (slots taken atomically) */
    size_t cap_pal;
    HookBuf warp, blend, blend2, pxtmp;      /* warped-motion 8x8 blocks; OBMC: blend_h stage, blend_v stage, pixel scratch (device only) */
    HookBuf scaled;                          /* predictions from references of another size (B200McScaledBlock) */
    HookBuf sr[2];                           /* super-resolution: the upscaled deblocked / CDEF pictures loop restoration reads (device only) */
    int n_scaled;
    int n_pred, n_comp, n_comp2, n_itx[19], n_warp, n_blend, n_blend2;       /* totals over the tiles, known when the frame completes */
    HookTile *tiles;
    int n_tiles, cap_tiles;
    void *sort_scratch;            /* cell map + wave numbers of b200hook_wave_sort, kept across frames */
    size_t sort_scratch_cap;
    int started;
    int pinned;                    /* never recycled for another key (the output-stage slots) */
    unsigned epoch;                /* b200hook_release generation the `users` references belong to */
    int users;                     /* threads whose thread-local cache points at this slot (under the table lock): only a slot
                                      nobody caches may be handed to another key — the lock-free fast path of b200hook_frame
                                      is taken by exactly those threads */
    const void *cur_pic;           /* f->cur.data[0] of the frame being emitted: a different picture means the previous frame of this
                                      context was abandoned half way (flush / close) and its records are stale */
    uint64_t last_use;             /* slot recycling: least recently used idle slot is taken over (its buffers are kept) */
    void *stream;
    /* a submitted job that has not been waited for yet (the frame's exit handler does): its output picture and what the
     * statistics will be told once it is done */
    int pending;
    struct HookRefPic *pending_out;
    double t_submit, pend_prep_ms;
    uint64_t pend_rec, pend_coef, pend_h2d, pend_d2h, pend_kinds[11];
    /* statistics */
    uint64_t frames, records;
    /* What every tile thread of a frame WRITES while it emits blocks lives on cache lines of its own, away from what the
     * threads only read per block (key, started, cur_pic, buffer pointers, capacities): with 8 - 16 threads on one frame a
     * shared line that is written once per block costs more than the emission itself. */
    int n_tx __attribute__((aligned(64)));             /* B200IntraTx records emitted so far (tx.host) */
    size_t n_coef __attribute__((aligned(64)));        /* coefficients staged so far (coef.host), in elements */
    size_t n_pal;                  /* bytes taken in the palette buffer */
    size_t n_tmp16, n_cmask, n_pxtmp;                  /* scratch offsets handed out to compound / OBMC / mask records */
    int n_ii, n_ibc;
    int unsupported;               /* a block used a tool the emitters do not translate (written at most a few times) */
    int is_inter;
    unsigned refs_used;            /* bit k: some prediction of this frame reads reference k (f->refp[k]) */
    char pad_tail[64];
} HookFrame;
HookFrame *b200hook_frame(const void *key);
int b200hook_wave_sort(const B200IntraTx *in, B200IntraTx *out, int n, const int32_t w4[3], const int32_t h4[3],
                       int ss_hor, int ss_ver, void **scratch, size_t *scratch_cap);
void *b200hook_append(HookBuf *b, int *n, size_t elem);
int b200hook_tiles_reset(HookFrame *hf, int n_tiles);
int b200hook_tiles_gather(HookFrame *hf, int list, HookBuf *dst, size_t elem);      /* total number of records, < 0 on failure */
void *b200hook_tile_grow(HookList *L, size_t elem);
/* one record at the end of a tile's list (zeroed); inline: it is called once or more per block */
static inline void *b200hook_tile_append(HookFrame *const hf, const int tile, const int list, const size_t elem)
{
    if ((unsigned)tile >= (unsigned)hf->n_tiles) return NULL;
    HookList *const L = &hf->tiles[tile].l[list];
    if (L->n == L->cap && !b200hook_tile_grow(L, elem)) return NULL;
    void *const p = L->data + (size_t)L->n++ * elem;
    __builtin_memset(p, 0, elem);
    return p;
}

/* device pictures that outlive their frame context: every decoded picture, keyed by the host picture's data[0]
 * (dav1d recycles a host buffer only when no reference to it is left, so a key is reused only for a dead picture) */
/* submitted: the picture's job is enqueued on its frame context's stream and `event` marks the end of its kernels — later
 * frames order their own jobs behind it on the device (b200_stream_wait_event) without waiting on the host; ready: the job
 * and the copy into the host picture are complete */
/* exported: an export into caller memory was enqueued and `export_event` marks its end — the entry's device buffer is not
 * handed to another picture before that event has completed */
/* pool: the key is a page-locked picture of the hooks' pool (b200_hooks.c) that dav1d held when the entry was made: the
 * entry is freed by b200hook_refpic_forget when dav1d releases the picture and is never recycled before */
typedef struct HookRefPic { const void *key; void *dev; size_t bytes; int ready, submitted; void *event; uint64_t last_use;
                            void *export_event; int exported, pool; } HookRefPic;
HookRefPic *b200hook_refpic(const void *key, size_t bytes, int create);
/* enqueues the export of n resident pictures r[0..n) on `stream` behind their own jobs (one wait per distinct job), and
 * records each entry's export-done event behind it: `jobs` is one B200ExportJob (b200_export_picture, n = 1) or, with
 * `tensor` set, n B200TensorJobs, their tone maps `tones` and their colour jitters `jitters` (each NULL: none; one
 * b200_export_tensor_jitter_batch call) */
int b200hook_export_submit(HookRefPic *const *r, int n, int tensor, const void *jobs, const B200ToneMap *const *tones,
                           const B200ColorJitter *const *jitters, void *stream);
/* a decoder context (Dav1dContext *) opened for device output: its frame jobs and film grain leave the pictures in device
 * memory and copy nothing back into the host pictures */
int b200hook_device_only(const void *ctx);
void b200hook_refpic_set_ready(HookRefPic *r, int ready);
void b200hook_refpic_wait(HookRefPic *r);
void b200hook_refpic_set_submitted(HookRefPic *r, int submitted);
void b200hook_refpic_wait_submitted(HookRefPic *r);
int b200hook_async(void);                /* B200HOOK_ASYNC != 0 (default): jobs are waited for in the frame's exit handler */
int b200hook_frame_finish(HookFrame *h); /* waits for the slot's pending job, accounts it, marks its picture ready */
void b200hook_job_enter(void);
void b200hook_job_leave(void);

typedef struct B200HookStats {
    uint64_t frames, records, coefs, h2d_bytes, d2h_bytes; double device_ms;
    uint64_t intra_tx, pred, comp, warp, blend, itx, inter_frames;      /* records by kind */
    double host_prep_ms;            /* frame completion on the host before the job: mask fix-ups, wavefront sort, staging */
    uint64_t interintra;            /* inter-intra records (a subset of intra_tx) */
    uint64_t palette_bytes;         /* palettes + index maps shipped for palette blocks */
    uint64_t ibc;                   /* intra block copy records (a subset of intra_tx) */
    uint64_t scaled;                /* predictions from references of another size */
    uint64_t ref_table, frame_table; /* entries the device-picture / frame-context tables hold now (chunks of 64; not reset,
                                        the device-picture table returns to 0 in b200hook_release) */
} B200HookStats;
void b200hook_account(uint64_t records, uint64_t coefs, uint64_t h2d, uint64_t d2h, double ms, const uint64_t kinds[11], double prep_ms);

#endif
