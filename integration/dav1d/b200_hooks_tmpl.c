/*
 * integration/dav1d/b200_hooks_tmpl.c — the dav1d `f->bd_fn` hooks (reference src/internal.h:247-262, typedefs
 * src/recon.h:39-70) as B200 record emitters. Compiled at BITDEPTH 8 and 16 against dav1d's internal headers.
 *
 * dav1d runs in its two-pass (frame-threaded) mode: pass 1 entropy-decodes every block into
 * f->frame_thread.{b,cbi,cf}; pass 2 calls the hooks below, which translate each block into the records of
 * include/b200av1.h instead of reconstructing it on the CPU:
 *   recon_b_intra   -> one B200IntraTx per transform block (mode, angle, edge availability, CFL parameters,
 *                      transform type / eob) + its dequantised coefficients copied into a pinned staging buffer
 *                      (what dav1d_recon_b_intra does per tx block, reference src/recon_tmpl.c:1176-1555)
 *   backup_ipred_edge -> "tile superblock row complete" marker; when the last one of a frame arrives the frame's
 *                      records, dav1d's own Av1Filter / level / Av1Restoration arrays and the frame-header
 *                      parameters are shipped to HBM, b200_frame_run_host reconstructs and filters the whole frame,
 *                      and the finished picture is copied into f->cur (what the output / reference logic reads)
 *   filter_sbrow_*  -> nothing left to do on the CPU (the device job already ran the whole post-filter sweep)
 *   recon_b_inter   -> B200McBlock (put / prep) per prediction incl. the shared 4x4 chroma of sub-8x8 blocks,
 *                      B200CompBlock per compound combination (avg, distance weights, wedge and difference-weighted
 *                      masks), one B200ItxBlock per leaf of the transform tree (reference src/recon_tmpl.c:1557-1985)
 *                      B200WarpBlock per 8x8 of a warped block (local and global motion), OBMC as neighbour predictions
 *                      into a pixel scratch + two ordered blend stages
 *   apply_grain / prep_grain / apply_grain_row (output stage, renamed in lib.c / thread_task.c) -> one device film
 *                      grain job on the HBM-resident picture, result copied into the output picture
 *                      inter-intra: an II record per plane (intra predictor over the block, blended into the inter
 *                      prediction by the intra dataflow kernel) + the block's residual as RESID records
 *                      palette blocks: a PAL record per plane (palette + dav1d's packed index map) + RESID records
 * Not translated yet (the frame fails loudly, there is no CPU fallback): intra block copy, scaled references.
 */
#include "config.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "common/attributes.h"
#include "common/bitdepth.h"
#include "common/frame.h"
#include "common/intops.h"
#include "src/internal.h"
#include "src/ipred_prepare.h"
#include "src/recon.h"
#include "src/tables.h"
#include "src/wedge.h"
#include "b200_hooks.h"

static inline double bitfn(now_ms)(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

/* device picture geometry derived from the host picture: same strides, planes back to back */
typedef struct PicGeom { int stride[3]; uint32_t off[3]; int rows[3]; size_t bytes; } PicGeom;
/* Monochrome (4:0:0): the device picture keeps two dummy chroma planes in 4:2:0 geometry (the frame-wide sweeps walk three
 * planes; nothing is predicted or transformed into them, chroma deblocking is off, nothing of them is downloaded), so the
 * luma path is exactly the 4:2:0 one. */
static void bitfn(geom_of)(const Dav1dPicture *const p, PicGeom *const g)
{
    const int mono = p->p.layout == DAV1D_PIXEL_LAYOUT_I400;
    const int ss_ver = mono || p->p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int rows = (p->p.h + 127) & ~127;
    g->stride[0] = (int)PXSTRIDE(p->stride[0]);
    g->stride[1] = g->stride[2] = mono ? g->stride[0] : (int)PXSTRIDE(p->stride[1]);
    g->rows[0] = rows; g->rows[1] = g->rows[2] = rows >> ss_ver;
    g->off[0] = 0;
    g->off[1] = (uint32_t)g->stride[0] * rows;
    g->off[2] = g->off[1] + (uint32_t)g->stride[1] * g->rows[1];
    g->bytes = ((size_t)g->off[2] + (size_t)g->stride[2] * g->rows[2]) * sizeof(pixel);
}
/* the picture being reconstructed (coded size) ... */
static void bitfn(pic_geom)(const Dav1dFrameContext *const f, PicGeom *const g) { bitfn(geom_of)(&f->cur, g); }
/* ... and the one that is output and referenced: the same picture, or with super-resolution the upscaled one (f->sr_cur) */
#define OUT_KEY(f) ((const void *)(f)->sr_cur.p.data[0])

/* first pass-2 hook call of a frame: its output picture (keyed by the host buffer) is not valid any more / yet */
static void bitfn(frame_started)(HookFrame *const hf, const Dav1dFrameContext *const f)
{
    if (__atomic_load_n(&hf->started, __ATOMIC_ACQUIRE) && hf->cur_pic == OUT_KEY(f)) return;
    pthread_mutex_lock(&hf->lock);
    if (hf->started && hf->cur_pic != OUT_KEY(f)) {
        /* the context's previous frame never completed (dav1d flushed or closed while it was being reconstructed) */
        hf->tile_sbrows_done = 0; hf->n_tx = 0; hf->n_coef = 0; hf->unsupported = 0;
        hf->n_pred = hf->n_comp = hf->n_comp2 = hf->n_warp = hf->n_blend = hf->n_blend2 = 0;
        hf->n_tmp16 = 0; hf->n_pxtmp = 0; hf->is_inter = 0; hf->n_ii = 0; hf->n_ibc = 0; hf->refs_used = 0;
        memset(hf->n_itx, 0, sizeof(hf->n_itx));
        hf->started = 0;
    }
    if (!hf->started) {
        hf->cur_pic = OUT_KEY(f);
        if (b200hook_tiles_reset(hf, f->frame_hdr->tiling.cols * f->frame_hdr->tiling.rows)) __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED);
        hf->n_cmask = (sizeof(dav1d_masks) + 63) & ~(size_t)63;      /* dav1d's wedge tables sit at the head of the mask buffer */
        PicGeom g;
        bitfn(geom_of)(&f->sr_cur.p, &g);
        HookRefPic *const out = b200hook_refpic(OUT_KEY(f), g.bytes, 1);
        if (out) b200hook_refpic_set_ready(out, 0);
        else __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED);
        /* intra records and coefficients are appended without a lock by every tile thread of the frame (slots are taken
         * with atomic counters), so their buffers are sized for the worst case up front: one record per 4x4 cell of each
         * plane, 16 coefficients per cell, over the 128-aligned frame area */
        const int ss_ver = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
        const size_t aw4 = (f->bw + 31) & ~31, ah4 = (f->bh + 31) & ~31;
        const size_t cells = aw4 * ah4 + (f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I400 ? 2 * ((aw4 >> ss_hor) * (ah4 >> ss_ver)) : 0);
        /* + the block-level records that come on top of the per-transform-block ones: a palette or inter-intra block emits
         * one PAL / II record per plane before its RESID records, and such a block covers at least one 8x8 luma area (2x2
         * cells: 4 luma + the chroma cells) — a quarter of the cells bounds their number (+ slack for ragged frame edges) */
        hf->cap_tx = (int)(cells + cells / 4 + 64); hf->cap_coef = cells * 16;
        /* palette blocks: 8 bytes of packed indices per 4x4 cell + 8 palette entries per block (>= 1 cell) */
        hf->cap_pal = f->frame_hdr->allow_screen_content_tools ? cells * (8 + 8 * sizeof(pixel)) : 0;
        hf->n_pal = 0;
        if (b200hook_buf_reserve(&hf->tx, (size_t)hf->cap_tx * sizeof(B200IntraTx), 1, 0) ||
            b200hook_buf_reserve(&hf->coef, cells * 16 * sizeof(coef), 1, 0) ||
            (hf->cap_pal && b200hook_buf_reserve(&hf->pal, hf->cap_pal, 1, 0))) {
            __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED);
            hf->cap_tx = 0; hf->cap_coef = 0; hf->cap_pal = 0;      /* nothing can be emitted: the frame fails when it completes */
        }
        __atomic_store_n(&hf->started, 1, __ATOMIC_RELEASE);
    }
    pthread_mutex_unlock(&hf->lock);
}

/* the job copies these dav1d structures byte for byte into their B200 twins (include/b200av1.h): a dav1d version or
 * configuration with another layout must not compile */
_Static_assert(sizeof(Av1Filter) == sizeof(B200Av1Filter), "Av1Filter layout");
_Static_assert(offsetof(Av1Filter, filter_uv) == offsetof(B200Av1Filter, filter_uv) && offsetof(Av1Filter, cdef_idx) == offsetof(B200Av1Filter, cdef_idx) &&
               offsetof(Av1Filter, noskip_mask) == offsetof(B200Av1Filter, noskip_mask), "Av1Filter members");
_Static_assert(sizeof(Av1Restoration) == sizeof(B200Av1Restoration) && sizeof(Av1RestorationUnit) == sizeof(B200RestorationUnit), "Av1Restoration layout");
_Static_assert(offsetof(Av1RestorationUnit, filter_h) == offsetof(B200RestorationUnit, filter_h) && offsetof(Av1RestorationUnit, filter_v) == offsetof(B200RestorationUnit, filter_v) &&
               offsetof(Av1RestorationUnit, sgr_weights) == offsetof(B200RestorationUnit, sgr_weights), "Av1RestorationUnit members");
_Static_assert(sizeof(Dav1dFilmGrainData) == sizeof(B200FilmGrainData), "Dav1dFilmGrainData layout");
_Static_assert(offsetof(Dav1dFilmGrainData, ar_coeffs_y) == offsetof(B200FilmGrainData, ar_coeffs_y) && offsetof(Dav1dFilmGrainData, ar_coeff_shift) == offsetof(B200FilmGrainData, ar_coeff_shift) &&
               offsetof(Dav1dFilmGrainData, uv_mult) == offsetof(B200FilmGrainData, uv_mult) && offsetof(Dav1dFilmGrainData, clip_to_restricted_range) == offsetof(B200FilmGrainData, clip_to_restricted_range),
               "Dav1dFilmGrainData members");
_Static_assert(sizeof(((Av1FilterLUT *)0)->e) == sizeof(((B200FilterLUT *)0)->e) && sizeof(((Av1FilterLUT *)0)->i) == sizeof(((B200FilterLUT *)0)->i) &&
               sizeof(((Av1FilterLUT *)0)->sharp) == sizeof(((B200FilterLUT *)0)->sharp), "Av1FilterLUT members");

/* ---- one transform block -> one record ------------------------------------------------------------------ */
typedef struct TxCtx {
    HookFrame *hf;
    const Dav1dTaskContext *t;
    const Av1Block *b;
    PicGeom g;
    int ii;                 /* the block is an inter-intra block: its residual goes through the intra kernel */
} TxCtx;

/* copies the block's coefficients out of dav1d's pass-1 buffer (and clears them there, as the reference's
 * inverse transform would have: the buffer must be all zero for the next frame's pass 1) */
static int bitfn(stage_coefs)(HookFrame *const hf, coef *const cf, const int n, uint32_t *const off)
{
    const size_t at = __atomic_fetch_add(&hf->n_coef, (size_t)n, __ATOMIC_RELAXED);
    if (at + n > hf->cap_coef) return -1;
    memcpy((coef *)hf->coef.host + at, cf, n * sizeof(coef));
    memset(cf, 0, n * sizeof(coef));
    *off = (uint32_t)at;
    return 0;
}

static B200IntraTx *bitfn(new_record)(HookFrame *const hf)
{
    const int at = __atomic_fetch_add(&hf->n_tx, 1, __ATOMIC_RELAXED);
    if (at >= hf->cap_tx) return NULL;
    B200IntraTx *const r = (B200IntraTx *)hf->tx.host + at;
    memset(r, 0, sizeof(*r));
    return r;
}

/* the residual of the transform block the tile's cbi / cf cursors point at (pass 2: reference
 * src/recon_tmpl.c:1296-1302, 1508-1514); advances the cursors exactly like the reference */
static int bitfn(take_residual)(TxCtx *const c, B200IntraTx *const r, const TxfmInfo *const td, const int chroma)
{
    Dav1dTileState *const ts = c->t->ts;
    const int p = c->t->frame_thread.pass & 1;
    r->eob = -1;
    if (c->b->skip) return 0;
    const int cbi = *ts->frame_thread[p].cbi++;
    coef *const cf = ts->frame_thread[p].cf;
    const int n = chroma ? td->w * td->h * 16 : imin(td->w, 8) * imin(td->h, 8) * 16;
    ts->frame_thread[p].cf = cf + n;
    r->eob = (int16_t)(cbi >> 5);
    r->txtp = (uint8_t)(cbi & 0x1f);
    if (r->eob >= 0) return bitfn(stage_coefs)(c->hf, cf, n, &r->coef_off);
    return 0;
}

/* the transform size with the dimensions of a w4 x h4 block (4-sample units), -1 if dav1d has none */
static int bitfn(tx_of_dims)(const int w4, const int h4)
{
    for (int tx = 0; tx < N_RECT_TX_SIZES; tx++)
        if (dav1d_txfm_dimensions[tx].w == w4 && dav1d_txfm_dimensions[tx].h == h4) return tx;
    return -1;
}

/* palette block of one plane (reference :1201-1223 luma, :1400-1419 chroma): a PAL record over the whole block, the
 * palette and dav1d's packed index map copied into the frame's palette buffer */
static int bitfn(emit_palette)(TxCtx *const c, const int pl, const int pw4, const int ph4, const uint32_t dst_off,
                               const int x4, const int y4, const pixel *const pal, const uint8_t *const idx)
{
    HookFrame *const hf = c->hf;
    const int tx = bitfn(tx_of_dims)(pw4, ph4);
    const size_t idx_bytes = (size_t)pw4 * ph4 * 8, need = (8 * sizeof(pixel) + idx_bytes + 15) & ~(size_t)15;
    if (tx < 0) { __atomic_fetch_or(&hf->unsupported, 1, __ATOMIC_RELAXED); return 0; }
    const size_t at = __atomic_fetch_add(&hf->n_pal, need, __ATOMIC_RELAXED);
    B200IntraTx *const r = bitfn(new_record)(hf);
    if (!r || at + need > hf->cap_pal) return -1;
    memcpy((uint8_t *)hf->pal.host + at, pal, 8 * sizeof(pixel));
    memcpy((uint8_t *)hf->pal.host + at + 8 * sizeof(pixel), idx, idx_bytes);
    r->mode = B200_INTRA_MODE_PAL; r->plane = pl; r->tx = tx; r->dst_off = dst_off; r->eob = -1;
    r->x4 = x4; r->y4 = y4;
    r->xend4 = c->t->ts->tiling.col_end >> (pl && c->t->f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444);
    r->yend4 = c->t->ts->tiling.row_end >> (pl && c->t->f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420);
    r->luma_off = (uint32_t)at;
    r->cfl_alpha = !c->b->skip;               /* residual records follow */
    return 0;
}

void bitfn(b200hook_recon_b_intra)(Dav1dTaskContext *const t, const enum BlockSize bs,
                                   const enum EdgeFlags intra_edge_flags, const Av1Block *const b)
{
    const Dav1dFrameContext *const f = t->f;
    Dav1dTileState *const ts = t->ts;
    HookFrame *const hf = b200hook_frame(f);
    if (!hf) { atomic_fetch_or(&((Dav1dFrameContext *)f)->task_thread.error, 1); return; }
    if (t->frame_thread.pass != 2) {
        /* single-pass decoding interleaves entropy decoding with reconstruction inside this hook; the B200 back end
         * needs dav1d's two-pass mode (n_threads >= 2 with max_frame_delay >= 2, reference src/lib.c get_num_threads) */
        __atomic_fetch_or(&hf->unsupported, 4, __ATOMIC_RELAXED);
        return;
    }
    TxCtx c = { .hf = hf, .t = t, .b = b };
    bitfn(pic_geom)(f, &c.g);
    const int ss_ver = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int ss_hor = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int bx = t->bx, by = t->by, bx4 = bx & 31, by4 = by & 31;
    const uint8_t *const dim = dav1d_block_dimensions[bs];
    const int bw4 = dim[0], bh4 = dim[1];
    const int w4 = imin(bw4, f->bw - bx), h4 = imin(bh4, f->bh - by);
    const int cw4 = (w4 + ss_hor) >> ss_hor, ch4 = (h4 + ss_ver) >> ss_ver;
    const int cbw4 = (bw4 + ss_hor) >> ss_hor, cbh4 = (bh4 + ss_ver) >> ss_ver;
    const int has_chroma = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I400 && (bw4 > ss_hor || bx & 1) && (bh4 > ss_ver || by & 1);
    const TxfmInfo *const yt = &dav1d_txfm_dimensions[b->tx], *const ct = &dav1d_txfm_dimensions[b->uvtx];
    const int edge_filter_bit = f->seq_hdr->intra_edge_filter << 10;
    const int layout_shift = f->cur.p.layout - 1;      /* EDGE_I420_* >> (layout - 1) selects this layout's chroma flags */

    bitfn(frame_started)(hf, f);
    /* palette: the colours live in f->frame_thread.pal (one entry per 8x8 area, indexed like the reference does), the
     * packed index maps are consumed from the tile's pal_idx cursor exactly like the reference consumes them */
    const pixel (*const pal)[8] = !(b->pal_sz[0] | b->pal_sz[1]) ? NULL :
        f->frame_thread.pal[((by >> 1) + (bx & 1)) * (f->b4_stride >> 1) + ((bx >> 1) + (by & 1))];
    const int pass_idx = t->frame_thread.pass & 1;
    /* the reference walks a block in 64x64-luma chunks: luma transform blocks of the chunk, then its chroma */
    for (int iy = 0; iy < h4; iy += 16) {
        const int y_end = imin(h4, iy + 16), cy_end = imin(ch4, (iy + 16) >> ss_ver);
        for (int ix = 0; ix < w4; ix += 16) {
            const int x_end = imin(w4, ix + 16), cx_end = imin(cw4, (ix + 16) >> ss_hor);
            /* ---- luma ---- */
            if (b->pal_sz[0]) {
                const uint8_t *const idx = ts->frame_thread[pass_idx].pal_idx;
                ts->frame_thread[pass_idx].pal_idx += bw4 * bh4 * 8;
                if (bitfn(emit_palette)(&c, 0, bw4, bh4, c.g.off[0] + (uint32_t)(4 * by) * c.g.stride[0] + 4 * bx, bx, by, pal[0], idx))
                    { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
            }
            const int y_flags = sm_flag(t->a, bx4) | sm_flag(&t->l, by4) | edge_filter_bit;
            const int chunk_tr = ix + 16 < w4 ? 1 : iy ? 0 : !!(intra_edge_flags & EDGE_I444_TOP_HAS_RIGHT);
            const int chunk_bl = ix ? 0 : iy + 16 < h4 ? 1 : !!(intra_edge_flags & EDGE_I444_LEFT_HAS_BOTTOM);
            for (int y = iy; y < y_end; y += yt->h)
                for (int x = ix; x < x_end; x += yt->w) {
                    if (b->pal_sz[0] && b->skip) continue;      /* palette block without residual: the PAL record is final */
                    B200IntraTx *const r = bitfn(new_record)(hf);
                    if (!r) { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
                    const int px = bx + x, py = by + y;
                    r->plane = 0; r->tx = b->tx;
                    r->x4 = px; r->y4 = py; r->xend4 = ts->tiling.col_end; r->yend4 = ts->tiling.row_end;
                    r->dst_off = c.g.off[0] + (uint32_t)(4 * py) * c.g.stride[0] + 4 * px;
                    r->mode = b->y_mode; r->angle = b->y_angle;
                    r->angle_flags = y_flags;
                    if (b->pal_sz[0]) r->mode = B200_INTRA_MODE_RESID;      /* the palette record predicted the whole block */
                    r->max_w = 4 * f->bw - 4 * px; r->max_h = 4 * f->bh - 4 * py;
                    const int last_col = x + yt->w >= x_end, last_row = y + yt->h >= y_end;
                    r->flags = (px > ts->tiling.col_start ? B200_INTRA_HAVE_LEFT : 0) |
                               (py > ts->tiling.row_start ? B200_INTRA_HAVE_TOP : 0) |
                               (((y > iy || !chunk_tr) && last_col) ? 0 : B200_INTRA_TOP_HAS_RIGHT) |
                               ((x > ix || (!chunk_bl && last_row)) ? 0 : B200_INTRA_LEFT_HAS_BOTTOM);
                    if (b->pal_sz[0]) r->flags = 0;
                    if (bitfn(take_residual)(&c, r, yt, 0)) { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
                }
            if (!has_chroma) continue;
            /* ---- chroma ---- */
            const int is_cfl = b->uv_mode == CFL_PRED;
            const int uv_flags = sm_uv_flag(t->a, bx4 >> ss_hor) | sm_uv_flag(&t->l, by4 >> ss_ver) | edge_filter_bit;
            const int uv_tr = ((ix + 16) >> ss_hor) < cw4 ? 1 : iy ? 0 :
                              !!(intra_edge_flags & (EDGE_I420_TOP_HAS_RIGHT >> layout_shift));
            const int uv_bl = ix ? 0 : ((iy + 16) >> ss_ver) < ch4 ? 1 :
                              !!(intra_edge_flags & (EDGE_I420_LEFT_HAS_BOTTOM >> layout_shift));
            /* CFL: the ac block is derived from the whole co-located luma block, padded past the frame edge
             * (reference :1342-1362; a CFL block is a single chunk and a single chroma transform block) */
            int cfl_wpad = 0, cfl_hpad = 0;
            if (is_cfl) {
                const int far_r = ((cw4 << ss_hor) + yt->w - 1) & ~(yt->w - 1);
                const int far_b = ((ch4 << ss_ver) + yt->h - 1) & ~(yt->h - 1);
                cfl_wpad = cbw4 - (far_r >> ss_hor); cfl_hpad = cbh4 - (far_b >> ss_ver);
            }
            const int uv_pal = !is_cfl && b->pal_sz[1];
            if (uv_pal) {
                const uint8_t *const idx = ts->frame_thread[pass_idx].pal_idx;
                ts->frame_thread[pass_idx].pal_idx += cbw4 * cbh4 * 8;
                for (int pl = 1; pl <= 2; pl++)
                    if (bitfn(emit_palette)(&c, pl, cbw4, cbh4, c.g.off[pl] + (uint32_t)(4 * (by >> ss_ver)) * c.g.stride[pl] + 4 * (bx >> ss_hor),
                                            bx >> ss_hor, by >> ss_ver, pal[pl], idx))
                        { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
            }
            for (int pl = 1; pl <= 2; pl++)
                for (int y = iy >> ss_ver; y < cy_end; y += ct->h)
                    for (int x = ix >> ss_hor; x < cx_end; x += ct->w) {
                        if (uv_pal && b->skip) continue;
                        B200IntraTx *const r = bitfn(new_record)(hf);
                        if (!r) { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
                        /* luma-unit position the reference's t->bx / t->by would hold here */
                        const int lx = bx + (x << ss_hor), ly = by + (y << ss_ver);
                        const int px = lx >> ss_hor, py = ly >> ss_ver;
                        r->plane = pl; r->tx = b->uvtx;
                        r->x4 = px; r->y4 = py;
                        r->xend4 = ts->tiling.col_end >> ss_hor; r->yend4 = ts->tiling.row_end >> ss_ver;
                        r->dst_off = c.g.off[pl] + (uint32_t)(4 * py) * c.g.stride[pl] + 4 * px;
                        r->max_w = (4 * f->bw + ss_hor - 4 * (lx & ~ss_hor)) >> ss_hor;
                        r->max_h = (4 * f->bh + ss_ver - 4 * (ly & ~ss_ver)) >> ss_ver;
                        r->angle_flags = uv_flags;
                        const int last_col = x + ct->w >= cx_end, last_row = y + ct->h >= cy_end;
                        r->flags = (px > (ts->tiling.col_start >> ss_hor) ? B200_INTRA_HAVE_LEFT : 0) |
                                   (py > (ts->tiling.row_start >> ss_ver) ? B200_INTRA_HAVE_TOP : 0);
                        if (is_cfl) {
                            r->mode = B200_INTRA_MODE_CFL;
                            r->cfl_alpha = b->cfl_alpha[pl - 1];
                            r->cfl_w_pad = cfl_wpad; r->cfl_h_pad = cfl_hpad;
                            r->luma_off = c.g.off[0] + (uint32_t)(4 * (by & ~ss_ver)) * c.g.stride[0] + 4 * (bx & ~ss_hor);
                        } else {
                            r->mode = b->uv_mode; r->angle = b->uv_angle;
                        }
                        if (uv_pal) { r->mode = B200_INTRA_MODE_RESID; r->flags = 0; }
                        else if (!is_cfl || !r->cfl_alpha)      /* alpha == 0 is a plain DC_PRED with the usual edge rules */
                            r->flags |= (((y > (iy >> ss_ver) || !uv_tr) && last_col) ? 0 : B200_INTRA_TOP_HAS_RIGHT) |
                                        ((x > (ix >> ss_hor) || (!uv_bl && last_row)) ? 0 : B200_INTRA_LEFT_HAS_BOTTOM);
                        if (bitfn(take_residual)(&c, r, ct, 1)) { __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED); goto out; }
                    }
        }
    }
out:;
}

/* ---- inter blocks (what dav1d_recon_b_inter does, reference src/recon_tmpl.c:1557-1985) -------------------- */
/* the tile the calling thread is reconstructing (set on entry of the inter hook): its record lists are this thread's alone */
static __thread int bitfn(tl_tile);
#define TILE_REC(list, type) ((type *)b200hook_tile_append(hf, bitfn(tl_tile), (list), sizeof(type)))
/* one motion-compensated prediction: the arguments of the reference's mc() (:938-988), as a B200McBlock.
 * Source samples outside the reference plane are clamped by the kernel (= emu_edge). */
static int bitfn(emit_mc)(HookFrame *const hf, const Dav1dFrameContext *const f, const int op, const uint32_t dst_off,
                          const int bw4, const int bh4, const int bx, const int by, const int pl, const mv mv,
                          const int refidx, const enum Filter2d filter_2d)
{
    const Dav1dThreadPicture *const refp = &f->refp[refidx];
    const int ss_ver = !!pl && f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int ss_hor = !!pl && f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int h_mul = 4 >> ss_hor, v_mul = 4 >> ss_ver;
    if (refp->p.p.w != f->cur.p.w || refp->p.p.h != f->cur.p.h) {
        /* a reference of another size (the scaled branch of mc(), reference :991-1046): the block's position in the reference
         * in 1/1024 sample units and the per-sample steps of f->svc[refidx]; the kernel clamps its loads to the reference
         * plane (= the emu_edge window of the reference) */
        const int orig_pos_y = (by * v_mul << 4) + mv.y * (1 << !ss_ver), orig_pos_x = (bx * h_mul << 4) + mv.x * (1 << !ss_hor);
        const int64_t tx = (int64_t)orig_pos_x * f->svc[refidx][0].scale + (f->svc[refidx][0].scale - 0x4000) * 8;
        const int64_t ty = (int64_t)orig_pos_y * f->svc[refidx][1].scale + (f->svc[refidx][1].scale - 0x4000) * 8;
        const int pos_x = apply_sign64((int)((llabs(tx) + 128) >> 8), tx) + 32, pos_y = apply_sign64((int)((llabs(ty) + 128) >> 8), ty) + 32;
        B200McScaledBlock *const r = TILE_REC(B200L_SCALED, B200McScaledBlock);
        if (!r) return -1;
        r->dst_off = dst_off;
        r->src_x = pos_x >> 10; r->src_y = pos_y >> 10;
        r->mx = pos_x & 0x3ff; r->my = pos_y & 0x3ff;
        r->dx = f->svc[refidx][0].step; r->dy = f->svc[refidx][1].step;
        r->w = bw4 * h_mul; r->h = bh4 * v_mul;
        r->filter2d = filter_2d; r->op = op; r->plane = pl; r->ref = refidx;
        if (!(__atomic_load_n(&hf->refs_used, __ATOMIC_RELAXED) & (1u << refidx))) __atomic_fetch_or(&hf->refs_used, 1u << refidx, __ATOMIC_RELAXED);      /* written once per reference, not once per block: the line is shared by every tile thread */
        return 0;
    }
    const int mx = mv.x & (15 >> !ss_hor), my = mv.y & (15 >> !ss_ver);
    B200McBlock *const r = TILE_REC(B200L_PRED, B200McBlock);
    if (!r) return -1;
    r->dst_off = dst_off;
    r->src_x = bx * h_mul + (mv.x >> (3 + ss_hor));
    r->src_y = by * v_mul + (mv.y >> (3 + ss_ver));
    r->w = bw4 * h_mul; r->h = bh4 * v_mul;
    r->mx = mx << !ss_hor; r->my = my << !ss_ver;
    r->filter2d = filter_2d; r->op = op; r->plane = pl; r->ref = refidx;      /* op: 0 put, 1 prep, 2 put into the pixel scratch */
    if (!(__atomic_load_n(&hf->refs_used, __ATOMIC_RELAXED) & (1u << refidx))) __atomic_fetch_or(&hf->refs_used, 1u << refidx, __ATOMIC_RELAXED);      /* written once per reference, not once per block: the line is shared by every tile thread */
    return 0;
}

/* warped motion: one B200WarpBlock per 8x8 of the block (warp_affine, :1115-1174); op 0 -> pixels at dst_off,
 * op 1 -> int16 prediction at dst_off in tmp (pitch tmp_stride) */
static int bitfn(emit_warp)(HookFrame *const hf, const Dav1dFrameContext *const f, const Dav1dTaskContext *const t, const int op,
                            const uint32_t dst_off, const int pitch, const uint8_t *const b_dim, const int pl, const int refidx,
                            const Dav1dWarpedMotionParams *const wmp)
{
    const Dav1dThreadPicture *const refp = &f->refp[refidx];
    if (refp->p.p.w != f->cur.p.w || refp->p.p.h != f->cur.p.h) { __atomic_fetch_or(&hf->unsupported, 32, __ATOMIC_RELAXED); return 0; }
    const int ss_ver = !!pl && f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int ss_hor = !!pl && f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int h_mul = 4 >> ss_hor, v_mul = 4 >> ss_ver;
    const int32_t *const mat = wmp->matrix;
    for (int y = 0; y < b_dim[1] * v_mul; y += 8) {
        const int src_y = t->by * 4 + ((y + 4) << ss_ver);
        const int64_t mat3_y = (int64_t)mat[3] * src_y + mat[0], mat5_y = (int64_t)mat[5] * src_y + mat[1];
        for (int x = 0; x < b_dim[0] * h_mul; x += 8) {
            const int src_x = t->bx * 4 + ((x + 4) << ss_hor);
            const int64_t mvx = ((int64_t)mat[2] * src_x + mat3_y) >> ss_hor, mvy = ((int64_t)mat[4] * src_x + mat5_y) >> ss_ver;
            B200WarpBlock *const r = TILE_REC(B200L_WARP, B200WarpBlock);
            if (!r) return -1;
            r->dst_off = dst_off + (uint32_t)y * pitch + x;
            r->src_x = (int)(mvx >> 16) - 4; r->src_y = (int)(mvy >> 16) - 4;
            r->mx = (((int)mvx & 0xffff) - wmp->u.p.alpha * 4 - wmp->u.p.beta * 7) & ~0x3f;
            r->my = (((int)mvy & 0xffff) - wmp->u.p.gamma * 4 - wmp->u.p.delta * 4) & ~0x3f;
            for (int k = 0; k < 4; k++) r->abcd[k] = wmp->u.abcd[k];
            r->tmp_stride = pitch; r->op = op; r->plane = pl; r->ref = refidx;
            if (!(__atomic_load_n(&hf->refs_used, __ATOMIC_RELAXED) & (1u << refidx))) __atomic_fetch_or(&hf->refs_used, 1u << refidx, __ATOMIC_RELAXED);      /* written once per reference, not once per block: the line is shared by every tile thread */
        }
    }
    return 0;
}

/* overlapped block motion compensation (obmc, :1052-1113): the block's top rows are blended with predictions made with
 * the motion of the blocks above (blend_h, first blend stage), then its left columns with those of the blocks to the left
 * (blend_v, second stage: the two overlap in the top-left corner and the order matters) */
static int bitfn(emit_obmc)(HookFrame *const hf, const Dav1dFrameContext *const f, const Dav1dTaskContext *const t,
                            const uint32_t dst_off, const int dst_stride, const uint8_t *const b_dim, const int pl,
                            const int bx4, const int by4, const int w4, const int h4)
{
    refmvs_block *const *const r = &t->rt.r[(t->by & 31) + 5];
    const int ss_ver = !!pl && f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int ss_hor = !!pl && f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int h_mul = 4 >> ss_hor, v_mul = 4 >> ss_ver;
    if (t->by > t->ts->tiling.row_start && (!pl || b_dim[0] * h_mul + b_dim[1] * v_mul >= 16))
        for (int i = 0, x = 0; x < w4 && i < imin(b_dim[2], 4); ) {
            const refmvs_block *const a_r = &r[-1][t->bx + x + 1];          /* odd column: the block covering it */
            const int step4 = iclip(dav1d_block_dimensions[a_r->bs][0], 2, 16);
            if (a_r->ref.ref[0] > 0) {
                const int ow4 = imin(step4, b_dim[0]), oh4 = imin(b_dim[1], 16) >> 1;
                const uint32_t scratch = (uint32_t)__atomic_fetch_add(&hf->n_pxtmp, (size_t)(ow4 * h_mul) * (((oh4 * 3 + 3) >> 2) * v_mul), __ATOMIC_RELAXED);
                if (bitfn(emit_mc)(hf, f, 2, scratch, ow4, (oh4 * 3 + 3) >> 2, t->bx + x, t->by, pl, a_r->mv.mv[0], a_r->ref.ref[0] - 1,
                                   dav1d_filter_2d[t->a->filter[1][bx4 + x + 1]][t->a->filter[0][bx4 + x + 1]])) return -1;
                B200BlendBlock *const bl = TILE_REC(B200L_BLEND, B200BlendBlock);
                if (!bl) return -1;
                bl->dst_off = dst_off + x * h_mul; bl->tmp_off = scratch;
                bl->w = h_mul * ow4; bl->h = v_mul * oh4; bl->op = B200_BLEND_H; bl->plane = pl;
                i++;
            }
            x += step4;
        }
    if (t->bx > t->ts->tiling.col_start)
        for (int i = 0, y = 0; y < h4 && i < imin(b_dim[3], 4); ) {
            const refmvs_block *const l_r = &r[y + 1][t->bx - 1];
            const int step4 = iclip(dav1d_block_dimensions[l_r->bs][1], 2, 16);
            if (l_r->ref.ref[0] > 0) {
                const int ow4 = imin(b_dim[0], 16) >> 1, oh4 = imin(step4, b_dim[1]);
                const uint32_t scratch = (uint32_t)__atomic_fetch_add(&hf->n_pxtmp, (size_t)(ow4 * h_mul) * (oh4 * v_mul), __ATOMIC_RELAXED);
                if (bitfn(emit_mc)(hf, f, 2, scratch, ow4, oh4, t->bx, t->by + y, pl, l_r->mv.mv[0], l_r->ref.ref[0] - 1,
                                   dav1d_filter_2d[t->l.filter[1][by4 + y + 1]][t->l.filter[0][by4 + y + 1]])) return -1;
                B200BlendBlock *const bl = TILE_REC(B200L_BLEND2, B200BlendBlock);
                if (!bl) return -1;
                bl->dst_off = dst_off + (uint32_t)(y * v_mul) * dst_stride; bl->tmp_off = scratch;
                bl->w = h_mul * ow4; bl->h = v_mul * oh4; bl->op = B200_BLEND_V; bl->plane = pl;
                i++;
            }
            y += step4;
        }
    return 0;
}

/* inter-intra (reference :1601-1626 luma, :1737-1777 chroma): one II record per plane of the block; the predictor runs
 * over the whole block, whose size is also a transform size (8x8 .. 32x32 luma, halved for sub-sampled chroma) */
static int bitfn(emit_interintra)(TxCtx *const c, const enum BlockSize bs, const int pl, const uint32_t dst_off,
                                  const int bx, const int by, const uint8_t *const mask)
{
    HookFrame *const hf = c->hf;
    const Dav1dFrameContext *const f = c->t->f;
    const Dav1dTileState *const ts = c->t->ts;
    const int ss_ver = pl && f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = pl && f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const uint8_t *const dim = dav1d_block_dimensions[bs];
    const int pw4 = (dim[0] + ss_hor) >> ss_hor, ph4 = (dim[1] + ss_ver) >> ss_ver;
    const int tx = bitfn(tx_of_dims)(pw4, ph4);
    if (tx < 0) { __atomic_fetch_or(&hf->unsupported, 256, __ATOMIC_RELAXED); return 0; }
    B200IntraTx *const r = bitfn(new_record)(hf);
    if (!r) return -1;
    const int px = bx >> ss_hor, py = by >> ss_ver;
    r->mode = B200_INTRA_MODE_II; r->plane = pl; r->tx = tx; r->dst_off = dst_off; r->eob = -1;
    r->angle = c->b->interintra_mode == II_SMOOTH_PRED ? SMOOTH_PRED : c->b->interintra_mode;     /* DC / VERT / HOR / SMOOTH */
    r->x4 = px; r->y4 = py; r->xend4 = ts->tiling.col_end >> ss_hor; r->yend4 = ts->tiling.row_end >> ss_ver;
    r->flags = (px > (ts->tiling.col_start >> ss_hor) ? B200_INTRA_HAVE_LEFT : 0) | (py > (ts->tiling.row_start >> ss_ver) ? B200_INTRA_HAVE_TOP : 0);
    r->luma_off = (uint32_t)(mask - (const uint8_t *)&dav1d_masks);
    r->cfl_alpha = !c->b->skip;               /* residual records follow */
    __atomic_fetch_add(&hf->n_ii, 1, __ATOMIC_RELAXED);
    return 0;
}

/* intra block copy (reference :1583-1596; the vector was clipped to the decoded part of the tile in src/decode.c:1286-1345):
 * mc() with the current picture as reference and the bilinear filter, bw4 x bh4 luma units at (bx, by), written as IBC records
 * of the intra machine (one per <= 64x64 piece whose shape is a transform size); the residual follows as RESID records */
static int bitfn(emit_ibc)(TxCtx *const c, const int pl, const uint32_t dst_off, const int bw4, const int bh4,
                           const int bx, const int by, const mv mv)
{
    HookFrame *const hf = c->hf;
    const Dav1dFrameContext *const f = c->t->f;
    const Dav1dTileState *const ts = c->t->ts;
    const int ss_ver = pl && f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = pl && f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int h_mul = 4 >> ss_hor, v_mul = 4 >> ss_ver;
    const int w = bw4 * h_mul, h = bh4 * v_mul;
    const int dx = bx * h_mul + (mv.x >> (3 + ss_hor)), dy = by * v_mul + (mv.y >> (3 + ss_ver));
    const int mx = (mv.x & (15 >> !ss_hor)) << !ss_hor, my = (mv.y & (15 >> !ss_ver)) << !ss_ver;
    if (dx < 0 || dy < 0 || dx + w > 65535 || dy + h > 65535) { __atomic_fetch_or(&hf->unsupported, 64, __ATOMIC_RELAXED); return 0; }
    int cw = imin(w, 64), ch = imin(h, 64);
    while (cw > 4 * ch) cw >>= 1;           /* e.g. the 8x64 chroma block of a 4:2:2 16x64 block: no such transform shape */
    while (ch > 4 * cw) ch >>= 1;
    const int tx = bitfn(tx_of_dims)(cw >> 2, ch >> 2);
    if (tx < 0) { __atomic_fetch_or(&hf->unsupported, 64, __ATOMIC_RELAXED); return 0; }
    const int px4 = (bx * h_mul) >> 2, py4 = (by * v_mul) >> 2;
    for (int yy = 0; yy < h; yy += ch)
        for (int xx = 0; xx < w; xx += cw) {
            B200IntraTx *const r = bitfn(new_record)(hf);
            if (!r) return -1;
            r->mode = B200_INTRA_MODE_IBC; r->plane = pl; r->tx = tx; r->eob = -1; r->flags = 0;
            r->dst_off = dst_off + (uint32_t)yy * c->g.stride[pl] + xx;
            r->x4 = px4 + (xx >> 2); r->y4 = py4 + (yy >> 2);
            r->xend4 = ts->tiling.col_end >> ss_hor; r->yend4 = ts->tiling.row_end >> ss_ver;
            r->luma_off = ((uint32_t)(dy + yy) << 16) | (uint32_t)(dx + xx);
            r->cfl_w_pad = mx; r->cfl_h_pad = my;
            r->cfl_alpha = !c->b->skip;           /* residual records follow */
            __atomic_fetch_add(&hf->n_ibc, 1, __ATOMIC_RELAXED);
        }
    return 0;
}

static int bitfn(emit_itx)(TxCtx *const c, const int tx, const int pl, const uint32_t dst_off, const int chroma)
{
    HookFrame *const hf = c->hf;
    if (c->ii) {
        /* inter-intra block: the residual is added by the intra dataflow kernel after the block's blend (a RESID record
         * per transform block, also when it has no coefficients: it turns the cells from "predicted" into "final") */
        B200IntraTx *const r = bitfn(new_record)(hf);
        if (!r || bitfn(take_residual)(c, r, &dav1d_txfm_dimensions[tx], chroma)) return -1;
        const int ss_ver = pl && c->t->f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = pl && c->t->f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
        const uint32_t rel = dst_off - c->g.off[pl];
        r->mode = B200_INTRA_MODE_RESID; r->plane = pl; r->tx = tx; r->dst_off = dst_off;
        r->y4 = (rel / c->g.stride[pl]) >> 2; r->x4 = (rel % c->g.stride[pl]) >> 2;
        r->xend4 = c->t->ts->tiling.col_end >> ss_hor; r->yend4 = c->t->ts->tiling.row_end >> ss_ver;
        return 0;
    }
    B200IntraTx tmp;          /* take_residual fills eob / txtp / coef_off of any record with these fields */
    memset(&tmp, 0, sizeof(tmp));
    if (bitfn(take_residual)(c, &tmp, &dav1d_txfm_dimensions[tx], chroma)) return -1;
    if (tmp.eob < 0) return 0;
    B200ItxBlock *const r = TILE_REC(B200L_ITX + tx, B200ItxBlock);
    if (!r) return -1;
    r->dst_off = dst_off; r->coef_off = tmp.coef_off; r->eob = tmp.eob; r->txtp = tmp.txtp; r->plane = pl;
    return 0;
}

/* the luma transform tree of an inter block (read_coef_tree, :731-822): (x4, y4) = position of this node */
static int bitfn(emit_tx_tree)(TxCtx *const c, const enum RectTxfmSize tx, const int depth, const uint16_t *const split,
                               const int x_off, const int y_off, const int x4, const int y4)
{
    const Dav1dFrameContext *const f = c->t->f;
    const TxfmInfo *const td = &dav1d_txfm_dimensions[tx];
    if (depth < 2 && split[depth] && (split[depth] & (1 << (y_off * 4 + x_off)))) {
        const enum RectTxfmSize sub = td->sub;
        const TxfmInfo *const sd = &dav1d_txfm_dimensions[sub];
        const int two_cols = td->w >= td->h && x4 + sd->w < f->bw, two_rows = td->h >= td->w && y4 + sd->h < f->bh;
        if (bitfn(emit_tx_tree)(c, sub, depth + 1, split, x_off * 2, y_off * 2, x4, y4)) return -1;
        if (two_cols && bitfn(emit_tx_tree)(c, sub, depth + 1, split, x_off * 2 + 1, y_off * 2, x4 + sd->w, y4)) return -1;
        if (two_rows) {
            if (bitfn(emit_tx_tree)(c, sub, depth + 1, split, x_off * 2, y_off * 2 + 1, x4, y4 + sd->h)) return -1;
            if (two_cols && bitfn(emit_tx_tree)(c, sub, depth + 1, split, x_off * 2 + 1, y_off * 2 + 1, x4 + sd->w, y4 + sd->h)) return -1;
        }
        return 0;
    }
    return bitfn(emit_itx)(c, tx, 0, c->g.off[0] + (uint32_t)(4 * y4) * c->g.stride[0] + 4 * x4, 0);
}

int bitfn(b200hook_recon_b_inter)(Dav1dTaskContext *const t, const enum BlockSize bs, const Av1Block *const b)
{
    const Dav1dFrameContext *const f = t->f;
    HookFrame *const hf = b200hook_frame(f);
    if (!hf) { atomic_fetch_or(&((Dav1dFrameContext *)f)->task_thread.error, 1); return -1; }
    if (t->frame_thread.pass != 2) {
        __atomic_fetch_or(&hf->unsupported, 4, __ATOMIC_RELAXED);
        return -1;
    }
    TxCtx c = { .hf = hf, .t = t, .b = b };
    bitfn(pic_geom)(f, &c.g);
    const PicGeom *const g = &c.g;
    const int ss_ver = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420;
    const int ss_hor = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int bx = t->bx, by = t->by, bx4 = bx & 31, by4 = by & 31;
    const uint8_t *const dim = dav1d_block_dimensions[bs];
    const int bw4 = dim[0], bh4 = dim[1];
    const int w4 = imin(bw4, f->bw - bx), h4 = imin(bh4, f->bh - by);
    const int cw4 = (w4 + ss_hor) >> ss_hor, ch4 = (h4 + ss_ver) >> ss_ver;
    const int cbw4 = (bw4 + ss_hor) >> ss_hor, cbh4 = (bh4 + ss_ver) >> ss_ver;
    const int has_chroma = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I400 && (bw4 > ss_hor || bx & 1) && (bh4 > ss_ver || by & 1);
    const int chr_layout_idx = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I400 ? 0 : DAV1D_PIXEL_LAYOUT_I444 - f->cur.p.layout;
    const uint32_t ydst = g->off[0] + (uint32_t)(4 * by) * g->stride[0] + 4 * bx;
    const uint32_t uvrel = (uint32_t)(4 * (by >> ss_ver)) * g->stride[1] + 4 * (bx >> ss_hor);   /* + g->off[pl] */
    int rc = -1;

    bitfn(frame_started)(hf, f);
    bitfn(tl_tile) = (int)(t->ts - f->ts);  /* no lock: inter records go to this tile's lists, intra records / coefficients / scratch offsets are taken atomically */
    if (IS_KEY_OR_INTRA(f->frame_hdr)) {
        /* intra block copy: prediction and residual both go through the intra machine (the source is this very picture) */
        c.ii = 1;
        if (bitfn(emit_ibc)(&c, 0, ydst, bw4, bh4, bx, by, b->mv[0])) goto out;
        if (has_chroma)
            for (int pl = 1; pl <= 2; pl++)
                if (bitfn(emit_ibc)(&c, pl, g->off[pl] + uvrel, bw4 << (bw4 == ss_hor), bh4 << (bh4 == ss_ver), bx & ~ss_hor, by & ~ss_ver, b->mv[0])) goto out;
        goto residual;
    }
    if (!__atomic_load_n(&hf->is_inter, __ATOMIC_RELAXED)) __atomic_store_n(&hf->is_inter, 1, __ATOMIC_RELAXED);
    if (b->comp_type == COMP_INTER_NONE) {
        const enum Filter2d filter_2d = b->filter2d;
        const int warp = (b->inter_mode == GLOBALMV && f->gmv_warp_allowed[b->ref[0]]) ||
                         (b->motion_mode == MM_WARP && t->warpmv.type > DAV1D_WM_TYPE_TRANSLATION);
        const Dav1dWarpedMotionParams *const wmp = b->motion_mode == MM_WARP ? &t->warpmv : &f->frame_hdr->gmv[b->ref[0]];
        c.ii = !!b->interintra_type;
        if (warp && imin(bw4, bh4) > 1) {
            if (bitfn(emit_warp)(hf, f, t, 0, ydst, g->stride[0], dim, 0, b->ref[0], wmp)) goto out;
        } else {
            if (bitfn(emit_mc)(hf, f, 0, ydst, bw4, bh4, bx, by, 0, b->mv[0], b->ref[0], filter_2d)) goto out;
            if (b->motion_mode == MM_OBMC && bitfn(emit_obmc)(hf, f, t, ydst, g->stride[0], dim, 0, bx4, by4, w4, h4)) goto out;
        }
        if (c.ii && bitfn(emit_interintra)(&c, bs, 0, ydst, bx, by, II_MASK(0, bs, b))) goto out;
        if (has_chroma) {
            /* a 4-wide / 4-tall luma block shares its 4x4 chroma block with its left / top neighbours: each quarter is
             * predicted with the motion of the luma block above it, if all of them are inter (:1652-1724) */
            int sub8 = bw4 == ss_hor || bh4 == ss_ver;
            refmvs_block *const *rr = NULL;
            if (sub8) {
                rr = &t->rt.r[(by & 31) + 5];
                if (bw4 == 1) sub8 &= rr[0][bx - 1].ref.ref[0] > 0;
                if (bh4 == ss_ver) sub8 &= rr[-1][bx].ref.ref[0] > 0;
                if (bw4 == 1 && bh4 == ss_ver) sub8 &= rr[-1][bx - 1].ref.ref[0] > 0;
            }
            if (sub8) {
                uint32_t h_off = 0, v_off = 0;
                if (bw4 == 1 && bh4 == ss_ver) {
                    const refmvs_block *const n = &rr[-1][bx - 1];
                    for (int pl = 1; pl <= 2; pl++)
                        if (bitfn(emit_mc)(hf, f, 0, g->off[pl] + uvrel, bw4, bh4, bx - 1, by - 1, pl, n->mv.mv[0], n->ref.ref[0] - 1,
                                           f->frame_thread.b[(by - 1) * f->b4_stride + bx - 1].filter2d)) goto out;
                    v_off = 2 * g->stride[1]; h_off = 2;
                }
                if (bw4 == 1) {
                    const refmvs_block *const n = &rr[0][bx - 1];
                    for (int pl = 1; pl <= 2; pl++)
                        if (bitfn(emit_mc)(hf, f, 0, g->off[pl] + uvrel + v_off, bw4, bh4, bx - 1, by, pl, n->mv.mv[0], n->ref.ref[0] - 1,
                                           f->frame_thread.b[by * f->b4_stride + bx - 1].filter2d)) goto out;
                    h_off = 2;
                }
                if (bh4 == ss_ver) {
                    const refmvs_block *const n = &rr[-1][bx];
                    for (int pl = 1; pl <= 2; pl++)
                        if (bitfn(emit_mc)(hf, f, 0, g->off[pl] + uvrel + h_off, bw4, bh4, bx, by - 1, pl, n->mv.mv[0], n->ref.ref[0] - 1,
                                           f->frame_thread.b[(by - 1) * f->b4_stride + bx].filter2d)) goto out;
                    v_off = 2 * g->stride[1];
                }
                for (int pl = 1; pl <= 2; pl++)
                    if (bitfn(emit_mc)(hf, f, 0, g->off[pl] + uvrel + h_off + v_off, bw4, bh4, bx, by, pl, b->mv[0], b->ref[0], filter_2d)) goto out;
            } else if (warp && imin(cbw4, cbh4) > 1) {
                for (int pl = 1; pl <= 2; pl++)
                    if (bitfn(emit_warp)(hf, f, t, 0, g->off[pl] + uvrel, g->stride[1], dim, pl, b->ref[0], wmp)) goto out;
            } else {
                for (int pl = 1; pl <= 2; pl++) {
                    if (bitfn(emit_mc)(hf, f, 0, g->off[pl] + uvrel, bw4 << (bw4 == ss_hor), bh4 << (bh4 == ss_ver),
                                       bx & ~ss_hor, by & ~ss_ver, pl, b->mv[0], b->ref[0], filter_2d)) goto out;
                    if (b->motion_mode == MM_OBMC && bitfn(emit_obmc)(hf, f, t, g->off[pl] + uvrel, g->stride[1], dim, pl, bx4, by4, w4, h4)) goto out;
                }
            }
            if (c.ii && !sub8)
                for (int pl = 1; pl <= 2; pl++)
                    if (bitfn(emit_interintra)(&c, bs, pl, g->off[pl] + uvrel, bx, by, II_MASK(chr_layout_idx, bs, b))) goto out;
        }
    } else {
        /* compound: two int16 predictions per plane, then avg / w_avg / mask / w_mask (:1782-1866) */
        const enum Filter2d filter_2d = b->filter2d;
        uint32_t mask_off = 0;          /* luma mask, then the mask the chroma planes read */
        for (int pl = 0; pl < (has_chroma ? 3 : 1); pl++) {
            const int pw = pl ? bw4 * 4 >> ss_hor : bw4 * 4, ph = pl ? bh4 * 4 >> ss_ver : bh4 * 4;
            uint32_t tmp_off[2];
            for (int i = 0; i < 2; i++) {
                tmp_off[i] = (uint32_t)__atomic_fetch_add(&hf->n_tmp16, (size_t)pw * ph, __ATOMIC_RELAXED);
                if (b->inter_mode == GLOBALMV_GLOBALMV && f->gmv_warp_allowed[b->ref[i]] && (!pl || imin(cbw4, cbh4) > 1)) {
                    if (bitfn(emit_warp)(hf, f, t, 1, tmp_off[i], pw, dim, pl, b->ref[i], &f->frame_hdr->gmv[b->ref[i]])) goto out;
                } else if (bitfn(emit_mc)(hf, f, 1, tmp_off[i], bw4, bh4, bx, by, pl, b->mv[i], b->ref[i], filter_2d)) goto out;
            }
            const int seg = b->comp_type == COMP_INTER_SEG;
            /* chroma of a difference-weighted block reads the mask its luma block writes: second compound stage */
            B200CompBlock *const r = (pl && seg) ? TILE_REC(B200L_COMP2, B200CompBlock) : TILE_REC(B200L_COMP, B200CompBlock);
            if (!r) goto out;
            r->dst_off = pl ? g->off[pl] + uvrel : ydst;
            r->w = pw; r->h = ph; r->plane = pl;
            r->tmp1_off = tmp_off[0]; r->tmp2_off = tmp_off[1];
            switch (b->comp_type) {
            case COMP_INTER_AVG: r->op = B200_COMP_AVG; break;
            case COMP_INTER_WEIGHTED_AVG: r->op = B200_COMP_W_AVG; r->param = f->jnt_weights[b->ref[0]][b->ref[1]]; break;
            default:
                r->tmp1_off = tmp_off[b->mask_sign]; r->tmp2_off = tmp_off[!b->mask_sign];
                if (!pl) {
                    if (seg) {
                        /* w_mask writes the (sub-sampled) mask the chroma planes blend with */
                        r->op = B200_COMP_W_MASK_444 + chr_layout_idx; r->param = b->mask_sign;
                        /* the counter stays a multiple of 64 (it starts as one and grows by rounded sizes) */
                        r->mask_off = mask_off = (uint32_t)__atomic_fetch_add(&hf->n_cmask, ((size_t)(bw4 * 4 >> ss_hor) * (bh4 * 4 >> ss_ver) + 63) & ~(size_t)63, __ATOMIC_RELAXED);
                    } else {
                        r->op = B200_COMP_MASK;
                        r->mask_off = (uint32_t)(WEDGE_MASK(0, bs, 0, b->wedge_idx) - (const uint8_t *)&dav1d_masks);
                        if (has_chroma)
                            mask_off = (uint32_t)(WEDGE_MASK(chr_layout_idx, bs, b->mask_sign, b->wedge_idx) - (const uint8_t *)&dav1d_masks);
                    }
                } else {
                    r->op = B200_COMP_MASK; r->mask_off = mask_off;
                }
            }
        }
    }
residual:
    /* residual (:1888-1983) */
    if (!b->skip) {
        const TxfmInfo *const uvtx = &dav1d_txfm_dimensions[b->uvtx], *const ytx = &dav1d_txfm_dimensions[b->max_ytx];
        const uint16_t tx_split[2] = { b->tx_split0, b->tx_split1 };
        for (int iy = 0; iy < bh4; iy += 16)
            for (int ix = 0; ix < bw4; ix += 16) {
                int y_off = !!iy;
                for (int y = iy; y < imin(h4, iy + 16); y += ytx->h, y_off++) {
                    int x_off = !!ix;
                    for (int x = ix; x < imin(w4, ix + 16); x += ytx->w, x_off++)
                        if (bitfn(emit_tx_tree)(&c, b->max_ytx, 0, tx_split, x_off, y_off, bx + x, by + y)) goto out;
                }
                if (has_chroma)
                    for (int pl = 1; pl <= 2; pl++)
                        for (int y = iy >> ss_ver; y < imin(ch4, (iy + 16) >> ss_ver); y += uvtx->h)
                            for (int x = ix >> ss_hor; x < imin(cw4, (ix + 16) >> ss_hor); x += uvtx->w)
                                if (bitfn(emit_itx)(&c, b->uvtx, pl, g->off[pl] + uvrel + (uint32_t)(4 * y) * g->stride[1] + 4 * x, 1)) goto out;
            }
    }
    rc = 0;
out:
    if (rc) __atomic_fetch_or(&hf->unsupported, 8, __ATOMIC_RELAXED);
    return 0;       /* problems are reported when the frame completes (the whole frame fails, loudly) */
}

/* ---- frame completion ------------------------------------------------------------------------------------- */

/* moves the edge at bit `bit` of a (classes x 2 halves) mask row into class min(current class, cap) */
static inline void bitfn(cap_edge_class)(uint16_t (*const m)[2], const int n_cls, const int bit, const int half_bits, const int cap)
{
    const int half = bit >= half_bits;
    const unsigned sel = 1u << (bit - half * half_bits);
    int cls = 0;
    for (int k = n_cls - 1; k > 0; k--)
        if (m[k][half] & sel) { cls = k; break; }
    for (int k = 0; k < n_cls; k++) m[k][half] &= ~sel;
    m[imin(cls, cap)][half] |= sel;
}

/* The deblocking masks pass 1 built describe each tile on its own; at tile boundaries the edge class is limited by
 * the transform size on the other side, which the reference patches in when it filters a superblock row
 * (reference src/lf_apply_tmpl.c:331-401). Same patch, applied to our staged copy for every superblock row. */
static void bitfn(fix_tile_edges)(const Dav1dFrameContext *const f, Av1Filter *const masks)
{
    const int is_sb64 = !f->seq_hdr->sb128, sbsz = 32 >> is_sb64, sbl2 = 5 - is_sb64;
    const int ss_ver = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int has_chroma = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I400;
    const int halign = (f->bh + 31) & ~31;
    for (int sby = 0; sby < f->sbh; sby++) {
        Av1Filter *const row = masks + (sby >> is_sb64) * f->sb128w;
        const int y0 = (sby & is_sb64) << 4, y1 = y0 + imin(f->h4 - sby * sbsz, sbsz);
        const int cy0 = y0 >> ss_ver, cy1 = (y1 + ss_ver) >> ss_ver;
        for (int tc = 1; ; tc++) {
            const int sbx = f->frame_hdr->tiling.col_start_sb[tc];
            if ((sbx << sbl2) >= f->bw) break;
            const int col4 = (sbx & is_sb64) ? 16 : 0;
            Av1Filter *const m = &row[sbx >> is_sb64];
            const uint8_t *const cap_y = &f->lf.tx_lpf_right_edge[0][(sby << sbl2) + (size_t)halign * (tc - 1)];
            for (int y = y0; y < y1; y++)
                bitfn(cap_edge_class)(m->filter_y[0][col4], 3, y, 16, cap_y[y - y0]);
            if (has_chroma) {
                const uint8_t *const cap_uv = &f->lf.tx_lpf_right_edge[1][(sby << (sbl2 - ss_ver)) + (size_t)(halign >> ss_ver) * (tc - 1)];
                for (int y = cy0; y < cy1; y++)
                    bitfn(cap_edge_class)(m->filter_uv[0][col4 >> ss_hor], 2, y, 16 >> ss_ver, cap_uv[y - cy0]);
            }
        }
        const int tile_row = f->lf.start_of_tile_row[sby];
        if (!tile_row) continue;
        const BlockContext *a = &f->a[f->sb128w * (tile_row - 1)];
        for (int x = 0; x < f->sb128w; x++, a++) {
            const int w = imin(32, f->w4 - (x << 5));
            for (int i = 0; i < w; i++)
                bitfn(cap_edge_class)(row[x].filter_y[1][y0], 3, i, 16, a->tx_lpf_y[i]);
            if (has_chroma) {
                const int cw = (w + ss_hor) >> ss_hor;
                for (int i = 0; i < cw; i++)
                    bitfn(cap_edge_class)(row[x].filter_uv[1][cy0], 2, i, 16 >> ss_hor, a->tx_lpf_uv[i]);
            }
        }
    }
}

static int bitfn(run_frame)(HookFrame *const hf, const Dav1dFrameContext *const f)
{
    const double t_enter = bitfn(now_ms)();
    /* B200HOOK_PROF=1: where the host-side completion of a frame spends its time (stderr, one line per frame) */
    static int prof = -1;
    if (prof < 0) { const char *e = getenv("B200HOOK_PROF"); prof = e && atoi(e) != 0; }
    double tp[6] = { t_enter, t_enter, t_enter, t_enter, t_enter, t_enter };
    const B200Backend *const be = b200hook_backend();
    if (!be) return -1;
    if (hf->unsupported) {
        fprintf(stderr, "b200hook: frame uses tools the emitters do not translate yet (%s%s%s%s)\n",
                hf->unsupported & 1 ? " palette" : "", hf->unsupported & 2 ? " inter" : "",
                hf->unsupported & 4 ? " single-pass-decoding" : "", hf->unsupported & 8 ? " out-of-memory" : "");
        fprintf(stderr, "b200hook: unsupported mask 0x%x (16 warped motion, 32 warp from a scaled reference, 64 intra block copy out of range, 256 inter-intra block size, 1024 super-resolution)\n", hf->unsupported);
        return -1;
    }
    PicGeom g, gs;            /* the picture as coded; the picture that is output / referenced (wider with super-resolution) */
    bitfn(pic_geom)(f, &g);
    bitfn(geom_of)(&f->sr_cur.p, &gs);
    const Dav1dFrameHeader *const hdr = f->frame_hdr;
    const int superres = hdr->width[0] != hdr->width[1];
    const int mono = f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I400;         /* dummy 4:2:0 chroma planes on the device (pic_geom) */
    const int ss_ver = mono || f->cur.p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = f->cur.p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int n_sb128 = f->sb128w * f->sb128h;
    const size_t mask_bytes = (size_t)n_sb128 * sizeof(Av1Filter), level_bytes = (size_t)n_sb128 * 32 * 32 * 4;
    const size_t lr_bytes = (size_t)f->sr_sb128w * f->sb128h * sizeof(Av1Restoration);
    if (!hf->stream && !(hf->stream = be->stream_create())) { fprintf(stderr, "b200hook: %s\n", be->last_error()); return -1; }
    for (int k = 0; k < 3; k++)
        if (b200hook_buf_reserve(&hf->pic[k], g.bytes, 0, 0)) return -1;
    if (b200hook_buf_reserve(&hf->mask, mask_bytes, 1, 0) || b200hook_buf_reserve(&hf->level, level_bytes, 1, 0) ||
        b200hook_buf_reserve(&hf->lr_mask, lr_bytes, 1, 0))
        return -1;
    if (hf->n_tx > hf->cap_tx || hf->n_coef > hf->cap_coef) { fprintf(stderr, "b200hook: record buffers overflowed\n"); return -1; }
    memcpy(hf->mask.host, f->lf.mask, mask_bytes);
    bitfn(fix_tile_edges)(f, (Av1Filter *)hf->mask.host);
    memcpy(hf->level.host, f->lf.level, level_bytes);
    memcpy(hf->lr_mask.host, f->lf.lr_mask, lr_bytes);
    tp[1] = bitfn(now_ms)();

    B200FrameJob j;
    memset(&j, 0, sizeof(j));
#if BITDEPTH == 8
    j.bitdepth_max = 255;
#else
    j.bitdepth_max = f->bitdepth_max;
#endif
    /* the finished picture goes into a buffer that outlives this frame context (later frames predict from it); the
     * other stages ping-pong through the context's own pictures */
    HookRefPic *const outp = b200hook_refpic(OUT_KEY(f), gs.bytes, 1);
    if (!outp) return -1;
    const int will_cdef = f->seq_hdr->cdef && (f->c->inloop_filters & DAV1D_INLOOPFILTER_CDEF);
    const int will_lr = f->lf.restore_planes && (f->c->inloop_filters & DAV1D_INLOOPFILTER_RESTORATION);
    /* super-resolution: reconstruction, deblocking and CDEF stay in the context's own pictures (coded width); the upscaled CDEF
     * picture u1 is the output itself unless loop restoration follows, which reads u1 and the upscaled deblocked picture u0 */
    if (superres && (b200hook_buf_reserve(&hf->sr[0], gs.bytes, 0, 0) || b200hook_buf_reserve(&hf->sr[1], gs.bytes, 0, 0))) return -1;
    void *const u0 = superres ? hf->sr[0].dev : NULL, *const u1 = superres ? (will_lr ? hf->sr[1].dev : outp->dev) : NULL;
    void *const p2 = will_lr ? outp->dev : hf->pic[2].dev;
    void *const p1 = !superres && !will_lr && will_cdef ? outp->dev : hf->pic[1].dev;
    void *const p0 = !superres && !will_lr && !will_cdef ? outp->dev : hf->pic[0].dev;
    j.mc.dst = p0;
    const int inter = hf->is_inter;
    HookRefPic *rps[7];
    int n_rps = 0;
    if (inter) {
        for (int k = 0; k < 7; k++) {
            /* only the references some block really predicts from: dav1d made this frame wait for those (their pass 2 has
             * begun, so their device picture exists and will become ready); a reference nobody reads may not even have
             * started its second pass yet */
            const void *const key = f->refp[k].p.data[0];
            if (!key || !(hf->refs_used & (1u << k))) continue;
            HookRefPic *const rp = b200hook_refpic(key, 0, 0);
            if (!rp || !rp->dev) { fprintf(stderr, "b200hook: reference %d was not decoded by this back end\n", k); return -1; }
            /* its device job (another frame context) must have been enqueued: this job is ordered behind it on the device
             * (event), the host does not wait for it to finish. Without events: wait for the finished picture. */
            if (rp->event && b200hook_async()) { b200hook_refpic_wait_submitted(rp); rps[n_rps++] = rp; }
            else b200hook_refpic_wait(rp);
            j.mc.ref[k] = rp->dev;
            const Dav1dPicture *const rpic = &f->refp[k].p;
            if (rpic->p.w != f->cur.p.w || rpic->p.h != f->cur.p.h) {
                /* a reference of another size: its own plane geometry (the layout pic_geom() gives a picture of its size) */
                B200RefGeom *const rg = &j.mc.ref_geom[k];
                const int rrows = (rpic->p.h + 127) & ~127;
                rg->stride[0] = (int)PXSTRIDE(rpic->stride[0]);
                rg->stride[1] = rg->stride[2] = mono ? rg->stride[0] : (int)PXSTRIDE(rpic->stride[1]);
                rg->plane_off[0] = 0; rg->plane_off[1] = (uint32_t)rg->stride[0] * rrows;
                rg->plane_off[2] = rg->plane_off[1] + (uint32_t)rg->stride[1] * (rrows >> ss_ver);
                for (int p = 0; p < 3; p++) {
                    rg->w[p] = p ? (rpic->p.w + ss_hor) >> ss_hor : rpic->p.w;
                    rg->h[p] = p ? (rpic->p.h + ss_ver) >> ss_ver : rpic->p.h;
                }
                j.mc.scaled_mask |= 1u << k;
            }
        }
        tp[2] = bitfn(now_ms)();
        for (int p = 0; p < 3; p++) {
            j.mc.ref_plane_off[p] = g.off[p]; j.mc.ref_stride[p] = g.stride[p];
            j.mc.ref_w[p] = p ? (f->cur.p.w + ss_hor) >> ss_hor : f->cur.p.w;
            j.mc.ref_h[p] = p ? (f->cur.p.h + ss_ver) >> ss_ver : f->cur.p.h;
        }
        if (b200hook_buf_reserve(&hf->tmp16, (hf->n_tmp16 + 1) * sizeof(int16_t), 0, 0) ||
            b200hook_buf_reserve(&hf->cmask, hf->n_cmask + 64, 1, 0) ||
            /* the tiles' record lists, concatenated into the pinned upload buffers */
            (hf->n_pred = b200hook_tiles_gather(hf, B200L_PRED, &hf->pred, sizeof(B200McBlock))) < 0 ||
            (hf->n_comp = b200hook_tiles_gather(hf, B200L_COMP, &hf->comp, sizeof(B200CompBlock))) < 0 ||
            (hf->n_comp2 = b200hook_tiles_gather(hf, B200L_COMP2, &hf->comp2, sizeof(B200CompBlock))) < 0 ||
            (hf->n_warp = b200hook_tiles_gather(hf, B200L_WARP, &hf->warp, sizeof(B200WarpBlock))) < 0 ||
            (hf->n_blend = b200hook_tiles_gather(hf, B200L_BLEND, &hf->blend, sizeof(B200BlendBlock))) < 0 ||
            (hf->n_blend2 = b200hook_tiles_gather(hf, B200L_BLEND2, &hf->blend2, sizeof(B200BlendBlock))) < 0 ||
            (hf->n_scaled = b200hook_tiles_gather(hf, B200L_SCALED, &hf->scaled, sizeof(B200McScaledBlock))) < 0 ||
            b200hook_buf_reserve(&hf->pxtmp, (hf->n_pxtmp + 1) * sizeof(pixel), 0, 0))
            return -1;
        memcpy(hf->cmask.host, &dav1d_masks, sizeof(dav1d_masks));
        j.mc.tmp = (int16_t *)hf->tmp16.dev; j.mc.mask = (uint8_t *)hf->cmask.dev;
        j.d_pred = (const B200McBlock *)hf->pred.dev; j.n_pred = hf->n_pred;
        j.d_comp = (const B200CompBlock *)hf->comp.dev; j.n_comp = hf->n_comp;
        j.d_comp2 = (const B200CompBlock *)hf->comp2.dev; j.n_comp2 = hf->n_comp2;
        j.mc.px_tmp = hf->pxtmp.dev;
        j.d_warp = (const B200WarpBlock *)hf->warp.dev; j.n_warp = hf->n_warp;
        j.d_blend = (const B200BlendBlock *)hf->blend.dev; j.n_blend = hf->n_blend;
        j.d_blend2 = (const B200BlendBlock *)hf->blend2.dev; j.n_blend2 = hf->n_blend2;
        j.d_scaled = (const B200McScaledBlock *)hf->scaled.dev; j.n_scaled = hf->n_scaled;
        for (int t = 0; t < N_RECT_TX_SIZES; t++) {
            if ((hf->n_itx[t] = b200hook_tiles_gather(hf, B200L_ITX + t, &hf->itx[t], sizeof(B200ItxBlock))) < 0) return -1;
            if (!hf->n_itx[t]) continue;
            j.d_itx[t] = (const B200ItxBlock *)hf->itx[t].dev; j.n_itx[t] = hf->n_itx[t];
        }
    }
    tp[3] = bitfn(now_ms)();
    j.d_coef = hf->coef.dev;
    for (int p = 0; p < 3; p++) { j.itx_stride[p] = g.stride[p]; j.mc.dst_stride[p] = g.stride[p]; }
    /* intra reconstruction */
    j.d_intra = (const B200IntraTx *)hf->tx.dev; j.n_intra = hf->n_tx;
    j.intra.pic = p0; j.intra.d_coef = hf->coef.dev;
    j.intra.ss_hor = ss_hor; j.intra.ss_ver = ss_ver;
    for (int p = 0; p < 3; p++) {
        j.intra.stride[p] = g.stride[p]; j.intra.plane_off[p] = g.off[p];
        j.intra.w4[p] = p ? (f->bw + ss_hor) >> ss_hor : f->bw;
        j.intra.h4[p] = p ? (f->bh + ss_ver) >> ss_ver : f->bh;
    }
    if (b200hook_buf_reserve(&hf->scratch, be->intra_scratch_bytes(&j.intra), 0, 0)) return -1;
    j.intra.scratch = hf->scratch.dev;
    j.intra.mask = inter ? (const uint8_t *)hf->cmask.dev : NULL;
    j.intra.pal = hf->n_pal ? (const uint8_t *)hf->pal.dev : NULL;
    if (hf->n_pal > hf->cap_pal) { fprintf(stderr, "b200hook: palette buffer overflowed\n"); return -1; }
    if (inter && hf->n_tx > 0) {
        /* intra blocks inside an inter frame: everything that is not an intra transform block is already final */
        const size_t total = be->intra_scratch_bytes(&j.intra);
        if (b200hook_buf_reserve(&hf->done_init, total, 1, 0)) return -1;
        uint8_t *const img = hf->done_init.host;
        memset(img, 0, 256); memset(img + 256, 1, total - 256);
        size_t moff[3], o = 256;
        for (int p = 0; p < 3; p++) { moff[p] = o; o += ((size_t)j.intra.w4[p] * j.intra.h4[p] + 255) & ~(size_t)255; }
        const B200IntraTx *const recs = (const B200IntraTx *)hf->tx.host;
        for (int i = 0; i < hf->n_tx; i++) {
            const B200IntraTx *const r = &recs[i];
            const TxfmInfo *const td = &dav1d_txfm_dimensions[r->tx];
            const int mw = j.intra.w4[r->plane], mh = j.intra.h4[r->plane];
            for (int y = r->y4; y < imin(r->y4 + td->h, mh); y++)
                memset(img + moff[r->plane] + (size_t)y * mw + r->x4, 0, imin(td->w, mw - r->x4));
        }
        j.intra.done_init = (const uint8_t *)hf->done_init.dev;
    }
    tp[4] = bitfn(now_ms)();
    /* decode order -> wavefront order (B200HOOK_WAVE_SORT=0 keeps decode order, which is also valid) */
    const HookBuf *txb = &hf->tx;
    static int wave_sort = -1;
    if (wave_sort < 0) { const char *e = getenv("B200HOOK_WAVE_SORT"); wave_sort = !e || atoi(e) != 0; }
    if (wave_sort && hf->n_tx > 0) {
        if (b200hook_buf_reserve(&hf->tx_sorted, (size_t)hf->n_tx * sizeof(B200IntraTx), 1, 0)) return -1;
        if (b200hook_wave_sort((const B200IntraTx *)hf->tx.host, (B200IntraTx *)hf->tx_sorted.host, hf->n_tx,
                               j.intra.w4, j.intra.h4, ss_hor, ss_ver, &hf->sort_scratch, &hf->sort_scratch_cap) < 0) return -1;
        txb = &hf->tx_sorted;
        j.d_intra = (const B200IntraTx *)txb->dev;
    }
    tp[5] = bitfn(now_ms)();
    if (prof) fprintf(stderr, "b200hook prof: masks %.2f  ref-submit wait %.2f  gather %.2f  done map %.2f  wave sort %.2f ms (%d intra records)\n",
                      tp[1] - tp[0], tp[2] - tp[1], tp[3] - tp[2], tp[4] - tp[3], tp[5] - tp[4], hf->n_tx);
    /* deblock (reference src/recon_tmpl.c:1987-2027), in place on p0 */
    const int do_lf = (f->c->inloop_filters & DAV1D_INLOOPFILTER_DEBLOCK) && (hdr->loopfilter.level_y[0] || hdr->loopfilter.level_y[1]);
    j.run_lf = do_lf;
    j.lf.pic = p0;
    for (int p = 0; p < 3; p++) { j.lf.plane_off[p] = g.off[p]; j.lf.stride[p] = g.stride[p]; }
    j.lf.w4 = f->w4; j.lf.h4 = f->h4; j.lf.sb128w = f->sb128w; j.lf.b4_stride = (int)f->b4_stride;
    j.lf.ss_hor = ss_hor; j.lf.ss_ver = ss_ver; j.lf.sb128 = f->seq_hdr->sb128;
    j.lf.filter_y = do_lf; j.lf.filter_uv = !mono && (hdr->loopfilter.level_u || hdr->loopfilter.level_v);
    j.lf.mask = (const B200Av1Filter *)hf->mask.dev;
    j.lf.level = (const uint8_t (*)[4])hf->level.dev;
    memcpy(j.lf.lut.e, f->lf.lim_lut.e, 64); memcpy(j.lf.lut.i, f->lf.lim_lut.i, 64);
    j.lf.lut.sharp[0] = f->lf.lim_lut.sharp[0]; j.lf.lut.sharp[1] = f->lf.lim_lut.sharp[1];
    /* CDEF (:2029-2058), p0 -> p1 */
    const int do_cdef = f->seq_hdr->cdef && (f->c->inloop_filters & DAV1D_INLOOPFILTER_CDEF);
    j.run_cdef = do_cdef;
    j.cdef.src = p0; j.cdef.dst = p1;
    for (int p = 0; p < 3; p++) { j.cdef.plane_off[p] = g.off[p]; j.cdef.stride[p] = g.stride[p]; }
    j.cdef.bw = f->bw; j.cdef.bh = f->bh; j.cdef.sb128w = f->sb128w; j.cdef.ss_hor = ss_hor; j.cdef.ss_ver = ss_ver;
    j.cdef.damping = hdr->cdef.damping;
    for (int i = 0; i < 8; i++) { j.cdef.y_strength[i] = hdr->cdef.y_strength[i]; j.cdef.uv_strength[i] = hdr->cdef.uv_strength[i]; }
    j.cdef.mask = (const B200Av1Filter *)hf->mask.dev;
    /* loop restoration (:2100-2109), -> p2 */
    const int do_lr = f->lf.restore_planes && (f->c->inloop_filters & DAV1D_INLOOPFILTER_RESTORATION);
    j.run_lr = do_lr;
    j.lr.cdef = superres ? u1 : do_cdef ? p1 : p0; j.lr.dbl = superres ? u0 : p0; j.lr.dst = p2;
    for (int p = 0; p < 3; p++) { j.lr.plane_off[p] = gs.off[p]; j.lr.stride[p] = gs.stride[p]; }
    if (superres) {
        /* the upscaling stage (dav1d_filter_sbrow_resize, :2053-2086; the rows loop restoration keeps of the deblocked picture
         * are upscaled the same way, src/lf_apply_tmpl.c:73-87) */
        j.run_resize = 1;
        for (int k = 0; k < 2; k++) {
            B200ResizeFrame *const rz = &j.resize[k];
            if (k && !do_lr) break;                      /* nobody reads the upscaled deblocked picture */
            rz->src = k ? p0 : (do_cdef ? p1 : p0); rz->dst = k ? u0 : u1;
            rz->n_planes = mono ? 1 : 3;
            for (int p = 0; p < 3; p++) {
                const int sh = p && ss_hor, sv = p && ss_ver;
                rz->src_plane_off[p] = g.off[p]; rz->dst_plane_off[p] = gs.off[p];
                rz->src_stride[p] = g.stride[p]; rz->dst_stride[p] = gs.stride[p];
                rz->src_w[p] = (4 * f->bw + sh) >> sh; rz->dst_w[p] = (f->sr_cur.p.p.w + sh) >> sh;
                rz->h[p] = (f->cur.p.h + sv) >> sv;
                rz->dx[p] = f->resize_step[!!p]; rz->mx0[p] = f->resize_start[!!p];
            }
        }
    }
    j.lr.w = f->sr_cur.p.p.w; j.lr.h = f->sr_cur.p.p.h; j.lr.ss_hor = ss_hor; j.lr.ss_ver = ss_ver;
    j.lr.sb128 = f->seq_hdr->sb128; j.lr.sr_sb128w = f->sr_sb128w;
    j.lr.unit_size_log2[0] = hdr->restoration.unit_size[0]; j.lr.unit_size_log2[1] = hdr->restoration.unit_size[1];
    j.lr.restore_planes = mono ? f->lf.restore_planes & 1 : f->lf.restore_planes;
    j.lr.lr_mask = (const B200Av1Restoration *)hf->lr_mask.dev;

    B200Xfer up[48];          /* 6 fixed + 8 inter lists + 19 transform sizes + done map: 34 at most */
    int n_up = 0;
#define UP(buf, nbytes) do { if (n_up >= 48) abort(); up[n_up].host = (buf).host; up[n_up].dev = (buf).dev; up[n_up].bytes = (uint64_t)(nbytes); n_up++; } while (0)
    UP(*txb, (size_t)hf->n_tx * sizeof(B200IntraTx));
    UP(hf->coef, hf->n_coef * sizeof(coef));
    UP(hf->mask, mask_bytes); UP(hf->level, level_bytes); UP(hf->lr_mask, lr_bytes);
    if (hf->n_pal) UP(hf->pal, hf->n_pal);
    if (inter) {
        UP(hf->pred, (size_t)hf->n_pred * sizeof(B200McBlock));
        UP(hf->comp, (size_t)hf->n_comp * sizeof(B200CompBlock));
        UP(hf->comp2, (size_t)hf->n_comp2 * sizeof(B200CompBlock));
        UP(hf->warp, (size_t)hf->n_warp * sizeof(B200WarpBlock));
        UP(hf->blend, (size_t)hf->n_blend * sizeof(B200BlendBlock));
        UP(hf->blend2, (size_t)hf->n_blend2 * sizeof(B200BlendBlock));
        UP(hf->scaled, (size_t)hf->n_scaled * sizeof(B200McScaledBlock));
        UP(hf->cmask, sizeof(dav1d_masks));
        for (int t = 0; t < N_RECT_TX_SIZES; t++)
            if (hf->n_itx[t]) UP(hf->itx[t], (size_t)hf->n_itx[t] * sizeof(B200ItxBlock));
        if (j.intra.done_init) UP(hf->done_init, be->intra_scratch_bytes(&j.intra));
    }
#undef UP
    uint8_t *const out = outp->dev;
    B200Xfer down[3];
    uint64_t d2h = 0, h2d = 0;
    /* a context opened for device output keeps its pictures in HBM: nothing is copied into the host picture */
    const int n_down = b200hook_device_only(f->c) ? 0 : mono ? 1 : 3;
    for (int p = 0; p < n_down; p++) {
        const int rows = p ? (f->cur.p.h + ss_ver) >> ss_ver : f->cur.p.h;
        down[p].host = f->sr_cur.p.data[p];
        down[p].dev = out + (size_t)gs.off[p] * sizeof(pixel);
        down[p].bytes = (uint64_t)rows * gs.stride[p] * sizeof(pixel);
        d2h += down[p].bytes;
    }
    for (int i = 0; i < n_up; i++) h2d += up[i].bytes;
    const double t0 = bitfn(now_ms)();
    /* enqueue: the frame's records (they depend on nothing on the device, so they go up while earlier frames still compute),
     * the wait for the reference pictures' jobs, the job, the event later frames will wait on, the copy into the host picture.
     * Nothing here waits on the host: that happens in the frame's exit handler (b200hook_frame_finish). */
    b200hook_job_enter();
    int r = 0;
    for (int i = 0; i < n_up && !r; i++)
        if (up[i].bytes) r = be->copy_async(up[i].dev, up[i].host, up[i].bytes, hf->stream);
    for (int i = 0; i < n_rps && !r; i++) r = be->stream_wait_event(hf->stream, rps[i]->event);
    if (!r) r = be->frame_submit_host(&j, NULL, 0, NULL, 0, hf->stream);
    if (!r && outp->event) r = be->event_record(outp->event, hf->stream);
    for (int i = 0; i < n_down && !r; i++) r = be->copy_async(down[i].host, down[i].dev, down[i].bytes, hf->stream);
    b200hook_job_leave();
    if (r) {
        fprintf(stderr, "b200hook: submitting the frame job failed (%d): %s\n", r, be->last_error());
        be->frame_wait(hf->stream);             /* whatever was enqueued must not outlive the buffers */
        return -1;
    }
    uint64_t n_rec = (uint64_t)hf->n_tx + hf->n_pred + hf->n_comp + hf->n_comp2 + hf->n_warp + hf->n_blend + hf->n_blend2 + (inter ? hf->n_scaled : 0);
    uint64_t n_itx = 0;
    for (int t = 0; t < N_RECT_TX_SIZES; t++) n_itx += hf->n_itx[t];
    n_rec += n_itx;
    const uint64_t kinds[11] = { (uint64_t)hf->n_tx, (uint64_t)hf->n_pred, (uint64_t)hf->n_comp + hf->n_comp2, (uint64_t)hf->n_warp,
                                (uint64_t)hf->n_blend + hf->n_blend2, n_itx, (uint64_t)inter, (uint64_t)hf->n_ii, (uint64_t)hf->n_pal, (uint64_t)hf->n_ibc, (uint64_t)(inter ? hf->n_scaled : 0) };
    hf->pending = 1; hf->pending_out = outp; hf->t_submit = t0; hf->pend_prep_ms = t0 - t_enter;
    hf->pend_rec = n_rec; hf->pend_coef = hf->n_coef; hf->pend_h2d = h2d; hf->pend_d2h = d2h;
    memcpy(hf->pend_kinds, kinds, sizeof(kinds));
    b200hook_refpic_set_submitted(outp, 1);
    if (!b200hook_async()) return b200hook_frame_finish(hf) ? -1 : 0;     /* B200HOOK_ASYNC=0: one job at a time per context, host waits here */
    return 0;
}

/* "tile superblock row reconstructed" (pass 2 calls this after every tile superblock row, reference
 * src/decode.c:2620-2635): the frame is complete when every tile has delivered all of its rows */
void bitfn(b200hook_backup_ipred_edge)(Dav1dTaskContext *const t)
{
    Dav1dFrameContext *const f = (Dav1dFrameContext *)t->f;
    HookFrame *const hf = b200hook_frame(f);
    if (!hf) { atomic_fetch_or(&f->task_thread.error, 1); return; }
    pthread_mutex_lock(&hf->lock);
    if (t->frame_thread.pass != 2) __atomic_fetch_or(&hf->unsupported, 4, __ATOMIC_RELAXED);
    const int total = f->sbh * f->frame_hdr->tiling.cols;
    if (++hf->tile_sbrows_done >= total) {
        if (bitfn(run_frame)(hf, f)) {
            atomic_fetch_or(&f->task_thread.error, 1);      /* the frame is reported as a decoding error */
            HookRefPic *const outp = b200hook_refpic(OUT_KEY(f), 0, 0);
            if (outp && !hf->pending) b200hook_refpic_set_ready(outp, 1);       /* after a failure nobody may wait for ever */
        }
        hf->tile_sbrows_done = 0; hf->n_tx = 0; hf->n_coef = 0; hf->unsupported = 0;
        hf->n_pred = hf->n_comp = hf->n_comp2 = hf->n_warp = hf->n_blend = hf->n_blend2 = 0;
        hf->n_tmp16 = 0; hf->n_pxtmp = 0; hf->started = 0; hf->is_inter = 0; hf->n_ii = 0; hf->n_ibc = 0; hf->refs_used = 0;
        memset(hf->n_itx, 0, sizeof(hf->n_itx));
    }
    pthread_mutex_unlock(&hf->lock);
}

/* the post-filter sweep already ran on the device as part of the frame job */
void bitfn(b200hook_filter_sbrow)(Dav1dFrameContext *const f, const int sby) { (void)f; (void)sby; }
void bitfn(b200hook_filter_sbrow_deblock_cols)(Dav1dFrameContext *const f, const int sby) { (void)f; (void)sby; }
void bitfn(b200hook_filter_sbrow_deblock_rows)(Dav1dFrameContext *const f, const int sby) { (void)f; (void)sby; }
void bitfn(b200hook_filter_sbrow_cdef)(Dav1dTaskContext *const tc, const int sby) { (void)tc; (void)sby; }
void bitfn(b200hook_filter_sbrow_resize)(Dav1dFrameContext *const f, const int sby) { (void)f; (void)sby; }
void bitfn(b200hook_filter_sbrow_lr)(Dav1dFrameContext *const f, const int sby) { (void)f; (void)sby; }


/* ---- film grain on the output copy (dav1d_apply_grain, reference src/lib.c:485-520; with worker threads the
 * delayed_fg tasks of src/thread_task.c:470-545 call prep_grain once and apply_grain_row per 32-row strip) ---------
 * The decoded picture is still in HBM (keyed by its host buffer), so the whole job — grain LUTs, scaling LUTs, every
 * strip of every plane — runs as one b200 frame job when `prep` is called; the per-row calls have nothing left to do. */
#include "src/fg_apply.h"
/* the context whose dsp table the film-grain call came through (lib.c and thread_task.c pass &c->dsp[bpc index].fg) */
static const Dav1dContext *bitfn(fg_context)(const Dav1dFilmGrainDSPContext *const dsp, const int bpc)
{
    const int idx = BITDEPTH == 8 ? 0 : (bpc >> 1) - 4;
    return (const Dav1dContext *)((const char *)dsp - offsetof(Dav1dDSPContext, fg) - (size_t)idx * sizeof(Dav1dDSPContext) -
                                  offsetof(Dav1dContext, dsp));
}
static void bitfn(fg_whole_picture)(const Dav1dFilmGrainDSPContext *const dsp, Dav1dPicture *const out, const Dav1dPicture *const in)
{
    const B200Backend *const be = b200hook_backend();
    if (!be) { fprintf(stderr, "b200hook: film grain: no back end\n"); abort(); }      /* no error channel here (void, like dav1d's), no CPU fallback */
    const int mono = in->p.layout == DAV1D_PIXEL_LAYOUT_I400;            /* device picture: dummy 4:2:0 chroma planes (pic_geom) */
    const int ss_ver = mono || in->p.layout == DAV1D_PIXEL_LAYOUT_I420, ss_hor = in->p.layout != DAV1D_PIXEL_LAYOUT_I444;
    const int rows = (in->p.h + 127) & ~127;
    const int st0 = (int)PXSTRIDE(in->stride[0]), st1 = mono ? st0 : (int)PXSTRIDE(in->stride[1]);
    const uint32_t off1 = (uint32_t)st0 * rows, off2 = off1 + (uint32_t)st1 * (rows >> ss_ver);
    const size_t bytes = ((size_t)off2 + (size_t)st1 * (rows >> ss_ver)) * sizeof(pixel);
    const int npl = mono ? 1 : 3;
    /* normally the decoded picture is still in HBM (keyed by its host buffer). It is not when it was decoded elsewhere and
     * handed to the public dav1d_apply_grain, or after b200hook_release(): then the host picture goes up first. */
    HookRefPic *const src = b200hook_refpic(in->data[0], 0, 0);
    const char *const force = getenv("B200HOOK_FG_UPLOAD");                /* tests: take the upload path although the picture is resident */
    const int resident = src && src->dev && src->bytes >= bytes && !(force && atoi(force));
    if (resident) b200hook_refpic_wait(src);
    const int same_pitch = out->stride[0] == in->stride[0] && (mono || out->stride[1] == in->stride[1]);
    /* device output: the grained picture gets a resident device copy of its own, keyed by its host buffer like every decoded
     * picture (the slot's pic[0] is overwritten by the next grained picture), and nothing is copied into the host picture */
    HookRefPic *dst = NULL;
    if (b200hook_device_only(bitfn(fg_context)(dsp, in->p.bpc))) {
        /* (the host picture holds no pixels to upload) */
        if (!resident || !same_pitch || !(dst = b200hook_refpic(out->data[0], bytes, 1))) { fprintf(stderr, "b200hook: film grain: no device picture\n"); abort(); }
        b200hook_refpic_set_ready(dst, 0);
    }
    static const char fg_slot_key = 0;
    HookFrame *const hf = b200hook_frame(&fg_slot_key);                  /* a slot of its own for the output stage */
    if (!hf) { fprintf(stderr, "b200hook: film grain: no slot\n"); abort(); }
    hf->pinned = 1;
    pthread_mutex_lock(&hf->lock);
    if ((!hf->stream && !(hf->stream = be->stream_create())) || b200hook_buf_reserve(&hf->pic[0], bytes, 0, 0) ||
        (!resident && b200hook_buf_reserve(&hf->pic[1], bytes, 0, 0)) ||
        b200hook_buf_reserve(&hf->scratch, B200_FG_SCRATCH_BYTES, 0, 0)) {
        fprintf(stderr, "b200hook: film grain: %s\n", be->last_error());
        abort();
    }
    B200FrameJob j;
    memset(&j, 0, sizeof(j));
#if BITDEPTH == 8
    j.bitdepth_max = 255;
#else
    j.bitdepth_max = (1 << in->p.bpc) - 1;
#endif
    j.run_fg = 1;
    j.fg.in = resident ? src->dev : hf->pic[1].dev; j.fg.out = dst ? dst->dev : hf->pic[0].dev; j.fg.scratch = hf->scratch.dev;
    j.fg.plane_off[0] = 0; j.fg.plane_off[1] = off1; j.fg.plane_off[2] = off2;
    j.fg.stride[0] = st0; j.fg.stride[1] = j.fg.stride[2] = st1;
    j.fg.w = in->p.w; j.fg.h = in->p.h; j.fg.ss_hor = ss_hor; j.fg.ss_ver = ss_ver;
    j.fg.is_id = in->seq_hdr->mtrx == DAV1D_MC_IDENTITY;
    memcpy(&j.fg.data, &in->frame_hdr->film_grain.data, sizeof(j.fg.data));
    b200hook_job_enter();
    int r = 0;
    for (int p = 0; p < npl && !resident && !r; p++) {
        const int prow = p ? (in->p.h + ss_ver) >> ss_ver : in->p.h;
        r = be->copy_async((uint8_t *)hf->pic[1].dev + (size_t)j.fg.plane_off[p] * sizeof(pixel), in->data[p],
                           (size_t)prow * j.fg.stride[p] * sizeof(pixel), hf->stream);
    }
    if (!r) r = be->frame_submit_host(&j, NULL, 0, NULL, 0, hf->stream);
    if (!r && dst && dst->event) r = be->event_record(dst->event, hf->stream);
    for (int p = 0; p < npl && !r && !dst; p++) {
        const int prow = p ? (in->p.h + ss_ver) >> ss_ver : in->p.h, pw = p ? (in->p.w + ss_hor) >> ss_hor : in->p.w;
        const uint8_t *const d = (const uint8_t *)hf->pic[0].dev + (size_t)j.fg.plane_off[p] * sizeof(pixel);
        if (same_pitch) r = be->copy_async(out->data[p], d, (size_t)prow * j.fg.stride[p] * sizeof(pixel), hf->stream);
        else            /* an output copy with another pitch (a caller's own allocator): row by row */
            for (int y = 0; y < prow && !r; y++)
                r = be->copy_async((uint8_t *)out->data[p] + (ptrdiff_t)y * out->stride[!!p], d + (size_t)y * j.fg.stride[p] * sizeof(pixel),
                                   (size_t)pw * sizeof(pixel), hf->stream);
    }
    const int r2 = be->frame_wait(hf->stream);
    b200hook_job_leave();
    pthread_mutex_unlock(&hf->lock);
    if (r || r2) { fprintf(stderr, "b200hook: film grain job failed: %s\n", be->last_error()); abort(); }
    if (dst) b200hook_refpic_set_ready(dst, 1);
}

void bitfn(b200hook_apply_grain)(const Dav1dFilmGrainDSPContext *const dsp, Dav1dPicture *const out, const Dav1dPicture *const in)
{
    bitfn(fg_whole_picture)(dsp, out, in);
}
void bitfn(b200hook_prep_grain)(const Dav1dFilmGrainDSPContext *const dsp, Dav1dPicture *const out, const Dav1dPicture *const in,
                                uint8_t scaling[3][SCALING_SIZE], entry grain_lut[3][GRAIN_HEIGHT + 1][GRAIN_WIDTH])
{
    (void)scaling; (void)grain_lut;
    bitfn(fg_whole_picture)(dsp, out, in);
}
void bitfn(b200hook_apply_grain_row)(const Dav1dFilmGrainDSPContext *const dsp, Dav1dPicture *const out, const Dav1dPicture *const in,
                                     const uint8_t scaling[3][SCALING_SIZE], const entry grain_lut[3][GRAIN_HEIGHT + 1][GRAIN_WIDTH],
                                     const int row)
{
    (void)dsp; (void)out; (void)in; (void)scaling; (void)grain_lut; (void)row;      /* done by the job prep started */
}

/* ---- export of an output picture from its device copy (b200hook_export_picture / _tensor_batch in b200_hooks.c) --------------
 * Ungrained pictures are the frame job's output entry (OUT_KEY: with super-resolution the upscaled picture), grained ones the
 * entry film grain made for them; either is keyed by the picture's data[0] and laid out as geom_of() says. Both jobs take
 * the same source fields from it. */
#define EXPORT_SOURCE(j, r, g, p) do { \
        const int mono_ = (p)->p.layout == DAV1D_PIXEL_LAYOUT_I400; \
        (j).src = (r)->dev; \
        for (int k = 0; k < 3; k++) { (j).plane_off[k] = (g).off[k]; (j).stride[k] = (g).stride[k]; } \
        (j).w = (p)->p.w; (j).h = (p)->p.h; (j).mono = mono_; \
        (j).ss_hor = (p)->p.layout != DAV1D_PIXEL_LAYOUT_I444; (j).ss_ver = mono_ || (p)->p.layout == DAV1D_PIXEL_LAYOUT_I420; \
        (j).bitdepth_max = (1 << (p)->p.bpc) - 1; \
    } while (0)
static HookRefPic *bitfn(export_source)(const Dav1dPicture *const p, PicGeom *const g)
{
    bitfn(geom_of)(p, g);
    HookRefPic *const r = b200hook_refpic(p->data[0], 0, 0);
    if (!r || !r->dev || r->bytes < g->bytes) { fprintf(stderr, "b200hook: export: the picture has no device copy\n"); return NULL; }
    b200hook_refpic_wait(r);
    return r;
}
int bitfn(b200hook_export_picture)(const Dav1dPicture *const p, const B200ExportJob *const tmpl, void *const stream)
{
    PicGeom g;
    HookRefPic *r = bitfn(export_source)(p, &g);
    if (!r) return -1;
    B200ExportJob j = *tmpl;
    EXPORT_SOURCE(j, r, g, p);
    return b200hook_export_submit(&r, 1, 0, &j, NULL, NULL, stream);
}
/* fills the source fields of tensor job *j from the picture's device copy: that entry, NULL when it has none or when `box`
 * (top, left, height, width, or NULL for the whole picture) is not a box of the picture whose chroma keeps its siting
 * (include/b200av1.h B200TensorJob); the box's sub-picture is then the source */
HookRefPic *bitfn(b200hook_tensor_source)(const Dav1dPicture *const p, const int32_t *const box, B200TensorJob *const j)
{
    if (box) {
        const int mono = p->p.layout == DAV1D_PIXEL_LAYOUT_I400;
        const int ssh = !mono && p->p.layout != DAV1D_PIXEL_LAYOUT_I444, ssv = p->p.layout == DAV1D_PIXEL_LAYOUT_I420;
        const int64_t top = box[0], left = box[1], bh = box[2], bw = box[3];
        if (top < 0 || left < 0 || bh < 1 || bw < 1 || top + bh > p->p.h || left + bw > p->p.w || (top & ssv) || (left & ssh)) {
            fprintf(stderr, "b200hook: export: bad crop box (top %lld, left %lld, %lld x %lld) of a %d x %d picture\n",
                    (long long)top, (long long)left, (long long)bw, (long long)bh, p->p.w, p->p.h);
            return NULL;
        }
    }
    PicGeom g;
    HookRefPic *const r = bitfn(export_source)(p, &g);
    if (!r) return NULL;
    EXPORT_SOURCE(*j, r, g, p);
    if (box) {
        j->plane_off[0] += (uint32_t)((int64_t)box[0] * j->stride[0] + box[1]);
        for (int k = 1; k < 3 && !j->mono; k++)
            j->plane_off[k] += (uint32_t)((int64_t)(box[0] >> j->ss_ver) * j->stride[k] + (box[1] >> j->ss_hor));
        j->h = box[2]; j->w = box[3];
    }
    return r;
}
#undef EXPORT_SOURCE
