"""Host side of the whole-frame job (include/b200av1.h, B200FrameJob).

FrameBuffers turns one frame's records (numpy arrays in dav1d's layouts, e.g. from synth.py — the
role dav1d's pass-1 entropy decode plays in a real integration) into device buffers + a B200FrameJob,
and runs it. `alloc` abstracts where the buffers live: torch CUDA tensors on the GPU, or plain numpy
when the same C ABI is bound to the test-only host emulator.
"""
import ctypes as C
import numpy as np

from . import _lib


class TorchAlloc:
    """device buffers as torch CUDA tensors (torch is plumbing: memory + streams only)"""

    def __init__(self, device=None):
        import torch
        self.torch = torch
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())

    def upload(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(self.device)
        return t, t.data_ptr()

    def zeros(self, nbytes):
        t = self.torch.zeros(max(nbytes, 16), dtype=self.torch.uint8, device=self.device)
        return t, t.data_ptr()

    def download(self, t, like):
        return t.cpu().numpy()[:like.nbytes].view(like.dtype)

    def pinned(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).pin_memory()
        return t, t.data_ptr()

    def sync(self):
        self.torch.cuda.synchronize()

    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def new_stream(self):
        s = self.torch.cuda.Stream(device=self.device)
        return s, s.cuda_stream


class NumpyAlloc:
    """'device' == host: only valid with the emulated library (tests/emu)"""

    def upload(self, a):
        c = np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()
        return c, c.ctypes.data

    def zeros(self, nbytes):
        c = np.zeros(max(nbytes, 16), np.uint8)
        return c, c.ctypes.data

    def download(self, t, like):
        return t[:like.nbytes].view(like.dtype)

    def pinned(self, a):
        return self.upload(a)

    def sync(self):
        pass

    def stream(self):
        return None

    def new_stream(self):
        return None, None


# ---- the stage descriptors of a frame: S's geometry and parameters, buffers as plain addresses ----
def mc_frame(S):
    """B200McFrame geometry: every reference has S's planes (the callers set the buffer pointers)"""
    fr = _lib.McFrame()
    ssh, ssv = [0, S["ss_hor"], S["ss_hor"]], [0, S["ss_ver"], S["ss_ver"]]
    for p in range(3):
        fr.ref_plane_off[p] = S["off"][p]; fr.ref_stride[p] = fr.dst_stride[p] = S["stride"][p]
        fr.ref_w[p] = (S["W"] + ssh[p]) >> ssh[p]; fr.ref_h[p] = (S["H"] + ssv[p]) >> ssv[p]
    return fr


def intra_frame(S, pic, coef):
    """B200IntraFrame geometry over the picture at `pic` and the dense coefficients at `coef`"""
    fr = _lib.IntraFrame()
    fr.pic, fr.d_coef = pic, coef
    fr.ss_hor, fr.ss_ver = S["ss_hor"], S["ss_ver"]
    for p in range(3):
        ssh, ssv = (S["ss_hor"], S["ss_ver"]) if p else (0, 0)
        fr.stride[p], fr.plane_off[p] = S["stride"][p], S["off"][p]
        fr.w4[p], fr.h4[p] = S["w4"] >> ssh, S["h4"] >> ssv
    return fr


def lf_frame(S, pic, mask, level):
    """B200LfFrame: deblocks the picture at `pic` in place. S["sb128"] (default 0) is the superblock walk order and
    S["filter_uv"] (default 1) whether chroma is filtered; luma always is."""
    fr = _lib.LfFrame()
    fr.pic, fr.mask, fr.level = pic, mask, level
    for p in range(3):
        fr.plane_off[p] = S["off"][p]; fr.stride[p] = S["stride"][p]
    fr.w4, fr.h4, fr.sb128w, fr.b4_stride = S["w4"], S["h4"], S["sb128w"], S["b4_stride"]
    fr.ss_hor, fr.ss_ver, fr.sb128 = S["ss_hor"], S["ss_ver"], S.get("sb128", 0)
    fr.filter_y, fr.filter_uv = 1, S.get("filter_uv", 1)
    for k in range(64):
        fr.lut.e[k], fr.lut.i[k] = int(S["lut_e"][k]), int(S["lut_i"][k])
    fr.lut.sharp[0], fr.lut.sharp[1] = S["lut_sharp"]
    return fr


def cdef_frame(S, src, dst, mask):
    """B200CdefFrame: the picture at `src` filtered into `dst`"""
    fr = _lib.CdefFrame()
    fr.src, fr.dst, fr.mask = src, dst, mask
    for p in range(3):
        fr.plane_off[p] = S["off"][p]; fr.stride[p] = S["stride"][p]
    fr.bw, fr.bh, fr.sb128w, fr.ss_hor, fr.ss_ver, fr.damping = S["bw"], S["bh"], S["sb128w"], S["ss_hor"], S["ss_ver"], S["damping"]
    for i in range(8):
        fr.y_strength[i], fr.uv_strength[i] = S["y_strength"][i], S["uv_strength"][i]
    return fr


def lr_frame(S, cdef, dbl, dst, lr_mask):
    """B200LrFrame: the CDEF output at `cdef` (and the deblocked picture at `dbl`, for the stripe edges) restored
    into `dst`"""
    fr = _lib.LrFrame()
    fr.cdef, fr.dbl, fr.dst, fr.lr_mask = cdef, dbl, dst, lr_mask
    for p in range(3):
        fr.plane_off[p] = S["off"][p]; fr.stride[p] = S["stride"][p]
    fr.w, fr.h, fr.ss_hor, fr.ss_ver, fr.sb128 = S["W"], S["H"], S["ss_hor"], S["ss_ver"], S["sb128"]
    fr.sr_sb128w = (S["W"] + 127) >> 7
    fr.unit_size_log2[0], fr.unit_size_log2[1] = S["us"]
    fr.restore_planes = S["rp"]
    return fr


def fg_frame(S, src, dst):
    """B200FgFrame: film grain S["fg"] applied to the picture at `src`, written to `dst` (the caller sets the scratch)"""
    fr = _lib.FgFrame()
    fr.in_, fr.out = src, dst
    for p in range(3):
        fr.plane_off[p] = S["off"][p]; fr.stride[p] = S["stride"][p]
    fr.w, fr.h, fr.ss_hor, fr.ss_ver, fr.is_id = S["W"], S["H"], S["ss_hor"], S["ss_ver"], 0
    fr.data = S["fg"]
    return fr


def band_plan(S, band_rows, compact=False, fused=False):
    """Cut a frame's records into horizontal bands of `band_rows` luma rows (a multiple of 64: blocks never straddle a
    band). Returns (S2, bands, need): S2 = shallow copy of S whose record arrays are stably sorted by band (the by-area
    order is kept inside a band), bands = list of dicts {y0, y1, last, <record list>: (first, count)} and need[k][ref] =
    (luma rows, chroma rows) of reference `ref` that band k's predictions read — the `lowest_pixel` of dav1d's
    check_tile (reference src/thread_task.c:415, src/decode.c lowest_pixel bookkeeping); expand = the compact coefficient
    stream, its band-sorted B200CoefBlock records and the per-size block offsets into it (itx_compact_offsets) when `compact`. Intra records (S["intra_tx"]) are sorted by band too
    (bands[k]["intra"]); see check_intra_bands for what they may read."""
    assert band_rows % 64 == 0 and band_rows > 0
    H, off, stride = S["H"], S["off"], S["stride"]
    ssv = [0, S["ss_ver"], S["ss_ver"]]
    nb = -(-H // band_rows)
    S2 = dict(S)

    def luma_y(dst_off, plane):
        pl = np.asarray(plane).astype(np.int64)
        o = np.asarray(off, np.int64)[pl]; st = np.asarray(stride, np.int64)[pl]
        return ((np.asarray(dst_off).astype(np.int64) - o) // st) << np.asarray(ssv, np.int64)[pl]

    def sort_by_band(arr, y):
        band = (y // band_rows).astype(np.int64)
        assert not len(band) or (band.min() >= 0 and band.max() < nb)
        order = np.argsort(band, kind="stable")
        cnt = np.bincount(band, minlength=nb)
        first = np.concatenate([[0], np.cumsum(cnt)[:-1]])
        return arr[order], first, cnt, band[order]

    ranges = {}
    # compound records first: they tell where the int16 predictions (op 1, addressed in `tmp`) belong
    tmp_y = {}
    for name in ("comp", "comp2"):
        a = S[name]
        y = luma_y(a["dst_off"], a["plane"]) if len(a) else np.zeros(0, np.int64)
        for t1, t2, yy in zip(a["tmp1_off"].tolist(), a["tmp2_off"].tolist(), y.tolist()):
            tmp_y[t1] = yy; tmp_y[t2] = yy
        S2[name], f, c, _ = sort_by_band(a, y)
        ranges[name] = (f, c)
    # blends (OBMC): they tell where the overlapped predictions (op 2, addressed in `px_tmp`) belong; 8x8 warps
    lap_y = {}
    for name in ("blend", "blend2", "warp"):
        if name in S:
            a = S[name]
            y = luma_y(a["dst_off"], a["plane"]) if len(a) else np.zeros(0, np.int64)
            if name != "warp":
                for t, yy in zip(a["tmp_off"].tolist(), y.tolist()):
                    lap_y[t] = yy
            S2[name], f, c, _ = sort_by_band(a, y)
            ranges[name] = (f, c)
    pname = "pred_single" if (fused and "cfused" in S) else "pred"
    a = S[pname]
    y = np.zeros(len(a), np.int64)
    put, prep, lap = a["op"] == 0, a["op"] == 1, a["op"] == 2
    if put.any():
        y[put] = luma_y(a["dst_off"][put], a["plane"][put])
    if prep.any():
        y[prep] = [tmp_y[t] for t in a["dst_off"][prep].tolist()]
    if lap.any():
        y[lap] = [lap_y[t] for t in a["dst_off"][lap].tolist()]
    S2[pname], f, c, pband = sort_by_band(a, y)
    ranges["pred"] = (f, c)
    for name in ("cfused", "cfused2"):
        if fused and name in S:
            a = S[name]
            S2[name], f, c, _ = sort_by_band(a, luma_y(a["dst_off"], a["plane"]) if len(a) else np.zeros(0, np.int64))
            ranges[name] = (f, c)
    S2["itx"] = {}
    itx_ranges = {}
    for tx in range(19):
        a = S["itx"][tx]
        S2["itx"][tx], f, c, _ = sort_by_band(a, luma_y(a["dst_off"], a["plane"]) if len(a) else np.zeros(0, np.int64))
        itx_ranges[tx] = (f, c)
    # intra-machine records (intra, CFL, palette, inter-intra, intra block copy) by the luma row of their top: the stable sort
    # keeps the wavefront order, so the records of every band stay in a topological order
    iband = None
    it = S.get("intra_tx")
    if it is not None and len(it):
        S2["intra_tx"], f, c, iband = sort_by_band(it, luma_y(it["dst_off"], it["plane"]))
        ranges["intra"] = (f, c)
        check_intra_bands(S, S2["intra_tx"], iband, band_rows, nb)
    expand = None
    if compact:
        from . import synth
        cc, ex = synth.compact_coefs(S2)
        # compact_coefs emits its records size class after size class, each in the (band-sorted) order of S2["itx"][tx]
        per_tx = [np.repeat(np.arange(nb), itx_ranges[tx][1]) for tx in range(19) if len(S2["itx"][tx])]       # empty: every inter block skipped
        # ... followed by the coded intra records, size class after size class, in the (band-sorted) order of S2["intra_tx"]
        if iband is not None:
            it2 = S2["intra_tx"]
            per_tx += [iband[(it2["tx"] == tx) & (it2["eob"] >= 0)] for tx in range(19)]
        eb = np.concatenate(per_tx).astype(np.int64) if per_tx else np.zeros(0, np.int64)
        assert len(eb) == len(ex)
        order = np.argsort(eb, kind="stable")
        cnt = np.bincount(eb, minlength=nb)
        expand = (cc, ex[order], itx_compact_offsets(S2, ex))
        ranges["expand"] = (np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
    bands = []
    for k in range(nb):
        b = {"y0": k * band_rows, "y1": min(H, (k + 1) * band_rows), "last": int(k == nb - 1)}
        for name, (f, c) in ranges.items():
            b[name] = (int(f[k]), int(c[k]))
        b["itx"] = [(int(itx_ranges[tx][0][k]), int(itx_ranges[tx][1][k])) for tx in range(19)]
        bands.append(b)
    # rows of each reference that a band reads: block bottom + 4 rows of filter support (8-tap: 3 above, 4 below)
    P = S2[pname]
    n_refs = len(S["refs"])
    need = np.zeros((nb, max(n_refs, 1), 2), np.int64)
    if len(P):
        low = P["src_y"].astype(np.int64) + P["h"] + 4
        cls = (P["plane"] > 0).astype(np.int64)
        np.maximum.at(need, (pband, P["ref"].astype(np.int64), cls), low)
    ph = [H, (H + ssv[1]) >> ssv[1]]
    need[:, :, 0] = np.minimum(need[:, :, 0], ph[0]); need[:, :, 1] = np.minimum(need[:, :, 1], ph[1])
    return S2, bands, need, expand


def itx_compact_offsets(S, ex):
    """B200FrameJob.d_itx_coff: per transform size, where the coefficients of each block of S["itx"][tx] start in the compact
    stream. synth.compact_coefs emits its B200CoefBlock records `ex` size after size, each in the order of S["itx"][tx]
    (the coded intra records follow); that order is checked and kept, so a band's range of S["itx"][tx] indexes the
    offsets too."""
    out, pos = {}, 0
    for tx in range(19):
        a = S["itx"][tx]
        if len(a):
            r = ex[pos:pos + len(a)]
            assert len(r) == len(a) and (r["tx"] == tx).all() and (r["dense_off"] == a["coef_off"]).all()
            out[tx] = r["compact_off"].astype("<u4")
            pos += len(a)
    return out


def check_intra_bands(S, tx, band, band_rows, nb):
    """No intra record of a band may read a row at or below the band's bottom: those rows are reconstructed by a later
    band, so the intra kernel would wait for their cells forever (or, for cells of inter blocks, which the done map marks
    final from the start, read pixels that are not there yet). Checks the cells the kernel waits for: bottom-left edges,
    intra block copy sources and the luma blocks of CFL records. The bottom band reads nothing below itself."""
    from . import levels as L, synth
    if nb == 1 or not len(tx):
        return
    ssv = np.where(tx["plane"] > 0, S["ss_ver"], 0).astype(np.int64)
    th = (np.asarray(L.TX_H)[tx["tx"]] // 4).astype(np.int64)
    y, ye = tx["y4"].astype(np.int64), tx["yend4"].astype(np.int64)
    h4 = np.where(tx["plane"] > 0, S["h4"] >> S["ss_ver"], S["h4"])
    mode, fl = tx["mode"], tx["flags"].astype(np.int64)
    reach = y + th                                                   # end of the rows read, plane 4-sample units
    edges = (mode != synth.MODE_RESID) & (mode != synth.MODE_IBC)
    bl = edges & ((fl & 9) == 9) & (y + th < ye)                    # HAVE_LEFT | LEFT_HAS_BOTTOM
    reach = np.where(bl, y + th + np.minimum(th, ye - y - th), reach)
    ibc = mode == synth.MODE_IBC
    sy = (tx["luma_off"] >> 16).astype(np.int64)
    reach = np.where(ibc, np.minimum((sy + 4 * th - 1 + (tx["cfl_h_pad"] != 0)) >> 2, h4 - 1) + 1, reach)
    cfl = (mode == synth.MODE_CFL) & (tx["cfl_alpha"] != 0)          # CFL: end of the luma block, luma 4-sample units
    ly4 = y << ssv
    lum = np.where(cfl, ly4 + np.minimum((th - tx["cfl_h_pad"].astype(np.int64)) << ssv, S["h4"] - ly4), 0)
    y1 = (band + 1) * band_rows
    bad = (band < nb - 1) & (((reach * 4) << ssv > y1) | (lum * 4 > y1))
    assert not bad.any(), "intra record %d (plane %d, y4 %d, mode %d) reads rows below its band [.., %d)" % (
        int(np.argmax(bad)), int(tx["plane"][bad][0]), int(y[bad][0]), int(mode[bad][0]), int(y1[bad][0]))


def run_batch(fbs, stream=None):
    """b200_frame_run_batch over several FrameBuffers (same library, same bit depth) on one stream: their intra
    stages share launches (frames are the parallel axis of intra decoding)."""
    lib = fbs[0].lib
    arr = (C.POINTER(_lib.FrameJob) * len(fbs))(*[C.pointer(fb.job) for fb in fbs])
    st = fbs[0].alloc.stream() if stream is None else stream
    lib.check(lib.b200_frame_run_batch(arr, len(fbs), st), "b200_frame_run_batch")


class FrameGroup:
    """Several FrameBuffers driven as one unit on one stream (b200_frame_run_batch / b200_frame_submit_host_batch)."""

    def __init__(self, fbs):
        self.fbs, self.lib = fbs, fbs[0].lib
        self.jobs = (C.POINTER(_lib.FrameJob) * len(fbs))(*[C.pointer(fb.job) for fb in fbs])
        self._stream = None
        self._host = False

    def stream(self):
        if self._stream is None:
            self._stream = self.fbs[0].alloc.new_stream()
        return self._stream[1]

    def run(self, stream=None):
        self.lib.check(self.lib.b200_frame_run_batch(self.jobs, len(self.fbs), self.stream() if stream is None else stream),
                       "b200_frame_run_batch")

    def submit_host(self):
        if not self._host:
            ups, downs = [], []
            for fb in self.fbs:
                fb.prepare_host(); fb._host = True
                ups += list(fb._ups); downs += list(fb._downs)
            self._ups = (_lib.Xfer * len(ups))(*ups); self._downs = (_lib.Xfer * len(downs))(*downs)
            self._host = True
        self.lib.check(self.lib.b200_frame_submit_host_batch(self.jobs, len(self.fbs), self._ups, len(self._ups), self._downs,
                                                             len(self._downs), self.stream()), "b200_frame_submit_host_batch")

    def wait(self):
        self.lib.check(self.lib.b200_frame_wait(self.stream()), "b200_frame_wait")


class FrameBuffers:
    def __init__(self, S, lib=None, alloc=None, run_lf=True, run_cdef=True, run_lr=True, intra_grid=0, compact=False, intra_sb=False, fused=False,
                 band_rows=0):
        self.bands = None
        expand = None
        if band_rows:            # records sorted by band + the B200FrameBand list (b200_frame_run_band)
            S, plan, self.band_need, expand = band_plan(S, band_rows, compact=compact, fused=fused)
            self.bands = (_lib.FrameBand * len(plan))()
            for k, b in enumerate(plan):
                fbn = self.bands[k]
                fbn.y0, fbn.y1, fbn.last = b["y0"], b["y1"], b["last"]
                for name in ("pred", "warp", "comp", "comp2", "blend", "blend2", "cfused", "cfused2", "expand", "intra"):
                    if name in b:
                        getattr(fbn, name)[0], getattr(fbn, name)[1] = b[name]
                for tx in range(19):
                    fbn.itx[tx][0], fbn.itx[tx][1] = b["itx"][tx]
        self.S, self.lib = S, lib or _lib.get_lib()
        self.alloc = alloc or TorchAlloc()
        A = self.alloc
        self.keep = {}
        px = S["pic"].itemsize

        def up(name, arr):
            self.keep[name] = A.upload(arr)
            return self.keep[name][1]

        def zeros(name, nbytes):
            self.keep[name] = A.zeros(nbytes)
            return self.keep[name][1]
        nbytes = S["pic"].nbytes
        refs = [up("ref%d" % i, r) for i, r in enumerate(S["refs"])]
        p0, p1, p2 = zeros("p0", nbytes), zeros("p1", nbytes), zeros("p2", nbytes)
        tmp = zeros("tmp", S["tmp_len"] * 2)
        mask = up("mask", S["mask"])
        j = _lib.FrameJob()
        j.bitdepth_max, j.zero_coefs = S["bd"], 0
        j.mc = mc_frame(S)
        for i, r in enumerate(refs):
            j.mc.ref[i] = r
        for p in range(3):
            j.itx_stride[p] = S["stride"][p]
        j.mc.dst, j.mc.tmp, j.mc.mask, j.mc.px_tmp = p0, tmp, mask, (zeros("px_tmp", S["px_tmp_len"] * px) if S.get("px_tmp_len") else None)
        self.uploads = []          # (name, host array) re-sent per frame on the end-to-end path

        def rec(field_ptr, field_n, name, arr):
            if len(arr):
                setattr(j, field_ptr, up(name, arr)); setattr(j, field_n, len(arr))
                self.uploads.append((name, arr))
        if fused and "cfused" in S:      # compound blocks: both predictions + the combination in one kernel
            rec("d_pred", "n_pred", "pred", S["pred_single"])
            rec("d_cfused", "n_cfused", "cfused", S["cfused"])
            rec("d_cfused2", "n_cfused2", "cfused2", S["cfused2"])
        else:
            rec("d_pred", "n_pred", "pred", S["pred"])
            rec("d_comp", "n_comp", "comp", S["comp"])
            rec("d_comp2", "n_comp2", "comp2", S["comp2"])
        for name in ("warp", "blend", "blend2"):      # warped blocks; OBMC blends (stage 1: rows from above, stage 2: columns from the left)
            if name in S:
                rec("d_" + name, "n_" + name, name, S[name])
        for tx in range(19):
            a = S["itx"][tx]
            if len(a):
                j.d_itx[tx] = up("itx%d" % tx, a); j.n_itx[tx] = len(a)
                self.uploads.append(("itx%d" % tx, a))
        if compact:
            # the emitter ships coefficients 0 .. eob in scan order. Without intra records the inverse transforms read them
            # in place through per-block offsets (B200FrameJob.d_itx_coff); with intra records, whose kernels read the dense
            # buffer, the job zeroes + rebuilds it from the B200CoefBlock records. The dense buffer stays allocated either way
            # (b200_itx_add_frame takes it).
            from . import synth
            if expand is not None:
                cc, ex, coffs = expand
            else:
                cc, ex = synth.compact_coefs(S)
                coffs = itx_compact_offsets(S, ex)
            j.d_coef = zeros("coef", S["coefs"].nbytes)
            j.coef_bytes = S["coefs"].nbytes
            j.d_ccoef = up("ccoef", cc); self.uploads.append(("ccoef", cc))
            if (S.get("intra_tx") is None or not len(S["intra_tx"])) and coffs:
                allo = np.concatenate([coffs[tx] for tx in sorted(coffs)])       # one upload, one pointer per size into it
                base, pos = up("itx_coff", allo), 0
                self.uploads.append(("itx_coff", allo))
                for tx in sorted(coffs):
                    j.d_itx_coff[tx] = base + 4 * pos
                    pos += len(coffs[tx])
            elif len(ex):
                j.d_expand = up("expand", ex); j.n_expand = len(ex); self.uploads.append(("expand", ex))
        else:
            j.d_coef = up("coef", S["coefs"]); self.uploads.append(("coef", S["coefs"]))
        if len(S["mask"]) > 1:
            self.uploads.append(("mask", S["mask"]))
        if S.get("intra_tx") is not None and len(S["intra_tx"]):
            j.intra = intra_frame(S, p0, j.d_coef)
            it = j.intra
            it.grid = intra_grid
            it.mask = mask                            # blend masks of inter-intra (II) records
            nb = self.lib.b200_intra_scratch_bytes(C.byref(it)) if hasattr(self.lib, "b200_intra_scratch_bytes") else 1 << 22
            it.scratch = zeros("intra_scratch", nb)
            if intra_sb:     # superblock-granular schedule (records grouped by 64x64 superblock)
                j.d_intra = up("intra_tx", S["intra_tx_sb"]); j.n_intra = len(S["intra_tx_sb"])
                self.uploads.append(("intra_tx", S["intra_tx_sb"]))
                it.sb = up("intra_sb", S["intra_sb"]); it.n_sb = len(S["intra_sb"])
                it.sb_w, it.sb_h = S["intra_sb_grid"]
                self.uploads.append(("intra_sb", S["intra_sb"]))
            else:
                j.d_intra = up("intra_tx", S["intra_tx"]); j.n_intra = len(S["intra_tx"])
                self.uploads.append(("intra_tx", S["intra_tx"]))
                if S.get("done_init") is not None:       # a frame that mixes inter and intra blocks: inter cells are final already
                    it.done_init = up("done_init", S["done_init"])
                    self.uploads.append(("done_init", S["done_init"]))
        # post filters
        j.run_lf, j.run_cdef, j.run_lr = int(run_lf), int(run_cdef), int(run_lr)
        d_masks = up("masks", S["masks"]); self.uploads.append(("masks", S["masks"]))
        d_level = up("level", S["level"]); self.uploads.append(("level", S["level"]))
        d_lrm = up("lr_mask", S["lr_mask"]); self.uploads.append(("lr_mask", S["lr_mask"]))
        j.lf = lf_frame(S, p0, d_masks, d_level)
        j.cdef = cdef_frame(S, p0, p1, d_masks)
        j.lr = lr_frame(S, p1 if run_cdef else p0, p0, p2, d_lrm)
        self.out_name = "p2" if run_lr else ("p1" if run_cdef else "p0")
        if self.bands is not None and len(self.bands) > 1 and j.n_intra:
            # the pre-filter bottom rows of the bands, which the first row of intra records of the next band reads
            edge = zeros("intra_edge", self.lib.b200_band_edge_bytes(C.byref(j)))
            for b in self.bands:
                b.intra_edge = edge
        self.ref_name = self.out_name          # the picture later frames predict from (never the grained copy)
        if S.get("fg") is not None:
            # film grain goes into a separate display copy; the un-grained picture stays the reference picture
            j.fg = fg_frame(S, self.keep[self.out_name][1], zeros("p3", nbytes))
            j.run_fg = 1
            j.fg.scratch = zeros("fg_scratch", 256 * 1024)
            self.ref_name, self.out_name = self.out_name, "p3"
        self.job = j
        self._host = None

    # ---- device-resident run (records already in HBM) ----
    def run(self, stream=None):
        st = self.alloc.stream() if stream is None else stream
        self.lib.check(self.lib.b200_frame_run(C.byref(self.job), st), "b200_frame_run")

    # ---- band by band (b200_frame_run_band): same result as run(); what the frame pipeline over GPUs schedules ----
    def n_bands(self):
        return len(self.bands) if self.bands is not None else 0

    def run_band(self, k, stream=None):
        st = self.alloc.stream() if stream is None else stream
        self.lib.check(self.lib.b200_frame_run_band(C.byref(self.job), C.byref(self.bands[k]), st), "b200_frame_run_band")

    def run_band_phase(self, k, phases, stream=None):
        """1 = reconstruction of band k, 2 = its post filters (b200_frame_run_band_phase)"""
        st = self.alloc.stream() if stream is None else stream
        self.lib.check(self.lib.b200_frame_run_band_phase(C.byref(self.job), C.byref(self.bands[k]), phases, st), "b200_frame_run_band_phase")

    def run_bands(self, stream=None):
        for k in range(len(self.bands)):
            self.run_band(k, stream)

    def band_progress(self, k, plane):
        """rows of `plane` of the restored picture that are final after band k"""
        b = self.bands[k]
        return self.lib.b200_band_progress(C.byref(self.job), b.y1, b.last, plane)

    def set_refs(self, ptrs):
        for i, p in enumerate(ptrs):
            self.job.mc.ref[i] = p

    def output(self, name=None):
        return self.alloc.download(self.keep[name or self.out_name][0], self.S["pic"])

    def picture_ptr(self, name=None):
        return self.keep[name or self.out_name][1]

    # ---- end-to-end run: records from pinned host memory, picture back to the host ----
    def prepare_host(self):
        A = self.alloc
        ups = []
        self._host_keep = []
        for name, arr in self.uploads:
            t, p = A.pinned(arr)
            self._host_keep.append(t)
            ups.append((p, self.keep[name][1], arr.nbytes))
        out_t, out_p = A.pinned(np.zeros(self.S["pic"].nbytes, np.uint8))
        self._host_out = out_t
        self._ups = (_lib.Xfer * len(ups))(*[_lib.Xfer(h, d, n) for h, d, n in ups])
        self._downs = (_lib.Xfer * 1)(_lib.Xfer(out_p, self.keep[self.out_name][1], self.S["pic"].nbytes))
        self.h2d_bytes = sum(n for _, _, n in ups)
        self.d2h_bytes = self.S["pic"].nbytes

    def h2d_bytes_estimate(self):
        return sum(a.nbytes for _, a in self.uploads)

    def run_host(self, stream=None):
        if self._host is None:
            self.prepare_host(); self._host = True
        st = self.alloc.stream() if stream is None else stream
        self.lib.check(self.lib.b200_frame_run_host(C.byref(self.job), self._ups, len(self._ups), self._downs, 1, st),
                       "b200_frame_run_host")

    # frame-threaded variant: each FrameBuffers owns a stream; submit() returns at once, wait() joins
    def submit_host(self):
        if self._host is None:
            self.prepare_host(); self._host = True
        if getattr(self, "_own_stream", None) is None:
            self._own_stream = self.alloc.new_stream()
        self.lib.check(self.lib.b200_frame_submit_host(C.byref(self.job), self._ups, len(self._ups), self._downs, 1,
                                                       self._own_stream[1]), "b200_frame_submit_host")

    def wait(self):
        self.lib.check(self.lib.b200_frame_wait(self._own_stream[1]), "b200_frame_wait")

    def host_output(self):
        t = self._host_out
        a = t.numpy() if hasattr(t, "numpy") else t
        return a[:self.S["pic"].nbytes].view(self.S["pic"].dtype)
