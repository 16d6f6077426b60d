"""Whole-frame parity: reconstruction (prediction + compound + inverse transforms) followed by the
post-filter sweep (deblock -> CDEF -> loop restoration) over one synthetic inter frame, CUDA job vs the
oracle running the same stages in the same order on the CPU (each stage of the oracle is itself pinned
against the reference: test_itx / test_mc / test_loopfilter / test_cdef / test_looprestoration)."""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import synth, frame
import test_loopfilter as TLF
import test_cdef as TCD
import test_looprestoration as TLR


def oracle_frame(S, run_lf=True, run_cdef=True, run_lr=True):
    """returns dict of the pictures after each stage"""
    o = refs.oracle()
    bd = S["bd"]
    pic = np.zeros_like(S["pic"])
    tmp = np.zeros(S["tmp_len"], np.int16)
    mask = S["mask"].copy()
    fr = frame.mc_frame(S)
    keep = [r.copy() for r in S["refs"]]
    for i, r in enumerate(keep):
        fr.ref[i] = r.ctypes.data
    fr.dst, fr.tmp, fr.mask = pic.ctypes.data, tmp.ctypes.data, mask.ctypes.data
    px_tmp = np.zeros(S.get("px_tmp_len", 1), pic.dtype)
    fr.px_tmp = px_tmp.ctypes.data
    o.oracle_mc_batch(bd, C.byref(fr), S["pred"].ctypes.data, len(S["pred"]))
    if "warp" in S:
        o.oracle_mc_warp_batch(bd, C.byref(fr), S["warp"].ctypes.data, len(S["warp"]))
    o.oracle_mc_comp_batch(bd, C.byref(fr), S["comp"].ctypes.data, len(S["comp"]))
    o.oracle_mc_comp_batch(bd, C.byref(fr), S["comp2"].ctypes.data, len(S["comp2"]))
    for name in ("blend", "blend2"):            # OBMC: rows from the blocks above, then columns from the blocks to the left
        if name in S:
            o.oracle_mc_blend_batch(bd, C.byref(fr), S[name].ctypes.data, len(S[name]))
    st = (C.c_int32 * 3)(*S["stride"])
    coefs = S["coefs"].copy()
    for tx in range(19):
        a = S["itx"][tx]
        if len(a):
            assert o.oracle_itx_add_batch(bd, tx, a.ctypes.data, len(a), coefs.ctypes.data, pic.ctypes.data, st, 0) == 0
    if S.get("intra_tx") is not None and len(S["intra_tx"]):
        # intra blocks of a mixed frame: record by record, after every inter block is in the picture
        fr_i = frame.intra_frame(S, pic.ctypes.data, coefs.ctypes.data)
        fr_i.mask = mask.ctypes.data
        tx = np.ascontiguousarray(S["intra_tx_decode_order"])
        fn = o.oracle_intra_frame
        fn.restype = None
        fn(C.c_int(bd), C.byref(fr_i), C.c_void_p(tx.ctypes.data), C.c_int(len(tx)))
    out = {"recon": pic.copy()}
    S2 = dict(S); S2["pic"] = pic
    if run_lf:
        pic = TLF.lf_frame_oracle(S2); S2["pic"] = pic
    out["dbl"] = pic.copy()
    if run_cdef:
        cd = TCD.cdef_frame_oracle(S2)
    else:
        cd = pic
    out["cdef"] = cd
    if run_lr:
        S3 = dict(S2); S3["cdef"], S3["dbl"] = cd, pic
        out["lr"] = TLR.lr_frame_oracle(S3)
    if S.get("fg") is not None:
        import test_filmgrain as TFG
        out["fg"] = TFG.run_oracle_frame(frame.fg_frame(S, None, None), np.ascontiguousarray(out["lr"]), S["bpc"])
    return out


def check_frame(S, fb, exp):
    """the frame area of every stage's picture must match"""
    got_recon_dbl = fb.output("p0")
    assert TCD.frame_area_equal(S, got_recon_dbl, exp["dbl"]), "reconstruction + deblock mismatch"
    assert TCD.frame_area_equal(S, fb.output("p1"), exp["cdef"]), "cdef mismatch"
    assert TLR.picture_equal(S, fb.output("p2"), exp["lr"]), "loop restoration mismatch"
    if "fg" in exp:
        assert TLR.picture_equal(S, fb.output("p3"), exp["fg"]), "film grain mismatch"


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 200, 136, 1, 1), (10, 136, 72, 1, 1)])
def test_emu_frame(bpc, W, H, ssh, ssv):
    S = synth.make_inter_frame(np.random.default_rng(600 + bpc), bpc, W, H, ssh, ssv, film_grain=bpc > 8)
    exp = oracle_frame(S)
    assert (exp["recon"] != 0).mean() > 0.3 and not np.array_equal(exp["recon"], exp["dbl"])
    fb = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    fb.run()
    check_frame(S, fb, exp)
    fbf = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc(), fused=True)     # fused compound prediction
    assert fbf.job.n_cfused > 0 and fbf.job.n_comp == 0
    fbf.run()
    check_frame(S, fbf, exp)
    # the host-buffer path must give the same picture
    fb2 = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    fb2.run_host()
    last = exp["fg"] if "fg" in exp else exp["lr"]
    assert TLR.picture_equal(S, fb2.host_output(), last)
    fb3 = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc(), compact=True)   # compact coefficient upload
    assert fb3.h2d_bytes_estimate() < fb2.h2d_bytes_estimate()
    fb3.submit_host(); fb3.wait()
    assert TLR.picture_equal(S, fb3.host_output(), last)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 640, 360, 1, 1), (10, 648, 368, 1, 1), (12, 328, 200, 0, 0), (8, 1920, 1080, 1, 1)])
def test_gpu_frame(bpc, W, H, ssh, ssv):
    S = synth.make_inter_frame(np.random.default_rng(610 + bpc + W), bpc, W, H, ssh, ssv, film_grain=bpc > 8)
    exp = oracle_frame(S)
    fb = frame.FrameBuffers(S)
    fb.run()
    fb.alloc.sync()
    check_frame(S, fb, exp)
    fbf = frame.FrameBuffers(S, fused=True, compact=True)
    fbf.run()
    fbf.alloc.sync()
    check_frame(S, fbf, exp)
    last = exp["fg"] if "fg" in exp else exp["lr"]
    fb2 = frame.FrameBuffers(S)
    fb2.run_host()
    assert TLR.picture_equal(S, fb2.host_output(), last)
    # two frames in flight on their own streams (frame-threaded end-to-end path)
    fb3, fb4 = frame.FrameBuffers(S, compact=True), frame.FrameBuffers(S, compact=True)
    for _ in range(3):
        fb3.submit_host(); fb4.submit_host()
        fb3.wait(); fb4.wait()
    assert TLR.picture_equal(S, fb3.host_output(), last) and TLR.picture_equal(S, fb4.host_output(), last)


def _banded_variants(S, **kw):
    """band-sliced jobs of frame S that must all reproduce the whole-frame job (b200_frame_run_band)"""
    out = []
    for rows, opts in ((64, {}), (128, dict(compact=True)), (64, dict(fused=True, compact=True))):
        fb = frame.FrameBuffers(S, band_rows=rows, **opts, **kw)
        assert fb.n_bands() == -(-S["H"] // rows)
        out.append(fb)
    return out


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 200, 264, 1, 1), (10, 136, 200, 1, 1), (8, 72, 136, 0, 0)])
def test_emu_frame_bands(bpc, W, H, ssh, ssv):
    """a frame cut into 64 / 128-row bands (reconstruction, deblock, and the CDEF / LR / grain rows each band makes final)
    equals the whole-frame job and the oracle; the progress a band reports is really final at that point"""
    S = synth.make_inter_frame(np.random.default_rng(630 + bpc + H), bpc, W, H, ssh, ssv, film_grain=bpc > 8)
    exp = oracle_frame(S)
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    for fb in _banded_variants(S, **kw):
        fb.run_bands()
        check_frame(S, fb, exp)
    # progress: after band k the rows b200_band_progress reports must already hold their final values
    fb = frame.FrameBuffers(S, band_rows=64, **kw)
    final = exp["lr"]
    hs = [S["H"], (S["H"] + ssv) >> ssv, (S["H"] + ssv) >> ssv]
    ws = [S["W"], (S["W"] + ssh) >> ssh, (S["W"] + ssh) >> ssh]
    prev = [0, 0, 0]
    for k in range(fb.n_bands()):
        fb.run_band(k)
        got = fb.output("p2")
        for pl in range(3):
            rows = fb.band_progress(k, pl)
            assert prev[pl] <= rows <= hs[pl]
            prev[pl] = rows
            o, st = S["off"][pl], S["stride"][pl]
            a = got[o:o + hs[pl] * st].reshape(hs[pl], st)[:rows, :ws[pl]]
            b = final[o:o + hs[pl] * st].reshape(hs[pl], st)[:rows, :ws[pl]]
            assert np.array_equal(a, b), "band %d plane %d: rows reported final are not" % (k, pl)
    assert prev == hs
    # the rows a band's predictions read from each reference stay inside the picture and grow with the band
    assert (fb.band_need[:, :, 0] <= S["H"]).all() and (fb.band_need[-1].max() > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 640, 360, 1, 1), (10, 648, 520, 1, 1)])
def test_gpu_frame_bands(bpc, W, H, ssh, ssv):
    S = synth.make_inter_frame(np.random.default_rng(640 + bpc), bpc, W, H, ssh, ssv, film_grain=bpc > 8)
    exp = oracle_frame(S)
    for fb in _banded_variants(S):
        fb.run_bands()
        fb.alloc.sync()
        check_frame(S, fb, exp)


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H", [(8, 264, 200), (10, 200, 136)])
def test_emu_mixed_frame(bpc, W, H):
    """an inter frame in which a share of the blocks is intra coded (what real inter frames contain): the intra kernel runs
    on top of the inter stages from a pre-marked done map; equals the oracle, whole-frame and as a single band"""
    S = synth.make_inter_frame(np.random.default_rng(650 + bpc), bpc, W, H, p_intra=0.25, film_grain=bpc > 8)
    assert len(S["intra_tx"]) > 30 and S["intra_waves"] > 2
    exp = oracle_frame(S)
    S0 = dict(S); S0["intra_tx"] = S["intra_tx"][:0]
    assert not np.array_equal(exp["recon"], oracle_frame(S0)["recon"])
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    fb = frame.FrameBuffers(S, **kw)
    fb.run()
    check_frame(S, fb, exp)
    fb1 = frame.FrameBuffers(S, band_rows=-(-H // 64) * 64, compact=True, **kw)      # the pipeline's whole-frame band
    assert fb1.n_bands() == 1
    fb1.run_bands()
    check_frame(S, fb1, exp)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H", [(8, 648, 520), (10, 1288, 720)])
def test_gpu_mixed_frame(bpc, W, H):
    S = synth.make_inter_frame(np.random.default_rng(660 + bpc), bpc, W, H, p_intra=0.15, film_grain=bpc > 8)
    exp = oracle_frame(S)
    for kw in (dict(), dict(band_rows=-(-H // 64) * 64, compact=True)):
        fb = frame.FrameBuffers(S, **kw)
        fb.run_bands() if kw else fb.run()
        fb.alloc.sync()
        check_frame(S, fb, exp)


MOTION = dict(p_obmc=0.2, p_warp=0.15, p_ii=0.15)


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,p_intra", [(8, 264, 200, 0.1), (10, 200, 136, 0.0), (8, 328, 264, 0.0)])
def test_emu_motion_mode_frame(bpc, W, H, p_intra):
    """the remaining inter tools of real frames in the synthetic records: overlapped block motion compensation (op-2 predictions
    + blend_h / blend_v stages), affine warps (8x8 records) and inter-intra blends (II + RESID records of the intra machine),
    alone and next to intra blocks; equals the oracle; without intra-machine records also cut into bands"""
    S = synth.make_inter_frame(np.random.default_rng(670 + bpc + H), bpc, W, H, p_intra=p_intra, film_grain=bpc > 8, **MOTION)
    assert len(S["warp"]) > 10 and len(S["blend"]) > 10 and len(S["blend2"]) > 10 and (S["intra_tx"]["mode"] == 15).sum() > 5
    assert (S["intra_tx"]["mode"] == 16).sum() > 5 and (S["pred"]["op"] == 2).sum() > 20
    exp = oracle_frame(S)
    for drop in ("warp", "blend", "blend2"):         # every list matters
        S0 = dict(S); S0[drop] = S[drop][:0]
        assert not np.array_equal(exp["recon"], oracle_frame(S0)["recon"]), drop
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    fb = frame.FrameBuffers(S, **kw)
    fb.run()
    check_frame(S, fb, exp)
    fb1 = frame.FrameBuffers(S, band_rows=-(-H // 64) * 64, compact=True, **kw)
    fb1.run_bands()
    check_frame(S, fb1, exp)


@pytest.mark.emu
def test_emu_mixed_frame_whose_inter_blocks_are_all_skipped():
    """found by tools/fuzz_frames.py: no inter transform block at all, coefficients only in the intra blocks — the band plan of the
    whole-frame band (compact upload) used to fail on the empty list"""
    S = synth.make_inter_frame(np.random.default_rng(702), 8, 200, 136, p_skip=0.2, p_intra=0.3)
    S["itx"] = {t: a[:0] for t, a in S["itx"].items()}          # as if every inter block had been skipped
    assert (S["intra_tx"]["eob"] >= 0).sum() > 10
    exp = oracle_frame(S)
    fb = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc(), band_rows=192, compact=True)
    fb.run_bands()
    check_frame(S, fb, exp)


@pytest.mark.emu
def test_emu_motion_mode_frame_bands():
    """OBMC and warp records sorted into 64-row bands (inter-intra needs the intra machine: whole-frame band only)"""
    S = synth.make_inter_frame(np.random.default_rng(681), 8, 264, 328, p_obmc=0.25, p_warp=0.2)
    assert "intra_tx" not in S and len(S["warp"]) and len(S["blend"])
    exp = oracle_frame(S)
    for rows in (64, 128):
        fb = frame.FrameBuffers(S, lib=refs.emu_lib(), alloc=frame.NumpyAlloc(), band_rows=rows, compact=True)
        assert fb.n_bands() > 2
        fb.run_bands()
        check_frame(S, fb, exp)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,p_intra", [(8, 648, 520, 0.1), (10, 1288, 720, 0.05)])
def test_gpu_motion_mode_frame(bpc, W, H, p_intra):
    S = synth.make_inter_frame(np.random.default_rng(690 + bpc), bpc, W, H, p_intra=p_intra, film_grain=bpc > 8, **MOTION)
    exp = oracle_frame(S)
    for kw in (dict(), dict(band_rows=-(-H // 64) * 64, compact=True)):
        fb = frame.FrameBuffers(S, **kw)
        fb.run_bands() if kw else fb.run()
        fb.alloc.sync()
        check_frame(S, fb, exp)
    S = synth.make_inter_frame(np.random.default_rng(691 + bpc), bpc, W, H, p_obmc=0.25, p_warp=0.2)
    exp = oracle_frame(S)
    fb = frame.FrameBuffers(S, band_rows=128, compact=True)
    fb.run_bands()
    fb.alloc.sync()
    check_frame(S, fb, exp)


def reference_frame(S):
    """the same job through the reference's own functions on the CPU (oracle/refdriver: refdrv_frame_run)"""
    fb = frame.FrameBuffers(S, lib=object(), alloc=frame.NumpyAlloc())
    fn = refs.ref().refdrv_frame_run_8bpc if S["bpc"] == 8 else refs.ref().refdrv_frame_run_16bpc
    fn(C.byref(fb.job))
    return fb


@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 328, 200, 1, 1), (10, 264, 136, 1, 1), (12, 136, 200, 0, 0)])
def test_oracle_frame_vs_reference_functions(bpc, W, H, ssh, ssv):
    """whole-frame pin of the oracle: every stage run by dav1d's own C functions / frame drivers"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = synth.make_inter_frame(np.random.default_rng(620 + bpc), bpc, W, H, ssh, ssv, film_grain=bpc > 8)
    exp = oracle_frame(S)
    fb = reference_frame(S)
    check_frame(S, fb, exp)
    # ... and with intra blocks, OBMC, warps and inter-intra blends in the records
    S = synth.make_inter_frame(np.random.default_rng(625 + bpc), bpc, W, H, ssh, ssv, p_intra=0.1, **MOTION)
    S["intra_tx"] = S["intra_tx_decode_order"]
    exp = oracle_frame(S)
    fb = reference_frame(S)
    check_frame(S, fb, exp)
