"""Parity tests for intra-frame reconstruction (device-side dav1d_prepare_intra_edges + predictors + itx in a
dependency-driven kernel; include/b200av1.h B200IntraTx / b200_intra_frame).

The oracle restatement (oracle/intra.c) is pinned against the reference's own dav1d_prepare_intra_edges,
intra_pred / cfl_ac / cfl_pred and itxfm_add functions driven record by record (oracle/refdriver); the CUDA
kernel is then checked against the oracle, with the records in decode order and in wavefront order.
"""
import ctypes as C
import os
import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, synth, frame

CASES = [(8, 136, 72, 1, 1), (10, 200, 136, 1, 1), (12, 72, 136, 0, 0), (8, 264, 136, 1, 0)]


def run_cpu(fn, S, order="intra_tx"):
    pic = np.zeros_like(S["pic"]); coefs = S["coefs"].copy()
    fr = frame.intra_frame(S, pic.ctypes.data, coefs.ctypes.data)
    tx = np.ascontiguousarray(S[order])
    fn.restype = None
    fn(C.c_int(S["bd"]), C.byref(fr), C.c_void_p(tx.ctypes.data), C.c_int(len(tx)))
    assert np.array_equal(coefs, S["coefs"])
    return pic


def oracle_intra(S, order="intra_tx"):
    return run_cpu(refs.oracle().oracle_intra_frame, S, order)


def reference_intra(S, order="intra_tx"):
    r = refs.ref()
    return run_cpu(r.refdrv_intra_frame_8bpc if S["bpc"] == 8 else r.refdrv_intra_frame_16bpc, S, order)


def planes_equal(S, a, b):
    ssh, ssv = [0, S["ss_hor"], S["ss_hor"]], [0, S["ss_ver"], S["ss_ver"]]
    for p in range(3):
        w, h = S["W"] >> ssh[p], S["H"] >> ssv[p]
        st, o = S["stride"][p], S["off"][p]
        va = a[o:o + st * h].reshape(h, st)[:, :w]; vb = b[o:o + st * h].reshape(h, st)[:, :w]
        if not np.array_equal(va, vb):
            ys, xs = np.nonzero(va != vb)
            return False, (p, int(ys[0]), int(xs[0]), int(va[ys[0], xs[0]]), int(vb[ys[0], xs[0]]), len(ys))
    return True, None


@pytest.mark.parametrize("bpc,W,H,ssh,ssv", CASES)
def test_oracle_intra_vs_reference_functions(bpc, W, H, ssh, ssv):
    if not refs.have_ref():
        pytest.skip("oracle/_ref not built")
    S = synth.make_intra_frame(np.random.default_rng(700 + bpc + W), bpc, W, H, ssh, ssv)
    a = reference_intra(S); b = oracle_intra(S)
    ok, where = planes_equal(S, a, b)
    assert ok, where
    assert (a != 0).mean() > 0.15
    # any topological order gives the same picture: decode order vs wavefront order
    c = oracle_intra(S, "intra_tx_decode_order")
    ok, where = planes_equal(S, a, c)
    assert ok, where
    if W * H >= 200 * 136:
        modes = set(S["intra_tx"]["mode"].tolist())
        assert modes >= set(range(13)) | {synth.MODE_CFL, synth.MODE_FILTER}, modes


def run_lib(lib, alloc, S, order="intra_tx", compact=False, sb=False):
    S2 = dict(S); S2["intra_tx"] = np.ascontiguousarray(S[order])
    fb = frame.FrameBuffers(S2, lib=lib, alloc=alloc, run_lf=False, run_cdef=False, run_lr=False, compact=compact, intra_sb=sb)
    fb.run()
    fb.alloc.sync()
    return fb.output("p0")


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", CASES)
def test_emu_intra_frame(bpc, W, H, ssh, ssv):
    S = synth.make_intra_frame(np.random.default_rng(720 + bpc + W), bpc, W, H, ssh, ssv)
    exp = oracle_intra(S)
    got = run_lib(refs.emu_lib(), frame.NumpyAlloc(), S)
    ok, where = planes_equal(S, exp, got)
    assert ok, where
    got = run_lib(refs.emu_lib(), frame.NumpyAlloc(), S, compact=True)      # coefficients shipped in scan order up to eob
    ok, where = planes_equal(S, exp, got)
    assert ok, where
    got = run_lib(refs.emu_lib(), frame.NumpyAlloc(), S, sb=True)            # superblock-granular schedule
    ok, where = planes_equal(S, exp, got)
    assert ok, ("sb", where)


IBC_CASES = [(8, 328, 264, 1, 1), (10, 264, 200, 1, 1), (12, 200, 264, 0, 0), (8, 264, 264, 1, 0)]


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", IBC_CASES)
def test_intra_block_copy_oracle_reference_and_kernel(bpc, W, H, ssh, ssv):
    """intra block copy records (B200_INTRA_MODE_IBC + RESID): blocks copied with the bilinear put from arbitrary (unaligned,
    odd-vector) positions in the superblock rows above; the oracle's restatement, dav1d's own emu_edge + mc[BILINEAR] and the
    intra machine (wavefront order and decode order) give the same picture"""
    S = synth.make_intra_frame(np.random.default_rng(740 + bpc + W), bpc, W, H, ssh, ssv, p_ibc=0.3)
    t = S["intra_tx"]
    assert (t["mode"] == synth.MODE_IBC).sum() > 12 and (t["mode"] == synth.MODE_RESID).sum() > 12
    if ssh:
        assert ((t["mode"] == synth.MODE_IBC) & (t["cfl_w_pad"] == 8)).sum() > 3, "no half-sample chroma phase"
    exp = oracle_intra(S)
    S0 = dict(S); S0["intra_tx"] = t[t["mode"] != synth.MODE_IBC]
    assert not planes_equal(S, exp, oracle_intra(S0))[0]                   # the copies matter
    if refs.have_ref():
        ok, where = planes_equal(S, reference_intra(S), exp)
        assert ok, ("reference", where)
    for order in ("intra_tx", "intra_tx_decode_order"):
        got = run_lib(refs.emu_lib(), frame.NumpyAlloc(), S, order=order, compact=order == "intra_tx")
        ok, where = planes_equal(S, exp, got)
        assert ok, (order, where)


def check_cta_kernel():
    """The CTA-per-block kernel against the oracle: an intra block copy frame, an intra frame in wavefront and in decode
    order, a mixed PAL / II / RESID frame. Runs in a process started with B200_INTRA_CTA=1 (test_emu_intra_cta_kernel)."""
    emu = refs.emu_lib()
    bpc, W, H, ssh, ssv = IBC_CASES[0]
    S = synth.make_intra_frame(np.random.default_rng(740 + bpc + W), bpc, W, H, ssh, ssv, p_ibc=0.3)
    ok, where = planes_equal(S, oracle_intra(S), run_lib(emu, frame.NumpyAlloc(), S))
    assert ok, ("ibc", where)
    bpc, W, H, ssh, ssv = CASES[1]
    S = synth.make_intra_frame(np.random.default_rng(720 + bpc + W), bpc, W, H, ssh, ssv)
    exp = oracle_intra(S)
    for order in ("intra_tx", "intra_tx_decode_order"):
        ok, where = planes_equal(S, exp, run_lib(emu, frame.NumpyAlloc(), S, order=order))
        assert ok, (order, where)
    bpc, W, H, ssh, ssv = CASES[0]
    rng = np.random.default_rng(900 + bpc + W)
    S = make_mixed(synth.make_intra_frame(rng, bpc, W, H, ssh, ssv), rng)
    ok, where = planes_equal(S, run_mixed(refs.oracle().oracle_intra_frame, S), run_mixed(None, S, emu=emu))
    assert ok, ("mixed", where)


@pytest.mark.emu
def test_emu_intra_cta_kernel():
    """the CTA-per-block kernel is chosen once per process from B200_INTRA_CTA, so it is checked in a process of its own"""
    import subprocess, sys
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_intra\n"
            "test_intra.check_cta_kernel()\n"
            "print('RESULT ok')\n") % (refs.ROOT, os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800,
                         env=dict(os.environ, B200_INTRA_CTA="1"))
    assert "RESULT ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


def check_batch(lib, alloc_fn, n, bpc=8, W=136, H=72, with_lf=True):
    """n different frames through b200_frame_run_batch (one intra launch for all of them) against the oracle"""
    import test_loopfilter as TLF
    import test_cdef as TCD
    Ss = [synth.make_intra_frame(np.random.default_rng(780 + k), bpc, W, H) for k in range(n)]
    fbs = [frame.FrameBuffers(S, lib=lib, alloc=alloc_fn(), run_lf=with_lf, run_cdef=False, run_lr=False, compact=k & 1, intra_grid=7, intra_sb=bool(k & 2))
           for k, S in enumerate(Ss)]
    frame.run_batch(fbs)
    fbs[0].alloc.sync()
    for S, fb in zip(Ss, fbs):
        rec = oracle_intra(S)
        if with_lf:
            S2 = dict(S); S2["pic"] = rec
            assert TCD.frame_area_equal(S, fb.output("p0"), TLF.lf_frame_oracle(S2))
        else:
            ok, where = planes_equal(S, rec, fb.output("p0"))
            assert ok, where


@pytest.mark.emu
def test_emu_intra_batch():
    check_batch(refs.emu_lib(), frame.NumpyAlloc, 4)


@pytest.mark.gpu
def test_gpu_intra_batch():
    check_batch(_lib.get_lib(), frame.TorchAlloc, 30, W=264, H=136)      # > 24 frames: two launches


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", CASES + [(8, 1920, 1080, 1, 1), (10, 1280, 720, 1, 1)])
def test_gpu_intra_frame(bpc, W, H, ssh, ssv):
    S = synth.make_intra_frame(np.random.default_rng(740 + bpc + W), bpc, W, H, ssh, ssv)
    exp = oracle_intra(S)
    for order in ("intra_tx", "intra_tx_decode_order"):
        got = run_lib(_lib.get_lib(), None, S, order, compact=order == "intra_tx")
        ok, where = planes_equal(S, exp, got)
        assert ok, (order, where)
    got = run_lib(_lib.get_lib(), None, S, sb=True, compact=True)
    ok, where = planes_equal(S, exp, got)
    assert ok, ("sb", where)


@pytest.mark.gpu
def test_gpu_intra_frame_with_deblock():
    """BASELINE configs[1]: intra reconstruction followed by the deblocking sweeps, whole job through the C ABI"""
    import test_loopfilter as TLF
    S = synth.make_intra_frame(np.random.default_rng(760), 8, 640, 360)
    rec = oracle_intra(S)
    S2 = dict(S); S2["pic"] = rec
    exp = TLF.lf_frame_oracle(S2)
    fb = frame.FrameBuffers(S, run_cdef=False, run_lr=False)
    fb.run(); fb.alloc.sync()
    import test_cdef as TCD
    assert TCD.frame_area_equal(S, fb.output("p0"), exp)


# ---- record kinds of mixed frames: palette blocks, inter-intra blends, residual-only transform blocks -----------------
def make_mixed(S, rng, p_pal=0.2, p_ii=0.25):
    """Turns a share of the transform blocks of a synthetic intra frame into PAL / II records (+ a RESID record when the
    block had a residual), the way the dav1d hooks emit palette and inter-intra blocks (include/b200av1.h). The picture
    starts as random pixels: what the prediction stage would have left in an inter-intra block."""
    px = 2 if S["bpc"] > 8 else 1
    bd = S["bd"]
    src = S["intra_tx_decode_order"]
    out, pal, mask = [], bytearray(), bytearray()
    from dav1d_b200 import levels as L
    for r in src:
        w, h = L.TX_W[r["tx"]], L.TX_H[r["tx"]]
        u = rng.random()
        if r["mode"] == synth.MODE_CFL or u >= p_pal + p_ii:
            out.append(r.copy()); continue
        head = r.copy()
        head["eob"] = -1; head["flags"] = int(r["flags"]) & 3; head["angle_flags"] = 0
        head["cfl_alpha"] = 1 if r["eob"] >= 0 else 0
        if u < p_pal:
            head["mode"], head["flags"], head["angle"] = 17, 0, 0
            while len(pal) % 16:
                pal.append(0)
            head["luma_off"] = len(pal)
            cols = rng.integers(0, bd + 1, 8).astype(np.uint16 if px == 2 else np.uint8)
            idx = rng.integers(0, 8, (h, w)).astype(np.uint8)
            pal += cols.tobytes() + (idx[:, 0::2] | (idx[:, 1::2] << 4)).astype(np.uint8).tobytes()
        else:
            head["mode"] = 15
            head["angle"] = int(rng.choice([0, 1, 2, 9]))            # DC / VERT / HOR / SMOOTH
            head["luma_off"] = len(mask)
            mask += rng.integers(0, 65, w * h).astype(np.uint8).tobytes()
        out.append(head)
        if r["eob"] >= 0:
            res = r.copy()
            res["mode"], res["flags"], res["angle"], res["angle_flags"] = 16, 0, 0, 0
            out.append(res)
    S2 = dict(S)
    S2["mixed_tx"] = np.array(out, dtype=src.dtype)
    S2["mixed_pal"] = np.frombuffer(bytes(pal) + b"\0" * 16, np.uint8).copy()
    S2["mixed_mask"] = np.frombuffer(bytes(mask) + b"\0" * 16, np.uint8).copy()
    S2["mixed_pic0"] = rng.integers(0, bd + 1, len(S["pic"])).astype(S["pic"].dtype)
    return S2


def run_mixed(fn, S, emu=None):
    pic = S["mixed_pic0"].copy(); coefs = S["coefs"].copy()
    fr = frame.intra_frame(S, pic.ctypes.data, coefs.ctypes.data)
    fr.mask, fr.pal = S["mixed_mask"].ctypes.data, S["mixed_pal"].ctypes.data
    tx = np.ascontiguousarray(S["mixed_tx"])
    if emu is None:
        fn.restype = None
        fn(C.c_int(S["bd"]), C.byref(fr), C.c_void_p(tx.ctypes.data), C.c_int(len(tx)))
    else:
        scratch = np.zeros(int(emu.b200_intra_scratch_bytes(C.byref(fr))) + 256, np.uint8)
        fr.scratch = scratch.ctypes.data
        emu.check(emu.b200_intra_frame(S["bd"], C.byref(fr), tx.ctypes.data, len(tx), None), "b200_intra_frame")
    return pic


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", CASES)
def test_mixed_record_kinds_oracle_reference_and_kernel(bpc, W, H, ssh, ssv):
    """PAL / II / RESID records: oracle restatement == the reference's own pal_pred / prepare_intra_edges / intra_pred /
    blend / itxfm_add driven record by record == the kernel (host emulator build)"""
    if not refs.have_ref():
        pytest.skip("oracle/_ref not built")
    rng = np.random.default_rng(900 + bpc + W)
    S = make_mixed(synth.make_intra_frame(rng, bpc, W, H, ssh, ssv), rng)
    kinds = set(S["mixed_tx"]["mode"].tolist())
    assert {15, 16, 17} <= kinds, kinds
    r = refs.ref()
    a = run_mixed(r.refdrv_intra_frame_8bpc if bpc == 8 else r.refdrv_intra_frame_16bpc, S)
    b = run_mixed(refs.oracle().oracle_intra_frame, S)
    ok, where = planes_equal(S, a, b)
    assert ok, ("oracle vs reference", where)
    c = run_mixed(None, S, emu=refs.emu_lib())
    ok, where = planes_equal(S, b, c)
    assert ok, ("kernel vs oracle", where)
