"""Inverse transforms fed straight from the compact coefficient stream (B200FrameJob.d_itx_coff).

A frame job without intra records whose transform blocks carry offsets into the compact stream (per block the coefficients
0 .. eob in the scan order of its class) runs the transforms on that stream: the dense coefficient plane is neither zeroed
nor expanded into, nor read. The arithmetic after the load is the dense form's, so the pictures must be byte-identical to
the dense job and to the oracle:

  * every transform size x every defined transform type (WHT_WHT included), eob = 0, 1, small and the whole coded region,
    coefficients over the full dequantised range, 8 / 10 / 12 bit;
  * whole frames and 64- / 192-row bands, post filters on;
  * jobs with intra records keep the dense path (the intra kernels read the dense plane) even when offsets are given.

Each compact job runs with the dense plane filled with a sentinel: it must come out unchanged (no memset, no expansion)
while the picture stays right (nothing read it). The launch counter shows the expansion launches that are gone.
"""
import ctypes as C

import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, frame, synth
from dav1d_b200 import levels as L
import test_coef_range as CR
import test_frame as TF
import test_itx as TX

SENTINEL = 0x5A


def oracle_prototypes():
    """Declare the prototypes of the prediction batches that test_frame.oracle_frame calls with raw addresses. Without them
    ctypes passes each address as a C int, keeping its low 32 bits only, so a buffer allocated above 4 GB (mmap, another
    arena) is read at a wrong address."""
    o = refs.oracle()
    for name in ("oracle_mc_batch", "oracle_mc_comp_batch", "oracle_mc_blend_batch", "oracle_mc_warp_batch"):
        fn = getattr(o, name)
        fn.argtypes, fn.restype = [C.c_int, C.c_void_p, C.c_void_p, C.c_int], None


def compact_batch(rng, bpc, tx):
    """blocks of size tx over a random picture (test_itx.make_batch layout): every defined type with eob 0, 1, small and
    full, coefficients up to eob (in the scan order of the type's class) uniform over the legal range or at its ends"""
    types = [tp for tp in range(17) if L.itx_defined(tx, tp)]
    sw, sh = L.tx_coef_dims(tx)
    n = sw * sh
    eobs = [0, 1, int(rng.integers(2, min(n, 24))), n - 1]
    cases = [(tp, e) for tp in types for e in eobs]
    blocks, coefs, pic, stride = TX.make_batch(rng, bpc, tx, len(cases))
    hi, lo = CR.cf_max(bpc), -CR.cf_max(bpc) - 1
    for i, (tp, eob) in enumerate(cases):
        order = CR.scan_order(tx, tp)
        c = np.zeros(n, np.int64)
        pick = rng.random()
        if pick < 0.25:
            c[order[:eob + 1]] = hi
        elif pick < 0.5:
            c[order[:eob + 1]] = lo
        else:
            c[order[:eob + 1]] = rng.integers(lo, hi + 1, eob + 1)
        if c[order[eob]] == 0:
            c[order[eob]] = 1
        off = int(blocks[i]["coef_off"])
        coefs[off:off + n] = c
        blocks[i]["eob"], blocks[i]["txtp"] = eob, tp
    bdmax = (1 << bpc) - 1
    m = rng.random(pic.shape) < 0.33
    pic[m] = rng.choice(np.array([0, bdmax], pic.dtype), int(m.sum()))
    return blocks, coefs, pic, stride


def run_itx_job(lib, bpc, tx, blocks, pic, stride, coefs=None, compact=None):
    """a frame job holding only the transform blocks of one size: dense (coefs) or compact ((stream, offsets))"""
    j = _lib.FrameJob()
    j.bitdepth_max = (1 << bpc) - 1
    j.d_itx[tx], j.n_itx[tx] = blocks.ctypes.data, len(blocks)
    j.mc.dst = pic.ctypes.data
    for p in range(3):
        j.itx_stride[p] = stride
    keep = [blocks, pic]
    if compact is not None:
        cc, coff = compact
        dense = np.full(coefs.shape, SENTINEL, coefs.dtype)
        j.d_ccoef, j.d_itx_coff[tx], j.d_coef = cc.ctypes.data, coff.ctypes.data, dense.ctypes.data
        keep += [cc, coff, dense]
    else:
        j.d_coef = coefs.ctypes.data
    before = lib.b200_launch_count()
    lib.check(lib.b200_frame_run(C.byref(j), None), "b200_frame_run")
    if compact is not None:
        assert (dense == SENTINEL).all(), "the compact job touched the dense coefficient plane"
    return lib.b200_launch_count() - before


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_compact_itx_every_size_and_type(bpc):
    lib = refs.emu_lib()
    rng = np.random.default_rng(900 + bpc)
    bdmax = (1 << bpc) - 1
    for tx in range(19):
        blocks, coefs, pic, stride = compact_batch(rng, bpc, tx)
        exp, ec = pic.copy(), coefs.copy()        # (named: the oracle reads them through raw pointers)
        st = (C.c_int32 * 3)(stride, stride, stride)
        assert refs.oracle().oracle_itx_add_batch(bdmax, tx, blocks.ctypes.data, len(blocks), ec.ctypes.data,
                                                  exp.ctypes.data, st, 0) == 0
        dense = pic.copy()
        assert run_itx_job(lib, bpc, tx, blocks, dense, stride, coefs=coefs.copy()) == 1
        S = {"coefs": coefs, "itx": {t: blocks if t == tx else blocks[:0] for t in range(19)}}
        cc, ex = synth.compact_coefs(S)
        assert set(ex["tx_class"].tolist()) >= ({0, 1, 2} if L.itx_defined(tx, L.V_DCT) else {0})
        coff = frame.itx_compact_offsets(S, ex)[tx]
        got = pic.copy()
        assert run_itx_job(lib, bpc, tx, blocks, got, stride, coefs=coefs, compact=(cc, coff)) == 1
        for name, a in (("dense job", dense), ("compact job", got)):
            if not np.array_equal(a, exp):
                bad = int(np.nonzero((a != exp).reshape(-1))[0][0])
                i = int(np.nonzero(blocks["dst_off"] <= bad)[0][-1]) if (blocks["dst_off"] <= bad).any() else -1
                raise AssertionError("%s %dbpc tx=%s: pixel %d differs from the oracle (block %d, txtp %d, eob %d)" % (
                    name, bpc, L.TX_NAMES[tx], bad, i, int(blocks["txtp"][i]), int(blocks["eob"][i])))


def legacy_compact(fb, S, rows):
    """fb (a compact job without intra records) turned back into the dense form of the compact upload: no offsets, the
    B200CoefBlock records (band-sorted for a banded job), so that the job zeroes and expands the dense plane"""
    ex = frame.band_plan(S, rows, compact=True)[3][1] if rows else synth.compact_coefs(S)[1]
    ex = np.ascontiguousarray(ex)
    fb.keep["expand_legacy"] = fb.alloc.upload(ex)
    for tx in range(19):
        fb.job.d_itx_coff[tx] = None
    fb.job.d_expand, fb.job.n_expand = fb.keep["expand_legacy"][1], len(ex)
    return fb


def check_compact_frame(S, kw, rows_list=(0, 64, 192), sentinel=None):
    lib = kw.get("lib") or _lib.get_lib()
    oracle_prototypes()
    exp = TF.oracle_frame(S)
    fb = frame.FrameBuffers(S, **kw)
    fb.run()
    fb.alloc.sync()
    TF.check_frame(S, fb, exp)
    dense_out = fb.output("p2")

    def count(fn):
        fb.alloc.sync()
        b = lib.b200_launch_count()
        fn()
        fb.alloc.sync()
        return lib.b200_launch_count() - b
    for rows in rows_list:
        fbc = frame.FrameBuffers(S, compact=True, band_rows=rows, **kw)
        j = fbc.job
        assert j.n_expand == 0 and all(j.d_itx_coff[tx] for tx in range(19) if j.n_itx[tx])
        names = [n for n, _ in fbc.uploads]
        assert "itx_coff" in names and "expand" not in names
        sentinel(fbc.keep["coef"][0], fill=True)
        n_new = count(fbc.run_bands if rows else fbc.run)
        assert sentinel(fbc.keep["coef"][0]), "compact job (band_rows %d) zeroed or filled the dense coefficient plane" % rows
        TF.check_frame(S, fbc, exp)
        assert np.array_equal(fbc.output("p2"), dense_out)
        fbl = legacy_compact(frame.FrameBuffers(S, compact=True, band_rows=rows, **kw), S, rows)
        n_old = count(fbl.run_bands if rows else fbl.run)
        TF.check_frame(S, fbl, exp)
        # one coef_expand launch less per band that has transform blocks
        n_bands = sum(1 for b in fbl.bands if b.expand[1] > 0) if rows else 1
        assert n_old - n_new == n_bands, (rows, n_old, n_new, n_bands)


def numpy_sentinel(a, fill=False):
    if fill:
        a[:] = SENTINEL
        return True
    return bool((a == SENTINEL).all())


def torch_sentinel(t, fill=False):
    if fill:
        t.fill_(SENTINEL)
        return True
    return bool((t == SENTINEL).all().item())


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 200, 264, 1, 1), (10, 200, 200, 1, 0), (12, 136, 264, 0, 0)])
def test_emu_compact_frame_jobs(bpc, W, H, ssh, ssv):
    rng = np.random.default_rng(910 + bpc)
    S = CR.harden(synth.make_inter_frame(rng, bpc, W, H, ssh, ssv, film_grain=bpc > 8), rng)
    assert S.get("intra_tx") is None or not len(S["intra_tx"])
    assert S["hard_stats"]["1d"] > 5 and S["hard_stats"]["wht"] > 0, S["hard_stats"]
    check_compact_frame(S, dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc()), sentinel=numpy_sentinel)


@pytest.mark.emu
def test_emu_compact_job_with_intra_records_keeps_the_dense_path():
    """offsets on a job with intra records are ignored: the job zeroes and expands the dense plane the intra kernels read"""
    lib = refs.emu_lib()
    kw = dict(lib=lib, alloc=frame.NumpyAlloc())
    rng = np.random.default_rng(920)
    S = CR.harden(synth.make_inter_frame(rng, 10, 200, 136, 1, 1, p_intra=0.2), rng)
    assert len(S["intra_tx"]) > 10
    oracle_prototypes()
    exp = TF.oracle_frame(S)
    fb = frame.FrameBuffers(S, compact=True, **kw)
    assert fb.job.n_expand > 0 and not any(fb.job.d_itx_coff[tx] for tx in range(19))
    b = lib.b200_launch_count()
    fb.run()
    n_plain = lib.b200_launch_count() - b
    TF.check_frame(S, fb, exp)
    fbo = frame.FrameBuffers(S, compact=True, **kw)
    cc, ex = synth.compact_coefs(S)
    coff = frame.itx_compact_offsets(S, ex)
    for tx, o in coff.items():
        fbo.keep["coff%d" % tx] = fbo.alloc.upload(o)
        fbo.job.d_itx_coff[tx] = fbo.keep["coff%d" % tx][1]
    fbo.keep["coef"][0][:] = SENTINEL
    b = lib.b200_launch_count()
    fbo.run()
    assert lib.b200_launch_count() - b == n_plain, "a job with intra records must take the dense path (memset + coef_expand)"
    assert not (fbo.keep["coef"][0] == SENTINEL).all(), "a job with intra records must rebuild the dense plane"
    TF.check_frame(S, fbo, exp)


def test_compact_offsets_follow_the_band_order():
    """band_plan's offsets index the band-sorted records of every size: a band's range of d_itx[tx] is its range of offsets"""
    rng = np.random.default_rng(930)
    S = synth.make_inter_frame(rng, 8, 200, 264)
    S2, bands, _, (cc, ex_sorted, coff) = frame.band_plan(S, 64, compact=True)
    by_dense = {int(r["dense_off"]): int(r["compact_off"]) for r in ex_sorted}
    total = 0
    for tx in range(19):
        a = S2["itx"][tx]
        if not len(a):
            assert tx not in coff
            continue
        assert len(coff[tx]) == len(a) and coff[tx].dtype == np.dtype("<u4")
        assert [by_dense[int(o)] for o in a["coef_off"]] == coff[tx].tolist()
        total += len(a)
    assert total == len(ex_sorted)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 1920, 1080, 1, 1), (10, 1280, 720, 1, 0), (12, 1288, 720, 0, 0)])
def test_gpu_compact_frame_jobs(bpc, W, H, ssh, ssv):
    rng = np.random.default_rng(940 + bpc)
    S = CR.harden(synth.make_inter_frame(rng, bpc, W, H, ssh, ssv, film_grain=bpc > 8), rng, share=0.3)
    check_compact_frame(S, {}, rows_list=(0, 64, 192), sentinel=torch_sentinel)
