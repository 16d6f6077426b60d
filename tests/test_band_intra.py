"""Band-sliced frame jobs whose frames contain intra-machine records (intra, filter-intra, CFL, palette, inter-intra, intra
block copy): b200_frame_run_band with B200FrameBand.intra / intra_edge. The records on a band's first row read the row above
from the copy the previous band saved before its post filters ran (dav1d's saved intra edge, reference src/recon_tmpl.c
`top_sb_edge`), so every band plan and every phase order must give the whole-frame job's picture and the oracle's.

CPU: the host emulator. The intra kernel stops on a dependency that never arrives, so ordering mistakes are found here.
GPU: the same frames at larger sizes, and a mixed dependent GOP over two ranks with peer puts, eager and with graph replay."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, frame, synth
import test_frame as TF
import test_intra as TI

MOTION = dict(p_obmc=0.2, p_warp=0.15, p_ii=0.2)
VARIANTS = ((64, {}), (128, dict(compact=True)), (192, dict(compact=True, fused=True)), (64, dict(fused=True)))


def _mixed(seed, bpc, W, H, ssh, ssv, p_intra):
    return synth.make_inter_frame(np.random.default_rng(seed), bpc, W, H, ssh, ssv, p_intra=p_intra, film_grain=bpc > 8, **MOTION)


def _boundary_rows_filtered(S, exp, rows):
    """some band's bottom row changes in the deblocking sweep: reading it from the picture would be wrong"""
    o, st = S["off"][0], S["stride"][0]
    return any(not np.array_equal(exp["recon"][o + (y - 1) * st:o + y * st], exp["dbl"][o + (y - 1) * st:o + y * st])
               for y in range(rows, S["H"], rows))


def run_phase_order(fb):
    """RECON 0, RECON 1, POST 0, RECON 2, POST 1, ...: the reconstruction of band k+1 before the post filters of band k.
    Yields k after POST k."""
    n = fb.n_bands()
    fb.run_band_phase(0, 1)
    for k in range(n):
        if k + 1 < n:
            fb.run_band_phase(k + 1, 1)
        fb.run_band_phase(k, 2)
        yield k


def check_progress(S, fb, final, k, prev):
    """after band k the rows b200_band_progress reports hold their final values"""
    ssh, ssv = S["ss_hor"], S["ss_ver"]
    hs = [S["H"], (S["H"] + ssv) >> ssv, (S["H"] + ssv) >> ssv]
    ws = [S["W"], (S["W"] + ssh) >> ssh, (S["W"] + ssh) >> ssh]
    got = fb.output("p2")
    for pl in range(3):
        rows = fb.band_progress(k, pl)
        assert prev[pl] <= rows <= hs[pl]
        prev[pl] = rows
        o, st = S["off"][pl], S["stride"][pl]
        a = got[o:o + hs[pl] * st].reshape(hs[pl], st)[:rows, :ws[pl]]
        b = final[o:o + hs[pl] * st].reshape(hs[pl], st)[:rows, :ws[pl]]
        assert np.array_equal(a, b), "band %d plane %d: rows reported final are not" % (k, pl)
    return hs


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv,p_intra", [(8, 200, 264, 1, 1, 0.1), (10, 136, 328, 1, 1, 0.4),
                                                      (8, 136, 264, 0, 0, 0.25), (10, 136, 200, 0, 0, 0.3)])
def test_emu_mixed_frame_bands(bpc, W, H, ssh, ssv, p_intra):
    """mixed inter frames (intra blocks, OBMC, warps, inter-intra; 10-bit with film grain) in 64-, 128- and 192-row bands, with
    the compact and fused variants: equal to the whole-frame job and the oracle, in band order and in the order in which the
    reconstruction of band k+1 runs before the post filters of band k"""
    S = _mixed(1100 + bpc + W + H, bpc, W, H, ssh, ssv, p_intra)
    assert len(S["intra_tx"]) > 20 and (S["intra_tx"]["mode"] == 15).sum() > 0
    exp = TF.oracle_frame(S)
    assert _boundary_rows_filtered(S, exp, 64)
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    whole = frame.FrameBuffers(S, **kw)
    whole.run()
    TF.check_frame(S, whole, exp)
    last = "p3" if "fg" in exp else "p2"
    for rows, opts in VARIANTS:
        fb = frame.FrameBuffers(S, band_rows=rows, **opts, **kw)
        assert fb.n_bands() == -(-H // rows)
        assert sum(b.intra[1] for b in fb.bands) == len(S["intra_tx"])
        if fb.n_bands() > 1:
            assert fb.bands[0].intra_edge and all(b.intra_edge == fb.bands[0].intra_edge for b in fb.bands)
        fb.run_bands()
        TF.check_frame(S, fb, exp)
        assert np.array_equal(fb.output(last), whole.output(last)), (rows, opts)
    # phase order RECON0, RECON1, POST0, RECON2, POST1, ...; the progress after every band is final
    for rows in (64, 128):
        fb = frame.FrameBuffers(S, band_rows=rows, compact=True, **kw)
        prev = [0, 0, 0]
        for k in run_phase_order(fb):
            hs = check_progress(S, fb, exp["lr"], k, prev)
        assert prev == hs
        TF.check_frame(S, fb, exp)


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 200, 264, 1, 1), (10, 136, 200, 1, 1), (12, 72, 200, 0, 0), (8, 264, 200, 1, 0)])
def test_emu_intra_frame_bands(bpc, W, H, ssh, ssv):
    """intra-only frames (every block intra, CFL, filter-intra) banded with deblocking, CDEF and loop restoration on: equal to
    the whole-frame job, and their reconstruction to the oracle's"""
    S = synth.make_intra_frame(np.random.default_rng(1200 + bpc + W), bpc, W, H, ssh, ssv)
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc())
    whole = frame.FrameBuffers(S, **kw)
    whole.run()
    rec = TI.oracle_intra(S)
    S2 = dict(S); S2["pic"] = rec
    import test_loopfilter as TLF
    import test_cdef as TCD
    assert TCD.frame_area_equal(S, whole.output("p0"), TLF.lf_frame_oracle(S2))
    for rows, compact in ((64, False), (128, True)):
        fb = frame.FrameBuffers(S, band_rows=rows, compact=compact, **kw)
        assert fb.n_bands() > 1
        fb.run_bands()
        for name in ("p0", "p1", "p2"):
            assert np.array_equal(fb.output(name), whole.output(name)), (rows, name)
    fb = frame.FrameBuffers(S, band_rows=64, **kw)
    for _ in run_phase_order(fb):
        pass
    assert np.array_equal(fb.output("p2"), whole.output("p2"))


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 264, 264, 1, 1), (10, 200, 328, 0, 0)])
def test_emu_intra_block_copy_frame_bands(bpc, W, H, ssh, ssv):
    """intra block copy (filters off, as AV1 requires): copies read rows of earlier bands from the picture; equal to the
    whole-frame job and the oracle"""
    S = synth.make_intra_frame(np.random.default_rng(1300 + bpc + W), bpc, W, H, ssh, ssv, p_ibc=0.3)
    assert (S["intra_tx"]["mode"] == synth.MODE_IBC).sum() > 8
    exp = TI.oracle_intra(S)
    kw = dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc(), run_lf=False, run_cdef=False, run_lr=False)
    whole = frame.FrameBuffers(S, **kw)
    whole.run()
    for rows, compact in ((64, True), (128, False)):
        fb = frame.FrameBuffers(S, band_rows=rows, compact=compact, **kw)
        fb.run_bands()
        assert np.array_equal(fb.output("p0"), whole.output("p0")), rows
        ok, where = TI.planes_equal(S, exp, fb.output("p0"))
        assert ok, (rows, where)


@pytest.mark.emu
def test_emu_band_plan_rejects_records_that_read_below_their_band():
    """a bottom-left edge that reaches into the next band would be a dependency the kernel waits for forever: the band plan
    refuses it on the host"""
    S = synth.make_intra_frame(np.random.default_rng(1400), 8, 136, 200)
    t = S["intra_tx"].copy()
    # a luma block that ends on the bottom row of the first superblock row, with a left neighbour
    th = np.asarray(synth._L.TX_H)[t["tx"]] // 4
    i = int(np.nonzero((t["plane"] == 0) & (t["y4"] + th == 16) & ((t["flags"] & 1) > 0))[0][0])
    t["flags"][i] |= 8
    S["intra_tx"] = t
    frame.band_plan(S, 256)                       # one band: nothing below
    with pytest.raises(AssertionError, match="reads rows below its band"):
        frame.band_plan(S, 64)


@pytest.mark.emu
def test_emu_band_intra_abi_errors():
    """superblock-mode intra in a band that is not the whole frame, a missing intra_edge and an intra range outside the job
    are bad arguments (-2) with a message"""
    lib = refs.emu_lib()
    kw = dict(lib=lib, alloc=frame.NumpyAlloc())
    S = synth.make_intra_frame(np.random.default_rng(1500), 8, 136, 200)

    def rc(fb, b):
        return lib.b200_frame_run_band(C.byref(fb.job), C.byref(b), None), lib.b200_last_error().decode()

    fb = frame.FrameBuffers(S, band_rows=64, intra_sb=True, **kw)
    r, msg = rc(fb, fb.bands[0])
    assert r == -2 and "superblock" in msg
    fb = frame.FrameBuffers(S, band_rows=64, **kw)
    b = _lib.FrameBand.from_buffer_copy(fb.bands[1])
    b.intra_edge = None
    r, msg = rc(fb, b)
    assert r == -2 and "intra_edge" in msg
    for first, count in ((-1, 4), (0, fb.job.n_intra + 1), (fb.job.n_intra, 1)):
        b = _lib.FrameBand.from_buffer_copy(fb.bands[0])
        b.intra[0], b.intra[1] = first, count
        r, msg = rc(fb, b)
        assert r == -2 and "intra range" in msg, (first, count)
    whole = frame.FrameBuffers(S, band_rows=256, intra_sb=True, **kw)     # superblock mode as the whole-frame band is fine
    assert whole.n_bands() == 1 and rc(whole, whole.bands[0])[0] == 0


# whole-frame jobs and jobs without intra records launch what they launched before band-sliced intra existed
LAUNCHES = {"mixed_whole": 14, "mixed_one_band": 15, "intra_whole": 3, "intra_sb_whole": 5, "inter_bands64": 44, "intra_batch4": 9}


@pytest.mark.emu
def test_emu_launch_counts_of_unbanded_jobs_unchanged():
    lib = refs.emu_lib()
    kw = dict(lib=lib, alloc=frame.NumpyAlloc())

    def count(fn):
        b = lib.b200_launch_count()
        fn()
        return lib.b200_launch_count() - b
    out = {}
    S = synth.make_inter_frame(np.random.default_rng(11), 10, 200, 136, p_intra=0.2, film_grain=True, p_obmc=0.2, p_warp=0.15, p_ii=0.15)
    out["mixed_whole"] = count(frame.FrameBuffers(S, **kw).run)
    out["mixed_one_band"] = count(frame.FrameBuffers(S, band_rows=192, compact=True, **kw).run_bands)
    Si = synth.make_intra_frame(np.random.default_rng(12), 8, 200, 136)
    out["intra_whole"] = count(frame.FrameBuffers(Si, run_cdef=False, run_lr=False, **kw).run)
    out["intra_sb_whole"] = count(frame.FrameBuffers(Si, intra_sb=True, **kw).run)
    Sb = synth.make_inter_frame(np.random.default_rng(13), 8, 200, 264, film_grain=True)
    out["inter_bands64"] = count(frame.FrameBuffers(Sb, band_rows=64, **kw).run_bands)
    fbs = [frame.FrameBuffers(synth.make_intra_frame(np.random.default_rng(14 + k), 8, 136, 72), run_cdef=False, run_lr=False, **kw)
           for k in range(4)]
    out["intra_batch4"] = count(lambda: frame.run_batch(fbs))
    assert out == LAUNCHES
    # a banded mixed frame adds one intra launch per band with records and one edge copy per band boundary
    fb = frame.FrameBuffers(S, band_rows=64, compact=True, **kw)
    n = count(fb.run_bands)
    assert n > LAUNCHES["mixed_one_band"]


# ------------------------------------------------------------------------------------------ dependent GOP over ranks
def _gop_frames(w=200, h=264, n=6, bpc=8, seed=1600):
    return [synth.make_inter_frame(np.random.default_rng(seed + k), bpc, w, h, p_intra=0.15, **MOTION) for k in range(n)]


def _worker_emu_bands(rank, world, port, outdir):
    sys.path.insert(0, os.path.dirname(__file__))
    import torch.distributed as dist
    import test_multigpu as TM
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pics = TM._decode_emu(rank, world, _gop_frames(), band_rows=64)
        np.savez(os.path.join(outdir, "r%d.npz" % rank), **{str(k): v for k, v in pics.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.emu
@pytest.mark.parametrize("world", [2, 3])
def test_ranks_shard_mixed_frames_in_bands(tmp_path, world):
    """a dependent GOP of mixed frames (264 rows: five 64-row bands) over gloo ranks: every frame equals the single-rank decode
    and the oracle's chained decode"""
    import torch.multiprocessing as mp
    import test_multigpu as TM
    port = 29500 + (os.getpid() + 41 + world) % 2000
    mp.spawn(_worker_emu_bands, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    frames = _gop_frames()
    got = TM._collect(str(tmp_path), world, len(frames))
    single = TM._decode_emu(0, 1, frames, band_rows=64)
    exp = TM.oracle_gop(frames)
    for k in range(len(frames)):
        assert np.array_equal(got[k], single[k]), "frame %d: sharded decode differs from the single-rank decode" % k
        assert np.array_equal(got[k], exp[k]), "frame %d differs from the oracle's chained decode" % k


# ------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H", [(8, 648, 520), (10, 1288, 720)])
def test_gpu_mixed_frame_bands(bpc, W, H):
    S = _mixed(1700 + bpc, bpc, W, H, 1, 1, 0.15)
    exp = TF.oracle_frame(S)
    for rows, opts in VARIANTS:
        fb = frame.FrameBuffers(S, band_rows=rows, **opts)
        fb.run_bands()
        fb.alloc.sync()
        TF.check_frame(S, fb, exp)
    # the reconstruction of band k+1 before the post filters of band k, on one stream
    fb = frame.FrameBuffers(S, band_rows=64, compact=True)
    for _ in run_phase_order(fb):
        pass
    fb.alloc.sync()
    TF.check_frame(S, fb, exp)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H", [(8, 648, 520), (10, 1288, 720), (8, 1920, 1080)])
def test_gpu_intra_frame_bands(bpc, W, H):
    """intra-only frames banded with deblocking on (a 1080p key frame among them), and with intra block copy (filters off)"""
    import test_loopfilter as TLF
    import test_cdef as TCD
    S = synth.make_intra_frame(np.random.default_rng(1800 + bpc + W), bpc, W, H)
    rec = TI.oracle_intra(S)
    S2 = dict(S); S2["pic"] = rec
    dbl = TLF.lf_frame_oracle(S2)
    for rows in (64, 192):
        fb = frame.FrameBuffers(S, band_rows=rows, compact=True, run_cdef=False, run_lr=False)
        fb.run_bands()
        fb.alloc.sync()
        assert TCD.frame_area_equal(S, fb.output("p0"), dbl), rows
    S = synth.make_intra_frame(np.random.default_rng(1850 + bpc + W), bpc, W, H, p_ibc=0.3)
    exp = TI.oracle_intra(S)
    fb = frame.FrameBuffers(S, band_rows=64, compact=True, run_lf=False, run_cdef=False, run_lr=False)
    fb.run_bands()
    fb.alloc.sync()
    ok, where = TI.planes_equal(S, exp, fb.output("p0"))
    assert ok, where


GW, GH = 648, 520


def _gpu_gop_frames(n, seed):
    return [synth.make_inter_frame(np.random.default_rng(seed + k), 8, GW, GH, p_intra=0.1, **MOTION) for k in range(n)]


def _worker_gpu_bands(rank, world, port, outdir):
    import test_multigpu as TM
    TM._gpu_rank_setup(rank, world, port)
    import torch.distributed as dist
    try:
        from dav1d_b200 import shard, get_lib
        frames = _gpu_gop_frames(6, 1900)

        def make(S, rows):
            return frame.FrameBuffers(S, band_rows=rows, compact=True)
        pics = shard.decode_gop(frames, make, dist, rank, world, get_lib(), exchange="peer", band_rows=64)
        np.savez(os.path.join(outdir, "r%d.npz" % rank), **{str(k): v for k, v in pics.items()})
    finally:
        dist.destroy_process_group()


def _worker_gpu_graph(rank, world, port, outdir, per_rank):
    import test_multigpu as TM
    TM._gpu_rank_setup(rank, world, port)
    import torch.distributed as dist
    try:
        from dav1d_b200 import shard, get_lib
        lib = get_lib()
        n_sets = 4
        base = {(r, i): _gpu_gop_frames(1, 1950 + 16 * r + i)[0] for r in range(world) for i in range(n_sets)}
        sets = [frame.FrameBuffers(base[(rank, i)], band_rows=64, compact=True) for i in range(n_sets)]
        x = shard.PeerExchange(lib, dist, rank, world, base[(0, 0)]["pic"].nbytes, 2)
        pipe = shard.GopPipeline(lib, rank, world, sets, exchange=x, graphs=True)
        for _ in range(per_rank):
            pipe.submit()
        pipe.sync()
        dist.barrier()
        out = {str((per_rank - n_sets + i) * world + rank): pipe.output(per_rank - n_sets + i) for i in range(n_sets)}
        np.savez(os.path.join(outdir, "g%d.npz" % rank), **out)
        x.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_gpu_ranks_shard_mixed_frames_in_bands(tmp_path):
    """a mixed dependent GOP over two ranks in 64-row bands, reference rows as peer puts: equal to the oracle's chained decode"""
    import test_multigpu as TM
    port = 29500 + (os.getpid() + 53) % 2000
    TM._spawn_ranks(_worker_gpu_bands, (2, port, str(tmp_path)), 2)
    frames = _gpu_gop_frames(6, 1900)
    got = TM._collect(str(tmp_path), 2, len(frames))
    exp = TM.oracle_gop(frames)
    for k in range(len(frames)):
        assert np.array_equal(got[k], exp[k]), "frame %d differs from the oracle's chained decode" % k


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_gpu_graph_replay_mixed_frames_in_bands(tmp_path):
    """the same over two ranks as an endless stream: from a set's second frame on, every frame (its banded intra launches and
    edge copies included) is one CUDA graph launch"""
    import test_multigpu as TM
    per_rank, world, n_sets = 10, 2, 4
    port = 29500 + (os.getpid() + 59) % 2000
    TM._spawn_ranks(_worker_gpu_graph, (world, port, str(tmp_path), per_rank), world)
    base = {(r, i): _gpu_gop_frames(1, 1950 + 16 * r + i)[0] for r in range(world) for i in range(n_sets)}
    seq = [base[(n % world, (n // world) % n_sets)] for n in range(per_rank * world)]
    exp = TM.oracle_gop(seq)
    for r in range(world):
        z = np.load(os.path.join(str(tmp_path), "g%d.npz" % r))
        assert len(z.files) == n_sets
        for k in z.files:
            assert np.array_equal(z[k], exp[int(k)]), "frame %s (rank %d) differs from the oracle's chained decode" % (k, r)
