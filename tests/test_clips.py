"""Clip batches (stream.DeviceDecoder.clips) and the batched tensor export behind them (b200_export_tensor_batch,
dav1d_b200/csrc/export.cu; b200hook_export_tensor_batch, integration/dav1d/b200_hooks.c). Every x[i, t] must be
stream.tensor_reference applied to stock dav1d's picture start_i + t * step of stream i, bit for bit; a batch of jobs must
write exactly what one b200_export_tensor per job writes. CPU tests run the CUDA sources on the host emulator (numpy
destinations), GPU tests run the CUDA library into torch CUDA tensors."""
import ctypes as C
import threading

import numpy as np
import pytest

import refs
from dav1d_b200 import obu, stream

import test_stream_device_output as DO
import test_tensor_export as TE

BATCH_MAX = 24                          # B200_TENSOR_BATCH_MAX, include/b200av1.h


def _alloc(shape, dtype):
    return np.full(shape, 0x5a, np.float32 if dtype == "float32" else np.uint16)


def _check_clips(dec, streams, frames, step, start, size=None, dtype="float32", layout="chw", sitings=None, colors=None,
                 matrix="auto", mean=None, std=None, alloc=_alloc, d2h=0, **kw):
    """clips() against tensor_reference on stock dav1d's pictures; sitings[i] / colors[i] = what "auto" siting / matrix and
    range resolve to for stream i (default "left" / ("bt709", limited)); d2h=None: device-to-host traffic of other decoders
    is expected"""
    starts = [start] * len(streams) if isinstance(start, int) else start
    dec.stats(reset=True)
    x = dec.clips(streams, frames=frames, step=step, start=start, size=size, dtype=dtype, layout=layout, mean=mean, std=std,
                  matrix=matrix, alloc=alloc, **kw)
    assert x.shape[:2] == (len(streams), frames)
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        name, full = (colors or {}).get(i, ("bt709", False))
        name = name if matrix == "auto" else matrix
        for t in range(frames):
            w, h, bpc, lay, rp = ref[starts[i] + t * step]
            want = stream.tensor_reference(rp, bpc, lay, size, name, full, (sitings or {}).get(i, "left"), mean, std)
            if layout == "hwc":
                want = want.transpose(1, 2, 0)
            assert tuple(x[i, t].shape) == want.shape, (i, t)
            assert np.array_equal(TE._host_bits(x[i, t], dtype), TE._bits(want, dtype)), "stream %d clip picture %d (%s, %s)" % (i, t, dtype, layout)
    assert d2h is None or dec.stats(reset=True)["d2h_bytes"] == d2h
    return x


# matrix and range "auto" resolves to, per stream of _mixed_streams (the others have no colour description)
MIXED_COLORS = {0: ("bt601", True), 3: ("bt2020", False)}


def _mixed_streams():
    """4:2:0 8 bit with hidden frames (BT.601 full range), 4:2:2 10 bit with grain, 4:4:4 12 bit, 4:0:0 10 bit (BT.2020),
    4:2:0 colocated chroma, odd sizes"""
    import test_stream as TS
    return [obu.inter_stream(41, 99, 67, n_frames=7, bpc=8, motion_modes=1, hidden_every=2, color=(5, 1)),
            TS._valid_422("inter", 96, 64, 10, 1, motion_modes=1, film_grain=1)[0],
            obu.intra_stream(43, 72, 50, n_frames=6, bpc=12, layout="444", film_grain=1),
            obu.inter_stream(44, 61, 45, n_frames=6, bpc=10, layout="400", color=(9, 0)),
            obu.inter_stream(45, 83, 57, n_frames=7, bpc=8, chroma_sample_position=2, film_grain=1)]


@pytest.fixture(scope="module")
def emu_dec(hooked_library):
    refs.emu_lib()
    d = stream.DeviceDecoder(backend=DO._emu_path(), serialize=True, apply_grain=1)
    yield d
    d.release()


@pytest.fixture(scope="module")
def hooked_library():
    stream.build_hooked()
    if not __import__("os").path.exists(stream.HOOKED_SO):
        pytest.skip("%s not built" % stream.HOOKED_SO)


# ---- decoder level, emulator --------------------------------------------------------------------------------------
@pytest.mark.emu
@pytest.mark.parametrize("dtype", list(stream.TENSOR_DTYPES))
@pytest.mark.parametrize("layout", list(stream.TENSOR_LAYOUTS))
def test_clips_match_definition_emu(emu_dec, dtype, layout):
    streams = _mixed_streams()
    counts = [len(DO._ref_pictures(s)) for s in streams]
    starts = [max(0, c - 3 - k % 2) for k, c in enumerate(counts)]       # pictures start, start + 2: at or near the end
    kw = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)) if dtype != "float32" else {}
    _check_clips(emu_dec, streams, 2, 2, starts, size=(23, 37), dtype=dtype, layout=layout, sitings={4: "topleft"},
                 colors=MIXED_COLORS, workers=3 if layout == "chw" else None, **kw)


@pytest.mark.emu
def test_clips_native_size_emu(emu_dec):
    """size=None: pictures of one size keep it; every stream its own start, two workers for three streams"""
    streams = [obu.inter_stream(50 + k, 64, 48, n_frames=5, bpc=8 + 2 * (k % 2), film_grain=k % 2) for k in range(3)]
    x = _check_clips(emu_dec, streams, 2, 2, [0, 1, 0], workers=2, dtype="float16", layout="hwc")
    assert x.shape == (3, 2, 48, 64, 3)


@pytest.mark.emu
def test_clips_capacity_emu(emu_dec):
    """32 streams decoded at once, 4 frame contexts each, references refreshed at random: more than 64 device pictures and
    more than 64 frame contexts are alive at once, so both tables of the hooks grow past their first chunk of 64 (which a
    table fixed at 64 entries cannot serve: live entries would be recycled or refused). Every clip must still be right, and
    a HookedDecoder decoding in another thread at the same time still matches stock dav1d."""
    streams = [obu.inter_stream(60 + k, 64, 48, n_frames=12, bpc=8, motion_modes=1, film_grain=k % 2) for k in range(32)]
    dec = stream.DeviceDecoder(backend=DO._emu_path(), serialize=True, n_threads=4, max_frame_delay=4)
    dec.release()                                   # nothing decodes now: the device-picture table starts empty
    other = obu.inter_stream(70, 96, 64, n_frames=6, bpc=10, motion_modes=2)
    r0, _, out0 = stream.decode_stream(C.CDLL(refs.REF_SO), other, apply_grain=1)
    res = {}

    def side():
        res["r"] = stream.HookedDecoder(backend=DO._emu_path(), serialize=True).decode(other, apply_grain=1)
    th = threading.Thread(target=side)
    th.start()
    _check_clips(dec, streams, 3, 2, 5, size=(20, 30), workers=32, d2h=None)
    th.join()
    st = dec.stats()
    assert st["ref_table"] > 64 and st["frame_table"] > 64, (st["ref_table"], st["frame_table"])
    r1, _, out1 = res["r"]
    assert r1 == r0 and np.array_equal(out0, out1)


@pytest.mark.emu
def test_clips_errors_emu(emu_dec):
    good = [obu.inter_stream(80 + k, 64, 48, n_frames=4, bpc=8) for k in range(3)]
    before = threading.active_count()
    with pytest.raises(ValueError, match="stream 1 "):
        emu_dec.clips([good[0], good[1][:2], good[2]], frames=2, step=2, alloc=_alloc)
    assert threading.active_count() == before
    other_size = obu.inter_stream(90, 80, 48, n_frames=4, bpc=8)
    with pytest.raises(ValueError, match="size"):
        emu_dec.clips([good[0], other_size], frames=2, alloc=_alloc)
    assert threading.active_count() == before
    for kw in (dict(workers=0), dict(workers=stream.CLIP_MAX_WORKERS + 1), dict(start=-1), dict(start=[0, 1]),
               dict(frames=0), dict(step=0), dict(dtype="int8"), dict(size=(0, 4))):
        args = dict(frames=2, alloc=_alloc)
        args.update(kw)
        with pytest.raises(ValueError):
            emu_dec.clips(good, **args)
    with pytest.raises(ValueError):
        emu_dec.clips([], frames=1, alloc=_alloc)
    bad = list(good[1])
    bad[2] = bytes([0x32, 0x05]) + b"\xff" * 6                  # an OBU dav1d rejects
    with pytest.raises(RuntimeError, match="stream 1"):
        emu_dec.clips([good[0], bad, good[2]], frames=4, workers=3, alloc=_alloc)
    assert threading.active_count() == before
    _check_clips(emu_dec, good, 2, 1, 1)                      # the decoder is still usable


# ---- the batch ABI, emulator --------------------------------------------------------------------------------------
def _batch_cases(rng, n, dtype, lay):
    out = []
    for k in range(n):
        bpc = (8, 10, 12)[int(rng.integers(3))] if k % 3 else 8
        layout = int(rng.integers(4))
        w, h = int(rng.integers(5, 70)), int(rng.integers(3, 50))
        size = None if k % 4 == 0 else (int(rng.integers(1, 60)), int(rng.integers(1, 60)))
        matrix = "identity" if layout == 3 and k % 5 == 0 else ["bt601", "bt709", "bt2020"][k % 3]
        out.append(TE.Case(bpc, layout, w, h, size, dtype, lay, list(stream.SITINGS)[k % 3], matrix, bool(k % 2), offset=k % 2, pad=k % 3))
    return out


def _batch_setup(cases, seed, ptr_of=lambda a: a.ctypes.data):
    """per job: sources, job, and the expected bits of its destination slice; all destinations in one guarded buffer"""
    rng = np.random.default_rng(seed)
    et = np.uint32 if cases[0].dtype == "float32" else np.uint16
    guard = et(0x7fc0dead if et is np.uint32 else 0x7e57)
    srcs, spans, at = [], [], TE.GUARD
    for c in cases:
        planes = TE._planes(rng, c)
        src, offs, strides = TE._source(planes, c.layout)
        pc, py, n = TE._pitches(c)
        srcs.append((c, planes, src, offs, strides, pc, py, n))
        spans.append(at + c.offset)
        at += c.offset + n + TE.GUARD
    return srcs, spans, np.full(at, guard, et), guard


@pytest.mark.emu
@pytest.mark.parametrize("n", [1, BATCH_MAX, BATCH_MAX + 5, 2 * BATCH_MAX + 5])
@pytest.mark.parametrize("dtype,lay", [("float32", "chw"), ("bfloat16", "hwc"), ("float16", "chw")])
def test_batch_matches_single_jobs_emu(n, dtype, lay):
    lib = refs.emu_lib()
    cases = _batch_cases(np.random.default_rng(n), n, dtype, lay)
    if n > 2 * BATCH_MAX:                  # both bit-depth classes are split into several launches
        assert min(sum(c.bpc == 8 for c in cases), sum(c.bpc > 8 for c in cases)) > BATCH_MAX
    srcs, spans, buf, guard = _batch_setup(cases, 500 + n)
    jobs = (stream.TensorJob * n)()
    want = np.full_like(buf, guard)
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        want[at:at + m] = TE._expected(c, planes, pc, py, m, guard)
    assert lib.b200_export_tensor_batch(jobs, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)
    single = np.full_like(buf, guard)
    for k, (c, planes, src, offs, strides, pc, py, m) in enumerate(srcs):
        j = stream.TensorJob.from_buffer_copy(jobs[k])
        j.dst = single.ctypes.data + spans[k] * single.itemsize
        assert lib.b200_export_tensor(C.byref(j), None) == 0
    assert np.array_equal(buf, single)


@pytest.mark.emu
def test_batch_bad_arguments_emu():
    lib = refs.emu_lib()
    cases = _batch_cases(np.random.default_rng(9), 6, "float32", "chw")
    srcs, spans, buf, guard = _batch_setup(cases, 9)
    jobs = (stream.TensorJob * 6)()
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
    assert lib.b200_export_tensor_batch(None, 1, None) == -2
    assert lib.b200_export_tensor_batch(jobs, 0, None) == -2
    assert lib.b200_export_tensor_batch(jobs, -3, None) == -2
    for field, value in [("dtype", 1), ("layout", 1), ("bitdepth_max", 511), ("src", None), ("out_w", 0), ("pitch_y", 1)]:
        bad = (stream.TensorJob * 6).from_buffer_copy(jobs)
        setattr(bad[4], field, value)
        buf[:] = guard
        assert lib.b200_export_tensor_batch(bad, 6, None) == -2, field
        assert lib.b200_last_error()
        assert np.all(buf == guard), "a rejected batch wrote %s" % field       # nothing launched


# ---- on the device ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
def test_clips_gpu(hooked_library, dtype, monkeypatch):
    """four 1080p 8-bit streams (one with grain) and one 4K 10-bit stream into one [5, 8, 3, 224, 224] batch on a
    non-default stream"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)         # stock dav1d's 16 4K 10-bit pictures, packed
    streams = [obu.inter_stream(600 + k, 1920, 1080, n_frames=17, bpc=8, log2_cols=2, log2_rows=1, motion_modes=1,
                                film_grain=int(k == 1)) for k in range(4)]
    streams.append(obu.inter_stream(610, 3840, 2160, n_frames=16, bpc=10, log2_cols=2, log2_rows=1, motion_modes=1))
    dec = stream.DeviceDecoder(n_threads=4, max_frame_delay=2)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = _check_clips(dec, streams, 8, 2, [0, 1, 0, 1, 0], size=(224, 224), dtype=dtype, alloc=None, workers=5,
                         mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
    assert x.is_cuda and tuple(x.shape) == (5, 8, 3, 224, 224)
    dec.release()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["1080p8", "4k10", "mixed"])
def test_batch_matches_single_jobs_gpu(mix):
    """b200_export_tensor_batch against one b200_export_tensor per job on full-size device pictures, into 224 x 224"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    kinds = {"1080p8": [(8, 1920, 1080)] * 30, "4k10": [(10, 3840, 2160)] * 6, "mixed": [(8, 1920, 1080), (10, 3840, 2160)] * 14}[mix]
    rng = np.random.default_rng(len(kinds))
    cases = [TE.Case(bpc, 1, w, h, (224, 224), "bfloat16", "chw", "left", "bt709", bool(k % 2)) for k, (bpc, w, h) in enumerate(kinds)]
    srcs = []
    for c in cases:
        planes = TE._planes(rng, c)
        src, offs, strides = TE._source(planes, c.layout, extra=64)
        srcs.append((torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda(), offs, strides))
    pc, py, m = TE._pitches(cases[0])
    slot = m + TE.GUARD
    a = torch.full((len(cases) * slot + TE.GUARD,), 0x7e57, dtype=torch.int16, device="cuda")
    b = a.clone()
    jobs = (stream.TensorJob * len(cases))()
    for k, (c, (d, offs, strides)) in enumerate(zip(cases, srcs)):
        jobs[k] = TE._job(c, d.data_ptr(), offs, strides, a.data_ptr() + (TE.GUARD + k * slot) * 2, pc, py)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    assert lib.b200_export_tensor_batch(jobs, len(cases), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
    for k in range(len(cases)):
        j = stream.TensorJob.from_buffer_copy(jobs[k])
        j.dst = b.data_ptr() + (TE.GUARD + k * slot) * 2
        assert lib.b200_export_tensor(C.byref(j), C.c_void_p(s.cuda_stream)) == 0
    s.synchronize()
    assert torch.equal(a, b)
    c, (d, offs, strides) = cases[0], srcs[0]
    want = TE._expected(c, TE._planes(np.random.default_rng(len(kinds)), c), pc, py, m, np.uint16(0x7e57))
    assert np.array_equal(TE._host_bits(a, "bfloat16")[TE.GUARD:TE.GUARD + m], want)     # and the batch is the definition
