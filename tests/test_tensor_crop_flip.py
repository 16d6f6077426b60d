"""Crop boxes and horizontal flips in the tensor export (B200TensorJob.flip and a cropped source, include/b200av1.h;
tensor_store in dav1d_b200/csrc/export.cu; the boxes of b200hook_export_tensor_batch; crop= / flip= of
stream.DeviceDecoder.tensors and clips). A crop is only a change of source: the export of a box must be exactly
stream.tensor_reference of stream.crop_planes of the picture. A flip is only a mirrored store: out'[.., x] = out[.., OW-1-x]
bit for bit. CPU tests run the CUDA sources on the host emulator, GPU tests run the CUDA library into torch CUDA tensors."""
import ctypes as C

import numpy as np
import pytest

import refs
from dav1d_b200 import obu, stream

import test_clips as TC
import test_stream_device_output as DO
import test_tensor_export as TE

DTYPES = list(stream.TENSOR_DTYPES)
IMAGENET = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))


def _mirror(ref, flip):
    return ref[:, :, ::-1].copy() if flip else ref


# ---- the alignment rule -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout,box,want", [
    (1, (3, 5, 10, 7), (2, 4, 11, 8)), (1, (2, 4, 1, 1), (2, 4, 1, 1)), (1, (1, 1, 1, 1), (0, 0, 2, 2)),
    (2, (3, 5, 10, 7), (3, 4, 10, 8)), (3, (3, 5, 10, 7), (3, 5, 10, 7)), (0, (3, 5, 10, 7), (3, 5, 10, 7)),
    (1, (0, 0, 20, 30), (0, 0, 20, 30)), (1, (19, 29, 1, 1), (18, 28, 2, 2))])
def test_align_crop(layout, box, want):
    """odd top / left move to even on subsampled axes only; the bottom / right edge stays"""
    got = stream.align_crop(box, 30, 20, layout)
    assert got == want
    assert got[0] + got[2] == box[0] + box[2] and got[1] + got[3] == box[1] + box[3]


@pytest.mark.parametrize("box", [(-1, 0, 2, 2), (0, -1, 2, 2), (0, 0, 0, 2), (0, 0, 2, 0), (19, 0, 2, 2), (0, 29, 2, 2),
                                 (0, 0, 21, 30), (0, 0, 20, 31), (0, 0, 2), (0, 0, 2.0, 2), "abcd", None])
def test_align_crop_rejects(box):
    with pytest.raises(ValueError):
        stream.align_crop(box, 30, 20, 1)


def test_crop_planes():
    planes = [np.arange(20 * 30).reshape(20, 30), np.arange(10 * 15).reshape(10, 15), -np.arange(10 * 15).reshape(10, 15)]
    y, u, v = stream.crop_planes(planes, 1, (2, 4, 5, 7))
    assert np.array_equal(y, planes[0][2:7, 4:11]) and np.array_equal(u, planes[1][1:4, 2:6]) and np.array_equal(v, planes[2][1:4, 2:6])
    y, u, _ = stream.crop_planes([planes[0], planes[0][:, :15], planes[0][:, :15]], 2, (3, 2, 4, 4))
    assert u.shape == (4, 2)
    assert len(stream.crop_planes(planes[:1], 0, (1, 1, 1, 1))) == 1


# ---- kernel level -------------------------------------------------------------------------------------------------
def _expected(c, planes, pc, py, n, guard, aa, flip):
    ref = _mirror(stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std,
                                          antialias=aa), flip)
    bits = TE._bits(ref, c.dtype)
    out = np.full(n, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        out[ch * pc + y * py + x if c.lay == "chw" else y * py + 3 * x + ch] = bits[ch]
    return out


def _run(c, seed, aa, flip, lib, device=False):
    """one job into a guarded destination: (what was written, what the definition says)"""
    rng = np.random.default_rng(seed)
    planes = TE._planes(rng, c)
    src, offs, strides = TE._source(planes, c.layout, extra=64 if device else 7)
    pc, py, n = TE._pitches(c)
    et = np.uint32 if c.dtype == "float32" else np.uint16
    guard = et(0x7fc0dead if et is np.uint32 else 0x7e57)
    total = n + 2 * TE.GUARD + c.offset
    if device:
        import torch
        d_src = torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda()
        buf = torch.full((total,), int(guard.astype(np.int32 if et is np.uint32 else np.int16)),
                         dtype=torch.int32 if et is np.uint32 else torch.int16, device="cuda")
        j = TE._job(c, d_src.data_ptr(), offs, strides, buf.data_ptr() + (TE.GUARD + c.offset) * buf.element_size(), pc, py)
        j.antialias, j.flip = aa, flip
        assert lib.b200_export_tensor(C.byref(j), None) == 0, lib.b200_last_error()
        torch.cuda.synchronize()
        got = TE._host_bits(buf, c.dtype)
    else:
        buf = np.full(total, guard, et)
        j = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + (TE.GUARD + c.offset) * buf.itemsize, pc, py)
        j.antialias, j.flip = aa, flip
        assert lib.b200_export_tensor(C.byref(j), None) == 0, lib.b200_last_error()
        got = buf
    want = np.full(total, guard, et)
    want[TE.GUARD + c.offset:TE.GUARD + c.offset + n] = _expected(c, planes, pc, py, n, guard, aa, flip)
    return got, want


def _kernel_cases():
    """(case, antialias): every dtype x layout x bit depth x chroma layout on both kernels, with output widths below 4, not
    a multiple of 4 and a multiple of 4, odd pitches and destinations misaligned by one element"""
    geo = [(45, 27, (13, 22)), (38, 21, (9, 3)), (64, 48, (5, 1)), (97, 13, (40, 2)), (33, 31, (100, 11)), (61, 33, (7, 16)),
           (200, 150, (30, 45)), (9, 260, (4, 5))]
    cases, k = [], 0
    for bpc in (8, 10, 12):
        for layout in (0, 1, 2, 3):
            for dtype in DTYPES:
                for lay in ("chw", "hwc"):
                    w, h, size = geo[k % len(geo)]
                    siting = list(stream.SITINGS)[k % 3]
                    matrix = "identity" if layout == 3 and k % 4 == 0 else ["bt601", "bt709", "bt2020"][k % 3]
                    kw = IMAGENET if k % 3 == 1 else {}
                    cases.append((TE.Case(bpc, layout, w, h, size, dtype, lay, siting, matrix, bool(k % 2), offset=(k // 2) % 2,
                                          pad=(1, 0, 3)[k % 3], **kw), k % 2))
                    k += 1
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_flip_kernel_emu(idx):
    """flip = 1 writes the flip = 0 output mirrored, bit for bit, and nothing outside it"""
    c, aa = KERNEL_CASES[idx]
    lib = refs.emu_lib()
    got, want = _run(c, 5000 + idx, aa, 1, lib)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s)" % (bad.size, bad[0], c.__dict__)


def _batch(n, dtype, lay, seed):
    """a mixed batch on host sources: (jobs, destination, what it must hold, job offsets, guard, sources to keep alive)"""
    rng = np.random.default_rng(seed)
    cases = TC._batch_cases(rng, n, dtype, lay)
    aa, flips = [], []
    for k, c in enumerate(cases):
        if k % 2:
            c.size = (max(1, c.h // (2 + k % 5)), max(1, c.w // (1 + k % 3)))
        aa.append(int(k % 4 != 0))
        flips.append(int(k % 3 != 1))
    srcs, spans, buf, guard = TC._batch_setup(cases, seed)
    jobs = (stream.TensorJob * n)()
    want = np.full_like(buf, guard)
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        jobs[k].antialias, jobs[k].flip = aa[k], flips[k]
        want[at:at + m] = _expected(c, planes, pc, py, m, guard, aa[k], flips[k])
    return jobs, buf, want, spans, guard, srcs


@pytest.mark.emu
@pytest.mark.parametrize("n", [1, TC.BATCH_MAX, TC.BATCH_MAX + 5])
@pytest.mark.parametrize("dtype,lay", [("float32", "hwc"), ("bfloat16", "chw"), ("float16", "hwc")])
def test_batch_mixing_flips_emu(n, dtype, lay):
    """flipped and unflipped, antialiased and bilinear jobs of both bit-depth classes in one call: each is the definition,
    and writes what it writes alone"""
    lib = refs.emu_lib()
    jobs, buf, want, spans, guard, _keep = _batch(n, dtype, lay, 900 + n)
    assert lib.b200_export_tensor_batch(jobs, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)
    single = np.full_like(buf, guard)
    for k in range(n):
        j = stream.TensorJob.from_buffer_copy(jobs[k])
        j.dst = single.ctypes.data + spans[k] * single.itemsize
        assert lib.b200_export_tensor(C.byref(j), None) == 0
    assert np.array_equal(buf, single)


@pytest.mark.emu
def test_bad_flip_emu():
    """flip outside 0 .. 1 on one job of a batch: -2 and nothing written"""
    lib = refs.emu_lib()
    jobs, buf, _, _, guard, _keep = _batch(6, "float32", "chw", 17)
    for value in (2, -1):
        bad = (stream.TensorJob * 6).from_buffer_copy(jobs)
        bad[3].flip = value
        buf[:] = guard
        assert lib.b200_export_tensor_batch(bad, 6, None) == -2
        assert lib.b200_last_error()
        assert np.all(buf == guard)
        assert lib.b200_export_tensor(C.byref(bad[3]), None) == -2
    assert C.sizeof(stream.TensorJob) == 168 and 24 * C.sizeof(stream.TensorJob) <= 4096


# ---- decoder level ------------------------------------------------------------------------------------------------
def _check_tensors(dec, tus, crop, flip, size=None, dtype="float32", layout="chw", alloc=TE._np_alloc, antialias=False,
                   matrix="auto", want_siting="left", **kw):
    """tensors(crop=, flip=) against tensor_reference(crop_planes(stock dav1d's picture)), mirrored where flipped"""
    ref = DO._ref_pictures(tus)
    dec.stats(reset=True)
    got = list(dec.tensors(tus, size=size, dtype=dtype, layout=layout, alloc=alloc, antialias=antialias, matrix=matrix,
                           crop=crop, flip=flip, **kw))
    items = [t for g in got for t in g] if kw.get("batch") else got
    assert len(items) == len(ref)
    name = "bt709" if matrix == "auto" else matrix
    for k, ((w, h, bpc, lay, rp), g) in enumerate(zip(ref, items)):
        box = stream.align_crop(crop(k, h, w) if callable(crop) else crop, w, h, lay)
        fl = flip(k) if callable(flip) else flip
        want = _mirror(stream.tensor_reference(stream.crop_planes(rp, lay, box), bpc, lay, size, name, False, want_siting,
                                               kw.get("mean"), kw.get("std"), antialias=antialias), fl)
        if layout == "hwc":
            want = want.transpose(1, 2, 0)
        assert tuple(g.shape) == want.shape, k
        assert np.array_equal(TE._host_bits(g, dtype), TE._bits(want, dtype)), "picture %d differs (box %s, flip %s)" % (k, box, fl)
    assert dec.stats(reset=True)["d2h_bytes"] == 0
    return got


def _random_box(k, h, w):
    rng = np.random.default_rng(k)
    bh, bw = int(rng.integers(1, h + 1)), int(rng.integers(1, w + 1))
    return int(rng.integers(0, h - bh + 1)), int(rng.integers(0, w - bw + 1)), bh, bw


DECODER_CASES = [
    ("4:2:0 8 bit, top-left box, odd size", lambda: obu.inter_stream(31, 99, 67, n_frames=3, bpc=8, motion_modes=1),
     dict(crop=(0, 0, 61, 93), flip=True, size=(24, 40))),
    ("4:2:0 10 bit, bottom-right box at odd top / left, antialiased", lambda: obu.inter_stream(32, 130, 70, n_frames=3, bpc=10,
                                                                                                film_grain=1),
     dict(crop=(13, 37, 57, 93), flip=lambda k: k % 2 == 0, size=(9, 14), antialias=True, dtype="bfloat16", layout="hwc",
          **IMAGENET)),
    ("4:2:0 8 bit, random boxes and flips per picture, batched", lambda: obu.inter_stream(33, 96, 64, n_frames=4, bpc=8),
     dict(crop=_random_box, flip=lambda k: k != 1, size=(17, 23), antialias=True, batch=3, dtype="float16")),
    ("4:0:0 10 bit, 1x1 box at odd position, native size", lambda: obu.inter_stream(34, 61, 45, n_frames=2, bpc=10, layout="400"),
     dict(crop=(7, 9, 1, 1), flip=True)),
    ("4:0:0 10 bit, odd box, antialiased", lambda: obu.inter_stream(34, 61, 45, n_frames=2, bpc=10, layout="400"),
     dict(crop=(3, 5, 41, 55), flip=False, size=(6, 5), antialias=True)),
    ("4:2:2 10 bit, odd top, odd left rounded, native size",
     lambda: __import__("test_stream")._valid_422("inter", 96, 64, 10, 1, motion_modes=1, film_grain=1)[0],
     dict(crop=(5, 3, 51, 88), flip=True, layout="hwc", chroma_siting="topleft", want_siting="topleft")),
    ("4:4:4 8 bit, odd box, antialiased", lambda: obu.intra_stream(35, 72, 50, n_frames=2, bpc=8, layout="444"),
     dict(crop=(1, 3, 49, 69), flip=True, size=(11, 30), antialias=True, matrix="identity")),
    ("4:4:4 10 bit, box touching right and bottom, enlarged", lambda: obu.intra_stream(36, 72, 50, n_frames=2, bpc=10, layout="444"),
     dict(crop=(41, 63, 9, 9), flip=True, size=(20, 13))),
    ("4:2:0 10 bit, 1x1 box at the bottom-right corner", lambda: obu.inter_stream(37, 83, 57, n_frames=2, bpc=10),
     dict(crop=(56, 82, 1, 1), flip=True, size=(3, 5))),
]


@pytest.mark.emu
@pytest.mark.parametrize("name,make,kw", DECODER_CASES, ids=[c[0] for c in DECODER_CASES])
def test_tensors_crop_flip_emu(emu_dec, name, make, kw):
    _check_tensors(emu_dec, make(), **kw)


@pytest.mark.emu
def test_tensors_size_none_is_the_aligned_box_emu(emu_dec):
    tus = obu.inter_stream(38, 64, 48, n_frames=2, bpc=8)
    got = _check_tensors(emu_dec, tus, (3, 5, 20, 30), False)
    assert all(tuple(g.shape) == (3, 21, 31) for g in got)


@pytest.mark.emu
def test_clips_crop_flip_emu(emu_dec):
    """per-stream boxes and flips: every picture of a clip is what tensors() of its stream exports with that box and flip;
    a callable box is asked once per stream, with the size of its first sampled picture"""
    streams = TC._mixed_streams()
    counts = [len(DO._ref_pictures(s)) for s in streams]
    starts = [max(0, c - 4) for c in counts]
    boxes = [(3, 5, 40, 61), (0, 1, 64, 95), (11, 13, 39, 59), (44, 60, 1, 1), (1, 0, 56, 83)]
    flips = [True, False, True, True, False]
    kw = dict(size=(13, 9), dtype="float16", layout="hwc", antialias=True, **IMAGENET)
    x = emu_dec.clips(streams, frames=2, step=2, start=starts, alloc=TC._alloc, crop=boxes, flip=flips, **kw)
    for i, tus in enumerate(streams):
        t_all = list(emu_dec.tensors(tus, alloc=TE._np_alloc, crop=boxes[i], flip=flips[i], **kw))
        name, full = TC.MIXED_COLORS.get(i, ("bt709", False))
        for t in range(2):
            g = TE._host_bits(x[i, t], "float16")
            assert np.array_equal(g, TE._host_bits(t_all[starts[i] + 2 * t], "float16")), (i, t)
            w, h, bpc, lay, rp = DO._ref_pictures(tus)[starts[i] + 2 * t]
            want = _mirror(stream.tensor_reference(stream.crop_planes(rp, lay, stream.align_crop(boxes[i], w, h, lay)), bpc, lay,
                                                   (13, 9), name, full, "topleft" if i == 4 else "left", antialias=True,
                                                   **IMAGENET), flips[i]).transpose(1, 2, 0)
            assert np.array_equal(g, TE._bits(want, "float16")), (i, t)
    calls = []

    def crop(i, h, w):
        calls.append((i, h, w))
        return (h // 4, w // 3, h // 2, w // 2)
    streams = streams[:3]
    x = emu_dec.clips(streams, frames=2, step=1, start=0, size=(8, 12), alloc=TC._alloc, crop=crop, flip=True)
    assert sorted(calls) == sorted((i, DO._ref_pictures(s)[0][1], DO._ref_pictures(s)[0][0]) for i, s in enumerate(streams))
    for i, tus in enumerate(streams):
        name, full = TC.MIXED_COLORS.get(i, ("bt709", False))
        for t in range(2):
            w, h, bpc, lay, rp = DO._ref_pictures(tus)[t]
            box = stream.align_crop((h // 4, w // 3, h // 2, w // 2), w, h, lay)
            want = _mirror(stream.tensor_reference(stream.crop_planes(rp, lay, box), bpc, lay, (8, 12), name, full, "left"), True)
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)


@pytest.mark.emu
def test_crop_flip_errors_emu(emu_dec):
    """boxes outside the picture and bad arguments raise ValueError naming the picture or stream; nothing is left open"""
    tus = obu.inter_stream(39, 64, 48, n_frames=3, bpc=8)
    for kw, match in [(dict(crop=(0, 0, 49, 10)), "picture 0"), (dict(crop=(40, 0, 9, 10)), "picture 0"),
                      (dict(crop=(0, 60, 10, 5)), "picture 0"), (dict(crop=(0, 0, 0, 5)), "picture 0"),
                      (dict(crop=lambda k, h, w: (0, 0, h, w + k)), "picture 1"), (dict(crop=(1, 2, 3)), "crop"),
                      (dict(crop="box"), "crop"), (dict(flip=1), "flip"), (dict(flip="yes"), "flip"),
                      (dict(flip=lambda k: k), "picture 0"), (dict(crop=lambda k, h, w: None if k else (0, 0, 1.5, 2)), "picture 0")]:
        with pytest.raises(ValueError, match=match):
            list(emu_dec.tensors(tus, alloc=TE._np_alloc, **kw))
    good = [obu.inter_stream(80 + k, 64, 48, n_frames=4, bpc=8) for k in range(3)]
    for kw, match in [(dict(crop=[(0, 0, 8, 8), (0, 0, 49, 8), (0, 0, 8, 8)]), "stream 1 picture"),
                      (dict(crop=lambda i, h, w: (0, 0, h, w + (i == 2))), "stream 2 picture"),
                      (dict(crop=[(0, 0, 8, 8)] * 2), "crop"), (dict(flip=[True, False]), "flip"), (dict(flip=1), "flip"),
                      (dict(crop=(0, 0, 8)), "crop")]:
        with pytest.raises(ValueError, match=match):
            emu_dec.clips(good, frames=2, alloc=TC._alloc, **kw)
    TC._check_clips(emu_dec, good, 2, 1, 1)                   # the decoder is still usable


@pytest.mark.emu
def test_hook_rejects_bad_boxes_emu(emu_dec):
    """b200hook_export_tensor takes boxes as they are: one outside the picture or at an odd chroma offset is an error and
    exports nothing"""
    tus = obu.inter_stream(40, 64, 48, n_frames=1, bpc=8)
    out = TE._np_alloc((3, 4, 4), "float32")
    rcs = []

    def export(h, info):
        job = emu_dec._tensor_job(h, info, out.ctypes.data, 4, 4, "float32", "chw", None, None, "auto", None, "left", False, True)
        pic = emu_dec.dll.refdrv_stream_picture(h)
        for box in ((1, 0, 4, 4), (0, 1, 4, 4), (0, 0, 49, 4), (0, 0, 4, 65), (-2, 0, 4, 4), (0, 0, 0, 4)):
            rcs.append(emu_dec.dll.b200hook_export_tensor(pic, C.byref(job), (C.c_int32 * 4)(*box), None))
        return None
    list(emu_dec._decode(tus, export))
    assert rcs == [-1] * 6
    assert (out.view(np.uint32) == np.full(1, 0x5a, np.float32).view(np.uint32)).all()


@pytest.fixture(scope="module")
def emu_dec(hooked_library):
    refs.emu_lib()
    d = stream.DeviceDecoder(backend=DO._emu_path(), serialize=True, apply_grain=1)
    yield d
    d.release()


@pytest.fixture(scope="module")
def hooked_library():
    import os
    stream.build_hooked()
    if not os.path.exists(stream.HOOKED_SO):
        pytest.skip("%s not built" % stream.HOOKED_SO)


# ---- on the device ------------------------------------------------------------------------------------------------
GPU_CASES = [(TE.Case(8, 1, 1920, 1080, (224, 224), "bfloat16", "chw", "left", "bt709", False, **IMAGENET), 1),
             (TE.Case(8, 1, 1920, 1080, (223, 221), "float32", "hwc", "left", "bt709", False, offset=1), 0),
             (TE.Case(10, 1, 3840, 2160, (224, 224), "bfloat16", "chw", "left", "bt2020", True, **IMAGENET), 1),
             (TE.Case(10, 1, 3840, 2160, (1080, 1918), "float16", "hwc", "center", "bt709", False, offset=1), 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GPU_CASES)))
def test_flip_kernel_gpu(idx):
    from dav1d_b200 import _lib
    c, aa = GPU_CASES[idx]
    got, want = _run(c, 6000 + idx, aa, 1, _lib.get_lib(), device=True)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


@pytest.mark.gpu
def test_batch_of_30_gpu():
    """30 cropped, antialiased jobs of 1080p 8 bit and 4K 10 bit pictures into 224 x 224 in one call (two launches of the
    8-bit class would be needed at more than 24), every other one flipped: each is the definition"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    rng = np.random.default_rng(30)
    kinds = [(8, 1920, 1080)] * 26 + [(10, 3840, 2160)] * 4
    c0 = TE.Case(8, 1, 1, 1, (224, 224), "bfloat16", "chw")
    pc, py, m = TE._pitches(c0)
    slot = m + TE.GUARD
    a = torch.full((len(kinds) * slot + TE.GUARD,), 0x7e57, dtype=torch.int16, device="cuda")
    jobs = (stream.TensorJob * len(kinds))()
    keep, wants = [], []
    for k, (bpc, w, h) in enumerate(kinds):
        full = TE.Case(bpc, 1, w, h, (224, 224), "bfloat16", "chw", "left", "bt709", bool(k % 2), **IMAGENET)
        planes = TE._planes(rng, full)
        box = stream.align_crop(_random_box(k + 100, h, w), w, h, 1)
        cp = stream.crop_planes(planes, 1, box)
        c = TE.Case(bpc, 1, box[3], box[2], (224, 224), "bfloat16", "chw", "left", "bt709", bool(k % 2), **IMAGENET)
        src, offs, strides = TE._source(planes, 1, extra=64)
        offs = [offs[0] + box[0] * strides[0] + box[1]] + [offs[p] + (box[0] >> 1) * strides[p] + (box[1] >> 1) for p in (1, 2)]
        d = torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda()
        keep.append(d)
        jobs[k] = TE._job(c, d.data_ptr(), offs, strides, a.data_ptr() + (TE.GUARD + k * slot) * 2, pc, py)
        jobs[k].antialias, jobs[k].flip = 1, k % 2
        wants.append(_expected(c, cp, pc, py, m, np.uint16(0x7e57), 1, k % 2))
    assert lib.b200_export_tensor_batch(jobs, len(kinds), None) == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    got = TE._host_bits(a, "bfloat16")
    for k in range(len(kinds)):
        assert np.array_equal(got[TE.GUARD + k * slot:TE.GUARD + k * slot + m], wants[k]), k
    assert (got[:TE.GUARD] == 0x7e57).all()


@pytest.mark.gpu
def test_tensors_and_clips_gpu(hooked_library, monkeypatch):
    """RandomResizedCrop + flip through tensors() and clips() on a non-default stream: 1080p 8 bit with grain and 4K 10
    bit to 224 x 224 bf16, antialiased, a random box and flip per picture / per stream"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)
    streams = [obu.inter_stream(630, 1920, 1080, n_frames=5, bpc=8, log2_cols=2, log2_rows=1, motion_modes=1, film_grain=1),
               obu.inter_stream(631, 3840, 2160, n_frames=5, bpc=10, log2_cols=2, log2_rows=1, motion_modes=1)]
    dec = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for tus in streams:
            got = _check_tensors(dec, tus, _random_box, lambda k: k % 2 == 1, size=(224, 224), dtype="bfloat16", alloc=None,
                                 antialias=True, batch=4, **IMAGENET)
            assert [g.shape[0] for g in got] == [4, 1] and all(g.is_cuda for g in got)
        boxes = [(101, 333, 871, 1201), (2000, 3000, 159, 839)]
        x = dec.clips(streams, frames=2, step=2, size=(224, 224), dtype="float32", antialias=True, crop=boxes, flip=[True, False])
    s.synchronize()
    assert x.is_cuda and tuple(x.shape) == (2, 2, 3, 224, 224)
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        for t in range(2):
            w, h, bpc, lay, rp = ref[2 * t]
            box = stream.align_crop(boxes[i], w, h, lay)
            want = _mirror(stream.tensor_reference(stream.crop_planes(rp, lay, box), bpc, lay, (224, 224), "bt709", False, "left",
                                                   antialias=True), i == 0)
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)
    dec.release()
