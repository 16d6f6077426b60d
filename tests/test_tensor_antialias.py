"""Antialiased tensor export (B200TensorJob.antialias = 1, export_tensor_aa_kernel in dav1d_b200/csrc/export.cu;
antialias=True in stream.DeviceDecoder.tensors / clips). The numpy statement of include/b200av1.h (stream.tensor_reference
with antialias=True, stream.tensor_weights) is pinned against torch's interpolate(antialias=True), against a float64
statement of the triangle filter and against ramps that show the siting; the kernel must equal it bit for bit, and must
leave every export without a reduced luma axis exactly as the bilinear export writes it. CPU tests run the CUDA sources on
the host emulator, GPU tests run the CUDA library into torch CUDA tensors."""
import ctypes as C

import numpy as np
import pytest

import refs
from dav1d_b200 import obu, stream

import test_clips as TC
import test_stream_device_output as DO
import test_tensor_export as TE

DTYPES = list(stream.TENSOR_DTYPES)
SITINGS = list(stream.SITINGS)
IMAGENET = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))


def _triangle(out, inn, n):
    """float64 [out, n] weights of torch's antialiased bilinear resize along one axis, stated directly: a triangle of
    half-width inn / out around the output's centre, clipped to the picture and renormalised; plain bilinear (clamped
    taps) where the axis is not reduced"""
    scale = inn / out
    c = (np.arange(out) + 0.5) * scale - 0.5
    j = np.arange(n)[None, :]
    if scale <= 1:
        c = np.maximum(c, 0)
        i0 = np.minimum(np.floor(c).astype(int), n - 1)
        f = c - np.floor(c)
        W = np.zeros((out, n))
        np.add.at(W, (np.arange(out), i0), 1 - f)
        np.add.at(W, (np.arange(out), np.minimum(i0 + 1, n - 1)), f)
        return W
    W = np.maximum(0, 1 - np.abs(j - c[:, None]) / scale)
    return W / W.sum(1, keepdims=True)


def _random_rgb(rng, shape, bpc):
    bdmax = (1 << bpc) - 1
    return [rng.integers(0, bdmax + 1, shape) for _ in range(3)], bdmax


GEOMETRIES = [((37, 53), (17, 29)), ((64, 48), (15, 7)), ((9, 200), (40, 3)), ((1080, 1920), (224, 224)),
              ((100, 100), (99, 51)), ((300, 500), (299, 7)), ((120, 90), (7, 90)), ((61, 400), (100, 13)),
              ((184, 291), (72, 1)), ((480, 640), (1, 1)), ((5, 333), (1, 9)), ((101, 101), (100, 100)),
              ((256, 64), (4, 1))]


# ---- the numpy statement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,size", GEOMETRIES)
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_reference_is_torch_antialias(shape, size, bpc):
    """identity matrix on 4:4:4: torch's interpolate(bilinear, antialias=True) within the quantisation of positions to
    1/256 sample (3/256 + 1/4 code value; 1/256 when both axes are reduced 2x or more), for outputs of length >= 2 (torch's
    own kernel is off for length 1); the float64 triangle formula within the same bound everywhere"""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(bpc * 1000 + shape[0] + size[1])
    planes, bdmax = _random_rgb(rng, shape, bpc)
    got = stream.tensor_reference(planes, bpc, 3, size, "identity", True, "left", antialias=True)
    rgb = np.stack([planes[2], planes[0], planes[1]]).astype(np.float64) / bdmax
    tol = 3 / 256 + 1 / (4 * bdmax) + 1e-6
    exact = _triangle(size[0], shape[0], shape[0]) @ rgb @ _triangle(size[1], shape[1], shape[1]).T
    assert np.abs(got - exact).max() <= tol
    if min(size) >= 2:
        want = F.interpolate(torch.from_numpy(rgb)[None], size=size, mode="bilinear", align_corners=False, antialias=True)[0].numpy()
        reduced2 = shape[0] >= 2 * size[0] and shape[1] >= 2 * size[1]
        assert np.abs(got - want).max() <= (1 / 256 + 1e-6 if reduced2 else tol)


@pytest.mark.parametrize("out,inn,s,k", [(224, 1920, 0, 0), (224, 1080, 1, 1), (7, 4000, 0, 0), (1, 65536, 0, 0),
                                         (3, 5, 1, 0), (100, 101, 0, 0), (13, 8, 1, 1), (1, 2, 1, 1)])
def test_weights_sum_and_taps(out, inn, s, k):
    """every row sums to 2^14 exactly, no weight is negative, and each is within 2^-14 of the exact share t_j / T"""
    n = (inn + s) >> s
    W = stream.tensor_weights(out, inn, n, s, k)
    assert W.shape == (out, n) and (W >= 0).all() and (W.sum(1) == 1 << 14).all()
    sigma = inn * (1 << (8 - s)) // out
    if sigma > 256:
        x = np.arange(out)
        P = ((2 * x + 1) * inn - (1 + k) * out) * (1 << (7 - s)) // out
        t = np.maximum(sigma - np.abs(256 * np.arange(n)[None, :] - P[:, None]), 0).astype(np.float64)
        assert np.abs(W - t / t.sum(1, keepdims=True) * (1 << 14)).max() <= 1


@pytest.mark.parametrize("siting", SITINGS)
@pytest.mark.parametrize("ratio", [4, 8])
def test_siting_ramps(siting, ratio):
    """a luma ramp and a 4:2:0 chroma ramp through reduced axes give, where no tap is clipped, the ramp's value at the
    output's centre (luma position (x + 1/2) * IN / OUT - 1/2, chroma as sited) within 1 Q unit. The reductions keep the
    triangle's half-width a whole number of samples on both planes, where its samples are centred exactly."""
    a, b, w, h = 100, 16, 240, 120
    ow, oh = int(w / ratio), int(h / ratio)
    kx, ky = stream.SITINGS[siting]
    for s, k, n, inn, out in ((0, 0, w, w, ow), (1, kx, w // 2, w, ow), (1, ky, h // 2, h, oh)):
        ramp = a + b * np.arange(n)
        q = (stream.tensor_weights(out, inn, n, s, k) @ ramp + (1 << 8)) >> 9       # H' of one row
        q = (q * (1 << 14) + (1 << 16)) >> 17                                        # Q of a flat column
        c = ((2 * np.arange(out) + 1) * inn / out - 1 - k) / (1 << (1 + s))
        half = inn / out / (1 << s)
        inner = (c - half >= 0) & (c + half <= n - 1)
        assert inner.sum() >= out // 2
        assert np.abs(q[inner] - 4 * (a + b * c[inner])).max() <= 1, (s, k)


def _noop_geometries():
    return [((37, 53), None), ((20, 30), (61, 97)), ((64, 48), (64, 48)), ((299, 300), (299, 299)), ((9, 200), (40, 200)),
            ((100, 100), (300, 100)), ((1, 1), (5, 7))]


@pytest.mark.parametrize("shape,size", _noop_geometries())
def test_reference_noop_without_reduction(shape, size):
    rng = np.random.default_rng(shape[0])
    planes, _ = _random_rgb(rng, shape, 10)
    planes = [planes[0], planes[1][:(shape[0] + 1) // 2, :(shape[1] + 1) // 2], planes[2][:(shape[0] + 1) // 2, :(shape[1] + 1) // 2]]
    for siting in SITINGS:
        a = stream.tensor_reference(planes, 10, 1, size, "bt709", False, siting)
        b = stream.tensor_reference(planes, 10, 1, size, "bt709", False, siting, antialias=True)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- kernel level, emulator ---------------------------------------------------------------------------------------
def _expected(c, planes, pitch_c, pitch_y, n_elems, guard, antialias):
    ref = stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std,
                                  antialias=antialias)
    bits = TE._bits(ref, c.dtype)
    out = np.full(n_elems, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        idx = ch * pitch_c + y * pitch_y + x if c.lay == "chw" else y * pitch_y + 3 * x + ch
        out[idx] = bits[ch]
    return out


def _run(c, seed, antialias=1, lib=None, device=False):
    """one job into a guarded destination; returns (what was written, what the definition says)"""
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
        j.antialias = antialias
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        assert lib.b200_export_tensor(C.byref(j), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
        s.synchronize()
        got = TE._host_bits(buf, c.dtype)
    else:
        buf = np.full(total, guard, et)
        j = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + (TE.GUARD + c.offset) * buf.itemsize, pc, py)
        j.antialias = antialias
        assert lib.b200_export_tensor(C.byref(j), None) == 0, lib.b200_last_error()
        got = buf
    want = np.full(total, guard, et)
    want[TE.GUARD + c.offset:TE.GUARD + c.offset + n] = _expected(c, planes, pc, py, n, guard, antialias)
    return got, want


def _kernel_cases():
    """(bpc, layout, w, h, size): reductions from 1.01x to 64x on either axis or both, one axis reduced and the other
    enlarged, 1 x 1 and 1 x N outputs, extreme aspect ratios, odd sizes; every dtype x layout x siting cycles through"""
    geo = [(101, 73, (72, 100)), (45, 27, (13, 22)), (61, 33, (33, 4)), (64, 48, (1, 1)), (97, 13, (40, 3)),
           (300, 7, (2, 5)), (9, 260, (4, 30)), (512, 9, (9, 8)), (130, 140, (2, 140)), (33, 31, (100, 11)),
           (200, 150, (75, 100)), (38, 21, (21, 37)), (256, 128, (2, 4)), (5, 400, (1, 3))]
    cases, k = [], 0
    for bpc in (8, 10, 12):
        for layout in (0, 1, 2, 3):
            for w, h, size in geo[(bpc + layout) % 3::3]:
                dtype, lay, siting = DTYPES[k % 3], ("chw", "hwc")[(k // 3) % 2], SITINGS[(k // 2) % 3]
                matrix = "identity" if layout == 3 and k % 4 == 0 else ["bt601", "bt709", "bt2020"][k % 3]
                kw = IMAGENET if k % 3 == 1 else {}
                cases.append(TE.Case(bpc, layout, w, h, size, dtype, lay, siting, matrix, bool(k % 2), offset=k % 2,
                                     pad=3 * (k % 3), **kw))
                k += 1
    for dtype in DTYPES:
        for lay in ("chw", "hwc"):
            for siting in SITINGS:
                cases.append(TE.Case(10, 1, 95, 61, (11, 23), dtype, lay, siting, "bt709", False, offset=1, pad=1))
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_kernel_matches_reference_emu(idx):
    got, want = _run(KERNEL_CASES[idx], 3000 + idx, lib=refs.emu_lib())
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s)" % (bad.size, bad[0], KERNEL_CASES[idx].__dict__)


@pytest.mark.emu
@pytest.mark.parametrize("shape,size", _noop_geometries())
def test_kernel_noop_without_reduction_emu(shape, size):
    """antialias = 1 writes exactly what antialias = 0 writes when no luma axis is reduced"""
    lib = refs.emu_lib()
    for k, siting in enumerate(SITINGS):
        c = TE.Case(10, 1, shape[1], shape[0], size, DTYPES[k], ("chw", "hwc")[k % 2], siting, "bt709", False, pad=1)
        a, _ = _run(c, 7, antialias=0, lib=lib)
        b, want = _run(c, 7, antialias=1, lib=lib)
        assert np.array_equal(a, b) and np.array_equal(b, want)


def _batch_cases(rng, n, dtype, lay):
    """TC's mixed batch, with every other job reduced 2 .. 20x and antialiased (a few antialiased jobs that reduce
    nothing go the bilinear way)"""
    cases = TC._batch_cases(rng, n, dtype, lay)
    aa = []
    for k, c in enumerate(cases):
        if k % 2:
            f = 2 + k % 19
            c.size = (max(1, c.h // f), max(1, c.w // (1 + k % 3)))
        aa.append(int(k % 4 != 0))
    return cases, aa


@pytest.mark.emu
@pytest.mark.parametrize("n", [1, TC.BATCH_MAX, TC.BATCH_MAX + 5, 2 * TC.BATCH_MAX + 5])
@pytest.mark.parametrize("dtype,lay", [("float32", "chw"), ("bfloat16", "hwc")])
def test_batch_matches_single_jobs_emu(n, dtype, lay):
    """antialiased and bilinear jobs of both bit-depth classes in one call: each writes what it writes alone, which is the
    definition"""
    lib = refs.emu_lib()
    cases, aa = _batch_cases(np.random.default_rng(n + 7), n, dtype, lay)
    srcs, spans, buf, guard = TC._batch_setup(cases, 700 + n)
    jobs = (stream.TensorJob * n)()
    want = np.full_like(buf, guard)
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        jobs[k].antialias = aa[k]
        want[at:at + m] = _expected(c, planes, pc, py, m, guard, aa[k])
    assert lib.b200_export_tensor_batch(jobs, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)
    single = np.full_like(buf, guard)
    for k in range(n):
        j = stream.TensorJob.from_buffer_copy(jobs[k])
        j.dst = single.ctypes.data + spans[k] * single.itemsize
        assert lib.b200_export_tensor(C.byref(j), None) == 0
    assert np.array_equal(buf, single)


@pytest.mark.emu
def test_batch_bad_arguments_emu():
    """antialias other than 0 / 1, and the other bad fields, on one job of a mixed batch: -2 and nothing written"""
    lib = refs.emu_lib()
    cases, aa = _batch_cases(np.random.default_rng(11), 6, "float32", "chw")
    srcs, spans, buf, guard = TC._batch_setup(cases, 11)
    jobs = (stream.TensorJob * 6)()
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        jobs[k].antialias = aa[k]
    for field, value in [("antialias", 2), ("antialias", -1), ("dtype", 1), ("bitdepth_max", 511), ("out_h", 0), ("src", None)]:
        for victim in (1, 4):
            bad = (stream.TensorJob * 6).from_buffer_copy(jobs)
            setattr(bad[victim], field, value)
            buf[:] = guard
            assert lib.b200_export_tensor_batch(bad, 6, None) == -2, field
            assert lib.b200_last_error()
            assert np.all(buf == guard), "a rejected batch wrote (%s)" % field
            if victim == 1 and field != "dtype":            # a dtype of its own is bad only within a batch
                assert lib.b200_export_tensor(C.byref(bad[1]), None) == -2
    assert lib.b200_export_tensor_batch(jobs, 6, None) == 0


# ---- decoder level, emulator --------------------------------------------------------------------------------------
def _check_tensors(dec, tus, size, dtype="float32", layout="chw", batch=None, want_siting="left", matrix="auto", full_range=None,
                   mean=None, std=None, alloc=TE._np_alloc, **kw):
    ref = DO._ref_pictures(tus)
    dec.stats(reset=True)
    got = list(dec.tensors(tus, size=size, dtype=dtype, layout=layout, mean=mean, std=std, matrix=matrix, full_range=full_range,
                           batch=batch, alloc=alloc, antialias=True, **kw))
    items = [t for g in got for t in g] if batch else got
    assert len(items) == len(ref)
    name = "bt709" if matrix == "auto" else matrix
    for k, ((w, h, bpc, layout_, rp), g) in enumerate(zip(ref, items)):
        want = stream.tensor_reference(rp, bpc, layout_, size, name, bool(full_range), want_siting, mean, std, antialias=True)
        if layout == "hwc":
            want = want.transpose(1, 2, 0)
        assert np.array_equal(TE._host_bits(g, dtype), TE._bits(want, dtype)), "picture %d differs (%s, %s)" % (k, dtype, layout)
    st = dec.stats(reset=True)
    assert st["d2h_bytes"] == 0 and st["frames"] > 0
    return got


DECODER_CASES = [
    ("10 bit odd size, grain", lambda: obu.inter_stream(21, 201, 135, n_frames=3, bpc=10, film_grain=1, motion_modes=2),
     dict(size=(24, 40), dtype="bfloat16", layout="hwc", batch=2, **IMAGENET)),
    ("4:0:0", lambda: obu.inter_stream(22, 131, 67, n_frames=2, bpc=10, layout="400"), dict(size=(9, 130), dtype="float16", full_range=True)),
    ("12 bit 4:4:4", lambda: obu.intra_stream(23, 96, 64, n_frames=2, bpc=12, layout="444", film_grain=1),
     dict(size=(150, 11), matrix="identity")),
    ("4:2:2", lambda: __import__("test_stream")._valid_422("inter", 128, 64, 10, 1, motion_modes=1, film_grain=1)[0],
     dict(size=(5, 31), chroma_siting="topleft", want_siting="topleft", layout="hwc", batch=3)),
]


@pytest.mark.emu
@pytest.mark.parametrize("name,make,kw", DECODER_CASES, ids=[c[0] for c in DECODER_CASES])
def test_tensors_antialias_emu(emu_dec, name, make, kw):
    _check_tensors(emu_dec, make(), **kw)


@pytest.mark.emu
def test_clips_antialias_emu(emu_dec):
    streams = TC._mixed_streams()
    counts = [len(DO._ref_pictures(s)) for s in streams]
    starts = [max(0, c - 3) for c in counts]
    x = emu_dec.clips(streams, frames=2, step=1, start=starts, size=(13, 9), dtype="float16", layout="chw", alloc=TC._alloc,
                      antialias=True, **IMAGENET)
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        name, full = TC.MIXED_COLORS.get(i, ("bt709", False))
        for t in range(2):
            w, h, bpc, lay, rp = ref[starts[i] + t]
            want = stream.tensor_reference(rp, bpc, lay, (13, 9), name, full, "topleft" if i == 4 else "left",
                                           antialias=True, **IMAGENET)
            assert np.array_equal(TE._host_bits(x[i, t], "float16"), TE._bits(want, "float16")), (i, t)


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
GPU_CASES = [TE.Case(8, 1, 1920, 1080, (224, 224), d, l, "left", "bt709", False, **IMAGENET) for d, l in
             (("bfloat16", "chw"), ("float32", "hwc"))] + \
    [TE.Case(10, 1, 3840, 2160, (224, 398), d, l, s, "bt2020", True, offset=1, **IMAGENET) for d, l, s in
     (("bfloat16", "chw", "left"), ("float16", "hwc", "center"))] + \
    [TE.Case(8, 1, 3840, 2160, (1080, 1920), "float16", "chw", "topleft", "bt709", False),
     TE.Case(12, 3, 1920, 1080, (1, 1), "float32", "chw", "left", "identity", False)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GPU_CASES)))
def test_kernel_matches_reference_gpu(idx):
    from dav1d_b200 import _lib
    got, want = _run(GPU_CASES[idx], 4000 + idx, lib=_lib.get_lib(), device=True)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


@pytest.mark.gpu
def test_batch_gpu():
    """24 antialiased jobs (1080p 8 bit and 4K 10 bit into 224 x 224) in one call equal the definition"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    kinds = [(8, 1920, 1080), (10, 3840, 2160)] * 12
    rng = np.random.default_rng(24)
    cases = [TE.Case(bpc, 1, w, h, (224, 224), "bfloat16", "chw", "left", "bt709", bool(k % 2)) for k, (bpc, w, h) in enumerate(kinds)]
    pc, py, m = TE._pitches(cases[0])
    slot = m + TE.GUARD
    a = torch.full((len(cases) * slot + TE.GUARD,), 0x7e57, dtype=torch.int16, device="cuda")
    jobs = (stream.TensorJob * len(cases))()
    planes, keep = [], []
    for k, c in enumerate(cases):
        p = TE._planes(rng, c)
        src, offs, strides = TE._source(p, c.layout, extra=64)
        d = torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda()
        keep.append(d)
        planes.append(p)
        jobs[k] = TE._job(c, d.data_ptr(), offs, strides, a.data_ptr() + (TE.GUARD + k * slot) * 2, pc, py)
        jobs[k].antialias = 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    assert lib.b200_export_tensor_batch(jobs, len(cases), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
    s.synchronize()
    got = TE._host_bits(a, "bfloat16")
    for k, c in enumerate(cases):
        want = _expected(c, planes[k], pc, py, m, np.uint16(0x7e57), 1)
        assert np.array_equal(got[TE.GUARD + k * slot:TE.GUARD + k * slot + m], want), k
    assert (got[:TE.GUARD] == 0x7e57).all()


@pytest.mark.gpu
def test_tensors_and_clips_gpu(hooked_library, monkeypatch):
    """tensors() and clips() with antialias=True into torch CUDA tensors on a non-default stream: 1080p 8 bit with grain
    and 4K 10 bit to 224 x 224"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)
    streams = [obu.inter_stream(620, 1920, 1080, n_frames=5, bpc=8, log2_cols=2, log2_rows=1, motion_modes=1, film_grain=1),
               obu.inter_stream(621, 3840, 2160, n_frames=5, bpc=10, log2_cols=2, log2_rows=1, motion_modes=1)]
    dec = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for tus in streams:
            got = _check_tensors(dec, tus, (224, 224), dtype="bfloat16", batch=4, alloc=None, **IMAGENET)
            assert [g.shape[0] for g in got] == [4, 1] and all(g.is_cuda for g in got)
        x = dec.clips(streams, frames=2, step=2, size=(224, 224), dtype="float32", antialias=True)
    s.synchronize()
    assert x.is_cuda and tuple(x.shape) == (2, 2, 3, 224, 224)
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        for t in range(2):
            w, h, bpc, lay, rp = ref[2 * t]
            want = stream.tensor_reference(rp, bpc, lay, (224, 224), "bt709", False, "left", antialias=True)
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)
    assert dec.stats()["d2h_bytes"] == 0
    dec.release()
