"""Bicubic tensor export (B200TensorJob.interpolation = B200_TENSOR_BICUBIC, the kCubic export_tensor_aa_kernel in
dav1d_b200/csrc/export.cu; interpolation="bicubic" in stream.DeviceDecoder.tensors / clips). The numpy statement of
include/b200av1.h (stream.tensor_reference with interpolation="bicubic", stream.cubic_weights) is pinned against torch's
interpolate(mode="bicubic") with and without antialias, against a float64 Keys statement and against ramps; the kernel
must equal it bit for bit. CPU tests run the CUDA sources on the host emulator, GPU tests run the CUDA library into torch
CUDA tensors."""
import ctypes as C

import numpy as np
import pytest

import refs
from dav1d_b200 import obu, stream

import test_clips as TC
import test_stream_device_output as DO
import test_tensor_antialias as TA
import test_tensor_export as TE

DTYPES = list(stream.TENSOR_DTYPES)
SITINGS = list(stream.SITINGS)
IMAGENET = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))


def _keys(x, a):
    x = np.abs(x)
    return np.where(x < 1, (a + 2) * x ** 3 - (a + 3) * x ** 2 + 1, np.where(x < 2, a * x ** 3 - 5 * a * x ** 2 + 8 * a * x - 4 * a, 0))


def _cubic(out, inn, n, antialias, centres=None):
    """float64 [out, n] weights of torch's bicubic resize along one axis, stated directly: Keys (a = -3/4) at four taps
    around the output's centre with the edge replicated; antialiased, Keys (a = -1/2) stretched by max(scale, 1), clipped
    to the picture and renormalised. centres: the outputs' positions in samples of this axis (by default luma's)"""
    scale = inn / out
    c = (np.arange(out) + 0.5) * scale - 0.5 if centres is None else centres
    W = np.zeros((out, n))
    if not antialias:
        f0 = np.floor(c).astype(int)
        for d in range(-1, 3):
            np.add.at(W, (np.arange(out), np.clip(f0 + d, 0, n - 1)), _keys(f0 + d - c, -0.75))
        return W
    support = max(scale, 1.0)
    W = _keys((np.arange(n)[None, :] - c[:, None]) / support, -0.5)
    return W / W.sum(1, keepdims=True)


def _mid_rgb(rng, shape, bpc):
    """planes drawn from the middle half of the code range: no clip of H' or Q fires"""
    bdmax = (1 << bpc) - 1
    return [rng.integers(bdmax // 4, 3 * bdmax // 4 + 1, shape) for _ in range(3)], bdmax


GEOMETRIES = TA.GEOMETRIES + [((20, 30), (61, 97)), ((7, 9), (50, 40)), ((64, 48), (64, 96)), ((33, 17), (100, 17)),
                              ((1, 5), (3, 11))]


# ---- the numpy statement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,size", GEOMETRIES)
@pytest.mark.parametrize("bpc", [8, 10, 12])
@pytest.mark.parametrize("antialias", [False, True])
def test_reference_is_torch_bicubic(shape, size, bpc, antialias):
    """identity matrix on 4:4:4, mid-range planes: torch's interpolate(mode="bicubic") within the quantisation of
    positions to 1/256 sample (3/256 + 1/4 code value) where torch's kernel is defined (outputs of length >= 2), the
    float64 Keys statement within the same bound everywhere"""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(bpc * 1000 + shape[0] + size[1] + antialias)
    planes, bdmax = _mid_rgb(rng, shape, bpc)
    got = stream.tensor_reference(planes, bpc, 3, size, "identity", True, "left", antialias=antialias, interpolation="bicubic")
    rgb = np.stack([planes[2], planes[0], planes[1]]).astype(np.float64) / bdmax
    tol = 3 / 256 + 1 / (4 * bdmax) + 1e-6
    exact = _cubic(size[0], shape[0], shape[0], antialias) @ rgb @ _cubic(size[1], shape[1], shape[1], antialias).T
    assert np.abs(got - exact).max() <= tol
    if min(size) >= 2:
        want = F.interpolate(torch.from_numpy(rgb)[None], size=size, mode="bicubic", align_corners=False, antialias=antialias)[0].numpy()
        assert np.abs(got - want).max() <= tol


SWEEP = [(224, 1920, 0, 0), (224, 1080, 1, 1), (398, 3840, 0, 0), (7, 4000, 0, 0), (1, 65536, 0, 0), (3, 5, 1, 0), (100, 101, 0, 0),
         (13, 8, 1, 1), (1, 2, 1, 1), (1, 1, 0, 0), (50, 1, 0, 0), (1080, 720, 0, 0), (1080, 720, 1, 1), (9, 2, 1, 0), (4, 256, 1, 1)]


@pytest.mark.parametrize("out,inn,s,k", SWEEP)
@pytest.mark.parametrize("antialias", [False, True])
def test_weights_sum_and_taps(out, inn, s, k, antialias):
    """every row sums to 2^14 exactly and each weight is within 1 of its exact share t_j / T; antialiased, T > 0 and no
    tap outside u_j < 512; plain, the weights of the four unclamped taps are a function of f = P & 255 alone"""
    n = (inn + s) >> s
    W = stream.cubic_weights(out, inn, n, s, k, antialias)
    assert W.shape == (out, n) and (W.sum(1) == 1 << 14).all()
    x = np.arange(out)
    P = ((2 * x + 1) * inn - (1 + k) * out) * (1 << (7 - s)) // out
    if antialias:
        sg = max(inn * (1 << (8 - s)) // out, 256)
        u = np.abs(256 * np.arange(n)[None, :] - P[:, None]) * 256 // sg
        t = stream._keys(u, -2)
        T = t.sum(1, keepdims=True)
        assert (T > 0).all()
        assert (W[u >= 512] == 0).all()
        assert np.abs(W - t / T * (1 << 14)).max() <= 1
    else:
        taps = (P >> 8)[:, None] + np.arange(-1, 3)
        t = stream._keys(np.abs(256 * taps - P[:, None]), -3)
        assert (t.sum(1) == 1 << 26).all()
        R = (np.cumsum(t, 1) + (1 << 11)) >> 12
        w4 = np.diff(R, axis=1, prepend=0)
        assert np.abs(w4 - t / (1 << 12)).max() <= 1
        by_f = {}
        for f, row in zip(P & 255, w4):
            assert by_f.setdefault(int(f), tuple(row)) == tuple(row)
        want = np.zeros((out, n), np.int64)
        np.add.at(want, (np.repeat(x, 4), np.clip(taps, 0, n - 1).ravel()), w4.ravel())
        assert np.array_equal(W, want)


def test_plain_weights_of_every_phase():
    """the 256 phases f of the plain rule: four weights that sum to 2^14, each within 1 of Keys (a = -3/4) at f / 256"""
    f = np.arange(256)
    P = 256 * 10 + f
    W = stream.cubic_weights(1, 1, 1, 0, 0)             # shape check of the n = 1 fold
    assert W.tolist() == [[1 << 14]]
    t = stream._keys(np.abs(256 * ((P >> 8)[:, None] + np.arange(-1, 3)) - P[:, None]), -3)
    w = np.diff((np.cumsum(t, 1) + (1 << 11)) >> 12, axis=1, prepend=0)
    exact = _keys(np.arange(-1, 3)[None, :] - f[:, None] / 256, -0.75) * (1 << 14)
    assert (w.sum(1) == 1 << 14).all() and np.abs(w - exact).max() <= 1


@pytest.mark.parametrize("antialias", [False, True])
@pytest.mark.parametrize("geo", [((2160, 3840), (224, 398)), ((1080, 1920), (224, 224)), ((720, 1280), (1080, 1920)),
                                 ((64, 64), (7, 5)), ((64, 64), (500, 300))])
def test_no_int32_overflow_on_checkerboards(antialias, geo):
    """0 / 4095 checkerboards at 12 bit (the largest |H| and V a cubic's negative lobes allow): H and V stay inside int32"""
    (h, w), (oh, ow) = geo
    for phase in (0, 1):
        p = np.where((np.add.outer(np.arange(h), np.arange(w)) + phase) % 2, 4095, 0).astype(np.int64)
        wx = stream.cubic_weights(ow, w, w, 0, 0, antialias)
        wy = stream.cubic_weights(oh, h, h, 0, 0, antialias)
        H = p @ wx.T
        assert np.abs(H).max() < 2 ** 31
        hq = np.clip((H + (1 << 9)) >> 10, 0, 16 * 4095)
        V = wy @ hq
        assert np.abs(V).max() < 2 ** 31
        # and every partial sum the kernel forms on the way (positive and negative parts apart) as well
        assert (np.maximum(wx, 0) @ np.full(w, 4095)).max() < 2 ** 31 and (np.maximum(wy, 0) @ np.full(h, 16 * 4095)).max() < 2 ** 31


@pytest.mark.parametrize("antialias", [False, True])
@pytest.mark.parametrize("bpc", [8, 12])
def test_constant_picture_stays_constant(antialias, bpc):
    for (h, w), size in [((37, 53), (17, 29)), ((20, 30), (61, 97)), ((1080, 1920), (224, 224)), ((5, 333), (1, 9))]:
        v = (1 << bpc) // 3
        planes = [np.full((h, w), v)] * 3
        got = stream.tensor_reference(planes, bpc, 3, size, "identity", True, antialias=antialias, interpolation="bicubic")
        assert (got == np.float32(4 * v) * stream.tensor_scale_bias(bpc)[0][0]).all()


@pytest.mark.parametrize("siting", SITINGS)
@pytest.mark.parametrize("antialias", [False, True])
@pytest.mark.parametrize("ratio", [0.5, 0.75, 4])
def test_siting_ramps(siting, antialias, ratio):
    """a luma ramp and a 4:2:0 chroma ramp, away from the edges: what the float64 Keys filter centred on the output's
    position (luma (x + 1/2) * IN / OUT - 1/2, chroma as sited) gives, within 1 Q unit. Antialiased (a = -1/2, which
    reproduces linear functions) that is the ramp's value at the centre; plain (a = -3/4) it is not quite."""
    a, b, w, h = 100, 16, 240, 120
    ow, oh = int(w / ratio), int(h / ratio)
    kx, ky = stream.SITINGS[siting]
    for s, k, n, inn, out in ((0, 0, w, w, ow), (1, kx, w // 2, w, ow), (1, ky, h // 2, h, oh)):
        ramp = a + b * np.arange(n)
        q = np.clip((stream.cubic_weights(out, inn, n, s, k, antialias) @ ramp + (1 << 9)) >> 10, 0, 16 * 4095)  # H' of one row
        q = (q * (1 << 14) + (1 << 15)) >> 16                                                                    # Q of a flat column
        c = ((2 * np.arange(out) + 1) * inn / out - 1 - k) / (1 << (1 + s))
        half = 2 * max(inn / out / (1 << s), 1)
        inner = (c - half >= 0) & (c + half <= n - 1)
        assert inner.sum() >= out // 2
        want = 4 * _cubic(out, inn >> s, n, antialias, c) @ ramp
        assert np.abs(q[inner] - want[inner]).max() <= 1, (s, k)
        if antialias:
            assert np.abs(q[inner] - 4 * (a + b * c[inner])).max() <= 1, (s, k)


def test_plain_replicates_and_antialiased_renormalises():
    """at the left edge of an enlargement: plain bicubic adds the weights of the taps left of the picture to sample 0,
    antialiased bicubic drops them and renormalises the rest, so the two differ exactly there"""
    out, inn = 40, 10
    plain, aa = stream.cubic_weights(out, inn, inn), stream.cubic_weights(out, inn, inn, antialias=True)
    # output 0 sits at -0.375: plain taps -2 .. 1 clamp to 0, 0, 0, 1
    assert plain[0, 2:].sum() == 0 and plain[0, 0] + plain[0, 1] == 1 << 14 and plain[0, 0] > 1 << 14
    x = (np.arange(out) + 0.5) * inn / out - 0.5
    for r in range(out):
        P = ((2 * r + 1) * inn - out) * 128 // out
        taps = np.arange((P >> 8) - 1, (P >> 8) + 3)
        if taps.min() >= 0 and taps.max() <= inn - 1:           # no tap beyond an edge: the weights of a = -3/4
            assert np.abs(plain[r, taps] - _keys(taps - x[r], -0.75) * (1 << 14)).max() <= 2
    exact = _cubic(out, inn, inn, True)
    assert np.abs(aa - exact * (1 << 14)).max() <= 2
    assert not np.array_equal(plain[0], aa[0]) and (aa[0] >= -(1 << 14)).all()


@pytest.mark.parametrize("antialias", [False, True])
def test_same_size_444_is_the_bilinear_export(antialias):
    """a same-size 4:4:4 export is Q = 4 S under either cubic rule: bit for bit the bilinear export"""
    rng = np.random.default_rng(5)
    for bpc in (8, 10, 12):
        planes, _ = TA._random_rgb(rng, (23, 41), bpc)
        for matrix in ("identity", "bt709"):
            a = stream.tensor_reference(planes, bpc, 3, None, matrix, False)
            b = stream.tensor_reference(planes, bpc, 3, None, matrix, False, antialias=antialias, interpolation="bicubic")
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_reference_rejects_other_interpolations():
    planes = [np.zeros((4, 4), np.int64)] * 3
    for bad in ("nearest", "BICUBIC", 1, None):
        with pytest.raises(ValueError):
            stream.tensor_reference(planes, 8, 3, (2, 2), interpolation=bad)


# ---- kernel level, emulator ---------------------------------------------------------------------------------------
def _expected(c, planes, pitch_c, pitch_y, n_elems, guard, antialias, interpolation, flip=False):
    ref = stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std,
                                  antialias=antialias, interpolation=interpolation)
    if flip:
        ref = ref[:, :, ::-1].copy()
    bits = TE._bits(ref, c.dtype)
    out = np.full(n_elems, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        idx = ch * pitch_c + y * pitch_y + x if c.lay == "chw" else y * pitch_y + 3 * x + ch
        out[idx] = bits[ch]
    return out


INTERP = ("bilinear", "bicubic")


def _run(c, seed, antialias, lib, device=False, flip=False, interpolation="bicubic", planes=None):
    """one job into a guarded destination; returns (what was written, what the definition says)"""
    rng = np.random.default_rng(seed)
    planes = TE._planes(rng, c) if planes is None else planes
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
    else:
        buf = np.full(total, guard, et)
        j = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + (TE.GUARD + c.offset) * buf.itemsize, pc, py)
    j.antialias, j.flip, j.interpolation = int(antialias), int(flip), stream.TENSOR_INTERPOLATIONS[interpolation]
    if device:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        assert lib.b200_export_tensor(C.byref(j), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
        s.synchronize()
        got = TE._host_bits(buf, c.dtype)
    else:
        assert lib.b200_export_tensor(C.byref(j), None) == 0, lib.b200_last_error()
        got = buf
    want = np.full(total, guard, et)
    want[TE.GUARD + c.offset:TE.GUARD + c.offset + n] = _expected(c, planes, pc, py, n, guard, antialias, interpolation, flip)
    return got, want


def _kernel_cases():
    """(bpc, layout, w, h, size, antialias, flip): 1 -> N, N -> 1, up to 64x reductions, enlargements, one axis reduced and
    the other enlarged, odd sizes; every dtype x layout x siting cycles through, with ragged and misaligned stores"""
    geo = [(101, 73, (72, 100)), (45, 27, (13, 22)), (61, 33, (33, 4)), (64, 48, (1, 1)), (97, 13, (40, 3)), (1, 1, (5, 7)),
           (300, 7, (2, 5)), (9, 260, (4, 30)), (512, 9, (9, 8)), (13, 17, (40, 29)), (33, 31, (100, 11)), (1, 9, (3, 1)),
           (200, 150, (75, 100)), (38, 21, (21, 37)), (256, 128, (2, 4)), (5, 400, (1, 3)), (20, 12, (61, 97)), (7, 1, (2, 9))]
    cases, k = [], 0
    for bpc in (8, 10, 12):
        for layout in (0, 1, 2, 3):
            for w, h, size in geo[(bpc + layout) % 3::3]:
                dtype, lay, siting = DTYPES[k % 3], ("chw", "hwc")[(k // 3) % 2], SITINGS[(k // 2) % 3]
                matrix = "identity" if layout == 3 and k % 4 == 0 else ["bt601", "bt709", "bt2020"][k % 3]
                kw = IMAGENET if k % 3 == 1 else {}
                cases.append((TE.Case(bpc, layout, w, h, size, dtype, lay, siting, matrix, bool(k % 2), offset=k % 2,
                                      pad=3 * (k % 3), **kw), bool(k % 2 == (k // 7) % 2), k % 5 == 2))
                k += 1
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_kernel_matches_reference_emu(idx):
    c, aa, flip = KERNEL_CASES[idx]
    got, want = _run(c, 5000 + idx, aa, refs.emu_lib(), flip=flip)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s, antialias %s)" % (bad.size, bad[0], c.__dict__, aa)


@pytest.mark.emu
@pytest.mark.parametrize("antialias", [False, True])
def test_kernel_long_taps_emu(antialias):
    """64x reductions and a 1000 -> 1 axis: antialiased columns span several tap windows and rows several chunks, so the
    running sums cross both; on 12-bit checkerboards with extreme codes, where the clips of H' and Q fire"""
    lib = refs.emu_lib()
    for k, (w, h, size) in enumerate([(1000, 70, (1, 3)), (64 * 3, 64 * 2, (2, 3)), (130, 900, (2, 1))]):
        c = TE.Case(12, 3, w, h, size, "float32", "chw", "left", "identity", True)
        board = np.where(np.add.outer(np.arange(h), np.arange(w)) % 2, 4095, 0).astype(np.uint16)
        got, want = _run(c, 0, antialias, lib, planes=[board, 4095 - board, board])
        assert np.array_equal(got, want), (w, h, size)
        got, want = _run(c, 6000 + k, antialias, lib)
        assert np.array_equal(got, want), (w, h, size)


@pytest.mark.emu
def test_kernel_same_size_444_is_the_bilinear_export_emu():
    lib = refs.emu_lib()
    for k, bpc in enumerate((8, 10, 12)):
        c = TE.Case(bpc, 3, 37, 29, None, DTYPES[k], ("chw", "hwc")[k % 2], "left", "bt709", False, pad=1)
        a, _ = _run(c, 9, False, lib, interpolation="bilinear")
        for aa in (False, True):
            b, want = _run(c, 9, aa, lib)
            assert np.array_equal(a, b) and np.array_equal(b, want)


def _batch_cases(rng, n, dtype, lay):
    """TC's mixed batch of both bit-depth classes, cycling through bilinear, antialiased bilinear (triangle), plain and
    antialiased bicubic jobs, with every other job reduced 2 .. 20x"""
    cases = TC._batch_cases(rng, n, dtype, lay)
    kinds = []
    for k, c in enumerate(cases):
        if k % 2:
            f = 2 + k % 19
            c.size = (max(1, c.h // f), max(1, c.w // (1 + k % 3)))
        kinds.append((("bilinear", "bicubic")[(k // 2) % 2], bool(k % 3), bool(k % 5 == 1)))
    return cases, kinds


@pytest.mark.emu
@pytest.mark.parametrize("n", [1, 7, TC.BATCH_MAX + 5, 2 * TC.BATCH_MAX + 5])
@pytest.mark.parametrize("dtype,lay", [("float32", "chw"), ("bfloat16", "hwc")])
def test_batch_matches_single_jobs_emu(n, dtype, lay):
    """bilinear, triangle, plain and antialiased cubic jobs, flipped and not, of both bit-depth classes in one call: each
    writes what it writes alone, which is the definition"""
    lib = refs.emu_lib()
    cases, kinds = _batch_cases(np.random.default_rng(n + 17), n, dtype, lay)
    srcs, spans, buf, guard = TC._batch_setup(cases, 900 + n)
    jobs = (stream.TensorJob * n)()
    want = np.full_like(buf, guard)
    for k, ((c, planes, src, offs, strides, pc, py, m), at, (interp, aa, flip)) in enumerate(zip(srcs, spans, kinds)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        jobs[k].antialias, jobs[k].flip, jobs[k].interpolation = int(aa), int(flip), stream.TENSOR_INTERPOLATIONS[interp]
        want[at:at + m] = _expected(c, planes, pc, py, m, guard, aa, interp, flip)
    assert lib.b200_export_tensor_batch(jobs, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)
    single = np.full_like(buf, guard)
    for k in range(n):
        j = stream.TensorJob.from_buffer_copy(jobs[k])
        j.dst = single.ctypes.data + spans[k] * single.itemsize
        assert lib.b200_export_tensor(C.byref(j), None) == 0
    assert np.array_equal(buf, single)


@pytest.mark.emu
def test_bad_interpolation_emu():
    """interpolation other than 0 / 1 on one job of a batch, or alone: -2 and nothing written"""
    lib = refs.emu_lib()
    cases, kinds = _batch_cases(np.random.default_rng(11), 6, "float32", "chw")
    srcs, spans, buf, guard = TC._batch_setup(cases, 11)
    jobs = (stream.TensorJob * 6)()
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        jobs[k] = TE._job(c, src.ctypes.data, offs, strides, buf.ctypes.data + at * buf.itemsize, pc, py)
        jobs[k].interpolation = stream.TENSOR_INTERPOLATIONS[kinds[k][0]]
    for value in (2, -1, 1 << 30):
        bad = (stream.TensorJob * 6).from_buffer_copy(jobs)
        bad[3].interpolation = value
        buf[:] = guard
        assert lib.b200_export_tensor_batch(bad, 6, None) == -2
        assert b"interpolation" in lib.b200_last_error()
        assert np.all(buf == guard)
        assert lib.b200_export_tensor(C.byref(bad[3]), None) == -2
    assert lib.b200_export_tensor_batch(jobs, 6, None) == 0


# ---- decoder level, emulator --------------------------------------------------------------------------------------
def _check_tensors(dec, tus, size, dtype="float32", layout="chw", batch=None, want_siting="left", matrix="auto", full_range=None,
                   mean=None, std=None, alloc=TE._np_alloc, antialias=False, crop=None, flip=False, **kw):
    ref = DO._ref_pictures(tus)
    dec.stats(reset=True)
    got = list(dec.tensors(tus, size=size, dtype=dtype, layout=layout, mean=mean, std=std, matrix=matrix, full_range=full_range,
                           batch=batch, alloc=alloc, antialias=antialias, crop=crop, flip=flip, interpolation="bicubic", **kw))
    items = [t for g in got for t in g] if batch else got
    assert len(items) == len(ref)
    name = "bt709" if matrix == "auto" else matrix
    for k, ((w, h, bpc, lay, rp), g) in enumerate(zip(ref, items)):
        if crop is not None:
            rp = stream.crop_planes(rp, lay, stream.align_crop(crop, w, h, lay))
        want = stream.tensor_reference(rp, bpc, lay, size, name, bool(full_range), want_siting, mean, std, antialias=antialias,
                                       interpolation="bicubic")
        if flip:
            want = want[:, :, ::-1]
        if layout == "hwc":
            want = want.transpose(1, 2, 0)
        assert np.array_equal(TE._host_bits(g, dtype), TE._bits(np.ascontiguousarray(want), dtype)), "picture %d differs" % k
    st = dec.stats(reset=True)
    assert st["d2h_bytes"] == 0 and st["frames"] > 0
    return got


DECODER_CASES = [
    ("10 bit odd size, grain, antialiased", lambda: obu.inter_stream(21, 201, 135, n_frames=3, bpc=10, film_grain=1, motion_modes=2),
     dict(size=(24, 40), dtype="bfloat16", layout="hwc", batch=2, antialias=True, **IMAGENET)),
    ("4:0:0 enlarged", lambda: obu.inter_stream(22, 131, 67, n_frames=2, bpc=10, layout="400"), dict(size=(90, 150), dtype="float16", full_range=True)),
    ("12 bit 4:4:4", lambda: obu.intra_stream(23, 96, 64, n_frames=2, bpc=12, layout="444", film_grain=1),
     dict(size=(150, 11), matrix="identity", antialias=True)),
    ("4:2:2", lambda: __import__("test_stream")._valid_422("inter", 128, 64, 10, 1, motion_modes=1, film_grain=1)[0],
     dict(size=(5, 31), chroma_siting="topleft", want_siting="topleft", layout="hwc", batch=3)),
    ("8 bit 4:2:0, crop and flip", lambda: obu.inter_stream(24, 160, 96, n_frames=2, bpc=8),
     dict(size=(20, 24), crop=(13, 37, 57, 93), flip=True, antialias=True)),
]


@pytest.mark.emu
@pytest.mark.parametrize("name,make,kw", DECODER_CASES, ids=[c[0] for c in DECODER_CASES])
def test_tensors_bicubic_emu(emu_dec, name, make, kw):
    _check_tensors(emu_dec, make(), **kw)


@pytest.mark.emu
def test_clips_bicubic_emu(emu_dec):
    streams = TC._mixed_streams()
    counts = [len(DO._ref_pictures(s)) for s in streams]
    starts = [max(0, c - 3) for c in counts]
    for aa in (False, True):
        x = emu_dec.clips(streams, frames=2, step=1, start=starts, size=(13, 9), dtype="float16", layout="chw", alloc=TC._alloc,
                          antialias=aa, interpolation="bicubic", **IMAGENET)
        for i, tus in enumerate(streams):
            ref = DO._ref_pictures(tus)
            name, full = TC.MIXED_COLORS.get(i, ("bt709", False))
            for t in range(2):
                w, h, bpc, lay, rp = ref[starts[i] + t]
                want = stream.tensor_reference(rp, bpc, lay, (13, 9), name, full, "topleft" if i == 4 else "left",
                                               antialias=aa, interpolation="bicubic", **IMAGENET)
                assert np.array_equal(TE._host_bits(x[i, t], "float16"), TE._bits(want, "float16")), (aa, i, t)


@pytest.mark.emu
def test_bad_interpolation_is_a_value_error_emu(emu_dec):
    tus = obu.intra_stream(23, 32, 16, n_frames=1)
    for bad in ("bicubic ", "nearest", 1, None):
        with pytest.raises(ValueError, match="interpolation"):
            list(emu_dec.tensors(tus, size=(8, 8), alloc=TE._np_alloc, interpolation=bad))
        with pytest.raises(ValueError, match="interpolation"):
            emu_dec.clips([tus], frames=1, alloc=TC._alloc, interpolation=bad)


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
GPU_CASES = [(TE.Case(8, 1, 1920, 1080, (224, 224), "bfloat16", "chw", "left", "bt709", False, **IMAGENET), True),
             (TE.Case(8, 1, 1920, 1080, (224, 224), "float32", "hwc", "left", "bt709", False), False),
             (TE.Case(10, 1, 3840, 2160, (224, 398), "bfloat16", "chw", "left", "bt2020", True, offset=1, **IMAGENET), True),
             (TE.Case(10, 1, 3840, 2160, (224, 398), "float16", "hwc", "center", "bt709", False), False),
             (TE.Case(8, 1, 1920, 1080, (1080, 1920), "float16", "chw", "topleft", "bt709", False), True),
             (TE.Case(10, 1, 3840, 2160, (1080, 1920), "float16", "chw", "left", "bt709", False), True),
             (TE.Case(8, 1, 1280, 720, (1080, 1920), "bfloat16", "chw", "left", "bt709", False), False),
             (TE.Case(12, 3, 1920, 1080, (1, 1), "float32", "chw", "left", "identity", False), True)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GPU_CASES)))
def test_kernel_matches_reference_gpu(idx):
    from dav1d_b200 import _lib
    c, aa = GPU_CASES[idx]
    got, want = _run(c, 7000 + idx, aa, _lib.get_lib(), device=True, flip=idx % 3 == 1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


@pytest.mark.gpu
def test_batch_of_30_gpu():
    """30 jobs in one call (1080p 8 bit and 4K 10 bit into 224 x 224: bilinear, triangle, plain and antialiased cubic,
    flipped and not): each equals the definition"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    kinds = [(8, 1920, 1080), (10, 3840, 2160)] * 15
    rng = np.random.default_rng(30)
    cases = [TE.Case(bpc, 1, w, h, (224, 224), "bfloat16", "chw", "left", "bt709", bool(k % 2)) for k, (bpc, w, h) in enumerate(kinds)]
    modes = [(("bilinear", "bicubic")[(k // 2) % 2], bool((k // 4) % 2 or k % 3 == 0), k % 5 == 0) for k in range(len(cases))]
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
        interp, aa, flip = modes[k]
        jobs[k].antialias, jobs[k].flip, jobs[k].interpolation = int(aa), int(flip), stream.TENSOR_INTERPOLATIONS[interp]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    assert lib.b200_export_tensor_batch(jobs, len(cases), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
    s.synchronize()
    got = TE._host_bits(a, "bfloat16")
    for k, c in enumerate(cases):
        interp, aa, flip = modes[k]
        want = _expected(c, planes[k], pc, py, m, np.uint16(0x7e57), aa, interp, flip)
        assert np.array_equal(got[TE.GUARD + k * slot:TE.GUARD + k * slot + m], want), (k, modes[k])
    assert (got[:TE.GUARD] == 0x7e57).all()


@pytest.mark.gpu
def test_tensors_and_clips_gpu(hooked_library, monkeypatch):
    """tensors() and clips() with interpolation="bicubic" into torch CUDA tensors on a non-default stream: 1080p 8 bit with
    grain and 4K 10 bit, antialiased to 224 x 224 and plain to 1080p"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)
    streams = [obu.inter_stream(630, 1920, 1080, n_frames=5, bpc=8, log2_cols=2, log2_rows=1, motion_modes=1, film_grain=1),
               obu.inter_stream(631, 3840, 2160, n_frames=5, bpc=10, log2_cols=2, log2_rows=1, motion_modes=1)]
    dec = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for tus in streams:
            got = _check_tensors(dec, tus, (224, 224), dtype="bfloat16", batch=4, alloc=None, antialias=True, **IMAGENET)
            assert [g.shape[0] for g in got] == [4, 1] and all(g.is_cuda for g in got)
        _check_tensors(dec, streams[1], (1080, 1920), dtype="float16", alloc=None)
        x = dec.clips(streams, frames=2, step=2, size=(224, 224), dtype="float32", antialias=True, interpolation="bicubic")
    s.synchronize()
    assert x.is_cuda and tuple(x.shape) == (2, 2, 3, 224, 224)
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        for t in range(2):
            w, h, bpc, lay, rp = ref[2 * t]
            want = stream.tensor_reference(rp, bpc, lay, (224, 224), "bt709", False, "left", antialias=True, interpolation="bicubic")
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)
    assert dec.stats()["d2h_bytes"] == 0
    dec.release()
