"""Tensor export (b200_export_tensor, dav1d_b200/csrc/export.cu; stream.DeviceDecoder.tensors): decoded pictures resized,
converted to RGB and normalised in one kernel. The numpy statement of include/b200av1.h (stream.tensor_reference) is pinned
against torch's bilinear interpolation and against ramps that show the chroma siting; the kernel must equal it bit for bit,
on random planes and on stock dav1d's pictures. CPU tests run the CUDA sources on the host emulator (numpy destinations),
GPU tests run the CUDA library into torch CUDA tensors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import refs
from dav1d_b200 import obu, stream

import test_stream_device_output as DO

DTYPES = list(stream.TENSOR_DTYPES)
SITINGS = list(stream.SITINGS)


@pytest.fixture(scope="module")
def hooked_library():
    stream.build_hooked()
    if not os.path.exists(stream.HOOKED_SO):
        pytest.skip("%s not built" % stream.HOOKED_SO)


def _bits(a, dtype):
    """raw bits of a float32 array rounded to `dtype` the way the export rounds (nearest even)"""
    a = np.ascontiguousarray(a, np.float32)
    if dtype == "float32":
        return a.view(np.uint32)
    if dtype == "float16":
        return a.astype(np.float16).view(np.uint16)
    import torch
    return torch.from_numpy(a).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def _host_bits(t, dtype):
    t = t.cpu() if hasattr(t, "cpu") else t
    if hasattr(t, "numpy"):
        import torch
        t = t.view(torch.int32 if dtype == "float32" else torch.int16).numpy()
    return t.view(np.uint32 if dtype == "float32" else np.uint16)


def _layout_of(layout):
    return {0: (1, 1), 1: (1, 1), 2: (1, 0), 3: (0, 0)}[layout]      # ss_hor, ss_ver (4:0:0 as the hooks pass it)


# ---- the numpy statement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,size", [((37, 53), (37, 53)), ((37, 53), (17, 29)), ((20, 30), (61, 97)), ((64, 48), (15, 7)),
                                        ((9, 200), (40, 3))])
@pytest.mark.parametrize("bpc", [8, 10])
def test_reference_is_torch_bilinear(shape, size, bpc):
    """identity matrix on 4:4:4 float pictures: torch's interpolate(bilinear, align_corners=False) to within the
    quantisation of the positions to 1/256 sample (per axis) and of the samples to 1/4 code value"""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(bpc * 100 + shape[0] + size[1])
    bdmax = (1 << bpc) - 1
    planes = [rng.integers(0, bdmax + 1, shape) for _ in range(3)]
    got = stream.tensor_reference(planes, bpc, 3, size, "identity", True, "left")
    x = torch.from_numpy(np.stack([planes[2], planes[0], planes[1]]).astype(np.float64) / bdmax)[None]
    want = F.interpolate(x, size=size, mode="bilinear", align_corners=False)[0].numpy()
    assert got.dtype == np.float32 and got.shape == (3,) + size
    assert np.abs(got - want).max() <= 2 / 256 + 1 / (4 * bdmax) + 1e-6


def _q(plane, oh, ow, h, w, s_hor, s_ver, kx, ky):
    """Q (2 fractional bits) of one plane resampled the way tensor_reference does"""
    p = plane.astype(np.int64)
    x0, x1, fx = stream.tensor_taps(ow, w, p.shape[1], s_hor, kx if s_hor else 0)
    y0, y1, fy = stream.tensor_taps(oh, h, p.shape[0], s_ver, ky if s_ver else 0)
    a = p[np.ix_(y0, x0)] * (256 - fx) + p[np.ix_(y0, x1)] * fx
    b = p[np.ix_(y1, x0)] * (256 - fx) + p[np.ix_(y1, x1)] * fx
    return (a * (256 - fy)[:, None] + b * fy[:, None] + (1 << 13)) >> 14


@pytest.mark.parametrize("siting", SITINGS)
def test_siting_ramps(siting):
    """a 4:2:0 chroma ramp a + b*i read at interior luma column X (row Y) gives a + b*X/2 on the even-sample siting and
    a + b*(X - 1/2)/2 midway; luma ramps at native size and at half size (output x reads luma 2x + 1/2)"""
    a, b, w, h = 100, 64, 40, 24
    kx, ky = stream.SITINGS[siting]
    X, Y = np.arange(4, w - 4), np.arange(4, h - 4)
    cols = np.broadcast_to(a + b * np.arange(w // 2), (h // 2, w // 2))
    rows = np.broadcast_to((a + b * np.arange(h // 2))[:, None], (h // 2, w // 2))
    qx = _q(cols, h, w, h, w, 1, 1, kx, ky)
    qy = _q(rows, h, w, h, w, 1, 1, kx, ky)
    assert np.array_equal(qx[5, X], 4 * a + 4 * b * (X - 0.5 * kx) / 2)
    assert np.array_equal(qy[Y, 5], 4 * a + 4 * b * (Y - 0.5 * ky) / 2)
    luma = np.broadcast_to(a + b * np.arange(w), (h, w))
    assert np.array_equal(_q(luma, h, w, h, w, 0, 0, 0, 0)[3, X], 4 * (a + b * X))
    half = _q(luma, h // 2, w // 2, h, w, 0, 0, 0, 0)[3, 2:-2]
    assert np.array_equal(half, 4 * (a + b * (2 * np.arange(2, w // 2 - 2) + 0.5)))
    # the same through tensor_reference: 4:2:0 with constant luma, the chroma ramp on Cr, full-range BT.709 red
    s, bdmax = 2, 1023
    cr = np.broadcast_to(512 + 8 * np.arange(w // 2), (h // 2, w // 2))
    planes = [np.full((h, w), 512), np.full((h // 2, w // 2), 512), cr]
    got = stream.tensor_reference(planes, 10, 1, None, "bt709", True, siting)
    cy, rv = stream.rgb_coefficients("bt709", True)[:2]
    qcr = 4 * 512 + 4 * 8 * (X - 0.5 * kx) / 2
    red = np.clip((cy * (4 * 512) + rv * (qcr.astype(np.int64) - (512 << s)) + 8192) >> 14, 0, 4 * bdmax)
    assert np.array_equal(got[0, 7, X], (red.astype(np.float32) * np.float32(1 / (4 * bdmax))).astype(np.float32))


def test_scale_and_bias():
    scale, bias = stream.tensor_scale_bias(10, [0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
    assert scale.dtype == np.float32 and scale[0] == np.float32(1 / (4 * 1023 * 0.229)) and bias[2] == np.float32(-0.406 / 0.225)
    with pytest.raises(ValueError):
        stream.tensor_scale_bias(8, [0, 0], [1, 1, 1])


# ---- ABI ----------------------------------------------------------------------------------------------------------
def test_tensor_job_layout_matches_the_library():
    assert refs.emu_lib().b200_struct_size(23) == C.sizeof(stream.TensorJob)


def test_null_backend_compiles_and_binds(hooked_library, tmp_path):
    """tools/null_backend.c (the host-side timing aid) provides every entry point the hooks bind"""
    so = str(tmp_path / "libnull.so")
    subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-shared", "-fPIC", "-o", so, os.path.join(refs.ROOT, "tools", "null_backend.c")],
                   check=True)
    dec = stream.HookedDecoder(backend=so)
    assert stream._bound[stream.HOOKED_SO] == so
    dec.release()


# ---- kernel level -------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, bpc, layout, w, h, size=None, dtype="float32", lay="chw", siting="left", matrix="bt709", full_range=False,
                 mean=None, std=None, offset=0, pad=0):
        self.__dict__.update(locals())
        del self.__dict__["self"]


def _planes(rng, c):
    dims = stream.plane_dims(c.w, c.h, c.layout)
    return [rng.integers(0, 1 << c.bpc, (ph, pw)).astype(np.uint16 if c.bpc > 8 else np.uint8) for pw, ph in dims]


def _source(planes, layout, extra=7):
    """the planes in one buffer with strides wider than the rows: (buffer, plane_off, stride)"""
    offs, strides, parts, at = [0, 0, 0], [0, 0, 0], [], 0
    for k, p in enumerate(planes):
        st = p.shape[1] + extra
        buf = np.zeros((p.shape[0], st), p.dtype)
        buf[:, :p.shape[1]] = p
        offs[k], strides[k] = at, st
        parts.append(buf.ravel())
        at += buf.size
    return np.concatenate(parts), offs, strides


def _job(c, src_ptr, offs, strides, dst_ptr, pitch_c, pitch_y):
    j = stream.TensorJob()
    j.src = src_ptr
    for k in range(3):
        j.plane_off[k], j.stride[k] = offs[k], strides[k]
    j.w, j.h = c.w, c.h
    j.ss_hor, j.ss_ver = _layout_of(c.layout)
    j.mono = int(c.layout == 0)
    j.bitdepth_max = (1 << c.bpc) - 1
    oh, ow = c.size or (c.h, c.w)
    j.out_w, j.out_h = ow, oh
    j.dtype, j.layout = stream.TENSOR_DTYPES[c.dtype], stream.TENSOR_LAYOUTS[c.lay]
    j.full_range, j.identity = int(c.full_range), int(c.matrix == "identity")
    j.siting_x, j.siting_y = stream.SITINGS[c.siting]
    if c.matrix != "identity":
        j.cy, j.rv, j.gu, j.gv, j.bu = stream.rgb_coefficients(c.matrix, c.full_range)
    scale, bias = stream.tensor_scale_bias(c.bpc, c.mean, c.std)
    for k in range(3):
        j.scale[k], j.bias[k] = float(scale[k]), float(bias[k])
    j.dst, j.pitch_c, j.pitch_y = dst_ptr, pitch_c, pitch_y
    return j


def _pitches(c):
    """(pitch_c, pitch_y, elements of the destination) with c.pad elements of slack after every row and channel"""
    oh, ow = c.size or (c.h, c.w)
    if c.lay == "chw":
        py = ow + c.pad
        pc = oh * py + c.pad
        return pc, py, 3 * pc
    py = 3 * ow + c.pad
    return 1, py, oh * py


def _expected(c, planes, pitch_c, pitch_y, n_elems, guard):
    """the destination as the export must leave it: reference bits in the written elements, `guard` everywhere else"""
    ref = stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std)
    bits = _bits(ref, c.dtype)
    out = np.full(n_elems, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        idx = ch * pitch_c + y * pitch_y + x if c.lay == "chw" else y * pitch_y + 3 * x + ch
        out[idx] = bits[ch]
    return out


GUARD = 16


def _run_emu(c, seed):
    lib = refs.emu_lib()
    rng = np.random.default_rng(seed)
    planes = _planes(rng, c)
    src, offs, strides = _source(planes, c.layout)
    pc, py, n = _pitches(c)
    et = np.uint32 if c.dtype == "float32" else np.uint16
    guard = et(0x7fc0dead if et is np.uint32 else 0x7e57)
    buf = np.full(n + 2 * GUARD + c.offset, guard, et)
    j = _job(c, src.ctypes.data, offs, strides, buf.ctypes.data + (GUARD + c.offset) * buf.itemsize, pc, py)
    assert lib.b200_export_tensor(C.byref(j), None) == 0, lib.b200_last_error()
    want = np.full_like(buf, guard)
    want[GUARD + c.offset:GUARD + c.offset + n] = _expected(c, planes, pc, py, n, guard)
    bad = np.flatnonzero(buf != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s)" % (bad.size, bad[0], c.__dict__)


def _kernel_cases():
    cases = []
    k = 0
    for bpc in (8, 10, 12):
        for layout in (0, 1, 2, 3):
            w, h = (45, 27) if layout != 2 else (38, 21)
            sizes = [None, (13, 22), (4 * h, 4 * w - 3), (1, 1), (3, 97)]
            for size in sizes:
                dtype, lay, siting = DTYPES[k % 3], ("chw", "hwc")[(k // 3) % 2], SITINGS[(k // 2) % 3]
                matrix = ("identity" if layout == 3 and k % 4 == 0 else ["bt601", "bt709", "bt2020"][k % 3])
                full = bool(k % 2)
                mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if k % 3 == 1 else (None, None)
                cases.append(Case(bpc, layout, w, h, size, dtype, lay, siting, matrix, full, mean, std, offset=k % 2, pad=3 * (k % 3)))
                k += 1
    # every dtype x layout x siting once more on 4:2:0 10 bit, with a downscale
    for dtype in DTYPES:
        for lay in ("chw", "hwc"):
            for siting in SITINGS:
                cases.append(Case(10, 1, 31, 19, (11, 23), dtype, lay, siting, "bt709", False, offset=1, pad=1))
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_kernel_matches_reference_emu(idx):
    _run_emu(KERNEL_CASES[idx], 1000 + idx)


@pytest.mark.emu
def test_bad_arguments_emu():
    lib = refs.emu_lib()
    c = Case(10, 1, 32, 16)
    planes = _planes(np.random.default_rng(3), c)
    src, offs, strides = _source(planes, c.layout)
    pc, py, n = _pitches(c)
    buf = np.zeros(n + 8, np.float32)
    good = _job(c, src.ctypes.data, offs, strides, buf.ctypes.data, pc, py)
    assert lib.b200_export_tensor(C.byref(good), None) == 0
    mutations = [("bitdepth_max", 511), ("dtype", 3), ("dtype", -1), ("layout", 2), ("w", 0), ("h", -4), ("w", 65537),
                 ("out_w", 0), ("out_h", 65537), ("ss_hor", 2), ("siting_x", 2), ("siting_y", -1), ("identity", 1),
                 ("src", None), ("dst", None), ("dst", buf.ctypes.data + 2), ("pitch_y", 31), ("pitch_y", -32),
                 ("pitch_c", pc - 1), ("pitch_y", 1 << 50), ("pitch_c", 1 << 60), ("stride", (C.c_int32 * 3)(31, 16, 16)),
                 ("stride", (C.c_int32 * 3)(40, 15, 40))]
    for field, value in mutations:
        j = stream.TensorJob.from_buffer_copy(good)
        setattr(j, field, value)
        assert lib.b200_export_tensor(C.byref(j), None) == -2, (field, value)
        assert lib.b200_last_error()
    j = stream.TensorJob.from_buffer_copy(good)
    j.layout, j.pitch_y = 1, 3 * 32 - 1
    assert lib.b200_export_tensor(C.byref(j), None) == -2
    assert lib.b200_export_tensor(None, None) == -2


# ---- decoder level ------------------------------------------------------------------------------------------------
def _np_alloc(shape, dtype):
    return np.full(shape, 0x5a, np.float32 if dtype == "float32" else np.float16 if dtype == "float16" else np.uint16)


def _check_tensors(dec, tus, size=None, dtype="float32", layout="chw", batch=None, siting="auto", want_siting="left",
                   matrix="auto", full_range=None, mean=None, std=None, alloc=_np_alloc, **kw):
    ref = DO._ref_pictures(tus)
    dec.stats(reset=True)
    got = list(dec.tensors(tus, size=size, dtype=dtype, layout=layout, mean=mean, std=std, matrix=matrix, full_range=full_range,
                           chroma_siting=siting, batch=batch, alloc=alloc, **kw))
    items = [t for g in got for t in g] if batch else got
    assert len(items) == len(ref)
    name = "bt709" if matrix == "auto" else matrix
    for k, ((w, h, bpc, layout_, rp), g) in enumerate(zip(ref, items)):
        want = stream.tensor_reference(rp, bpc, layout_, size, name, bool(full_range), want_siting, mean, std)
        if layout == "hwc":
            want = want.transpose(1, 2, 0)
        assert tuple(g.shape) == want.shape, k
        assert np.array_equal(_host_bits(g, dtype), _bits(want, dtype)), "picture %d differs (%s, %s)" % (k, dtype, layout)
    st = dec.stats(reset=True)
    assert st["d2h_bytes"] == 0 and st["frames"] > 0
    return got, ref


DECODER_CASES = [
    ("10 bit odd size, grain", lambda: obu.inter_stream(21, 201, 135, n_frames=3, bpc=10, film_grain=1, motion_modes=2),
     dict(size=(64, 96), dtype="bfloat16", layout="hwc", mean=(0.5, 0.4, 0.3), std=(0.2, 0.3, 0.25))),
    ("4:0:0", lambda: obu.inter_stream(22, 131, 67, n_frames=2, bpc=10, layout="400"), dict(dtype="float16", full_range=True)),
    ("12 bit 4:4:4", lambda: obu.intra_stream(23, 96, 64, n_frames=2, bpc=12, layout="444", film_grain=1),
     dict(size=(150, 41), matrix="identity")),
    ("super-resolution", lambda: obu.intra_stream(900, 328, 200, n_frames=2, bpc=10, super_res=1, log2_cols=1),
     dict(size=(100, 164), siting="center", want_siting="center", matrix="bt2020")),
]


@pytest.mark.emu
@pytest.mark.parametrize("name,make,kw", DECODER_CASES, ids=[c[0] for c in DECODER_CASES])
def test_tensors_match_reference_emu(emu_device_decoder, name, make, kw):
    _check_tensors(emu_device_decoder, make(), **kw)


@pytest.mark.emu
def test_tensors_422_emu(emu_device_decoder):
    import test_stream as TS
    tus = TS._valid_422("inter", 128, 64, 10, 1, motion_modes=1, film_grain=1)[0]
    _check_tensors(emu_device_decoder, tus, size=(48, 80), siting="topleft", want_siting="topleft", layout="hwc")


@pytest.mark.emu
def test_tensors_auto_siting_emu(emu_device_decoder):
    """chroma_sample_position = colocated (2) in the sequence header: "auto" samples chroma on the even luma row"""
    tus = obu.inter_stream(24, 96, 64, n_frames=2, bpc=8, chroma_sample_position=2)
    _check_tensors(emu_device_decoder, tus, want_siting="topleft")
    _check_tensors(emu_device_decoder, obu.inter_stream(24, 96, 64, n_frames=2, bpc=8, chroma_sample_position=1), want_siting="left")


@pytest.mark.emu
def test_tensors_batches_with_changing_sizes_emu(emu_device_decoder):
    """scaled references with frame-size changes: with size=None a picture of another size closes the batch, with a size
    every batch is full but the last"""
    tus = obu.inter_stream(701, 320, 192, n_frames=6, sizes=[(256, 160), (320, 192), (200, 120), (320, 176)], bpc=10,
                           motion_modes=1, film_grain=1)
    got, ref = _check_tensors(emu_device_decoder, tus, batch=4, dtype="float16")
    runs = []
    for w, h, *_ in ref:
        if runs and runs[-1][0] == (w, h) and runs[-1][1] < 4:
            runs[-1][1] += 1
        else:
            runs.append([(w, h), 1])
    assert [tuple(g.shape) for g in got] == [(n, 3, h, w) for (w, h), n in runs]
    assert len(set((w, h) for w, h, *_ in ref)) > 1
    got, _ = _check_tensors(emu_device_decoder, tus, batch=4, size=(90, 150), layout="hwc", dtype="bfloat16")
    assert [tuple(g.shape) for g in got] == [(4, 90, 150, 3), (len(ref) - 4, 90, 150, 3)]


@pytest.mark.emu
def test_tensors_bad_arguments_emu(emu_device_decoder):
    tus = obu.intra_stream(1, 64, 64)
    for kw in (dict(dtype="uint8"), dict(layout="nchw"), dict(size=(0, 10)), dict(batch=0), dict(chroma_siting="bottom"),
               dict(mean=(0, 0)), dict(std=(1, 0, 1)), dict(matrix="identity")):
        with pytest.raises(ValueError):
            list(emu_device_decoder.tensors(tus, alloc=_np_alloc, **kw))


@pytest.fixture(scope="module")
def emu_device_decoder(hooked_library):
    refs.emu_lib()
    d = stream.DeviceDecoder(backend=DO._emu_path(), serialize=True, apply_grain=1)
    yield d
    d.release()


# ---- on the device ------------------------------------------------------------------------------------------------
def _run_gpu(c, seed):
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    rng = np.random.default_rng(seed)
    planes = _planes(rng, c)
    src, offs, strides = _source(planes, c.layout, extra=64)
    d_src = torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda()
    pc, py, n = _pitches(c)
    tdt = torch.int32 if c.dtype == "float32" else torch.int16
    guard = 0x7fc0dead if c.dtype == "float32" else 0x7e57
    buf = torch.full((n + 2 * GUARD + c.offset,), guard, dtype=tdt, device="cuda")
    j = _job(c, d_src.data_ptr(), offs, strides, buf.data_ptr() + (GUARD + c.offset) * buf.element_size(), pc, py)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    assert lib.b200_export_tensor(C.byref(j), C.c_void_p(s.cuda_stream)) == 0, lib.b200_last_error()
    s.synchronize()
    got = _host_bits(buf, c.dtype)
    et = got.dtype
    want = np.full(got.shape, et.type(guard), et)
    want[GUARD + c.offset:GUARD + c.offset + n] = _expected(c, planes, pc, py, n, et.type(guard))
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


GPU_KERNEL_CASES = [Case(8, 1, 1920, 1080, None, d, l, "left", "bt709", False) for d in DTYPES for l in ("chw", "hwc")] + \
    [Case(10, 1, 3840, 2160, (1080, 1920), d, l, s, "bt2020", True, (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), offset=o)
     for (d, l, s, o) in [("float32", "chw", "topleft", 0), ("float16", "hwc", "center", 1), ("bfloat16", "chw", "left", 1),
                          ("bfloat16", "hwc", "left", 0), ("float32", "hwc", "center", 1), ("float16", "chw", "left", 0)]] + \
    [Case(10, 1, 3840, 2160, None, "bfloat16", "hwc", "left", "bt709", False), Case(12, 3, 1920, 1080, (2160, 3840), "float16", "chw", "left", "identity", False),
     Case(8, 1, 1920, 1080, (360, 640), "float16", "chw", "left", "bt709", False, pad=5)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GPU_KERNEL_CASES)))
def test_kernel_matches_reference_gpu(idx):
    _run_gpu(GPU_KERNEL_CASES[idx], 2000 + idx)


@pytest.fixture(scope="module")
def gpu_device_decoder(hooked_library):
    d = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    yield d
    d.release()


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(1920, 1080, 8, 1), (3840, 2160, 10, 0)])
def test_tensors_gpu(gpu_device_decoder, case):
    """1080p 8 bit with film grain and 4K 10 bit into torch CUDA tensors on a non-default stream, in batches of 4, native
    and resized"""
    import torch
    w, h, bpc, fg = case
    tus = obu.inter_stream(300 + bpc, w, h, n_frames=5, bpc=bpc, log2_cols=2, log2_rows=1, motion_modes=2, film_grain=fg)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for kw in (dict(), dict(size=(h // 2, w // 2 + 6), dtype="bfloat16", layout="hwc"),
                   dict(size=(224, 224), dtype="float16", mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))):
            got, _ = _check_tensors(gpu_device_decoder, tus, batch=4, alloc=None, **kw)
            assert [g.shape[0] for g in got] == [4, 1] and all(g.is_cuda for g in got)
