"""HDR to SDR in the tensor export (B200ToneMap and b200_export_tensor_tone_batch, include/b200av1.h; tone_map in
dav1d_b200/csrc/export.cu; b200hook_export_tensor_tone_batch and refdrv_stream_color, integration/dav1d; tonemap= of
stream.DeviceDecoder.tensors and clips). The tables (stream.tone_tables) are checked against a float64 statement of the
standards written out here; the kernel must be stream.tensor_reference(..., tone=tables) bit for bit. CPU tests run the
CUDA sources on the host emulator, GPU tests run the CUDA library into torch CUDA tensors."""
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
TONE_MAX = 16                           # B200_TENSOR_TONE_BATCH_MAX, include/b200av1.h


# ---- the standards, in float64 ------------------------------------------------------------------------------------
def st2084_eotf(e):
    m1, m2, c1, c2, c3 = 0.1593017578125, 78.84375, 0.8359375, 18.8515625, 18.6875
    p = np.asarray(e, np.float64) ** (1 / m2)
    return 10000 * (np.maximum(p - c1, 0) / (c2 - c3 * p)) ** (1 / m1)


def st2084_inverse(lum):
    m1, m2, c1, c2, c3 = 0.1593017578125, 78.84375, 0.8359375, 18.8515625, 18.6875
    y = (np.asarray(lum, np.float64) / 10000) ** m1
    return ((c1 + c2 * y) / (1 + c3 * y)) ** m2


def hlg_inverse_oetf(e):
    a = 0.17883277
    b, c = 1 - 4 * a, 0.5 - a * np.log(4 * a)
    e = np.asarray(e, np.float64)
    return np.where(e <= 0.5, e ** 2 / 3, (np.exp((e - c) / a) + b) / 12)


def bt2390_eetf(lum, src_peak, dst_peak):
    """BT.2390 section 5.4 with Lb = Lmin = 0: display light in, display light out"""
    lb = st2084_inverse(0.0)
    lw = st2084_inverse(src_peak)
    e1 = np.clip((st2084_inverse(np.minimum(lum, src_peak)) - lb) / (lw - lb), 0, 1)
    max_lum = (st2084_inverse(dst_peak) - lb) / (lw - lb)
    ks = 1.5 * max_lum - 0.5
    out = np.empty_like(e1)
    for i, x in np.ndenumerate(e1):
        if x < ks:
            out[i] = x
        else:
            t = (x - ks) / (1 - ks)
            out[i] = (2 * t ** 3 - 3 * t ** 2 + 1) * ks + (t ** 3 - 2 * t ** 2 + t) * (1 - ks) + (-2 * t ** 3 + 3 * t ** 2) * max_lum
    return st2084_eotf(out * (lw - lb) + lb)


def bt709_oetf(v):
    a, b = 1.09929682680944, 0.018053968510807
    v = np.asarray(v, np.float64)
    return np.where(v < b, 4.5 * v, a * np.maximum(v, b) ** 0.45 - (a - 1))


def chain(transfer, e, peak, sdr_peak):
    """curve stage in float64: signal -> SDR-normalised light in [0, 1]"""
    if transfer == "pq":
        lum = st2084_eotf(e)
    else:
        lum = peak * hlg_inverse_oetf(e) ** (1.2 + 0.42 * np.log10(peak / 1000))
    if sdr_peak < peak:
        lum = bt2390_eetf(lum, peak, sdr_peak)
    return np.clip(np.minimum(lum, peak) / sdr_peak, 0, 1)


# ---- tables against the standards ---------------------------------------------------------------------------------
@pytest.mark.parametrize("transfer,bpc,peak", [("pq", 10, 1000), ("pq", 12, 4000), ("pq", 8, 600), ("pq", 10, 150),
                                               ("hlg", 10, 1000), ("hlg", 12, 2000), ("hlg", 8, 1000)])
def test_tables_follow_the_standards(transfer, bpc, peak):
    """at every curve index, and over a dense sweep of G, the float32 tables give the float64 chain within 2^-12 of full
    scale"""
    curve, m, oetf = stream.tone_tables(transfer, 9, bpc, peak)
    qmax = 4 * ((1 << bpc) - 1)
    assert curve.dtype == oetf.dtype == m.dtype == np.float32
    assert curve.shape == (qmax + 1,) and oetf.shape == ((1 << 16) + 1,) and m.shape == (3, 3)
    assert curve.min() >= 0 and curve.max() <= 1
    lin = chain(transfer, np.arange(qmax + 1) / qmax, peak, 203.0)
    got = oetf[np.rint(curve * np.float32(1 << 16)).astype(np.int64)] / qmax
    assert np.abs(got - bt709_oetf(lin)).max() <= 2.0 ** -12
    g = np.linspace(0, 1, 1_000_003)
    got = oetf[np.rint(g.astype(np.float32) * np.float32(1 << 16)).astype(np.int64)] / qmax
    assert np.abs(got - bt709_oetf(g)).max() <= 2.0 ** -12


def test_curve_points():
    """50 cd/m^2 lies below the knee (peak 1000, SDR 203) and passes unchanged; the source peak becomes 1.0; HLG's 75 %
    reference white is 203 cd/m^2 at Lw = 1000"""
    assert abs(stream.tone_light("pq", st2084_inverse(50.0), 1000.0, 203.0) - 50 / 203) < 1e-9
    assert abs(stream.tone_light("pq", st2084_inverse(1000.0), 1000.0, 203.0) - 1.0) < 1e-12
    assert abs(stream.tone_light("pq", st2084_inverse(4000.0), 1000.0, 203.0) - 1.0) < 1e-12      # above the peak: clipped
    assert abs(1000 * hlg_inverse_oetf(0.75) ** 1.2 - 203) < 1
    assert abs(1000 * stream.hlg_inverse_oetf(0.75) ** stream.hlg_gamma(1000.0) - 203) < 1
    # no compression when the SDR peak is at or above the source peak
    e = np.linspace(0, 1, 1001)
    assert np.allclose(stream.tone_light("pq", e, 150.0, 203.0), np.minimum(st2084_eotf(e), 150) / 203, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("peak,sdr_peak", [(1000.0, 203.0), (4000.0, 100.0), (600.0, 203.0), (10000.0, 300.0)])
def test_eetf_identity_below_knee_and_monotone(peak, sdr_peak):
    lum = st2084_eotf(np.linspace(0, st2084_inverse(peak), 200_001))
    out = stream.eetf(lum, peak, sdr_peak)
    assert np.all(np.diff(out) >= 0)
    assert np.allclose(out, bt2390_eetf(lum, peak, sdr_peak), rtol=1e-9, atol=1e-12)
    max_lum = st2084_inverse(sdr_peak) / st2084_inverse(peak)    # PQ(0) is below 1e-6: black is 0 on both sides
    ks = 1.5 * max_lum - 0.5
    below = st2084_inverse(lum) / st2084_inverse(peak) < ks - 1e-9
    assert below.any() and np.allclose(out[below], lum[below], rtol=1e-9)
    assert abs(stream.eetf(peak, peak, sdr_peak) - sdr_peak) < 1e-9 * sdr_peak


def test_gamut_matrices():
    """BT.2020 -> BT.709 is BT.2087's matrix; every matrix maps white to white; unknown primaries are an error"""
    bt2087 = np.array([[1.6605, -0.5876, -0.0728], [-0.1246, 1.1329, -0.0083], [-0.0182, -0.1006, 1.1187]])
    assert np.abs(stream.gamut_matrix(9) - bt2087).max() < 1e-4
    assert np.array_equal(stream.gamut_matrix(2), stream.gamut_matrix(9))
    assert np.array_equal(stream.gamut_matrix(1), np.eye(3))
    for pri in (1, 2, 9, 12):
        assert np.allclose(stream.gamut_matrix(pri).sum(1), 1, atol=1e-12)
        assert np.allclose(stream.tone_tables("pq", pri, 10)[1].astype(np.float64).sum(1), 1, atol=1e-6)
    p3 = stream.gamut_matrix(12)
    assert p3[0, 0] > 1.2 and p3[0, 1] < 0                      # P3 red lies outside BT.709
    for pri in (0, 4, 5, 6, 11, 22, "bt2020"):
        with pytest.raises(ValueError):
            stream.tone_tables("pq", pri, 10)
    for bad in (dict(transfer="sdr"), dict(transfer=1), dict(bpc=9), dict(peak=0), dict(peak=float("nan")), dict(sdr_peak=-1),
                dict(bits=7), dict(bits=17)):
        kw = dict(transfer="pq", primaries=9, bpc=10)
        kw.update(bad)
        with pytest.raises(ValueError):
            stream.tone_tables(**kw)
    assert np.array_equal(stream.tone_tables(16, 9, 10)[0], stream.tone_tables("pq", 9, 10)[0])


def test_tone_reference_rounds_each_operation():
    """tone_reference is the float32 stage written out: curve gather, the three products and two sums in order, clip,
    rint half to even on the exact product, OETF gather"""
    rng = np.random.default_rng(3)
    curve, m, oetf = stream.tone_tables("pq", 12, 10, 800)
    rgb = rng.integers(0, 4093, (3, 7, 9))
    got = stream.tone_reference(rgb, (curve, m, oetf))
    L = curve[rgb].astype(np.float64)
    for r in range(3):
        g = np.float32(np.float32(np.float32(m[r, 0]) * np.float32(L[0])) + np.float32(np.float32(m[r, 1]) * np.float32(L[1])))
        g = np.float32(g + np.float32(np.float32(m[r, 2]) * np.float32(L[2])))
        idx = np.rint(np.clip(g, 0, 1).astype(np.float64) * 65536).astype(np.int64)
        assert np.array_equal(got[r], oetf[idx])
    assert np.array_equal(stream.tone_reference(np.full((3, 1, 1), 4092), (curve, np.eye(3, dtype=np.float32), oetf)),
                          np.full((3, 1, 1), 4092, np.float32))


# ---- kernel level -------------------------------------------------------------------------------------------------
KINDS = {"bilinear": (0, "bilinear"), "triangle": (1, "bilinear"), "cubic": (0, "bicubic"), "cubic_aa": (1, "bicubic")}


def _tone_args(c, k):
    transfer = ("pq", "hlg")[k % 2]
    return stream.tone_tables(transfer, (9, 12, 1, 2)[k % 4], c.bpc, (1000.0, 600.0, 4000.0)[k % 3], (203.0, 100.0)[k % 2])


def _tone_struct(tables, keep, to_dev=None):
    curve, m, oetf = tables
    d = [to_dev(curve), to_dev(oetf)] if to_dev else [curve, oetf]
    keep.extend(d)
    t = stream.ToneMap()
    t.curve, t.oetf = stream._data_ptr(d[0]), stream._data_ptr(d[1])
    t.curve_len, t.oetf_bits = len(curve), 16
    for i in range(9):
        t.m[i] = float(m.ravel()[i])
    return t


def _expected(c, planes, pc, py, n, guard, kind, flip, tone):
    aa, interp = KINDS[kind]
    ref = stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std,
                                  antialias=aa, interpolation=interp, tone=tone)
    if flip:
        ref = ref[:, :, ::-1].copy()
    bits = TE._bits(ref, c.dtype)
    out = np.full(n, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        out[ch * pc + y * py + x if c.lay == "chw" else y * py + 3 * x + ch] = bits[ch]
    return out


def _crop_source(planes, layout, box, extra):
    """the source buffer of the whole picture with the job's plane_off moved to the box: (buffer, offs, strides)"""
    src, offs, strides = TE._source(planes, layout, extra=extra)
    if box:
        ssh, ssv = int(layout in (1, 2)), int(layout == 1)
        offs = [offs[0] + box[0] * strides[0] + box[1]] + [offs[p] + (box[0] >> ssv) * strides[p] + (box[1] >> ssh) for p in (1, 2)]
    return src, offs, strides


def _run(c, seed, kind, flip, box, lib, device=False):
    """one tone-mapped job (c: the full picture; box: a crop of it or None) into a guarded destination: (written, wanted)"""
    rng = np.random.default_rng(seed)
    planes = TE._planes(rng, c)
    tone = _tone_args(c, seed)
    src, offs, strides = _crop_source(planes, c.layout, box, 64 if device else 7)
    cj = TE.Case(**dict(c.__dict__, w=box[3], h=box[2])) if box else c
    pc, py, n = TE._pitches(cj)
    et = np.uint32 if c.dtype == "float32" else np.uint16
    guard = et(0x7fc0dead if et is np.uint32 else 0x7e57)
    total = n + 2 * TE.GUARD + c.offset
    keep = []
    aa, interp = KINDS[kind]
    if device:
        import torch
        d_src = torch.from_numpy(src.view(np.int16) if src.dtype == np.uint16 else src).cuda()
        buf = torch.full((total,), int(guard.astype(np.int32 if et is np.uint32 else np.int16)),
                         dtype=torch.int32 if et is np.uint32 else torch.int16, device="cuda")
        j = TE._job(cj, d_src.data_ptr(), offs, strides, buf.data_ptr() + (TE.GUARD + c.offset) * buf.element_size(), pc, py)
        tm = _tone_struct(tone, keep, lambda a: torch.from_numpy(a).cuda())
    else:
        buf = np.full(total, guard, et)
        j = TE._job(cj, src.ctypes.data, offs, strides, buf.ctypes.data + (TE.GUARD + c.offset) * buf.itemsize, pc, py)
        tm = _tone_struct(tone, keep)
    j.antialias, j.flip, j.interpolation = aa, flip, stream.TENSOR_INTERPOLATIONS[interp]
    tones = (C.POINTER(stream.ToneMap) * 1)(C.pointer(tm))
    assert lib.b200_export_tensor_tone_batch(C.byref(j), tones, 1, None) == 0, lib.b200_last_error()
    if device:
        torch.cuda.synchronize()
        buf = TE._host_bits(buf, c.dtype)
    want = np.full(total, guard, et)
    part = stream.crop_planes(planes, c.layout, box) if box else planes
    want[TE.GUARD + c.offset:TE.GUARD + c.offset + n] = _expected(cj, part, pc, py, n, guard, kind, flip, tone)
    return buf, want


def _kernel_cases():
    """every kind x bit depth x chroma layout (4:4:4 with the identity matrix), every dtype and layout, flips and crops,
    ragged widths and misaligned destinations"""
    geo = [(45, 27, (13, 22)), (38, 21, (9, 3)), (64, 48, (5, 1)), (33, 31, (40, 11)), (61, 33, (7, 16)), (30, 20, (45, 31))]
    cases, k = [], 0
    for kind in KINDS:
        for bpc in (8, 10, 12):
            for layout in (0, 1, 2, 3):
                w, h, size = geo[k % len(geo)]
                matrix = "identity" if layout == 3 else ["bt2020", "bt709", "bt601"][k % 3]
                kw = IMAGENET if k % 3 == 1 else {}
                c = TE.Case(bpc, layout, w, h, size, DTYPES[k % 3], ("chw", "hwc")[(k // 3) % 2], list(stream.SITINGS)[k % 3],
                            matrix, bool(k % 2), offset=(k // 2) % 2, pad=(1, 0, 3)[k % 3], **kw)
                box = (2, 4, h - 5, w - 7) if k % 3 == 2 else None
                cases.append((c, kind, k % 2, box))
                k += 1
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_tone_kernel_emu(idx):
    c, kind, flip, box = KERNEL_CASES[idx]
    got, want = _run(c, 7000 + idx, kind, flip, box, refs.emu_lib())
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s %s)" % (bad.size, bad[0], kind, c.__dict__)


def _mixed_plan(k):
    """(kind, flip, tone map) of job k of a mixed batch: tone-mapped (even k) and plain jobs each take every kind"""
    return list(KINDS)[(k // 2) % 4], k % 3 == 0, k % 2 == 0


def _mixed_cases(n, dtype, lay, seed):
    rng = np.random.default_rng(seed)
    cases = TC._batch_cases(rng, n, dtype, lay)
    for k, c in enumerate(cases):
        if k % 2 or k % 8 == 2:                 # reduced, so that antialiased bilinear jobs take the triangle kernel
            c.size = (max(1, c.h // (2 + k % 5)), max(1, c.w // (1 + k % 3)))
    return cases


def _uniform_cases(n, dtype, lay, seed):
    """n 10-bit 4:2:0 pictures reduced to 20 x 30: one bit-depth class and, with antialias, one kernel kind"""
    return [TE.Case(10, 1, 64 + k % 5, 48 + k % 3, (20, 30), dtype, lay, "left", "bt2020", bool(k % 2), offset=k % 2)
            for k in range(n)]


def _uniform_plan(k):
    """a tone-mapped triangle job without a flip, but every fourth job plain (its own launch group)"""
    return "triangle", False, k % 4 != 3


def _batch(cases, seed, plan, to_dev=None, ptr_of=lambda a: a.ctypes.data):
    """the jobs of `cases` as plan(k) = (kind, flip, tone map) says: (jobs, tones, destination, what it must hold, spans,
    guard, keep)"""
    n = len(cases)
    srcs, spans, buf, guard = TC._batch_setup(cases, seed, ptr_of)
    jobs = (stream.TensorJob * n)()
    tones = (C.POINTER(stream.ToneMap) * n)()
    want = np.full_like(buf, guard)
    keep = []
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        kind, flip, has_tone = plan(k)
        aa, interp = KINDS[kind]
        jobs[k] = TE._job(c, ptr_of(src), offs, strides, ptr_of(buf) + at * buf.itemsize, pc, py)
        jobs[k].antialias, jobs[k].flip, jobs[k].interpolation = aa, flip, stream.TENSOR_INTERPOLATIONS[interp]
        tone = _tone_args(c, k) if has_tone else None
        if tone is not None:
            tones[k] = C.pointer(_tone_struct(tone, keep, to_dev))
        want[at:at + m] = _expected(c, planes, pc, py, m, guard, kind, flip, tone)
    return jobs, tones, buf, want, spans, guard, (srcs, keep)


def _check_plain_jobs(lib, jobs, tones, buf, spans, guard):
    """the plain jobs of a mixed batch wrote what b200_export_tensor_batch writes, and tones = NULL is that function"""
    n = len(jobs)
    plain = np.full_like(buf, guard)
    pj = (stream.TensorJob * n).from_buffer_copy(jobs)
    for k in range(n):
        pj[k].dst = plain.ctypes.data + spans[k] * plain.itemsize
    assert lib.b200_export_tensor_batch(pj, n, None) == 0
    for k in range(n):
        if not tones[k]:
            s = slice(spans[k], spans[k + 1] if k + 1 < n else None)
            assert np.array_equal(plain[s], buf[s]), k
    again = np.full_like(buf, guard)
    for k in range(n):
        pj[k].dst = again.ctypes.data + spans[k] * again.itemsize
    assert lib.b200_export_tensor_tone_batch(pj, None, n, None) == 0
    assert np.array_equal(again, plain)


@pytest.mark.emu
@pytest.mark.parametrize("n,dtype,lay", [(2 * TONE_MAX + 5, "float32", "hwc"), (TONE_MAX + 1, "bfloat16", "chw")])
def test_batch_mixing_tone_and_plain_jobs_emu(n, dtype, lay):
    """tone-mapped and plain jobs of every kind, both bit-depth classes and flips in one call: each is the definition, and
    the plain ones write what b200_export_tensor_batch writes"""
    lib = refs.emu_lib()
    jobs, tones, buf, want, spans, guard, _keep = _batch(_mixed_cases(n, dtype, lay, 1200 + n), 1200 + n, _mixed_plan)
    assert lib.b200_export_tensor_tone_batch(jobs, tones, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)
    _check_plain_jobs(lib, jobs, tones, buf, spans, guard)


@pytest.mark.emu
@pytest.mark.parametrize("n_tone", [TONE_MAX, 2 * TONE_MAX + 3])
def test_tone_jobs_split_into_launches_emu(n_tone):
    """more tone-mapped jobs of one bit-depth class, kind and flip than one launch takes, between plain jobs of the same
    group: every job is the definition, and the tone-mapped ones take ceil(n / B200_TENSOR_TONE_BATCH_MAX) launches"""
    lib = refs.emu_lib()
    n = n_tone + n_tone // 3
    cases = _uniform_cases(n, "bfloat16", "chw", 1300 + n)
    jobs, tones, buf, want, spans, guard, _keep = _batch(cases, 1300 + n, _uniform_plan)
    assert sum(bool(t) for t in tones) == n_tone
    before = lib.b200_launch_count()
    assert lib.b200_export_tensor_tone_batch(jobs, tones, n, None) == 0, lib.b200_last_error()
    assert lib.b200_launch_count() - before == -(-n_tone // TONE_MAX) + 1          # and one launch of the plain jobs
    assert np.array_equal(buf, want)
    _check_plain_jobs(lib, jobs, tones, buf, spans, guard)


@pytest.mark.emu
def test_bad_tone_maps_emu():
    """a NULL table, a curve of the wrong length for the job's bit depth, oetf_bits outside 8 .. 16 or a matrix entry that
    is not finite: -2 with the error set, and nothing written by any job of the batch"""
    lib = refs.emu_lib()
    jobs, tones, buf, _, _, guard, _keep = _batch(_mixed_cases(6, "float32", "chw", 31), 31, _mixed_plan)
    good = stream.ToneMap.from_buffer_copy(tones[2].contents)
    bdmax = jobs[2].bitdepth_max
    for field, value in [("curve", None), ("oetf", None), ("curve_len", 4 * bdmax), ("curve_len", 4 * bdmax + 2),
                         ("curve_len", 4 * 1023 + 1 if bdmax != 1023 else 4 * 255 + 1), ("oetf_bits", 7), ("oetf_bits", 17),
                         ("m", float("nan")), ("m", float("inf")), ("m", float("-inf"))]:
        bad = stream.ToneMap.from_buffer_copy(good)
        if field == "m":
            bad.m[4] = value
        else:
            setattr(bad, field, value)
        t = (C.POINTER(stream.ToneMap) * 6)(*[tones[k] for k in range(6)])
        t[2] = C.pointer(bad)
        buf[:] = guard
        assert lib.b200_export_tensor_tone_batch(jobs, t, 6, None) == -2, field
        assert b"tone" in lib.b200_last_error()
        assert np.all(buf == guard)
    bad_job = (stream.TensorJob * 6).from_buffer_copy(jobs)
    bad_job[3].flip = 2
    assert lib.b200_export_tensor_tone_batch(bad_job, tones, 6, None) == -2
    assert lib.b200_export_tensor_tone_batch(None, tones, 1, None) == -2
    assert lib.b200_export_tensor_tone_batch(jobs, tones, 0, None) == -2
    assert np.all(buf == guard)


def test_tone_map_abi():
    """B200ToneMap is 64 bytes in ctypes and in the library (checked on load), and 16 jobs with their tone maps fit the 4 KB
    parameter block"""
    from dav1d_b200 import _lib
    assert C.sizeof(stream.ToneMap) == 64 and C.sizeof(stream.TensorJob) == 168
    assert TONE_MAX * (C.sizeof(stream.ToneMap) + C.sizeof(stream.TensorJob)) <= 4096
    assert _lib.ABI_STRUCTS[24] is stream.ToneMap
    assert "b200_export_tensor_tone_batch" in _lib.B200Lib.symbols()


@pytest.mark.emu
def test_tone_map_size_in_the_library_emu():
    lib = refs.emu_lib()
    assert lib.b200_struct_size(24) == C.sizeof(stream.ToneMap)


# ---- decoder level ------------------------------------------------------------------------------------------------
def _pq_stream(seed=50, cll=(1000, 400), mdcv=None, w=96, h=64, n_frames=3, pri=9, trc=16, bpc=10, **kw):
    md = ([obu.metadata_hdr_cll(*cll)] if cll else []) + ([obu.metadata_hdr_mdcv(*mdcv)] if mdcv else [])
    return obu.inter_stream(seed, w, h, n_frames=n_frames, bpc=bpc, color=(9, 0, pri, trc), metadata=md, **kw)


def _check_tensors(dec, tus, tonemap, transfer, primaries, want_peak, size=None, dtype="float32", layout="chw", alloc=TE._np_alloc,
                   matrix="bt2020", sdr_peak=203.0, **kw):
    """tensors(tonemap=) against tensor_reference(stock dav1d's picture, tone=tone_tables(transfer, primaries, bpc,
    want_peak)); transfer None: no tone"""
    ref = DO._ref_pictures(tus)
    got = list(dec.tensors(tus, size=size, dtype=dtype, layout=layout, alloc=alloc, tonemap=tonemap, sdr_peak=sdr_peak, **kw))
    items = [t for g in got for t in g] if kw.get("batch") else got
    assert len(items) == len(ref)
    opts = {k: v for k, v in kw.items() if k in ("mean", "std", "antialias", "interpolation")}
    for k, ((w, h, bpc, lay, rp), g) in enumerate(zip(ref, items)):
        tone = stream.tone_tables(transfer, primaries, bpc, want_peak, sdr_peak) if transfer else None
        want = stream.tensor_reference(rp, bpc, lay, size, matrix, False, "left", tone=tone, **opts)
        if layout == "hwc":
            want = want.transpose(1, 2, 0)
        assert np.array_equal(TE._host_bits(g, dtype), TE._bits(want, dtype)), "picture %d differs" % k
    return items


@pytest.mark.emu
def test_color_metadata_emu(emu_dec):
    """refdrv_stream_color: primaries, transfer, MaxCLL / MaxFALL and the mastering display's luminances on every picture"""
    tus = _pq_stream(cll=(1234, 321), mdcv=(4000, 0.005), pri=12)
    seen = []
    list(emu_dec._decode(tus, lambda h, info: seen.append(emu_dec.color(h))))
    assert len(seen) == 3
    for c in seen:
        assert (c["primaries"], c["transfer"], c["max_cll"], c["max_fall"]) == (12, 16, 1234, 321)
        assert c["mastering_max"] == 4000 and abs(c["mastering_min"] - 0.005) < 1e-4
    seen = []
    list(emu_dec._decode(obu.inter_stream(51, 64, 48, n_frames=1), lambda h, info: seen.append(emu_dec.color(h))))
    assert seen == [dict(primaries=2, transfer=2, max_cll=0, max_fall=0, mastering_max=0.0, mastering_min=0.0)]


@pytest.mark.emu
def test_tensors_pq_auto_emu(emu_dec):
    """a 10-bit BT.2020 PQ stream with MaxCLL 1000: tonemap="auto" is the definition with the metadata's peak, resized,
    normalised, batched"""
    tus = _pq_stream()
    _check_tensors(emu_dec, tus, "auto", "pq", 9, 1000, size=(24, 40), dtype="bfloat16", batch=2, **IMAGENET)
    _check_tensors(emu_dec, tus, "auto", "pq", 9, 1000, size=(17, 31), antialias=True, interpolation="bicubic", layout="hwc")


@pytest.mark.emu
def test_tensors_pq_peak_follows_the_metadata_emu(emu_dec):
    """MaxCLL sets the curve; without it the mastering display's maximum does, and without either 1000 cd/m^2; peak=
    overrides all of them"""
    outs = []
    for cll, mdcv, peak in [((600, 100), None, 600), ((4000, 100), (1000, 0.01), 4000), (None, (2000, 0.01), 2000),
                            ((0, 0), (1500, 0.01), 1500), (None, None, 1000)]:
        tus = _pq_stream(cll=cll, mdcv=mdcv, n_frames=2)
        outs.append(_check_tensors(emu_dec, tus, "auto", "pq", 9, peak, size=(16, 24))[0])
    assert not np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[1], outs[2])
    tus = _pq_stream(cll=(600, 100), n_frames=2)
    _check_tensors(emu_dec, tus, "auto", "pq", 9, 350, size=(16, 24), peak=350)
    _check_tensors(emu_dec, tus, "pq", "pq", 9, 600, size=(16, 24), sdr_peak=100.0)


@pytest.mark.emu
def test_tensors_hlg_and_forced_emu(emu_dec):
    """HLG with P3 primaries through "auto"; "pq" and "hlg" forced on a stream without a colour description (BT.2020
    assumed), and on an SDR-labelled one; "auto" leaves an unlabelled stream alone"""
    hlg = _pq_stream(seed=52, cll=None, pri=12, trc=18)
    _check_tensors(emu_dec, hlg, "auto", "hlg", 12, 1000, size=(20, 30), antialias=True)
    plain = obu.inter_stream(53, 80, 56, n_frames=2, bpc=10)
    _check_tensors(emu_dec, plain, "pq", "pq", 2, 1000, size=(20, 30), matrix="bt709")
    _check_tensors(emu_dec, plain, "hlg", "hlg", 2, 1200, size=(20, 30), matrix="bt709", peak=1200)
    _check_tensors(emu_dec, plain, "auto", None, None, None, size=(20, 30), matrix="bt709")
    sdr = _pq_stream(seed=54, cll=None, pri=1, trc=1)
    _check_tensors(emu_dec, sdr, "hlg", "hlg", 1, 1000, size=(20, 30))


@pytest.mark.emu
def test_tonemap_auto_leaves_sdr_streams_alone_emu(emu_dec):
    """"auto" on SDR streams (every layout and bit depth, odd sizes, crops, flips, bicubic) is bit for bit tonemap=None"""
    streams = TC._mixed_streams() + [obu.inter_stream(55, 64, 48, n_frames=2, bpc=10, color=(9, 0, 9, 14))]
    for i, tus in enumerate(streams):
        kw = dict(size=(13, 9 + i), dtype=DTYPES[i % 3], alloc=TE._np_alloc, antialias=bool(i % 2), flip=i % 3 == 0,
                  interpolation=("bilinear", "bicubic")[i % 2], crop=(1, 2, 20, 30) if i % 2 else None)
        a = list(emu_dec.tensors(tus, **kw))
        b = list(emu_dec.tensors(tus, tonemap="auto", **kw))
        assert len(a) == len(b) and all(np.array_equal(TE._host_bits(x, kw["dtype"]), TE._host_bits(y, kw["dtype"]))
                                        for x, y in zip(a, b)), i


@pytest.mark.emu
def test_clips_mix_hdr_and_sdr_emu(emu_dec):
    """clips(tonemap="auto") over PQ, HLG and SDR streams: each picture is what tensors() exports for it"""
    streams = [_pq_stream(seed=56, n_frames=4), TC._mixed_streams()[0], _pq_stream(seed=57, cll=None, pri=12, trc=18, n_frames=4),
               obu.inter_stream(58, 61, 45, n_frames=4, bpc=10, layout="400", color=(9, 0)),
               _pq_stream(seed=59, cll=(3000, 100), n_frames=4, bpc=12, layout="444")]
    kw = dict(size=(11, 14), dtype="float16", layout="hwc", antialias=True, tonemap="auto", **IMAGENET)
    x = emu_dec.clips(streams, frames=2, step=1, start=1, alloc=TC._alloc, **kw)
    for i, tus in enumerate(streams):
        t_all = list(emu_dec.tensors(tus, alloc=TE._np_alloc, **kw))
        for t in range(2):
            assert np.array_equal(TE._host_bits(x[i, t], "float16"), TE._host_bits(t_all[1 + t], "float16")), (i, t)
    w, h, bpc, lay, rp = DO._ref_pictures(streams[4])[1]
    want = stream.tensor_reference(rp, bpc, lay, (11, 14), "bt2020", False, "left", antialias=True,
                                   tone=stream.tone_tables("pq", 9, 12, 3000), **IMAGENET).transpose(1, 2, 0)
    assert np.array_equal(TE._host_bits(x[4, 0], "float16"), TE._bits(want, "float16"))


@pytest.mark.emu
def test_tonemap_errors_emu(emu_dec):
    tus = _pq_stream(n_frames=1)
    for kw, match in [(dict(tonemap="hdr10"), "tonemap"), (dict(tonemap=True), "tonemap"), (dict(tonemap="auto", peak=0), "peak"),
                      (dict(tonemap="auto", peak="1000"), "peak"), (dict(tonemap="auto", sdr_peak=-5.0), "sdr_peak"),
                      (dict(tonemap="auto", sdr_peak=float("nan")), "sdr_peak")]:
        with pytest.raises(ValueError, match=match):
            list(emu_dec.tensors(tus, alloc=TE._np_alloc, **kw))
        with pytest.raises(ValueError, match=match):
            emu_dec.clips([tus], frames=1, alloc=TC._alloc, **kw)
    odd = _pq_stream(seed=60, cll=None, pri=4, n_frames=1)          # BT.470M primaries: not known to the tone map
    with pytest.raises(ValueError, match="color_primaries"):
        list(emu_dec.tensors(odd, alloc=TE._np_alloc, tonemap="auto"))
    assert len(list(emu_dec.tensors(odd, alloc=TE._np_alloc))) == 1


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
GPU_CASES = [(TE.Case(10, 1, 3840, 2160, (224, 224), "bfloat16", "chw", "left", "bt2020", False, **IMAGENET), "triangle", 0, None),
             (TE.Case(10, 1, 3840, 2160, (224, 224), "bfloat16", "chw", "left", "bt2020", False, **IMAGENET), "cubic_aa", 1, None),
             (TE.Case(10, 1, 3840, 2160, (1080, 1920), "float16", "hwc", "left", "bt2020", False, offset=1), "bilinear", 0, None),
             (TE.Case(10, 1, 1920, 1080, (224, 224), "float32", "chw", "center", "bt2020", True), "cubic", 1, (101, 333, 871, 1201)),
             (TE.Case(12, 3, 640, 360, (223, 221), "float32", "hwc", "left", "identity", False), "triangle", 1, None),
             (TE.Case(8, 0, 1280, 720, (300, 500), "bfloat16", "chw", "left", "bt709", False), "bilinear", 1, (7, 9, 600, 1000)),
             (TE.Case(10, 2, 1920, 1080, (224, 224), "float16", "hwc", "topleft", "bt2020", False), "cubic_aa", 0, (10, 20, 700, 900)),
             (TE.Case(12, 2, 1280, 720, (720, 1280), "bfloat16", "chw", "left", "bt2020", True), "cubic", 1, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES) + len(GPU_CASES)))
def test_tone_kernel_gpu(idx):
    """the emulator's cases, then full-size pictures"""
    from dav1d_b200 import _lib
    c, kind, flip, box = (KERNEL_CASES + GPU_CASES)[idx]
    got, want = _run(c, 8000 + idx, kind, flip, box, _lib.get_lib(), device=True)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["mixed", "uniform"])
def test_batch_mixing_tone_and_plain_jobs_gpu(mix):
    """a 37-job batch of every kind, class and flip; 35 tone-mapped jobs of one group between plain ones (three launches)"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    on_device = {}                          # id of a host array -> (the array, its device copy)

    def ptr_of(a):
        if id(a) not in on_device:
            on_device[id(a)] = (a, torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda())
        return on_device[id(a)][1].data_ptr()
    if mix == "mixed":
        n = 2 * TONE_MAX + 5
        cases, plan = _mixed_cases(n, "bfloat16", "chw", 77), _mixed_plan
    else:
        n = 2 * TONE_MAX + 3 + 11
        cases, plan = _uniform_cases(n, "float32", "hwc", 78), _uniform_plan
    jobs, tones, buf, want, spans, guard, _keep = _batch(cases, 77, plan, lambda a: torch.from_numpy(a).cuda(), ptr_of)
    d_buf = on_device[id(buf)][1]
    assert lib.b200_export_tensor_tone_batch(jobs, tones, n, None) == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    assert np.array_equal(d_buf.cpu().numpy().view(buf.dtype), want)


@pytest.mark.gpu
def test_tensors_and_clips_gpu(hooked_library, monkeypatch):
    """PQ (4K and 1080p, MaxCLL), HLG and SDR streams through tensors() and clips(tonemap="auto") on a non-default stream:
    each picture is the definition"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)
    pq4k = _pq_stream(seed=640, cll=(1500, 300), w=3840, h=2160, n_frames=3, log2_cols=2, log2_rows=1)
    hlg = _pq_stream(seed=641, cll=None, pri=9, trc=18, w=1920, h=1080, n_frames=3, log2_cols=2)
    sdr = obu.inter_stream(642, 1920, 1080, n_frames=3, bpc=8, log2_cols=2, film_grain=1)
    dec = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for kw in (dict(antialias=True, dtype="bfloat16", size=(224, 224), **IMAGENET),
                   dict(antialias=True, interpolation="bicubic", dtype="bfloat16", size=(224, 224), **IMAGENET),
                   dict(dtype="float16", size=(1080, 1920), layout="hwc"),
                   dict(interpolation="bicubic", dtype="float32", size=(360, 640))):
            got = _check_tensors(dec, pq4k, "auto", "pq", 9, 1500, alloc=None, **kw)
            assert all(g.is_cuda for g in got)
        _check_tensors(dec, hlg, "auto", "hlg", 9, 1000, alloc=None, size=(224, 224), antialias=True, interpolation="bicubic")
        x = dec.clips([pq4k, hlg, sdr], frames=2, step=1, size=(224, 224), dtype="float32", antialias=True, tonemap="auto")
    s.synchronize()
    for i, (tus, tone, matrix) in enumerate([(pq4k, ("pq", 9, 1500), "bt2020"), (hlg, ("hlg", 9, 1000), "bt2020"),
                                             (sdr, None, "bt709")]):
        for t, (w, h, bpc, lay, rp) in enumerate(DO._ref_pictures(tus)[:2]):
            want = stream.tensor_reference(rp, bpc, lay, (224, 224), matrix, False, "left", antialias=True,
                                           tone=stream.tone_tables(*tone[:2], bpc, tone[2]) if tone else None)
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)
    dec.release()
