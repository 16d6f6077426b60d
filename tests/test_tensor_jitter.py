"""Colour jitter and grayscale in the tensor export (B200ColorJitter and b200_export_tensor_jitter_batch, include/b200av1.h;
color_jitter and the contrast pass in dav1d_b200/csrc/export.cu; b200hook_export_tensor_jitter_batch, integration/dav1d;
jitter= / grayscale= of stream.DeviceDecoder.tensors and clips). The numpy statement (stream.jitter_reference) is checked
against torchvision's functional ops; the kernel must be stream.tensor_reference(..., jitter=, grayscale=) bit for bit.
CPU tests run the CUDA sources on the host emulator, GPU tests run the CUDA library into torch CUDA tensors."""
import ctypes as C
import itertools

import numpy as np
import pytest

import refs
from dav1d_b200 import stream

import test_clips as TC
import test_stream_device_output as DO
import test_tensor_export as TE
import test_tensor_tonemap as TT

DTYPES = list(stream.TENSOR_DTYPES)
IMAGENET = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
JITTER_MAX = 14                         # B200_TENSOR_JITTER_BATCH_MAX, include/b200av1.h


def _random_jitter(rng, p_none=0.25):
    """a ColorJitter(0.4, 0.4, 0.4, 0.1).get_params-like tuple, some factors None"""
    order = [int(v) for v in rng.permutation(4)]
    f = [float(rng.uniform(0.6, 1.4)) for _ in range(3)] + [float(rng.uniform(-0.1, 0.1))]
    return tuple([order] + [None if rng.random() < p_none else v for v in f])


# ---- the statement against torchvision -----------------------------------------------------------------------------
def _images(rng, h=13, w=17):
    """random pictures, plus grays, primaries, secondaries, saturated colours, ties and values at the hue sector edges"""
    x = rng.random((3, h, w), dtype=np.float32)
    special = [(0, 0, 0), (1, 1, 1), (0.5, 0.5, 0.5), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (0, 1, 1), (1, 0, 1),
               (1, 0.5, 0), (0.5, 1, 0), (0, 1, 0.5), (0, 0.5, 1), (0.5, 0, 1), (1, 0, 0.5), (0.9, 0.9, 0.1), (0.2, 0.7, 0.7),
               (1, 1e-7, 0), (1, 0, 1e-7), (0.25, 0.75, 0.75), (1e-3, 0, 0), (0.999, 1, 0.999)]
    for k, c in enumerate(special):
        x[:, k // w, k % w] = c
    return x


def _torchvision_chain(x, jitter, v2):
    import torch
    if v2:
        from torchvision.transforms.v2 import functional as F
        fns = [F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue]
    else:
        from torchvision.transforms import _functional_tensor as F
        fns = [F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue]
    t = torch.from_numpy(x.copy())
    for op in jitter[0]:
        if jitter[1 + op] is not None:
            t = fns[op](t, jitter[1 + op])
    return t.numpy()


def _check_statement(x, jitter, tol=1e-5):
    pytest.importorskip("torchvision")
    got = stream.jitter_reference(x, jitter)
    for v2 in (False, True):
        want = _torchvision_chain(x, jitter, v2)
        assert np.abs(got - want).max() <= tol, (jitter, v2, np.abs(got - want).max())


@pytest.mark.parametrize("op,factor", [(op, f) for op in range(3) for f in (0.0, 0.3, 1.0, 1.7, 2.0)] +
                         [(3, f) for f in (-0.5, -0.25, -0.01, 0.0, 0.01, 0.25, 0.5)])
def test_statement_one_op(op, factor):
    """each op alone at its edge factors (0 and 2 for the blends, +-0.5 for hue: the remainder wraps)"""
    rng = np.random.default_rng(op * 100 + int(factor * 100))
    jitter = tuple([[op] + [k for k in range(4) if k != op]] + [factor if k == op else None for k in range(4)])
    _check_statement(_images(rng), jitter)


@pytest.mark.parametrize("order", list(itertools.permutations(range(4))))
def test_statement_every_order(order):
    rng = np.random.default_rng(sum(v * 4 ** k for k, v in enumerate(order)))
    for _ in range(3):
        f = [float(rng.uniform(0, 2)) for _ in range(3)] + [float(rng.uniform(-0.5, 0.5))]
        _check_statement(_images(rng), tuple([list(order)] + f))


def test_statement_grayscale_and_sector_edges():
    """grayscale is torchvision's rgb_to_grayscale on 3 channels; hue on colours whose h lands on the sector edges"""
    pytest.importorskip("torchvision")
    import torch
    from torchvision.transforms import _functional_tensor as F
    rng = np.random.default_rng(5)
    x = _images(rng)
    got = stream.jitter_reference(x, None, grayscale=True)
    want = F.rgb_to_grayscale(torch.from_numpy(x), num_output_channels=3).numpy()
    assert np.array_equal(got, want)
    # hues k / 6 (sector edges) and just beside them, shifted across the wrap at 0 / 1
    hs = np.array([k / 6 + d for k in range(7) for d in (-1e-7, 0, 1e-7)], np.float32) % 1
    import colorsys
    rgb = np.array([colorsys.hsv_to_rgb(h, 0.8, 0.9) for h in hs], np.float32).T.reshape(3, 3, 7)
    for hue in (-0.5, -1 / 6, -1e-7, 0.0, 1e-7, 1 / 6, 0.5):
        _check_statement(rgb, ([3, 0, 1, 2], None, None, None, hue))


def test_factors_follow_torchvision():
    """c1 and s1 are f32(1.0 - factor) of the float64 difference; disabled ops are neutral; the enable bits follow None"""
    order, enabled, b, c, s, h, c1, s1 = stream.jitter_factors(([2, 0, 3, 1], 0.1, 1.1, None, -0.2))
    assert order == [2, 0, 3, 1] and enabled == 0b1011
    assert (b, c, s, h) == (np.float32(0.1), np.float32(1.1), np.float32(1), np.float32(-0.2))
    assert c1 == np.float32(1.0 - 1.1) and s1 == 0
    assert stream.jitter_factors(([0, 1, 2, 3], None, None, None, None))[1] == 0


def test_bad_jitter_tuples():
    for bad in [None, (1, 2, 3), ([0, 1, 2], 1, 1, 1, 0), ([0, 1, 2, 2], 1, 1, 1, 0), ([0, 1, 2, 4], 1, 1, 1, 0),
                ([0, 1, 2, 3], -0.1, 1, 1, 0), ([0, 1, 2, 3], 1, -1, 1, 0), ([0, 1, 2, 3], 1, 1, -2, 0),
                ([0, 1, 2, 3], 1, 1, 1, 0.6), ([0, 1, 2, 3], 1, 1, 1, -0.51), ([0, 1, 2, 3], float("nan"), 1, 1, 0),
                ([0, 1, 2, 3], 1, float("inf"), 1, 0), ([0, 1, 2, 3], "1", 1, 1, 0), ([0, 1, 2, 3], True, 1, 1, 0)]:
        with pytest.raises(ValueError):
            stream.jitter_factors(bad)


# ---- kernel level -------------------------------------------------------------------------------------------------
KINDS = TT.KINDS


def _jitter_struct(jitter, gray, acc_ptr):
    return stream.color_jitter(jitter, gray, acc=acc_ptr)


def _expected(c, planes, pc, py, n, guard, kind, flip, tone, jitter, gray):
    aa, interp = KINDS[kind]
    ref = stream.tensor_reference(planes, c.bpc, c.layout, c.size, c.matrix, c.full_range, c.siting, c.mean, c.std,
                                  antialias=aa, interpolation=interp, tone=tone, jitter=jitter, grayscale=gray)
    if flip:
        ref = ref[:, :, ::-1].copy()
    bits = TE._bits(ref, c.dtype)
    out = np.full(n, guard, bits.dtype)
    _, oh, ow = ref.shape
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    for ch in range(3):
        out[ch * pc + y * py + x if c.lay == "chw" else y * py + 3 * x + ch] = bits[ch]
    return out


def _jobs_scale(j, c):
    scale, bias = stream.tensor_scale_bias(c.bpc, c.mean, c.std, jittered=True)
    for k in range(3):
        j.scale[k], j.bias[k] = float(scale[k]), float(bias[k])


def _run(c, seed, kind, flip, box, tone_on, jitter, gray, lib, device=False):
    """one jittered job (c: the full picture; box: a crop of it or None) into a guarded destination: (written, wanted)"""
    rng = np.random.default_rng(seed)
    planes = TE._planes(rng, c)
    tone = TT._tone_args(c, seed) if tone_on else None
    src, offs, strides = TT._crop_source(planes, c.layout, box, 64 if device else 7)
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
        acc = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
        j = TE._job(cj, d_src.data_ptr(), offs, strides, buf.data_ptr() + (TE.GUARD + c.offset) * buf.element_size(), pc, py)
        tm = TT._tone_struct(tone, keep, lambda a: torch.from_numpy(a).cuda()) if tone_on else None
        acc_ptr = acc.data_ptr()
    else:
        buf = np.full(total, guard, et)
        acc = np.full(1, 12345, np.uint64)
        j = TE._job(cj, src.ctypes.data, offs, strides, buf.ctypes.data + (TE.GUARD + c.offset) * buf.itemsize, pc, py)
        tm = TT._tone_struct(tone, keep) if tone_on else None
        acc_ptr = acc.ctypes.data
    j.antialias, j.flip, j.interpolation = aa, flip, stream.TENSOR_INTERPOLATIONS[interp]
    _jobs_scale(j, cj)
    jt = _jitter_struct(jitter, gray, acc_ptr)
    tones = (C.POINTER(stream.ToneMap) * 1)(C.pointer(tm)) if tone_on else None
    jits = (C.POINTER(stream.ColorJitter) * 1)(C.pointer(jt))
    assert lib.b200_export_tensor_jitter_batch(C.byref(j), tones, jits, 1, None) == 0, lib.b200_last_error()
    if device:
        torch.cuda.synchronize()
        buf = TE._host_bits(buf, c.dtype)
    want = np.full(total, guard, et)
    part = stream.crop_planes(planes, c.layout, box) if box else planes
    want[TE.GUARD + c.offset:TE.GUARD + c.offset + n] = _expected(cj, part, pc, py, n, guard, kind, flip, tone, jitter, gray)
    return buf, want


def _kernel_cases():
    """every kind x bit depth x chroma layout (4:4:4 with the identity matrix), every dtype and layout, flips, crops, tone
    maps and grayscale, ragged widths and misaligned destinations; contrast in most jitters"""
    geo = [(45, 27, (13, 22)), (38, 21, (9, 3)), (64, 48, (5, 1)), (33, 31, (40, 11)), (61, 33, (7, 16)), (30, 20, (45, 31))]
    rng = np.random.default_rng(77)
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
                jitter = None if k % 11 == 5 else _random_jitter(rng)
                cases.append((c, kind, k % 2, box, k % 4 == 1, jitter, k % 5 == 3 or jitter is None))
                k += 1
    return cases


KERNEL_CASES = _kernel_cases()


@pytest.mark.emu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES)))
def test_jitter_kernel_emu(idx):
    c, kind, flip, box, tone, jitter, gray = KERNEL_CASES[idx]
    got, want = _run(c, 9000 + idx, kind, flip, box, tone, jitter, gray, refs.emu_lib())
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d (%s %s %s)" % (bad.size, bad[0], kind, jitter, c.__dict__)


@pytest.mark.emu
@pytest.mark.parametrize("jitter", [([1, 0, 2, 3], 0.0, 2.0, 0.0, 0.5), ([3, 2, 1, 0], 2.0, 0.0, 2.0, -0.5),
                                    ([0, 3, 1, 2], 1.0, 1.0, 1.0, 0.0), ([2, 3, 0, 1], 1e-39, 1e-30, 1e-20, 1e-40)])
def test_jitter_edge_factors_emu(jitter):
    """neutral, zero, doubling and +-0.5 factors, and factors small enough to reach subnormal products"""
    c = TE.Case(10, 1, 40, 30, (17, 23), "float32", "chw", "left", "bt709", False)
    got, want = _run(c, 91, "triangle", 0, None, False, jitter, False, refs.emu_lib())
    assert np.array_equal(got, want)


def _mixed_plan(k):
    """(kind, flip, tone map, jitter, grayscale) of job k of a mixed batch: jittered (k % 3 != 2), tone-mapped (k % 4 == 0)
    and plain jobs of every kind"""
    rng = np.random.default_rng(500 + k)
    jit = k % 3 != 2
    return list(KINDS)[(k // 3) % 4], k % 5 == 0, k % 4 == 0, _random_jitter(rng) if jit else None, jit and k % 7 == 1


def _batch(cases, seed, plan, acc, acc_ptr, to_dev=None, ptr_of=lambda a: a.ctypes.data):
    """the jobs of `cases` as plan(k) says: (jobs, tones, jitters, destination, what it must hold, keep)"""
    n = len(cases)
    srcs, spans, buf, guard = TC._batch_setup(cases, seed, ptr_of)
    jobs = (stream.TensorJob * n)()
    tones = (C.POINTER(stream.ToneMap) * n)()
    jits = (C.POINTER(stream.ColorJitter) * n)()
    want = np.full_like(buf, guard)
    keep = []
    for k, ((c, planes, src, offs, strides, pc, py, m), at) in enumerate(zip(srcs, spans)):
        kind, flip, has_tone, jitter, gray = plan(k)
        aa, interp = KINDS[kind]
        jobs[k] = TE._job(c, ptr_of(src), offs, strides, ptr_of(buf) + at * buf.itemsize, pc, py)
        jobs[k].antialias, jobs[k].flip, jobs[k].interpolation = aa, flip, stream.TENSOR_INTERPOLATIONS[interp]
        tone = TT._tone_args(c, k) if has_tone else None
        if tone is not None:
            tones[k] = C.pointer(TT._tone_struct(tone, keep, to_dev))
        if jitter is not None or gray:
            _jobs_scale(jobs[k], c)
            keep.append(_jitter_struct(jitter, gray, acc_ptr + 8 * k))
            jits[k] = C.pointer(keep[-1])
        want[at:at + m] = _expected(c, planes, pc, py, m, guard, kind, flip, tone, jitter, gray)
    return jobs, tones, jits, buf, want, (srcs, keep)


@pytest.mark.emu
@pytest.mark.parametrize("n,dtype,lay", [(3 * JITTER_MAX + 5, "float32", "hwc"), (JITTER_MAX + 1, "bfloat16", "chw")])
def test_batch_mixing_jitter_tone_and_plain_jobs_emu(n, dtype, lay):
    """jittered (with and without tone maps), tone-mapped and plain jobs of every kind, both bit-depth classes and flips,
    beyond the jitter batch cap, in one call: each is the definition"""
    lib = refs.emu_lib()
    cases = TT._mixed_cases(n, dtype, lay, 1500 + n)
    acc = np.zeros(n, np.uint64)
    jobs, tones, jits, buf, want, _keep = _batch(cases, 1500 + n, _mixed_plan, acc, acc.ctypes.data)
    assert lib.b200_export_tensor_jitter_batch(jobs, tones, jits, n, None) == 0, lib.b200_last_error()
    assert np.array_equal(buf, want)


@pytest.mark.emu
def test_jitter_jobs_split_into_launches_emu():
    """2 * cap + 3 jittered jobs of one group: ceil(n / cap) groups, each a zero launch, a contrast pass and the export;
    a group without contrast takes the export alone"""
    lib = refs.emu_lib()
    n = 2 * JITTER_MAX + 3
    cases = TT._uniform_cases(n, "float16", "hwc", 1600)
    acc = np.zeros(n, np.uint64)
    plan = lambda k: ("triangle", False, False, ([1, 0, 2, 3], 1.2, 0.8, 1.1, 0.05), False)
    jobs, tones, jits, buf, want, _keep = _batch(cases, 1600, plan, acc, acc.ctypes.data)
    before = lib.b200_launch_count()
    assert lib.b200_export_tensor_jitter_batch(jobs, tones, jits, n, None) == 0, lib.b200_last_error()
    assert lib.b200_launch_count() - before == 3 * -(-n // JITTER_MAX)
    assert np.array_equal(buf, want)
    plan = lambda k: ("triangle", False, False, ([1, 0, 2, 3], 1.2, None, 1.1, 0.05), k % 2 == 0)
    jobs, tones, jits, buf, want, _keep = _batch(cases, 1600, plan, acc, acc.ctypes.data)
    before = lib.b200_launch_count()
    assert lib.b200_export_tensor_jitter_batch(jobs, tones, jits, n, None) == 0, lib.b200_last_error()
    assert lib.b200_launch_count() - before == -(-n // JITTER_MAX)
    assert np.array_equal(buf, want)


@pytest.mark.emu
def test_null_jitters_are_the_tone_batch_emu():
    """jitters = NULL, or all NULL entries, writes what b200_export_tensor_tone_batch writes"""
    lib = refs.emu_lib()
    n = 9
    cases = TT._mixed_cases(n, "float32", "chw", 33)
    acc = np.zeros(n, np.uint64)
    plan = lambda k: TT._mixed_plan(k) + (None, False)
    jobs, tones, jits, buf, want, _keep = _batch(cases, 33, plan, acc, acc.ctypes.data)
    g = buf[0]
    for j in (None, jits):
        buf[:] = g
        assert lib.b200_export_tensor_jitter_batch(jobs, tones, j, n, None) == 0
        assert np.array_equal(buf, want)
    again = np.full_like(buf, g)
    for k in range(n):
        jobs[k].dst = again.ctypes.data + (jobs[k].dst - buf.ctypes.data)
    assert lib.b200_export_tensor_tone_batch(jobs, tones, n, None) == 0
    assert np.array_equal(again, want)


@pytest.mark.emu
def test_bad_jitters_emu():
    """a factor that is not finite, negative blend factors, a hue outside [-0.5, 0.5], an order that is not a permutation,
    stray enabled bits, a bad grayscale, a NULL or misaligned acc with contrast: -2, the error set, nothing written"""
    lib = refs.emu_lib()
    n = 6
    cases = TT._mixed_cases(n, "float32", "chw", 31)
    acc = np.zeros(n + 1, np.uint64)
    plan = lambda k: ("bilinear", False, False, ([0, 1, 2, 3], 1.1, 0.9, 1.2, 0.1), False)
    jobs, tones, jits, buf, _, _keep = _batch(cases, 31, plan, acc, acc.ctypes.data)
    guard = buf.copy()
    good = stream.ColorJitter.from_buffer_copy(jits[2].contents)
    for field, value in [("brightness", float("nan")), ("contrast", float("inf")), ("saturation", float("-inf")),
                         ("hue", float("nan")), ("contrast1", float("inf")), ("saturation1", float("nan")),
                         ("brightness", -1e-3), ("contrast", -1.0), ("saturation", -0.5), ("hue", 0.5001), ("hue", -0.6),
                         ("order", (0, 1, 2, 2)), ("order", (0, 1, 2, 4)), ("order", (-1, 1, 2, 3)), ("enabled", 16),
                         ("enabled", -1), ("grayscale", 2), ("acc", None), ("acc", acc.ctypes.data + 4)]:
        bad = stream.ColorJitter.from_buffer_copy(good)
        if field == "order":
            bad.order[:] = value
        else:
            setattr(bad, field, value)
        t = (C.POINTER(stream.ColorJitter) * n)(*[jits[k] for k in range(n)])
        t[2] = C.pointer(bad)
        assert lib.b200_export_tensor_jitter_batch(jobs, None, t, n, None) == -2, field
        assert b"jitter" in lib.b200_last_error()
        assert np.array_equal(buf, guard)
    ok = stream.ColorJitter.from_buffer_copy(good)
    ok.enabled, ok.acc = 0b1101, None                   # no contrast: no scratch needed
    t = (C.POINTER(stream.ColorJitter) * n)(*[jits[k] for k in range(n)])
    t[2] = C.pointer(ok)
    assert lib.b200_export_tensor_jitter_batch(jobs, None, t, n, None) == 0, lib.b200_last_error()


def test_jitter_abi():
    """B200ColorJitter is 56 bytes; 14 jobs with their tone maps and jitters fit the 4 KB parameter block"""
    from dav1d_b200 import _lib
    assert C.sizeof(stream.ColorJitter) == 56
    assert JITTER_MAX * (C.sizeof(stream.ColorJitter) + C.sizeof(stream.ToneMap) + C.sizeof(stream.TensorJob)) + 4 <= 4096
    assert _lib.ABI_STRUCTS[25] is stream.ColorJitter
    assert "b200_export_tensor_jitter_batch" in _lib.B200Lib.symbols()


@pytest.mark.emu
def test_jitter_size_in_the_library_emu():
    assert refs.emu_lib().b200_struct_size(25) == C.sizeof(stream.ColorJitter)


# ---- decoder level ------------------------------------------------------------------------------------------------
def _want(rp, bpc, lay, size, kw, jitter, gray, tone=None, flip=False, matrix="bt709"):
    opts = {k: v for k, v in kw.items() if k in ("mean", "std", "antialias", "interpolation")}
    want = stream.tensor_reference(rp, bpc, lay, size, matrix, False, "left", tone=tone, jitter=jitter, grayscale=gray, **opts)
    return want[:, :, ::-1] if flip else want


@pytest.mark.emu
def test_tensors_jitter_emu(emu_dec):
    """tensors(jitter=callable, grayscale=callable): each picture its own parameters (None: the plain export), each
    picture's own contrast mean, batched and not"""
    tus = TC._mixed_streams()[0]
    ref = DO._ref_pictures(tus)
    rng = np.random.default_rng(4)
    params = [_random_jitter(rng, 0.1) if k % 3 else None for k in range(len(ref))]
    grays = [k % 4 == 2 for k in range(len(ref))]
    for kw in (dict(size=(24, 40), dtype="bfloat16", batch=3, **IMAGENET),
               dict(size=(17, 31), antialias=True, interpolation="bicubic", layout="hwc", flip=True)):
        got = list(emu_dec.tensors(tus, alloc=TE._np_alloc, jitter=lambda k: params[k], grayscale=lambda k: grays[k],
                                   matrix="bt601", full_range=True, **kw))
        items = [t for g in got for t in g] if kw.get("batch") else got
        assert len(items) == len(ref)
        for k, ((w, h, bpc, lay, rp), g) in enumerate(zip(ref, items)):
            want = stream.tensor_reference(rp, bpc, lay, kw["size"], "bt601", True, "left", jitter=params[k], grayscale=grays[k],
                                           **{o: v for o, v in kw.items() if o in ("mean", "std", "antialias", "interpolation")})
            if kw.get("flip"):
                want = want[:, :, ::-1]
            if kw.get("layout") == "hwc":
                want = want.transpose(1, 2, 0)
            assert np.array_equal(TE._host_bits(g, kw["dtype"] if "dtype" in kw else "float32"),
                                  TE._bits(np.ascontiguousarray(want), kw.get("dtype", "float32"))), k


@pytest.mark.emu
def test_jitter_none_is_the_plain_export_emu(emu_dec):
    """jitter=None, grayscale=False (and a callable returning None / False) export exactly as without the arguments"""
    for i, tus in enumerate(TC._mixed_streams()[:3]):
        kw = dict(size=(13, 9 + i), dtype=DTYPES[i % 3], alloc=TE._np_alloc, antialias=bool(i % 2), flip=i % 2 == 0)
        a = list(emu_dec.tensors(tus, **kw))
        for extra in (dict(jitter=None, grayscale=False), dict(jitter=lambda k: None, grayscale=lambda k: False)):
            b = list(emu_dec.tensors(tus, **extra, **kw))
            assert len(a) == len(b) and all(np.array_equal(TE._host_bits(x, kw["dtype"]), TE._host_bits(y, kw["dtype"]))
                                            for x, y in zip(a, b)), i


@pytest.mark.emu
def test_clips_jitter_emu(emu_dec):
    """clips(): per-stream parameters held across each clip (a callable asked once per stream, returning None for one),
    per-picture contrast means, and a batch mixing jittered, HDR and plain streams"""
    streams = TC._mixed_streams()[:3] + [TT._pq_stream(seed=70, n_frames=4), TC._mixed_streams()[3]]
    rng = np.random.default_rng(8)
    params = {0: _random_jitter(rng, 0), 1: None, 2: ([1, 3, 0, 2], 1.3, 0.5, 1.6, -0.3), 3: _random_jitter(rng, 0), 4: None}
    asked = []

    def pick(i):
        asked.append(i)
        return params[i]
    grays = [False, False, True, False, True]
    kw = dict(size=(11, 14), dtype="float32", layout="chw", antialias=True, tonemap="auto", **IMAGENET)
    x = emu_dec.clips(streams, frames=2, step=1, start=1, alloc=TC._alloc, jitter=pick, grayscale=grays, flip=[False, True, False, True, True],
                      **kw)
    assert sorted(asked) == list(range(5))
    for i, tus in enumerate(streams):
        ref = DO._ref_pictures(tus)
        tone = stream.tone_tables("pq", 9, 10, 1000) if i == 3 else None
        matrix = {0: "bt601", 3: "bt2020", 4: "bt2020"}.get(i, "bt709")
        full = i == 0
        for t in range(2):
            w, h, bpc, lay, rp = ref[1 + t]
            want = stream.tensor_reference(rp, bpc, lay, (11, 14), matrix, full, "left", antialias=True, tone=tone,
                                           jitter=params[i], grayscale=grays[i], **IMAGENET)
            if i in (1, 3, 4):
                want = want[:, :, ::-1]
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(np.ascontiguousarray(want), "float32")), (i, t)
    # one tuple for every stream, and one per stream
    one = ([2, 1, 0, 3], 0.8, 1.2, None, 0.2)
    a = emu_dec.clips(streams[:2], frames=1, alloc=TC._alloc, jitter=one, size=(9, 9))
    b = emu_dec.clips(streams[:2], frames=1, alloc=TC._alloc, jitter=[one, one], size=(9, 9))
    assert np.array_equal(a, b)


@pytest.mark.emu
def test_jitter_errors_emu(emu_dec):
    """malformed tuples, out-of-range factors and bad grayscale values: ValueError naming the picture or the stream"""
    tus = TC._mixed_streams()[0]
    bad = ([0, 1, 2, 3], 1.0, -1.0, 1.0, 0.0)
    for kw, match in [(dict(jitter=bad), "contrast"), (dict(jitter=(1, 2)), "jitter"), (dict(grayscale=1), "grayscale"),
                      (dict(jitter=lambda k: bad if k == 2 else None), "picture 2"),
                      (dict(grayscale=lambda k: "yes"), "picture 0")]:
        with pytest.raises(ValueError, match=match):
            list(emu_dec.tensors(tus, alloc=TE._np_alloc, **kw))
    for kw, match in [(dict(jitter=[None, bad]), "stream 1"), (dict(jitter=lambda i: bad if i else None), "stream 1"),
                      (dict(grayscale=[True]), "grayscale"), (dict(jitter=[None]), "jitter")]:
        with pytest.raises(ValueError, match=match):
            emu_dec.clips([tus, tus], frames=1, alloc=TC._alloc, **kw)


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
GPU_CASES = [(TE.Case(10, 1, 3840, 2160, (224, 224), "bfloat16", "chw", "left", "bt2020", False, **IMAGENET), "triangle", 0, None, False),
             (TE.Case(10, 1, 3840, 2160, (224, 224), "bfloat16", "chw", "left", "bt2020", False, **IMAGENET), "cubic_aa", 1, None, True),
             (TE.Case(8, 1, 1920, 1080, (224, 224), "float16", "hwc", "left", "bt709", False), "triangle", 1, (101, 333, 871, 1201), False),
             (TE.Case(10, 1, 3840, 2160, (1080, 1920), "float16", "hwc", "left", "bt2020", False, offset=1), "bilinear", 0, None, True),
             (TE.Case(12, 3, 640, 360, (223, 221), "float32", "hwc", "left", "identity", False), "cubic", 1, None, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(KERNEL_CASES) + len(GPU_CASES)))
def test_jitter_kernel_gpu(idx):
    """the emulator's cases through the C ABI, then full-size pictures"""
    from dav1d_b200 import _lib
    if idx < len(KERNEL_CASES):
        c, kind, flip, box, tone, jitter, gray = KERNEL_CASES[idx]
    else:
        c, kind, flip, box, tone = GPU_CASES[idx - len(KERNEL_CASES)]
        jitter, gray = _random_jitter(np.random.default_rng(idx), 0), idx % 2 == 0
    got, want = _run(c, 9500 + idx, kind, flip, box, tone, jitter, gray, _lib.get_lib(), device=True)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d elements differ, first at %d" % (bad.size, bad[0])


@pytest.mark.gpu
def test_batch_mixing_jitter_tone_and_plain_jobs_gpu():
    """a 47-job batch of every kind, class, flip and epilogue, beyond the jitter batch cap"""
    import torch
    from dav1d_b200 import _lib
    lib = _lib.get_lib()
    on_device = {}

    def ptr_of(a):
        if id(a) not in on_device:
            on_device[id(a)] = (a, torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda())
        return on_device[id(a)][1].data_ptr()
    n = 3 * JITTER_MAX + 5
    acc = torch.zeros(n, dtype=torch.int64, device="cuda")
    cases = TT._mixed_cases(n, "bfloat16", "chw", 88)
    jobs, tones, jits, buf, want, _keep = _batch(cases, 88, _mixed_plan, acc, acc.data_ptr(), lambda a: torch.from_numpy(a).cuda(),
                                                  ptr_of)
    d_buf = on_device[id(buf)][1]
    assert lib.b200_export_tensor_jitter_batch(jobs, tones, jits, n, None) == 0, lib.b200_last_error()
    torch.cuda.synchronize()
    assert np.array_equal(d_buf.cpu().numpy().view(buf.dtype), want)


@pytest.mark.gpu
def test_tensors_and_clips_gpu(hooked_library, monkeypatch):
    """4K and 1080p streams through tensors() and clips() with jitter on a non-default stream: each picture is the
    definition"""
    import torch
    monkeypatch.setattr(stream.decode_stream, "capacity", 1 << 30)
    from dav1d_b200 import obu
    big = obu.inter_stream(740, 3840, 2160, n_frames=3, bpc=10, log2_cols=2, log2_rows=1)
    pq = TT._pq_stream(seed=741, cll=(1500, 300), w=1920, h=1080, n_frames=3, log2_cols=2)
    sdr = obu.inter_stream(742, 1920, 1080, n_frames=3, bpc=8, log2_cols=2, film_grain=1)
    dec = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    rng = np.random.default_rng(9)
    params = [_random_jitter(rng, 0) for _ in range(3)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        kw = dict(antialias=True, dtype="bfloat16", size=(224, 224), **IMAGENET)
        got = list(dec.tensors(big, jitter=lambda k: params[k], grayscale=lambda k: k == 1, **kw))
        x = dec.clips([big, pq, sdr], frames=2, step=1, size=(224, 224), dtype="float32", antialias=True, tonemap="auto",
                      jitter=[params[0], None, params[2]], grayscale=[False, True, False], flip=[True, False, False])
    s.synchronize()
    for k, (w, h, bpc, lay, rp) in enumerate(DO._ref_pictures(big)):
        want = stream.tensor_reference(rp, bpc, lay, (224, 224), "bt709", False, "left", antialias=True, jitter=params[k],
                                       grayscale=k == 1, **IMAGENET)
        assert np.array_equal(TE._host_bits(got[k], "bfloat16"), TE._bits(want, "bfloat16")), k
    for i, (tus, tone, matrix, jit, gray, fl) in enumerate([(big, None, "bt709", params[0], False, True),
                                                             (pq, stream.tone_tables("pq", 9, 10, 1500), "bt2020", None, True, False),
                                                             (sdr, None, "bt709", params[2], False, False)]):
        for t, (w, h, bpc, lay, rp) in enumerate(DO._ref_pictures(tus)[:2]):
            want = stream.tensor_reference(rp, bpc, lay, (224, 224), matrix, False, "left", antialias=True, tone=tone,
                                           jitter=jit, grayscale=gray)
            if fl:
                want = np.ascontiguousarray(want[:, :, ::-1])
            assert np.array_equal(TE._host_bits(x[i, t], "float32"), TE._bits(want, "float32")), (i, t)
    dec.release()
