"""Device output (stream.DeviceDecoder): pictures stay in the decoder's device memory and one export kernel
(dav1d_b200/csrc/export.cu) writes them into caller memory as planes or as RGB. The planes must be stock dav1d's pictures
byte for byte, the RGB the numpy statement of the export's formula (stream.rgb_reference) applied to stock dav1d's pictures.
CPU tests bind the hooks to the host emulator (its "device" memory is host memory: numpy destinations); GPU tests bind the
CUDA library and export into torch CUDA tensors."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import refs
from dav1d_b200 import cli, obu, stream

MATRICES = ["bt601", "bt709", "bt2020"]


@pytest.fixture(scope="module", autouse=True)
def hooked_library():
    stream.build_hooked()
    if not os.path.exists(stream.HOOKED_SO):
        pytest.skip("%s not built" % stream.HOOKED_SO)


def _emu_path():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(refs.ROOT, "tests", "emu", "build_emu.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return m.build()


@pytest.fixture(scope="module")
def emu_device_decoder():
    refs.emu_lib()
    d = stream.DeviceDecoder(backend=_emu_path(), serialize=True, apply_grain=1)
    yield d
    d.release()


def _host(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else a
    return a.view(np.uint16) if a.dtype == np.int16 else a


def _ref_pictures(tus, apply_grain=1):
    r, info, packed = stream.decode_stream(C.CDLL(refs.REF_SO), tus, apply_grain=apply_grain, max_pics=len(tus) + 8)
    assert r > 0, "stock dav1d could not decode the stream (%d)" % r
    return [(int(i[0]), int(i[1]), int(i[2]), int(i[3]), planes) for i, (_, _, _, planes) in zip(info, cli.frames_of(info, packed))]


def _np_alloc(shape, dtype):
    return np.full(shape, 0x5a, dtype)          # not zero: a sample the export does not write shows up


def _check_planes(dec, tus, alloc=_np_alloc, **kw):
    ref = _ref_pictures(tus)
    dec.stats(reset=True)
    got = list(dec.pictures(tus, alloc=alloc, **kw))
    assert len(got) == len(ref)
    for k, ((w, h, bpc, layout, rp), gp) in enumerate(zip(ref, got)):
        assert len(gp) == len(rp), k
        for pl, (a, b) in enumerate(zip(gp, rp)):
            assert a.dtype == (np.uint8 if bpc == 8 else np.int16) or str(a.dtype) == ("torch.uint8" if bpc == 8 else "torch.int16")
            assert np.array_equal(_host(a), b), "picture %d plane %d differs" % (k, pl)
    st = dec.stats(reset=True)
    assert st["d2h_bytes"] == 0 and st["frames"] > 0
    return ref


def _check_rgb(dec, tus, matrix, full_range, alloc=_np_alloc, **kw):
    ref = _ref_pictures(tus)
    got = list(dec.pictures(tus, format="rgb", matrix=matrix, full_range=full_range, alloc=alloc, **kw))
    assert len(got) == len(ref)
    name = "bt709" if matrix == "auto" else matrix
    for k, ((w, h, bpc, layout, rp), g) in enumerate(zip(ref, got)):
        assert tuple(g.shape) == (3, h, w)
        want = stream.rgb_reference(rp, bpc, layout, name, bool(full_range))
        assert np.array_equal(_host(g).astype(np.int64), want), "picture %d: RGB differs (%s, full range %s)" % (k, matrix, full_range)
    dec.stats(reset=True)


PLANE_CASES = [
    ("key 8 bit", lambda: obu.intra_stream(1, 256, 192, n_frames=2, log2_cols=1)),
    ("inter 10 bit, odd size", lambda: obu.inter_stream(2, 201, 135, n_frames=4, bpc=10, motion_modes=2)),
    ("inter 12 bit 4:4:4", lambda: obu.inter_stream(3, 200, 136, n_frames=3, bpc=12, layout="444", motion_modes=2)),
    ("inter 8 bit 4:0:0, odd size", lambda: obu.inter_stream(4, 199, 121, n_frames=3, layout="400", motion_modes=1)),
    ("inter 10 bit film grain", lambda: obu.inter_stream(5, 320, 192, n_frames=4, bpc=10, film_grain=1, motion_modes=2)),
    ("key 12 bit 4:0:0 film grain", lambda: obu.intra_stream(6, 200, 136, n_frames=2, bpc=12, layout="400", film_grain=1)),
    ("super-resolution key frames", lambda: obu.intra_stream(900, 328, 200, n_frames=2, bpc=10, super_res=1, log2_cols=1)),
    ("super-resolution inter frames, grain", lambda: obu.inter_stream(950, 320, 192, n_frames=5, super_res=1, film_grain=1)),
    ("scaled references", lambda: obu.inter_stream(701, 320, 192, n_frames=6, sizes=[(256, 160), (320, 192), (200, 120), (320, 176)],
                                                   bpc=10, motion_modes=1, film_grain=1)),
    ("hidden frames shown later, grain", lambda: obu.inter_stream(30, 256, 192, n_frames=7, bpc=10, film_grain=1, motion_modes=2, hidden_every=2)),
]


@pytest.mark.emu
@pytest.mark.parametrize("name,make", PLANE_CASES, ids=[c[0] for c in PLANE_CASES])
def test_planes_match_stock_dav1d_emu(emu_device_decoder, name, make):
    _check_planes(emu_device_decoder, make())


@pytest.mark.emu
def test_planes_422_and_intra_block_copy_emu(emu_device_decoder):
    """4:2:2 key and inter frames, and key frames with intra block copy (streams stock dav1d accepts, drawn like test_stream.py does)"""
    import test_stream as TS
    streams = TS._valid_422("inter", 128, 64, 10, 1, motion_modes=1, film_grain=1) + TS._valid_422("intra", 128, 128, 8, 1) + \
        TS._valid_intrabc(256, 192, 1, bpc=8, layout="444") + TS._valid_intrabc(192, 128, 1, bpc=10)
    assert len(streams) == 4
    for tus in streams:
        _check_planes(emu_device_decoder, tus)


@pytest.mark.emu
@pytest.mark.parametrize("matrix", MATRICES)
@pytest.mark.parametrize("full_range", [False, True])
def test_rgb_matches_reference_formula_emu(emu_device_decoder, matrix, full_range):
    """every matrix x range on 4:2:0 (odd size: the last chroma sample covers one luma column / row) and on 4:2:2"""
    _check_rgb(emu_device_decoder, obu.inter_stream(8, 203, 131, n_frames=3, bpc=10, motion_modes=1, film_grain=1), matrix, full_range)
    import test_stream as TS
    _check_rgb(emu_device_decoder, TS._valid_422("intra", 64, 64, 8, 1)[0], matrix, full_range)


@pytest.mark.emu
def test_rgb_identity_mono_auto_and_12bit_emu(emu_device_decoder):
    """identity matrix (4:4:4: R = V, G = Y, B = U), monochrome (Cb' = Cr' = 0), the sequence header's choice (no colour
    description: BT.709, limited range) and 12-bit clipping"""
    _check_rgb(emu_device_decoder, obu.inter_stream(9, 130, 66, n_frames=2, layout="444", motion_modes=1), "identity", None)
    _check_rgb(emu_device_decoder, obu.inter_stream(10, 131, 67, n_frames=2, bpc=10, layout="400"), "bt601", True)
    _check_rgb(emu_device_decoder, obu.intra_stream(11, 192, 128, n_frames=2, bpc=12, layout="444", film_grain=1), "auto", None)
    _check_rgb(emu_device_decoder, obu.intra_stream(12, 96, 64, n_frames=1, bpc=12), "bt2020", True)
    with pytest.raises(ValueError):
        list(emu_device_decoder.pictures(obu.intra_stream(1, 64, 64), format="rgb", matrix="identity", alloc=_np_alloc))


@pytest.mark.emu
def test_host_decoder_in_the_same_process_keeps_host_pictures_emu(emu_device_decoder):
    """device output is a setting of one decoder context: a HookedDecoder.decode() run while a device-output decode is half
    way through still gets its pictures copied into host memory"""
    tus = obu.inter_stream(13, 256, 192, n_frames=5, bpc=10, film_grain=1, motion_modes=2)
    ref = _ref_pictures(tus)
    r0, _, packed0 = stream.decode_stream(C.CDLL(refs.REF_SO), tus, apply_grain=1)
    host = stream.HookedDecoder(backend=_emu_path(), serialize=True)
    gen = emu_device_decoder.pictures(tus, alloc=_np_alloc)
    first = next(gen)
    emu_device_decoder.stats(reset=True)
    r1, _, packed1 = host.decode(tus, apply_grain=1)
    assert r1 == r0 and np.array_equal(packed0, packed1)
    assert host.stats(reset=True)["d2h_bytes"] > 0
    rest = list(gen)
    for (_, _, _, _, rp), gp in zip(ref, [first] + rest):
        assert all(np.array_equal(_host(a), b) for a, b in zip(gp, rp))


@pytest.mark.emu
def test_more_pictures_than_the_picture_table_emu(emu_device_decoder):
    """72 output pictures (the hooks' table of device pictures has 64 entries), film grain on every other one: entries and
    device buffers are recycled as pictures are released; a decode stopped half way leaves nothing behind"""
    tus = obu.inter_stream(14, 64, 64, n_frames=72, film_grain=1, motion_modes=1)
    _check_planes(emu_device_decoder, tus)
    gen = emu_device_decoder.pictures(tus, alloc=_np_alloc)
    for _ in range(5):
        next(gen)
    gen.close()
    _check_planes(emu_device_decoder, tus[:10])


def test_export_job_layout_matches_the_library():
    assert refs.emu_lib().b200_struct_size(22) == C.sizeof(stream.ExportJob)


def test_rgb_coefficients():
    """the five integers of each matrix: 1.0 = 1 << 14; full-range BT.709 R = Y + 1.5748 Cr"""
    assert stream.rgb_coefficients("bt709", True) == (16384, 25802, 3069, 7670, 30402)
    assert stream.rgb_coefficients("bt601", False)[0] == round(16384 * 255 / 219)


# ---- on the device ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_device_decoder():
    d = stream.DeviceDecoder(n_threads=8, max_frame_delay=4)
    yield d
    d.release()


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(1920, 1080, 8, 1), (3840, 2160, 10, 0)])
def test_device_output_gpu(gpu_device_decoder, case):
    """1080p 8 bit with film grain and 4K 10 bit: planes and RGB in torch CUDA tensors, exported on a non-default stream"""
    import torch
    w, h, bpc, fg = case
    tus = obu.inter_stream(300 + bpc, w, h, n_frames=3, bpc=bpc, log2_cols=2, log2_rows=1, motion_modes=2, film_grain=fg)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _check_planes(gpu_device_decoder, tus, alloc=None)
        for matrix, full in (("auto", None), ("bt2020", True)):
            _check_rgb(gpu_device_decoder, tus, matrix, full, alloc=None)
    # a HookedDecoder in the same process still gets host pictures
    r, _, packed = stream.HookedDecoder().decode(tus, apply_grain=1)
    r0, _, packed0 = stream.decode_stream(C.CDLL(refs.REF_SO), tus, apply_grain=1)
    assert r == r0 == 3 and np.array_equal(packed, packed0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["key_8bit_tiles", "inter_10bit_all_tools", "inter_444_12bit", "gen_422_10bit_all_tools", "gen_sparse_8bit"])
def test_golden_streams_device_output_gpu_md5(name, capsys):
    """the committed streams through `--output-path device`, grain applied: the digest over the exported planes is the one of
    the stock reference's output (needs neither the reference sources nor libdav1d_ref.so)"""
    want = json.load(open(os.path.join(refs.ROOT, "tests", "golden", "stream_golden.json")))[name]
    path = os.path.join(refs.ROOT, "tests", "golden", "stream_%s.obu" % name)
    capsys.readouterr()
    assert cli.main(["-i", path, "--output-path", "device", "--muxer", "md5", "--verify", want["md5"]]) == 0
    assert capsys.readouterr().out.split()[0] == want["md5"]
