"""Host glue for decoding AV1 elementary streams with the B200 back end behind a real dav1d front end.

`oracle/_ref/hooked-<digest>/libdav1d_b200.so` is the unmodified dav1d library whose `f->bd_fn` hooks are the record
emitters of integration/dav1d/ (built by oracle/hooked.mk where the reference sources exist; elsewhere the prebuilt
oracle/_ref/ is used). This module binds its stream driver (dav1d's public API: dav1d_open / dav1d_send_data / dav1d_get_picture)
and points the hooks at dav1d_b200/libb200av1.so. No CPU fallback: without the CUDA library the decode fails."""
import ctypes as C
import os
import queue
import threading

import numpy as np

from ._lib import ColorJitter, ExportJob, TensorJob, ToneMap  # noqa: F401  (the B200 structs DeviceDecoder fills)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hooked_dir():
    """oracle/_ref/hooked-<digest>: the hooked libraries are compiled from this tree's own sources (integration/dav1d/, the C
    ABI header, the recipe), so the directory they are built into is named by a digest of those sources. A library built
    from other sources (an older checkout, a build directory restored from elsewhere, objects make judged up to date by
    their times) is then never loaded in their place: its symbols and struct layouts would not be the ones this module
    binds."""
    import hashlib
    h = hashlib.sha256()
    hk = os.path.join(ROOT, "integration", "dav1d")
    files = [os.path.join(hk, f) for f in sorted(os.listdir(hk))] + [os.path.join(ROOT, "include", "b200av1.h"),
                                                                    os.path.join(ROOT, "oracle", "hooked.mk")]
    for f in files:
        if os.path.isfile(f):
            with open(f, "rb") as fh:
                h.update(os.path.relpath(f, ROOT).encode()); h.update(fh.read())
    return os.path.join(ROOT, "oracle", "_ref", "hooked-" + h.hexdigest()[:16])


HOOKED_DIR = _hooked_dir()
HOOKED_SO = os.path.join(HOOKED_DIR, "libdav1d_b200.so")
LEVEL1_SO = os.path.join(HOOKED_DIR, "libdav1d_b200_l1.so")
# hooked library -> the back end its hooks are bound to: the binding and everything the hooks hold (device pictures, frame
# slots, page-locked pictures) is process-wide state of the library, shared by every HookedDecoder of the process
_bound = {}
FAMILIES = {"itx": 1, "mc": 2, "ipred": 4, "loopfilter": 8, "cdef": 16, "looprestoration": 32, "filmgrain": 64}


class HookStats(C.Structure):
    _fields_ = [("frames", C.c_uint64), ("records", C.c_uint64), ("coefs", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("device_ms", C.c_double), ("intra_tx", C.c_uint64), ("pred", C.c_uint64),
                ("comp", C.c_uint64), ("warp", C.c_uint64), ("blend", C.c_uint64), ("itx", C.c_uint64),
                ("inter_frames", C.c_uint64), ("host_prep_ms", C.c_double), ("interintra", C.c_uint64), ("palette_bytes", C.c_uint64), ("ibc", C.c_uint64), ("scaled", C.c_uint64),
                ("ref_table", C.c_uint64), ("frame_table", C.c_uint64)]


def build_hooked(verbose=False):
    """(Re)build HOOKED_SO (+ the Level-1 variant) where the reference sources exist; otherwise a no-op."""
    import subprocess
    oracle = os.path.join(ROOT, "oracle")
    r = subprocess.run(["make", "-j8", "-C", oracle, "hooked", "OUT=" + os.path.relpath(HOOKED_DIR, oracle)], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("oracle/hooked.mk build failed:\n" + r.stderr[-3000:])
    if verbose:
        print(r.stdout[-500:])
    return HOOKED_SO


def plane_dims(w, h, layout):
    """(width, height) of the planes of a picture; layout = enum Dav1dPixelLayout (0 4:0:0, 1 4:2:0, 2 4:2:2, 3 4:4:4)"""
    if layout == 0:
        return [(w, h)]
    cw = w if layout == 3 else (w + 1) // 2
    ch = (h + 1) // 2 if layout == 1 else h
    return [(w, h), (cw, ch), (cw, ch)]


def decode_stream(dll, tus, n_threads=4, max_frame_delay=2, max_pics=64, apply_grain=0):
    """Decode a list of temporal units with `dll` (a CDLL exporting refdrv_decode_stream: the hooked library or the
    stock checker). Returns (n_pictures or negative dav1d error, info[n][4] = w, h, bpc, layout, packed pictures)."""
    data = b"".join(tus)
    sz = (C.c_uint64 * len(tus))(*[len(t) for t in tus])
    info = np.zeros(4 * max_pics, np.int32)
    # output size is not known before the sequence header is parsed by the decoder: bound it from the stream's own
    # sequence header (max_frame_width / height live in the first OBU_SEQ_HDR) -> the caller passes generous capacity
    cap = int(decode_stream.capacity)
    out = np.empty(cap, np.uint8)
    dll.refdrv_decode_stream.restype = C.c_int
    dll.refdrv_decode_stream.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint64,
                                         C.c_void_p, C.c_int]
    r = dll.refdrv_decode_stream(data, sz, len(tus), n_threads, max_frame_delay, apply_grain, out.ctypes.data, cap,
                                 info.ctypes.data, max_pics)
    n = 0
    for i in range(max(r, 0)):
        w, h, bpc, layout = (int(v) for v in info[4 * i:4 * i + 4])
        n += sum(pw * ph for pw, ph in plane_dims(w, h, layout)) * (2 if bpc > 8 else 1)
    return r, info[:4 * max(r, 0)].reshape(-1, 4).copy(), out[:n]


decode_stream.capacity = 256 << 20


class HookedDecoder:
    """dav1d front end + B200 back end. `backend` = path of the C-ABI library the hooks bind (default: the CUDA
    library); `serialize` = one device job at a time (for back ends that are not re-entrant)."""

    def __init__(self, backend=None, serialize=False):
        if not os.path.exists(HOOKED_SO):
            build_hooked()
            if not os.path.exists(HOOKED_SO):
                raise RuntimeError("%s missing (it is built where the reference sources exist)" % HOOKED_SO)
        if backend is None:
            from . import _lib
            _lib.get_lib()                       # builds / loads the CUDA library or raises
            backend = _lib.get_lib().path
        self.dll = C.CDLL(HOOKED_SO)
        self.backend, self.serialize = backend, serialize
        self._bind()

    def _bind(self):
        """bind the hooks to this decoder's back end unless they already are; what they hold from another back end (another
        decoder of this process) is released through that back end first"""
        if _bound.get(HOOKED_SO) != self.backend:
            if HOOKED_SO in _bound:
                self.dll.b200hook_release()
            if self.dll.b200hook_set_backend(self.backend.encode()) != 0:
                raise RuntimeError("b200hook_set_backend(%s) failed" % self.backend)
            _bound[HOOKED_SO] = self.backend
        self.dll.b200hook_set_serialize(1 if self.serialize else 0)

    def decode(self, tus, **kw):
        self._bind()
        return decode_stream(self.dll, tus, **kw)

    def output_times_ns(self):
        """when each picture of the last decode() came out of dav1d_get_picture: nanoseconds since the call began"""
        buf = (C.c_uint64 * 4096)()
        self.dll.refdrv_output_times_ns.restype = C.c_int
        n = self.dll.refdrv_output_times_ns(buf, 4096)
        return [int(buf[i]) for i in range(n)]

    def stats(self, reset=False):
        s = HookStats()
        self.dll.b200hook_get_stats(C.byref(s), 1 if reset else 0)
        return {k: getattr(s, k) for k, _ in HookStats._fields_}

    def release(self):
        self.dll.b200hook_release()


EXPORT_FORMATS = {"planes": 0, "rgb": 1}
# (Kr, Kb) of the YCbCr matrices the RGB export knows; the sequence header's matrix_coefficients (enum Dav1dMatrixCoefficients)
# -> one of them ("identity": R = V, G = Y, B = U)
MATRICES = {"bt601": (0.299, 0.114), "bt709": (0.2126, 0.0722), "bt2020": (0.2627, 0.0593)}
MTRX_TO_MATRIX = {0: "identity", 1: "bt709", 5: "bt601", 6: "bt601", 9: "bt2020", 10: "bt2020"}


def rgb_coefficients(matrix, full_range):
    """(cy, rv, gu, gv, bu) of the RGB export, 1.0 = 1 << 14: R = cy*Y' + rv*Cr', G = cy*Y' - gu*Cb' - gv*Cr', B = cy*Y' + bu*Cb'.
    Limited range stretches luma by 255/219 and chroma by 255/224 (whatever the bit depth)."""
    kr, kb = MATRICES[matrix]
    kg = 1.0 - kr - kb
    ys, cs = (1.0, 1.0) if full_range else (255.0 / 219.0, 255.0 / 224.0)
    f = [ys, 2 * (1 - kr) * cs, 2 * kb * (1 - kb) / kg * cs, 2 * kr * (1 - kr) / kg * cs, 2 * (1 - kb) * cs]
    return tuple(int(round(v * (1 << 14))) for v in f)


def rgb_reference(planes, bpc, layout, matrix, full_range):
    """numpy statement of the RGB export (include/b200av1.h B200ExportJob) for one picture's planes: [3, h, w] int64"""
    y = planes[0].astype(np.int64)
    h, w = y.shape
    if layout == 0:
        u = v = None
    else:
        ssh, ssv = int(layout != 3), int(layout == 1)
        yi, xi = np.arange(h)[:, None] >> ssv, np.arange(w)[None, :] >> ssh
        u, v = planes[1].astype(np.int64)[yi, xi], planes[2].astype(np.int64)[yi, xi]
    if matrix == "identity":
        return np.stack([v, y, u])
    s, bdmax = bpc - 8, (1 << bpc) - 1
    cy, rv, gu, gv, bu = rgb_coefficients(matrix, full_range)
    yy = cy * (y - (0 if full_range else 16 << s)) + 8192
    cb, cr = (0, 0) if u is None else (u - (128 << s), v - (128 << s))
    return np.clip(np.stack([(yy + rv * cr) >> 14, (yy - gu * cb - gv * cr) >> 14, (yy + bu * cb) >> 14]), 0, bdmax)


TENSOR_DTYPES = {"float32": 0, "float16": 1, "bfloat16": 2}
TENSOR_LAYOUTS = {"chw": 0, "hwc": 1}
# chroma siting of the tensor export -> (horizontal, vertical): 1 = the chroma sample lies midway between two luma samples,
# 0 = on the even one. "left" is the MPEG-2 convention (4:2:0 chroma co-sited with luma horizontally, midway vertically).
SITINGS = {"left": (0, 1), "topleft": (0, 0), "center": (1, 1)}
# the sequence header's chroma_sample_position (enum Dav1dChromaSamplePosition: 0 unknown, 1 vertical, 2 colocated) -> siting
CHR_TO_SITING = {0: "left", 1: "left", 2: "topleft"}


def tensor_scale_bias(bpc, mean=None, std=None, jittered=False):
    """float32 (scale, bias) per channel of the tensor export: out = R * scale + bias with R in 0 .. 4 * bdmax, so that
    out = (R / (4 * bdmax) - mean) / std; mean 0 and std 1 by default (outputs in [0, 1]). jittered=True: the scale of a
    colour-jittered job (B200ColorJitter), whose J is in [0, 1] already: out = (J - mean) / std"""
    bdmax = (1 << bpc) - 1
    mean = [0.0] * 3 if mean is None else [float(v) for v in mean]
    std = [1.0] * 3 if std is None else [float(v) for v in std]
    if len(mean) != 3 or len(std) != 3 or not all(v > 0 for v in std):
        raise ValueError("mean and std need 3 values each, std > 0")
    scale = np.array([1.0 / (s if jittered else 4 * bdmax * s) for s in std], np.float32)
    bias = np.array([-m / s for m, s in zip(mean, std)], np.float32)
    return scale, bias


def tensor_taps(out, inn, n, s=0, k=0):
    """(i0, i1, f) of the tensor export's bilinear sampling along one axis (include/b200av1.h B200TensorJob): `out` output
    samples from a plane of n samples whose luma axis has `inn`, sub-sampled by s, chroma sited by k"""
    x = np.arange(out, dtype=np.int64)
    pos = np.maximum(0, (2 * x + 1) * inn - (1 + k) * out) * (1 << (7 - s)) // out
    i0 = np.minimum(pos >> 8, n - 1)
    return i0, np.minimum(i0 + 1, n - 1), pos & 255


def tensor_weights(out, inn, n, s=0, k=0):
    """[out, n] int64 weights (1/2^14, each row summing to 2^14) of the antialiased tensor export along one axis
    (include/b200av1.h B200TensorJob, antialias = 1); arguments as in tensor_taps. An axis that this plane does not reduce
    (sigma <= 256) gets its bilinear taps as weights; a reduced one the triangle of half-width sigma, clipped at the edges,
    with cumulative rounding."""
    x = np.arange(out, dtype=np.int64)
    P = ((2 * x + 1) * inn - (1 + k) * out) * (1 << (7 - s)) // out
    sigma = inn * (1 << (8 - s)) // out
    W = np.zeros((out, n), np.int64)
    if sigma <= 256:
        i0, i1, f = tensor_taps(out, inn, n, s, k)
        np.add.at(W, (x, i0), (256 - f) * 64)
        np.add.at(W, (x, i1), f * 64)
        return W
    t = np.maximum(sigma - np.abs(256 * np.arange(n, dtype=np.int64)[None, :] - P[:, None]), 0)
    T = t.sum(1, keepdims=True)
    R = (np.cumsum(t, axis=1) * (1 << 15) + T) // (2 * T)
    return np.diff(R, axis=1, prepend=0)


TENSOR_INTERPOLATIONS = {"bilinear": 0, "bicubic": 1}


def _keys(u, a4):
    """4 * 256^3 * K(u / 256) of the Keys cubic with a = a4 / 4 (int64 u >= 0), as include/b200av1.h states it"""
    return np.where(u < 256, (a4 + 8) * u ** 3 - (a4 + 12) * u ** 2 * 256 + 4 * 256 ** 3,
                    np.where(u < 512, a4 * u ** 3 - 5 * a4 * u ** 2 * 256 + 8 * a4 * u * 256 ** 2 - 4 * a4 * 256 ** 3, 0))


def cubic_weights(out, inn, n, s=0, k=0, antialias=False):
    """[out, n] int64 weights (1/2^14, each row summing to 2^14) of the bicubic tensor export along one axis
    (include/b200av1.h B200TensorJob, interpolation = B200_TENSOR_BICUBIC); arguments as in tensor_taps. antialias=False:
    torch's bicubic (a = -3/4), four taps around the unclamped position with the weights of taps beyond the edge added to
    the edge sample; antialias=True: torch's antialiased bicubic (a = -1/2, half-support 2 * max(scale, 1)), taps clipped
    at the edges and the weights renormalised. Both with cumulative rounding."""
    x = np.arange(out, dtype=np.int64)
    P = ((2 * x + 1) * inn - (1 + k) * out) * (1 << (7 - s)) // out
    if antialias:
        sg = max(inn * (1 << (8 - s)) // out, 256)
        u = np.abs(256 * np.arange(n, dtype=np.int64)[None, :] - P[:, None]) * 256 // sg
        t = _keys(u, -2)
        T = t.sum(1, keepdims=True)
        R = (np.cumsum(t, axis=1) * (1 << 15) + T) // (2 * T)
        return np.diff(R, axis=1, prepend=0)
    taps = (P >> 8)[:, None] + np.arange(-1, 3)
    R = (np.cumsum(_keys(np.abs(256 * taps - P[:, None]), -3), axis=1) + (1 << 11)) >> 12
    W = np.zeros((out, n), np.int64)
    np.add.at(W, (np.repeat(x, 4), np.clip(taps, 0, n - 1).ravel()), np.diff(R, axis=1, prepend=0).ravel())
    return W


# ---- HDR to SDR (B200ToneMap, include/b200av1.h): the curves in float64 --------------------------------------------
# the sequence header's transfer_characteristics (enum Dav1dTransferCharacteristics) of the transfers tone_tables knows
TRANSFERS = {"pq": 16, "hlg": 18}
# color_primaries (enum Dav1dColorPrimaries) -> CIE 1931 xy of R, G, B; 2 (unspecified) is taken as BT.2020 for PQ / HLG
PRIMARIES = {1: ((0.640, 0.330), (0.300, 0.600), (0.150, 0.060)),      # BT.709
             9: ((0.708, 0.292), (0.170, 0.797), (0.131, 0.046)),      # BT.2020
             12: ((0.680, 0.320), (0.265, 0.690), (0.150, 0.060))}     # P3-D65 (SMPTE EG 432-1)
PRIMARIES[2] = PRIMARIES[9]
D65 = (0.3127, 0.3290)
SDR_PEAK = 203.0                         # cd/m^2: BT.2408's HDR reference white, where SDR white lands
HDR_PEAK = 1000.0                        # cd/m^2: the source peak without metadata, and HLG's nominal display peak
PQ_M1, PQ_M2 = 2610 / 16384, 2523 / 4096 * 128
PQ_C1, PQ_C2, PQ_C3 = 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32
HLG_A = 0.17883277
HLG_B, HLG_C = 1 - 4 * HLG_A, 0.5 - HLG_A * np.log(4 * HLG_A)
BT709_ALPHA, BT709_BETA = 1.09929682680944, 0.018053968510807


def pq_eotf(e):
    """SMPTE ST 2084: non-linear signal e in [0, 1] -> display light in cd/m^2"""
    p = np.power(np.clip(np.asarray(e, np.float64), 0, 1), 1 / PQ_M2)
    return 10000 * np.power(np.maximum(p - PQ_C1, 0) / (PQ_C2 - PQ_C3 * p), 1 / PQ_M1)


def pq_inverse_eotf(lum):
    """display light in cd/m^2 (0 .. 10000) -> the ST 2084 signal"""
    y = np.power(np.clip(np.asarray(lum, np.float64) / 10000, 0, 1), PQ_M1)
    return np.power((PQ_C1 + PQ_C2 * y) / (1 + PQ_C3 * y), PQ_M2)


def hlg_inverse_oetf(e):
    """BT.2100 HLG: non-linear signal e in [0, 1] -> normalised scene light E in [0, 1]"""
    e = np.clip(np.asarray(e, np.float64), 0, 1)
    return np.where(e <= 0.5, e * e / 3, (np.exp((e - HLG_C) / HLG_A) + HLG_B) / 12)


def hlg_gamma(lw):
    """the HLG system gamma of a display of peak lw cd/m^2 (BT.2100)"""
    return 1.2 + 0.42 * np.log10(lw / 1000.0)


def eetf(lum, peak, sdr_peak):
    """BT.2390 EETF on display light (cd/m^2): the PQ-domain Hermite knee from source peak `peak` to target peak `sdr_peak`,
    black at 0 on both sides. Light above `peak` clips to it; with sdr_peak >= peak nothing is compressed."""
    lum = np.minimum(np.asarray(lum, np.float64), peak)
    if sdr_peak >= peak:
        return lum
    black, white = pq_inverse_eotf(0.0), pq_inverse_eotf(peak)
    e1 = np.clip((pq_inverse_eotf(lum) - black) / (white - black), 0, 1)
    max_lum = (pq_inverse_eotf(sdr_peak) - black) / (white - black)
    ks = 1.5 * max_lum - 0.5
    t = (e1 - ks) / (1 - ks)
    knee = (2 * t ** 3 - 3 * t ** 2 + 1) * ks + (t ** 3 - 2 * t ** 2 + t) * (1 - ks) + (-2 * t ** 3 + 3 * t ** 2) * max_lum
    e2 = np.where(e1 < ks, e1, knee)
    return pq_eotf(e2 * (white - black) + black)


def bt709_oetf(lin):
    """the BT.709 OETF with its exact constants: linear light in [0, 1] -> R', G', B' in [0, 1]"""
    lin = np.clip(np.asarray(lin, np.float64), 0, 1)
    return np.where(lin < BT709_BETA, 4.5 * lin, BT709_ALPHA * np.power(lin, 0.45) - (BT709_ALPHA - 1))


def _rgb_to_xyz(prim):
    xy = np.array(prim, np.float64)
    m = np.stack([xy[:, 0] / xy[:, 1], np.ones(3), (1 - xy[:, 0] - xy[:, 1]) / xy[:, 1]])
    white = np.array([D65[0] / D65[1], 1.0, (1 - D65[0] - D65[1]) / D65[1]])
    return m * np.linalg.solve(m, white)[None, :]


def gamut_matrix(primaries):
    """float64 [3, 3]: linear RGB in the primaries of `primaries` (color_primaries code 1, 2, 9 or 12) -> linear BT.709 RGB,
    both with a D65 white. ValueError for any other code."""
    if primaries not in PRIMARIES:
        raise ValueError("tone mapping knows color_primaries 1 (BT.709), 2 (unspecified: BT.2020), 9 (BT.2020) and 12 "
                         "(P3-D65), not %r" % (primaries,))
    if PRIMARIES[primaries] == PRIMARIES[1]:
        return np.eye(3)
    return np.linalg.solve(_rgb_to_xyz(PRIMARIES[1]), _rgb_to_xyz(PRIMARIES[primaries]))


def tone_light(transfer, e, peak, sdr_peak=SDR_PEAK):
    """float64 statement of the curve table: signal e in [0, 1] -> the EETF's display light over sdr_peak, in [0, 1].
    PQ: the ST 2084 EOTF; HLG: peak * E^gamma per channel on the scene light E (peak = the display's Lw)."""
    if transfer == "pq":
        lum = pq_eotf(e)
    else:
        lum = peak * np.power(hlg_inverse_oetf(e), hlg_gamma(peak))
    return np.clip(eetf(lum, peak, sdr_peak) / sdr_peak, 0, 1)


def tone_tables(transfer, primaries, bpc, peak=None, sdr_peak=SDR_PEAK, bits=16):
    """(curve, m, oetf) of a B200ToneMap (include/b200av1.h), computed in float64 and rounded once to float32: curve
    [4 * bdmax + 1] = tone_light of R / (4 * bdmax), m [3, 3] = gamut_matrix(primaries), oetf [2^bits + 1] =
    4 * bdmax * bt709_oetf(i / 2^bits). transfer: "pq" or "hlg" (or its transfer_characteristics code, 16 or 18); peak: the
    source peak in cd/m^2 (None: 1000); sdr_peak: the light that becomes SDR white."""
    transfer = {v: k for k, v in TRANSFERS.items()}.get(transfer, transfer)
    if transfer not in TRANSFERS:
        raise ValueError("transfer must be 'pq' or 'hlg', not %r" % (transfer,))
    if bpc not in (8, 10, 12) or not 8 <= int(bits) <= 16:
        raise ValueError("bpc must be 8, 10 or 12 and bits 8 .. 16")
    peak = HDR_PEAK if peak is None else float(peak)
    if not (np.isfinite(peak) and peak > 0 and np.isfinite(sdr_peak) and sdr_peak > 0):
        raise ValueError("peak and sdr_peak must be positive (cd/m^2)")
    qmax = 4 * ((1 << bpc) - 1)
    curve = tone_light(transfer, np.arange(qmax + 1) / qmax, peak, float(sdr_peak)).astype(np.float32)
    oetf = (qmax * bt709_oetf(np.arange((1 << bits) + 1) / (1 << bits))).astype(np.float32)
    return curve, gamut_matrix(primaries).astype(np.float32), oetf


def tone_reference(rgb, tone):
    """the tone stage of B200ToneMap (include/b200av1.h) on the matrix's integer R, G, B ([3, ...], 0 .. 4 * bdmax):
    float32 T on the same scale, exactly as the kernel computes it (numpy rounds each float32 operation on its own)"""
    curve, m, oetf = (np.asarray(a, np.float32) for a in tone)
    m = m.reshape(3, 3)
    bits = (len(oetf) - 1).bit_length() - 1
    L = curve[rgb]
    G = [(m[r, 0] * L[0] + m[r, 1] * L[1]) + m[r, 2] * L[2] for r in range(3)]
    return np.stack([oetf[np.rint(np.clip(g, np.float32(0), np.float32(1)) * np.float32(1 << bits)).astype(np.int64)] for g in G])


# ---- colour jitter (B200ColorJitter, include/b200av1.h): torchvision's ColorJitter in float32 ------------------------
JITTER_OPS = ("brightness", "contrast", "saturation", "hue")     # torchvision's numbering of fn_idx


def _is_jitter(j):
    """whether j has the shape of what torchvision.transforms.ColorJitter.get_params returns: (fn_idx, b, c, s, h)"""
    if not isinstance(j, (tuple, list)) or len(j) != 5:
        return False
    try:
        return len(j[0]) == 4
    except TypeError:
        return False


def jitter_factors(jitter):
    """(order, enabled, b, c, s, hue, c1, s1) of B200ColorJitter for jitter = (fn_idx, b, c, s, h), the tuple
    torchvision.transforms.ColorJitter.get_params returns (None: that op is off). The factors are float32, c1 and s1 are
    f32(1.0 - factor) with the difference taken in float64, as torchvision's _blend does; a disabled op gets a neutral
    factor. ValueError for a fn_idx that is not a permutation of 0 .. 3, a factor that is not a finite number, a negative
    brightness, contrast or saturation, or a hue outside [-0.5, 0.5]."""
    if not _is_jitter(jitter):
        raise ValueError("jitter must be None or (fn_idx, brightness, contrast, saturation, hue) as ColorJitter.get_params "
                         "returns it, not %r" % (jitter,))
    try:
        order = [int(v) for v in jitter[0]]
    except (TypeError, ValueError):
        order = None
    if order is None or sorted(order) != [0, 1, 2, 3]:
        raise ValueError("jitter fn_idx must be a permutation of 0 .. 3, not %r" % (jitter[0],))
    enabled, f = 0, []
    for op, v in enumerate(jitter[1:]):
        if v is None:
            f.append(0.0 if op == 3 else 1.0)
            continue
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(v):
            raise ValueError("jitter %s factor must be a finite number, not %r" % (JITTER_OPS[op], v))
        v = float(v)
        if (op < 3 and v < 0) or (op == 3 and not -0.5 <= v <= 0.5):
            raise ValueError("jitter %s factor %r is out of range (%s)" % (JITTER_OPS[op], v, ">= 0" if op < 3 else "-0.5 .. 0.5"))
        enabled |= 1 << op
        f.append(v)
    b, c, s, h = f
    c1, s1 = (1.0 - c if enabled & 2 else 0.0), (1.0 - s if enabled & 4 else 0.0)
    return (order, enabled) + tuple(np.float32(v) for v in (b, c, s, h, c1, s1))


def color_jitter(jitter, grayscale=False, acc=None):
    """the B200ColorJitter of jitter (jitter_factors; None: no op) and grayscale, its contrast scratch at address acc"""
    if not _is_flag(grayscale):
        raise ValueError("grayscale must be a bool, not %r" % (grayscale,))
    order, enabled, b, c, s, h, c1, s1 = jitter_factors(jitter) if jitter is not None else ([0, 1, 2, 3], 0) + (1, 1, 1, 0, 0, 0)
    t = ColorJitter()
    t.brightness, t.contrast, t.saturation, t.hue, t.contrast1, t.saturation1 = (float(v) for v in (b, c, s, h, c1, s1))
    t.order[:] = order
    t.enabled, t.grayscale, t.acc = enabled, int(grayscale), acc
    return t


# float32 operations as the export kernels compute them under -ftz: a subnormal operand or result is a zero of its sign
_TINY = np.float32(2.0 ** -126)


def _ftz(a):
    a = np.asarray(a, np.float32)
    return np.where(np.abs(a) < _TINY, np.copysign(np.float32(0), a), a).astype(np.float32)


def _fmul(a, b):
    return _ftz(_ftz(a) * _ftz(b))


def _fadd(a, b):
    return _ftz(_ftz(a) + _ftz(b))


def _fsub(a, b):
    return _ftz(_ftz(a) - _ftz(b))


def _fdiv(a, b):
    return _ftz(_ftz(a) / _ftz(b))


def _unit_clip(a):
    return np.minimum(np.maximum(a, np.float32(0)), np.float32(1))


def jitter_gray(x):
    """torchvision's rgb_to_grayscale of x [3, ...] in float32: ((0.2989 r + 0.587 g) + 0.114 b)"""
    f = np.float32
    return _fadd(_fadd(_fmul(f(0.2989), x[0]), _fmul(f(0.587), x[1])), _fmul(f(0.114), x[2]))


def _jitter_hue(x, hue):
    """torchvision's adjust_hue on x [3, ...]: _rgb2hsv, remainder(h + hue, 1), _hsv2rgb"""
    f = np.float32
    r, g, b = x
    maxc, minc = np.maximum(np.maximum(r, g), b), np.minimum(np.minimum(r, g), b)
    eqc = maxc == minc
    cr = _fsub(maxc, minc)
    s = _fdiv(cr, np.where(eqc, f(1), maxc))
    d = np.where(eqc, f(1), cr)
    rc, gc, bc = (_fdiv(_fsub(maxc, c), d) for c in (r, g, b))
    h = np.where(maxc == r, _fsub(bc, gc), np.where(maxc == g, _fsub(_fadd(f(2), rc), bc), _fsub(_fadd(f(4), gc), rc)))
    h = np.fmod(_fadd(_fdiv(h, f(6)), f(1)), f(1))
    h = np.fmod(_fadd(h, hue), f(1))
    h = np.where(h < 0, _fadd(h, f(1)), h)
    h6 = _fmul(h, f(6))
    fi = np.floor(h6)
    fr = _fsub(h6, fi)
    p = _unit_clip(_fmul(maxc, _fsub(f(1), s)))
    q = _unit_clip(_fmul(maxc, _fsub(f(1), _fmul(s, fr))))
    t = _unit_clip(_fmul(maxc, _fsub(f(1), _fmul(s, _fsub(f(1), fr)))))
    i = fi.astype(np.int64) % 6
    return np.stack([np.choose(i, [maxc, q, p, p, t, maxc]), np.choose(i, [t, maxc, maxc, q, p, p]),
                     np.choose(i, [p, p, t, maxc, maxc, q])]).astype(np.float32)


def contrast_mean(gray):
    """M of B200ColorJitter: the mean of gray over the picture, f32(f64(S) / (f64(n) * 2^24)) with the exact
    S = sum of rint(gray * 2^24)"""
    total = int(np.rint(_fmul(gray, np.float32(1 << 24))).astype(np.int64).sum())
    return np.float32(float(total) / (float(gray.size) * float(1 << 24)))


def jitter_reference(x, jitter, grayscale=False):
    """numpy statement of the colour jitter stage (include/b200av1.h B200ColorJitter) on one picture x = float32
    [3, H, W] in [0, 1]: the enabled ops of jitter = (fn_idx, b, c, s, h) (ColorJitter.get_params; None: none) in the
    order fn_idx gives, contrast against the picture's mean gray M (contrast_mean), then with grayscale the gray on all
    three channels. Each float32 operation is rounded on its own and flushed like the kernels'."""
    x = _ftz(x).copy()
    if jitter is not None:
        order, enabled, b, c, s, h, c1, s1 = jitter_factors(jitter)
        for op in order:
            if not (enabled >> op) & 1:
                continue
            if op == 0:
                x = _unit_clip(_fmul(b, x))
            elif op == 1:
                x = _unit_clip(_fadd(_fmul(c, x), _fmul(c1, contrast_mean(jitter_gray(x)))))
            elif op == 2:
                x = _unit_clip(_fadd(_fmul(s, x), _fmul(s1, jitter_gray(x))))
            else:
                x = _jitter_hue(x, h)
    if grayscale:
        x = np.broadcast_to(jitter_gray(x), x.shape).astype(np.float32)
    return x


def tensor_antialiased(w, h, size, antialias):
    """whether an export of a w x h picture to size = (OH, OW) takes the antialiased definition: antialias and a luma axis
    reduced (sigma > 256)"""
    oh, ow = size
    return bool(antialias) and (w * 256 // ow > 256 or h * 256 // oh > 256)


def tensor_reference(planes, bpc, layout, size=None, matrix="bt709", full_range=False, siting="left", mean=None, std=None,
                     antialias=False, interpolation="bilinear", tone=None, jitter=None, grayscale=False):
    """numpy statement of the tensor export (include/b200av1.h B200TensorJob) for one picture's planes (layout = enum
    Dav1dPixelLayout): float32 [3, OH, OW] of R, G, B; size = (OH, OW), by default the picture's. antialias=True: the
    antialiased definition (triangle filter on reduced axes), which leaves exports without a reduced luma axis unchanged.
    interpolation="bicubic": the bicubic definition instead, plain or (antialias=True) antialiased on every axis.
    tone=(curve, m, oetf), e.g. tone_tables(...): the HDR to SDR stage of B200ToneMap between the matrix and the output.
    jitter=(fn_idx, b, c, s, h) (ColorJitter.get_params) and / or grayscale=True: the colour jitter stage of
    B200ColorJitter after it (jitter_reference), with its output rule."""
    h, w = planes[0].shape
    oh, ow = size or (h, w)
    ssh, ssv = int(layout in (1, 2)), int(layout == 1)
    kx, ky = SITINGS[siting]
    s, bdmax = bpc - 8, (1 << bpc) - 1
    _check_interpolation(interpolation)
    aa = tensor_antialiased(w, h, (oh, ow), antialias)

    def sample(p, sh, sv, kx, ky):
        p = p.astype(np.int64)
        if interpolation == "bicubic":
            wx = cubic_weights(ow, w, p.shape[1], sh, kx if sh else 0, antialias)
            wy = cubic_weights(oh, h, p.shape[0], sv, ky if sv else 0, antialias)
            # exact in float64, as below: every partial sum is an integer below 2^31
            hq = np.clip((np.rint(p.astype(np.float64) @ wx.T.astype(np.float64)).astype(np.int64) + (1 << 9)) >> 10, 0, 16 * bdmax)
            return np.clip((np.rint(wy.astype(np.float64) @ hq.astype(np.float64)).astype(np.int64) + (1 << 15)) >> 16, 0, 4 * bdmax)
        if aa:
            wx = tensor_weights(ow, w, p.shape[1], sh, kx if sh else 0)
            wy = tensor_weights(oh, h, p.shape[0], sv, ky if sv else 0)
            # float64 products are exact here (every partial sum is an integer below 2^31) and take the BLAS path
            hq = (np.rint(p.astype(np.float64) @ wx.T.astype(np.float64)).astype(np.int64) + (1 << 8)) >> 9
            return (np.rint(wy.astype(np.float64) @ hq.astype(np.float64)).astype(np.int64) + (1 << 16)) >> 17
        x0, x1, fx = tensor_taps(ow, w, p.shape[1], sh, kx if sh else 0)
        y0, y1, fy = tensor_taps(oh, h, p.shape[0], sv, ky if sv else 0)
        a = p[np.ix_(y0, x0)] * (256 - fx) + p[np.ix_(y0, x1)] * fx
        b = p[np.ix_(y1, x0)] * (256 - fx) + p[np.ix_(y1, x1)] * fx
        return (a * (256 - fy)[:, None] + b * fy[:, None] + (1 << 13)) >> 14

    y = sample(planes[0], 0, 0, 0, 0)
    u, v = (None, None) if layout == 0 else (sample(planes[1], ssh, ssv, kx, ky), sample(planes[2], ssh, ssv, kx, ky))
    if matrix == "identity":
        rgb = np.stack([v, y, u])
    else:
        cy, rv, gu, gv, bu = rgb_coefficients(matrix, full_range)
        yy = cy * (y - (0 if full_range else 64 << s)) + 8192
        cb, cr = (0, 0) if u is None else (u - (512 << s), v - (512 << s))
        rgb = np.clip(np.stack([(yy + rv * cr) >> 14, (yy - gu * cb - gv * cr) >> 14, (yy + bu * cb) >> 14]), 0, 4 * bdmax)
    t = rgb.astype(np.float32) if tone is None else tone_reference(rgb, tone)
    if jitter is None and not grayscale:
        scale, bias = tensor_scale_bias(bpc, mean, std)
        return t * scale[:, None, None] + bias[:, None, None]
    scale, bias = tensor_scale_bias(bpc, mean, std, jittered=True)
    x = jitter_reference(_fmul(t, np.float32(1) / np.float32(4 * bdmax)), jitter, grayscale)
    return _fadd(_fmul(x, scale[:, None, None]), bias[:, None, None])


def crop_planes(planes, layout, box):
    """the planes of the box (top, left, height, width) of a picture (layout = enum Dav1dPixelLayout), the source a cropped
    tensor export reads (include/b200av1.h B200TensorJob): luma [top, top + height) x [left, left + width), chroma the
    samples from top >> ssv, left >> ssh that cover it"""
    top, left, height, width = box
    ssh, ssv = int(layout in (1, 2)), int(layout == 1)
    return [planes[0][top:top + height, left:left + width]] + \
        [p[top >> ssv:(top + height + ssv) >> ssv, left >> ssh:(left + width + ssh) >> ssh] for p in planes[1:]]


def align_crop(box, w, h, layout):
    """the box (top, left, height, width) of a w x h picture that the tensor export takes for `box`: on a chroma-subsampled
    axis (layout = enum Dav1dPixelLayout) an odd top / left is moved up / left by one sample and the height / width grown
    by one, so that the bottom / right edge stays put and the box's chroma keeps the picture's siting. ValueError when box
    is not 4 integers with height, width >= 1 inside the picture."""
    if not _is_box(box):
        raise ValueError("a crop box is 4 integers (top, left, height, width), not %r" % (box,))
    top, left, height, width = (int(v) for v in box)
    if top < 0 or left < 0 or height < 1 or width < 1 or top + height > h or left + width > w:
        raise ValueError("crop box (top %d, left %d, height %d, width %d) is not inside the %dx%d picture" % (top, left, height, width, w, h))
    ssh, ssv = int(layout in (1, 2)), int(layout == 1)
    dt, dl = top & ssv, left & ssh
    return top - dt, left - dl, height + dt, width + dl


def _is_box(b):
    return isinstance(b, (tuple, list, np.ndarray)) and len(b) == 4 and all(isinstance(v, (int, np.integer)) for v in b)


def _is_flag(f):
    return isinstance(f, (bool, np.bool_))


def _check_interpolation(interpolation):
    if not isinstance(interpolation, str) or interpolation not in TENSOR_INTERPOLATIONS:
        raise ValueError("interpolation must be 'bilinear' or 'bicubic', not %r" % (interpolation,))


class DeviceDecoder:
    """dav1d front end + B200 back end whose output pictures never leave the device: each one is exported by one kernel from
    its HBM copy into memory the caller allocates, and released at once.

        dec = DeviceDecoder()
        for y, u, v in dec.pictures(tus):                      # torch.uint8 (8 bit) / torch.int16 (10, 12 bit) CUDA tensors
            ...
        for rgb in dec.pictures(tus, format="rgb"):             # [3, h, w], same dtype rule, stream bit depth
        for x in dec.tensors(tus, size=(224, 224), dtype="bfloat16", batch=8):   # [n, 3, 224, 224] model input
        x = dec.clips([tus_0, tus_1, ...], frames=16, step=2, size=(224, 224))  # [N, 16, 3, 224, 224] clip batch

    `backend` = path of the C-ABI library the hooks bind (default: the CUDA library); `serialize` = one device job at a time
    (for back ends that are not re-entrant, like the host emulator)."""

    def __init__(self, backend=None, n_threads=4, max_frame_delay=2, apply_grain=1, serialize=False):
        self._hooked = HookedDecoder(backend=backend, serialize=serialize)
        self.dll = self._hooked.dll
        self.n_threads, self.max_frame_delay, self.apply_grain = n_threads, max_frame_delay, apply_grain
        d = self.dll
        d.refdrv_stream_open.restype = C.c_void_p
        d.refdrv_stream_open.argtypes = [C.c_int, C.c_int, C.c_int]
        for fn in ("refdrv_stream_context", "refdrv_stream_picture"):
            getattr(d, fn).restype = C.c_void_p
            getattr(d, fn).argtypes = [C.c_void_p]
        d.refdrv_stream_send.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
        d.refdrv_stream_get.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        d.refdrv_stream_release.argtypes = [C.c_void_p]
        d.refdrv_stream_close.argtypes = [C.c_void_p]
        d.b200hook_set_device_only.argtypes = [C.c_void_p, C.c_int]
        d.b200hook_export_picture.argtypes = [C.c_void_p, C.POINTER(ExportJob), C.c_void_p]
        d.b200hook_export_tensor.argtypes = [C.c_void_p, C.POINTER(TensorJob), C.c_void_p, C.c_void_p]
        d.b200hook_export_tensor_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        d.refdrv_stream_chroma_position.argtypes = [C.c_void_p]
        d.refdrv_stream_color.argtypes = [C.c_void_p, C.c_void_p]
        d.b200hook_export_tensor_tone_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        d.b200hook_export_tensor_jitter_batch.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
        self._tones = {}                         # (transfer, primaries, bpc, peak, sdr_peak, device) -> (ToneMap, tables)
        self._accs = {}                          # (device, stream) -> the contrast scratch of jittered exports, grown

    def stats(self, reset=False):
        return self._hooked.stats(reset)

    def release(self):
        self._drop_tables()
        self._hooked.release()

    def pictures(self, tus, format="planes", matrix="auto", full_range=None, alloc=None, stream=None):
        """Decodes the temporal units `tus` and yields one item per output picture: a tuple of planes (Y, U, V; Y alone for
        4:0:0) for format="planes", a [3, h, w] array of R, G, B for format="rgb".
        matrix: "auto" (the sequence header's matrix_coefficients; BT.709 when unspecified), "bt601", "bt709", "bt2020" or
        "identity" (4:4:4 only); full_range: None = the sequence header's color_range.
        alloc(shape, dtype) returns the destination (dtype "uint8" at 8 bit, "int16" above, holding the sample values): by
        default torch.empty(..., device="cuda") on the current device. The export runs on `stream` (a torch.cuda.Stream or a
        cudaStream_t handle), by default torch.cuda.current_stream() with the default alloc and the legacy default stream
        otherwise."""
        if format not in EXPORT_FORMATS:
            raise ValueError("format must be 'planes' or 'rgb'")
        if matrix != "auto" and matrix != "identity" and matrix not in MATRICES:
            raise ValueError("unknown matrix %r" % (matrix,))
        alloc, stream = _default_alloc(alloc, stream)
        yield from self._decode(tus, lambda h, info: self._export(h, info, format, matrix, full_range, alloc, stream))

    def tensors(self, tus, size=None, dtype="float32", layout="chw", mean=None, std=None, matrix="auto", full_range=None,
                chroma_siting="auto", batch=None, alloc=None, stream=None, antialias=False, crop=None, flip=False,
                interpolation="bilinear", tonemap=None, peak=None, sdr_peak=SDR_PEAK, jitter=None, grayscale=False):
        """Decodes the temporal units `tus` and yields every output picture as a model input: R, G, B resized to
        size = (height, width) (default: the picture's own) by bilinear sampling at half-sample centres, like
        torch.nn.functional.interpolate(mode="bilinear", align_corners=False) (chroma upsampling is part of the same
        sampling), then (x - mean) / std with x in [0, 1], as a [3, OH, OW] (layout="chw") or [OH, OW, 3] ("hwc") tensor of
        dtype "float32", "float16" or "bfloat16". One kernel per picture (include/b200av1.h, B200TensorJob).
        antialias=True filters reduced axes with a triangle as wide as the reduction, like interpolate(mode="bilinear",
        antialias=True) and torchvision's Resize: what vision models are trained on. It changes nothing when no luma axis
        is reduced.
        interpolation="bicubic" resamples with a Keys cubic instead, chroma upsampling included: like
        interpolate(mode="bicubic", align_corners=False) (edge samples replicated), or with antialias=True like
        interpolate(mode="bicubic", antialias=True), torchvision's Resize(BICUBIC) and PIL's BICUBIC, which filter every
        axis, enlarged ones too. CLIP, SigLIP and most timm models are trained on the antialiased one.
        batch=N: yields [n, ...] tensors of up to N pictures, each picture exported straight into its slot; a picture of
        another size (size=None with frame-size changes) closes the batch early.
        matrix and full_range: as in pictures(). chroma_siting: "auto" (the sequence header's chroma_sample_position:
        colocated -> "topleft", vertical or unknown -> "left", the MPEG-2 convention), "left", "topleft" or "center".
        alloc(shape, dtype) receives "float32", "float16" or "bfloat16"; alloc and stream otherwise mean what they mean in
        pictures().
        crop: a box (top, left, height, width) in luma samples of the picture, or a callable (k, height, width) -> box for
        output picture k of that size: the export reads the box alone as its picture, taps stopping at its edge
        (torchvision's resized_crop; RandomResizedCrop with a random box). On a chroma-subsampled axis an odd top / left
        is rounded down and the box grown to keep its bottom / right edge (align_crop). size=None exports the box at that
        (aligned) size. flip: True, or a callable k -> bool, mirrors the output horizontally after resizing
        (torchvision's hflip). ValueError, naming the picture, for a box outside the picture.
        tonemap: None (the default) exports every stream as it is coded. "auto" tone-maps streams whose sequence header says
        PQ (transfer_characteristics 16) or HLG (18) to SDR BT.709 (include/b200av1.h B200ToneMap; tone_tables states the
        curves) and exports every other stream exactly as None does; "pq" or "hlg" force that transfer, for streams without
        a colour description. peak: the source peak in cd/m^2, by default MaxCLL, else the mastering display's maximum
        luminance, else 1000 (HLG: 1000); sdr_peak: the light that becomes SDR white (203 cd/m^2, BT.2408). The colour
        primaries come from the header (unspecified: BT.2020). The tone map applies to the resized signal.
        jitter: None (the default), the tuple (fn_idx, brightness, contrast, saturation, hue) that
        torchvision.transforms.ColorJitter.get_params returns (None entries: those ops off), or a callable k -> tuple or
        None for output picture k (RandomApply(ColorJitter, p) returns None with probability 1 - p): torchvision's colour
        jitter, in the order fn_idx gives, on the resized (and tone-mapped) picture in [0, 1], contrast against that
        picture's own mean gray (include/b200av1.h B200ColorJitter; jitter_reference states it). grayscale: a bool, or a
        callable k -> bool: the gray of the jittered picture on all three channels (RandomGrayscale). mean / std apply
        after both. ValueError, naming the picture, for a malformed tuple or an out-of-range factor."""
        if dtype not in TENSOR_DTYPES or layout not in TENSOR_LAYOUTS:
            raise ValueError("dtype must be one of %s, layout 'chw' or 'hwc'" % ", ".join(TENSOR_DTYPES))
        if matrix != "auto" and matrix != "identity" and matrix not in MATRICES:
            raise ValueError("unknown matrix %r" % (matrix,))
        if chroma_siting != "auto" and chroma_siting not in SITINGS:
            raise ValueError("unknown chroma siting %r" % (chroma_siting,))
        if size is not None:
            size = tuple(int(v) for v in size)
            if len(size) != 2 or not all(1 <= v <= 65536 for v in size):
                raise ValueError("size must be (height, width), each 1 .. 65536")
        if batch is not None and int(batch) < 1:
            raise ValueError("batch must be >= 1")
        if crop is not None and not callable(crop) and not _is_box(crop):
            raise ValueError("crop must be None, a box (top, left, height, width) or a callable")
        if not callable(flip) and not _is_flag(flip):
            raise ValueError("flip must be a bool or a callable")
        _check_interpolation(interpolation)
        _check_tonemap(tonemap, peak, sdr_peak)
        if jitter is not None and not callable(jitter):
            jitter_factors(jitter)
        if not callable(grayscale) and not _is_flag(grayscale):
            raise ValueError("grayscale must be a bool or a callable")
        tensor_scale_bias(8, mean, std)                          # checks mean / std
        alloc, stream = _default_alloc(alloc, stream)
        esize = 4 if dtype == "float32" else 2
        state = {"buf": None, "n": 0, "shape": None, "k": 0}
        tone_kw = dict(tonemap=tonemap, peak=peak, sdr_peak=sdr_peak)

        def export(h, info):
            k = state["k"]
            state["k"] += 1
            box = _picture_box(crop(k, int(info[1]), int(info[0])) if callable(crop) else crop, info, "picture %d" % k)
            fl = flip(k) if callable(flip) else flip
            if not _is_flag(fl):
                raise ValueError("picture %d: flip must be a bool, not %r" % (k, fl))
            jit = _picture_jitter(jitter(k) if callable(jitter) else jitter, grayscale(k) if callable(grayscale) else grayscale,
                                  "picture %d" % k)
            oh, ow = size or ((box[2], box[3]) if box else (int(info[1]), int(info[0])))
            shape = (3, oh, ow) if layout == "chw" else (oh, ow, 3)
            if batch is None:
                out = alloc(shape, dtype)
                self._export_tensor(h, info, _data_ptr(out), oh, ow, dtype, layout, mean, std, matrix, full_range, chroma_siting,
                                    antialias, stream, box, fl, interpolation, self._tone(h, info, out, **tone_kw),
                                    self._jitter(jit, out, stream))
                return [out]
            done = []
            if state["buf"] is not None and state["shape"] != shape:       # another size closes the batch
                done.append(state["buf"][:state["n"]])
                state["buf"] = None
            if state["buf"] is None:
                state.update(buf=alloc((int(batch),) + shape, dtype), n=0, shape=shape)
            dst = _data_ptr(state["buf"]) + state["n"] * 3 * oh * ow * esize
            self._export_tensor(h, info, dst, oh, ow, dtype, layout, mean, std, matrix, full_range, chroma_siting, antialias, stream,
                                box, fl, interpolation, self._tone(h, info, state["buf"], **tone_kw),
                                self._jitter(jit, state["buf"], stream))
            state["n"] += 1
            if state["n"] == batch:
                done.append(state["buf"])
                state["buf"] = None
            return done

        for outs in self._decode(tus, export):
            yield from outs
        if state["buf"] is not None:
            yield state["buf"][:state["n"]]

    def clips(self, streams, frames, step=1, start=0, size=None, dtype="float32", layout="chw", mean=None, std=None,
              matrix="auto", full_range=None, chroma_siting="auto", workers=None, alloc=None, stream=None, antialias=False,
              crop=None, flip=False, interpolation="bilinear", tonemap=None, peak=None, sdr_peak=SDR_PEAK, jitter=None,
              grayscale=False):
        """Decodes N streams (each a list of temporal units) concurrently and returns one clip per stream as a
        [N, frames, 3, OH, OW] tensor (layout="hwc": [N, frames, OH, OW, 3]): x[i, t] is output picture
        start_i + t * step of stream i, exported exactly as tensors() exports it. `start` is one int or one per stream.
        size=None needs every sampled picture to have the same size. The tensor options (antialias and interpolation included), alloc and
        stream mean what they mean in tensors(); "auto" matrix, range and siting are resolved per stream from its own headers.
        crop: one box (top, left, height, width) for every stream, one box per stream, or a callable (i, height, width) -> box
        called once per stream i on its first sampled picture; flip: one bool, or one per stream. Every picture of a clip
        takes its stream's box and flip (tensors() says what they do), so a clip stays consistent in time. tonemap, peak and
        sdr_peak: as in tensors(), resolved per stream from its own headers and metadata ("auto" converts the PQ and HLG
        streams of a batch and exports the others as they are, in the same batched launches). jitter: one tuple (as
        tensors() takes it) for every stream, one tuple or None per stream, or a callable i -> tuple or None called once per
        stream; grayscale: one bool, or one per stream. Every picture of a clip takes its stream's jitter and grayscale, as
        it takes its box and flip, and contrast uses each picture's own mean gray, as torchvision's ColorJitter does on a
        [T, 3, H, W] clip.
        Each stream has a dav1d context of its own (this decoder's n_threads / max_frame_delay) driven by a host thread of
        its own; at most `workers` streams are open at once (default min(N, CLIP_WORKERS), at most CLIP_MAX_WORKERS).
        Pictures that are not sampled are released unexported, and a stream is closed once its last sampled picture is
        exported. The calling thread exports every sampled picture that is waiting with one batched kernel launch
        (b200_export_tensor_batch) straight into its slot of the result. ValueError when a stream has too few pictures (it
        names the stream); a dav1d error in any stream stops the others and is raised here; no thread outlives the call."""
        streams = list(streams)
        n = len(streams)
        frames, step = int(frames), int(step)
        starts = [int(start)] * n if isinstance(start, (int, np.integer)) else [int(v) for v in start]
        workers = min(n, CLIP_WORKERS) if workers is None else int(workers)
        if n < 1 or frames < 1 or step < 1 or len(starts) != n or min(starts) < 0:
            raise ValueError("clips needs >= 1 stream, frames >= 1, step >= 1 and one start >= 0 per stream")
        if not 1 <= workers <= CLIP_MAX_WORKERS:
            raise ValueError("workers must be 1 .. %d" % CLIP_MAX_WORKERS)
        if dtype not in TENSOR_DTYPES or layout not in TENSOR_LAYOUTS:
            raise ValueError("dtype must be one of %s, layout 'chw' or 'hwc'" % ", ".join(TENSOR_DTYPES))
        if matrix != "auto" and matrix != "identity" and matrix not in MATRICES:
            raise ValueError("unknown matrix %r" % (matrix,))
        if chroma_siting != "auto" and chroma_siting not in SITINGS:
            raise ValueError("unknown chroma siting %r" % (chroma_siting,))
        if size is not None:
            size = tuple(int(v) for v in size)
            if len(size) != 2 or not all(1 <= v <= 65536 for v in size):
                raise ValueError("size must be (height, width), each 1 .. 65536")
        if crop is None or callable(crop) or _is_box(crop):
            crops = [crop] * n
        elif isinstance(crop, (list, tuple)) and len(crop) == n and all(_is_box(b) for b in crop):
            crops = list(crop)
        else:
            raise ValueError("crop must be None, a box (top, left, height, width), one box per stream or a callable")
        if _is_flag(flip):
            flips = [bool(flip)] * n
        elif isinstance(flip, (list, tuple, np.ndarray)) and len(flip) == n and all(_is_flag(f) for f in flip):
            flips = [bool(f) for f in flip]
        else:
            raise ValueError("flip must be a bool or one bool per stream")
        if jitter is None or callable(jitter) or _is_jitter(jitter):
            jits = [jitter] * n
        elif isinstance(jitter, (list, tuple)) and len(jitter) == n and all(j is None or _is_jitter(j) for j in jitter):
            jits = list(jitter)
        else:
            raise ValueError("jitter must be None, a ColorJitter.get_params tuple, one tuple or None per stream or a callable")
        if _is_flag(grayscale):
            grays = [bool(grayscale)] * n
        elif isinstance(grayscale, (list, tuple, np.ndarray)) and len(grayscale) == n and all(_is_flag(g) for g in grayscale):
            grays = [bool(g) for g in grayscale]
        else:
            raise ValueError("grayscale must be a bool or one bool per stream")
        for i in range(n):
            if not callable(jits[i]):
                jits[i] = _picture_jitter(jits[i], grays[i], "stream %d" % i)
        _check_interpolation(interpolation)
        _check_tonemap(tonemap, peak, sdr_peak)
        tensor_scale_bias(8, mean, std)                          # checks mean / std
        alloc, stream = _default_alloc(alloc, stream)
        self._hooked._bind()
        esize = 4 if dtype == "float32" else 2
        todo = queue.Queue()                     # stream indices not started yet
        for i in range(n):
            todo.put(i)
        ready = queue.Queue()                    # (stream, t, handle, info, event) of a held sampled picture, or an error
        stop = threading.Event()
        threads = [threading.Thread(target=self._clip_worker, args=(streams, starts, frames, step, todo, ready, stop), daemon=True)
                   for _ in range(workers)]
        out, hw, left = None, None, n * frames
        try:
            for t in threads:
                t.start()
            while left:
                items = [ready.get()]
                while True:
                    try:
                        items.append(ready.get_nowait())
                    except queue.Empty:
                        break
                try:
                    errors = [it for it in items if isinstance(it, BaseException)]
                    if errors:
                        raise errors[0]
                    jobs = (TensorJob * len(items))()
                    pics = (C.c_void_p * len(items))()
                    boxes = (C.c_int32 * (4 * len(items)))() if crop is not None else None
                    tones = (C.POINTER(ToneMap) * len(items))()
                    jitters = (C.POINTER(ColorJitter) * len(items))()
                    keep = []
                    for k, (i, t, h, info, _) in enumerate(items):
                        if callable(crops[i]):                  # the stream's box, from its first sampled picture
                            crops[i] = crops[i](i, int(info[1]), int(info[0]))
                        if callable(jits[i]):                   # the stream's jitter, asked for once
                            jits[i] = _picture_jitter(jits[i](i), grays[i], "stream %d" % i)
                        box = _picture_box(crops[i], info, "stream %d picture %d" % (i, starts[i] + t * step))
                        if box:
                            boxes[4 * k:4 * k + 4] = box
                        oh, ow = size or ((box[2], box[3]) if box else (int(info[1]), int(info[0])))
                        if out is None:
                            hw = (oh, ow)
                            out = alloc((n, frames) + ((3, oh, ow) if layout == "chw" else (oh, ow, 3)), dtype)
                        elif (oh, ow) != hw:
                            raise ValueError("stream %d picture %d is %dx%d, not %dx%d like the others: pass size= for "
                                             "pictures of different sizes" % (i, starts[i] + t * step, ow, oh, hw[1], hw[0]))
                        dst = _data_ptr(out) + (i * frames + t) * 3 * oh * ow * esize
                        jobs[k] = self._tensor_job(h, info, dst, oh, ow, dtype, layout, mean, std, matrix, full_range, chroma_siting,
                                                   antialias, flips[i], interpolation, jits[i] is not None)
                        pics[k] = self.dll.refdrv_stream_picture(h)
                        tm = self._tone(h, info, out, tonemap, peak, sdr_peak)
                        if tm is not None:
                            tones[k] = C.pointer(tm)
                        if jits[i] is not None:
                            keep.append(color_jitter(*jits[i], acc=self._acc(out, stream, len(items)) + 8 * k))
                            jitters[k] = C.pointer(keep[-1])
                    if self.dll.b200hook_export_tensor_jitter_batch(pics, jobs, boxes, tones if any(tones) else None,
                                                                    jitters if any(jitters) else None, len(items),
                                                                    C.c_void_p(stream)) != 0:
                        raise RuntimeError("exporting pictures failed (see stderr)")
                    left -= len(items)
                finally:
                    for it in items:                 # the pictures go back to their workers: enqueued, or abandoned
                        if not isinstance(it, BaseException):
                            it[4].set()
        finally:
            stop.set()
            while any(t.is_alive() for t in threads):
                try:                                 # workers blocked on a handed-over picture are let go
                    it = ready.get(timeout=0.01)
                    if not isinstance(it, BaseException):
                        it[4].set()
                except queue.Empty:
                    pass
            for t in threads:
                t.join()
        return out

    def _clip_worker(self, streams, starts, frames, step, todo, ready, stop):
        """one host thread of clips(): decodes streams taken from `todo` one after the other, hands each sampled picture
        to the calling thread and waits until its export has been enqueued; errors go to `ready` and stop the others"""
        try:
            while not stop.is_set():
                try:
                    i = todo.get_nowait()
                except queue.Empty:
                    return
                want = {starts[i] + t * step: t for t in range(frames)}
                last, k = max(want), 0

                def take(h, info):
                    nonlocal k
                    t = want.get(k)
                    k += 1
                    if t is not None and not stop.is_set():
                        done = threading.Event()
                        ready.put((i, t, h, info.copy(), done))
                        done.wait()
                    return k > last or stop.is_set()          # True: the stream's last sampled picture is out

                try:
                    for finished in self._decode(streams[i], take):
                        if finished:
                            break
                except RuntimeError as e:
                    raise RuntimeError("stream %d: %s" % (i, e)) from None
                if k <= last and not stop.is_set():
                    raise ValueError("stream %d has %d pictures; the clip needs picture %d" % (i, k, last))
        except BaseException as e:                          # noqa: B036  (handed to the calling thread)
            stop.set()
            ready.put(e)

    def _decode(self, tus, export):
        """the decode loop of pictures() and tensors(): export(h, info) runs for every output picture while the stream
        holds it (info = w, h, bpc, layout, matrix_coefficients, color_range), and what it returns is yielded"""
        self._hooked._bind()
        d = self.dll
        h = d.refdrv_stream_open(self.n_threads, self.max_frame_delay, self.apply_grain)
        if not h:
            raise RuntimeError("dav1d_open failed")
        ctx = d.refdrv_stream_context(h)
        try:
            if d.b200hook_set_device_only(ctx, 1):
                raise RuntimeError("too many decoders with device output open")
            info = np.zeros(6, np.int32)
            for tu in list(tus) + [None]:
                pending = 1 if tu is not None else 0
                if tu is not None:
                    pending = d.refdrv_stream_send(h, tu, len(tu))
                while True:
                    while True:
                        r = d.refdrv_stream_get(h, info.ctypes.data, 0 if tu is not None else 1)
                        if r == _EAGAIN:
                            break
                        if r < 0:
                            raise RuntimeError("decoding failed: dav1d error %d" % r)
                        try:
                            out = export(h, info)
                        finally:
                            d.refdrv_stream_release(h)
                        yield out
                    if pending < 0:
                        raise RuntimeError("decoding failed: dav1d error %d" % pending)
                    if pending == 0:
                        break
                    pending = d.refdrv_stream_send(h, None, 0)
        finally:
            d.refdrv_stream_close(h)                # frames still in flight are flushed as device-output frames
            d.b200hook_set_device_only(ctx, 0)

    @staticmethod
    def _matrix(matrix, mtrx, layout):
        name = MTRX_TO_MATRIX.get(mtrx, "bt709") if matrix == "auto" else matrix
        if name == "identity" and layout != 3:
            if matrix == "identity":
                raise ValueError("the identity matrix needs a 4:4:4 picture")
            name = "bt709"
        return name

    def _export_tensor(self, h, info, dst, oh, ow, dtype, layout, mean, std, matrix, full_range, siting, antialias, stream, box,
                       flip, interpolation, tone=None, jitter=None):
        job = self._tensor_job(h, info, dst, oh, ow, dtype, layout, mean, std, matrix, full_range, siting, antialias, flip,
                               interpolation, jitter is not None)
        box = (C.c_int32 * 4)(*box) if box else None
        pic = self.dll.refdrv_stream_picture(h)
        tones = (C.POINTER(ToneMap) * 1)(C.pointer(tone)) if tone is not None else None
        if jitter is not None:
            rc = self.dll.b200hook_export_tensor_jitter_batch((C.c_void_p * 1)(pic), C.byref(job), box, tones,
                                                              (C.POINTER(ColorJitter) * 1)(C.pointer(jitter)), 1, C.c_void_p(stream))
        elif tone is None:
            rc = self.dll.b200hook_export_tensor(pic, C.byref(job), box, C.c_void_p(stream))
        else:
            rc = self.dll.b200hook_export_tensor_tone_batch((C.c_void_p * 1)(pic), C.byref(job), box, tones, 1, C.c_void_p(stream))
        if rc != 0:
            raise RuntimeError("exporting a picture failed (see stderr)")

    def color(self, h):
        """the colour description and HDR metadata of the picture stream h holds: dict of primaries, transfer (codes of the
        sequence header), max_cll, max_fall (cd/m^2) and mastering_max / mastering_min (cd/m^2), 0 where absent"""
        out = np.zeros(6, np.int32)
        if self.dll.refdrv_stream_color(h, out.ctypes.data) != 0:
            raise RuntimeError("no picture is held")
        pri, trc, cll, fall, mx, mn = (int(v) for v in out)
        return dict(primaries=pri, transfer=trc, max_cll=cll, max_fall=fall, mastering_max=(mx & 0xffffffff) / 256.0,
                    mastering_min=(mn & 0xffffffff) / 16384.0)

    def _tone(self, h, info, out, tonemap, peak, sdr_peak):
        """the B200ToneMap of the picture stream h holds, None when it is exported as it is coded. Its tables are built once
        per (transfer, primaries, bit depth, peak, SDR peak) and kept by this decoder, until release(), on the device of
        the destination `out` (host arrays for a host destination), so they outlive every launch that reads them."""
        if tonemap is None:
            return None
        col = self.color(h)
        transfer = {v: k for k, v in TRANSFERS.items()}.get(col["transfer"]) if tonemap == "auto" else tonemap
        if transfer is None:
            return None
        if peak is None:
            peak = (col["max_cll"] or col["mastering_max"] or HDR_PEAK) if transfer == "pq" else HDR_PEAK
        bpc = int(info[2])
        device = out.device if getattr(out, "is_cuda", False) else None
        key = (transfer, col["primaries"], bpc, float(peak), float(sdr_peak), str(device))
        if key not in self._tones:
            curve, m, oetf = tone_tables(transfer, col["primaries"], bpc, peak, sdr_peak)
            tables = [_on_device(curve, device), _on_device(oetf, device)]
            tm = ToneMap()
            tm.curve, tm.oetf = _data_ptr(tables[0]), _data_ptr(tables[1])
            tm.curve_len, tm.oetf_bits = len(curve), (len(oetf) - 1).bit_length() - 1
            for k in range(9):
                tm.m[k] = float(m.ravel()[k])
            self._tones[key] = (tm, tables)
        return self._tones[key][0]

    def _jitter(self, jit, out, stream):
        """the B200ColorJitter of jit = (jitter tuple or None, grayscale) as _picture_jitter gives it (None: no jitter),
        with contrast scratch from _acc"""
        if jit is None:
            return None
        return color_jitter(*jit, acc=self._acc(out, stream, 1))

    def _acc(self, out, stream, n):
        """the address of n uint64 contrast sums (B200ColorJitter.acc) on the device of the destination `out` (host memory
        for a host destination), for exports on `stream`. Each (device, stream) has its own, so exports on different streams
        never share one; on one stream, the export of the next call waits for the last. Kept until release()."""
        device = out.device if getattr(out, "is_cuda", False) else None
        bufs = self._accs.setdefault((str(device), stream), [])
        if not bufs or len(bufs[-1]) < n:
            size = max(n, 2 * len(bufs[-1]) if bufs else 16)
            if device is None:
                bufs.append(np.zeros(size, np.uint64))
            else:
                import torch
                bufs.append(torch.empty(size, dtype=torch.int64, device=device))
        return _data_ptr(bufs[-1])

    def _drop_tables(self):
        """frees the tone tables and the contrast scratch once the launches that may still read them have completed"""
        import sys
        if "torch" in sys.modules:
            arrays = [t for _, tables in self._tones.values() for t in tables] + [a for bufs in self._accs.values() for a in bufs]
            for dev in {t.device for t in arrays if getattr(t, "is_cuda", False)}:
                sys.modules["torch"].cuda.synchronize(dev)
        self._tones.clear()
        self._accs.clear()

    def _tensor_job(self, h, info, dst, oh, ow, dtype, layout, mean, std, matrix, full_range, siting, antialias, flip,
                    interpolation="bilinear", jittered=False):
        """the B200TensorJob of the picture stream h holds (info as _decode gives it): "auto" matrix, range and siting come
        from that stream's own headers"""
        w, hh, bpc, pl, mtrx, color_range = (int(v) for v in info)
        job = TensorJob()
        job.out_w, job.out_h, job.dtype, job.layout = ow, oh, TENSOR_DTYPES[dtype], TENSOR_LAYOUTS[layout]
        name = self._matrix(matrix, mtrx, pl)
        job.identity = name == "identity"
        job.full_range = int(bool(color_range if full_range is None else full_range))
        if not job.identity:
            job.cy, job.rv, job.gu, job.gv, job.bu = rgb_coefficients(name, job.full_range)
        if siting == "auto":
            siting = CHR_TO_SITING.get(self.dll.refdrv_stream_chroma_position(h), "left")
        job.siting_x, job.siting_y = SITINGS[siting]
        scale, bias = tensor_scale_bias(bpc, mean, std, jittered)
        for c in range(3):
            job.scale[c], job.bias[c] = float(scale[c]), float(bias[c])
        job.antialias = int(bool(antialias))
        job.flip = int(flip)
        job.interpolation = TENSOR_INTERPOLATIONS[interpolation]
        job.dst = dst
        job.pitch_y, job.pitch_c = (ow, oh * ow) if layout == "chw" else (3 * ow, 1)
        return job

    def _export(self, h, info, format, matrix, full_range, alloc, stream):
        w, hh, bpc, layout, mtrx, color_range = (int(v) for v in info)
        dtype = "uint8" if bpc == 8 else "int16"
        job = ExportJob()
        job.format = EXPORT_FORMATS[format]
        if format == "planes":
            outs = [alloc((ph, pw), dtype) for pw, ph in plane_dims(w, hh, layout)]
            for k, o in enumerate(outs):
                job.dst[k], job.dst_pitch[k] = _data_ptr(o), plane_dims(w, hh, layout)[k][0]
            result = tuple(outs)
        else:
            name = self._matrix(matrix, mtrx, layout)
            job.identity = name == "identity"
            job.full_range = int(bool(color_range if full_range is None else full_range))
            if not job.identity:
                job.cy, job.rv, job.gu, job.gv, job.bu = rgb_coefficients(name, job.full_range)
            result = alloc((3, hh, w), dtype)
            base = _data_ptr(result)
            for k in range(3):
                job.dst[k], job.dst_pitch[k] = base + k * hh * w * (1 if bpc == 8 else 2), w
        if self.dll.b200hook_export_picture(self.dll.refdrv_stream_picture(h), C.byref(job), C.c_void_p(stream)) != 0:
            raise RuntimeError("exporting a picture failed (see stderr)")
        return result


_EAGAIN = -11
# clips(): streams decoded at once by default and at most. Each open stream is a device-output dav1d context (the hooks
# register up to 64) holding up to 8 reference pictures + its frames in flight + its output in the hooks' pool of 1024
# page-locked pictures.
CLIP_WORKERS = 4
CLIP_MAX_WORKERS = 32


def _default_alloc(alloc, stream):
    """(alloc, cudaStream_t handle) of an export: torch CUDA tensors on the current stream unless the caller brings its own"""
    if alloc is None:
        import torch
        alloc = lambda shape, dtype: torch.empty(shape, dtype=getattr(torch, dtype), device="cuda")
        if stream is None:
            stream = torch.cuda.current_stream()
    return alloc, getattr(stream, "cuda_stream", stream) or 0


def _check_tonemap(tonemap, peak, sdr_peak):
    if tonemap is not None and tonemap != "auto" and tonemap not in TRANSFERS:
        raise ValueError("tonemap must be None, 'auto', 'pq' or 'hlg', not %r" % (tonemap,))
    for name, v in (("peak", peak), ("sdr_peak", sdr_peak)):
        if v is not None and not (isinstance(v, (int, float, np.integer, np.floating)) and np.isfinite(v) and v > 0):
            raise ValueError("%s must be a positive number of cd/m^2, not %r" % (name, v))
    if sdr_peak is None:
        raise ValueError("sdr_peak must be a positive number of cd/m^2")


def _on_device(a, device):
    """the numpy array a as a CUDA tensor on `device`, its copy complete when this returns, or a itself for device None"""
    if device is None:
        return a
    import torch
    t = torch.from_numpy(a).to(device)
    torch.cuda.synchronize(device)
    return t


def _picture_jitter(jitter, grayscale, who):
    """(jitter, grayscale) of one picture or stream, checked (ValueError naming `who`), or None when it has neither"""
    if not _is_flag(grayscale):
        raise ValueError("%s: grayscale must be a bool, not %r" % (who, grayscale))
    if jitter is None and not grayscale:
        return None
    if jitter is not None:
        try:
            jitter_factors(jitter)
        except ValueError as e:
            raise ValueError("%s: %s" % (who, e)) from None
    return jitter, bool(grayscale)


def _picture_box(box, info, who):
    """align_crop of box (None: no crop) on the picture of `info`; ValueError naming `who`"""
    if box is None:
        return None
    try:
        return align_crop(box, int(info[0]), int(info[1]), int(info[3]))
    except ValueError as e:
        raise ValueError("%s: %s" % (who, e)) from None


def _data_ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


class Level1Decoder:
    """dav1d with its own reconstruction code, but every DSP table slot (`Dav1dDSPContext`: itx, mc, ipred, loopfilter,
    cdef, looprestoration, filmgrain) overridden by libb200av1's Level-1 functions — the architecture-hook form of the
    drop-in (integration/dav1d/b200_level1.c). One kernel launch per DSP call: a parity harness, not a throughput path.
    `families` = iterable of FAMILIES keys (default: all seven)."""

    def __init__(self, backend=None, families=None):
        if not os.path.exists(LEVEL1_SO):
            build_hooked()
            if not os.path.exists(LEVEL1_SO):
                raise RuntimeError("%s missing (it is built where the reference sources exist)" % LEVEL1_SO)
        if backend is None:
            from . import _lib
            backend = _lib.get_lib().path
        self.dll = C.CDLL(LEVEL1_SO)
        mask = sum(FAMILIES[f] for f in (families or FAMILIES))
        if self.dll.b200l1_set_backend(backend.encode(), mask) != 0:
            raise RuntimeError("b200l1_set_backend(%s) failed" % backend)

    def c_slots_left(self):
        """(slots still on dav1d's C functions after the back end's init, slots replaced): the first must be 0"""
        return int(self.dll.b200l1_c_slots_left()), int(self.dll.b200l1_slots_replaced())

    def decode(self, tus, **kw):
        kw.setdefault("n_threads", 1)            # the Level-1 thunks serialise on one lock anyway
        kw.setdefault("max_frame_delay", 1)
        return decode_stream(self.dll, tus, **kw)
