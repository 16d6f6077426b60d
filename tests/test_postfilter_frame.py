"""The CDEF and loop-restoration frame kernels (cdef_frame_kernel behind b200_cdef_frame, lr_frame_kernel behind
b200_lr_frame, and both band by band in the frame job) on content that reaches their branches, in every layout, at odd
picture sizes and at band seams.

The frames keep synth.make_lf_frame's tilings and masks, synth.make_cdef_params' cdef_idx / noskip layout and
synth.make_lr_params' lr_mask layout, and repaint the pictures:
  CDEF: each 8x8 block is a straight edge at one of 32 angles, exactly flat (variance 0: the luma primary strength
        adjusts to 0), full-range noise (high variance: it keeps its full value), or, next to the picture edges, pinned at
        0 or bitdepth_max with a small checkerboard. The strength tables hold every class (primary + secondary, primary
        only, secondary only, neither) at primary 15 / secondary 4 and primary 1 / secondary 1; damping runs 3 to 6, and
        damping 3 with chroma primary 15 clamps the primary shift at 0.
  LR:   16x16 cells that are flat (bright ones at bitdepth_max, where 12-bit SGR products pass 2^31), hard edges and
        checkerboards between 0 and bitdepth_max, noise and ramps; the deblocked picture is the CDEF picture with its top
        bit flipped, so a sample read from the wrong one moves the output. A share of the Wiener units takes the extreme
        taps of test_postfilter_mapping.WIENER_EXTREMES.

The oracle counts the branches each case takes (oracle_cdef_counts / oracle_lr_counts); the CPU tests assert every
counter against the floors stated below and the oracle against dav1d's own frame drivers. The cases run on the host
emulator and the GPU against the oracle, and the GPU also compares with dav1d's driver where oracle/_ref exists.
Band seams: a frame job with no reconstruction records runs {CDEF}, {LR}, {CDEF, LR} and {LF, CDEF, LR} through
b200_frame_run_band, and every row b200_band_progress reports after a band must already be final.
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, get_lib, synth
from test_cdef import cdef_frame_struct
from test_looprestoration import lr_frame_struct
from test_postfilter_mapping import WIENER_EXTREMES
import test_deblock_frame as TDF

LAYOUTS = {"420": (1, 1), "422": (1, 0), "444": (0, 0), "400": (1, 1)}

CDEF_COUNTERS = ("skip_idx", "skip_noskip", "skip_zero", "pri_sec", "pri", "sec", "adj_zero", "adj_full", "shift_clamp",
                 *("dir%d" % d for d in range(8)), "edge_l", "edge_r", "edge_t", "edge_b", "clamp_px", "tap_dropped")
LR_COUNTERS = ("none", "wiener", "sgr5", "sgr3", "sgr_mix", "ext_h", "pulled_up", "hor_clip_lo", "hor_clip_hi",
               "out_clip_lo", "out_clip_hi", "z0", "z255", "sgr_big", "top", "no_top", "bot", "no_bot", "bot_clamp")


def plane(S, pic, p):
    return pic[S["off"][p]:S["off"][p] + S["stride"][p] * S["rows"][p]].reshape(S["rows"][p], S["stride"][p])


def base_frame(rng, lay, bpc, W, H):
    """synth.make_lf_frame's geometry, tilings and masks; 4:0:0 in the hooks' device picture (two dummy 4:2:0 chroma
    planes at the luma stride)"""
    ssh, ssv = LAYOUTS[lay]
    S = synth.make_lf_frame(rng, bpc, W, H, ssh, ssv)
    if lay == "400":
        st, rows = S["stride"][0], S["rows"][0]
        S["stride"], S["rows"] = [st, st, st], [rows, rows >> 1, rows >> 1]
        S["off"] = [0, st * rows, st * rows + st * (rows >> 1)]
        S["pic"] = np.zeros(S["off"][2] + st * (rows >> 1), S["pic"].dtype)
    S["lay"] = lay
    return S


def relayout(S, pad):
    """the same planes in a buffer whose strides and plane offsets are `pad` samples past a multiple of 4"""
    T = dict(S)
    T["stride"] = [s + pad for s in S["stride"]]
    off, o = [], pad
    for p in range(3):
        off.append(o)
        o += T["stride"][p] * S["rows"][p] + pad
    T["off"] = off
    for key in ("pic", "cdef", "dbl"):
        if key in S:
            a = np.zeros(o, S[key].dtype)
            for p in range(3):
                plane(T, a, p)[:, :S["stride"][p]] = plane(S, S[key], p)
            T[key] = a
    return T


# ---------------------------------------------------------------------------------------- CDEF content
# strength index: (y, uv). Luma: pri 15 + sec 4, pri 1 + sec 1, pri 15 only, sec 4 only, sec 1 only, none, pri 15 + sec 2;
# chroma likewise in other slots; index 7 is 0 / 0 (the whole 64x64 area is skipped)
Y_STRENGTH = [63, 5, 60, 3, 1, 0, 62, 0]
UV_STRENGTH = [63, 5, 3, 60, 0, 4, 61, 0]


def paint_cdef_plane(rng, dst, bpc, aw, ah):
    """8x8 blocks of the classes in the module docstring; dst is the whole plane, (aw, ah) the filtered area"""
    bd, sc = (1 << bpc) - 1, 1 << (bpc - 8)
    rows, stride = dst.shape
    nby, nbx = -(-rows // 8), -(-stride // 8)
    # 0 edges, 1 flat, 2 noise, 3 edges with low contrast, 6 one noiseless hard edge with single-sample dips and peaks (the
    # combined filter overshoots its taps there and the min / max clamp acts)
    cat = rng.choice([0, 1, 2, 3, 6], (nby, nbx), p=[0.25, 0.15, 0.1, 0.1, 0.4])
    # pinned clusters (2x2 blocks) next to the picture edges: at 0 or at bitdepth_max
    byy, bxx = np.mgrid[0:nby, 0:nbx]
    near = (bxx * 8 < 16) | (bxx * 8 >= aw - 24) | (byy * 8 < 16) | (byy * 8 >= ah - 24)
    cl = rng.random((nby // 2 + 1, nbx // 2 + 1))[byy // 2, bxx // 2]
    cat[near & (cl < 0.25)] = 4
    cat[near & (cl > 0.75)] = 5
    ang = rng.integers(0, 32, (nby, nbx)) * np.pi / 32
    phase = rng.random((nby, nbx)) * 2 * np.pi
    mid = rng.integers(bd // 4, 3 * bd // 4 + 1, (nby, nbx))
    amp = np.where(cat == 3, rng.integers(2, 12, (nby, nbx)) * sc, rng.integers(bd // 8, bd // 2 + 1, (nby, nbx)))
    flat = rng.integers(0, bd + 1, (nby, nbx))
    ys, xs = np.mgrid[0:rows, 0:stride]
    by, bx, yy, xx = ys >> 3, xs >> 3, ys & 7, xs & 7
    a = ang[by, bx]
    edge = mid[by, bx] + amp[by, bx] * np.sign(np.sin((np.cos(a) * xx + np.sin(a) * yy) * 1.7 + phase[by, bx]))
    edge = edge + rng.integers(-2 * sc, 2 * sc + 1, (rows, stride))
    c = cat[by, bx]
    chk = ((xx + yy) & 1) * rng.choice([2, 3], (rows, stride)) * sc
    v = np.where(c <= 0, edge, 0)
    v = np.where(c == 3, edge, v)
    v = np.where(c == 1, flat[by, bx], v)
    imp = np.where(rng.random((rows, stride)) < 0.1, rng.choice([-4, -3, -2, 2, 3, 4], (rows, stride)) * sc, 0)
    one = np.where(np.cos(a) * (xx - 3.5) + np.sin(a) * (yy - 3.5) > phase[by, bx] - np.pi, bd // 4, -(bd // 4))
    v = np.where(c == 6, np.clip(mid[by, bx] + one, 4 * sc, bd - 4 * sc) + imp, v)
    v = np.where(c == 2, rng.integers(0, bd + 1, (rows, stride)), v)
    v = np.where(c == 4, chk, v)
    v = np.where(c == 5, bd - chk, v)
    dst[:] = np.clip(v, 0, bd)


def make_cdef_case(lay, bpc, W, H, damping, seed):
    rng = np.random.default_rng(seed)
    S = base_frame(rng, lay, bpc, W, H)
    S["bw"], S["bh"] = S["w4"], S["h4"]
    synth.make_cdef_params(rng, S["bw"], S["bh"], S["sb128w"], S["masks"])     # noskip
    # -1 and every strength index, evenly over the 64x64 areas inside the picture
    idx = S["masks"]["cdef_idx"].reshape(-1, S["sb128w"], 2, 2)
    ay, ax = np.nonzero(np.ones(((S["bh"] + 15) // 16, (S["bw"] + 15) // 16), bool))
    idx[ay // 2, ax // 2, ay & 1, ax & 1] = rng.permutation(len(ay)) % 9 - 1
    S["damping"] = damping
    S["y_strength"] = list(Y_STRENGTH)
    S["uv_strength"] = [0] * 8 if lay == "400" else list(UV_STRENGTH)          # 4:0:0 has no chroma strengths
    for p in range(3):
        sh, sv = (S["ss_hor"], S["ss_ver"]) if p else (0, 0)
        paint_cdef_plane(rng, plane(S, S["pic"], p), bpc, (S["bw"] * 4) >> sh, (S["bh"] * 4) >> sv)
    return S


def cdef_oracle(S):
    dst = S["pic"].copy()
    refs.oracle().oracle_cdef_frame(S["bd"], C.byref(cdef_frame_struct(S, S["pic"].ctypes.data, dst.ctypes.data, S["masks"].ctypes.data)))
    return dst


def cdef_reference(S):
    pic = S["pic"].copy()
    fr = cdef_frame_struct(S, pic.ctypes.data, None, S["masks"].ctypes.data)
    (refs.ref().refdrv_cdef_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_cdef_frame_16bpc)(S["bd"], C.byref(fr))
    return pic


def cdef_counts():
    out = np.zeros(2 * len(CDEF_COUNTERS), np.int64)
    assert refs.oracle().oracle_cdef_counts(C.c_void_p(out.ctypes.data)) == len(CDEF_COUNTERS)
    return [dict(zip(CDEF_COUNTERS, map(int, r))) for r in out.reshape(2, -1)]


def cdef_area_diff(S, a, b):
    """per plane: samples that differ inside the bw x bh area (the rest of the planes is not CDEF output)"""
    out = []
    for p in range(3):
        sh, sv = (S["ss_hor"], S["ss_ver"]) if p else (0, 0)
        w, h = (S["bw"] * 4) >> sh, (S["bh"] * 4) >> sv
        out.append(int((plane(S, a, p)[:h, :w] != plane(S, b, p)[:h, :w]).sum()))
    return out


# (W, H): bw / bh odd / odd, odd / even, odd / even, even / odd; 258, 331, 270 are not multiples of 4
CDEF_GEOMS = [(258, 146), (331, 198), (196, 134), (270, 178)]
CDEF_CASES = [(lay, bpc, *CDEF_GEOMS[(i + j) % 4], 3 + (i + 2 * j) % 4) for i, lay in enumerate(LAYOUTS) for j, bpc in enumerate((8, 10, 12))]


def cdef_case_id(c):
    return "%s-%dbit-%dx%d-damp%d" % c


def cdef_frame(c):
    return make_cdef_case(*c, seed=1100 + sum(c[1:]) + 100 * list(LAYOUTS).index(c[0]))


# floors, as a share of the plane class's filtered blocks (at least 1); a counter missing here has its own rule below
# (a small frame has few filtered blocks on its right or bottom edge: the edge counters are floors over all cases)
CDEF_FLOOR = {"pri_sec": 0.1, "pri": 0.02, "sec": 0.05, "clamp_px": 0.005, "adj_zero": 0.01, "adj_full": 0.01, "tap_dropped": 0.5,
              **{"dir%d" % d: 0.01 for d in range(8)}, "skip_idx": 0, "skip_noskip": 0.02, "skip_zero": 0}


def cdef_below_floor(S, counts):
    low = []
    chroma = S["lay"] != "400"
    for pc, c in enumerate(counts):
        blocks = c["pri_sec"] + c["pri"] + c["sec"]
        if pc and not chroma:
            if blocks:
                low.append((pc, "chroma filtered", blocks, 0))
            continue
        for k, share in CDEF_FLOOR.items():
            if pc and k in ("adj_zero", "adj_full"):
                continue                  # only luma adjusts its primary strength
            if pc and k in ("dir1", "dir3") and S["ss_hor"] and not S["ss_ver"]:
                continue                  # 4:2:2 chroma maps the luma direction onto 7 0 2 4 5 6 6 6
            floor = max(1, int(share * blocks))
            if c[k] < floor:
                low.append((pc, k, c[k], floor))
        # the primary shift clamps at 0 only for chroma at damping 3 (damping - 1 - ulog2(15) < 0)
        if (c["shift_clamp"] > 0) != (pc == 1 and S["damping"] == 3):
            low.append((pc, "shift_clamp", c["shift_clamp"], S["damping"]))
    return low


@pytest.mark.parametrize("case", CDEF_CASES, ids=cdef_case_id)
def test_cdef_content_reaches_every_branch(case):
    S = cdef_frame(case)
    cdef_counts()
    cdef_oracle(S)
    counts = cdef_counts()
    assert not cdef_below_floor(S, counts), (cdef_below_floor(S, counts), counts)


def test_cdef_edges_over_the_cases():
    total = np.zeros((2, 4), np.int64)
    for case in CDEF_CASES:
        cdef_counts()
        cdef_oracle(cdef_frame(case))
        total += [[c[k] for k in ("edge_l", "edge_r", "edge_t", "edge_b")] for c in cdef_counts()]
    assert (total >= 50).all(), total


def test_cdef_cases_cover_layouts_depths_damping_geometry():
    assert {(c[0], c[1]) for c in CDEF_CASES} == {(lay, bpc) for lay in LAYOUTS for bpc in (8, 10, 12)}
    assert {c[4] for c in CDEF_CASES} == {3, 4, 5, 6}
    assert any(c[4] == 3 and c[0] != "400" for c in CDEF_CASES)
    w4s, h4s = {(c[2] + 3) // 4 for c in CDEF_CASES}, {(c[3] + 3) // 4 for c in CDEF_CASES}
    assert any(w & 1 for w in w4s) and any(h & 1 for h in h4s) and any(not h & 1 for h in h4s)
    assert any(c[2] % 4 for c in CDEF_CASES)


@pytest.mark.parametrize("case", CDEF_CASES, ids=cdef_case_id)
def test_cdef_oracle_vs_reference_driver(case):
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = cdef_frame(case)
    exp = cdef_oracle(S)
    assert cdef_area_diff(S, exp, cdef_reference(S)) == [0, 0, 0]
    assert sum(cdef_area_diff(S, exp, S["pic"])[:1 if S["lay"] == "400" else 3]) > 0


class Pics:
    """named pictures of a case where the library reads them: host memory for the emulator, HBM for the GPU"""

    def __init__(self, gpu, **arrays):
        self.gpu, self.dtype = gpu, next(iter(arrays.values())).dtype
        self.lib = get_lib() if gpu else refs.emu_lib()
        self.a = {}
        for k, v in arrays.items():
            if gpu:
                import torch
                self.a[k] = torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).copy()).cuda()
            else:
                self.a[k] = np.ascontiguousarray(v).copy()

    def ptr(self, k):
        return self.a[k].data_ptr() if self.gpu else self.a[k].ctypes.data

    def get(self, k):
        if not self.gpu:
            return self.a[k].copy()
        import torch
        torch.cuda.synchronize()
        return self.a[k].cpu().numpy().view(self.dtype)


def run_cdef(S, gpu):
    d = Pics(gpu, src=S["pic"], dst=np.zeros_like(S["pic"]), mask=S["masks"].view(np.uint8))
    d.lib.check(d.lib.b200_cdef_frame(S["bd"], C.byref(cdef_frame_struct(S, d.ptr("src"), d.ptr("dst"), d.ptr("mask"))), None), "b200_cdef_frame")
    return d.get("dst")


def check_cdef(S, gpu, reference=False):
    got, exp = run_cdef(S, gpu), cdef_oracle(S)
    assert cdef_area_diff(S, got, exp) == [0, 0, 0]
    if reference and refs.have_ref():
        assert cdef_area_diff(S, got, cdef_reference(S)) == [0, 0, 0]


@pytest.mark.emu
@pytest.mark.parametrize("case", CDEF_CASES, ids=cdef_case_id)
def test_emu_cdef_frame(case):
    check_cdef(cdef_frame(case), False)


def check_cdef_misaligned(gpu):
    """stride / plane offsets that are not 4-sample multiples: -2, and dst untouched"""
    S = relayout(cdef_frame(CDEF_CASES[0]), 1)
    d = Pics(gpu, src=S["pic"], dst=np.full_like(S["pic"], 7), mask=S["masks"].view(np.uint8))
    fr = cdef_frame_struct(S, d.ptr("src"), d.ptr("dst"), d.ptr("mask"))
    assert d.lib.b200_cdef_frame(S["bd"], C.byref(fr), None) == -2
    assert b"4-sample aligned" in d.lib.b200_last_error()
    assert (d.get("dst") == 7).all()


@pytest.mark.emu
def test_emu_cdef_misaligned_planes():
    check_cdef_misaligned(False)


# ---------------------------------------------------------------------------------------- LR content
def paint_lr_plane(rng, dst, bpc):
    """16x16 cells: flat (a share at bitdepth_max), hard edges and checkerboards between 0 and bitdepth_max, noise, ramps"""
    bd, sc = (1 << bpc) - 1, 1 << (bpc - 8)
    rows, stride = dst.shape
    ny, nx = -(-rows // 16), -(-stride // 16)
    cat = rng.choice(6, (ny, nx), p=[0.2, 0.15, 0.2, 0.1, 0.15, 0.2])
    ys, xs = np.mgrid[0:rows, 0:stride]
    cy, cx, yy, xx = ys >> 4, xs >> 4, ys & 15, xs & 15
    c = cat[cy, cx]
    flat = np.where(rng.random((ny, nx)) < 0.5, bd - rng.integers(0, 2, (ny, nx)), rng.integers(0, bd + 1, (ny, nx)))
    cut = rng.integers(3, 13, (ny, nx))
    vert = rng.random((ny, nx)) < 0.5
    side = np.where(vert[cy, cx], xx, yy) < cut[cy, cx]
    edge = np.where(side, 0, bd)
    period = rng.choice([1, 2, 4], (ny, nx))[cy, cx]
    checker = np.where(((xx // period) + (yy // period)) & 1, bd, 0)
    noise = rng.integers(0, bd + 1, (rows, stride))
    slope = rng.integers(-6, 7, (ny, nx))[cy, cx] * sc
    ramp = rng.integers(0, bd + 1, (ny, nx))[cy, cx] + slope * (xx + yy) + rng.integers(-sc, sc + 1, (rows, stride))
    v = np.select([c == 0, c == 1, c == 2, c == 3, c == 4], [flat[cy, cx], edge, checker, noise, ramp], ramp)
    dst[:] = np.clip(v, 0, bd)


def make_lr_case(lay, bpc, W, H, us, rp, sb128, seed):
    rng = np.random.default_rng(seed)
    S = base_frame(rng, lay, bpc, W, H)
    cdef = S["pic"]
    for p in range(3):
        paint_lr_plane(rng, plane(S, cdef, p), bpc)
    S["cdef"] = cdef
    S["dbl"] = cdef ^ np.asarray(1 << (bpc - 1), cdef.dtype)            # every sample differs by half the range
    m = synth.make_lr_params(rng, W, H, p_none=0.15)
    S["lr_mask"], S["sb128"], S["us"], S["rp"] = m, sb128, us, (rp & 1 if lay == "400" else rp)
    u = m["lr"]
    # the units the stripes look up (in either superblock size) take none, Wiener, SGR 5x5, 3x3 and both in turn
    for p in range(3):
        seen = sorted({e for sb in (0, 1) for e in lr_units(dict(S, sb128=sb), p)})
        cycle = [0, 2, 17, 13, 3, 2, 18, 14, 8, 15, 12, 16]
        for k, i in enumerate(rng.permutation(len(seen))):
            u["type"][seen[i][0], p, seen[i][1]] = cycle[k % len(cycle)]
    idx = np.clip(u["type"].astype(np.int32) - 3, 0, 15)
    s0 = np.array([q[0] for q in synth.SGR_PARAMS])[idx]; s1 = np.array([q[1] for q in synth.SGR_PARAMS])[idx]
    u["sgr_weights"][..., 0] = np.where(s0 > 0, rng.integers(-96, 32, idx.shape), 0)
    u["sgr_weights"][..., 1] = np.where(s1 > 0, rng.integers(-32, 96, idx.shape), 95)
    wiener = u["type"] == 2
    ext = wiener & (rng.random(u["type"].shape) < 0.7)
    taps = np.array(WIENER_EXTREMES, np.int8)
    u["filter_h"][ext] = taps[rng.integers(0, len(taps), ext.sum())]
    u["filter_v"][ext] = taps[rng.integers(0, len(taps), ext.sum())]
    u["filter_h"][:, 1:, :, 0] = 0; u["filter_v"][:, 1:, :, 0] = 0        # chroma uses the 5-tap form
    return S


def plane_dims(S, p):
    sh, sv = (S["ss_hor"], S["ss_ver"]) if p else (0, 0)
    return (S["W"] + sh) >> sh, (S["H"] + sv) >> sv


def stripes(S, p):
    """[(y0, y1)] of the 64-row stripes of plane p (8 rows shorter at the top; halved when vertically subsampled)"""
    sv = S["ss_ver"] if p else 0
    h, out, y0, k = plane_dims(S, p)[1], [], 0, 0
    while y0 < h:
        y1 = min(h, (64 * (k + 1) - 8) >> sv)
        out.append((y0, y1))
        y0, k = y1, k + 1
    return out


def lr_unit_row(S, p, y0):
    """lr_mask index of the first unit of the unit row stripe y0 of plane p looks up, and its unit_idx"""
    sv = S["ss_ver"] if p else 0
    h, unit = plane_dims(S, p)[1], 1 << S["us"][min(p, 1)]
    sby = ((y0 << sv) + (8 if y0 else 0)) >> (6 + S["sb128"])
    aligned = ((sby << (6 + S["sb128"])) >> sv) & ~(unit - 1)
    pulled = bool(aligned and aligned + unit // 2 > h)
    aligned = (aligned - unit * pulled) << sv
    return (aligned >> 7) * ((S["W"] + 127) >> 7), ((aligned >> 6) & 1) << 1, pulled


def lr_units(S, p):
    """[(lr_mask index, unit index)] of the units plane p's stripes look up (lr_sbrow's walk)"""
    w = plane_dims(S, p)[0]
    unit, shift_hor = 1 << S["us"][min(p, 1)], 7 - (S["ss_hor"] if p else 0)
    out = []
    for y0, _ in stripes(S, p):
        sb_idx, unit_idx, _ = lr_unit_row(S, p, y0)
        x = 0
        while x < w:
            out.append((sb_idx + (x >> shift_hor), unit_idx + ((x >> (shift_hor - 1)) & 1)))
            x += unit if x + unit + unit // 2 <= w else w - x
    return out


def lr_geometry(S):
    """per plane class: the counters that follow from the geometry alone (a restatement of lr_sbrow's unit walk)"""
    out = [dict.fromkeys(("ext_h", "pulled_up", "top", "no_top", "bot", "no_bot", "bot_clamp"), 0) for _ in range(2)]
    for p in range(3):
        if not S["rp"] & (1 << p):
            continue
        c = out[min(p, 1)]
        w, h = plane_dims(S, p)
        unit = 1 << S["us"][min(p, 1)]
        n_units = max(1, (w + unit // 2) // unit)
        ext = n_units * unit < w
        for y0, y1 in stripes(S, p):
            c["pulled_up"] += lr_unit_row(S, p, y0)[2]
            c["ext_h"] += ext
            c["top" if y0 else "no_top"] += 1
            c["bot" if y1 < h else "no_bot"] += 1
            c["bot_clamp"] += y1 < h and y1 + 1 > h - 1
    return out


def last_stripe_rows(S, p):
    y0, y1 = stripes(S, p)[-1]
    return y1 - y0


def lr_oracle(S):
    dst = np.zeros_like(S["cdef"])
    fr = lr_frame_struct(S, S["cdef"].ctypes.data, S["dbl"].ctypes.data, dst.ctypes.data, S["lr_mask"].ctypes.data)
    refs.oracle().oracle_lr_frame(S["bd"], C.byref(fr))
    return dst


def lr_reference(S):
    c2 = S["cdef"].copy()
    fr = lr_frame_struct(S, c2.ctypes.data, S["dbl"].ctypes.data, None, S["lr_mask"].ctypes.data)
    (refs.ref().refdrv_lr_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_lr_frame_16bpc)(S["bd"], C.byref(fr))
    return c2


def lr_counts():
    out = np.zeros(2 * len(LR_COUNTERS), np.int64)
    assert refs.oracle().oracle_lr_counts(C.c_void_p(out.ctypes.data)) == len(LR_COUNTERS)
    return [dict(zip(LR_COUNTERS, map(int, r))) for r in out.reshape(2, -1)]


def lr_diff(S, a, b):
    """per plane: samples that differ inside the picture"""
    out = []
    for p in range(3):
        w, h = plane_dims(S, p)
        out.append(int((plane(S, a, p)[:h, :w] != plane(S, b, p)[:h, :w]).sum()))
    return out


# (layout, bpc, W, H, (unit_size_log2 luma, chroma), restore_planes, sb128). Heights put the last stripe of each plane at
# 1 (h - y1s == 1 for the stripe above), 2, 7 and 8 rows over the cases of each layout: luma H mod 64 = 57, 58, 63, 0;
# 4:2:0 chroma ceil(H / 2) mod 32 = 29, 30, 3, 4 (H = 121 / 186, 124, 134, 136). Widths are odd or not multiples
# of 4; the unit sizes make the last unit of a row wider than a unit in some planes and narrower in others, and pull the
# unit row of the last stripes up in some.
LR_CASES = [("420", 8, 258, 121, (6, 5), 7, 0), ("420", 10, 331, 186, (7, 6), 7, 1), ("420", 12, 197, 124, (5, 5), 7, 0),
            ("420", 8, 290, 136, (8, 7), 5, 0), ("420", 10, 226, 134, (7, 6), 3, 1), ("420", 12, 305, 127, (7, 5), 6, 0), ("420", 8, 270, 192, (6, 6), 7, 0),
            ("422", 8, 333, 121, (7, 7), 7, 0), ("422", 10, 258, 122, (7, 7), 7, 1), ("422", 12, 198, 127, (5, 6), 7, 0),
            ("422", 10, 270, 128, (8, 8), 6, 0),
            ("444", 8, 197, 128, (8, 8), 7, 1), ("444", 10, 262, 121, (8, 6), 7, 0), ("444", 12, 331, 186, (7, 7), 5, 0),
            ("444", 12, 226, 127, (5, 7), 7, 0),
            ("400", 8, 333, 122, (6, 5), 7, 0), ("400", 10, 258, 127, (8, 7), 1, 1), ("400", 12, 197, 121, (5, 5), 1, 0),
            ("400", 8, 270, 128, (7, 5), 7, 0)]


def lr_case_id(c):
    return "%s-%dbit-%dx%d-us%d.%d-rp%d-sb%d" % (c[0], c[1], c[2], c[3], c[4][0], c[4][1], c[5], c[6])


def lr_frame(c):
    return make_lr_case(*c, seed=1300 + c[1] + c[2] + c[3] + 100 * list(LAYOUTS).index(c[0]))


# A frame of the small cases has few units (one per stripe where the unit is as wide as the plane), so the unit types and
# the clips they reach are floors over all cases, per plane class; the counters that follow from the geometry must equal
# the restatement in every case. Floors: samples or units, at least; sgr_big over the 12-bit cases (x * sum * 455 or
# * 164 passes 2^31 only at 12 bit). Chroma Wiener filters are 5-tap: their horizontal intermediate clips rarely.
LR_FLOOR = {"none": 10, "wiener": 10, "sgr5": 10, "sgr3": 10, "sgr_mix": 10, "hor_clip_lo": 100, "hor_clip_hi": 100,
            "out_clip_lo": 100, "out_clip_hi": 100, "z0": 1000, "z255": 1000, "sgr_big": 100}


def lr_geometry_mismatch(S, counts):
    low = []
    for pc, (c, g) in enumerate(zip(counts, lr_geometry(S))):
        units = sum(c[k] for k in ("none", "wiener", "sgr5", "sgr3", "sgr_mix"))
        if not S["rp"] & (1 if pc == 0 else 6) and units:
            low.append((pc, "unrestored plane filtered", units))
        low += [(pc, k, c[k], "geometry says %d" % v) for k, v in g.items() if c[k] != v]
    return low


def lr_below_floor(total):
    floor = [LR_FLOOR, dict(LR_FLOOR, hor_clip_lo=1, hor_clip_hi=1)]
    return [(pc, k, total[pc][k], f) for pc in range(2) for k, f in floor[pc].items() if total[pc][k] < f]


@pytest.mark.parametrize("case", LR_CASES, ids=lr_case_id)
def test_lr_stripes_and_units_follow_the_geometry(case):
    S = lr_frame(case)
    lr_counts()
    lr_oracle(S)
    counts = lr_counts()
    assert not lr_geometry_mismatch(S, counts), (lr_geometry_mismatch(S, counts), counts)


def test_lr_content_reaches_every_branch():
    total = [dict.fromkeys(LR_COUNTERS, 0) for _ in range(2)]
    for case in LR_CASES:
        lr_counts()
        lr_oracle(lr_frame(case))
        for pc, c in enumerate(lr_counts()):
            for k, v in c.items():
                total[pc][k] += v if k != "sgr_big" or case[1] == 12 else 0
    assert not lr_below_floor(total), (lr_below_floor(total), total)


def test_lr_cases_cover_layouts_stripes_units_and_planes():
    assert {(c[0], c[1]) for c in LR_CASES} == {(lay, bpc) for lay in LAYOUTS for bpc in (8, 10, 12)}
    for lay in LAYOUTS:
        frames = [make_lr_case(*c, seed=0) for c in LR_CASES if c[0] == lay]
        for p in ((0,) if lay == "400" else (0, 1)):
            assert {last_stripe_rows(S, p) for S in frames} >= {1, 2, 7, 8}, (lay, p)
    geo = [lr_geometry(make_lr_case(*c, seed=0)) for c in LR_CASES]
    for pc in range(2):
        for k in ("ext_h", "pulled_up", "bot_clamp"):
            assert any(g[pc][k] for g in geo) and any(not g[pc][k] for g in geo if g[pc]["top"]), (pc, k)
    assert {c[4][0] for c in LR_CASES} == {5, 6, 7, 8} and {c[4][1] for c in LR_CASES} == {5, 6, 7, 8}
    assert {c[5] for c in LR_CASES} >= {1, 3, 5, 6, 7} and {c[6] for c in LR_CASES} == {0, 1}
    assert all(sb128_legal(make_lr_case(*c, seed=0)) for c in LR_CASES if c[6])
    assert sum(sb128_legal(make_lr_case(*c, seed=0)) for c in LR_CASES) >= 8


def sb128_legal(S):
    """AV1 gives frames with 128x128 superblocks restoration units of 128 or 256 (4:2:0 chroma: 64 and up). Only then
    does the last stripe of a picture that ends inside the 8 rows above a superblock row boundary look up the unit row
    dav1d's superblock-row walk gives it."""
    return S["us"][0] >= 7 and S["us"][1] >= (6 if S["ss_hor"] and S["ss_ver"] else 7)


@pytest.mark.parametrize("case", LR_CASES, ids=lr_case_id)
def test_lr_oracle_vs_reference_driver(case):
    """in both superblock sizes where the unit sizes allow it: sb128 changes which unit row a stripe's lookup lands on"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = lr_frame(case)
    for sb128 in (0, 1) if sb128_legal(S) else (0,):
        S["sb128"] = sb128
        exp = lr_oracle(S)
        assert lr_diff(S, exp, lr_reference(S)) == [0, 0, 0], sb128


def run_lr(S, gpu):
    d = Pics(gpu, cdef=S["cdef"], dbl=S["dbl"], dst=np.zeros_like(S["cdef"]), mask=S["lr_mask"].view(np.uint8))
    fr = lr_frame_struct(S, d.ptr("cdef"), d.ptr("dbl"), d.ptr("dst"), d.ptr("mask"))
    d.lib.check(d.lib.b200_lr_frame(S["bd"], C.byref(fr), None), "b200_lr_frame")
    return d.get("dst")


def check_lr(S, gpu, reference=False):
    got, exp = run_lr(S, gpu), lr_oracle(S)
    assert lr_diff(S, got, exp) == [0, 0, 0]
    if reference and refs.have_ref():
        assert lr_diff(S, got, lr_reference(S)) == [0, 0, 0]


@pytest.mark.emu
@pytest.mark.parametrize("case", LR_CASES, ids=lr_case_id)
def test_emu_lr_frame(case):
    check_lr(lr_frame(case), False)


# planes whose stride and offset are 1 and 2 samples past a multiple of 4: the tiles take the per-sample staging path
LR_MISALIGNED = [(LR_CASES[0], 1), (LR_CASES[7], 2), (LR_CASES[12], 1)]


@pytest.mark.emu
@pytest.mark.parametrize("case,pad", LR_MISALIGNED, ids=lambda v: lr_case_id(v) if isinstance(v, tuple) else str(v))
def test_emu_lr_misaligned_planes(case, pad):
    check_lr(relayout(lr_frame(case), pad), False)


# ---------------------------------------------------------------------------------------- band seams
FILTER_SETS = {"cdef": (0, 1, 0), "lr": (0, 0, 1), "cdef_lr": (0, 1, 1), "lf_cdef_lr": (1, 1, 1)}
# odd final heights; the last luma stripes are 1, 57, 7 and 18 rows long
BAND_CASES = [("420", 8, 330, 313), ("422", 10, 262, 249), ("444", 12, 198, 311), ("400", 10, 262, 186)]


def band_frame(lay, bpc, W, H):
    """one frame for every stage: deblocking levels / masks, CDEF content and strengths, LR units"""
    c = (lay, bpc, W, H, 3 + bpc % 4)
    S = make_cdef_case(*c, seed=1500 + bpc + W)
    S2 = TDF.make_case(lay, bpc, W, H, 2, 1, seed=1600 + bpc + W)     # deblocking levels and masks of the same geometry
    S["level"], S["lut_e"], S["lut_i"], S["lut_sharp"] = S2["level"], S2["lut_e"], S2["lut_i"], S2["lut_sharp"]
    S["filter_uv"] = int(lay != "400")
    S["masks"]["filter_y"], S["masks"]["filter_uv"] = S2["masks"]["filter_y"], S2["masks"]["filter_uv"]
    rng = np.random.default_rng(1700 + W)
    m = synth.make_lr_params(rng, W, H, p_none=0.15)
    S["lr_mask"], S["sb128"], S["us"], S["rp"] = m, 0, (6, 5), 1 if lay == "400" else 7
    return S


def chain_oracle(S, run_lf, run_cdef, run_lr):
    """the oracle's pictures after each enabled stage, as the hooks wire them: LR reads p0 when CDEF is off"""
    p0 = TDF.run_oracle(S) if run_lf else S["pic"].copy()
    T = dict(S, pic=p0)
    p1 = cdef_oracle(T) if run_cdef else None
    p2 = None
    if run_lr:
        p2 = lr_oracle(dict(S, cdef=p1 if run_cdef else p0, dbl=p0))
    return p0, p1, p2


class Job:
    """a frame job with no reconstruction records over p0 (deblocked in place) -> p1 (CDEF) -> p2 (LR)"""

    def __init__(self, S, gpu, run_lf, run_cdef, run_lr):
        self.S = S
        z = np.zeros_like(S["pic"])
        self.d = Pics(gpu, p0=S["pic"], p1=z, p2=z, mask=S["masks"].view(np.uint8), level=S["level"].reshape(-1),
                      lrm=S["lr_mask"].view(np.uint8))
        d = self.d
        job = _lib.FrameJob()
        job.bitdepth_max, job.run_lf, job.run_cdef, job.run_lr = S["bd"], run_lf, run_cdef, run_lr
        job.lf = TDF.lf_struct(S, d.ptr("p0"), d.ptr("mask"), d.ptr("level"))      # lf.h4 / ss_ver: the band geometry
        job.cdef = cdef_frame_struct(S, d.ptr("p0"), d.ptr("p1"), d.ptr("mask"))
        job.lr = lr_frame_struct(S, d.ptr("p1" if run_cdef else "p0"), d.ptr("p0"), d.ptr("p2"), d.ptr("lrm"))
        self.job, self.out = job, "p2" if run_lr else "p1" if run_cdef else "p0"

    def run(self):
        self.d.lib.check(self.d.lib.b200_frame_run(C.byref(self.job), None), "b200_frame_run")

    def run_band(self, y0, y1, last):
        self.d.lib.check(self.d.lib.b200_frame_run_band(C.byref(self.job), C.byref(TDF.band(y0, y1, last)), None), "b200_frame_run_band")

    def progress(self, y1, last, p):
        return self.d.lib.b200_band_progress(C.byref(self.job), y1, last, p)


def final_diff(S, a, b, rows=None):
    """per plane: samples that differ in the first `rows[p]` rows of the picture (all rows by default)"""
    out = []
    for p in range(3):
        w, h = plane_dims(S, p)
        h = h if rows is None else rows[p]
        out.append(int((plane(S, a, p)[:h, :w] != plane(S, b, p)[:h, :w]).sum()))
    return out


def check_bands(S, gpu, sets=FILTER_SETS):
    H = S["H"]
    for name, flags in sets.items():
        exp = chain_oracle(S, *flags)[2 if flags[2] else 1 if flags[1] else 0]
        j = Job(S, gpu, *flags)
        j.run()
        assert final_diff(S, j.d.get(j.out), exp) == [0, 0, 0], (name, "whole frame")
        for rows in (64, 128, 192):
            j = Job(S, gpu, *flags)
            prev = [0, 0, 0]
            for y0 in range(0, H, rows):
                y1, last = min(y0 + rows, H), int(y0 + rows >= H)
                j.run_band(y0, y1, last)
                claim = [j.progress(y1, last, p) for p in range(3)]
                # rows reported final are final; the claim moves forward and reaches the plane height at the last band
                assert all(prev[p] <= claim[p] for p in range(3)), (name, rows, y1, prev, claim)
                assert final_diff(S, j.d.get(j.out), exp, claim) == [0, 0, 0], (name, rows, y1, claim)
                prev = claim
            assert prev == [plane_dims(S, p)[1] for p in range(3)], (name, rows, prev)
            assert final_diff(S, j.d.get(j.out), exp) == [0, 0, 0], (name, rows)


def test_band_cases_cover_layouts_and_short_stripes():
    assert {c[0] for c in BAND_CASES} == set(LAYOUTS) and all(c[3] & 1 or c[0] == "400" for c in BAND_CASES)
    lens = {last_stripe_rows(make_lr_case(*c, (6, 5), 7, 0, seed=0), 0) for c in BAND_CASES}
    assert min(lens) == 1, lens


@pytest.mark.emu
@pytest.mark.parametrize("case", BAND_CASES, ids=lambda c: "%s-%dbit-%dx%d" % c)
@pytest.mark.parametrize("sets", list(FILTER_SETS))
def test_emu_band_seams(case, sets):
    check_bands(band_frame(*case), False, {sets: FILTER_SETS[sets]})


# ---------------------------------------------------------------------------------------- H100
# 1080p 8-bit 4:2:0, 4K and 8K 10-bit 4:2:0, 720p 10-bit 4:2:2 and 12-bit 4:4:4; odd bh, and last luma stripes of 4, 2,
# 4, 3 and 3 rows
GPU_LARGE = [("420", 8, 1918, 1084), ("420", 10, 3836, 2170), ("420", 10, 7678, 4284), ("422", 10, 1280, 699),
             ("444", 12, 1284, 699)]


@pytest.mark.gpu
def test_gpu_postfilter_cases():
    for case in CDEF_CASES:
        check_cdef(cdef_frame(case), True, reference=True)
    for case in LR_CASES:
        check_lr(lr_frame(case), True, reference=True)
    for case, pad in LR_MISALIGNED:
        check_lr(relayout(lr_frame(case), pad), True)
    check_cdef_misaligned(True)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_LARGE, ids=lambda c: "%s-%dbit-%dx%d" % c)
def test_gpu_postfilter_large(case):
    lay, bpc, W, H = case
    assert ((H + 3) // 4) & 1 and last_stripe_rows(make_lr_case(lay, bpc, W, H, (7, 6), 7, 0, seed=0), 0) < 8
    S = make_cdef_case(lay, bpc, W, H, 3 + W % 4, seed=1800 + W)
    cdef_counts()
    check_cdef(S, True, reference=True)
    counts = cdef_counts()
    assert not cdef_below_floor(S, counts), counts
    S = make_lr_case(lay, bpc, W, H, (7, 6), 7, 0, seed=1900 + W)
    lr_counts()
    check_lr(S, True, reference=True)
    counts = lr_counts()
    if bpc != 12:
        for c in counts:
            c["sgr_big"] = LR_FLOOR["sgr_big"]
    assert not lr_geometry_mismatch(S, counts) and not lr_below_floor(counts), counts


@pytest.mark.gpu
def test_gpu_band_seams():
    for case in BAND_CASES:
        check_bands(band_frame(*case), True)
