"""The deblocking frame sweep (lf_cols_kernel / lf_rows_kernel behind b200_lf_frame and the band-sliced frame job) on
content that takes every filter branch, at picture sizes whose last 4x4 unit column and row are odd, and at band seams.

The pictures keep the transform tilings, masks and levels of synth.make_lf_frame, but every transform block is painted
with a flat DC value. Neighbouring DC values differ by geometric steps (scaled by 1 << (bpc - 8)), so the steps across
edges straddle the E / I thresholds. A share of blocks is textured (the narrow filter, with and without hev), a share
is flat at the edge but offset inside (flat8in without flat8out on 16-wide edges: the 16-to-8 fallthrough), and about
5 % each are pinned at 0 and at bitdepth_max, in clusters, with a checkerboard texture against the limit in some (the
narrow filter's output clipping). Blocks on the 128x128 area boundaries often get level 0, so the kernels' fallback to
the left / above level crosses areas in every level slot.

The oracle counts the edge lines that take each branch (oracle_lf_branch_counts); the CPU tests assert that every case
reaches every branch, that the oracle equals dav1d's own frame driver in both superblock walk orders, and the cases run
on the host emulator and the GPU against the oracle. Band seams: the deblocking stage of a frame job with no
reconstruction records (run_lf only) runs band by band through b200_frame_run_band.
"""
import ctypes as C
import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, synth
from test_loopfilter import lf_frame_struct

BRANCHES = ("fm_fail", "narrow_hev", "narrow", "flat6", "flat8", "flat8_of16", "flat16", "narrow_clip")
LAYOUTS = {"420": (1, 1), "422": (1, 0), "444": (0, 0), "400": (1, 1)}
# branches each plane class can take: chroma edges are 4 or 6 wide, luma edges 4, 8 or 16
LUMA_BRANCHES = ("fm_fail", "narrow_hev", "narrow", "flat8", "flat8_of16", "flat16", "narrow_clip")
CHROMA_BRANCHES = ("fm_fail", "narrow_hev", "narrow", "flat6", "narrow_clip")

# (W, H): w4 mod 32 = 1, 31, 18, 13; w4 / h4 odd / odd, odd / odd, even / even, odd / odd; 434 and 322 are not multiples of 4
GEOMS = [(516, 292), (508, 388), (456, 264), (434, 322)]
# every layout at every bit depth, the geometries and all eight sharpness values spread over them
CASES = [(lay, bpc, *GEOMS[(i + j) % 4], (3 * i + j) % 8, 1) for i, lay in enumerate(LAYOUTS) for j, bpc in enumerate((8, 10, 12))]
# luma deblocked, chroma not (level_u = level_v = 0); 4:0:0 is always so
CASES += [("420", 8, 516, 292, 5, 0), ("444", 10, 456, 264, 2, 0)]
# more frames with odd h4 where the chroma rows are subsampled or the units are narrow: the last chroma unit row and
# column are a small share of a frame, so one frame per layout could pass a clamp that drops them
ODD = [(lay, bpc, W, H, sharp, 1) for lay, bpc in (("420", 8), ("420", 10), ("422", 12), ("420", 12))
       for W, H, sharp in ((580, 324, 0), (428, 260, 6), (644, 228, 3))]


def case_id(c):
    return "%s-%dbit-%dx%d-sharp%d%s" % (c[0], c[1], c[2], c[3], c[4], "" if c[5] else "-luma_only")


def plane(S, pic, p):
    return pic[S["off"][p]:S["off"][p] + S["stride"][p] * S["rows"][p]].reshape(S["rows"][p], S["stride"][p])


def paint_plane(rng, dst, til, bpc, cell_units, pin=0.05, textured=0.3, framed=0.35):
    """Flat transform blocks with geometric DC steps, textured, framed and pinned blocks (see the module docstring).
    dst: the whole plane (rows x stride); blocks at the right and bottom edge run on past the unit grid unclipped."""
    bd, sc = (1 << bpc) - 1, 1 << (bpc - 8)
    bx, by, lw, lh = til
    ph4, pw4 = bx.shape
    key = by.astype(np.int64) * pw4 + bx
    uniq, inv = np.unique(key, return_inverse=True)
    n = len(uniq)
    ox, oy = (uniq % pw4).astype(np.int32), (uniq // pw4).astype(np.int32)
    first = np.unique(inv.reshape(-1), return_index=True)[1]        # one unit of each block
    bw, bh = 4 << lw.reshape(-1)[first].astype(np.int32), 4 << lh.reshape(-1)[first].astype(np.int32)
    # a gentle field (about 1.5 levels per unit at 8 bit) plus a geometric step of random sign per block; a tenth of the
    # field's nodes lie past 0 or bitdepth_max, so that whole regions sit at the clip limits
    g = rng.integers(bd * 3 // 10, bd * 7 // 10 + 1, (ph4 // 64 + 2, pw4 // 64 + 2)).astype(np.float64)
    ext = rng.random(g.shape)
    g[ext < 0.05] = -0.1 * bd
    g[ext > 0.95] = 1.1 * bd
    fy, fx = oy / 64.0, ox / 64.0
    iy, ix = fy.astype(np.int32), fx.astype(np.int32)
    ty, tx = fy - iy, fx - ix
    base = (1 - ty) * ((1 - tx) * g[iy, ix] + tx * g[iy, ix + 1]) + ty * ((1 - tx) * g[iy + 1, ix] + tx * g[iy + 1, ix + 1])
    u = rng.uniform(-1.5, 6.5, n)
    step = np.where(u < 0, 0, np.round(2.0 ** u)) * sc
    dc = np.clip(np.round(base) + np.where(rng.random(n) < 0.5, -step, step), 0, bd).astype(np.int32)
    # pinned blocks, in cells of twice the largest block so that pinned blocks meet pinned blocks; one cell of each at least
    cell = rng.random((ph4 // cell_units + 1, pw4 // cell_units + 1))
    cell.reshape(-1)[rng.choice(cell.size, 2, replace=False)] = (0, 1)
    cell = cell[oy // cell_units, ox // cell_units]
    dc[cell < pin] = 0
    dc[cell > 1 - pin] = bd
    side = np.where(dc == bd, -1, np.where(dc == 0, 1, 0)).astype(np.int32)
    tex = rng.random(n) < np.where(side != 0, 0.6, textured)
    amp = np.where(tex, rng.choice([1, 2, 3, 5], n) * sc, 0).astype(np.int32)
    # textured blocks at 0 / bitdepth_max: a checkerboard of the limit and a value 2 or 3 (x scale) inside the range;
    # where its p1 (or q1) sits at the limit and hev is off, the narrow filter's output p1 + g (q1 - g) overshoots it
    cb = np.where(side != 0, side * rng.choice([2, 3], n) * sc, 0).astype(np.int32)
    frm = ~tex & (bw >= 16) & (bh >= 16) & (rng.random(n) < framed)
    delta = np.where(frm, rng.choice([-4, -3, -2, 2, 3, 4], n) * sc, 0).astype(np.int32)
    rows, stride = dst.shape
    # block index of every sample: the unit map expanded 4x, replicated past the last unit row / column
    idx = np.repeat(np.repeat(inv.reshape(ph4, pw4).astype(np.int32), 4, 0), 4, 1)
    idx = np.pad(idx, ((0, rows - idx.shape[0]), (0, stride - idx.shape[1])), mode="edge")
    xs = np.arange(stride, dtype=np.int32)[None, :]
    for y0 in range(0, rows, 256):      # in strips: an 8K plane would otherwise need several GB of temporaries
        b = idx[y0:y0 + 256]
        ys = np.arange(y0, y0 + b.shape[0], dtype=np.int32)[:, None]
        rx, ry = xs - ox[b] * 4, ys - oy[b] * 4
        inside = (rx >= 4) & (rx < bw[b] - 4) & (ry >= 4) & (ry < bh[b] - 4)
        a = amp[b]
        noise = (rng.random(b.shape, np.float32) * (2 * a + 1)).astype(np.int32) - a
        noise = np.where(side[b] != 0, cb[b] * ((xs + ys) & 1), noise)
        dst[y0:y0 + b.shape[0]] = np.clip(dc[b] + noise + np.where(inside, delta[b], 0), 0, bd)


def zero_levels_on_area_edges(rng, S):
    """level 0 for about half of the blocks that start on a 128x128 area boundary, in every level slot, so the kernels'
    fallback to the left / above unit reads across the boundary"""
    lv = S["level"].reshape(S["h4"] + 32, S["b4_stride"], 4)
    for slot in range(4):
        til = S["til_y"] if slot < 2 else S["til_uv"]
        ssh, ssv = (0, 0) if slot < 2 else (S["ss_hor"], S["ss_ver"])
        bx, by = til[0], til[1]
        ph4, pw4 = bx.shape
        on = ((bx > 0) & (bx % (32 >> ssh) == 0)) | ((by > 0) & (by % (32 >> ssv) == 0))
        key = by.astype(np.int64) * pw4 + bx
        drop = rng.random(int(key.max()) + 1) < 0.6
        lv[:ph4, :pw4, slot][on & drop[key]] = 0


def make_case(lay, bpc, W, H, sharp, filter_uv, seed):
    ssh, ssv = LAYOUTS[lay]
    rng = np.random.default_rng(seed)
    S = synth.make_lf_frame(rng, bpc, W, H, ssh, ssv, sharp=sharp)
    if lay == "400":        # the hooks' device picture: two dummy 4:2:0 chroma planes at the luma stride
        st, rows = S["stride"][0], S["rows"][0]
        S["stride"], S["rows"] = [st, st, st], [rows, rows >> 1, rows >> 1]
        S["off"] = [0, st * rows, st * rows + st * (rows >> 1)]
        S["pic"] = np.zeros(S["off"][2] + st * (rows >> 1), S["pic"].dtype)
    for p in range(3):
        paint_plane(rng, plane(S, S["pic"], p), S["til_y"] if p == 0 else S["til_uv"], bpc, 32 if p == 0 else 16)
    zero_levels_on_area_edges(rng, S)
    S["filter_uv"] = int(filter_uv and lay != "400")
    S["sharp"] = sharp
    return S


def case_frame(c):
    return make_case(*c, seed=900 + sum(c[1:4]) + 10 * c[4] + 1000 * list(LAYOUTS).index(c[0]))


def lf_struct(S, pic_ptr, mask_ptr, level_ptr, sb128=0):
    fr = lf_frame_struct(S, pic_ptr, mask_ptr, level_ptr)
    fr.filter_uv = S["filter_uv"]
    fr.sb128 = sb128
    return fr


def run_oracle(S, masks=None):
    pic = S["pic"].copy()
    masks = S["masks"] if masks is None else masks
    refs.oracle().oracle_lf_frame(S["bd"], C.byref(lf_struct(S, pic.ctypes.data, masks.ctypes.data, S["level"].ctypes.data)))
    return pic


def branch_counts():
    """oracle counters since the last call: {(plane class, direction): {branch: lines}}"""
    out = np.zeros(2 * 2 * len(BRANCHES), np.int64)
    assert refs.oracle().oracle_lf_branch_counts(C.c_void_p(out.ctypes.data)) == len(BRANCHES)
    out = out.reshape(2, 2, len(BRANCHES))
    return {(pc, d): dict(zip(BRANCHES, map(int, out[pc, d]))) for pc in range(2) for d in range(2)}


def run_reference(S, sb128):
    pic = S["pic"].copy()
    masks = S["masks"].copy()     # the real driver patches masks at tile edges in place
    fr = lf_struct(S, pic.ctypes.data, masks.ctypes.data, S["level"].ctypes.data, sb128)
    (refs.ref().refdrv_lf_frame_8bpc if S["bpc"] == 8 else refs.ref().refdrv_lf_frame_16bpc)(S["bd"], C.byref(fr))
    return pic


class Device:
    """the picture, masks and levels of a case where the library reads them: host memory for the emulator, HBM for the GPU"""

    def __init__(self, S, gpu):
        self.S, self.gpu = S, gpu
        if gpu:
            import torch
            from dav1d_b200 import get_lib
            self.lib = get_lib()
            self.pic = torch.from_numpy(S["pic"].view(np.uint8).copy()).cuda()
            self.mask = torch.from_numpy(S["masks"].view(np.uint8).copy()).cuda()
            self.level = torch.from_numpy(S["level"].reshape(-1).copy()).cuda()
            ptrs = self.pic.data_ptr(), self.mask.data_ptr(), self.level.data_ptr()
        else:
            self.lib = refs.emu_lib()
            self.pic, self.mask, self.level = S["pic"].copy(), S["masks"], S["level"]
            ptrs = self.pic.ctypes.data, self.mask.ctypes.data, self.level.ctypes.data
        self.fr = lf_struct(S, *ptrs)

    def result(self):
        if not self.gpu:
            return self.pic
        import torch
        torch.cuda.synchronize()
        return self.pic.cpu().numpy().view(self.S["pic"].dtype)


def run_frame(S, gpu):
    d = Device(S, gpu)
    d.lib.check(d.lib.b200_lf_frame(S["bd"], C.byref(d.fr), None), "b200_lf_frame")
    return d.result()


def lf_job(d):
    job = _lib.FrameJob()           # no reconstruction records: band_recon enqueues nothing
    job.bitdepth_max, job.run_lf, job.lf = d.S["bd"], 1, d.fr
    return job


def band(y0, y1, last):
    b = _lib.FrameBand()
    b.y0, b.y1, b.last = y0, y1, last
    return b


def run_bands(S, gpu, band_rows):
    d = Device(S, gpu)
    job, H = lf_job(d), S["h4"] * 4
    for y0 in range(0, H, band_rows):
        y1 = min(y0 + band_rows, H)
        d.lib.check(d.lib.b200_frame_run_band(C.byref(job), C.byref(band(y0, y1, int(y1 == H))), None), "b200_frame_run_band")
    return d.result()


def chroma_untouched(S, got):
    return all(np.array_equal(plane(S, got, p), plane(S, S["pic"], p)) for p in (1, 2))


def check_case(S, got, exp):
    assert np.array_equal(got, exp), [(p, int((plane(S, got, p) != plane(S, exp, p)).sum())) for p in range(3)]
    if not S["filter_uv"]:
        assert chroma_untouched(S, got)


# ---------------------------------------------------------------------------------------- what the content reaches
# floors per plane class and direction, as a share of the edge lines tested (fm pass or fail); at least 1 line
FLOOR_SHARE = {"fm_fail": 0.05, "narrow_hev": 0.01, "narrow": 0.03, "flat6": 0.03, "flat8": 0.005, "flat8_of16": 0.003,
               "flat16": 0.005, "narrow_clip": 0.001}


def below_floor(counts, filter_uv):
    """[(plane class, direction, branch, lines, floor)] of the branches below their floor"""
    low = []
    for (pc, d), c in counts.items():
        lines = c["fm_fail"] + sum(c[b] for b in BRANCHES if b not in ("fm_fail", "narrow_clip"))
        if pc and not filter_uv:
            if lines:
                low.append((pc, d, "chroma filtered", lines, 0))
            continue
        for b in (CHROMA_BRANCHES if pc else LUMA_BRANCHES):
            floor = max(1, int(FLOOR_SHARE[b] * lines))
            if c[b] < floor:
                low.append((pc, d, b, c[b], floor))
    return low


def area_fallbacks(S):
    """per level slot: edges on a 128x128 area boundary whose unit has level 0 and whose neighbour across the edge
    (left for column edges, above for row edges) has a nonzero level"""
    lv = S["level"].reshape(S["h4"] + 32, S["b4_stride"], 4)
    out = []
    for slot in range(4):
        til = S["til_y"] if slot < 2 else S["til_uv"]
        ssh, ssv = (0, 0) if slot < 2 else (S["ss_hor"], S["ss_ver"])
        bx, by = til[0], til[1]
        ph4, pw4 = bx.shape
        L = lv[:ph4, :pw4, slot].astype(np.int32)
        xs, ys = np.arange(pw4)[None, :], np.arange(ph4)[:, None]
        n = 0
        if slot != 1:   # column edges: slot 0 and the chroma slots
            e = (bx == xs) & (xs > 0) & (xs % (32 >> ssh) == 0)
            n += int((e[:, 1:] & (L[:, 1:] == 0) & (L[:, :-1] != 0)).sum())
        if slot != 0:   # row edges: slot 1 and the chroma slots
            e = (by == ys) & (ys > 0) & (ys % (32 >> ssv) == 0)
            n += int((e[1:] & (L[1:] == 0) & (L[:-1] != 0)).sum())
        out.append(n)
    return out


@pytest.mark.parametrize("case", CASES + ODD, ids=case_id)
def test_content_reaches_every_branch(case):
    S = case_frame(case)
    branch_counts()
    run_oracle(S)
    counts = branch_counts()
    assert not below_floor(counts, S["filter_uv"]), (below_floor(counts, S["filter_uv"]), counts)
    fb = area_fallbacks(S)
    assert all(fb[:2]) and (all(fb[2:]) or not S["filter_uv"]), fb


def test_cases_cover_layouts_depths_sharpness_geometry():
    assert {(c[0], c[1]) for c in CASES} == {(lay, bpc) for lay in LAYOUTS for bpc in (8, 10, 12)}
    assert {c[4] for c in CASES} == set(range(8))
    w4s = {(W + 3) // 4 for _, _, W, _, _, _ in CASES}
    h4s = {(H + 3) // 4 for _, _, _, H, _, _ in CASES}
    assert {w % 32 for w in w4s} >= {1, 31} and len({w % 32 for w in w4s}) >= 3
    assert any(w & 1 for w in w4s) and any(not w & 1 for w in w4s) and any(h & 1 for h in h4s) and any(not h & 1 for h in h4s)
    assert any(W % 4 for _, _, W, _, _, _ in CASES)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_oracle_vs_reference_driver(case):
    """the oracle against dav1d's own dav1d_loopfilter_sbrow_cols / _rows on the same frame, in both walk orders"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    S = case_frame(case)
    exp = run_oracle(S)
    assert (exp != S["pic"]).mean() > 0.01
    for sb128 in (0, 1):
        assert np.array_equal(run_reference(S, sb128), exp), sb128
    if not S["filter_uv"]:
        assert chroma_untouched(S, exp)


@pytest.mark.emu
@pytest.mark.parametrize("case", CASES + ODD, ids=case_id)
def test_emu_lf_frame(case):
    S = case_frame(case)
    check_case(S, run_frame(S, False), run_oracle(S))


# ---------------------------------------------------------------------------------------- band seams
# (layout, bpc, W, H): h4 = 97 and 73, odd; bands end on 64-row multiples except the last
BAND_CASES = [("420", 8, 516, 388), ("422", 10, 644, 292), ("444", 12, 580, 388)]


def band_frame(lay, bpc, W, H):
    return make_case(lay, bpc, W, H, 0, 1, seed=960 + bpc + W)


def seam_flat16(S, out):
    """per band seam y (64, 128, ... inside the picture): luma columns whose row edge at y is 16 wide and where rows
    y - 6 / y - 5 changed in the row pass. Only the 16-wide flat filter of the edge at y writes there: a 16-wide edge
    has blocks at least 16 rows tall on both sides, and the row edges 16 rows up write rows <= y - 11."""
    rows_off = S["masks"].copy()
    rows_off["filter_y"][:, 1] = 0
    rows_off["filter_uv"][:, 1] = 0
    cols_only = plane(S, run_oracle(S, rows_off), 0)
    out = plane(S, out, 0)
    by, lh = S["til_y"][1], S["til_y"][3]
    res = []
    for y in range(64, S["h4"] * 4, 64):
        y4 = y // 4
        wd16 = (by[y4] == y4) & (np.minimum(lh[y4], lh[y4 - 1]) >= 2)
        x = np.nonzero(np.repeat(wd16, 4))[0]
        res.append(int(((out[y - 6, x] != cols_only[y - 6, x]) | (out[y - 5, x] != cols_only[y - 5, x])).sum()))
    return res


def check_bands(S, gpu):
    whole = run_frame(S, gpu)
    exp = run_oracle(S)
    assert np.array_equal(whole, exp)
    for rows in (64, 128, 192):
        got = run_bands(S, gpu, rows)
        assert np.array_equal(got, exp), (rows, [(p, int((plane(S, got, p) != plane(S, exp, p)).sum())) for p in range(3)])
    return exp


@pytest.mark.parametrize("case", BAND_CASES)
def test_band_seams_take_flat16(case):
    """the wide row filter really fires at every 64-row seam: band k's row pass rewrites band k - 1's bottom rows"""
    S = band_frame(*case)
    assert S["h4"] & 1
    assert min(seam_flat16(S, run_oracle(S))) >= 3, seam_flat16(S, run_oracle(S))


@pytest.mark.emu
@pytest.mark.parametrize("case", BAND_CASES)
def test_emu_band_seams(case):
    check_bands(band_frame(*case), False)


def check_bad_bands(S, gpu):
    d = Device(S, gpu)
    job, H = lf_job(d), S["h4"] * 4
    for y0, y1, last in ((0, 68, 0), (4, 64, 0), (64, 96, 0), (0, H - 4, 1), (32, H, 1)):
        assert d.lib.b200_frame_run_band(C.byref(job), C.byref(band(y0, y1, last)), None) == -2, (y0, y1, last)
        assert b"64-row aligned" in d.lib.b200_last_error()
    assert np.array_equal(d.result(), S["pic"])


@pytest.mark.emu
def test_emu_bad_band_bounds():
    check_bad_bands(band_frame(*BAND_CASES[0]), False)


# ---------------------------------------------------------------------------------------- H100
# 1080p, 4K, 8K 10-bit 4:2:0, 720p 12-bit 4:4:4 and 10-bit 4:2:2, each with odd h4 (heights 4 rows past the usual ones);
# 1918 is not a multiple of 4, 3836 gives w4 = 959 (mod 32 = 31), 1284 gives w4 mod 32 = 1
GPU_CASES = [("420", 8, 1918, 1084, 0, 1), ("420", 8, 3836, 2164, 4, 1), ("420", 10, 7680, 4324, 2, 1),
             ("444", 12, 1284, 724, 7, 1), ("422", 10, 1280, 724, 5, 1), ("400", 10, 1918, 1084, 3, 0),
             ("422", 8, 1284, 724, 6, 0)]
GPU_BANDS = [("420", 8, 1918, 1084), ("422", 10, 1280, 724), ("444", 12, 1284, 724)]


@pytest.mark.gpu
def test_gpu_lf_frame_cases():
    for case in CASES + ODD:
        S = case_frame(case)
        check_case(S, run_frame(S, True), run_oracle(S))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=case_id)
def test_gpu_lf_frame_large(case):
    S = case_frame(case)
    branch_counts()
    exp = run_oracle(S)
    counts = branch_counts()
    assert not below_floor(counts, S["filter_uv"]), counts
    if refs.have_ref():
        assert np.array_equal(run_reference(S, 1), exp)
    check_case(S, run_frame(S, True), exp)


@pytest.mark.gpu
def test_gpu_band_seams():
    for case in BAND_CASES + GPU_BANDS:
        S = band_frame(*case)
        exp = check_bands(S, True)
        assert min(seam_flat16(S, exp)) >= 3, case
    check_bad_bands(band_frame(*GPU_BANDS[0]), True)
