"""lr_frame_kernel's U / V pairs: where the chroma restoration units are 32 wide (4:2:0 and 4:2:2 here), one CTA restores
the U and the V tile at the same place, 128 threads each, with one barrier schedule whatever the two units' types.

The frames are test_postfilter_frame's LR content with the chroma units the stripes look up retyped so that the U / V
pairs take all 9 (U, V) combinations of none / Wiener / self-guided (parameter sets 0, 10 and 14 in turn). The widths
leave a last column tile narrower than 32 and the heights a short last stripe; restore_planes also leaves out U or V,
so that half copies its tile while the other restores. Checked on the host emulator and the GPU against the oracle,
and on the GPU against dav1d's driver where oracle/_ref exists.
"""
import numpy as np
import pytest

from dav1d_b200 import synth
import test_postfilter_frame as PF

KINDS = ("none", "wiener", "sgr")
SGR_TYPES = (3, 13, 17)           # 3 + parameter set: 0 (both passes), 10 (3x3 only), 14 (5x5 only)
COMBOS = [(a, b) for a in KINDS for b in KINDS]

# (layout, W, H): chroma 165 x 67 (last tile 5 wide, last stripe 7 rows) and 129 x 121 (last tile 1 wide, 1 row)
GEOMS = [("420", 330, 134), ("422", 258, 121)]
CASES = [(lay, bpc, W, H, rp) for lay, W, H in GEOMS for bpc in (8, 10) for rp in (7, 3, 5)]


def unit_type(kind, i):
    return {"none": 0, "wiener": 2, "sgr": SGR_TYPES[i % 3]}[kind]


def pair_frame(lay, bpc, W, H, rp):
    S = PF.make_lr_case(lay, bpc, W, H, (6, 5), rp, 0, seed=2100 + bpc + W + rp)
    u = S["lr_mask"]["lr"]
    units = PF.lr_units(S, 1)
    assert units == PF.lr_units(S, 2)
    rng = np.random.default_rng(2200 + W)
    for i, (mi, ui) in enumerate(dict.fromkeys(units)):
        cu, cv = COMBOS[i % len(COMBOS)]
        for p, kind in ((1, cu), (2, cv)):
            t = unit_type(kind, i + p)
            u["type"][mi, p, ui] = t
            if t >= 3:
                s0, s1 = synth.SGR_PARAMS[t - 3]
                u["sgr_weights"][mi, p, ui, 0] = rng.integers(-96, 32) if s0 else 0
                u["sgr_weights"][mi, p, ui, 1] = rng.integers(-32, 96) if s1 else 95
    return S


def case_id(c):
    return "%s-%dbit-%dx%d-rp%d" % c


def test_pair_cases_cover_types_edges_and_planes():
    seen, sgr = set(), set()
    for c in CASES:
        S = pair_frame(*c)
        t = S["lr_mask"]["lr"]["type"]
        for mi, ui in PF.lr_units(S, 1):
            kinds = tuple("none" if v == 0 else "wiener" if v == 2 else "sgr" for v in (t[mi, 1, ui], t[mi, 2, ui]))
            seen.add(kinds)
            sgr |= {int(v) for v in (t[mi, 1, ui], t[mi, 2, ui]) if v >= 3}
        w, h = PF.plane_dims(S, 1)
        assert w % 32 and PF.last_stripe_rows(S, 1) < 8, c
    assert seen == set(COMBOS) and sgr == set(SGR_TYPES)
    assert {c[4] for c in CASES} == {7, 3, 5} and {c[1] for c in CASES} == {8, 10}


@pytest.mark.emu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_emu_lr_pairs(case):
    PF.check_lr(pair_frame(*case), False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_lr_pairs(case):
    PF.check_lr(pair_frame(*case), True, reference=True)
