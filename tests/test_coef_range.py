"""Inverse transforms at the edges of the legal coefficient range, on every transform path.

dav1d clamps dequantised coefficients to cf_max = ~(~127U << bpc) (reference src/recon_tmpl.c:599): [-32768, 32767] at 8 bit,
[-131072, 131071] at 10 bit and [-524288, 524287] at 12 bit. At that scale the intermediate clips of the 2-D transform
(src/itx_tmpl.c:77-113: the row clip, then the column clip after the first pass) decide the result, and a narrow store or a
missing clip shows. The checkasm-style blocks of test_itx and the Laplace residuals of synth stay far below it, and synth
never draws the 1-D transform classes (V_* / H_*) or lossless WHT_WHT for a frame job or an intra kernel.

Here every coefficient block is a hard one (hard_block): saturated blocks of either sign, alternating signs, a single extreme
coefficient (DC-only blocks among them), uniform values over the whole range, and for identity first passes the value whose
first pass lands exactly on the column clip. Frame jobs and intra frames get such blocks with transform types drawn from
dav1d's transform sets (legal_txtps), so every case is one a stream can produce.

  not gpu : the oracle against the unmodified reference C path (oracle/_ref); the CUDA sources on the host emulator
            against the oracle: the Level-1 table, the Level-2 batches, frame jobs (dense and compact upload, whole
            frame and 64-row bands, post filters on) and the three intra kernels
  gpu     : the same paths at real frame sizes
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import refs
from dav1d_b200 import _lib, frame, synth
from dav1d_b200 import levels as L
import test_frame as TF
import test_intra as TI
import test_itx as TX


def cf_max(bpc):
    """largest dequantised coefficient magnitude dav1d hands the transforms (reference src/recon_tmpl.c:599)"""
    return ~(~127 << bpc)


def col_clip(bpc):
    """(col_lo, col_hi): the clip of the first pass's output (reference src/itx_tmpl.c:76-84)"""
    lo = -32768 if bpc == 8 else (~((1 << bpc) - 1)) << 5
    return lo, ~lo


# ------------------------------------------------------------------------------------------ transform sets
_INTRA2 = [L.IDTX, L.DCT_DCT, L.ADST_ADST, L.ADST_DCT, L.DCT_ADST]
_INTRA1 = _INTRA2 + [L.V_DCT, L.H_DCT]
_INTER2 = [L.IDTX, L.V_DCT, L.H_DCT] + list(range(L.IDTX))
_INTER1 = list(range(L.N_TX_TYPES))
_UV_INTRA = [L.DCT_DCT, L.ADST_DCT, L.DCT_ADST, L.ADST_ADST]


def legal_txtps(tx, inter, chroma=False, lossless=False):
    """The transform types a stream can give a block of size tx: dav1d's decode_coefs (reference src/recon_tmpl.c:351-401),
    with the sets of src/tables.c dav1d_tx_types_per_set, chroma of intra blocks from dav1d_txtp_from_uvmode and chroma of
    inter blocks from get_uv_inter_txtp (src/env.h:120-133), which never leaves the luma set of its size.
      lossless            : WHT_WHT, 4x4 only
      longest side 64     : DCT_DCT
      longest side 32     : DCT_DCT (intra), DCT_DCT / IDTX (inter, residual-only and intra block copy records)
      intra, shortest 16  : IDTX and the DCT / ADST pairs; V_DCT / H_DCT only when the shortest side is <= 8
      inter, shortest 16  : every 2-D type, IDTX, V_DCT, H_DCT; all 16 types when the shortest side is <= 8"""
    if lossless:
        return [L.WHT_WHT] if tx == L.TX_4X4 else []
    mx, mn = max(L.TX_W[tx], L.TX_H[tx]), min(L.TX_W[tx], L.TX_H[tx])
    if mx == 64 or (mx == 32 and not inter):
        return [L.DCT_DCT]
    if mx == 32:
        return [L.DCT_DCT, L.IDTX]
    if not inter:
        return list(_UV_INTRA) if chroma else list(_INTRA2 if mn == 16 else _INTRA1)
    return list(_INTER2 if mn == 16 else _INTER1)


def test_legal_txtps_are_defined_slots():
    for tx in range(L.N_RECT_TX_SIZES):
        for inter in (False, True):
            for chroma in (False, True):
                tps = legal_txtps(tx, inter, chroma)
                assert tps and all(L.itx_defined(tx, tp) for tp in tps), (tx, inter, chroma)
    assert legal_txtps(L.TX_4X4, True, lossless=True) == [L.WHT_WHT] and not legal_txtps(L.TX_8X8, True, lossless=True)
    # every defined slot but WHT_WHT is reachable from some inter block
    assert {(tx, tp) for tx in range(19) for tp in legal_txtps(tx, True)} == \
        {(tx, tp) for tx in range(19) for tp in range(16) if L.itx_defined(tx, tp)}


# ------------------------------------------------------------------------------------------ hard coefficient blocks
_SHIFT = {(4, 4): 0, (4, 8): 0, (4, 16): 1, (8, 4): 0, (8, 8): 1, (8, 16): 1, (8, 32): 2, (16, 4): 1, (16, 8): 1, (16, 16): 2,
          (16, 32): 1, (16, 64): 2, (32, 8): 2, (32, 16): 1, (32, 32): 2, (32, 64): 1, (64, 16): 2, (64, 32): 1, (64, 64): 2}
_FIRST_IDENTITY = (L.IDTX, L.V_DCT, L.V_ADST, L.V_FLIPADST)       # the row (first) pass is the identity
KINDS = ("max", "min", "alt", "single", "uniform", "edge")


def scan_order(tx, txtp):
    """coefficient index (layout cf[y + x * sh]) of scan position k, as decode_coefs walks it (reference
    src/recon_tmpl.c:458-467, 548-576): dav1d_scans for the 2-D classes, rc = k for TX_CLASS_H, x * sh + y for TX_CLASS_V"""
    sw, sh = L.tx_coef_dims(tx)
    k = np.arange(sw * sh)
    cls = refs.tx_class(txtp)
    if txtp == L.WHT_WHT or cls == refs._TX_CLASS_2D:
        return synth.scan_table(tx)
    if cls == refs._TX_CLASS_H:
        return k
    return (k % sw) * sh + k // sw


def first_pass_identity(v, tx):
    """output of the first pass of an identity row for a row of coefficients all equal to v, before the column clip
    (reference src/itx_tmpl.c:96-110, src/itx_1d.c identity)"""
    w, h = L.TX_W[tx], L.TX_H[tx]
    if w * 2 == h or h * 2 == w:
        v = (v * 181 + 128) >> 8
    if w == 4:
        v = v + ((v * 1697 + 2048) >> 12)
    elif w == 8:
        v = v * 2
    elif w == 16:
        v = 2 * v + ((v * 1697 + 1024) >> 11)
    else:
        v = v * 4
    s = _SHIFT[(w, h)]
    return (v + ((1 << s) >> 1)) >> s


def edge_values(tx, bpc):
    """(v_hi, v_lo): the smallest coefficient whose identity first pass reaches col_hi and the largest that reaches col_lo,
    within the legal range (the range end where the column clip is out of reach)"""
    hi, lo = cf_max(bpc), -cf_max(bpc) - 1
    col_lo, col_hi = col_clip(bpc)
    a, b = 0, hi                            # smallest v in [a, b] with f(v) >= col_hi
    if first_pass_identity(hi, tx) < col_hi:
        v_hi = hi
    else:
        while a < b:
            m = (a + b) // 2
            a, b = (m + 1, b) if first_pass_identity(m, tx) < col_hi else (a, m)
        v_hi = a
    a, b = lo, 0                            # largest v in [a, b] with f(v) <= col_lo
    if first_pass_identity(lo, tx) > col_lo:
        v_lo = lo
    else:
        while a < b:
            m = (a + b + 1) // 2
            a, b = (a, m - 1) if first_pass_identity(m, tx) > col_lo else (m, b)
        v_lo = a
    return v_hi, v_lo


def kinds_for(txtp):
    return KINDS if txtp in _FIRST_IDENTITY else KINDS[:-1]


def hard_block(rng, tx, txtp, bpc, kind):
    """(coef[sw * sh] in the layout itxfm_add reads, eob): a block dav1d's coefficient decoder can hand the transforms, with
    every coefficient past eob (in the scan order of its class) zero and the one at eob non-zero
      max / min : every coefficient up to eob at +cf_max / -(cf_max + 1)
      alt       : +cf_max / -(cf_max + 1) in a checkerboard (the largest DCT and ADST outputs)
      single    : one extreme coefficient at eob (DC-only blocks among them)
      uniform   : uniform over the legal range, eob drawn like checkasm's sub-block classes (tests/checkasm/itx.c:252)
      edge      : (identity first passes) the values whose first pass lands exactly on col_hi / col_lo"""
    sw, sh = L.tx_coef_dims(tx)
    n = sw * sh
    order = scan_order(tx, txtp)
    hi, lo = cf_max(bpc), -cf_max(bpc) - 1
    c = np.zeros(n, np.int64)
    if kind == "single":
        eob = 0 if txtp == L.DCT_DCT and rng.random() < 0.4 else int(rng.integers(0, n))
        c[order[eob]] = hi if rng.random() < 0.5 else lo
        return c, eob
    if kind == "uniform":
        w, h = L.TX_W[tx], L.TX_H[tx]
        smax = refs.SUBSH_ITERS[int(np.log2(max(w, h))) - 2]
        _, eob = refs.gen_itx_coefs(rng, tx, txtp, int(rng.integers(1 if txtp else 0, smax)), (1 << bpc) - 1)
        c[order[:eob + 1]] = rng.integers(lo, hi + 1, eob + 1)
    else:
        eob = n - 1 if rng.random() < 0.5 else int(rng.integers(0, n))
        idx = order[:eob + 1]
        if kind == "max":
            c[idx] = hi
        elif kind == "min":
            c[idx] = lo
        elif kind == "alt":
            c[idx] = np.where(((idx % sh) + (idx // sh)) & 1, lo, hi)
        else:
            assert kind == "edge" and txtp in _FIRST_IDENTITY
            v_hi, v_lo = edge_values(tx, bpc)
            c[idx] = v_hi if rng.random() < 0.5 else v_lo
    if c[order[eob]] == 0:
        c[order[eob]] = 1
    return c, eob


def test_hard_blocks_reach_the_clips():
    """the generator does what it claims: eob contract, legal range, identity first passes on the column clip"""
    rng = np.random.default_rng(1)
    for bpc in (8, 10, 12):
        hi = cf_max(bpc)
        col_lo, col_hi = col_clip(bpc)
        for tx in range(L.N_RECT_TX_SIZES):
            for tp in range(L.N_TX_TYPES_PLUS_LL):
                if not L.itx_defined(tx, tp):
                    continue
                order = scan_order(tx, tp)
                assert sorted(order.tolist()) == list(range(len(order)))
                for kind in kinds_for(tp):
                    c, eob = hard_block(rng, tx, tp, bpc, kind)
                    assert c.min() >= -hi - 1 and c.max() <= hi and c[order[eob]] != 0
                    assert not c[order[eob + 1:]].any()
                if tp in _FIRST_IDENTITY:
                    v_hi, v_lo = edge_values(tx, bpc)
                    assert first_pass_identity(v_hi, tx) >= col_hi or v_hi == hi
                    assert first_pass_identity(v_hi - 1, tx) < col_hi
                    assert first_pass_identity(v_lo, tx) <= col_lo or v_lo == -hi - 1
                    assert first_pass_identity(v_lo + 1, tx) > col_lo
    # the worked case: 12-bit 32x32 IDTX saturates the first pass at col_hi = 131071
    assert col_clip(12) == (-131072, 131071) and first_pass_identity(cf_max(12), L.TX_32X32) > 131071
    assert col_clip(10) == col_clip(8) == (-32768, 32767)


# ------------------------------------------------------------------------------------------ Level-1 table
def hard_slots(bpc_list=(8, 10, 12)):
    for bpc in bpc_list:
        for tx in range(L.N_RECT_TX_SIZES):
            for tp in range(L.N_TX_TYPES_PLUS_LL):
                if L.itx_defined(tx, tp):
                    for kind in kinds_for(tp):
                        yield bpc, tx, tp, kind


def run_hard_itx(new_tbls, chk_tbls, cases, seed, neg_stride_every=7):
    """test_itx.run_checkasm_itx with hard blocks: destination rectangle with padding guards and the coefficient buffer
    after the call (the zeroing contract) must both be identical"""
    rng = np.random.default_rng(seed)
    PAD = TX.PAD
    n = 0
    for bpc, tx, tp, kind in cases:
        bdmax = (1 << bpc) - 1
        w, h = L.TX_W[tx], L.TX_H[tx]
        coef, eob = hard_block(rng, tx, tp, bpc, kind)
        cbuf = rng.integers(-32768, 32767, 32 * 32).astype(refs.coef_dtype(bpc))
        cbuf[:len(coef)] = coef.astype(refs.coef_dtype(bpc))
        # pictures at both ends of the range: a saturated residual clips to 0 / bdmax
        canvas = rng.choice(np.array([0, 1, bdmax - 1, bdmax, bdmax // 2]), (h + 2 * PAD, w + 2 * PAD)) if n % 2 else \
            rng.integers(0, bdmax + 1, (h + 2 * PAD, w + 2 * PAD))
        canvas = canvas.astype(refs.pixel_dtype(bpc))
        c_chk, c_new = canvas.copy(), canvas.copy()
        k_chk, k_new = cbuf.copy(), cbuf.copy()
        n += 1
        if n % neg_stride_every == 0:
            d_chk, d_new = c_chk[PAD + h - 1:, PAD:], c_new[PAD + h - 1:, PAD:]
            stride = -canvas.strides[0]
        else:
            d_chk, d_new = c_chk[PAD:, PAD:], c_new[PAD:, PAD:]
            stride = canvas.strides[0]
        chk_tbls[bpc][tx][tp](d_chk, stride, k_chk, eob)
        new_tbls[bpc][tx][tp](d_new, stride, k_new, eob)
        what = "%dbpc %s %s %s eob=%d" % (bpc, L.TX_NAMES[tx], L.TXTP_NAMES[tp], kind, eob)
        if not np.array_equal(c_chk, c_new):
            ys, xs = np.nonzero(c_chk != c_new)
            raise AssertionError("dst mismatch: %s at (%d, %d): expected %d got %d (%d pixels)" % (
                what, ys[0] - PAD, xs[0] - PAD, c_chk[ys[0], xs[0]], c_new[ys[0], xs[0]], len(ys)))
        assert np.array_equal(k_chk, k_new), "coef (zeroing contract) mismatch: " + what
    return n


@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_oracle_vs_reference_hard_blocks(bpc):
    """pins the oracle at the extremes: every defined (tx, txtp) slot, every kind of hard block"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    n = run_hard_itx({bpc: refs.oracle_itxfm_add(bpc)}, {bpc: refs.ref_itx_table(bpc)}, list(hard_slots((bpc,))) * 3,
                     seed=300 + bpc)
    assert n == 3 * (156 * 5 + 39)             # the 39 IDTX / V_* slots also get the edge kind


@pytest.mark.parametrize("bpc", [10])
def test_oracle_vs_reference_garbage_10bit(bpc):
    """test_itx's out-of-contract check (full-range coefficients everywhere, arbitrary eob) at 10 bit"""
    if not refs.have_ref():
        pytest.skip("reference build (oracle/_ref) not present")
    rng = np.random.default_rng(7 + bpc)
    bdmax = (1 << bpc) - 1
    rt, ot = refs.ref_itx_table(bpc), refs.oracle_itxfm_add(bpc)
    amp = cf_max(bpc) + 1
    for tx in range(19):
        w, h = L.TX_W[tx], L.TX_H[tx]
        sw, sh = L.tx_coef_dims(tx)
        for tp in range(17):
            if not L.itx_defined(tx, tp):
                continue
            for it in range(6):
                cf = rng.integers(-amp, amp + 1, sw * sh).astype(refs.coef_dtype(bpc))
                eob = int(rng.integers(0, sw * sh))
                dst = rng.integers(0, bdmax + 1, (h, w)).astype(refs.pixel_dtype(bpc))
                d1, d2, c1, c2 = dst.copy(), dst.copy(), cf.copy(), cf.copy()
                rt[tx][tp](d1, d1.strides[0], c1, eob)
                ot[tx][tp](d2, d2.strides[0], c2, eob)
                assert np.array_equal(d1, d2) and np.array_equal(c1, c2), (bpc, tx, tp, eob)


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_itx_level1_hard_blocks(bpc):
    from dav1d_b200.dsp import InvTxfmDSPContext
    new = {bpc: InvTxfmDSPContext(bpc, lib=refs.emu_lib()).itxfm_add}
    run_hard_itx(new, {bpc: refs.oracle_itxfm_add(bpc)}, list(hard_slots((bpc,))), seed=310 + bpc)


@pytest.mark.gpu
def test_gpu_itx_level1_hard_blocks():
    from dav1d_b200.dsp import InvTxfmDSPContext
    new = {bpc: InvTxfmDSPContext(bpc).itxfm_add for bpc in (8, 10, 12)}
    for name, chk in TX._checkers():
        run_hard_itx(new, chk, list(hard_slots()) * 4, seed=320)


# ------------------------------------------------------------------------------------------ Level-2 batches
def make_hard_batch(rng, bpc, tx, n):
    """test_itx.make_batch with every other block (in random positions) replaced by a hard block of a random defined type"""
    blocks, coefs, pic, stride = TX.make_batch(rng, bpc, tx, n)
    sw, sh = L.tx_coef_dims(tx)
    types = [tp for tp in range(17) if L.itx_defined(tx, tp)]
    bdmax = (1 << bpc) - 1
    for i in np.nonzero(rng.random(n) < 0.5)[0]:
        tp = types[int(rng.integers(0, len(types)))]
        kinds = kinds_for(tp)
        c, eob = hard_block(rng, tx, tp, bpc, kinds[int(rng.integers(0, len(kinds)))])
        off = int(blocks[i]["coef_off"])
        coefs[off:off + sw * sh] = c
        blocks[i]["eob"], blocks[i]["txtp"] = eob, tp
    # a third of the picture at the ends of the range
    m = rng.random(pic.shape) < 0.33
    pic[m] = rng.choice(np.array([0, bdmax], pic.dtype), int(m.sum()))
    return blocks, coefs, pic, stride


def check_hard_batches(lib, device, bpc, seed, n_small, n_large, host_path=True):
    import torch
    from dav1d_b200 import batch
    rng = np.random.default_rng(seed)
    bdmax = (1 << bpc) - 1
    for tx in range(19):
        n = n_large if max(L.TX_W[tx], L.TX_H[tx]) >= 32 else n_small
        blocks, coefs, pic, stride = make_hard_batch(rng, bpc, tx, n)
        exp_pic, exp_coef = pic.copy(), coefs.copy()
        st = (C.c_int32 * 3)(stride, stride, stride)
        assert refs.oracle().oracle_itx_add_batch(bdmax, tx, blocks.ctypes.data, n, exp_coef.ctypes.data,
                                                  exp_pic.ctypes.data, st, 1) == 0
        for zero in (1, 0):
            d_blocks = torch.from_numpy(blocks.view(np.uint8).copy()).to(device)
            d_coef = torch.from_numpy(coefs.copy()).to(device)
            d_pic = torch.from_numpy(pic.copy().view(np.int16 if bpc > 8 else np.uint8)).to(device)
            batch.itx_add_batch(bdmax, tx, d_blocks, d_coef, d_pic, [stride] * 3, zero_coefs=bool(zero),
                                stream=0 if device == "cpu" else None, lib=lib)
            if device != "cpu":
                torch.cuda.synchronize()
            got = d_pic.cpu().numpy().view(pic.dtype)
            if not np.array_equal(got, exp_pic):
                bad = int(np.nonzero((got != exp_pic).reshape(-1))[0][0])
                raise AssertionError("pic mismatch %dbpc tx=%s zero=%d at offset %d: expected %d got %d" % (
                    bpc, L.TX_NAMES[tx], zero, bad, exp_pic.reshape(-1)[bad], got.reshape(-1)[bad]))
            assert np.array_equal(d_coef.cpu().numpy(), exp_coef if zero else coefs), "coef mismatch tx=%s" % L.TX_NAMES[tx]
        if host_path:
            p2, c2 = pic.copy(), coefs.copy()
            batch.itx_add_batch_host(bdmax, tx, blocks, c2, p2, [stride] * 3, zero_coefs=True, lib=lib)
            assert np.array_equal(p2, exp_pic) and np.array_equal(c2, exp_coef), "host path tx=%s" % L.TX_NAMES[tx]


@pytest.mark.emu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_emu_itx_batch_hard_blocks(bpc):
    check_hard_batches(refs.emu_lib(), "cpu", bpc, 330 + bpc, 40, 12)


@pytest.mark.gpu
@pytest.mark.parametrize("bpc", [8, 10, 12])
def test_gpu_itx_batch_hard_blocks(bpc):
    check_hard_batches(None, "cuda", bpc, 340 + bpc, 1031, 257)


# ------------------------------------------------------------------------------------------ frames
INTRA_COPIES = ("intra_tx", "intra_tx_decode_order", "intra_tx_sb")


def harden(S, rng, share=0.5, force_idtx32=0.0):
    """A copy of frame S in which `share` of the coded transform blocks (inter records S["itx"][tx] and intra-machine records)
    carry hard blocks with a type from the block's transform set. Only coefficients, eob and txtp change, so wavefront order
    and band plan stay as synth made them. Residual-only records (RESID: inter-intra blends and intra block copies) are inter
    blocks; `force_idtx32` of them with a 32-sample side get IDTX."""
    S = dict(S)
    coefs = S["coefs"].copy()
    bpc = S["bpc"]
    stats = {"idtx32_resid": 0, "wht": 0, "1d": 0}

    def pick(tx, inter, chroma):
        tps = legal_txtps(tx, inter, chroma)
        one_d = [tp for tp in tps if tp > L.IDTX]
        if tx == L.TX_4X4 and rng.random() < 0.3:
            tp = L.WHT_WHT                                                  # a lossless block
        elif inter and max(L.TX_W[tx], L.TX_H[tx]) == 32 and rng.random() < force_idtx32:
            tp = L.IDTX
        elif one_d and rng.random() < 0.4:                                  # V_* / H_*: another coefficient order
            tp = one_d[int(rng.integers(0, len(one_d)))]
        else:
            tp = tps[int(rng.integers(0, len(tps)))]
        kinds = kinds_for(tp)
        c, eob = hard_block(rng, tx, tp, bpc, kinds[int(rng.integers(0, len(kinds)))])
        stats["wht"] += tp == L.WHT_WHT
        stats["1d"] += tp > L.IDTX and tp != L.WHT_WHT
        return c, eob, tp

    itx = {}
    for tx, a in S["itx"].items():
        a = a.copy()
        ncf = np.prod(L.tx_coef_dims(tx))
        for i in np.nonzero(rng.random(len(a)) < share)[0]:
            c, eob, tp = pick(tx, True, a["plane"][i] > 0)
            off = int(a["coef_off"][i])
            coefs[off:off + ncf] = c
            a["eob"][i], a["txtp"][i] = eob, tp
        itx[tx] = a
    S["itx"] = itx
    if S.get("intra_tx") is not None and len(S["intra_tx"]):
        src = S["intra_tx_decode_order"]
        new = {}
        for i in np.nonzero((src["eob"] >= 0) & (rng.random(len(src)) < share))[0]:
            r = src[i]
            tx = int(r["tx"])
            resid = int(r["mode"]) == synth.MODE_RESID
            c, eob, tp = pick(tx, resid, int(r["plane"]) > 0)
            off = int(r["coef_off"])
            coefs[off:off + len(c)] = c
            new[off] = (eob, tp)
            stats["idtx32_resid"] += resid and tp == L.IDTX and max(L.TX_W[tx], L.TX_H[tx]) == 32
        keys = np.array(sorted(new), np.int64)
        for name in INTRA_COPIES:
            if name not in S:
                continue
            t = S[name].copy()
            hit = (t["eob"] >= 0) & np.isin(t["coef_off"].astype(np.int64), keys)
            for j in np.nonzero(hit)[0]:
                t["eob"][j], t["txtp"][j] = new[int(t["coef_off"][j])]
            S[name] = t
    S["coefs"] = coefs
    S["hard_stats"] = stats
    return S


def check_hard_frame(S, kw, bands=(64,)):
    """frame job against the oracle: dense and compact upload, whole frame and bands, post filters on"""
    exp = TF.oracle_frame(S)
    fb = frame.FrameBuffers(S, **kw)
    fb.run()
    fb.alloc.sync()
    TF.check_frame(S, fb, exp)
    for compact in (True,):
        fb = frame.FrameBuffers(S, compact=compact, **kw)
        fb.run()
        fb.alloc.sync()
        TF.check_frame(S, fb, exp)
    for rows in bands:
        for compact in (False, True):
            fb = frame.FrameBuffers(S, band_rows=rows, compact=compact, **kw)
            assert fb.n_bands() == -(-S["H"] // rows)
            fb.run_bands()
            fb.alloc.sync()
            TF.check_frame(S, fb, exp)
    return exp


FRAME_EMU = [(8, 200, 136, 1, 1), (10, 200, 136, 1, 1), (12, 136, 136, 0, 0), (8, 200, 136, 1, 0)]


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", FRAME_EMU)
def test_emu_frame_hard_blocks(bpc, W, H, ssh, ssv):
    rng = np.random.default_rng(350 + bpc + W + 2 * ssv)
    S = harden(synth.make_inter_frame(rng, bpc, W, H, ssh, ssv, p_intra=0.2, film_grain=bpc > 8), rng)
    assert len(S["intra_tx"]) > 10 and S["hard_stats"]["1d"] > 5 and S["hard_stats"]["wht"] > 0, S["hard_stats"]
    check_hard_frame(S, dict(lib=refs.emu_lib(), alloc=frame.NumpyAlloc()))


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv", [(8, 1920, 1080, 1, 1), (12, 1288, 720, 0, 0), (10, 1280, 720, 1, 0)])
def test_gpu_frame_hard_blocks(bpc, W, H, ssh, ssv):
    rng = np.random.default_rng(360 + bpc + W)
    S = harden(synth.make_inter_frame(rng, bpc, W, H, ssh, ssv, p_intra=0.1, film_grain=bpc > 8), rng, share=0.3)
    check_hard_frame(S, {})


def test_compact_stream_round_trips_every_class():
    """the compact upload (coefficients 0 .. eob in the scan order of the block's class) expands back to the dense blocks"""
    rng = np.random.default_rng(370)
    S = harden(synth.make_inter_frame(rng, 8, 136, 72, p_intra=0.3), rng, share=0.8)
    assert S["hard_stats"]["1d"] > 5
    cc, ex = synth.compact_coefs(S)
    dense = np.zeros_like(S["coefs"])
    assert set(ex["tx_class"].tolist()) == {0, 1, 2}
    for r in ex:
        tx, eob = int(r["tx"]), int(r["eob"])
        order = scan_order(tx, (L.DCT_DCT, L.H_DCT, L.V_DCT)[int(r["tx_class"])])
        dense[int(r["dense_off"]) + order[:eob + 1]] = cc[int(r["compact_off"]):int(r["compact_off"]) + eob + 1]
    assert np.array_equal(dense, S["coefs"])


# ------------------------------------------------------------------------------------------ intra kernels
INTRA_EMU = [(8, 136, 136, 1, 1, 0.0), (10, 136, 136, 1, 1, 0.3), (12, 200, 264, 0, 0, 0.3), (12, 136, 136, 0, 0, 0.0),
             (8, 200, 136, 1, 0, 0.3)]


def hard_intra_frame(bpc, W, H, ssh, ssv, p_ibc, seed):
    rng = np.random.default_rng(seed)
    S = synth.make_intra_frame(rng, bpc, W, H, ssh, ssv, p_ibc=p_ibc)
    S = harden(S, rng, force_idtx32=0.8)
    if bpc == 12 and p_ibc:
        assert S["hard_stats"]["idtx32_resid"] > 0, "no 12-bit 32-sample IDTX residual"
    return S


def check_intra_kernels(lib, alloc, S, sb=True):
    """the superblock schedule orders a superblock after its left / top-left / top / top-right neighbours only
    (include/b200av1.h B200IntraSb), which does not cover synth's intra block copies from anywhere in the rows above:
    superblock mode runs on frames without them"""
    exp = TI.oracle_intra(S)
    runs = [dict(order="intra_tx"), dict(order="intra_tx_decode_order", compact=True)]
    if sb and not (S["intra_tx"]["mode"] == synth.MODE_IBC).any():
        runs += [dict(sb=True), dict(sb=True, compact=True)]
    for kw in runs:
        got = TI.run_lib(lib, alloc(), S, **kw)
        ok, where = TI.planes_equal(S, exp, got)
        assert ok, ("%dbpc %r: plane %d y %d x %d: expected %d got %d (%d pixels)" % ((S["bpc"], kw) + where[:3] + where[3:]))


@pytest.mark.emu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv,p_ibc", INTRA_EMU)
def test_emu_intra_hard_blocks(bpc, W, H, ssh, ssv, p_ibc):
    """the warp-per-block kernel (the default) and the superblock kernel"""
    S = hard_intra_frame(bpc, W, H, ssh, ssv, p_ibc, 380 + bpc + W)
    check_intra_kernels(refs.emu_lib(), frame.NumpyAlloc, S)


def check_cta_kernel():
    """the CTA-per-block kernel on the hard intra frames (run in a process started with B200_INTRA_CTA=1)"""
    for bpc, W, H, ssh, ssv, p_ibc in INTRA_EMU:
        S = hard_intra_frame(bpc, W, H, ssh, ssv, p_ibc, 380 + bpc + W)
        check_intra_kernels(refs.emu_lib(), frame.NumpyAlloc, S, sb=False)


@pytest.mark.emu
def test_emu_intra_cta_kernel_hard_blocks():
    """the CTA-per-block kernel is chosen once per process from B200_INTRA_CTA, so it is checked in a process of its own"""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_coef_range\n"
            "test_coef_range.check_cta_kernel()\n"
            "print('RESULT ok')\n") % (refs.ROOT, os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800,
                         env=dict(os.environ, B200_INTRA_CTA="1"))
    assert "RESULT ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize("bpc,W,H,ssh,ssv,p_ibc", [(8, 1920, 1080, 1, 1, 0.0), (12, 1288, 720, 0, 0, 0.3), (12, 1288, 720, 0, 0, 0.0),
                                                    (10, 1280, 720, 1, 0, 0.3)])
def test_gpu_intra_hard_blocks(bpc, W, H, ssh, ssv, p_ibc):
    S = hard_intra_frame(bpc, W, H, ssh, ssv, p_ibc, 390 + bpc + W)
    check_intra_kernels(_lib.get_lib(), lambda: None, S)
