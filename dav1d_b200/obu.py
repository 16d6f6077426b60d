"""Synthetic AV1 elementary streams (low-overhead OBU format, AV1 spec section 5) for driving a real dav1d
front end: hand-written sequence / frame headers in front of tile payloads of random bytes.

There is no AV1 encoder in this environment. An AV1 tile payload is one arithmetic-coded symbol stream, and
every byte string decodes to *some* legal symbol sequence, so random tile bytes behind valid headers give
frames that exercise the whole block layer of the decoder (partitions, every intra mode, directional deltas,
filter-intra, CFL, transform sizes / types, coefficient magnitudes up to the clipping range, per-block
delta-q / delta-lf, CDEF indices, loop-restoration units) with the contexts and CDF adaptation of a real
stream. The header syntax follows the order in which the reference parses it (reference src/obu.c:
parse_seq_hdr :71-307, parse_frame_hdr :399-1164, parse_tile_hdr :1166-1180; tile size bytes src/decode.c,
dav1d_decode_frame_init_cdf).

Used by tests/test_stream.py and bench.py's `stream` workloads; not a general AV1 muxer."""
import numpy as np


class BitWriter:
    def __init__(self):
        self.bits = []

    def f(self, n, v):
        v = int(v)
        assert 0 <= v < (1 << n), (n, v)
        for i in range(n - 1, -1, -1):
            self.bits.append((v >> i) & 1)

    def su(self, n, v):                      # signed, n bits two's complement (dav1d_get_sbits)
        self.f(n, v & ((1 << n) - 1))

    def align(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def trailing(self):                      # trailing_bits(): a one, then zeros up to the byte boundary
        self.bits.append(1)
        self.align()

    def bytes(self):
        assert len(self.bits) % 8 == 0
        a = np.array(self.bits, np.uint8).reshape(-1, 8)
        return bytes(np.packbits(a, axis=1).reshape(-1))


def leb128(v):
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def obu(obu_type, payload):
    # obu_header: forbidden 0 | type(4) | extension 0 | has_size_field 1 | reserved 0
    return bytes([(obu_type << 3) | 2]) + leb128(len(payload)) + payload


OBU_SEQ_HDR, OBU_TD, OBU_FRAME_HDR, OBU_METADATA, OBU_FRAME = 1, 2, 3, 5, 6
METADATA_HDR_CLL, METADATA_HDR_MDCV = 1, 2


# 4:2:2 (layout="422") is expressible in the headers below, but random tile payloads are only sometimes legal 4:2:2 streams:
# partitions whose chroma blocks would be 2 samples wide are forbidden there and the decoder rejects them (reference
# src/decode.c, decode_sb). Small frames (a few superblocks) pass for a good share of the seeds: callers draw seeds until
# the stock decoder accepts the stream (tests/test_stream.py::_valid_422).
def _profile(bpc, layout):
    """seq_profile for a bit depth / chroma layout: 0 = 4:2:0 (and 4:0:0) 8 / 10 bit, 1 = 4:4:4 8 / 10 bit, 2 = 4:2:2 and everything 12 bit"""
    if bpc == 12 or layout == "422":
        return 2
    return 1 if layout == "444" else 0


def sequence_header(w, h, bpc=8, sb128=0, film_grain=0, filter_intra=1, intra_edge_filter=1, cdef=1, restoration=1,
                    inter_intra=1, masked_compound=1, warped_motion=1, screen_content=0, layout="420", super_res=0,
                    chroma_sample_position=0, color=None):
    """chroma_sample_position (4:2:0 only): enum Dav1dChromaSamplePosition, 0 unknown, 1 vertical, 2 colocated;
    color = (matrix_coefficients, color_range): a colour description with BT.709 primaries and transfer (matrix 0, identity,
    is not supported here), or (matrix_coefficients, color_range, color_primaries, transfer_characteristics); None writes
    none and limited range"""
    b = BitWriter()
    profile = _profile(bpc, layout)
    b.f(3, profile)
    b.f(1, 0); b.f(1, 0)                     # still_picture, reduced_still_picture_header
    b.f(1, 0)                                # timing_info_present
    b.f(1, 0)                                # initial_display_delay_present
    b.f(5, 0)                                # operating_points_cnt_minus_1
    b.f(12, 0)                               # operating_point_idc
    b.f(3, 3); b.f(2, 1)                     # seq_level_idx (major 5, minor 1)
    b.f(1, 0)                                # seq_tier (major level > 3)
    wn, hn = max(1, int(w - 1).bit_length()), max(1, int(h - 1).bit_length())
    b.f(4, wn - 1); b.f(4, hn - 1)
    b.f(wn, w - 1); b.f(hn, h - 1)
    b.f(1, 0)                                # frame_id_numbers_present
    b.f(1, sb128); b.f(1, filter_intra); b.f(1, intra_edge_filter)
    b.f(1, inter_intra); b.f(1, masked_compound); b.f(1, warped_motion); b.f(1, 1)   # ..., dual filter
    b.f(1, 1)                                # enable_order_hint
    b.f(1, 1); b.f(1, 0)                     # jnt_comp, ref_frame_mvs
    b.f(1, 0); b.f(1, screen_content)        # seq_choose_screen_content_tools = 0, seq_force_screen_content_tools
    if screen_content:
        b.f(1, 0); b.f(1, 0)                 # seq_choose_integer_mv = 0, seq_force_integer_mv = 0
    b.f(3, 6)                                # order_hint_bits_minus_1
    b.f(1, super_res); b.f(1, cdef); b.f(1, restoration)   # superres, cdef, restoration
    b.f(1, 1 if bpc > 8 else 0)              # high_bitdepth
    if profile == 2 and bpc > 8:
        b.f(1, 1 if bpc == 12 else 0)        # twelve_bit
    mono = layout == "400"
    if profile != 1:
        b.f(1, 1 if mono else 0)             # mono_chrome
    b.f(1, color is not None)                # color_description_present
    if color is not None:
        assert color[0] != 0, "identity matrix_coefficients need the sRGB special case"
        pri, trc = color[2:4] if len(color) == 4 else (1, 1)
        b.f(8, pri); b.f(8, trc); b.f(8, color[0])   # color_primaries, transfer_characteristics, matrix_coefficients
    b.f(1, color[1] if color is not None else 0)  # color_range
    if not mono:
        if profile == 2 and bpc == 12:       # explicit subsampling
            b.f(1, 0 if layout == "444" else 1)
            if layout != "444":
                b.f(1, 1 if layout == "420" else 0)
        if layout == "420":
            b.f(2, chroma_sample_position)   # chroma_sample_position
        b.f(1, 0)                            # separate_uv_delta_q
    b.f(1, film_grain)
    b.trailing()
    return obu(OBU_SEQ_HDR, b.bytes())


def _tile_log2(sz, tgt):
    k = 0
    while (sz << k) < tgt:
        k += 1
    return k


def _frame_common(b, rng, w, h, sb128, log2_cols, log2_rows, q, lf, cdef, restoration, delta_q, cdef_on, restoration_on, layout="420",
                  segmentation=0, intrabc=0):
    """tile info, quantizer, segmentation, delta q / lf, loop filter, CDEF, loop restoration (same syntax in key and
    inter frames when primary_ref_frame is NONE)"""
    # tile info (uniform)
    sbl = 6 + sb128
    sbw, sbh = (w + (1 << sbl) - 1) >> sbl, (h + (1 << sbl) - 1) >> sbl
    b.f(1, 1)
    min_cols = _tile_log2(4096 >> sbl, sbw)
    max_cols, max_rows = _tile_log2(1, min(sbw, 64)), _tile_log2(1, min(sbh, 64))
    min_tiles = max(_tile_log2(4096 * 2304 >> (2 * sbl), sbw * sbh), min_cols)
    log2_cols = min(max(log2_cols, min_cols), max_cols)
    for _ in range(min_cols, log2_cols):
        b.f(1, 1)
    if log2_cols < max_cols:
        b.f(1, 0)
    min_rows = max(min_tiles - log2_cols, 0)
    log2_rows = min(max(log2_rows, min_rows), max_rows)
    for _ in range(min_rows, log2_rows):
        b.f(1, 1)
    if log2_rows < max_rows:
        b.f(1, 0)
    tile_w = 1 + ((sbw - 1) >> log2_cols); cols = (sbw + tile_w - 1) // tile_w
    tile_h = 1 + ((sbh - 1) >> log2_rows); rows = (sbh + tile_h - 1) // tile_h
    if log2_cols or log2_rows:
        b.f(log2_cols + log2_rows, 0)        # context_update_tile_id
        b.f(2, 3)                            # tile_size_bytes_minus_1
    # quantizer
    q = int(rng.integers(40, 200)) if q is None else q
    b.f(8, q)
    mono = layout == "400"
    b.f(1, 0)                                # no y dc delta
    if not mono:
        b.f(1, 0); b.f(1, 0)                 # no u dc / u ac deltas
    b.f(1, 0)                                # using_qmatrix
    b.f(1, segmentation)                     # segmentation_enabled (primary_ref_frame NONE: map and data are always updated)
    if segmentation:
        for _ in range(8):
            # per segment: quantiser delta (may reach qidx 0 = lossless: 4x4 Walsh-Hadamard blocks, no filtering), four
            # loop-filter deltas, forced reference, forced skip, forced global motion
            if rng.random() < 0.5:
                b.f(1, 1); b.su(9, int(rng.choice([-q, int(rng.integers(-60, 61))])))
            else:
                b.f(1, 0)
            for _k in range(4):
                if rng.random() < 0.3:
                    b.f(1, 1); b.su(7, int(rng.integers(-30, 31)))
                else:
                    b.f(1, 0)
            if rng.random() < 0.2:
                b.f(1, 1); b.f(3, int(rng.integers(0, 8)))
            else:
                b.f(1, 0)
            b.f(1, int(rng.random() < 0.15))
            b.f(1, int(rng.random() < 0.15))
    if q:
        b.f(1, 1 if delta_q else 0)          # delta_q_present
        if delta_q:
            b.f(2, int(rng.integers(0, 4)))
            if not intrabc:
                b.f(1, 1); b.f(2, int(rng.integers(0, 4))); b.f(1, int(rng.integers(0, 2)))   # delta_lf present, res, multi
    # a frame that allows intra block copy carries no loop filter, CDEF or restoration parameters: the picture it copies
    # from is the unfiltered one, so the filters are off (reference src/obu.c:807, 835, 879, 895)
    if intrabc:
        return cols, rows, tile_w, tile_h, sbw, sbh
    # loop filter
    lf = [int(rng.integers(1, 64)), int(rng.integers(1, 64)), int(rng.integers(0, 64)), int(rng.integers(0, 64))] if lf is None else lf
    b.f(6, lf[0]); b.f(6, lf[1])
    if (lf[0] or lf[1]) and not mono:
        b.f(6, lf[2]); b.f(6, lf[3])
    b.f(3, int(rng.integers(0, 8)))          # sharpness
    b.f(1, 1); b.f(1, 0)                     # mode_ref_delta_enabled, no update
    if cdef_on:
        nb = int(rng.integers(0, 4)) if cdef else 0
        b.f(2, int(rng.integers(0, 4))); b.f(2, nb)
        for _ in range(1 << nb):
            b.f(6, int(rng.integers(0, 64)) if cdef else 0)
            if not mono:
                b.f(6, int(rng.integers(0, 64)) if cdef else 0)
    if restoration_on:
        types = [int(rng.integers(0, 4)) for _ in range(3)] if restoration else [0, 0, 0]
        if mono:
            types[1] = types[2] = 0
        for t in (types[:1] if mono else types):
            b.f(2, t)
        if any(types):
            if sb128:
                b.f(1, int(rng.integers(0, 2)))
            else:
                s = int(rng.integers(0, 2)); b.f(1, s)
                if s:
                    b.f(1, int(rng.integers(0, 2)))
            if (types[1] or types[2]) and layout == "420":
                b.f(1, int(rng.integers(0, 2)))
    return cols, rows, tile_w, tile_h, sbw, sbh


# stream generator (tests/streamgen.py): an iterator of tile payloads that replace the random ones (the random bytes are
# still drawn, so that every later header choice is the same as in the run that produced the payloads)
PAYLOADS = None


def _tile_group(b, rng, cols, rows, tile_w, tile_h, sbw, sbh, sb128, payload_bytes_per_sb64):
    b.align()
    n_tiles = cols * rows
    if n_tiles > 1:
        b.f(1, 0)                            # tile_start_and_end_present_flag
    b.align()
    out = bytearray(b.bytes())
    for t in range(n_tiles):
        tc, tr = t % cols, t // cols
        nsb = (min(sbw, (tc + 1) * tile_w) - tc * tile_w) * (min(sbh, (tr + 1) * tile_h) - tr * tile_h)
        n = max(64, (payload_bytes_per_sb64 << (2 * sb128)) * nsb)   # the symbol decoder must never run dry (src/decode.c:2743)
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        if PAYLOADS is not None:
            data = next(PAYLOADS)
        if t < n_tiles - 1:
            out += int(len(data) - 1).to_bytes(4, "little")
        out += data
    return bytes(out)


def key_frame(rng, w, h, sb128=0, log2_cols=0, log2_rows=0, payload_bytes_per_sb64=3000, q=None, lf=None, cdef=True,
              restoration=True, delta_q=True, cdef_on=1, restoration_on=1, film_grain_seq=0, screen_content=0, layout="420",
              intra_only=None, segmentation=0, super_res=0, intrabc=0):
    """One shown key frame (OBU_FRAME), or with intra_only=(order_hint, refresh_frame_flags) a shown INTRA_ONLY frame
    (intra coded, but it only replaces the reference slots it names). Returns the OBU bytes. `cdef_on` / `restoration_on` must match the sequence
    header (the fields are absent when the sequence disables the tool)."""
    b = BitWriter()
    b.f(1, 0)                                # show_existing_frame
    if intra_only is None:
        b.f(2, 0); b.f(1, 1)                 # frame_type KEY, show_frame
    else:
        b.f(2, 2); b.f(1, 1)                 # frame_type INTRA_ONLY, show_frame
        b.f(1, 0)                            # error_resilient_mode
    b.f(1, 0)                                # disable_cdf_update
    b.f(1, 0)                                # frame_size_override
    b.f(7, 0 if intra_only is None else intra_only[0])   # order_hint
    if intra_only is not None:
        b.f(8, intra_only[1])                # refresh_frame_flags (a shown key frame refreshes all slots implicitly)
    cw = w
    if super_res:
        cd = int(rng.integers(0, 8))
        b.f(1, 1); b.f(3, cd)                # use_superres, coded_denom: the frame is coded (cw wide) and upscaled to w after CDEF
        cw = (w * 8 + (9 + cd) // 2) // (9 + cd)
    b.f(1, 0)                                # render_and_frame_size_different
    intrabc = 1 if (intrabc and screen_content and not super_res) else 0
    if screen_content and not super_res:
        b.f(1, intrabc)                      # allow_intrabc
    b.f(1, 0)                                # disable_frame_end_update_cdf
    cols, rows, tile_w, tile_h, sbw, sbh = _frame_common(b, rng, cw, h, sb128, log2_cols, log2_rows, q, lf, cdef, restoration, delta_q, cdef_on, restoration_on, layout, segmentation, intrabc)
    b.f(1, 1)                                # tx_mode_select
    b.f(1, int(rng.integers(0, 2)))          # reduced_tx_set
    if film_grain_seq:
        _film_grain_params(b, rng, 0, layout)
    return obu(OBU_FRAME, _tile_group(b, rng, cols, rows, tile_w, tile_h, sbw, sbh, sb128, payload_bytes_per_sb64))


def metadata_hdr_cll(max_cll, max_fall):
    """OBU_METADATA of type HDR_CLL (AV1 spec 5.8.3): MaxCLL and MaxFALL in cd/m^2, for a temporal unit ahead of its frame"""
    b = BitWriter()
    b.f(16, max_cll); b.f(16, max_fall)
    b.trailing()
    return obu(OBU_METADATA, leb128(METADATA_HDR_CLL) + b.bytes())


def metadata_hdr_mdcv(max_luminance, min_luminance, primaries=((0.708, 0.292), (0.170, 0.797), (0.131, 0.046)),
                      white=(0.3127, 0.3290)):
    """OBU_METADATA of type HDR_MDCV (AV1 spec 5.8.4): the mastering display's max / min luminance in cd/m^2 (stored as
    24.8 / 18.14 fixed point), its primaries (R, G, B) and white point as CIE 1931 xy (0.16 fixed point)"""
    b = BitWriter()
    for x, y in list(primaries) + [white]:
        b.f(16, round(x * 65536)); b.f(16, round(y * 65536))
    b.f(32, round(max_luminance * 256)); b.f(32, round(min_luminance * 16384))
    b.trailing()
    return obu(OBU_METADATA, leb128(METADATA_HDR_MDCV) + b.bytes())


def temporal_unit(*obus):
    return obu(OBU_TD, b"") + b"".join(obus)


def intra_stream(seed, w, h, n_frames=1, bpc=8, sb128=0, log2_cols=0, log2_rows=0, film_grain=0, screen_content=0, layout="420",
                 super_res=0, chroma_sample_position=0, **kw):
    """A list of temporal units (bytes), each holding one shown key frame."""
    rng = np.random.default_rng(seed)
    seq = sequence_header(w, h, bpc=bpc, sb128=sb128, film_grain=film_grain, screen_content=screen_content, layout=layout, super_res=super_res,
                          chroma_sample_position=chroma_sample_position)
    kw = dict(kw, layout=layout, super_res=super_res)
    if film_grain:
        kw = dict(kw, film_grain_seq=1)
    if screen_content:
        kw = dict(kw, screen_content=1)
    tus = []
    for i in range(n_frames):
        fr = key_frame(rng, w, h, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows, **kw)
        tus.append(temporal_unit(seq, fr) if i == 0 else temporal_unit(fr))
    return tus


def _film_grain_params(b, rng, inter, layout="420"):
    """film_grain_params() with apply_grain = 1 and fresh parameters (reference src/obu.c:1064-1155): random scaling
    points, auto-regression lag 0..3 with random coefficients, overlap, optional chroma-from-luma scaling"""
    b.f(1, 1)                                # apply_grain
    b.f(16, int(rng.integers(0, 1 << 16)))   # grain_seed
    if inter:
        b.f(1, 1)                            # update_grain
    ny = int(rng.integers(0, 15))
    b.f(4, ny)
    xs = sorted(rng.choice(256, ny, replace=False).tolist())
    for x in xs:
        b.f(8, x); b.f(8, int(rng.integers(0, 256)))
    mono = layout == "400"
    csfl = 0 if mono else int(rng.integers(0, 2))
    if not mono:
        b.f(1, csfl)
    nuv = [0, 0]
    if not (mono or csfl or (layout == "420" and ny == 0)):   # 4:2:0 without luma points carries no chroma points either
        n = int(rng.integers(0, 11))
        nuv = [n, int(rng.integers(1, 11)) if n else 0] if layout == "420" else [n, int(rng.integers(0, 11))]   # 4:2:0: both or neither
        for pl in range(2):
            b.f(4, nuv[pl])
            for x in sorted(rng.choice(256, nuv[pl], replace=False).tolist()):
                b.f(8, x); b.f(8, int(rng.integers(0, 256)))
    b.f(2, int(rng.integers(0, 4)))          # grain_scaling_minus_8
    lag = int(rng.integers(0, 4))
    b.f(2, lag)
    npos = 2 * lag * (lag + 1)
    if ny:
        for _ in range(npos):
            b.f(8, int(rng.integers(0, 256)))
    for pl in range(2):
        if nuv[pl] or csfl:
            for _ in range(npos + (1 if ny else 0)):
                b.f(8, int(rng.integers(0, 256)))
    b.f(2, int(rng.integers(0, 4)))          # ar_coeff_shift_minus_6
    b.f(2, int(rng.integers(0, 4)))          # grain_scale_shift
    for pl in range(2):
        if nuv[pl]:
            b.f(8, int(rng.integers(0, 256))); b.f(8, int(rng.integers(0, 256))); b.f(9, int(rng.integers(0, 512)))
    b.f(1, int(rng.integers(0, 2)))          # overlap_flag
    b.f(1, int(rng.integers(0, 2)))          # clip_to_restricted_range


def _subexp_near_ref(b, rng, steps=2):
    """one dav1d_get_bits_subexp() field (reference src/getbits.c:139-164) whose decoded value is the prediction plus or
    minus a few units: `k` escape bits, a stop bit, then the 3 + max(k - 1, 0) literal bits of that bucket"""
    k = int(rng.integers(0, steps + 1))
    for _ in range(k):
        b.f(1, 1)
    b.f(1, 0)
    nb = 3 if k == 0 else 3 + k - 1
    b.f(nb, int(rng.integers(0, 1 << nb)))


def _global_motion_params(b, rng, hp):
    """global_motion_params() for the 7 references with primary_ref_frame = NONE (predictions = the default parameters,
    reference src/obu.c:1014-1060): a mix of identity, translation, rotation-zoom and affine models close to identity, so
    that the shear parameters are valid and GLOBALMV blocks are really warped"""
    for _ in range(7):
        kind = int(rng.integers(0, 4))           # 0 identity, 1 translation, 2 rot-zoom, 3 affine
        if kind == 0:
            b.f(1, 0); continue
        b.f(1, 1)
        if kind == 2:
            b.f(1, 1)
        else:
            b.f(1, 0); b.f(1, 1 if kind == 1 else 0)
        if kind >= 2:
            _subexp_near_ref(b, rng); _subexp_near_ref(b, rng)          # mat[2], mat[3]
            if kind == 3:
                _subexp_near_ref(b, rng); _subexp_near_ref(b, rng)      # mat[4], mat[5]
        _subexp_near_ref(b, rng, 3); _subexp_near_ref(b, rng, 3)        # mat[0], mat[1] (translation part)


def _poc_diff(bits, a, b):
    mask = 1 << (bits - 1)
    d = a - b
    return (d & (mask - 1)) - (d & mask)


def inter_frame(rng, w, h, order_hint, ref_hints, sb128=0, log2_cols=0, log2_rows=0, payload_bytes_per_sb64=3000, q=None,
                lf=None, cdef=True, restoration=True, delta_q=True, cdef_on=1, restoration_on=1, film_grain_seq=0,
                refresh=None, switchable_motion_mode=0, warped_motion_seq=0, comp_refs=1, allow_warped_motion=0, layout="420",
                show_frame=1, global_motion=0, segmentation=0, max_size=None, super_res=0):
    """One shown inter frame (OBU_FRAME), primary_ref_frame = NONE. `ref_hints` = order hints held by the 8 reference slots
    (updated in place for the slots this frame refreshes). Global motion is identity. max_size = (W, H) of the sequence
    header when this frame is coded at another size (w, h): frame_size_override with an explicit size, so that its references
    — decoded at other sizes — are scaled references (reference src/obu.c read_frame_size, src/recon_tmpl.c:991-1046)."""
    bits = 7
    b = BitWriter()
    b.f(1, 0)                                # show_existing_frame
    b.f(2, 1); b.f(1, show_frame)            # frame_type INTER, show_frame
    if not show_frame:
        b.f(1, 1)                            # showable_frame: a later show_existing_frame header outputs it
    b.f(1, 0)                                # error_resilient_mode
    b.f(1, 0)                                # disable_cdf_update
    override = max_size is not None and tuple(max_size) != (w, h)
    b.f(1, 1 if override else 0)             # frame_size_override
    b.f(bits, order_hint)
    b.f(3, 7)                                # primary_ref_frame NONE
    refresh = int(rng.integers(1, 256)) if refresh is None else refresh
    b.f(8, refresh)
    b.f(1, 0)                                # frame_refs_short_signaling
    refidx = [int(rng.integers(0, 8)) for _ in range(7)]
    for r in refidx:
        b.f(3, r)
    if override:
        for _ in range(7):
            b.f(1, 0)                        # found_ref: the size is not taken from a reference ...
        wn, hn = max(1, int(max_size[0] - 1).bit_length()), max(1, int(max_size[1] - 1).bit_length())
        b.f(wn, w - 1); b.f(hn, h - 1)       # ... but written out (frame_width_minus_1, frame_height_minus_1)
    cw = w
    if super_res:                            # superres_params() of frame_size(): the sequence enables the tool, this frame may use it
        use = int(rng.integers(0, 4) > 0)
        b.f(1, use)
        if use:
            cd = int(rng.integers(0, 8))
            b.f(3, cd)
            cw = (w * 8 + (9 + cd) // 2) // (9 + cd)
    b.f(1, 0)                                # render_and_frame_size_different
    hp = int(rng.integers(0, 2))
    b.f(1, hp)                               # allow_high_precision_mv
    if rng.integers(0, 2):
        b.f(1, 1)                            # is_filter_switchable
    else:
        b.f(1, 0); b.f(2, int(rng.integers(0, 4)))
    b.f(1, switchable_motion_mode)
    b.f(1, 0)                                # disable_frame_end_update_cdf
    cols, rows, tile_w, tile_h, sbw, sbh = _frame_common(b, rng, cw, h, sb128, log2_cols, log2_rows, q, lf, cdef, restoration, delta_q, cdef_on, restoration_on, layout, segmentation)
    b.f(1, 1)                                # tx_mode_select
    b.f(1, comp_refs)                        # reference_select
    if comp_refs:                            # skip_mode_present exists only when two suitable references do (src/obu.c:929-987)
        off_before = off_after = -1
        for r in refidx:
            rp = ref_hints[r]
            d = _poc_diff(bits, rp, order_hint)
            if d > 0:
                if off_after < 0 or _poc_diff(bits, off_after, rp) > 0:
                    off_after = rp
            elif d < 0 and (off_before < 0 or _poc_diff(bits, rp, off_before) > 0):
                off_before = rp
        allowed = False
        if off_before >= 0 and off_after >= 0:
            allowed = True
        elif off_before >= 0:
            off2 = -1
            for r in refidx:
                rp = ref_hints[r]
                if _poc_diff(bits, rp, off_before) < 0 and (off2 < 0 or _poc_diff(bits, rp, off2) > 0):
                    off2 = rp
            allowed = off2 >= 0
        if allowed:
            b.f(1, int(rng.integers(0, 2)))  # skip_mode_present
    if warped_motion_seq:
        b.f(1, allow_warped_motion)
    b.f(1, int(rng.integers(0, 2)))          # reduced_tx_set
    if global_motion:
        _global_motion_params(b, rng, hp)
    else:
        for _ in range(7):
            b.f(1, 0)                        # is_global: identity
    if film_grain_seq:
        _film_grain_params(b, rng, 1, layout)
    for i in range(8):
        if refresh & (1 << i):
            ref_hints[i] = order_hint
    return obu(OBU_FRAME, _tile_group(b, rng, cols, rows, tile_w, tile_h, sbw, sbh, sb128, payload_bytes_per_sb64))


def show_existing_frame(slot):
    """a frame header OBU that outputs the (hidden, showable) frame held by reference slot `slot`"""
    b = BitWriter()
    b.f(1, 1)                                # show_existing_frame
    b.f(3, slot)                             # frame_to_show_map_idx
    b.trailing()
    return obu(OBU_FRAME_HDR, b.bytes())


def inter_stream(seed, w, h, n_frames=3, bpc=8, sb128=0, log2_cols=0, log2_rows=0, motion_modes=0, film_grain=0, screen_content=0, layout="420",
                 hidden_every=0, intra_only_every=0, sizes=None, super_res=0, chroma_sample_position=0, color=None, metadata=(), **kw):
    """Temporal units: one key frame, then n_frames - 1 inter frames (single and compound references incl. wedge /
    difference-weighted masks and distance weights, switchable interpolation filters, variable transform trees, intra
    blocks; identity global motion). motion_modes=1 additionally enables the per-block motion mode (overlapped block
    motion compensation, locally warped motion), motion_modes=2 inter-intra prediction as well. hidden_every=k makes
    every k-th inter frame a hidden future frame (decoded early, referenced with backward prediction, output later by a
    show_existing_frame header). color: the sequence header's colour description (sequence_header); metadata: OBUs
    (metadata_hdr_cll, metadata_hdr_mdcv) placed behind the sequence header, which dav1d attaches to every later picture."""
    rng = np.random.default_rng(seed)
    seq = sequence_header(w, h, bpc=bpc, sb128=sb128, inter_intra=1 if motion_modes >= 2 else 0, warped_motion=1 if motion_modes else 0, film_grain=film_grain, screen_content=screen_content, layout=layout, super_res=super_res,
                          chroma_sample_position=chroma_sample_position, color=color)
    kw = dict(kw, layout=layout)
    if super_res:                            # every frame may then be coded narrower and upscaled; its references keep their upscaled size
        kw = dict(kw, super_res=1)
    if motion_modes:
        kw = dict(kw, switchable_motion_mode=1, warped_motion_seq=1, allow_warped_motion=1)
    if film_grain:
        kw = dict(kw, film_grain_seq=1)
    hints = [0] * 8
    tus = [temporal_unit(seq, *metadata, key_frame(rng, w, h, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows, film_grain_seq=film_grain, screen_content=screen_content, layout=layout, super_res=super_res))]
    for i in range(1, n_frames):
        if intra_only_every and i % intra_only_every == 0:
            refresh = int(rng.integers(1, 255))
            tus.append(temporal_unit(key_frame(rng, w, h, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows, film_grain_seq=film_grain,
                                               screen_content=screen_content, layout=layout, intra_only=(i % 128, refresh), super_res=super_res)))
            for k in range(8):
                if refresh & (1 << k):
                    hints[k] = i % 128
            continue
        if hidden_every and i % hidden_every == 0:
            # an "alt-ref": decoded now into slot 7 but not shown (it carries a later order hint), then a shown frame in
            # the same temporal unit, and one unit later a show_existing_frame header that outputs the hidden frame
            hid = inter_frame(rng, w, h, (i + 1) % 128, hints, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows, show_frame=0,
                              refresh=0x80, **kw)
            shown = inter_frame(rng, w, h, i % 128, hints, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows, refresh=int(rng.integers(1, 128)), **kw)
            tus.append(temporal_unit(hid, shown))
            tus.append(temporal_unit(show_existing_frame(7)))
        else:
            # sizes = [(w, h), ...]: inter frame i is coded at sizes[(i - 1) % len(sizes)] (each within a factor 2 down / 16 up of
            # every picture still held as a reference, as AV1 requires): its references are then scaled references
            fw, fh = sizes[(i - 1) % len(sizes)] if sizes else (w, h)
            tus.append(temporal_unit(inter_frame(rng, fw, fh, i % 128, hints, sb128=sb128, log2_cols=log2_cols, log2_rows=log2_rows,
                                                 max_size=(w, h) if sizes else None, **kw)))
    return tus
