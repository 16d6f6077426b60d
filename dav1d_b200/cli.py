"""Command-line decoder: dav1d's front end with the B200 back end, the way `tools/dav1d.c` drives libdav1d
(reference tools/dav1d.c:94-138, tools/output/{y4m2,md5}.c; SURVEY.md §8 row f4).

    python -m dav1d_b200.cli -i stream.obu -o out.y4m            # Section-5 ("low overhead") OBU file -> y4m
    python -m dav1d_b200.cli -i stream.obu --muxer md5            # md5 of the decoded frames (like `dav1d --muxer md5`)
    python -m dav1d_b200.cli -i clip.ivf --verify <md5>           # IVF / Annex B input too; exit status 2 on a mismatch
    python -m dav1d_b200.cli --synth inter:1280x720:10:8:grain,mm --muxer md5   # synthetic stream (dav1d_b200/obu.py)
    python -m dav1d_b200.cli --synth key:640x360:8:2 -w s.obu     # just write the synthetic stream to a file

There is one back end: libb200av1 (`--backend` takes the path of another build of the same C ABI; without a CUDA device the
decode fails). Comparisons with stock dav1d live in tests/test_stream.py, which decodes the same file with the reference
library and compares the md5. Input demuxing is limited to what the stream driver needs: the file is
split into temporal units at OBU_TEMPORAL_DELIMITER boundaries (every OBU must carry obu_has_size_field, which is what
`dav1d -o x.obu` and aomenc --obu write)."""
import argparse
import hashlib
import os
import sys
import time

import numpy as np

from . import obu, stream


def split_temporal_units(data):
    """Section 5 byte stream -> list of temporal units (each starts with an OBU_TEMPORAL_DELIMITER)."""
    tus, pos, start = [], 0, 0
    n = len(data)
    while pos < n:
        hdr = data[pos]
        obu_type, ext, has_size = (hdr >> 3) & 15, (hdr >> 2) & 1, (hdr >> 1) & 1
        if not has_size:
            raise ValueError("OBU at byte %d has no size field (Annex B streams are not supported)" % pos)
        p = pos + 1 + ext
        size, shift = 0, 0
        while True:
            b = data[p]; p += 1
            size |= (b & 0x7f) << shift; shift += 7
            if not b & 0x80:
                break
        if obu_type == obu.OBU_TD and pos > start:
            tus.append(bytes(data[start:pos])); start = pos
        pos = p + size
    if pos != n:
        raise ValueError("truncated OBU at the end of the file")
    if n > start:
        tus.append(bytes(data[start:n]))
    return tus


def split_ivf(data):
    """IVF container (reference tools/input/ivf.c): 32-byte file header ('DKIF', fourcc 'AV01'), then per frame a 12-byte
    header (payload size u32, timestamp u64) and one temporal unit of Section-5 OBUs"""
    if data[:4] != b"DKIF" or data[8:12] not in (b"AV01", b"av01"):
        raise ValueError("not an AV1 IVF file")
    pos, tus = int.from_bytes(data[6:8], "little"), []
    while pos + 12 <= len(data):
        sz = int.from_bytes(data[pos:pos + 4], "little")
        pos += 12
        if pos + sz > len(data):
            raise ValueError("truncated IVF frame")
        tus.append(bytes(data[pos:pos + sz])); pos += sz
    return tus


def _leb128(data, pos):
    v, shift = 0, 0
    while True:
        b = data[pos]; pos += 1
        v |= (b & 0x7f) << shift; shift += 7
        if not b & 0x80:
            return v, pos


def split_annexb(data):
    """Annex B length-delimited stream (reference tools/input/annexb.c): temporal_unit_size, frame_unit_size, obu_length
    prefixes; the OBUs inside carry no size field, so each is rewritten into the Section-5 form (has_size_field = 1) the
    stream driver feeds to dav1d"""
    pos, tus = 0, []
    while pos < len(data):
        tu_size, pos = _leb128(data, pos)
        tu_end, out = pos + tu_size, bytearray()
        while pos < tu_end:
            fu_size, pos = _leb128(data, pos)
            fu_end = pos + fu_size
            while pos < fu_end:
                ol, pos = _leb128(data, pos)
                hdr = data[pos]
                ext = (hdr >> 2) & 1
                if hdr & 2:                      # already carries a size field: keep as is
                    out += data[pos:pos + ol]
                else:
                    payload = data[pos + 1 + ext:pos + ol]
                    out += bytes([hdr | 2]) + data[pos + 1:pos + 1 + ext] + obu.leb128(len(payload)) + payload
                pos += ol
        tus.append(bytes(out))
    return tus


def demux(data, kind="auto"):
    if kind == "auto":
        kind = "ivf" if data[:4] == b"DKIF" else "obu"
    return {"ivf": split_ivf, "obu": split_temporal_units, "annexb": split_annexb}[kind](data)


def synth_stream(spec, seed=1):
    """kind:WxH:bpc:frames[:opts] with kind in key / inter, opts a comma list of grain, screen, mm (motion modes + inter-intra)"""
    f = spec.split(":")
    kind, (w, h), bpc, frames = f[0], (int(v) for v in f[1].split("x")), int(f[2]), int(f[3])
    opts = set(f[4].split(",")) if len(f) > 4 else set()
    kw = dict(bpc=bpc, film_grain=int("grain" in opts), screen_content=int("screen" in opts), log2_cols=1, log2_rows=1)
    if kind == "key":
        return obu.intra_stream(seed, w, h, n_frames=frames, **kw)
    if kind == "inter":
        return obu.inter_stream(seed, w, h, n_frames=frames, motion_modes=2 if "mm" in opts else 0, **kw)
    raise ValueError("unknown synthetic stream kind %r" % kind)


def frames_of(info, packed):
    """(w, h, bpc, [Y, U, V] arrays) per decoded picture out of the driver's packed output"""
    pos = 0
    for w, h, bpc, layout in info:
        px = 2 if bpc > 8 else 1
        dt = np.uint16 if px == 2 else np.uint8
        planes = []
        for pw, ph in stream.plane_dims(int(w), int(h), int(layout)):
            nbytes = pw * ph * px
            planes.append(packed[pos:pos + nbytes].view(dt).reshape(ph, pw)); pos += nbytes
        yield int(w), int(h), int(bpc), planes


def write_y4m(path, frames, fps=(25, 1)):
    """YUV4MPEG2 like tools/output/y4m2.c: C420jpeg / C420p10 / Cmono, little-endian 16-bit samples above 8 bit"""
    with open(path, "wb") as fh:
        first = True
        for w, h, bpc, planes in frames:
            if first:
                ss = "mono" if len(planes) == 1 else {1: "420", 2: "422", 3: "444"}[1 if planes[1].shape[0] < h else (2 if planes[1].shape[1] < w else 3)]
                cs = ("420jpeg" if ss == "420" else ss) if bpc == 8 else (ss + str(bpc) if ss == "mono" else "%sp%d" % (ss, bpc))
                fh.write(("YUV4MPEG2 W%d H%d F%d:%d Ip C%s\n" % (w, h, fps[0], fps[1], cs)).encode())
                first = False
            fh.write(b"FRAME\n")
            for p in planes:
                fh.write(np.ascontiguousarray(p).tobytes())


def md5_of(frames):
    """one digest over all frames' planes in output order (what `dav1d --muxer md5` prints)"""
    m = hashlib.md5()
    n = 0
    for _, _, _, planes in frames:
        for p in planes:
            m.update(np.ascontiguousarray(p).tobytes())
        n += 1
    return m.hexdigest(), n


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m dav1d_b200.cli", description=__doc__.split("\n")[0])
    ap.add_argument("-i", "--input", help="input file: Section-5 OBU stream, IVF, or Annex B")
    ap.add_argument("--demuxer", choices=["auto", "obu", "ivf", "annexb"], default="auto")
    ap.add_argument("--verify", metavar="MD5", help="compare the md5 of the decoded frames with this digest (like `dav1d --verify`)")
    ap.add_argument("--synth", help="synthetic stream kind:WxH:bpc:frames[:grain,screen,mm]")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("-w", "--write-stream", help="write the (synthetic) stream to this .obu file")
    ap.add_argument("-o", "--output", help="output file (.y4m)")
    ap.add_argument("--muxer", choices=["y4m", "md5", "null"], default=None)
    ap.add_argument("--threads", type=int, default=min(os.cpu_count() or 2, 16))
    ap.add_argument("--framedelay", type=int, default=4, help="dav1d max_frame_delay (frames in flight, >= 2)")
    ap.add_argument("--filmgrain", type=int, default=1, help="apply film grain (dav1d --filmgrain)")
    ap.add_argument("--backend", default="b200", help="b200 (default) or the path of another build of the libb200av1 C ABI")
    ap.add_argument("--one-job-at-a-time", action="store_true", help="serialise the device jobs (for back ends that are not re-entrant)")
    ap.add_argument("--frametimes", metavar="FILE", help="write one line per output frame: nanoseconds since the previous one (like `dav1d --frametimes`)")
    ap.add_argument("-q", "--quiet", action="store_true", help="no progress / speed line")
    ap.add_argument("--output-path", choices=["host", "device"], default="host",
                    help="device: pictures stay in device memory and are exported as planes (stream.DeviceDecoder); md5 / null only")
    args = ap.parse_args(argv)
    if bool(args.input) == bool(args.synth):
        ap.error("give exactly one of -i / --synth")
    if args.output_path == "device" and (args.output or args.muxer == "y4m" or args.frametimes):
        ap.error("--output-path device supports --muxer md5 / null and --verify")
    tus = synth_stream(args.synth, args.seed) if args.synth else demux(open(args.input, "rb").read(), args.demuxer)
    if args.write_stream:
        with open(args.write_stream, "wb") as fh:
            fh.write(b"".join(tus))
        if not (args.output or args.muxer or args.verify):
            print("wrote %d temporal units, %d bytes" % (len(tus), sum(map(len, tus))))
            return 0
    if args.output_path == "device":
        return _main_device(args, tus)
    kw = dict(n_threads=max(2, args.threads), max_frame_delay=max(2, args.framedelay), apply_grain=args.filmgrain, max_pics=len(tus) + 8)
    t0 = time.perf_counter()
    dec = stream.HookedDecoder(backend=None if args.backend == "b200" else args.backend, serialize=args.one_job_at_a_time)
    n, info, packed = dec.decode(tus, **kw)
    times = dec.output_times_ns()
    dec.release()
    dt = time.perf_counter() - t0
    if args.frametimes:
        # tools/dav1d.c synchronize(): elapsed time between consecutive output frames, in nanoseconds, one per line
        with open(args.frametimes, "w") as fh:
            last = 0
            for t in times:
                fh.write("%d\n" % (t - last)); last = t
    if n < 0:
        print("decoding failed: dav1d error %d" % n, file=sys.stderr)
        return 1
    muxer = args.muxer or ("y4m" if args.output else "md5")
    if muxer == "y4m":
        if not args.output:
            ap.error("--muxer y4m needs -o")
        write_y4m(args.output, frames_of(info, packed))
    elif muxer == "md5":
        digest, cnt = md5_of(frames_of(info, packed))
        print(digest)
    if args.verify:
        digest, _ = md5_of(frames_of(info, packed))
        if digest != args.verify.lower():
            print("md5 mismatch: %s != %s" % (digest, args.verify), file=sys.stderr)
            return 2
    px = sum(int(w) * int(h) for w, h, _, _ in info)
    if not args.quiet:
        # tools/dav1d.c print_stats(): "Decoded n/num frames (100.0%) - x fps" (the decoder's own clock: first byte in to last frame out)
        d_fps = 1e9 * n / times[-1] if times and times[-1] else n / dt
        print("Decoded %d/%d frames (100.0%%) - %.2f fps (%.1f Mpixels/s; %.3f s incl. start-up)" % (n, n, d_fps, px * d_fps / max(n, 1) / 1e6, dt), file=sys.stderr)
    return 0


def _main_device(args, tus):
    """--output-path device: the md5 / --verify digest is taken over the planes the export kernel wrote. A --backend other
    than the CUDA library is a host build of the C ABI (the emulator), whose device memory is host memory: numpy planes."""
    alloc = None if args.backend == "b200" else (lambda shape, dtype: np.empty(shape, dtype))
    dec = stream.DeviceDecoder(backend=None if args.backend == "b200" else args.backend, n_threads=max(2, args.threads),
                               max_frame_delay=max(2, args.framedelay), apply_grain=args.filmgrain, serialize=args.one_job_at_a_time)
    t0 = time.perf_counter()
    m, n, px = hashlib.md5(), 0, 0
    try:
        for planes in dec.pictures(tus, alloc=alloc):
            for p in planes:
                m.update(np.ascontiguousarray(p.cpu().numpy() if hasattr(p, "cpu") else p).tobytes())
            n += 1
            px += planes[0].shape[0] * planes[0].shape[1]
    except RuntimeError as e:
        print(e, file=sys.stderr)
        return 1
    finally:
        dec.release()
    dt = time.perf_counter() - t0
    digest = m.hexdigest()
    if (args.muxer or "md5") == "md5":
        print(digest)
    if args.verify and digest != args.verify.lower():
        print("md5 mismatch: %s != %s" % (digest, args.verify), file=sys.stderr)
        return 2
    if not args.quiet:
        print("Decoded %d/%d frames (100.0%%) - %.2f fps (%.1f Mpixels/s; %.3f s incl. start-up, device output)" % (n, n, n / dt, px / dt / 1e6, dt), file=sys.stderr)
    return 0


if __name__ == "__main__":
    sys.exit(main())
