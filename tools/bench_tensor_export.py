"""The tensor export (b200_export_tensor) against the torch chain it replaces (run on a GPU machine):

    python tools/bench_tensor_export.py [--launches 200] [--rounds 5] [--reps 3] [--antialias] [--crop-flip] [--kernel-only]
                                        [--interpolation bilinear | bicubic] [--tonemap] [--jitter] [--baseline-lib SO]
                                        [--out FILE]

Kernel level, one JSON line per configuration, on synthetic device pictures (random planes, 4:2:0):
  fused        one b200_export_tensor launch
  torch_chain  b200_export_picture (RGB at the stream's bit depth, nearest chroma), then x.float() / bdmax,
               interpolate(bilinear, align_corners=False) when resizing, (x - mean) / std, .to(dtype), and for HWC
               .permute(1, 2, 0).contiguous()
  Each is timed with CUDA events around --launches back-to-back launches after a warm-up (a sleep kernel holds the stream
  while they are enqueued, so the events time the GPU, not the host); the two alternate for --rounds
  rounds in the same run, and the median and min of the rounds' per-launch times are reported. `bytes` are algorithmic
  (computed from the shapes: every tensor each step reads and writes, once), `share_of_3.35TBps` their rate against the
  H100 SXM data sheet.
Decoder level, one JSON line per stream workload of bench.py: pictures per second of
  DeviceDecoder.tensors(size, dtype="bfloat16", batch=8) against DeviceDecoder.pictures(format="rgb") followed by the
  torch chain and torch.stack of every 8, the whole stream per run (median, min and max of --reps runs, alternated).
--antialias: the kernel level only, on AA_CONFIGS, with B200TensorJob.antialias = 1 against the chain with
  interpolate(..., antialias=True); a config with a batch runs that many pictures as one b200_export_tensor_batch call
  (the chain then loops over them). --kernel-only skips the decoder level.
--crop-flip: the kernel level only, on CROP_FLIP_CONFIGS: a RandomResizedCrop-style box (area 1/2, aspect 4:3) exported to
  224 x 224 bf16 CHW, antialiased and flipped (B200TensorJob source moved to the box, flip = 1), against the chain a user
  writes otherwise: the RGB export of the whole picture, the slice, interpolate(antialias=True), (x - mean) / std,
  .flip(-1), .to(bfloat16).
--interpolation bicubic: the kernel level only, on BICUBIC_CONFIGS (or CROP_FLIP_CONFIGS with --crop-flip), with
  B200TensorJob.interpolation = B200_TENSOR_BICUBIC (antialiased with --antialias or --crop-flip) against the chain with
  interpolate(mode="bicubic", ...).
--tonemap: the kernel level only, on TONEMAP_CONFIGS: 10-bit BT.2020 PQ or HLG pictures tone-mapped to SDR BT.709
  (b200_export_tensor_tone_batch, one job with the tables of stream.tone_tables) against the chain with the same
  definition: the RGB export, .float(), the curve gather, the 3 x 3 matrix, clamp, the OETF gather, interpolate,
  (x - mean) / std, .to(dtype).
--jitter: the kernel level only, on JITTER_CONFIGS: colour jitter (B200ColorJitter: brightness, contrast, saturation and
  hue, contrast taking its pass over the picture) and grayscale fused into an antialiased export, one b200_export_tensor_jitter_batch call
  for all pictures, against the same export without jitter (`fused_no_jitter`: what the jitter stage and the contrast
  pass cost) and the torch chain: the RGB export, .float() / bdmax, the crop, interpolate(antialias=True),
  torchvision.transforms.v2.functional's adjust_* in the same order, rgb_to_grayscale(num_output_channels=3), the flip,
  (x - mean) / std, .to(dtype).
--baseline-lib SO: the kernel level times the same jobs (flip = 0) through another build of the library (an earlier
  commit's libb200av1.so) instead of the torch chain, alternated with this tree's, as `fused_baseline`.
The GPU's name, power limit and SM clock are read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from dav1d_b200 import _lib, stream  # noqa: E402
from bench_device_output import HBM_BYTES_PER_S, gpu_info, workload_tus  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
ESIZE = {"float32": 4, "float16": 2, "bfloat16": 2}
CONFIGS = [  # (name, source w, h, bpc, output (h, w) or None, dtype, layout)
    ("1080p8 native fp32 chw", 1920, 1080, 8, None, "float32", "chw"),
    ("1080p8 native bf16 hwc", 1920, 1080, 8, None, "bfloat16", "hwc"),
    ("4k10 native fp32 chw", 3840, 2160, 10, None, "float32", "chw"),
    ("4k10 native bf16 hwc", 3840, 2160, 10, None, "bfloat16", "hwc"),
    ("4k10 -> 1920x1080 bf16 chw", 3840, 2160, 10, (1080, 1920), "bfloat16", "chw"),
    ("1080p8 -> 640x360 fp16 chw", 1920, 1080, 8, (360, 640), "float16", "chw"),
]

# the batched launch (B200_TENSOR_BATCH_MAX jobs per launch) of the bilinear kernel, fields as in AA_CONFIGS
BATCH_CONFIG = ("64 x 1080p8 -> 224x224 bf16 chw, one batch call", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 64)


AA_CONFIGS = [  # (name, source w, h, bpc, output (h, w), dtype, layout, pictures per call)
    ("aa 1080p8 -> 224x224 bf16 chw", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 1),
    ("aa 4k10 -> 398x224 bf16 chw", 3840, 2160, 10, (224, 398), "bfloat16", "chw", 1),
    ("aa 4k8 -> 1920x1080 fp16 chw", 3840, 2160, 8, (1080, 1920), "float16", "chw", 1),
    ("aa 1080p8 -> 640x360 fp32 hwc", 1920, 1080, 8, (360, 640), "float32", "hwc", 1),
    ("aa 64 x 1080p8 -> 224x224 bf16 chw, one batch call", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 64),
]


BICUBIC_CONFIGS = [  # AA_CONFIGS' fields: CLIP-style inputs, a downscale to 1080p and an upscale from 720p
    ("1080p8 -> 224x224 bf16 chw", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 1),
    ("4k10 -> 398x224 bf16 chw", 3840, 2160, 10, (224, 398), "bfloat16", "chw", 1),
    ("4k8 -> 1920x1080 fp16 chw", 3840, 2160, 8, (1080, 1920), "float16", "chw", 1),
    ("720p8 -> 1920x1080 bf16 chw", 1280, 720, 8, (1080, 1920), "bfloat16", "chw", 1),
]


CROP_FLIP_CONFIGS = [  # AA_CONFIGS' fields, then the box (top, left, height, width)
    ("crop+flip 1080p8 -> 224x224 bf16 chw", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 1, (100, 372, 882, 1176)),
    ("crop+flip 4k10 -> 224x224 bf16 chw", 3840, 2160, 10, (224, 224), "bfloat16", "chw", 1, (200, 744, 1764, 2352)),
]


TONEMAP_CONFIGS = [  # AA_CONFIGS' fields, no box, then (transfer, antialias, interpolation)
    ("pq 4k10 -> 224x224 bf16 chw, aa bilinear", 3840, 2160, 10, (224, 224), "bfloat16", "chw", 1, None, ("pq", 1, "bilinear")),
    ("pq 4k10 -> 224x224 bf16 chw, aa bicubic", 3840, 2160, 10, (224, 224), "bfloat16", "chw", 1, None, ("pq", 1, "bicubic")),
    ("pq 4k10 -> 1920x1080 fp16 chw, bilinear", 3840, 2160, 10, (1080, 1920), "float16", "chw", 1, None, ("pq", 0, "bilinear")),
    ("hlg 1080p10 -> 224x224 bf16 chw, aa bilinear", 1920, 1080, 10, (224, 224), "bfloat16", "chw", 1, None, ("hlg", 1, "bilinear")),
]


JITTER = ([1, 0, 3, 2], 1.2, 0.8, 1.3, 0.05)    # ColorJitter.get_params-style: contrast first, every op on
JITTER_CONFIGS = [  # AA_CONFIGS' fields, the box, no tone map
    ("jitter 4k10 -> 224x224 bf16 chw, aa", 3840, 2160, 10, (224, 224), "bfloat16", "chw", 1, None, None),
    ("jitter crop+flip 1080p8 -> 224x224 bf16 chw, aa", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 1, (100, 372, 882, 1176), None),
    ("jitter 8 x 16-frame clips 1080p8 -> 224x224 bf16 chw, aa, one batch call", 1920, 1080, 8, (224, 224), "bfloat16", "chw", 128,
     None, None),
]


def jitter_chain(x, bdmax, size, dtype, mean, std, flip):
    """the jittered export in torch: x / bdmax -> interpolate(antialias) -> v2 adjust_* in JITTER's order -> grayscale ->
    normalise"""
    from torchvision.transforms.v2 import functional as TF
    x = F.interpolate((x.float() / bdmax)[None], size=size, mode="bilinear", align_corners=False, antialias=True)[0]
    ops = [TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue]
    for op in JITTER[0]:
        x = ops[op](x, JITTER[1 + op])
    x = TF.rgb_to_grayscale(x, num_output_channels=3)
    x = x.flip(-1) if flip else x
    return ((x - mean) / std).to(getattr(torch, dtype))


def tone_chain(rgb, bdmax, tables, size, dtype, mean, std, antialias, mode):
    """the tone-mapped export in torch: R, G, B at the stream's bit depth -> curve -> matrix -> clamp -> OETF -> resize"""
    curve, m, oetf = tables
    L = curve[rgb.long() * 4]                        # R on the 0 .. 4 * bdmax scale of the curve
    G = torch.einsum("rc,chw->rhw", m, L).clamp_(0, 1)
    x = oetf[torch.round(G * 65536).long()] / (4 * bdmax)
    if size is not None:
        x = F.interpolate(x[None], size=size, mode=mode, align_corners=False, antialias=antialias)[0]
    return ((x - mean) / std).to(getattr(torch, dtype))


def torch_chain(rgb, bdmax, size, dtype, layout, mean, std, antialias=False, flip=False, mode="bilinear"):
    x = rgb.float() / bdmax
    if size is not None:
        x = F.interpolate(x[None], size=size, mode=mode, align_corners=False, antialias=antialias)[0]
    x = (x - mean) / std
    x = (x.flip(-1) if flip else x).to(getattr(torch, dtype))
    return x.permute(1, 2, 0).contiguous() if layout == "hwc" else x


def chain_bytes(w, h, sb, size, dtype, layout, box=None, tone=False):
    """algorithmic bytes of the torch chain: each step reads its input and writes its output once"""
    px, (oh, ow) = w * h, size or (h, w)
    op = oh * ow
    b = w * h * 3 // 2 * sb + 3 * px * sb            # export: YUV in, RGB out
    if box is not None:                              # the steps after the export see the box
        px = box[2] * box[3]
        b += 2 * 3 * op * 4                          # .flip(-1)
    b += 3 * px * sb + 3 * px * 4 + 2 * 3 * px * 4   # .float(), / bdmax
    if tone:                                         # int64 curve index, gather, matrix, clamp, OETF index, gather
        b += 3 * px * (sb + 8) + 3 * px * (8 + 4) + 3 * px * (4 + 4) + 2 * 3 * px * 4 + 3 * px * (4 + 8) + 3 * px * (8 + 4)
    if size is not None:
        b += 3 * px * 4 + 3 * op * 4                 # interpolate
    b += 2 * (2 * 3 * op * 4)                        # - mean, / std
    b += 3 * op * 4 + 3 * op * ESIZE[dtype]          # .to(dtype)
    if layout == "hwc":
        b += 2 * 3 * op * ESIZE[dtype]               # .contiguous()
    return b


def baseline_lib(path):
    """the tensor export entry points of another build of the library, whose B200TensorJob may be of another size (so not
    through _lib.B200Lib, which insists on this tree's layout)"""
    dll = C.CDLL(os.path.abspath(path))
    dll.b200_struct_size.restype = C.c_int
    dll.b200_export_tensor.argtypes = [C.c_void_p, C.c_void_p]
    dll.b200_export_tensor_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    dll.b200_last_error.restype = C.c_char_p

    def check(rc, what):
        if rc != 0:
            raise RuntimeError("%s failed (%d): %s" % (what, rc, dll.b200_last_error().decode()))
    dll.check = check
    return dll


def kernel_level(args):
    lib = _lib.get_lib()
    s = torch.cuda.Stream()
    lines = []
    bicubic = args.interpolation == "bicubic"
    configs = JITTER_CONFIGS if args.jitter else TONEMAP_CONFIGS if args.tonemap else CROP_FLIP_CONFIGS if args.crop_flip else BICUBIC_CONFIGS if bicubic else \
        AA_CONFIGS if args.antialias else [c + (1,) for c in CONFIGS] + [BATCH_CONFIG]
    base = baseline_lib(args.baseline_lib) if args.baseline_lib else None
    for name, w, h, bpc, size, dtype, layout, pics, *extra in configs:
        box = extra[0] if extra else None
        tone = extra[1] if len(extra) > 1 else None
        antialias = tone[1] if tone else args.antialias or args.jitter or box is not None
        interpolation = tone[2] if tone else args.interpolation
        rng = np.random.default_rng(w + bpc)
        bdmax, sb = (1 << bpc) - 1, 1 if bpc == 8 else 2
        planes = [rng.integers(0, bdmax + 1, (ph, pw)).astype(np.uint8 if bpc == 8 else np.int16) for pw, ph in stream.plane_dims(w, h, 1)]
        src = torch.from_numpy(np.concatenate([p.ravel() for p in planes])).cuda()
        offs = [0, planes[0].size, planes[0].size + planes[1].size]
        oh, ow = size or (h, w)
        shape = (3, oh, ow) if layout == "chw" else (oh, ow, 3)
        out = torch.empty(shape, dtype=getattr(torch, dtype), device="cuda")
        tj = stream.TensorJob()
        tj.src = src.data_ptr()
        for k in range(3):
            tj.plane_off[k], tj.stride[k] = offs[k], planes[k].shape[1]
        tj.w, tj.h, tj.ss_hor, tj.ss_ver, tj.bitdepth_max = w, h, 1, 1, bdmax
        tj.out_w, tj.out_h = ow, oh
        tj.dtype, tj.layout, tj.siting_x, tj.siting_y = stream.TENSOR_DTYPES[dtype], stream.TENSOR_LAYOUTS[layout], 0, 1
        tj.cy, tj.rv, tj.gu, tj.gv, tj.bu = stream.rgb_coefficients("bt2020" if tone else "bt709", False)
        scale, bias = stream.tensor_scale_bias(bpc, MEAN, STD)
        for c in range(3):
            tj.scale[c], tj.bias[c] = float(scale[c]), float(bias[c])
        tj.dst, tj.pitch_c, tj.pitch_y = out.data_ptr(), (oh * ow if layout == "chw" else 1), (ow if layout == "chw" else 3 * ow)
        tj.antialias = int(antialias)
        tj.interpolation = stream.TENSOR_INTERPOLATIONS[interpolation]
        if tone:                                 # BT.2020 primaries, source peak 1000 cd/m^2, SDR white at 203
            tables = stream.tone_tables(tone[0], 9, bpc)
            d_tables = [torch.from_numpy(t).cuda() for t in tables]
            tm = stream.ToneMap()
            tm.curve, tm.oetf, tm.curve_len, tm.oetf_bits = d_tables[0].data_ptr(), d_tables[2].data_ptr(), len(tables[0]), 16
            for k in range(9):
                tm.m[k] = float(tables[1].ravel()[k])
            tones = (C.POINTER(stream.ToneMap) * 1)(C.pointer(tm))
        if box is not None:                      # the box is the source; the output is mirrored
            top, left, tj.h, tj.w = box
            tj.plane_off[0] += top * tj.stride[0] + left
            for k in (1, 2):
                tj.plane_off[k] += (top >> 1) * tj.stride[k] + (left >> 1)
            tj.flip = 1
        if pics > 1 or args.jitter:              # the same picture into pics slots, one call
            out = torch.empty((pics,) + shape, dtype=getattr(torch, dtype), device="cuda")
            tjs = (stream.TensorJob * pics)()
            for k in range(pics):
                tjs[k] = stream.TensorJob.from_buffer_copy(tj)
                tjs[k].dst = out[k].data_ptr()
        if args.jitter:                          # J in [0, 1]: scale 1 / std; one acc per picture
            jscale, jbias = stream.tensor_scale_bias(bpc, MEAN, STD, jittered=True)
            jjobs = (stream.TensorJob * pics).from_buffer_copy(tjs)
            for k in range(pics):
                for c in range(3):
                    jjobs[k].scale[c], jjobs[k].bias[c] = float(jscale[c]), float(jbias[c])
            acc = torch.zeros(pics, dtype=torch.int64, device="cuda")
            jts = [stream.color_jitter(JITTER, True, acc=acc.data_ptr() + 8 * k) for k in range(pics)]
            jits = (C.POINTER(stream.ColorJitter) * pics)(*[C.pointer(t) for t in jts])
        rgb = torch.empty((3, h, w), dtype=torch.uint8 if bpc == 8 else torch.int16, device="cuda")
        ej = stream.ExportJob()
        ej.src, ej.format = src.data_ptr(), 1
        for k in range(3):
            ej.plane_off[k], ej.stride[k] = offs[k], planes[k].shape[1]
            ej.dst[k], ej.dst_pitch[k] = rgb.data_ptr() + k * h * w * sb, w
        ej.w, ej.h, ej.ss_hor, ej.ss_ver, ej.bitdepth_max = w, h, 1, 1, bdmax
        ej.cy, ej.rv, ej.gu, ej.gv, ej.bu = tj.cy, tj.rv, tj.gu, tj.gv, tj.bu
        mean = torch.tensor(MEAN, device="cuda").view(3, 1, 1)
        std = torch.tensor(STD, device="cuda").view(3, 1, 1)
        sp = C.c_void_p(s.cuda_stream)

        def fused():
            if args.jitter:
                lib.check(lib.b200_export_tensor_jitter_batch(jjobs, None, jits, pics, sp), "b200_export_tensor_jitter_batch")
            elif tone:
                lib.check(lib.b200_export_tensor_tone_batch(C.byref(tj), tones, 1, sp), "b200_export_tensor_tone_batch")
            elif pics > 1:
                lib.check(lib.b200_export_tensor_batch(tjs, pics, sp), "b200_export_tensor_batch")
            else:
                lib.check(lib.b200_export_tensor(C.byref(tj), sp), "b200_export_tensor")

        def chain():
            for _ in range(pics):
                lib.check(lib.b200_export_picture(C.byref(ej), sp), "b200_export_picture")
                x = rgb if box is None else rgb[:, box[0]:box[0] + box[2], box[1]:box[1] + box[3]]
                if args.jitter:
                    jitter_chain(x, bdmax, size, dtype, mean, std, box is not None)
                elif tone:
                    tone_chain(x, bdmax, d_tables, size, dtype, mean, std, antialias, interpolation)
                else:
                    torch_chain(x, bdmax, size, dtype, layout, mean, std, antialias, box is not None, interpolation)

        arms = {"fused": fused}
        if args.jitter:
            arms["fused_no_jitter"] = lambda: lib.check(lib.b200_export_tensor_batch(tjs, pics, sp), "b200_export_tensor_batch")
        if base is not None:                     # the same jobs in the other build's struct layout
            bsz = base.b200_struct_size(23)
            packed = (C.c_char * (bsz * pics))()
            for k in range(pics):
                C.memmove(C.addressof(packed) + k * bsz, C.addressof(tjs[k] if pics > 1 else tj), bsz)

            def fused_baseline():
                if pics > 1:
                    base.check(base.b200_export_tensor_batch(packed, pics, sp), "b200_export_tensor_batch")
                else:
                    base.check(base.b200_export_tensor(packed, sp), "b200_export_tensor")
            arms["fused_baseline"] = fused_baseline
        else:
            arms["torch_chain"] = chain
        times = {k: [] for k in arms}
        with torch.cuda.stream(s):
            for f in arms.values():
                for _ in range(20):
                    f()
            for _ in range(args.rounds):
                for key, f in arms.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda._sleep(50_000_000)            # holds the stream while the launches are enqueued
                    a.record(s)
                    for _ in range(args.launches):
                        f()
                    b.record(s)
                    b.synchronize()
                    times[key].append(1e3 * a.elapsed_time(b) / args.launches)
        sw, sh = (box[3], box[2]) if box else (w, h)
        fused_bytes = pics * (sw * sh * 3 // 2 * sb + 3 * oh * ow * ESIZE[dtype])
        line = {"config": name, "gpu": gpu_info(), "launches_per_round": args.launches, "rounds": args.rounds, "us": {}, "bytes": {
            "fused": fused_bytes, "fused_baseline": fused_bytes, "fused_no_jitter": fused_bytes, "torch_chain": pics * chain_bytes(w, h, sb, size, dtype, layout, box, bool(tone))},
            "GBps": {}, "share_of_3.35TBps": {}}
        line["bytes"] = {k: v for k, v in line["bytes"].items() if k in times}
        if antialias:
            line["antialias"] = True
        if interpolation == "bicubic":
            line["interpolation"] = "bicubic"
        if tone:
            line["tonemap"] = {"transfer": tone[0], "primaries": "bt2020", "peak": 1000.0, "sdr_peak": 203.0}
        if box is not None:
            line["crop_box"], line["flip"] = list(box), True
        if args.jitter:
            line["jitter"] = {"fn_idx": JITTER[0], "factors": list(JITTER[1:]), "grayscale": True}
        if base is not None:
            line["baseline_lib"] = args.baseline_lib
        for key, v in times.items():
            med = float(np.median(v))
            line["us"][key] = {"median": round(med, 2), "min": round(min(v), 2)}
            line["GBps"][key] = round(line["bytes"][key] / (med * 1e-6) / 1e9, 1)
            line["share_of_3.35TBps"][key] = round(line["bytes"][key] / (med * 1e-6) / HBM_BYTES_PER_S, 3)
        other = "fused_baseline" if base is not None else "torch_chain"
        line["speedup_median"] = round(line["us"][other]["median"] / line["us"]["fused"]["median"], 3)
        print(json.dumps(line), flush=True)
        lines.append(line)
    return lines


def decoder_level(args):
    import bench
    lines = []
    for name in ("stream1080p8_inter", "stream4k10"):
        W = bench.STREAM_WORKLOADS[name]
        tus = workload_tus(name)
        fg = int(W.get("film_grain", 0))
        nthr = min(os.cpu_count() or 2, 32)
        mfd = min(8, W["frames"], nthr)
        dev = stream.DeviceDecoder(n_threads=nthr, max_frame_delay=mfd, apply_grain=fg)
        size, bdmax = (W["H"] // 2, W["W"] // 2), (1 << W["bpc"]) - 1
        mean = torch.tensor(MEAN, device="cuda").view(3, 1, 1)
        std = torch.tensor(STD, device="cuda").view(3, 1, 1)
        s = torch.cuda.Stream()

        def fused():
            n = 0
            for b in dev.tensors(tus, size=size, dtype="bfloat16", batch=8, mean=MEAN, std=STD, stream=s):
                n += b.shape[0]
            return n

        def chain():
            n, pend = 0, []
            for rgb in dev.pictures(tus, format="rgb", stream=s):
                pend.append(torch_chain(rgb, bdmax, size, "bfloat16", "chw", mean, std))
                if len(pend) == 8:
                    n += torch.stack(pend).shape[0]
                    pend = []
            return n + (torch.stack(pend).shape[0] if pend else 0)

        arms = {"tensors_bf16_batch8": fused, "pictures_rgb_plus_torch_chain": chain}
        dts = {k: [] for k in arms}
        with torch.cuda.stream(s):
            for f in arms.values():
                f()
            for _ in range(args.reps):
                for k, f in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    assert f() == W["frames"], k
                    torch.cuda.synchronize()
                    dts[k].append(time.perf_counter() - t0)
        line = {"workload": name, "gpu": gpu_info(), "frames": W["frames"], "output": "%dx%d bf16 chw, batches of 8" % (size[1], size[0]),
                "dav1d_threads": nthr, "frames_in_flight": mfd, "reps": args.reps,
                "fps": {k: round(W["frames"] / float(np.median(v)), 2) for k, v in dts.items()},
                "fps_min_max": {k: [round(W["frames"] / max(v), 2), round(W["frames"] / min(v), 2)] for k, v in dts.items()}}
        dev.release()
        print(json.dumps(line), flush=True)
        lines.append(line)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--antialias", action="store_true")
    ap.add_argument("--crop-flip", action="store_true")
    ap.add_argument("--interpolation", choices=list(stream.TENSOR_INTERPOLATIONS), default="bilinear")
    ap.add_argument("--tonemap", action="store_true")
    ap.add_argument("--jitter", action="store_true")
    ap.add_argument("--baseline-lib", help="another build of libb200av1.so: time its export of the same jobs instead of the chain")
    ap.add_argument("--kernel-only", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    if args.baseline_lib and (args.interpolation != "bilinear" or args.tonemap or args.jitter):
        ap.error("--baseline-lib compares the bilinear and triangle exports, which an earlier library also has")
    assert torch.cuda.is_available(), "needs a CUDA device"
    kernel_only = args.antialias or args.crop_flip or args.tonemap or args.jitter or args.kernel_only or args.interpolation != "bilinear"
    lines = kernel_level(args) + ([] if kernel_only else decoder_level(args))
    if args.out:
        with open(args.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
