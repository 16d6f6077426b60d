"""Clip batches: DeviceDecoder.clips against sequential tensors() calls, and the batched tensor export against one launch
per picture (run on a GPU machine):

    python tools/bench_clips.py [--streams 8] [--threads 16] [--reps 3] [--launches 200] [--rounds 5] [--baseline DIR]
                                [--out FILE]

Decoder level, one JSON line per stream workload: sampled pictures per second of clips([N streams], frames=8, step=2,
size=(224, 224), bf16 CHW) with workers = 1, 2, 4, 8, and of the reference arm, N sequential tensors() calls (every
picture of each stream exported at 224 x 224, the sampled ones counted). Every arm gets the same host thread budget
(--threads): clips with w workers gives each stream's dav1d context threads // w threads and max_frame_delay 2,
tensors() gets all of them and max_frame_delay min(8, threads), its best single-stream setting (the line lists both).
Arms alternate within each of --reps rounds; median, min and max of the rounds. The streams are N 1080p 8-bit inter
streams of obu.inter_stream and, where oracle/_ref/libdav1d_gen.so exists, N sparse generator streams (bench.py's
stream1080p8_sparse recipe, one seed per stream).
Kernel level, one JSON line per source: 64 pictures (1080p 8 bit, 4K 10 bit, 4:2:0) into 224 x 224 bf16 CHW, one
b200_export_tensor_batch call against 64 b200_export_tensor calls, CUDA events around --launches repetitions (a sleep
kernel holds the stream while they are enqueued), --rounds rounds alternated, median and min per repetition in us.
Baseline (--baseline DIR: a built checkout of an earlier commit): tools/bench_tensor_export.py of DIR and of this tree,
run alternately twice each in this call; one JSON line with the single-picture export times (median us) of both.
The GPU's name, power limit and SM clock are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from dav1d_b200 import _lib, obu, stream  # noqa: E402
from bench_device_output import gpu_info  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
FRAMES, STEP, SIZE = 8, 2, (224, 224)


def workload_streams(name, n, n_frames):
    """n different 1080p 8-bit streams of n_frames pictures"""
    W = bench.STREAM_WORKLOADS["stream1080p8_inter"] if name == "inter" else bench.STREAM_WORKLOADS["stream1080p8_sparse"]
    out = []
    for k in range(n):
        build = lambda k=k: obu.inter_stream(100 + k, W["W"], W["H"], n_frames=n_frames, bpc=8, log2_cols=W["log2_cols"],
                                             log2_rows=W["log2_rows"], motion_modes=2)
        if name == "inter":
            out.append(build())
        else:
            import streamgen
            out.append(streamgen.generate(build, seed=100 + k, check=False, **W["gen"])[0])
    return out


def decoder_level(args):
    lines = []
    gen_so = os.path.join(ROOT, "oracle", "_ref", "libdav1d_gen.so")
    n_pics = FRAMES * STEP
    for name in ("inter", "sparse"):
        if name == "sparse" and not os.path.exists(gen_so):
            lines.append({"workload": "clips 1080p8 sparse", "skipped": "oracle/_ref/libdav1d_gen.so absent: not measured"})
            continue
        streams = workload_streams(name, args.streams, n_pics)
        s = torch.cuda.Stream()
        arms = {}
        for w in (1, 2, 4, 8):
            dec = stream.DeviceDecoder(n_threads=max(2, args.threads // w), max_frame_delay=2)
            arms["clips_workers_%d" % w] = (lambda dec=dec, w=w: dec.clips(streams, frames=FRAMES, step=STEP, size=SIZE, dtype="bfloat16",
                                                                            mean=MEAN, std=STD, workers=w, stream=s).shape[0] * FRAMES)
        ref = stream.DeviceDecoder(n_threads=args.threads, max_frame_delay=min(8, args.threads))

        def sequential():
            for tus in streams:
                for _ in ref.tensors(tus, size=SIZE, dtype="bfloat16", mean=MEAN, std=STD, batch=n_pics, stream=s):
                    pass
            return len(streams) * FRAMES
        arms["tensors_sequential"] = sequential
        dts = {k: [] for k in arms}
        with torch.cuda.stream(s):
            for f in arms.values():
                f()
            for _ in range(args.reps):
                for k, f in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    n = f()
                    torch.cuda.synchronize()
                    dts[k].append(time.perf_counter() - t0)
        n = len(streams) * FRAMES
        line = {"workload": "clips 1080p8 %s" % name, "gpu": gpu_info(), "streams": len(streams), "pictures_per_stream": n_pics,
                "clip": "frames=%d step=%d, 224x224 bf16 chw" % (FRAMES, STEP), "host_threads": args.threads,
                "dav1d_threads_per_stream": {k: (args.threads if k == "tensors_sequential" else max(2, args.threads // int(k.rsplit("_", 1)[1])))
                                             for k in arms},
                "max_frame_delay": {k: (min(8, args.threads) if k == "tensors_sequential" else 2) for k in arms},
                "cpu_count": os.cpu_count(), "reps": args.reps,
                "sampled_fps": {k: round(n / float(np.median(v)), 2) for k, v in dts.items()},
                "sampled_fps_min_max": {k: [round(n / max(v), 2), round(n / min(v), 2)] for k, v in dts.items()}}
        print(json.dumps(line), flush=True)
        lines.append(line)
    return lines


def kernel_level(args):
    lib = _lib.get_lib()
    s = torch.cuda.Stream()
    lines = []
    for name, w, h, bpc in (("1080p8", 1920, 1080, 8), ("4k10", 3840, 2160, 10)):
        rng = np.random.default_rng(w + bpc)
        bdmax = (1 << bpc) - 1
        dims = stream.plane_dims(w, h, 1)
        srcs = []
        for k in range(4):                  # 4 distinct pictures, each read by 16 of the 64 jobs
            planes = [rng.integers(0, bdmax + 1, (ph, pw)).astype(np.uint8 if bpc == 8 else np.int16) for pw, ph in dims]
            srcs.append(torch.from_numpy(np.concatenate([p.ravel() for p in planes])).cuda())
        offs = [0, dims[0][0] * dims[0][1], dims[0][0] * dims[0][1] + dims[1][0] * dims[1][1]]
        out = torch.empty((64, 3) + SIZE, dtype=torch.bfloat16, device="cuda")
        jobs = (stream.TensorJob * 64)()
        scale, bias = stream.tensor_scale_bias(bpc, MEAN, STD)
        for i in range(64):
            j = jobs[i]
            j.src = srcs[i % 4].data_ptr()
            for k in range(3):
                j.plane_off[k], j.stride[k] = offs[k], dims[k][0]
                j.scale[k], j.bias[k] = float(scale[k]), float(bias[k])
            j.w, j.h, j.ss_hor, j.ss_ver, j.bitdepth_max = w, h, 1, 1, bdmax
            j.out_w, j.out_h, j.dtype, j.layout, j.siting_x, j.siting_y = SIZE[1], SIZE[0], 2, 0, 0, 1
            j.cy, j.rv, j.gu, j.gv, j.bu = stream.rgb_coefficients("bt709", False)
            j.dst, j.pitch_c, j.pitch_y = out[i].data_ptr(), SIZE[0] * SIZE[1], SIZE[1]
        sp = C.c_void_p(s.cuda_stream)

        def batch():
            lib.check(lib.b200_export_tensor_batch(jobs, 64, sp), "b200_export_tensor_batch")

        def single():
            for i in range(64):
                lib.check(lib.b200_export_tensor(C.byref(jobs[i]), sp), "b200_export_tensor")

        with torch.cuda.stream(s):
            batch()
            s.synchronize()
            want = out.clone()
            out.zero_()
            single()
            s.synchronize()
            assert torch.equal(out, want), "batch and single-job exports differ"
            times = {"batch": [], "single_jobs": []}
            for _ in range(3):
                batch(); single()
            for _ in range(args.rounds):
                for key, f in (("batch", batch), ("single_jobs", single)):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda._sleep(200_000_000)
                    a.record(s)
                    for _ in range(args.launches):
                        f()
                    b.record(s)
                    b.synchronize()
                    times[key].append(1e3 * a.elapsed_time(b) / args.launches)
        line = {"config": "64 x %s 4:2:0 -> 224x224 bf16 chw" % name, "gpu": gpu_info(), "launches": {"batch": 3, "single_jobs": 64},
                "repetitions_per_round": args.launches, "rounds": args.rounds,
                "us_per_64_pictures": {k: {"median": round(float(np.median(v)), 2), "min": round(min(v), 2)} for k, v in times.items()}}
        line["speedup_median"] = round(line["us_per_64_pictures"]["single_jobs"]["median"] / line["us_per_64_pictures"]["batch"]["median"], 2)
        print(json.dumps(line), flush=True)
        lines.append(line)
    return lines


def baseline_comparison(args):
    """tools/bench_tensor_export.py of the checkout at args.baseline and of this tree, alternated: kernel times of
    b200_export_tensor (the "fused" arm) per configuration"""
    runs = {"before": [], "after": []}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(2):
            for key, root in (("before", os.path.abspath(args.baseline)), ("after", ROOT)):
                out = os.path.join(tmp, "%s_%d.jsonl" % (key, r))
                subprocess.run([sys.executable, os.path.join(root, "tools", "bench_tensor_export.py"), "--reps", "1",
                                "--launches", str(args.launches), "--rounds", str(args.rounds), "--out", out], cwd=root, check=True,
                               stdout=subprocess.DEVNULL)
                with open(out) as fh:
                    runs[key].append([json.loads(l) for l in fh])
    line = {"comparison": "b200_export_tensor of --baseline (before) and of this tree (after), tools/bench_tensor_export.py "
            "alternated before, after, before, after", "gpu": gpu_info(),
            "us_fused_median": {}}
    for k, c in enumerate(runs["before"][0]):
        if "config" in c:
            line["us_fused_median"][c["config"]] = {key: [run[k]["us"]["fused"]["median"] for run in runs[key]] for key in runs}
    print(json.dumps(line), flush=True)
    return [line]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-decoder", action="store_true")
    ap.add_argument("--baseline", help="a built checkout of an earlier commit: compare its single-picture export times")
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    lines = kernel_level(args) + ([] if args.skip_decoder else decoder_level(args))
    if args.baseline:
        lines += baseline_comparison(args)
    if args.out:
        with open(args.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
