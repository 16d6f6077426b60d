"""Host output against device output on the stream workloads of bench.py (run on a GPU machine):

    python tools/bench_device_output.py [--reps 5] [--out FILE]

Per workload one JSON line:
  fps          decoder pictures per second, the whole stream per run (median of --reps runs), for HookedDecoder.decode (every
               picture copied into a page-locked host picture, then packed into one numpy buffer) and DeviceDecoder.pictures
               in "planes" and in "rgb" (pictures exported into torch CUDA tensors); the three are alternated in one run
  d2h_bytes_per_picture   device-to-host bytes of the frame jobs per picture (HookStats)
  export_us    export kernel time per picture (CUDA events around each export over every picture of the runs; the stream is
               held busy by a sleep kernel while the export is enqueued, so the events time the kernel, not the host)
  export_bytes algorithmic bytes of one export (samples read + written) and their rate over export_us against 3.35 TB/s
The GPU's name, power limit and SM clock are read in the same run. The sparse workloads need oracle/_ref/libdav1d_gen.so."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from dav1d_b200 import obu, stream  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def workload_tus(name):
    """the stream run_stream of bench.py decodes for `name` (rank 0)"""
    W = bench.STREAM_WORKLOADS[name]
    gen = (lambda *a, **k: obu.inter_stream(*a, motion_modes=2, **k)) if W.get("inter") else obu.intra_stream
    build = lambda: gen(100, W["W"], W["H"], n_frames=W["frames"], bpc=W["bpc"], log2_cols=W["log2_cols"], log2_rows=W["log2_rows"],
                        film_grain=int(W.get("film_grain", 0)))
    if W.get("gen"):
        import streamgen
        return streamgen.generate(build, seed=100, check=False, **W["gen"])[0]
    return build()


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="stream1080p8_inter,stream4k10,stream1080p8_sparse,stream4k8_sparse")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    gen_so = os.path.join(ROOT, "oracle", "_ref", "libdav1d_gen.so")
    lines = []
    for name in args.workloads.split(","):
        W = bench.STREAM_WORKLOADS[name]
        if W.get("gen") and not os.path.exists(gen_so):
            lines.append({"workload": name, "skipped": "oracle/_ref/libdav1d_gen.so absent: not measured"})
            continue
        stream.decode_stream.capacity = (W["W"] * W["H"] * 3 // 2) * (2 if W["bpc"] > 8 else 1) * W["frames"] + (1 << 20)
        tus = workload_tus(name)
        fg = int(W.get("film_grain", 0))
        nthr = min(os.cpu_count() or 2, 32)
        mfd = min(8, W["frames"], nthr)
        host = stream.HookedDecoder()
        dev = stream.DeviceDecoder(n_threads=nthr, max_frame_delay=mfd, apply_grain=fg)
        s = torch.cuda.Stream()
        kern_ms = {"planes": [], "rgb": []}

        def run_device(fmt, timed):
            pending = []

            def alloc(shape, dtype):
                t = torch.empty(shape, dtype=getattr(torch, dtype), device="cuda")
                alloc.n += 1
                if timed and alloc.n == (3 if fmt == "planes" else 1):       # last destination of the picture (4:2:0)
                    torch.cuda._sleep(2_000_000)
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record(s)
                    pending.append(ev)
                return t
            alloc.n = 0
            n = 0
            with torch.cuda.stream(s):
                for _ in dev.pictures(tus, format=fmt, alloc=alloc, stream=s):
                    if timed:
                        pending[-1][1].record(s)
                    alloc.n = 0
                    n += 1
            s.synchronize()
            kern_ms[fmt] += [a.elapsed_time(b) for a, b in pending]
            return n

        arms = {"host": lambda timed: host.decode(tus, n_threads=nthr, max_frame_delay=mfd, apply_grain=fg)[0],
                "planes": lambda timed: run_device("planes", timed), "rgb": lambda timed: run_device("rgb", timed)}
        for arm in arms.values():                  # warm-up
            arm(False)
        host.stats(reset=True)
        dts = {k: [] for k in arms}
        d2h = {k: 0 for k in arms}
        for rep in range(args.reps):
            for k, arm in arms.items():
                t0 = time.perf_counter()
                n = arm(False)
                torch.cuda.synchronize()
                dts[k].append(time.perf_counter() - t0)
                assert n == W["frames"], (k, n)
                d2h[k] += host.stats(reset=True)["d2h_bytes"]
        for rep in range(args.reps):               # the kernel timings, in runs of their own (the sleep kernel is not in the fps)
            run_device("planes", True); run_device("rgb", True)
        px = W["W"] * W["H"]
        sb = 1 if W["bpc"] == 8 else 2
        yuv = px * 3 // 2 * sb
        bytes_ = {"planes": 2 * yuv, "rgb": yuv + 3 * px * sb}
        line = {"workload": name, "gpu": gpu_info(), "frames": W["frames"], "size": "%dx%d %d-bit 4:2:0" % (W["W"], W["H"], W["bpc"]),
                "dav1d_threads": nthr, "frames_in_flight": mfd, "reps": args.reps,
                "fps": {k: round(W["frames"] / float(np.median(v)), 2) for k, v in dts.items()},
                "d2h_bytes_per_picture": {k: d2h[k] // (args.reps * W["frames"]) for k in arms},
                "export_us": {}, "export_bytes": bytes_, "export_GBps": {}, "export_share_of_3.35TBps": {}}
        for fmt in ("planes", "rgb"):
            us = 1e3 * float(np.median(kern_ms[fmt]))
            line["export_us"][fmt] = {"median": round(us, 2), "min": round(1e3 * min(kern_ms[fmt]), 2), "pictures": len(kern_ms[fmt])}
            line["export_GBps"][fmt] = round(bytes_[fmt] / (us * 1e-6) / 1e9, 1)
            line["export_share_of_3.35TBps"][fmt] = round(bytes_[fmt] / (us * 1e-6) / HBM_BYTES_PER_S, 3)
        lines.append(line)
        dev.release()
        print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
