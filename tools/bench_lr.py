"""Loop restoration alone on bench.py's frame workloads: where the b200_lr_frame time goes.

Builds bench.py's frames (the same synth seeds), runs each frame job once so that the deblocked and post-CDEF pictures are
the pipeline's own, then times b200_lr_frame alone with CUDA events: launches rotate over the frame sets (more than 2x
the 50 MB L2 of distinct pictures, as bench.py does), in alternating rounds over the variants below, and each line
reports the median per launch.

Variants: the lr_mask as generated; every unit unrestored; every unit Wiener; every unit self-guided with both passes
(parameter set 0), 3x3 only (set 10), 5x5 only (set 14); and restore_planes luma only / chroma only.

usage: python tools/bench_lr.py [--workload 4k8_inter] [--sets 6] [--launches 50] [--rounds 5] [--out DIR] [--tag NAME]
Writes one JSON line per variant to DIR/bench_lr_<workload>.jsonl (and stdout), with the card's name, power limit and
SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (FRAME_WORKLOADS, make_workload_frame, workload_buffers, OURS)

# lr_mask unit types: 0 none, 2 Wiener, 3 + n self-guided with parameter set n
MASK_VARIANTS = {"as_generated": None, "none": 0, "wiener": 2, "sgr_both_idx0": 3, "sgr_3x3_idx10": 13, "sgr_5x5_idx14": 17}
PLANE_VARIANTS = {"luma_only": 1, "chroma_only": 6}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    return dict(zip(q.split(","), (v.strip() for v in line.split(",")))) if line else {"error": r.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="4k8_inter", choices=["4k8_inter", "4k10_full", "8k10_full"])
    ap.add_argument("--sets", type=int, default=6, help="frame sets the launches rotate over")
    ap.add_argument("--distinct", type=int, default=3, help="distinct synthetic frames among the sets")
    ap.add_argument("--launches", type=int, default=50, help="launches per timed round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for bench_lr_<workload>.jsonl")
    ap.add_argument("--tag", default="", help="build name written into every line")
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "bench_lr.py needs a CUDA device"
    from dav1d_b200 import get_lib
    lib = get_lib()
    lib.b200_set_pdl(1)         # as bench.py for one whole-frame band
    Ss = [bench.make_workload_frame(args.workload, 1 + k) for k in range(args.distinct)]
    fbs = [bench.workload_buffers(args.workload, Ss[k % args.distinct], **bench.OURS) for k in range(args.sets)]
    for fb in fbs:
        fb.run()
    torch.cuda.synchronize()
    S0 = Ss[0]
    pic_bytes = S0["pic"].nbytes

    # per variant and set: a copy of the job's B200LrFrame pointing at that variant's lr_mask / restore_planes
    masks = {}
    for name, typ in MASK_VARIANTS.items():
        per = []
        for k, fb in enumerate(fbs):
            m = Ss[k % args.distinct]["lr_mask"].copy()
            if typ is not None:
                m["lr"]["type"] = typ
            per.append(torch.from_numpy(m.view(np.uint8).reshape(-1).copy()).cuda())
        masks[name] = per
    frames = {}
    for name in list(MASK_VARIANTS) + list(PLANE_VARIANTS):
        fl = []
        for k, fb in enumerate(fbs):
            lr = type(fb.job.lr).from_buffer_copy(fb.job.lr)
            if name in MASK_VARIANTS:
                lr.lr_mask = masks[name][k].data_ptr()
            else:
                lr.restore_planes = PLANE_VARIANTS[name] & S0["rp"]
            fl.append(lr)
        frames[name] = fl

    bd = (1 << S0["bpc"]) - 1
    st = torch.cuda.current_stream().cuda_stream

    def launch(lr):
        r = lib.b200_lr_frame(bd, C.byref(lr), st)
        assert r == 0, lib.b200_last_error()

    for fl in frames.values():          # warm-up: every variant, every set
        for lr in fl:
            launch(lr)
    torch.cuda.synchronize()
    times = {n: [] for n in frames}
    for _ in range(args.rounds):
        for name, fl in frames.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.launches):
                launch(fl[i % args.sets])
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / args.launches)
    gpu = gpu_info()
    W, H = S0["W"], S0["H"]
    samples = W * H * (1 + 2 * ((W + S0["ss_hor"]) >> S0["ss_hor"]) * ((H + S0["ss_ver"]) >> S0["ss_ver"]) / (W * H))
    px = 2 if S0["bpc"] > 8 else 1
    out = []
    for name, t in times.items():
        med = float(np.median(t))
        line = {"tool": "bench_lr", "build": args.tag, "workload": args.workload, "variant": name,
                "us_per_launch_median": med, "us_per_launch_min": float(min(t)), "us_per_launch_max": float(max(t)),
                "rounds": args.rounds, "launches_per_round": args.launches, "sets": args.sets,
                "distinct_pictures_MB": round(args.sets * pic_bytes / 1e6, 1),
                "algorithmic_GBps": 2 * samples * px / (med * 1e-6) / 1e9,
                "restore_planes": PLANE_VARIANTS.get(name, S0["rp"]) & S0["rp"],
                "unit_size_log2": list(S0["us"]), "gpu": gpu}
        out.append(line)
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lr_%s.jsonl" % args.workload), "a") as f:
            for line in out:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
