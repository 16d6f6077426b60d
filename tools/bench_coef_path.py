"""Where the coefficient path of a frame job spends its time (run on a GPU machine):

    python tools/bench_coef_path.py [--workload 4k8_inter] [--reps 50] [--rounds 5] [--out FILE]

On bench.py's frame of the workload (same generator, same seed), each timed with CUDA events around --reps back-to-back
launches, after a warm-up, in --rounds alternating rounds (median and min of the per-launch times are reported):
  memset       cudaMemsetAsync of the dense coefficient plane (what a compact job without transform offsets does first)
  coef_expand  b200_coef_expand: the compact stream scattered into the dense plane (one warp per transform block)
  itx_dense    b200_itx_add_frame on the dense plane (the transforms of the dense form)
  itx_compact  the same transforms reading the compact stream through per-block offsets (B200FrameJob.d_itx_coff, a frame
               job holding only the transform blocks)
Each launch of a row runs on its own, not with its neighbours in a PDL chain as in the frame job. One JSON line; the GPU's
name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        return q[0] if q else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="4k8_inter")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import bench
    from dav1d_b200 import _lib, frame, synth
    assert torch.cuda.is_available(), "bench_coef_path needs a CUDA device"
    lib = _lib.get_lib()
    S = bench.make_workload_frame(a.workload, 1)
    bd = S["bd"]
    fb = frame.FrameBuffers(S, compact=True)
    j = fb.job
    assert j.n_intra == 0, "a workload without intra records"
    cc, ex = synth.compact_coefs(S)
    d_ex = torch.from_numpy(ex.view(np.uint8).copy()).cuda()
    st = torch.cuda.current_stream().cuda_stream
    # the transform-only compact job: the frame job's transform blocks, compact stream and offsets, nothing else
    tj = _lib.FrameJob()
    tj.bitdepth_max = bd
    for tx in range(19):
        tj.d_itx[tx], tj.n_itx[tx], tj.d_itx_coff[tx] = j.d_itx[tx], j.n_itx[tx], j.d_itx_coff[tx]
    tj.d_ccoef, tj.d_coef, tj.mc.dst = j.d_ccoef, j.d_coef, j.mc.dst
    for p in range(3):
        tj.itx_stride[p] = j.itx_stride[p]
    lib.b200_set_pdl(1)
    ops = {
        "memset": lambda: lib.check(lib.b200_dev_memset(j.d_coef, 0, j.coef_bytes, st), "memset"),
        "coef_expand": lambda: lib.check(lib.b200_coef_expand(bd, d_ex.data_ptr(), len(ex), j.d_ccoef, j.d_coef, st), "expand"),
        "itx_dense": lambda: lib.check(lib.b200_itx_add_frame(bd, j.d_itx, j.n_itx, j.d_coef, j.mc.dst, j.itx_stride, 0, st), "itx"),
        "itx_compact": lambda: lib.check(lib.b200_frame_run(C.byref(tj), st), "itx compact"),
    }
    # the dense plane holds this frame's coefficients for itx_dense
    ops["memset"](); ops["coef_expand"]()
    for fn in ops.values():
        for _ in range(5):
            fn()
    ops["memset"](); ops["coef_expand"]()
    torch.cuda.synchronize()
    times = {k: [] for k in ops}
    for _ in range(a.rounds):
        for k, fn in ops.items():          # (the dict order puts coef_expand after memset: itx_dense reads real coefficients)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e3 / a.reps)
    out = {"workload": a.workload, "reps": a.reps, "rounds": a.rounds, "unit": "us per launch",
           "tx_blocks": int(sum(j.n_itx[t] for t in range(19))), "dense_coef_bytes": int(j.coef_bytes),
           "compact_coef_bytes": int(cc.nbytes), "coef_block_record_bytes": int(ex.nbytes),
           "offset_bytes": int(4 * sum(j.n_itx[t] for t in range(19))),
           "median": {k: float(np.median(v)) for k, v in times.items()}, "min": {k: float(np.min(v)) for k, v in times.items()},
           "max": {k: float(np.max(v)) for k, v in times.items()}, "gpu": gpu_info()}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
