"""Times the pop-up depth map (pus_popup_depth) on the GPU against the CPU oracle on the same host.

Workloads: one 640x480 frame (the ground and 4 walls of tools/popup_cloud_bench.py, downsample on, ceiling 2.8) and a batch
of 64 such frames with jittered polygons.  Reports per frame: the kernels' time (CUDA events around the call's three kernels
would need the library's stream, so torch.profiler with CUDA activities, summed over the depth kernels of one call, in a
separate profiled pass), the end-to-end time of one capi.popup_depth call (host clock; uploads, kernels, the copy of the
maps to pageable host memory and allocation included), the device-to-host bytes, and the oracle's single-threaded CPU time.
The card's name and power limit are printed in the same run.  Not part of bench.py.

    python tools/popup_depth_bench.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import popup_cloud_bench as CB  # noqa: E402
import popup_depth_native as N  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402

W, H = 640, 480


def workload(n_frames, seed=0):
    rng = np.random.default_rng(seed)
    return N.batch([CB.tum_frame(rng, f) for f in range(n_frames)], W, H, True, 2.8)


def wall(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def kernel_ms(fn, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "depth" in e.key and "emcpy" not in e.key)
    return us / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib, orc = capi.load_library(), N.oracle_lib()
    for n in (1, 64):
        b = workload(n)
        gpu = lambda: capi.popup_depth(lib, **b)   # noqa: E731
        ref = lambda: capi.popup_depth(orc, prefix="orc_", **b)   # noqa: E731
        g, o = gpu(), ref()
        assert np.array_equal(g.view(np.uint32), o.view(np.uint32))
        e2e = wall(gpu, args.reps)
        k = kernel_ms(gpu, args.reps)
        cpu = wall(ref, max(3, args.reps // (10 if n > 1 else 1)))
        print(json.dumps({"frames": n, "written_pixels_per_frame": int((g != 0).sum() // n),
                          "kernel_ms_per_frame": round(k / n, 4), "end_to_end_ms_per_frame": round(e2e / n, 4),
                          "d2h_bytes_per_frame": W * H * 4, "oracle_cpu_ms_per_frame": round(cpu / n, 4), "card": card}))


if __name__ == "__main__":
    main()
