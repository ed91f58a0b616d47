"""Times the closed wall and ground polygons (pus_popup_polygons) on the GPU against the CPU oracle on the same host.

Workload: a batch of 64 synthetic frames (640x480, 1-8 ground segments each, walllength 3.0 and ceiling 2.5 as main_3d
runs it).  Reports: the kernels' time per frame (torch.profiler, CUDA activities, summed over the fit, polygon and pack
kernels of one call, in a separate profiled pass), the end-to-end time of one capi.popup_polygons call (host clock; its
size query and filling call, uploads, kernels, copies back and allocation included), and the oracle's single-threaded CPU time per frame.  The card's name and power
limit are printed in the same run.  Not part of bench.py.

    python tools/popup_polygon_bench.py [--reps 200]
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
import popup_polygon_native as N  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402

FRAMES = 64


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
    names = ("popup_kernel", "polygon_kernel", "pack_kernel")
    us = sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names))
    return us / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib, orc = capi.load_library(), N.oracle_lib()
    b = N.random_batch(0, FRAMES, 640, 480, 2.5, 3.0)
    gpu = lambda: capi.popup_polygons(lib, **b)   # noqa: E731
    ref = lambda: capi.popup_polygons(orc, prefix="orc_", **b)   # noqa: E731
    g, o = gpu(), ref()
    for k in ("bound", "cut", "world"):
        assert np.array_equal(g[k].view(np.uint32), o[k].view(np.uint32)), k
    # capi.popup_polygons makes two C-ABI calls, a size query and the filling call; both run the fit and polygon kernels
    e2e = wall(gpu, args.reps)
    k = kernel_ms(gpu, args.reps)
    cpu = wall(ref, max(3, args.reps // 10))
    print(json.dumps({"frames": FRAMES, "rows": int(len(b["segs"]) + FRAMES), "kernel_ms_per_frame": round(k / FRAMES, 5),
                      "end_to_end_ms_per_call": round(e2e, 4), "oracle_cpu_ms_per_frame": round(cpu / FRAMES, 5),
                      "card": card, "call": "capi.popup_polygons = size query + filling call"}))


if __name__ == "__main__":
    main()
