"""Times the dense plane clouds (pus_popup_clouds) on the GPU against the CPU oracle on the same host.

Workloads: one TUM-sized frame (640x480, the ground and 4 walls, downsample on, labels on) and a batch of 64 such frames
with jittered polygons.  Reports per frame: the kernels' time (torch.profiler, CUDA activities, summed over the cloud
kernels of one call, in a separate profiled pass), the end-to-end time of one C-ABI call (host clock; uploads, kernels,
copies back and allocation included), and the oracle's single-threaded CPU time.  The card's name and power limit are
printed in the same run.  Not part of bench.py.

    python tools/popup_cloud_bench.py [--reps 50]
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
import popup_cloud_native as N  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402

W, H = 640, 480


def tum_frame(rng, f):
    """camera 1 m above the floor looking horizontally; ground polygon below the horizon, 4 wall quads 3-4 m ahead"""
    R = np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]])
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = [0.01 * f, 0.0, 1.0]
    j = lambda: rng.uniform(-3, 3)   # noqa: E731
    polys = [np.array([[0 + j(), 250 + j()], [639 + j(), 250 + j()], [639, 479], [0, 479]], np.float32)]
    planes = [[0.0, 1.0, 0.0, -1.0]]
    for k in range(4):
        x0, x1 = 160 * k + j(), 160 * (k + 1) - 1 + j()
        polys.append(np.array([[x0, 40 + j()], [x1, 40 + j()], [x1, 250 + j()], [x0, 250 + j()]], np.float32))
        a = rng.uniform(-0.3, 0.3)
        planes.append([np.sin(a), 0.0, np.cos(a), -rng.uniform(3, 4)])
    return polys, np.array(planes, np.float32), T


def workload(n_frames, seed=0):
    rng = np.random.default_rng(seed)
    plane_ptr, poly_ptr, polys, planes, Ts = N.batch([tum_frame(rng, f) for f in range(n_frames)])
    return dict(plane_ptr=plane_ptr, poly_ptr=poly_ptr, polys=polys, planes_sensor=planes, Ts=Ts, invK=N.invK(W, H),
                width=W, height=H, images=np.stack([N.image(f, W, H) for f in range(n_frames)]), downsample=True, labels=True)


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
    us = sum(e.device_time_total for e in prof.key_averages() if "cloud" in e.key)
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
        cap = capi.popup_clouds(lib, points=False, **b)["total"]
        gpu = lambda: capi.popup_clouds(lib, capacity=cap, **b)   # noqa: E731
        ref = lambda: capi.popup_clouds(orc, capacity=cap, prefix="orc_", **b)   # noqa: E731
        g, o = gpu(), ref()
        assert np.array_equal(g["xyz"].view(np.uint32), o["xyz"].view(np.uint32)) and np.array_equal(g["labels"], o["labels"])
        e2e = wall(gpu, args.reps)
        k = kernel_ms(gpu, args.reps)
        cpu = wall(ref, max(3, args.reps // (10 if n > 1 else 1)))
        print(json.dumps({"frames": n, "points": int(g["total"]), "kernel_ms_per_frame": round(k / n, 4),
                          "end_to_end_ms_per_frame": round(e2e / n, 4), "oracle_cpu_ms_per_frame": round(cpu / n, 4),
                          "card": card}))


if __name__ == "__main__":
    main()
