"""Times the ground edges (pus_popup_edges) on the GPU against the CPU oracle on the same host.

Workloads: a 64-frame 640x480 batch of tools/make_popup_edge_golden.py frames (plus its 7 crafted ones), and single
frames of the same kind called one at a time (main_3d's pattern), downsample_contour on and off.  Reports per frame:
  - kernel_ms: the edge kernels of one call, from torch.profiler's CUDA activity records (the device's own start and end
    times of each kernel), in a separate profiled pass;
  - event_ms: CUDA events recorded on the default stream (where the library's copies and kernels run) around the timed
    calls; the calls are synchronous, so this also spans the host work between them;
  - end_to_end_ms: host clock around one capi.popup_edges call (size query and filling call);
  - the oracle's single-threaded CPU time.
The card's name and power limit are printed in the same run.  Not part of bench.py.

    python tools/popup_edges_bench.py [--reps 20]
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
import popup_edges_native as N  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402


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
    us = sum(e.device_time_total for e in prof.key_averages() if "edge_" in e.key and "emcpy" not in e.key)
    return us / reps / 1e3


def event_ms(fn, reps):
    import torch
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib, orc = capi.load_library(), N.oracle_lib()
    for down in (1, 0):
        b = N.random_batch(100 + down, 64, 640, 480, down)
        n = len(b["labels"])
        singles = []
        for f in range(8):   # the first 8 generated frames, one per call
            l0, l1 = b["line_ptr"][f], b["line_ptr"][f + 1]
            singles.append(dict(labels=b["labels"][f:f + 1], line_ptr=[0, l1 - l0], lines=b["lines"][l0:l1], params=b["params"]))
        for name, work, nf in [("batch", [b], n), ("single_frame", singles, 1)]:
            gpu = lambda: [capi.popup_edges(lib, **x) for x in work]   # noqa: E731
            ref = lambda: [capi.popup_edges(orc, prefix="orc_", **x) for x in work]   # noqa: E731
            for g, o in zip(gpu(), ref()):
                assert all(np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(o[k]).view(np.uint8)) for k in g)
            calls = len(work)
            k = kernel_ms(gpu, args.reps) / calls
            d = event_ms(gpu, args.reps) / calls
            e2e = wall(gpu, args.reps) / calls
            cpu = wall(ref, 2) / calls
            print(json.dumps({"workload": name, "frames_per_call": nf, "downsample_contour": down,
                              "kernel_ms_per_frame": round(k / nf, 4), "event_ms_per_frame": round(d / nf, 4),
                              "end_to_end_ms_per_frame": round(e2e / nf, 4), "oracle_cpu_ms_per_frame": round(cpu / nf, 4),
                              "card": card}), flush=True)


if __name__ == "__main__":
    main()
