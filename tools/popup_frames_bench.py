"""Per-frame end-to-end time of main_3d's pop-up chain (lines -> edges -> fit -> filter -> polygons -> clouds) on seeded
640x480 rendered rooms, four ways: the stage calls with the INTEGRATION.md glue (size queries included), the pop-up session
on host inputs, the session on device inputs (torch CUDA tensors, outputs left on the device), and the CPU oracles' chain.
Each arm runs one frame per call and 64-frame batches.  Host-clock timings around synchronised work, the arms alternated
round by round; min / median / max over the rounds are reported.  With --profile a separate torch.profiler run of one
batched session call gives the device kernel time.  The card's name and power limit are read in the same run.  Prints one
JSON line; --out also writes it to a file.

    python tools/popup_frames_bench.py [--frames 64] [--rounds 5] [--profile] [--out result.json]
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
import oracle_api  # noqa: E402
import popup_cloud_native as NC  # noqa: E402
import popup_depth_native as ND  # noqa: E402
import popup_edges_native as NE  # noqa: E402
import popup_frames_native as NF  # noqa: E402
import popup_lines_native as NL  # noqa: E402
import popup_polygon_native as NP  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402


def stats(ts):
    ts = sorted(ts)
    return {"min": ts[0], "median": ts[len(ts) // 2], "max": ts[-1], "n": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--single", type=int, default=8, help="frames timed one per call in each round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    lib = capi.load_library()
    orcs = (NL.oracle_lib(), NE.oracle_lib(), oracle_api.oracle_lib(), NP.oracle_lib(), NC.oracle_lib(), ND.oracle_lib())
    w, h, n = 640, 480, a.frames
    imgs, labs, Ts = NF.rooms(42, n, w, h)
    cfg = NF.config(w, h)
    sess = capi.PopupFrames(lib, cfg)
    d_in = [torch.from_numpy(x).cuda() for x in (imgs, labs, Ts)]

    def stage(sl):
        NF.chain((lib,) * 6, imgs[sl], labs[sl], Ts[sl], cfg)

    def host(sl):
        sess.run(imgs[sl], labs[sl], Ts[sl])

    def device(sl):
        sess.run(*[x[sl] for x in d_in])
        torch.cuda.synchronize()

    def cpu(sl):
        NF.chain(orcs, imgs[sl], labs[sl], Ts[sl], cfg, prefix="orc_")

    arms = {"stage_calls": stage, "session_host": host, "session_device": device, "cpu_oracles": cpu}
    whole, singles = slice(0, n), [slice(f, f + 1) for f in range(a.single)]
    for fn in arms.values():   # warm-up of both shapes
        fn(whole)
        fn(singles[0])
    t = {k: {"batch": [], "single": []} for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            if k == "cpu_oracles" and len(t[k]["batch"]) >= 2:
                continue   # seconds per round; two rounds show its spread
            t0 = time.perf_counter()
            fn(whole)
            t[k]["batch"].append(1e3 * (time.perf_counter() - t0) / n)
            t0 = time.perf_counter()
            for sl in singles:
                fn(sl)
            t[k]["single"].append(1e3 * (time.perf_counter() - t0) / len(singles))
    res = {"card": card, "frames": n, "size": [w, h],
           "ms_per_frame": {k: {m: stats(v) for m, v in d.items()} for k, d in t.items()}}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        device(whole)
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            device(whole)
        ev = [e for e in prof.key_averages() if e.device_type.name == "CUDA" and "Memcpy" not in e.key]
        total = sum(e.self_device_time_total for e in ev) / 1e3
        res["session_kernel_ms_per_frame"] = total / n
        res["top_kernels_ms"] = {e.key[:60]: e.self_device_time_total / 1e3
                                 for e in sorted(ev, key=lambda e: -e.self_device_time_total)[:6]}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
