"""Times pus_popup_lines end to end (host clock around the call, which ends in a device-to-host copy) for a 64-frame
batch and for one frame per call, with the CPU oracle per frame beside it, on seeded 640x480 room frames; the card's
name and power limit are read in the same run.  Prints one JSON line; --out also writes it to a file.

    python tools/popup_lines_bench.py [--frames 64] [--reps 5] [--out result.json]
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
import popup_lines_native as N  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402


def best(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    lib, orc = capi.load_library(), N.oracle_lib()
    res = {"card": card}
    for ch, ds in ((3, 0), (3, 1)):
        imgs = N.random_batch(42, a.frames, 640, 480, ch)
        capi.popup_lines(lib, imgs, downsample=ds)   # warm-up
        tb = best(lambda: capi.popup_lines(lib, imgs, downsample=ds), a.reps)
        t1 = best(lambda: [capi.popup_lines(lib, imgs[f:f + 1], downsample=ds) for f in range(8)], a.reps) / 8
        tc = best(lambda: [capi.popup_lines(orc, imgs[f:f + 1], downsample=ds, prefix="orc_") for f in range(4)], 2) / 4
        res[f"ds{ds}"] = {"batch_ms_per_frame": 1e3 * tb / a.frames, "single_ms_per_frame": 1e3 * t1,
                          "cpu_oracle_ms_per_frame": 1e3 * tc}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
