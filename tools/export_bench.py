"""Time the error / Jacobian export (pus_weighted_errors, pus_jacobian) on BASELINE configs 3 and 5.

For each config and Jacobian mode (closed form, then the reference's central differences) it reports, per call:
  - the kernel time of the errors-only export and of the full Jacobian export (CUDA events around the export kernel on the
    handle's stream, pus_stats.kernel_ms), summed over enough calls to exceed a second after a warm-up;
  - the device-to-host copy time and bytes (pus_stats.d2h_ms / d2h_bytes);
  - the bytes the kernel moves, computed from shapes, over kernel time, against the 3.35 TB/s HBM3 data-sheet figure.
Three repeats each; the spread is the range over the repeats.  The card's name and power limit are printed in the same run.

    python tools/export_bench.py [--configs 3 5] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pop_up_slam_b200 import graphgen as gg    # noqa: E402
from pop_up_slam_b200.capi import GpuGraphAPI  # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def kernel_bytes(a, nnz, jac):
    """bytes the export kernel reads and writes, from shapes: per pose-plane edge a pose (56 B), a plane (32 B), the
    measurement and sqrt-information (80 B) and the slot's indices (8 B); per pose factor two poses, 48 + 168 B of
    measurement / sqrt-information and 8 B of indices; per record its 16-byte table entry; out: the error rows, and with
    the Jacobian the values and rhs."""
    st = a.stats()
    E, Epf, Elp = st["n_pose_plane"], st["n_odometry"] + st["n_pose_prior"], st["n_plane_prior"]
    rows, _ = a.jacobian_dims()
    b = E * (56 + 32 + 80 + 8) + Epf * (2 * 56 + 48 + 168 + 8) + Elp * (32 + 80 + 4) + 16 * (E + Epf + Elp) + 8 * rows
    if jac:
        b += 8 * nnz + 8 * rows
    return b


def time_calls(a, fn, min_s=1.0):
    fn()   # warm-up (first call builds the layout tables)
    fn()
    n, k_ms, d_ms, t0 = 0, 0.0, 0.0, time.perf_counter()
    while time.perf_counter() - t0 < min_s or n < 5:
        fn()
        st = a.stats()
        k_ms += st["kernel_ms"]
        d_ms += st["d2h_ms"]
        n += 1
    st = a.stats()
    return k_ms / n, d_ms / n, st["d2h_bytes"], n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[3, 5])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    print("card:", card())
    out = []
    for cfg in args.configs:
        g = gg.make_config(cfg, seed=0)
        a = GpuGraphAPI()
        gg.build_bulk(a, g)
        gg.configure(a, g, max_iterations=2)
        a.upload()
        a.solve_resident()   # (fills the stats' graph sizes; the export then reads the resident estimate)
        rows, cols = a.jacobian_dims()
        for mode_name, mode in (("closed", 1), ("numeric", 0)):
            a.set_jacobian_mode(mode)
            nnz = a.jacobian()[0].nnz
            for what, jac in (("errors", False), ("jacobian", True)):
                fn = a.weighted_errors if not jac else a.jacobian
                reps = [time_calls(a, fn) for _ in range(args.repeats)]
                kb = kernel_bytes(a, nnz, jac)
                k = [r[0] for r in reps]
                d = [r[1] for r in reps]
                rec = dict(config=cfg, mode=mode_name, export=what, rows=rows, cols=cols, nnz=nnz, calls=[r[3] for r in reps],
                           kernel_ms=float(np.median(k)), kernel_ms_range=[min(k), max(k)],
                           d2h_ms=float(np.median(d)), d2h_ms_range=[min(d), max(d)], d2h_bytes=int(reps[-1][2]),
                           kernel_bytes=int(kb), kernel_GBps=kb / (np.median(k) * 1e-3) / 1e9,
                           share_of_hbm=kb / (np.median(k) * 1e-3) / HBM_BPS)
                print(json.dumps(rec), flush=True)
                out.append(rec)
        a.close()
    return out


if __name__ == "__main__":
    main()
