"""Dense-plane workload: LM iterations/s and the in-kernel phase split of device-resident solves of graphgen.make_dense graphs
whose 16-pose blocks are over the shared-memory limits of the PCG pose phase (> 256 distinct planes, or > 64 (tile, pose) runs),
next to a control graph of the same shape just within the limits.  The pose phase of an over-limit block keeps its vectors in the
global overflow scratch, so `pose_us_per_pcg_iter` (phase_ms[19] of a sub-phase-timed run) against the control is its cost.
usage: python tools/dense_planes_bench.py [n_poses=1600] [reps=5]      (one JSON line per graph)"""
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pop_up_slam_b200 import graphgen as gg  # noqa: E402
from pop_up_slam_b200.capi import GpuGraphAPI  # noqa: E402


def device():
    import torch
    out = dict(gpu=torch.cuda.get_device_name(0))
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        out["power_limit_w"] = None
    return out


def run(name, g, reps):
    a = GpuGraphAPI()
    gg.build_bulk(a, g)
    gg.configure(a, g)
    a.upload()
    a.solve_resident()   # warm-up (module load, first-touch of the buffers)
    nblk = int(a.debug_fetch("dims", 12)[6])
    over = int((a.debug_fetch("blk_ovf", nblk) >= 0).sum())
    iters, ms, pcg, phase = 0, 0.0, 0, [0.0] * 24
    for _ in range(reps):
        iters += a.solve_resident()
        st = a.stats()
        ms += st["kernel_ms"]
        pcg += st["pcg_iterations"]
        phase = [x + y for x, y in zip(phase, st["phase_ms"])]
    # the phase split from a run of its own: the sub-phase timers of the PCG loop (reserved[2] bit 0) perturb it slightly
    o = a.get_solver_options()
    o.reserved[2] = 1
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    a.solve_resident()
    fine = a.stats()
    ph = fine["phase_ms"]
    return dict(graph=name, n_poses=g.n_poses, n_planes=g.n_planes, edges=g.n_pose_plane, blocks=nblk, blocks_over_limit=over,
                lm_iters=iters // reps, pcg_iters=pcg // reps, kernel_ms=round(ms / reps, 3),
                lm_iters_per_s=round(iters / (ms * 1e-3), 2),
                phase_ms=[round(x / reps, 3) for x in phase[:13]],
                # per solve and per PCG iteration of the fine-timed run: plane-major sweep, fused pose phase
                sweep_ms=round(ph[16], 3), pose_ms=round(ph[19], 3),
                pose_us_per_pcg_iter=round(1e3 * ph[19] / max(1, fine["pcg_iterations"]), 2), sub_phase_ms=[round(x, 3) for x in ph[13:]])


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1600
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    dev = device()
    graphs = [("planes_control", dict(walls=30, advance=14)),   # 241 planes / block: within the limits
              ("planes_over", dict(walls=40, advance=20)),      # 341 planes / block
              ("runs_control", dict(walls=80, advance=6)),      # about 55 runs / block: within the limits
              ("runs_over", dict(walls=110, advance=6))]        # about 70 runs / block
    for name, kw in graphs:
        r = run(name, gg.make_dense(seed=0, n_poses=n, max_iterations=10, **kw), reps)
        print(json.dumps(dict(r, **dev)), flush=True)


if __name__ == "__main__":
    main()
