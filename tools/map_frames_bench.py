"""Per-frame time of the plane map (pus_map_process_frame) against the same mapping step chained on the host (path B of
tests/test_gpu_map.py: host-oracle association, capi add calls, the same solves, pus_refresh_bind / run over every mapped
frame, pus_project_to_planes), on two seeded corridors of explicit plane arrays: a TUM-length one (80 frames,
plane_3d_tum_far.yaml) and a 2 000-frame one with assoc_near_frames = 1000, run for one round (it takes minutes).

The chained path is split into association + graph edits, the solve, and refresh + re-projection.  pus_map_process_frame
is one call; it runs the same solve launches on the same graph as the chained path (the tests check the graphs are
bit-identical), so its solve is the chained path's solve time, and its other part is the call's time minus that,
reported as "rest" (association, edits, copy_plane, re-projection, refresh).  Host clock around synchronised calls; the
paths alternate round by round; min / median / max over rounds of the per-round median per frame.  The card's name and
power limit are read in the same run.  Prints one JSON line; --out also writes it.  No speed-up is claimed: both paths are
reported as measured.

    python tools/map_frames_bench.py [--rounds 3] [--long 2000] [--out result.json]
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
import map_native as M  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402


def new_handle():
    api = capi.GpuGraphAPI()
    p = api.get_properties()
    api.set_properties(method=1, mod_batch=1, epsilon2=p["epsilon2"] * 0.1, epsilon_abs=p["epsilon_abs"] * 0.1,
                       epsilon_rel=p["epsilon_rel"] * 0.1)   # Mapping.cpp:31-43
    return api


def run_a(frames, cfg):
    """path A: the whole pus_map_process_frame call per frame, in ms"""
    api = new_handle()
    pm = capi.PlaneMap(api, cfg)
    total = []
    for seq, fr in enumerate(frames):
        pm.predict_pose()
        t0 = time.perf_counter()
        pm.process_frame(seq, planes=fr)
        total.append(1e3 * (time.perf_counter() - t0))
    pm.close()
    api.close()
    return np.array(total)


def run_b(frames, cfg):
    """path B: (association + edits, solve, refresh + projection) per frame, in ms"""
    api = new_handle()
    B = M.PathB(api, cfg)
    for seq, fr in enumerate(frames):
        odom, _, _ = B.predict()
        B.frame(seq, fr, odom)
    api.close()
    t = np.array(B.times) * 1e3
    return t[:, 0], t[:, 1], t[:, 2]


def stats(rounds):
    med = [float(np.median(r)) for r in rounds]
    return dict(min=min(med), median=float(np.median(med)), max=max(med))


def workload(name, frames, cfg, n_rounds):
    a_tot, b_edit, b_solve, b_refresh = [], [], [], []
    for _ in range(n_rounds):
        a_tot.append(run_a(frames, cfg))
        e, s, r = run_b(frames, cfg)
        b_edit.append(e)
        b_solve.append(s)
        b_refresh.append(r)
    return dict(workload=name, frames=len(frames),
                map_ms_per_frame=dict(total=stats(a_tot), solve=stats(b_solve),
                                      rest=stats([t - s for t, s in zip(a_tot, b_solve)])),
                chained_ms_per_frame=dict(total=stats([e + s + r for e, s, r in zip(b_edit, b_solve, b_refresh)]),
                                          association_edit=stats(b_edit), solve=stats(b_solve),
                                          refresh_project=stats(b_refresh)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--long", type=int, default=2000)
    ap.add_argument("--out")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = dict(card=card, rounds=a.rounds, timing="host clock around synchronised calls; min / median / max over rounds of the "
               "per-round median per frame", results=[])
    tum = M.corridor(1, 80)
    res["results"].append(workload("tum_length_corridor_80", tum, capi.map_config("tum_far", M.INVK, init_wTo=tum[0]["T"]), a.rounds))
    long_ = M.corridor(2, a.long)
    res["results"].append(workload(f"corridor_{a.long}_near1000", long_,
                                   capi.map_config("tum_far", M.INVK, init_wTo=long_[0]["T"], assoc_near_frames=1000), 1))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
