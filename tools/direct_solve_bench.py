"""Direct linear solves (pus_set_linear_solver(h, 1) dense, (h, 2) band) against PCG: device-resident solves of the same
graphs in each mode, timed by CUDA events on the library's stream with a 256 MiB L2 flush before every timed solve (as
bench.py does).  Per workload: ms per solve and per LM trial step for each mode, the phase_ms split (11 assembly,
12 factorization, 13 right-hand side, 14 triangular solves in the direct modes), and the largest difference between the
estimates of PCG and each direct mode.  Workloads: configs 1 and 2, an 80-pose TUM-scale graph, the 600-pose Huber corridor,
sphere400 (loop closures, no planes) -- dense and band side by side -- then, band only (over the dense solve's 640 poses),
the 2 000-pose Huber corridor, sphere2500 and config 3; a batch of 64 config-2 graphs; with --config5, one band solve of
config 5.  Prints the GPU's name and power limit first.
usage: python tools/direct_solve_bench.py [reps=5] [warmup=2] [--config5]      (one JSON line per workload)"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pop_up_slam_b200 import capi, graphgen as gg  # noqa: E402
from pop_up_slam_b200.capi import GpuGraphAPI  # noqa: E402


def device():
    out = dict(gpu=torch.cuda.get_device_name(0))
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        out["power_limit_w"] = None
    return out


def sphere400(api):
    from make_sphere_golden import build
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "sphere400.json")))
    api.set_properties(**fx["properties"])
    edges = [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]]
    ids = build(api, edges)
    return dict(pose_ids=np.array(list(ids.values()) if isinstance(ids, dict) else ids), plane_ids=np.zeros(0, dtype=int))


def sphere2500(api):
    from make_sphere_golden import build, load_edge3
    api.set_properties(**dict(gg.PPS_PROPERTIES, max_iterations=6))
    ids = build(api, load_edge3(os.path.join(ROOT, "tests", "golden", "sphere2500.txt.xz")))
    return dict(pose_ids=np.array([ids[k] for k in sorted(ids)]), plane_ids=np.zeros(0, dtype=int))


WORKLOADS = [
    ("config1", lambda: gg.make_config(1, seed=0)),
    ("config2", lambda: gg.make_config(2, seed=0)),
    ("tum80", lambda: gg.make_config(2, seed=0, n_poses=80, n_planes=20)),
    ("huber600", lambda: gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=8)),
    ("sphere400", None),
    ("huber2000", lambda: gg.make_config(3, seed=0, n_poses=2000, n_planes=200, max_iterations=8)),
    ("sphere2500", None),
    ("config3", lambda: gg.make_config(3, seed=0)),
]
SPHERES = dict(sphere400=sphere400, sphere2500=sphere2500)


def make(name, g, direct, stream):
    a = GpuGraphAPI()
    a.set_stream(stream.cuda_stream)
    a.set_linear_solver(direct)
    if g is None:
        ids = SPHERES[name](a)
    else:
        ids = gg.build_bulk(a, g)
        gg.configure(a, g)
    a.upload()
    return a, ids


def timed(fn, reps, warmup, stream, flush):
    for _ in range(warmup):
        flush.fill_(1.0)
        fn()
    ms, its = [], []
    for k in range(reps):
        flush.fill_(float(k))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        its.append(fn())
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), its


def estimates(a, ids):
    x = [a.get_poses(ids["pose_ids"])[:, :3].ravel()]
    if len(ids["plane_ids"]):
        x.append(a.get_planes(ids["plane_ids"]).ravel())
    return np.concatenate(x)


def main():
    args = [x for x in sys.argv[1:] if not x.startswith("--")]
    reps = int(args[0]) if len(args) > 0 else 5
    warmup = int(args[1]) if len(args) > 1 else 2
    config5 = "--config5" in sys.argv
    dev = device()
    print(json.dumps(dev), flush=True)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    for name, mk in WORKLOADS:
        g = mk() if mk else None
        row = dict(workload=name)
        est = {}
        small = name not in ("huber2000", "sphere2500", "config3")   # (the dense solve takes at most 640 poses)
        for mode, kind in (("pcg", 0), ("direct", 1), ("band", 2)):
            if kind == 1 and not small:
                continue
            a, ids = make(name, g, kind, stream)
            ms, its = timed(a.solve_resident, reps, warmup, stream, flush)
            a.download()
            est[mode] = estimates(a, ids)
            row[mode] = dict(ms_per_solve=round(ms, 3), trial_steps=int(its[-1]), ms_per_trial_step=round(ms / max(1, its[-1]), 4),
                             phase_ms=[round(x, 3) for x in a.stats()["phase_ms"][:15]])
        for mode in ("direct", "band"):
            if mode in est:
                row[f"max_estimate_diff_pcg_{mode}"] = float(np.abs(est["pcg"] - est[mode]).max())
        if small:
            row["max_estimate_diff_direct_band"] = float(np.abs(est["direct"] - est["band"]).max())
        print(json.dumps(dict(row, **dev)), flush=True)
    if config5:   # one timed band solve, when the graph fits the band solve's device-memory budget
        g = gg.make_config(5, seed=0)
        row = dict(workload="config5")
        try:
            a, ids = make("config5", g, 2, stream)
            ms, its = timed(a.solve_resident, 1, 0, stream, flush)
            row["band"] = dict(ms_per_solve=round(ms, 3), trial_steps=int(its[-1]), ms_per_trial_step=round(ms / max(1, its[-1]), 4),
                               phase_ms=[round(x, 3) for x in a.stats()["phase_ms"][:15]],
                               device_bytes=int(a.debug_fetch("bbytes", 1)[0]))
        except capi.ApiError as e:
            row["band"] = dict(refused=str(e))
        print(json.dumps(dict(row, **dev)), flush=True)
    # a batch of 64 config-2 graphs
    graphs = [gg.make_config(2, seed=s) for s in range(64)]
    row = dict(workload="batch64_config2")
    est = {}
    for mode, direct in (("pcg", False), ("direct", True)):
        apis, idl = [], []
        for g in graphs:
            a, ids = make("b", g, direct, stream)
            apis.append(a)
            idl.append(ids)
        ms, its = timed(lambda: int(capi.solve_resident_many(apis).sum()), reps, warmup, stream, flush)
        for a in apis:
            a.download()
        est[mode] = np.concatenate([estimates(a, ids) for a, ids in zip(apis, idl)])
        row[mode] = dict(ms_per_batch=round(ms, 3), trial_steps=int(its[-1]), ms_per_trial_step=round(ms / max(1, its[-1]), 4))
    row["max_estimate_diff"] = float(np.abs(est["pcg"] - est["direct"]).max())
    print(json.dumps(dict(row, **dev)), flush=True)


if __name__ == "__main__":
    main()
