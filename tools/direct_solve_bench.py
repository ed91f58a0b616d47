"""Direct linear solves (pus_set_linear_solver(h, 1) dense, (h, 2) band in insertion order and in nested-dissection order
"nd") against PCG: device-resident solves of the same graphs in each mode, timed by CUDA events on the library's stream with
a 256 MiB L2 flush before every timed solve (as bench.py does).  Per workload: ms per solve and per LM trial step for each
mode, the phase_ms split (11 assembly, 12 factorization, 13 right-hand side, 14 triangular solves in the direct modes), and
the largest difference between the estimates of PCG and each direct mode; for the band and nd modes also the layout: stored
tiles, tile products of one factorization (nd), dependent steps (band: tile columns; nd: levels), device bytes and the host
time of the table build.  Workloads: configs 1 and 2, an 80-pose TUM-scale graph, the 600-pose Huber corridor, sphere400
(loop closures, no planes) -- dense and band side by side -- then, band only (over the dense solve's 640 poses), the
2 000-pose Huber corridor, sphere2500, config 3 and the revisited corridor (gg.make_revisit) at 2 000 and 5 000 poses; a batch
of 64 config-2 graphs; with --config5, one band and one nd solve of config 5 and of a revisited corridor of config 5's size
(or the refusal when a layout is over its budget).  Prints the GPU's name and power limit first.
usage: python tools/direct_solve_bench.py [reps=5] [warmup=2] [--config5]      (one JSON line per workload)"""
import json
import os
import subprocess
import sys
import time

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
    ("revisit2000", lambda: gg.make_revisit(seed=0, n_poses=2000, n_planes=100, max_iterations=8)),
    ("revisit5000", lambda: gg.make_revisit(seed=0, n_poses=5000, n_planes=250, max_iterations=8)),
]
MODES = (("pcg", 0, 0), ("direct", 1, 0), ("band", 2, 0), ("nd", 2, 1))
SPHERES = dict(sphere400=sphere400, sphere2500=sphere2500)


def make(name, g, direct, stream, order=0):
    a = GpuGraphAPI()
    a.set_stream(stream.cuda_stream)
    a.set_linear_solver(direct)
    a.set_direct_ordering(order)
    if g is None:
        ids = SPHERES[name](a)
    else:
        ids = gg.build_bulk(a, g)
        gg.configure(a, g)
    a.upload()
    return a, ids


def layout(a, order):
    """the band / nd layout of an uploaded handle, and the host time of its table build (a recompile of the graph)"""
    t0 = time.perf_counter()
    a._chk(a.lib.pus_debug_compile(a.h))
    out = dict(table_build_s=round(time.perf_counter() - t0, 3), device_bytes=int(a.debug_fetch("bbytes", 1)[0]),
               bordered=len(a.debug_fetch("bborder", 1 << 16)))
    if order == 0:
        first = a.debug_fetch("bfirst", 1 << 24).astype(np.int64)
        out.update(tiles=int(sum(i - first[i] + 1 for i in range(len(first)))), steps=len(first))
    else:
        cptr = a.debug_fetch("ndcptr", 1 << 24).astype(np.int64)
        m = np.diff(cptr) - 1
        out.update(tiles=int(cptr[-1]), tile_products=int((m * (m + 1) // 2).sum()),
                   levels=int(a.debug_fetch("ndlevel", 1 << 24).max()) + 1)
    return out


def run_mode(name, g, kind, order, reps, warmup, stream, flush):
    a, ids = make(name, g, kind, stream, order)
    ms, its = timed(a.solve_resident, reps, warmup, stream, flush)
    a.download()
    r = dict(ms_per_solve=round(ms, 3), trial_steps=int(its[-1]), ms_per_trial_step=round(ms / max(1, its[-1]), 4),
             phase_ms=[round(x, 3) for x in a.stats()["phase_ms"][:15]])
    if kind == 2:
        r.update(layout(a, order))
    return a, ids, r


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
        small = name in ("config1", "config2", "tum80", "huber600", "sphere400")   # (the dense solve takes at most 640 poses)
        for mode, kind, order in MODES:
            if kind == 1 and not small:
                continue
            try:
                a, ids, row[mode] = run_mode(name, g, kind, order, reps, warmup, stream, flush)
            except capi.ApiError as e:   # (a layout over its device-memory budget)
                row[mode] = dict(refused=str(e))
                continue
            est[mode] = estimates(a, ids)
        for mode in ("direct", "band", "nd"):
            if mode in est:
                row[f"max_estimate_diff_pcg_{mode}"] = float(np.abs(est["pcg"] - est[mode]).max())
        if "band" in est and "nd" in est:
            row["max_estimate_diff_band_nd"] = float(np.abs(est["band"] - est["nd"]).max())
        if small:
            row["max_estimate_diff_direct_band"] = float(np.abs(est["direct"] - est["band"]).max())
        print(json.dumps(dict(row, **dev)), flush=True)
    if config5:   # one timed solve per layout, when the graph fits the layout's device-memory budget
        for name, mk in (("config5", lambda: gg.make_config(5, seed=0)),
                         ("revisit50000", lambda: gg.make_revisit(seed=0, n_poses=50000, n_planes=5000, obs_per_pose=20,
                                                                  step=0.02, aisle=100.0, radius=2.0, max_iterations=50))):
            g = mk()
            row = dict(workload=name)
            for mode, kind, order in MODES[2:]:
                try:
                    row[mode] = run_mode(name, g, kind, order, 1, 0, stream, flush)[2]
                except capi.ApiError as e:
                    row[mode] = dict(refused=str(e))
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
