"""Direct linear solve (pus_set_linear_solver(h, 1)) against PCG: device-resident solves of the same graphs in both modes,
timed by CUDA events on the library's stream with a 256 MiB L2 flush before every timed solve (as bench.py does).  Per
workload: ms per solve and per LM trial step for each mode, and the largest difference between the two modes' estimates.
Workloads: configs 1 and 2, an 80-pose TUM-scale graph, the 600-pose Huber corridor, sphere400 (loop closures, no planes) and
a batch of 64 config-2 graphs.  Prints the GPU's name and power limit first.
usage: python tools/direct_solve_bench.py [reps=5] [warmup=2]      (one JSON line per workload)"""
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


WORKLOADS = [
    ("config1", lambda: gg.make_config(1, seed=0)),
    ("config2", lambda: gg.make_config(2, seed=0)),
    ("tum80", lambda: gg.make_config(2, seed=0, n_poses=80, n_planes=20)),
    ("huber600", lambda: gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=8)),
    ("sphere400", None),
]


def make(name, g, direct, stream):
    a = GpuGraphAPI()
    a.set_stream(stream.cuda_stream)
    a.set_linear_solver(direct)
    if g is None:
        ids = sphere400(a)
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
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    dev = device()
    print(json.dumps(dev), flush=True)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    for name, mk in WORKLOADS:
        g = mk() if mk else None
        row = dict(workload=name)
        est = {}
        for mode, direct in (("pcg", False), ("direct", True)):
            a, ids = make(name, g, direct, stream)
            ms, its = timed(a.solve_resident, reps, warmup, stream, flush)
            a.download()
            est[mode] = estimates(a, ids)
            row[mode] = dict(ms_per_solve=round(ms, 3), trial_steps=int(its[-1]), ms_per_trial_step=round(ms / max(1, its[-1]), 4),
                             phase_ms=[round(x, 3) for x in a.stats()["phase_ms"][:15]])
        row["max_estimate_diff"] = float(np.abs(est["pcg"] - est["direct"]).max())
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
