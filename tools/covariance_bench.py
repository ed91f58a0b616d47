"""All-node marginal covariances against one nested-dissection LM step (DESIGN.md section 5.4).

For each graph: the kernel time of the first pus_marginal_covariances call over every live node (linearisation, undamped
factorization, selected inversion, gather), of a second call that reads the stored Sigma, and of one LM step of the same
handle (max_iterations = 1: linearisation, factorization, solves, chi2), each the median of `reps` runs.  Prints one JSON
line per graph with the GPU name and power limit.

    python tools/covariance_bench.py [reps]
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pop_up_slam_b200 import graphgen as gg  # noqa: E402
from pop_up_slam_b200.capi import GpuGraphAPI  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def handle(build):
    a = GpuGraphAPI()
    a.set_linear_solver(2)
    a.set_direct_ordering(1)
    info = build(a)
    return a, [int(i) for i in info["pose_ids"]] + [int(i) for i in info["plane_ids"]]


def from_graph(g):
    def build(a):
        info = gg.build_bulk(a, g)
        gg.configure(a, g)
        return info
    return build


def sphere2500(a):
    from make_sphere_golden import build, load_edge3
    ids = build(a, load_edge3(os.path.join(ROOT, "tests", "golden", "sphere2500.txt.xz")))
    return dict(pose_ids=np.array([ids[k] for k in sorted(ids)]), plane_ids=np.zeros(0, dtype=int))


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    cases = [("config2", from_graph(gg.make_config(2, seed=0))), ("config3", from_graph(gg.make_config(3, seed=0))),
             ("sphere2500", sphere2500), ("revisit5000", from_graph(gg.make_revisit(seed=0, n_poses=5000, n_planes=250)))]
    dev = gpu_info()
    for name, build in cases:
        a, ids = handle(build)
        first, again, step = [], [], []
        for _ in range(reps):
            a.set_properties(max_iterations=1)
            a.upload()          # (invalidates the stored Sigma: the next call computes it)
            a.marginal_covariances(ids)
            first.append(a.stats()["kernel_ms"])
            a.marginal_covariances(ids)
            again.append(a.stats()["kernel_ms"])
            a.batch_optimize()
            step.append(a.stats()["kernel_ms"])
        print(json.dumps(dict(graph=name, nodes=len(ids), gpu=dev, marginals_first_ms=float(np.median(first)),
                              marginals_stored_ms=float(np.median(again)), lm_step_ms=float(np.median(step)),
                              bytes=int(a.debug_fetch("bbytes", 1)[0]), cov_bytes=int(a.debug_fetch("covbytes", 1)[0]))))


if __name__ == "__main__":
    main()
