"""The graphs and node pairs of the covariance fixture tests/golden/ref_covariances.npz, shared by its generator
(tools/make_cov_golden.py), its CPU check against the live reference (tests/test_covariance_reference.py) and the GPU
comparison (tests/test_gpu_covariance.py).  The reference's values are Slam::covariances().access right after one
Slam::update() from the generator's initial values: Optimizer::relinearize factors J^T J undamped at that point."""
import os

import numpy as np

from pop_up_slam_b200 import graphgen as gg

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_covariances.npz")
CASES = {
    "config1": lambda: gg.make_config(1, seed=0),
    "config2": lambda: gg.make_config(2, seed=0),
    "huber600": lambda: gg.make_config(3, seed=0, n_poses=600, n_planes=60),
}


def build(api, case):
    """the case on api (build_bulk + configure); returns (pairs, dims): every node's own block, then cross blocks"""
    g = CASES[case]()
    info = gg.build_bulk(api, g)
    gg.configure(api, g)
    P, L = [int(i) for i in info["pose_ids"]], [int(i) for i in info["plane_ids"]]
    pairs = [(i, i) for i in P + L]
    pairs += [(P[0], P[-1]), (P[-1], P[0]), (P[1], P[len(P) // 2]), (P[0], L[0]), (L[-1], P[2]), (L[0], L[-1]),
              (L[1], L[len(L) // 2])]
    ps = set(P)
    dims = [(6 if a in ps else 3, 6 if b in ps else 3) for a, b in pairs]
    return pairs, dims
