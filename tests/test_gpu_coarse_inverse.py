"""The coarse-operator inverse at a size where its block sweep runs many pivot steps with the triangle split over a large
team (the stage tests in test_gpu_stages.py use small graphs on small teams)."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle_api import OracleAPI
from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu

SP = 16


def test_coarse_inverse_large_team():
    g = gg.make_corridor(seed=3, n_poses=1500, n_planes=120, obs_per_pose=6, step=0.1, outlier_frac=0.03, robust_kind=1,
                         robust_b=1.0, odo_noise=(0.003, 0.0005), aisle=10.0, radius=1.5)
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    gg.build_bulk(gpu, g)
    gg.build_bulk(orc, g)
    gg.configure(gpu, g)
    gg.configure(orc, g)
    N, lam = g.n_poses, 1e-3
    gpu.upload()
    gpu.debug_run_stage(1, lam)
    assert gpu.stats()["grid_ctas"] >= 64

    # A_c = P^T S P with S = App - Apl All^-1 Apl^T, formed sparsely
    A, _ = orc.normal_equations(lam)
    A = A.tocsc()
    n_p = 6 * N
    App, Apl, All = A[:n_p, :n_p], A[:n_p, n_p:], A[n_p:, n_p:]
    nc = (N - 1 + SP - 1) // SP + 1
    rows, cols, vals = [], [], []
    for p in range(N):
        c0, t = p // SP, (p % SP) / SP
        for d in range(6):
            rows.append(6 * p + d); cols.append(6 * c0 + d); vals.append(1 - t)
            if t > 0:
                rows.append(6 * p + d); cols.append(6 * (c0 + 1) + d); vals.append(t)
    P = sp.csc_matrix((vals, (rows, cols)), shape=(n_p, 6 * nc))
    Q = (Apl.T @ P).tocsc()
    Ac = (P.T @ App @ P).toarray() - (Q.T @ spl.spsolve(All.tocsc(), Q)).toarray()

    ncp = (nc + 7) // 8 * 8
    assert 6 * ncp // 48 >= 10   # pivot steps
    Acinv = gpu.debug_fetch("Acinv", 36 * ncp * ncp).reshape(6 * ncp, 6 * ncp)
    assert np.abs(Acinv[:6 * nc, :6 * nc] - np.linalg.inv(Ac)).max() / np.abs(np.linalg.inv(Ac)).max() < 1e-7
    assert np.array_equal(Acinv, Acinv.T)
    assert np.allclose(Acinv[6 * nc:, 6 * nc:], np.eye(6 * (ncp - nc))) and np.all(Acinv[:6 * nc, 6 * nc:] == 0)
