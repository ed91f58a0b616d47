"""The stored coarse-preconditioner inverse is fp32: the fp64 inverse of A_c rounded once per entry after it is mirrored, so
the matrix the PCG applies is exactly symmetric and within half an fp32 unit of A_c^-1 (a 1 500-pose corridor, whose block
sweep runs many pivot steps over a large team)."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle_api import OracleAPI
from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu

SP = 16


def test_coarse_inverse_is_fp32_rounding_of_fp64_inverse():
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
    ref = np.linalg.inv(0.5 * (Ac + Ac.T))

    ncp = (nc + 7) // 8 * 8
    Acinv = gpu.debug_fetch("Acinv", 36 * ncp * ncp).reshape(6 * ncp, 6 * ncp)
    assert np.array_equal(Acinv.astype(np.float32).astype(np.float64), Acinv)   # fp32 values
    assert np.array_equal(Acinv, Acinv.T)                                       # rounded after the mirror
    got = Acinv[:6 * nc, :6 * nc]
    # half an fp32 spacing of the exact entry, plus what the fp64 sweep itself may be off by (far below that spacing for
    # the large entries, so there the stored value is the nearest fp32 number)
    half = 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    slack = 1e-9 * np.abs(ref).max()
    err = np.abs(got - ref)
    assert np.all(err <= half * (1 + 1e-6) + slack), float(np.max(err - half))
    big = np.abs(ref) >= 1e-3 * np.abs(ref).max()
    assert np.mean(got[big] == ref[big].astype(np.float32)) > 0.99
