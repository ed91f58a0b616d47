"""The error / Jacobian export on the device (pus_weighted_errors, pus_factor_errors, pus_jacobian, pus_normalized_chi2,
pus_local_chi2) against the oracle factor by factor, against the solver's own normal equations, and through the outlier
workflow it exists for: solve, rank the pose-plane factors by error, remove the worst, solve again."""
import json
import os
import sys

import numpy as np
import pytest

from export_api import OracleExportAPI
from pop_up_slam_b200 import geometry as geo, graphgen as gg
from pop_up_slam_b200.capi import ApiError, GpuGraphAPI

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def relerr(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(1e-300, np.abs(np.asarray(b)).max())


def relnorm(a, b):
    """norm-wise relative difference: the measure for error vectors, whose largest entries on the long dead-reckoned
    corridors (config 3 at its initial estimate) carry absolute rounding of 1e-12 of the largest one"""
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(1e-300, np.linalg.norm(np.asarray(b)))


def _build_factor2(api, g):
    from test_export_reference import _factor2   # rays as precompute_edge_ray forms them (float32 (x, y, 1))
    _factor2(api, g)


def _build_loopclose(api, g):
    """Mapper_mono::loopclose_merge's edit sequence (Mapping.cpp:659-700): duplicated walls merged into their landmark,
    the old factors and the duplicate planes removed -- a layout with tombstoned factors and nodes."""
    sys.path.insert(0, HERE)
    from test_reference_build import _loopclose_scenario
    ids = _loopclose_scenario(api, g)
    for k, dup in ids["dup_ids"].items():
        for f, e in ids["dup_facs"][k]:
            api.add_pose_plane(ids["pose_ids"][int(g.pp_pose[e])], ids["plane_ids"][k], api.get_measurement(f, 4), g.pp_sqrtinf[e])
            api.remove_factor(f)
    for k, dup in ids["dup_ids"].items():
        api.remove_node(dup)


def _build_sphere400(api, _):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    from make_sphere_golden import build
    fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
    build(api, [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]])


GRAPHS = {
    "config1": (lambda: gg.make_config(1, seed=0), gg.build_interleaved),
    "config2": (lambda: gg.make_config(2, seed=0), gg.build_interleaved),
    "config3": (lambda: gg.make_config(3, seed=0), gg.build_bulk),
    "sphere400": (lambda: None, _build_sphere400),
    "dense_mixed": (lambda: gg.make_dense(seed=0, **gg.DENSE_CASES["mixed"]), gg.build_bulk),
    "factor2": (lambda: gg.make_config(2, seed=6, n_poses=120, n_planes=30), _build_factor2),
    "loopclose": (lambda: gg.make_config(2, seed=5, n_poses=160, n_planes=30), _build_loopclose),
}


def make_pair(name, mode):
    """the same graph on the device and on the oracle; mode in the oracle's convention (0 numeric, 1 closed form)"""
    make, build = GRAPHS[name]
    g = make()
    gpu, orc = GpuGraphAPI(), OracleExportAPI()
    for api in (gpu, orc):
        build(api, g)
        if g is not None:
            gg.configure(api, g)
        api.set_jacobian_mode(mode)
    return g, gpu, orc


# Bars that differ from the defaults, with what was measured on an H100:
# - config 3 at its dead-reckoned initial estimate (a 500 m corridor): the errors differ from the oracle's (compiled without
#   FMA contraction) by 1.9e-12 norm-wise; 1e-11 there, 1e-12 elsewhere;
# - the closed-form blocks of Pose3d_Plane3d_Factor2 edges: the oracle has no closed form for them and differentiates
#   numerically in both modes, so the comparison measures the central differences' truncation error: 1.22e-4 of the largest
#   entry on this graph (the per-factor check in test_hostmath.py bounds it at 2e-5 of each factor's own scale).
ERR_TOL = {"config3": 1e-11}
VAL_TOL = {("factor2", 1): 3e-4}


def check_against(gpu, orc, mode, err_tol=1e-12, val_tol=1e-10):
    e_g, e_o = gpu.weighted_errors(), orc.weighted_errors()
    assert e_g.shape == e_o.shape
    assert relnorm(e_g, e_o) <= err_tol
    assert gpu.jacobian_dims() == orc.jacobian_dims()
    (J_g, rhs_g), (J_o, rhs_o) = gpu.jacobian(), orc.jacobian()
    assert J_g.shape == J_o.shape
    assert np.array_equal(J_g.indptr, J_o.indptr)
    assert np.array_equal(J_g.indices, J_o.indices)
    # numeric mode: both take the reference's central differences; closed form: the bar of the closed-form stage tests
    # against the oracle's analytic Jacobian
    assert relerr(J_g.data, J_o.data) <= val_tol
    assert relnorm(rhs_g, rhs_o) <= err_tol
    assert relnorm(rhs_g, -e_g) <= err_tol   # (mode 0: rhs at the Euler round trip of the estimate, as upstream)
    assert abs(gpu.normalized_chi2() - orc.normalized_chi2()) <= 1e-10 * abs(orc.normalized_chi2())
    nlive = len(orc.live_fids())
    for n in (0, 1, 7, nlive // 2, nlive, nlive + 5):
        lg, lo = gpu.local_chi2(n), orc.local_chi2(n)
        assert abs(lg - lo) <= 1e-10 * max(lo, 1e-12 * orc.normalized_chi2()), (n, lg, lo)
    fids = orc.live_fids()[::max(1, nlive // 50)][::-1]
    assert relnorm(gpu.factor_errors(fids), orc.factor_errors(fids)) <= err_tol


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", list(GRAPHS))
def test_export_matches_oracle(name, mode):
    g, gpu, orc = make_pair(name, mode)
    check_against(gpu, orc, mode, ERR_TOL.get(name, 1e-12), VAL_TOL.get((name, mode), 1e-10))


@pytest.mark.parametrize("mode", [0, 1])
def test_export_matches_the_solver_normal_equations(mode):
    """At the uploaded linearisation point (pus_upload + debug stage 0) the export's J^T J diagonal blocks and J^T rhs equal
    the device's own Hpp / Hll / gp / gl.  Sign convention: the lineariser accumulates g = J^T r with r the weighted
    residual, and rhs = -r, so g = -J^T rhs."""
    g = gg.make_corridor(seed=0, n_poses=150, n_planes=30, obs_per_pose=6, step=0.1, outlier_frac=0.03, robust_kind=1,
                         robust_b=1.0, odo_noise=(0.003, 0.0005), aisle=10.0, radius=1.5)
    gpu = GpuGraphAPI()
    gg.build_bulk(gpu, g)
    gg.configure(gpu, g)
    gpu.set_jacobian_mode(mode)
    gpu.upload()
    gpu.debug_run_stage(0)
    N, M = g.n_poses, g.n_planes
    Hpp = gpu.debug_fetch("Hpp", N * 36).reshape(N, 6, 6)
    gp = gpu.debug_fetch("gp", N * 6).reshape(N, 6)
    Hll = gpu.debug_fetch("Hll", M * 9).reshape(M, 3, 3)
    gl = gpu.debug_fetch("gl", M * 3).reshape(M, 3)
    pose_node = gpu.debug_fetch("pose_node", N).astype(int)
    plane_node = gpu.debug_fetch("plane_node", M).astype(int)
    J, rhs = gpu.jacobian()
    JtJ = (J.T @ J).tocsr()
    g_all = -(J.T @ rhs)
    for p in range(N):
        c = gpu.node_start(pose_node[p])
        assert relerr(JtJ[c:c + 6, c:c + 6].toarray(), Hpp[p]) <= 1e-12
        assert relerr(g_all[c:c + 6], gp[p]) <= 1e-12 or np.abs(g_all[c:c + 6] - gp[p]).max() <= 1e-12 * np.abs(gp).max()
    for l in range(M):
        c = gpu.node_start(plane_node[l])
        assert relerr(JtJ[c:c + 3, c:c + 3].toarray(), Hll[l]) <= 1e-12
        assert np.abs(g_all[c:c + 3] - gl[l]).max() <= 1e-12 * max(np.abs(gl[l]).max(), 1e-3 * np.abs(gl).max())


def test_chi2_identities():
    g = gg.make_config(2, seed=1)
    gpu = GpuGraphAPI()
    ids = gg.build_bulk(gpu, g)
    gg.configure(gpu, g)
    e = gpu.weighted_errors()
    chi2 = gpu.chi2()
    assert abs(np.sum(e ** 2) - chi2) <= 1e-13 * chi2
    rows, cols = gpu.jacobian_dims()
    assert rows == len(e) == g.dims()["rows"] and cols == g.dims()["state_dim"]
    assert abs(gpu.normalized_chi2() - np.sum(e ** 2) / (rows - cols)) <= 1e-13 * chi2 / (rows - cols)
    # bulk build: factor ids 0 .. n-1, all alive, in row order
    nf = gpu.num_factors()
    rows_of = [gpu.factor_row(f) for f in range(nf)] + [rows]
    for n in (0, 1, 2, 10, nf - 1, nf, nf + 100):
        lo = rows_of[max(0, nf - n)] if n > 0 else rows
        assert abs(gpu.local_chi2(n) - np.sum(e[lo:] ** 2)) <= 1e-13 * chi2
    for f in (0, ids["prior_fid"], ids["ground_fid"], int(ids["pp_fids"][17]), int(ids["odo_fids"][3])):
        r0 = gpu.factor_row(f)
        ef = gpu.factor_errors([f])
        assert np.array_equal(ef, e[r0:r0 + len(ef)])


def test_export_after_solve_and_after_init_pose():
    """after a solve the export reads the device-resident estimate; after pus_init_pose the host values are newer and the
    export re-uploads them first"""
    g = gg.make_config(2, seed=2)
    gpu, orc = GpuGraphAPI(), OracleExportAPI()
    ig, io = gg.build_interleaved(gpu, g), gg.build_interleaved(orc, g)
    for api in (gpu, orc):
        gg.configure(api, g)
        api.set_jacobian_mode(1)
    gpu.batch_optimize()
    orc.init_poses(io["pose_ids"], gpu.get_poses(ig["pose_ids"]))   # the oracle at the device's solution
    orc.init_planes(io["plane_ids"], gpu.get_planes(ig["plane_ids"]))
    check_against(gpu, orc, 1)
    p = int(ig["pose_ids"][g.n_poses // 2])
    moved = gpu.get_pose(p)
    moved[:3] += [0.05, -0.02, 0.01]
    gpu.init_pose(p, moved)
    orc.init_pose(p, moved)
    check_against(gpu, orc, 1)


def test_repeatable_and_independent_of_the_linear_solver():
    g = gg.make_config(2, seed=3)
    outs = []
    for direct in (False, False, True):
        gpu = GpuGraphAPI()
        gpu.set_linear_solver(direct)
        gg.build_bulk(gpu, g)
        gg.configure(gpu, g)
        for mode in (1, 0):
            gpu.set_jacobian_mode(mode)
            J, rhs = gpu.jacobian()
            outs.append((gpu.weighted_errors(), J.indptr, J.indices, J.data, rhs, gpu.normalized_chi2(), gpu.local_chi2(40)))
            again = (gpu.weighted_errors(), *gpu.jacobian()[0].data[None], gpu.local_chi2(40))
            assert np.array_equal(again[0], outs[-1][0]) and np.array_equal(again[1], outs[-1][3]) and again[2] == outs[-1][6]
    for k in range(2, len(outs)):
        for a, b in zip(outs[k], outs[k % 2]):
            assert np.array_equal(np.asarray(a), np.asarray(b))


def test_bad_calls_fail_with_a_message():
    gpu = GpuGraphAPI()
    with pytest.raises(ApiError, match="no live factors"):
        gpu.weighted_errors()
    g = gg.make_config(1, seed=0)
    gg.build_bulk(gpu, g)
    with pytest.raises(ApiError, match="bad factor id"):
        gpu.factor_errors([0, 10 ** 6])
    gpu.remove_factor(3)
    with pytest.raises(ApiError, match="bad factor id 3"):
        gpu.factor_errors([3])
    rows, _ = gpu.jacobian_dims()
    import ctypes as C
    from pop_up_slam_b200.capi import _dp
    out = np.zeros(rows)
    fn = gpu.lib.pus_weighted_errors
    fn.restype = C.c_longlong
    assert fn(gpu.h, _dp(out), C.c_longlong(rows - 1)) < 0
    assert b"capacity" in gpu.lib.pus_last_error()


def _injected_outliers(g):
    """The generator corrupts a measurement by a tangent step of 0.05..0.3 rad on top of 0.01-sigma noise: the observations
    whose measurement is over 0.05 rad from the true plane seen from the true pose are (nearly exactly) that set."""
    local = np.einsum("eji,ej->ei", np.array([geo.pose7_to_T(p) for p in g.poses_truth])[g.pp_pose], g.planes_truth[g.pp_plane])
    local /= np.linalg.norm(local, axis=1, keepdims=True)
    cosang = np.abs(np.sum(local * g.pp_meas, axis=1)).clip(0, 1)
    return np.nonzero(2 * np.arccos(cosang) > 0.05)[0]


def test_outlier_workflow_on_config3():
    """Solve under Huber, rank the pose-plane factors by the norm of their weighted error, remove the worst 5 % and solve
    again.  The removed set must recover most of the injected outliers, and the second solve must match the oracle's on
    the same edited graph."""
    g = gg.make_config(3, seed=0)
    gpu, orc = GpuGraphAPI(), OracleExportAPI()
    ig, io = gg.build_bulk(gpu, g), gg.build_bulk(orc, g)
    for api in (gpu, orc):
        gg.configure(api, g)
        api.set_jacobian_mode(1)
    gpu.batch_optimize()
    pp = ig["pp_fids"]
    err = gpu.factor_errors(pp).reshape(-1, 3)
    norms = np.linalg.norm(err, axis=1)
    k = int(round(0.05 * len(pp)))
    worst = np.argsort(-norms, kind="stable")[:k]
    injected = set(_injected_outliers(g).tolist())
    recall = len(injected & set(worst.tolist())) / max(1, len(injected))
    print(f"outliers injected {len(injected)}, removed {k}, recall {recall:.4f}")
    # Observed on an H100: 2 419 injected, 2 500 removed, recall 0.922.  The bar sits just under it: a change that ranks the
    # factors worse (wrong rows, wrong factor order) drops the recall far below.
    assert recall >= 0.9
    for e in worst:
        gpu.remove_factor(int(pp[e]))
        orc.remove_factor(int(io["pp_fids"][e]))
    # A wall whose every observation was removed is left as a plane node without factors: its columns of the system are zero
    # and the device's plane solve returns NaN for it (the LM then stops before its first step).  Such a landmark has been
    # dropped from the map, so the workflow removes the node as well, on both sides.
    orphans = [int(l) for l in ig["plane_ids"] if not gpu.node_factors(int(l))]
    print(f"planes left without observations: {len(orphans)}")
    for k, l in enumerate(ig["plane_ids"]):
        if int(l) in orphans:
            gpu.remove_node(int(l))
            orc.remove_node(int(io["plane_ids"][k]))
    keep = np.array([int(l) not in orphans for l in ig["plane_ids"]])
    # the second solve, from the device's first solution on both sides, to the oracle within the 1e-4 bar
    orc.init_poses(io["pose_ids"], gpu.get_poses(ig["pose_ids"]))
    orc.init_planes(io["plane_ids"][keep], gpu.get_planes(ig["plane_ids"][keep]))
    it_g, it_o = gpu.batch_optimize(), orc.batch_optimize()
    print(f"second solve: device {it_g} iterations chi2 {gpu.chi2():.6f}, oracle {it_o} iterations chi2 {orc.chi2():.6f}")
    assert it_g > 0
    c_g, c_o = gpu.chi2(), orc.chi2()
    assert abs(c_g - c_o) <= 1e-4 * c_o
    P_g, P_o = gpu.get_poses(ig["pose_ids"]), orc.get_poses(io["pose_ids"])
    assert np.abs(P_g[:, :3] - P_o[:, :3]).max() <= 1e-4 * max(1.0, np.abs(P_o[:, :3]).max())
    L_g, L_o = gpu.get_planes(ig["plane_ids"][keep]), orc.get_planes(io["plane_ids"][keep])
    assert np.abs(L_g * np.sign(np.sum(L_g * L_o, axis=1))[:, None] - L_o).max() <= 1e-4
    # and the edited graph exports as the oracle's does
    assert relnorm(gpu.weighted_errors(), orc.weighted_errors()) <= 1e-11


def test_facade_export_replay(tmp_path):
    """the façade's export methods after a solve (tests/facade_export_replay.cpp): the sum of squares of
    Slam::weighted_errors() is Slam::chi2(), normalized_chi2 divides it by rows - columns, local_chi2 covers the most recent
    factors (all of them for a count past the end), Factor::error is a slice of the stacked errors and the Jacobian's rhs is
    minus the errors"""
    import subprocess
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "facade_export_replay")
    libdir = os.path.join(root, "pop_up_slam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(root, "include"), os.path.join(HERE, "facade_export_replay.cpp"),
                           "-o", exe, "-L" + libdir, "-lpopup_gpu", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    vals = {}
    for line in out.splitlines():
        k, *v = line.split()
        vals.setdefault(k, []).append(v)
    chi2, sumsq, rows = float(vals["chi2"][0][0]), float(vals["sumsq"][0][0]), int(vals["rows"][0][0])
    jr, jc, jnnz, rhs_err = vals["jacobian"][0]
    assert int(jr) == rows and int(jc) == 12 * 6 + 4 * 3
    assert abs(sumsq - chi2) <= 1e-12 * chi2
    assert abs(float(vals["normalized_chi2"][0][0]) - chi2 / (rows - int(jc))) <= 1e-12 * chi2
    local = {int(v[0]): float(v[1]) for v in vals["local_chi2"]}
    assert local[0] == 0.0 and abs(local[1000] - chi2) <= 1e-12 * chi2 and 0 < local[1] <= local[5] <= local[1000]
    assert len(vals["factor_error"][0]) == 1 + 3   # factor 7 is a pose-plane factor: 3 rows
    assert float(rhs_err) <= 1e-12 * max(1.0, np.sqrt(chi2))
    assert int(jnnz) == 6 * 6 + 11 * 6 * 12 + 48 * 3 * 9   # prior, 11 odometry, 48 pose-plane factors; zeros stored
