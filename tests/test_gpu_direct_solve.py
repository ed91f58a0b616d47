"""The exact direct linear solve (pus_set_linear_solver(h, 1)): its stages against numpy on the oracle's normal equations,
whole LM / GN / update solves against the closed-form oracle on every trial step, reference-Jacobian + direct mode against the
reference's own LM runs, a façade replay through Slam::set_linear_solver, the reference's sphere400 fixture, bit-identical
estimates across team shapes and batch positions, a failed factorization, and the refusals (graphs over 640 poses, spanning)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse.linalg as spl

from oracle_api import OracleAPI
from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def pair(g, interleaved=False, direct=True, dup=None):
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    gpu.set_linear_solver(direct)
    out = []
    for api in (gpu, orc):
        info = gg.build_interleaved(api, g) if interleaved else gg.build_bulk(api, g)
        for e in (dup if dup is not None else []):
            m = g.pp_meas[e].copy()
            m[3] += 0.01
            api.add_pose_plane(int(info["pose_ids"][g.pp_pose[e]]), int(info["plane_ids"][g.pp_plane[e]]), m / np.linalg.norm(m),
                               g.pp_sqrtinf[e])
        gg.configure(api, g)
        out.append(info)
    return gpu, orc, out[0], out[1]


def relerr(a, b):
    return np.abs(a - b).max() / max(1e-300, np.abs(b).max())


STAGE_CASES = {
    "config1": lambda: gg.make_config(1, seed=0),
    "config2": lambda: gg.make_config(2, seed=0),
    "dense": lambda: gg.make_dense(seed=0),
    "n1": lambda: gg.make_config(2, seed=1, n_poses=1, n_planes=4),
    "n7": lambda: gg.make_config(2, seed=1, n_poses=7, n_planes=6),
    "n8": lambda: gg.make_config(2, seed=1, n_poses=8, n_planes=6),
}

@pytest.mark.parametrize("case", list(STAGE_CASES))
@pytest.mark.parametrize("lam", [0.0, 1e-6, 1e-2])
def test_stages_match_numpy(case, lam):
    g = STAGE_CASES[case]()
    gpu, orc, ig, io = pair(g)
    N, M = g.n_poses, g.n_planes
    A, b = orc.normal_equations(lam)
    A = A.tocsc()
    n = 6 * N
    App, Apl, All = A[:n, :n], A[:n, n:], A[n:, n:]
    S = App.toarray() - (Apl @ spl.spsolve(All.tocsc(), Apl.T.tocsc())).toarray() if M else App.toarray()
    gpu.upload()
    gpu.debug_run_stage(4, lam)
    Sd = gpu.debug_fetch("Sdir", n * n).reshape(n, n)
    e_s = relerr(Sd, np.tril(S))
    gpu.debug_run_stage(1, lam)
    L = gpu.debug_fetch("Ldir", n * n).reshape(n, n)
    e_l = relerr(L, np.linalg.cholesky(S))
    gpu.debug_run_stage(2, lam)
    got = gpu.debug_fetch("delta", n + 3 * M)
    ref = spl.spsolve(A, b)
    e_d = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    print(f"{case} lam={lam}: S {e_s:.2e}  L {e_l:.2e}  delta {e_d:.2e}")
    assert e_s < 1e-12
    assert e_l < 1e-10
    assert e_d < 1e-10


def test_641_poses_fail_and_launch_nothing():
    g = gg.make_corridor(seed=0, n_poses=641, n_planes=40, obs_per_pose=4)
    gpu = GpuGraphAPI()
    gpu.set_linear_solver(True)
    gg.build_bulk(gpu, g)
    gg.configure(gpu, g)
    with pytest.raises(capi.ApiError, match="at most 640"):
        gpu.batch_optimize()
    assert gpu.stats()["gpu_launches"] == 0


def step_err(a, b):
    """largest relative chi2 difference over the trial steps, each step against its own value"""
    a, b = np.asarray(a), np.asarray(b)
    return float(np.max(np.abs(a - b) / np.abs(b))) if len(b) else 0.0


def trace_match(gpu, orc, rtol=1e-8):
    tg, to = gpu.trace(), orc.trace()
    assert np.array_equal(tg["accepted"], to["accepted"])
    assert np.allclose(tg["lam"], to["lam"], rtol=1e-12)
    err = step_err(tg["chi2_new"], to["chi2_new"])
    assert np.all(tg["pcg"] == 0)
    assert err <= rtol, err
    return err


def estimates_match(gpu, orc, ig, io, tol=1e-8):
    P_g, P_o = gpu.get_poses(ig["pose_ids"]), orc.get_poses(io["pose_ids"])
    sq = np.sign(np.sum(P_g[:, 3:] * P_o[:, 3:], axis=1))[:, None]
    e = max(np.abs(P_g[:, :3] - P_o[:, :3]).max() / max(1.0, np.abs(P_o[:, :3]).max()), np.abs(P_g[:, 3:] * sq - P_o[:, 3:]).max())
    if len(ig["plane_ids"]):
        L_g, L_o = gpu.get_planes(ig["plane_ids"]), orc.get_planes(io["plane_ids"])
        sl = np.sign(np.sum(L_g * L_o, axis=1))[:, None]
        e = max(e, np.abs(L_g * sl - L_o).max())
    assert e <= tol, e
    return e


@pytest.mark.parametrize("cfg,seed", [(1, 0), (1, 1), (1, 2), (2, 0), (2, 1), (2, 2)])
def test_lm_matches_oracle_on_every_trial_step(cfg, seed):
    g = gg.make_config(cfg, seed=seed)
    gpu, orc, ig, io = pair(g, interleaved=True)
    assert gpu.batch_optimize() == orc.batch_optimize()
    e_t = trace_match(gpu, orc)
    e_x = estimates_match(gpu, orc, ig, io)
    assert gpu.stats()["pcg_iterations"] == 0
    print(f"config {cfg} seed {seed}: chi2_new {e_t:.2e}, estimates {e_x:.2e}")


def test_huber_corridor_matches_oracle_on_every_trial_step():
    g = gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=8)
    gpu, orc, ig, io = pair(g)
    assert gpu.batch_optimize() == orc.batch_optimize()
    print("600-pose Huber corridor:", trace_match(gpu, orc), estimates_match(gpu, orc, ig, io))


def test_repeated_observations_of_one_plane():
    g = gg.make_config(2, seed=4, n_poses=60, n_planes=15)
    dup = np.random.default_rng(0).choice(len(g.pp_pose), size=25, replace=False)
    gpu, orc, ig, io = pair(g, dup=dup)
    assert gpu.batch_optimize() == orc.batch_optimize()
    trace_match(gpu, orc)
    estimates_match(gpu, orc, ig, io)


def test_gauss_newton_and_update_match_oracle():
    g = gg.make_config(2, seed=1)
    for which in ("gn", "update"):
        gpu, orc = GpuGraphAPI(), OracleAPI()
        orc.set_jacobian_mode(1)
        gpu.set_linear_solver(True)
        ig, io = gg.build_bulk(gpu, g), gg.build_bulk(orc, g)
        gg.configure(gpu, g, method=0)
        gg.configure(orc, g, method=0)
        if which == "gn":
            assert gpu.batch_optimize() == orc.batch_optimize()
            trace_match(gpu, orc)
        else:
            for _ in range(3):
                gpu.update()
                orc.update()
        estimates_match(gpu, orc, ig, io)


def test_reference_sphere400_fixture():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    from make_sphere_golden import build
    fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
    edges = [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]]
    gpu = GpuGraphAPI()
    gpu.set_linear_solver(True)
    gpu.set_properties(**fx["properties"])
    ids = build(gpu, edges)
    assert gpu.batch_optimize() == fx["oracle"]["iterations"]
    assert abs(gpu.chi2() - fx["oracle"]["chi2_final"]) <= 1e-8 * fx["oracle"]["chi2_final"]
    P = gpu.get_poses(np.array([ids[k] for k in fx["oracle"]["pose_index"]]))
    Po = np.array(fx["oracle"]["poses"])
    assert np.abs(P[:, :3] - Po[:, :3]).max() <= 1e-6 * max(1.0, np.abs(Po[:, :3]).max())


def solve_with(g, team, cluster):
    a = GpuGraphAPI()
    a.set_linear_solver(True)
    ids = gg.build_bulk(a, g)
    gg.configure(a, g)
    o = a.get_solver_options()
    o.team_ctas = team
    o.reserved[2] = 0 if cluster else (1 << 16)   # bit 16: global-memory barrier team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    a.batch_optimize()
    return a, ids, np.concatenate([a.get_poses(ids["pose_ids"]).ravel(), a.get_planes(ids["plane_ids"]).ravel()]), a.trace()


def test_bit_identical_across_team_shapes():
    g = gg.make_config(2, seed=0)
    ref = None
    for team in (1, 2, 8, 16):
        for cluster in (True, False):
            a, ids, x, t = solve_with(g, team, cluster)
            if ref is None:
                ref = (x, t)
                a2, _, x2, t2 = solve_with(g, team, cluster)
                assert np.array_equal(x, x2)
                continue
            assert np.array_equal(x, ref[0]), (team, cluster)
            for k in ("lam", "accepted", "pcg"):
                assert np.array_equal(t[k], ref[1][k]), (team, cluster, k)
            # chi2 and |delta| are sums of the existing team reduction, whose order follows the team size: last bits only
            for k in ("chi2_new", "delta_norm"):
                assert np.allclose(t[k], ref[1][k], rtol=1e-14, atol=0), (team, cluster, k)


def test_mixed_batch_matches_single_solves():
    graphs = [gg.make_config(2, seed=s, n_poses=120, n_planes=24) for s in range(6)]
    many, single = [], []
    for i, g in enumerate(graphs):
        for lst in (many, single):
            a = GpuGraphAPI()
            a.set_linear_solver(i % 2 == 0)
            ids = gg.build_bulk(a, g)
            gg.configure(a, g)
            a.set_solver_options(team_ctas=2)
            lst.append((a, ids))
    its = capi.batch_optimize_many([a for a, _ in many])
    for (a, ids), (b, _), it in zip(many, single, its):
        assert b.batch_optimize() == it
        assert np.array_equal(a.get_poses(ids["pose_ids"]), b.get_poses(ids["pose_ids"]))
        assert np.array_equal(a.get_planes(ids["plane_ids"]), b.get_planes(ids["plane_ids"]))
        assert np.array_equal(a.trace()["chi2_new"], b.trace()["chi2_new"])


def test_spanning_refuses_direct_mode():
    g = gg.make_config(1, seed=0)
    hs = []
    for _ in range(2):
        a = GpuGraphAPI()
        a.set_linear_solver(True)
        gg.build_bulk(a, g)
        gg.configure(a, g)
        hs.append(a)
    arr = capi._handles(hs)
    its = np.zeros(1, dtype=np.int32)
    rc = hs[0].lib.pus_span_emulate_optimize(arr, 2, capi._ip(its))
    assert rc < 0 and b"direct" in hs[0].lib.pus_last_error()
    assert hs[0].stats()["gpu_launches"] == 0


REF = json.load(open(os.path.join(HERE, "golden", "reference_build.json")))


def _qdiff(a, b):
    a, b = np.asarray(a), np.asarray(b)
    s = np.sign(np.sum(a[..., 3:] * b[..., 3:], axis=-1))[..., None]
    return max(np.abs(a[..., :3] - b[..., :3]).max(), np.abs(a[..., 3:] * s - b[..., 3:]).max())


@pytest.mark.parametrize("name", ["config1_seed0", "config2_seed0", "config3_small_huber"])
def test_reference_jacobian_and_direct_mode_follow_the_reference_on_every_trial_step(name):
    """Reference-Jacobian mode + direct mode against the reference's own LM runs (tests/golden/reference_build.json): same
    iterations and lambda / accept / reject sequence; chi2 of every trial step the fixture records within 1e-6, and of every
    trial step, rejected ones included, within 1e-6 of the oracle in the reference's mode (numerical Jacobians, exact solve;
    the CPU suite pins that oracle to the same fixture); final chi2 and estimates within 1e-4."""
    r = REF["runs"][name]
    g = gg.make_config(r["config"], seed=r["seed"], **r["kw"])
    gpu, orc = GpuGraphAPI(), OracleAPI()
    gpu.set_jacobian_mode(0)          # GpuGraphAPI convention: 0 = the reference's numerical differences
    gpu.set_linear_solver(True)
    orc.set_jacobian_mode(0)
    orc.set_reuse_ordering(1)
    builder = gg.build_interleaved if r["builder"] == "build_interleaved" else gg.build_bulk
    ids, _ = builder(gpu, g), builder(orc, g)
    gg.configure(gpu, g)
    gg.configure(orc, g)
    assert gpu.batch_optimize() == r["iterations"] == orc.batch_optimize()
    tr, to = gpu.trace(), orc.trace()
    assert tr["accepted"].tolist() == r["accepted"] == to["accepted"].tolist()
    assert np.allclose(tr["lam"], r["lambda_trace"], rtol=1e-12)
    e_fix = max([abs(a - b) / b for a, b in zip(tr["chi2_new"], r["chi2_trace"]) if b is not None] + [0.0])
    e_all = step_err(tr["chi2_new"], to["chi2_new"])
    e_fin = abs(gpu.chi2() - r["chi2_final"]) / r["chi2_final"]
    P, L = gpu.get_poses(ids["pose_ids"]), gpu.get_planes(ids["plane_ids"])
    e_p = _qdiff(P[::r["stride"]], r["poses"]) / max(1.0, np.abs(np.array(r["poses"])[:, :3]).max())
    sg = np.sign(np.sum(L[::r["plane_stride"]] * np.array(r["planes"]), axis=1))[:, None]
    e_l = np.abs(L[::r["plane_stride"]] * sg - np.array(r["planes"])).max()
    print(f"{name}: chi2 vs fixture {e_fix:.2e}, every step vs oracle {e_all:.2e}, final {e_fin:.2e}, poses {e_p:.2e}, planes {e_l:.2e}")
    assert e_fix <= 1e-6 and e_all <= 1e-6
    assert e_fin <= 1e-4 and e_p <= 1e-4 and e_l <= 1e-4


def test_facade_replay_with_the_direct_solver(tmp_path):
    """tests/facade_direct_replay.cpp: the façade replay with Slam::set_linear_solver(LINEAR_SOLVER_DIRECT), against the
    closed-form oracle replaying the same frame sequence (batch every 5th frame, update() otherwise)."""
    from test_facade import write_frames
    from pop_up_slam_b200 import geometry as geo
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "facade_direct_replay")
    libdir = os.path.join(root, "pop_up_slam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", exe, os.path.join(HERE, "facade_direct_replay.cpp"),
                           "-L" + libdir, "-lpopup_gpu", "-Wl,-rpath," + libdir])
    g = gg.make_config(2, seed=6, n_poses=30, n_planes=10, sigma_mode="reference")
    sig = 1.0 / g.pp_sqrtinf[:, 0]
    path = tmp_path / "frames.txt"
    write_frames(g, path, sig.tolist())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, check=True).stdout.splitlines()
    chi2 = [float(t.split()[1]) for t in out if t.startswith("chi2")][0]
    poses = np.array([[float(x) for x in t.split()[1:]] for t in out if t.startswith("pose")])
    planes = np.array([[float(x) for x in t.split()[1:]] for t in out if t.startswith("plane")])
    o = OracleAPI()
    o.set_jacobian_mode(1)
    o.set_properties(**dict(gg.PPS_PROPERTIES))
    order = np.argsort(g.pp_pose, kind="stable")
    ptr = np.searchsorted(g.pp_pose[order], np.arange(g.n_poses + 1))
    pose_ut = gg.diag_ut([0.5] * 6)
    pid, lid = [], {}
    for i in range(g.n_poses):
        pid.append(o.add_pose(None))
        if i == 0:
            o.add_pose_prior(pid[0], g.prior_meas, pose_ut)
        else:
            o.add_odometry(pid[i - 1], pid[i], g.odo_meas[i - 1], pose_ut)
        for e in order[ptr[i]:ptr[i + 1]]:
            k = int(g.pp_plane[e])
            if k not in lid:
                lid[k] = o.add_plane(None)
                o.init_plane(lid[k], geo.plane_to_global(geo.pose7_to_T(o.get_pose(pid[i])), g.pp_meas[e]))
                if k == g.ground_plane:
                    o.add_plane_prior(lid[k], [0, 0, -1, 0], gg.diag_ut([20.0] * 3))
            o.add_pose_plane(pid[i], lid[k], g.pp_meas[e], gg.diag_ut([1.0 / sig[e]] * 3))
        if i % 5 == 0:
            o.batch_optimize()
        else:
            o.update()
    c_o = o.chi2()
    e_c = abs(chi2 - c_o) / c_o
    P_o = o.get_poses(pid)
    L_o = o.get_planes([lid[k] for k in sorted(lid, key=lambda k: lid[k])])
    sgn = np.sign(np.sum(planes * L_o, axis=1))[:, None]
    e_x = max(_qdiff(poses, P_o) / max(1.0, np.abs(P_o[:, :3]).max()), np.abs(planes * sgn - L_o).max())
    print(f"façade replay, direct mode: chi2 {e_c:.2e}, estimates {e_x:.2e}")
    assert e_c <= 1e-8 and e_x <= 1e-8


def with_isolated_pose(api, g):
    """config 1 plus one pose no factor touches: its diagonal block of S is exactly zero, so every factorization meets a
    zero pivot whatever the damping (the diagonal is scaled by 1 + lambda)"""
    ids = gg.build_bulk(api, g)
    gg.configure(api, g)
    api.add_pose(api.get_pose(int(ids["pose_ids"][0])))
    return ids


def test_failed_factorization():
    g = gg.make_config(1, seed=0)
    # debug stage: the step is delta = 0
    a = GpuGraphAPI()
    a.set_linear_solver(True)
    ids = with_isolated_pose(a, g)
    a.upload()
    a.debug_run_stage(2, 1e-3)
    assert np.all(a.debug_fetch("delta", 6 * (g.n_poses + 1) + 3 * g.n_planes) == 0.0)
    # LM: every trial step is a zero step with pcg = -1 (LM goes on to max_iterations instead of stopping on |delta| = 0),
    # and the estimates stay where they were (up to the rounding of the exmap of a zero step)
    a = GpuGraphAPI()
    a.set_linear_solver(True)
    ids = with_isolated_pose(a, g)
    a.set_properties(**dict(gg.PPS_PROPERTIES, max_iterations=5))
    P0 = a.get_poses(ids["pose_ids"])
    assert a.batch_optimize() == 5
    t = a.trace()
    assert np.all(t["pcg"] == -1) and np.all(t["delta_norm"] == 0.0)
    assert t["lam"][0] == 1e-6 and (t["accepted"][0] == 1 or np.isclose(t["lam"][1], 1e-5, rtol=1e-12))
    assert np.abs(a.get_poses(ids["pose_ids"]) - P0).max() < 1e-12
    # GN stops at once (|delta| = 0 <= epsilon2); update() applies delta = 0
    for which in ("gn", "update"):
        a = GpuGraphAPI()
        a.set_linear_solver(True)
        ids = with_isolated_pose(a, g)
        a.set_properties(**dict(gg.PPS_PROPERTIES, method=0))
        P0 = a.get_poses(ids["pose_ids"])
        if which == "gn":
            assert a.batch_optimize() == 0
        else:
            a.update()
        assert np.abs(a.get_poses(ids["pose_ids"]) - P0).max() < 1e-12
