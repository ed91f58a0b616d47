"""The band direct linear solve (pus_set_linear_solver(h, 2)): its stages against numpy on the bordered reduced system of the
oracle's normal equations, whole LM / GN / update solves against the closed-form oracle and against the dense direct solve
on every trial step, reference-Jacobian mode against the reference's own LM runs, bit-identical solves across team shapes and
in a batch mixing every kind, a failed factorization, banded ill-conditioned matrices through stage 5, the refusals, and a
façade replay over 640 poses."""
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
from test_gpu_direct_accuracy import check, lapack_factors
from test_gpu_direct_solve import STAGE_CASES, REF, _qdiff, estimates_match, relerr, step_err, trace_match

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
from make_sphere_golden import build as build_edges, load_edge3  # noqa: E402


def sphere_edges(name):
    if name == "sphere400":
        fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
        return [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]], fx["properties"]
    return load_edge3(os.path.join(HERE, "golden", "sphere2500.txt.xz")), dict(gg.PPS_PROPERTIES, max_iterations=6)


def several_walls():
    """a corridor whose ground plane and three more planes are seen from every pose: several bordered planes"""
    g = gg.make_config(3, seed=2, n_poses=400, n_planes=60)
    extra = [(p, l) for l in (1, 2, 3) for p in range(0, 400, 2)]
    return g, extra


def pose_chain(n):
    """the first n poses of sphere400 and the edges among them: a graph with no planes"""
    edges, props = sphere_edges("sphere400")
    return [e for e in edges if e[0] < n and e[1] < n], props


def build_graph(api, case):
    """builds the case on api; returns (ids, number of poses, number of planes)"""
    if case in ("sphere400", "noplanes"):
        edges, props = sphere_edges(case) if case == "sphere400" else pose_chain(100)
        api.set_properties(**props)
        ids = build_edges(api, edges)
        return dict(pose_ids=np.array([ids[k] for k in sorted(ids)]), plane_ids=np.zeros(0, dtype=int)), len(ids), 0
    if case == "several":
        g, extra = several_walls()
        info = gg.build_bulk(api, g)
        for p, l in extra:
            e = int(np.nonzero(g.pp_plane == l)[0][0])
            api.add_pose_plane(int(info["pose_ids"][p]), int(info["plane_ids"][l]), g.pp_meas[e], g.pp_sqrtinf[e])
        gg.configure(api, g)
        return info, g.n_poses, g.n_planes
    g = BAND_CASES[case]()
    info = gg.build_bulk(api, g)
    gg.configure(api, g)
    return info, g.n_poses, g.n_planes


BAND_CASES = dict(STAGE_CASES)
BAND_CASES.update({
    "corridor1200": lambda: gg.make_config(3, seed=0, n_poses=1200, n_planes=120),
})


def band_pair(case):
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    gpu.set_linear_solver(2)
    ig, N, M = build_graph(gpu, case)
    io, _, _ = build_graph(orc, case)
    return gpu, orc, ig, io, N, M


@pytest.mark.parametrize("case", list(BAND_CASES) + ["sphere400", "noplanes", "several"])
@pytest.mark.parametrize("lam", [0.0, 1e-6, 1e-2])
def test_stages_match_numpy(case, lam):
    gpu, orc, ig, io, N, M = band_pair(case)
    gpu.upload()
    border = gpu.debug_fetch("bborder", 1 << 16).astype(int).tolist()
    first = gpu.debug_fetch("bfirst", 1 << 20).astype(int)
    if case in ("corridor1200", "several"):
        assert len(border) >= (4 if case == "several" else 1)
    A, b = orc.normal_equations(lam)
    A = A.tocsc()
    n = 6 * N
    keep = np.concatenate([np.arange(n), [n + 3 * l + m for l in border for m in range(3)]]).astype(int)
    elim = np.setdiff1d(np.arange(n + 3 * M), keep)
    Akk, Ake, Aee = A[keep][:, keep].toarray(), A[keep][:, elim], A[elim][:, elim]
    S = Akk - (Ake @ spl.spsolve(Aee.tocsc(), Ake.T.tocsc())).toarray() if len(elim) else Akk
    nk = len(keep)
    gpu.debug_run_stage(4, lam)
    Sd = gpu.debug_fetch("Sdir", nk * nk).reshape(nk, nk)
    e_s = relerr(Sd, np.tril(S))
    gpu.debug_run_stage(1, lam)
    L = gpu.debug_fetch("Ldir", nk * nk).reshape(nk, nk)
    Lr = np.linalg.cholesky(S)
    e_l = relerr(L, Lr)
    # the envelope: the reference factor has no fill outside it (the fetch gives 0 there; the tiles are not stored)
    row_tile = np.array([r // 48 if r < n else (48 * ((n + 47) // 48) + r - n) // 48 for r in range(nk)])
    outside = row_tile[None, :] < first[row_tile][:, None]
    assert np.all(L[outside] == 0.0)
    assert np.abs(Lr[outside]).max(initial=0.0) <= 1e-12 * np.abs(Lr).max()
    gpu.debug_run_stage(2, lam)
    got = gpu.debug_fetch("delta", n + 3 * M)
    ref = spl.spsolve(A, b)
    e_d = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    res = np.linalg.norm(A @ got - b) / (spl.norm(A, 1) * np.linalg.norm(got))
    print(f"{case} lam={lam}: border {len(border)}  S {e_s:.2e}  L {e_l:.2e}  delta {e_d:.2e}  residual {res:.2e}")
    assert e_s < 1e-12
    assert e_l < 1e-10
    if case == "corridor1200" and lam < 1e-2:
        # the undamped 1 200-pose corridor is too ill-conditioned for a forward-error bar against spsolve (which has the
        # same rounding): the scaled residual shows the solve is backward stable
        assert res < 1e-12
    else:
        assert e_d < 1e-10


def lm_pair(g, kind=2, interleaved=False):
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    gpu.set_linear_solver(kind)
    out = []
    for api in (gpu, orc):
        out.append(gg.build_interleaved(api, g) if interleaved else gg.build_bulk(api, g))
        gg.configure(api, g)
    return gpu, orc, out[0], out[1]


@pytest.mark.parametrize("n", [1200, 2000])
def test_huber_corridor_matches_oracle_on_every_trial_step(n):
    g = gg.make_config(3, seed=0, n_poses=n, n_planes=n // 10, max_iterations=8)
    gpu, orc, ig, io = lm_pair(g)
    assert gpu.batch_optimize() == orc.batch_optimize()
    e_t = trace_match(gpu, orc, rtol=1e-9)
    e_x = estimates_match(gpu, orc, ig, io, tol=1e-8)
    print(f"{n}-pose Huber corridor: chi2 per step {e_t:.2e}, estimates {e_x:.2e}")


def test_sphere2500_matches_oracle_on_every_trial_step():
    edges, props = sphere_edges("sphere2500")
    gpu, orc = GpuGraphAPI(), OracleAPI()
    orc.set_jacobian_mode(1)
    gpu.set_linear_solver(2)
    ids = []
    for api in (gpu, orc):
        api.set_properties(**props)
        d = build_edges(api, edges)
        ids.append(np.array([d[k] for k in sorted(d)]))
    assert gpu.batch_optimize() == orc.batch_optimize()
    e_t = trace_match(gpu, orc, rtol=1e-9)
    P_g, P_o = gpu.get_poses(ids[0]), orc.get_poses(ids[1])
    e_x = _qdiff(P_g, P_o) / max(1.0, np.abs(P_o[:, :3]).max())
    print(f"sphere2500: chi2 per step {e_t:.2e}, estimates {e_x:.2e}")
    assert e_x <= 1e-8


def test_gauss_newton_and_update_match_oracle():
    g = gg.make_config(3, seed=1, n_poses=1200, n_planes=120)
    for which in ("gn", "update"):
        gpu, orc = GpuGraphAPI(), OracleAPI()
        orc.set_jacobian_mode(1)
        gpu.set_linear_solver(2)
        ig, io = gg.build_bulk(gpu, g), gg.build_bulk(orc, g)
        gg.configure(gpu, g, method=0, max_iterations=5)
        gg.configure(orc, g, method=0, max_iterations=5)
        if which == "gn":
            assert gpu.batch_optimize() == orc.batch_optimize()
            trace_match(gpu, orc, rtol=1e-9)
        else:
            for _ in range(3):
                gpu.update()
                orc.update()
        estimates_match(gpu, orc, ig, io, tol=1e-8)


@pytest.mark.parametrize("make", [lambda s: gg.make_config(1, seed=s), lambda s: gg.make_config(2, seed=s)], ids=["config1", "config2"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_band_matches_dense(make, seed):
    g = make(seed)
    _band_vs_dense(g)


def test_band_matches_dense_on_the_600_pose_corridor():
    _band_vs_dense(gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=8))


def _band_vs_dense(g):
    runs = []
    for kind in (1, 2):
        a = GpuGraphAPI()
        a.set_linear_solver(kind)
        gg.build_bulk(a, g)
        gg.configure(a, g)
        its = a.batch_optimize()
        runs.append((its, a.trace()))
    (i1, t1), (i2, t2) = runs
    assert i1 == i2
    assert np.array_equal(t1["accepted"], t2["accepted"]) and np.array_equal(t1["lam"], t2["lam"])
    e = step_err(t2["chi2_new"], t1["chi2_new"])
    assert e <= 1e-10, e


@pytest.mark.parametrize("name", ["config3_small_huber", "config3_full_20it"])
def test_reference_jacobian_band_mode_follows_the_reference_on_every_trial_step(name):
    r = REF["runs"][name]
    g = gg.make_config(r["config"], seed=r["seed"], **r["kw"])
    gpu = GpuGraphAPI()
    gpu.set_jacobian_mode(0)
    gpu.set_linear_solver(2)
    builder = gg.build_interleaved if r["builder"] == "build_interleaved" else gg.build_bulk
    ids = builder(gpu, g)
    gg.configure(gpu, g)
    assert gpu.batch_optimize() == r["iterations"]
    tr = gpu.trace()
    assert tr["accepted"].tolist() == r["accepted"]
    assert np.allclose(tr["lam"], r["lambda_trace"], rtol=1e-12)
    e_fix = max([abs(a - b) / b for a, b in zip(tr["chi2_new"], r["chi2_trace"]) if b is not None] + [0.0])
    e_fin = abs(gpu.chi2() - r["chi2_final"]) / r["chi2_final"]
    P, L = gpu.get_poses(ids["pose_ids"]), gpu.get_planes(ids["plane_ids"])
    e_p = _qdiff(P[::r["stride"]], r["poses"]) / max(1.0, np.abs(np.array(r["poses"])[:, :3]).max())
    sg = np.sign(np.sum(L[::r["plane_stride"]] * np.array(r["planes"]), axis=1))[:, None]
    e_l = np.abs(L[::r["plane_stride"]] * sg - np.array(r["planes"])).max()
    print(f"{name}: chi2 per step vs fixture {e_fix:.2e}, final {e_fin:.2e}, poses {e_p:.2e}, planes {e_l:.2e}")
    assert e_fix <= 1e-9 and e_fin <= 1e-10
    assert e_p <= 1e-8 and e_l <= 1e-8


def solve_with(g, team, cluster, kind=2):
    a = GpuGraphAPI()
    a.set_linear_solver(kind)
    ids = gg.build_bulk(a, g)
    gg.configure(a, g)
    o = a.get_solver_options()
    o.team_ctas = team
    o.reserved[2] = 0 if cluster else (1 << 16)   # bit 16: global-memory barrier team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    a.batch_optimize()
    return np.concatenate([a.get_poses(ids["pose_ids"]).ravel(), a.get_planes(ids["plane_ids"]).ravel()]), a.trace()


def test_bit_identical_across_team_shapes():
    g = gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=5)
    ref = None
    for team in (1, 2, 3, 16, 10_000):   # (10 000: clamped to the device's maximum)
        for cluster in (True, False):
            x, t = solve_with(g, team, cluster)
            if ref is None:
                ref = (x, t)
                continue
            assert np.array_equal(x, ref[0]), (team, cluster)
            for k in ("lam", "accepted", "pcg"):
                assert np.array_equal(t[k], ref[1][k]), (team, cluster, k)
            for k in ("chi2_new", "delta_norm"):   # team-reduction sums: last bits only
                assert np.allclose(t[k], ref[1][k], rtol=1e-14, atol=0), (team, cluster, k)


def test_mixed_batch_of_every_kind_matches_single_solves():
    graphs = [gg.make_config(2, seed=s, n_poses=120, n_planes=24) for s in range(6)]
    many, single = [], []
    for i, g in enumerate(graphs):
        for lst in (many, single):
            a = GpuGraphAPI()
            a.set_linear_solver(i % 3)
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


# ---------------------------------------------------------------- stage 5 on stored matrices of the band layout
_CARRIER = {}


def carrier():
    """an uploaded band-mode pose graph of 160 poses (no planes, loop closures): its envelope fixes where a stored S may
    have entries"""
    if not _CARRIER:
        edges, props = pose_chain(160)
        a = GpuGraphAPI()
        a.set_linear_solver(2)
        a.set_properties(**props)
        build_edges(a, edges)
        a.upload()
        first = a.debug_fetch("bfirst", 1 << 10).astype(int)
        _CARRIER["a"] = (a, first)
    return _CARRIER["a"]


def band_spd(n, first, p, rng):
    """L0 D L0^T with L0 unit lower triangular, non-zero only inside the envelope, and D log-uniform in [10^-p, 1]: an SPD
    matrix whose factor keeps to the envelope and whose conditioning follows D"""
    L0 = np.tril(rng.standard_normal((n, n)) / (2.0 * np.sqrt(n)), -1) + np.eye(n)   # (a well-conditioned unit factor)
    t = np.arange(n) // 48
    L0[t[None, :] < first[t][:, None]] = 0.0
    d = 10.0 ** (-p * rng.random(n))
    d[0], d[-1] = 1.0, 10.0 ** -p
    S = (L0 * d) @ L0.T
    return 0.5 * (S + S.T)


@pytest.mark.parametrize("p", [0, 4, 8, 10, 12, 13, 14])
@pytest.mark.parametrize("seed", [0, 1])
def test_banded_matrices_through_stage_5(p, seed):
    if p in (0, 4, 10) and seed == 1:
        pytest.skip("one seed at the easy ends")
    a, first = carrier()
    n = 6 * 160
    rng = np.random.default_rng(100 * p + seed)
    S = band_spd(n, first, p, rng)
    b = rng.standard_normal(n)
    assert lapack_factors(S)
    a.debug_store("Sdir", S)
    a.debug_store("b", b)
    a.debug_run_stage(5)
    assert int(a.debug_fetch("dflag", 1)[0]) == 0
    L = a.debug_fetch("Ldir", n * n).reshape(n, n)
    x = a.debug_fetch("x", n)
    check(f"banded p={p} seed={seed}", S, b, L, x, seed)


def test_indefinite_stored_matrix_sets_dflag():
    a, first = carrier()
    n = 6 * 160
    rng = np.random.default_rng(3)
    S = band_spd(n, first, 4, rng)
    S[500, 500] = -1.0
    a.debug_store("Sdir", S)
    a.debug_store("b", rng.standard_normal(n))
    a.debug_run_stage(5)
    assert int(a.debug_fetch("dflag", 1)[0]) == 1


def test_stored_matrix_outside_the_envelope_is_refused():
    a, first = carrier()
    n = 6 * 160
    S = np.eye(n)
    S[n - 1, 0] = S[0, n - 1] = 1e-3
    with pytest.raises(capi.ApiError, match="outside the band layout's envelope"):
        a.debug_store("Sdir", S)


# ---------------------------------------------------------------- refusals
def test_over_budget_graph_fails_and_launches_nothing():
    gpu = GpuGraphAPI()
    gpu.set_linear_solver(2)
    ut = gg.diag_ut([1.0] * 6)
    ids = [gpu.add_pose(None)]
    gpu.add_pose_prior(ids[0], [0, 0, 0, 0, 0, 0], ut)
    for i in range(1, 20000):
        ids.append(gpu.add_pose(None))
        gpu.add_odometry(ids[0], ids[i], [0.1 * i, 0, 0, 0, 0, 0], ut)
    with pytest.raises(capi.ApiError, match="band linear solver: the graph needs"):
        gpu.batch_optimize()
    assert gpu.stats()["gpu_launches"] == 0


def test_spanning_refuses_band_mode():
    g = gg.make_config(1, seed=0)
    hs = []
    for _ in range(2):
        a = GpuGraphAPI()
        a.set_linear_solver(2)
        gg.build_bulk(a, g)
        gg.configure(a, g)
        hs.append(a)
    arr = capi._handles(hs)
    its = np.zeros(1, dtype=np.int32)
    rc = hs[0].lib.pus_span_emulate_optimize(arr, 2, capi._ip(its))
    assert rc < 0 and b"direct" in hs[0].lib.pus_last_error()
    assert hs[0].stats()["gpu_launches"] == 0


def test_facade_replay_with_the_band_solver(tmp_path):
    """tests/facade_band_replay.cpp: the façade replay with Slam::set_linear_solver(LINEAR_SOLVER_BAND) on 700 poses (over
    the dense solve's 640), against the closed-form oracle replaying the same frame sequence"""
    import test_gpu_direct_solve as tds
    from test_facade import write_frames
    from pop_up_slam_b200 import geometry as geo
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "facade_band_replay")
    libdir = os.path.join(root, "pop_up_slam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", exe, os.path.join(HERE, "facade_band_replay.cpp"),
                           "-L" + libdir, "-lpopup_gpu", "-Wl,-rpath," + libdir])
    g = gg.make_config(2, seed=6, n_poses=700, n_planes=70, sigma_mode="reference")
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
    e_x = max(tds._qdiff(poses, P_o) / max(1.0, np.abs(P_o[:, :3]).max()), np.abs(planes * sgn - L_o).max())
    print(f"façade replay, band mode, 700 poses: chi2 {e_c:.2e}, estimates {e_x:.2e}")
    assert e_c <= 1e-8 and e_x <= 1e-8
