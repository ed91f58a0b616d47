"""The band direct solve in nested-dissection order (pus_set_linear_solver(h, 2) + pus_set_direct_ordering(h, 1)): its stages
against numpy on the bordered reduced system of the oracle's normal equations, whole LM / GN / update solves against the
closed-form oracle on every trial step, agreement with the insertion-order band solve, reference-Jacobian mode against the
reference's own LM run, bit-identical solves across team shapes and in a batch mixing every kind, ill-conditioned SPD
matrices with a non-band pattern through stage 5, a failed factorization, the refusals, and a revisited map that the
insertion-order layout cannot hold."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse.linalg as spl

from oracle_api import OracleAPI
from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI
from test_gpu_band_solve import build_edges, build_graph, pose_chain, sphere_edges
from test_gpu_direct_accuracy import check, lapack_factors
from test_gpu_direct_solve import REF, STAGE_CASES, _qdiff, estimates_match, relerr, step_err, trace_match

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def nd_api(kind=2, order=1):
    a = GpuGraphAPI()
    a.set_linear_solver(kind)
    a.set_direct_ordering(order)
    return a


ND_CASES = {
    "config1": STAGE_CASES["config1"], "config2": STAGE_CASES["config2"], "n7": STAGE_CASES["n7"],
    "corridor1200": lambda: gg.make_config(3, seed=0, n_poses=1200, n_planes=120),
    "revisit600": lambda: gg.make_revisit(seed=0, n_poses=600, n_planes=40),
}


def build_case(api, case):
    if case in ND_CASES:
        g = ND_CASES[case]()
        info = gg.build_bulk(api, g)
        gg.configure(api, g)
        return info, g.n_poses, g.n_planes
    return build_graph(api, case)


def row_order(n6, nbp, perm, nk):
    """the rows of the bordered order (6 N poses, then 3 per bordered plane) sorted by their row in the permuted layout"""
    pos = np.argsort(perm)
    padded = np.array([r if r < n6 else 48 * nbp + r - n6 for r in range(nk)])
    newrow = 48 * pos[padded // 48] + padded % 48
    return np.argsort(newrow, kind="stable"), newrow


@pytest.mark.parametrize("case", list(ND_CASES) + ["sphere400", "several"])
@pytest.mark.parametrize("lam", [0.0, 1e-6, 1e-2])
def test_stages_match_numpy(case, lam):
    gpu, orc = nd_api(), OracleAPI()
    orc.set_jacobian_mode(1)
    _, N, M = build_case(gpu, case)
    build_case(orc, case)
    gpu.upload()
    border = gpu.debug_fetch("bborder", 1 << 16).astype(int).tolist()
    perm = gpu.debug_fetch("ndtile", 1 << 20).astype(int)
    cptr, crow = gpu.debug_fetch("ndcptr", 1 << 20).astype(int), gpu.debug_fetch("ndcrow", 1 << 24).astype(int)
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
    p, newrow = row_order(n, max(1, (n + 47) // 48), perm, nk)
    Lr = np.linalg.cholesky(S[np.ix_(p, p)])
    e_l = relerr(L, Lr)
    # L's tile pattern: numpy's factor is zero outside it (the fetch gives 0 there; the tiles are not stored)
    nbt = len(perm)
    stored = np.zeros((nbt, nbt), dtype=bool)
    for j in range(nbt):
        stored[crow[cptr[j]:cptr[j + 1]], j] = True
    t = newrow[p] // 48
    outside = ~stored[t[:, None], t[None, :]] & (np.arange(nk)[:, None] >= np.arange(nk)[None, :])
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
    if case == "corridor1200" and lam < 1e-2:   # (as for the insertion order: too ill-conditioned for a forward-error bar)
        assert res < 1e-12
    else:
        assert e_d < 1e-10


def lm_pair(g, interleaved=False):
    gpu, orc = nd_api(), OracleAPI()
    orc.set_jacobian_mode(1)
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
    print(f"{n}-pose Huber corridor, ND order: chi2 per step {e_t:.2e}, estimates {e_x:.2e}")


def test_revisited_corridor_matches_oracle_on_every_trial_step():
    g = gg.make_revisit(seed=0, n_poses=2000, n_planes=100, max_iterations=8)
    gpu, orc, ig, io = lm_pair(g)
    assert gpu.batch_optimize() == orc.batch_optimize()
    e_t = trace_match(gpu, orc, rtol=1e-9)
    e_x = estimates_match(gpu, orc, ig, io, tol=1e-8)
    print(f"revisited 2000-pose corridor, ND order: chi2 per step {e_t:.2e}, estimates {e_x:.2e}")


def test_sphere2500_matches_oracle_on_every_trial_step():
    edges, props = sphere_edges("sphere2500")
    gpu, orc = nd_api(), OracleAPI()
    orc.set_jacobian_mode(1)
    ids = []
    for api in (gpu, orc):
        api.set_properties(**props)
        d = build_edges(api, edges)
        ids.append(np.array([d[k] for k in sorted(d)]))
    assert gpu.batch_optimize() == orc.batch_optimize()
    e_t = trace_match(gpu, orc, rtol=1e-9)
    P_g, P_o = gpu.get_poses(ids[0]), orc.get_poses(ids[1])
    e_x = _qdiff(P_g, P_o) / max(1.0, np.abs(P_o[:, :3]).max())
    print(f"sphere2500, ND order: chi2 per step {e_t:.2e}, estimates {e_x:.2e}")
    assert e_x <= 1e-8


def test_gauss_newton_and_update_match_oracle():
    g = gg.make_revisit(seed=1, n_poses=1200, n_planes=60)
    for which in ("gn", "update"):
        gpu, orc = nd_api(), OracleAPI()
        orc.set_jacobian_mode(1)
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


def _nd_vs_insertion(g):
    runs = []
    for order in (0, 1):
        a = nd_api(order=order)
        gg.build_bulk(a, g)
        gg.configure(a, g)
        its = a.batch_optimize()
        runs.append((its, a.trace()))
    (i1, t1), (i2, t2) = runs
    assert i1 == i2
    assert np.array_equal(t1["accepted"], t2["accepted"]) and np.array_equal(t1["lam"], t2["lam"])
    e = step_err(t2["chi2_new"], t1["chi2_new"])
    assert e <= 1e-10, e


@pytest.mark.parametrize("make", [lambda s: gg.make_config(1, seed=s), lambda s: gg.make_config(2, seed=s)], ids=["config1", "config2"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_nd_matches_insertion_order(make, seed):
    _nd_vs_insertion(make(seed))


def test_nd_matches_insertion_order_on_the_600_pose_corridor():
    _nd_vs_insertion(gg.make_config(3, seed=0, n_poses=600, n_planes=60, max_iterations=8))


def test_reference_jacobian_nd_mode_follows_the_reference_on_every_trial_step():
    r = REF["runs"]["config3_full_20it"]
    g = gg.make_config(r["config"], seed=r["seed"], **r["kw"])
    gpu = nd_api()
    gpu.set_jacobian_mode(0)
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
    print(f"config3_full_20it, ND order: chi2 per step vs fixture {e_fix:.2e}, final {e_fin:.2e}, poses {e_p:.2e}, planes {e_l:.2e}")
    assert e_fix <= 1e-9 and e_fin <= 1e-10
    assert e_p <= 1e-8 and e_l <= 1e-8


def solve_with(g, team, cluster):
    a = nd_api()
    ids = gg.build_bulk(a, g)
    gg.configure(a, g)
    o = a.get_solver_options()
    o.team_ctas = team
    o.reserved[2] = 0 if cluster else (1 << 16)   # bit 16: global-memory barrier team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    a.batch_optimize()
    return np.concatenate([a.get_poses(ids["pose_ids"]).ravel(), a.get_planes(ids["plane_ids"]).ravel()]), a.trace()


def test_bit_identical_across_team_shapes():
    g = gg.make_revisit(seed=0, n_poses=600, n_planes=40, max_iterations=5)
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
    """PCG, dense, band in insertion order and band in ND order in one batch"""
    graphs = [gg.make_config(2, seed=s, n_poses=120, n_planes=24) for s in range(8)]
    kinds = [(0, 0), (1, 0), (2, 0), (2, 1)]
    many, single = [], []
    for i, g in enumerate(graphs):
        for lst in (many, single):
            a = nd_api(*kinds[i % 4])
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


# ---------------------------------------------------------------- stage 5 on stored matrices of the ND layout
_CARRIER = {}


def carrier():
    """an uploaded ND-order pose graph of 160 poses (no planes, loop closures): its tile pattern fixes where a stored S may
    have entries"""
    if not _CARRIER:
        edges, props = pose_chain(160)
        a = nd_api()
        a.set_properties(**props)
        build_edges(a, edges)
        a.upload()
        perm = a.debug_fetch("ndtile", 1 << 10).astype(int)
        cptr, crow = a.debug_fetch("ndcptr", 1 << 10).astype(int), a.debug_fetch("ndcrow", 1 << 14).astype(int)
        nbt = len(perm)
        stored = np.zeros((nbt, nbt), dtype=bool)
        for j in range(nbt):
            stored[crow[cptr[j]:cptr[j + 1]], j] = True
        _CARRIER["a"] = (a, perm, stored)
    return _CARRIER["a"]


def pattern_spd(n, perm, stored, p, rng):
    """P^T (L0 D L0^T) P with L0 unit lower triangular, non-zero only inside L's tile pattern in the permuted order, and D
    log-uniform in [10^-p, 1]: an SPD matrix with a non-band pattern whose factor keeps to the pattern"""
    L0 = np.tril(rng.standard_normal((n, n)) / (2.0 * np.sqrt(n)), -1) + np.eye(n)
    t = np.arange(n) // 48
    L0[~stored[t[:, None], t[None, :]]] = 0.0
    d = 10.0 ** (-p * rng.random(n))
    d[0], d[-1] = 1.0, 10.0 ** -p
    Sp = (L0 * d) @ L0.T
    Sp = 0.5 * (Sp + Sp.T)
    newrow = 48 * np.argsort(perm)[np.arange(n) // 48] + np.arange(n) % 48   # original row -> permuted row
    return Sp[np.ix_(newrow, newrow)], newrow


@pytest.mark.parametrize("p", [0, 8, 12, 14])
def test_pattern_matrices_through_stage_5(p):
    a, perm, stored = carrier()
    n = 6 * 160
    rng = np.random.default_rng(200 + p)
    S, newrow = pattern_spd(n, perm, stored, p, rng)
    b = rng.standard_normal(n)
    assert lapack_factors(S)
    a.debug_store("Sdir", S)
    a.debug_store("b", b)
    a.debug_run_stage(5)
    assert int(a.debug_fetch("dflag", 1)[0]) == 0
    L = a.debug_fetch("Ldir", n * n).reshape(n, n)
    x = a.debug_fetch("x", n)
    q = np.argsort(newrow)   # the permuted order's rows
    check(f"ND pattern p={p}", S[np.ix_(q, q)], b[q], L, x[q], p)


def test_indefinite_stored_matrix_sets_dflag():
    a, perm, stored = carrier()
    n = 6 * 160
    rng = np.random.default_rng(3)
    S, _ = pattern_spd(n, perm, stored, 4, rng)
    S[500, 500] = -1.0
    a.debug_store("Sdir", S)
    a.debug_store("b", rng.standard_normal(n))
    a.debug_run_stage(5)
    assert int(a.debug_fetch("dflag", 1)[0]) == 1


def test_stored_matrix_outside_the_pattern_is_refused():
    a, perm, stored = carrier()
    n = 6 * 160
    pos = np.argsort(perm)
    nbt = len(perm)
    i, j = next((i, j) for i in range(nbt) for j in range(i) if not stored[i, j])
    r, q = 48 * perm[i], 48 * perm[j]   # original rows of the permuted tiles (i, j)
    S = np.eye(n)
    S[r, q] = S[q, r] = 1e-3
    assert pos[r // 48] == i
    with pytest.raises(capi.ApiError, match="outside the nested-dissection pattern"):
        a.debug_store("Sdir", S)


# ---------------------------------------------------------------- refusals and the revisited map
def test_spanning_refuses_nd_mode():
    g = gg.make_config(1, seed=0)
    hs = []
    for _ in range(2):
        a = nd_api()
        gg.build_bulk(a, g)
        gg.configure(a, g)
        hs.append(a)
    arr = capi._handles(hs)
    its = np.zeros(1, dtype=np.int32)
    rc = hs[0].lib.pus_span_emulate_optimize(arr, 2, capi._ip(its))
    assert rc < 0 and b"direct" in hs[0].lib.pus_last_error()
    assert hs[0].stats()["gpu_launches"] == 0


def test_revisited_map_over_the_band_budget_solves_exactly():
    """20 000 poses driven twice over: insertion order is refused over its budget; the ND order solves it, and one LM run
    capped at three iterations ends at the oracle's chi2"""
    g = gg.make_revisit(seed=0, n_poses=20000, n_planes=1000, max_iterations=3)
    band = nd_api(order=0)
    gg.build_bulk(band, g)
    gg.configure(band, g)
    with pytest.raises(capi.ApiError, match="band linear solver: the graph needs"):
        band.batch_optimize()
    gpu, orc, ig, io = lm_pair(g)
    it_g, it_o = gpu.batch_optimize(), orc.batch_optimize()
    c_g, c_o = gpu.chi2(), orc.chi2()
    print(f"revisited 20000 poses, ND order: {it_g} iterations, chi2 {c_g:.12g} vs oracle {c_o:.12g}, "
          f"{gpu.debug_fetch('bbytes', 1)[0] / 2**30:.2f} GiB")
    assert it_g == it_o
    assert abs(c_g - c_o) <= 1e-9 * c_o



def test_facade_replay_with_the_nd_order(tmp_path):
    """tests/facade_nd_replay.cpp: the façade replay with Slam::set_direct_ordering(ORDERING_NESTED_DISSECTION) on a band
    façade over 700 poses, against the closed-form oracle replaying the same frame sequence"""
    import subprocess
    from test_facade import write_frames
    from pop_up_slam_b200 import geometry as geo
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "facade_nd_replay")
    libdir = os.path.join(root, "pop_up_slam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", exe, os.path.join(HERE, "facade_nd_replay.cpp"),
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
    e_x = max(_qdiff(poses, P_o) / max(1.0, np.abs(P_o[:, :3]).max()), np.abs(planes * sgn - L_o).max())
    print(f"façade replay, ND order, 700 poses: chi2 {e_c:.2e}, estimates {e_x:.2e}")
    assert e_c <= 1e-8 and e_x <= 1e-8
