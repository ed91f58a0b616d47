"""Accuracy of the direct solve's factorization on ill-conditioned systems (DESIGN.md section 5.1).

Debug stage 5 factors a dense S stored with pus_debug_store("Sdir") and solves for a stored b, so the conditioning of S is
chosen by the test.  Each GPU result is measured against a plain host reference of the same S: LAPACK's float64 Cholesky
(scipy.linalg.cho_factor), and a solution x* refined with residuals computed in long double.  The bars are calibrated per
matrix by LAPACK's own errors on the same S, so no device number has to be guessed:
  backward error of L      max over 8 Gaussian probes v of |(S - L L^T) v| / (|S|_F |v|)  <= 10 max(LAPACK's, 1e-16)
  forward error of x       |x - x*| / |x*|                                               <= 10 max(LAPACK's, 1e-15)
  scaled residual of x     |b - S x| / (|S|_F |x|)                                       <= 10 max(LAPACK's, 1e-16)
Then: the factorization succeeds wherever LAPACK's does, reports an indefinite S through "dflag", is bitwise identical across
team shapes, and the assembly + factorization + solve of real graphs whose Schur complement is ill-conditioned at lambda = 0
meets the same bars."""
import ctypes

import numpy as np
import pytest
import scipy.linalg as sla

from oracle_api import OracleAPI
from pop_up_slam_b200 import graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu
LD = np.longdouble
ROWS = 256   # row chunk of the long-double products (bounds their memory at order 3 840)


# ---------------------------------------------------------------- host reference
def matmul_ld(S, V):
    """S V with S converted to long double a row chunk at a time"""
    V = np.asarray(V, dtype=LD)
    out = np.empty((S.shape[0],) + V.shape[1:], dtype=LD)
    for r in range(0, S.shape[0], ROWS):
        out[r:r + ROWS] = S[r:r + ROWS].astype(LD) @ V
    return out


def refined_solve(S, b, cf, rounds=5):
    """x* = S^-1 b: LAPACK's solve refined with residuals b - S x in long double"""
    x = sla.cho_solve(cf, b).astype(LD)
    for _ in range(rounds):
        r = (np.asarray(b, dtype=LD) - matmul_ld(S, x)).astype(np.float64)
        x = x + sla.cho_solve(cf, r).astype(LD)
    return x


def backward_error(S, L, V, normS):
    """max over the probe columns v of |(S - L L^T) v| / (|S|_F |v|), long-double products only"""
    R = matmul_ld(S, V) - matmul_ld(L, matmul_ld(L.T, V))
    return float(np.max(np.linalg.norm(R.astype(np.float64), axis=0) / (normS * np.linalg.norm(V, axis=0))))


def errors(S, b, L, x, xs, V, normS):
    """(backward error of L, forward error of x against x*, scaled residual of x)"""
    xs64 = xs.astype(np.float64)
    fwd = float(np.linalg.norm((np.asarray(x, dtype=LD) - xs).astype(np.float64)) / np.linalg.norm(xs64))
    res = float(np.linalg.norm((np.asarray(b, dtype=LD) - matmul_ld(S, x)).astype(np.float64)) / (normS * np.linalg.norm(x)))
    return backward_error(S, L, V, normS), fwd, res


def check(name, S, b, L, x, seed=0):
    """the GPU's L and x against LAPACK's on the same S, by the calibrated bars; returns the GPU's errors"""
    cf = sla.cho_factor(S, lower=True)
    L_ref = np.tril(cf[0])
    xs = refined_solve(S, b, cf)
    V = np.random.default_rng(seed).standard_normal((S.shape[0], 8))
    normS = np.linalg.norm(S)
    g = errors(S, b, L, x, xs, V, normS)
    r = errors(S, b, L_ref, sla.cho_solve(cf, b), xs, V, normS)
    print(f"{name}: backward {g[0]:.1e} (LAPACK {r[0]:.1e})  forward {g[1]:.1e} ({r[1]:.1e})  residual {g[2]:.1e} ({r[2]:.1e})")
    assert g[0] <= 10 * max(r[0], 1e-16), (name, "backward", g[0], r[0])
    assert g[1] <= 10 * max(r[1], 1e-15), (name, "forward", g[1], r[1])
    assert g[2] <= 10 * max(r[2], 1e-16), (name, "residual", g[2], r[2])
    return g


def lapack_factors(S):
    try:
        sla.cho_factor(S, lower=True)
        return True
    except np.linalg.LinAlgError:
        return False


# ---------------------------------------------------------------- test matrices (order n = 6 N)
def spd_spectrum(n, p, rng):
    """Q diag(ev) Q^T with ev log-uniform in [10^-p, 1], both ends included (cond = 10^p)"""
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    ev = 10.0 ** (-p * rng.random(n))
    ev[0], ev[-1] = 1.0, 10.0 ** -p
    S = (Q * ev) @ Q.T
    return 0.5 * (S + S.T)


def spd_bad_pivot(n, K, c, rng):
    """S = L L^T with well-conditioned blocks, except pivot block K of the Schur complement at step K, L_KK L_KK^T, whose
    cond is 10^c (its columns nearly dependent)"""
    L = np.tril(rng.standard_normal((n, n))) / np.sqrt(n)
    for k in range(0, n, 48):
        m = min(48, n - k)
        p = c if k == 48 * K else 0.3
        L[k:k + m, k:k + m] = np.linalg.cholesky(spd_spectrum(m, p, rng))
    return L @ L.T


def spd_graded(n, rng):
    """D A D with A well conditioned and D log-uniform in 10^[-8, 8]"""
    d = 10.0 ** rng.uniform(-8, 8, n)
    A = spd_spectrum(n, 1, rng)
    return d[:, None] * A * d[None, :]


# ---------------------------------------------------------------- device
_HANDLES = {}


def carrier(N):
    """an uploaded direct-mode handle of N poses (its graph only fixes the order 6 N of the stored S)"""
    if N not in _HANDLES:
        g = gg.make_config(2, seed=1, n_poses=N, n_planes=4)
        a = GpuGraphAPI()
        a.set_linear_solver(True)
        gg.build_bulk(a, g)
        gg.configure(a, g)
        a.upload()
        _HANDLES[N] = a
    return _HANDLES[N]


def set_team(a, team, cluster):
    o = a.get_solver_options()
    o.team_ctas = team
    o.reserved[2] = 0 if cluster else (1 << 16)   # bit 16: global-memory barrier team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))


def factor_on_gpu(S, b, team=0, cluster=True):
    """stage 5: (L, x, dflag) of the GPU's factorization of S and its solve for b"""
    n = S.shape[0]
    a = carrier(n // 6)
    set_team(a, team, cluster)
    a.debug_store("Sdir", S)
    a.debug_store("b", b)
    a.debug_run_stage(5)
    flag = int(a.debug_fetch("dflag", 1)[0])
    L = a.debug_fetch("Ldir", n * n).reshape(n, n)
    x = a.debug_fetch("x", n)
    return L, x, flag


def run_case(name, S, seed):
    b = np.random.default_rng(seed + 1000).standard_normal(S.shape[0])
    assert lapack_factors(S), name
    L, x, flag = factor_on_gpu(S, b)
    assert flag == 0, (name, "a pivot failed on the GPU where LAPACK's factorization succeeds")
    return check(name, S, b, L, x, seed)


# ---------------------------------------------------------------- matrix families through stage 5
@pytest.mark.parametrize("N", [8, 32, 80])
@pytest.mark.parametrize("p", [0, 8, 12, 14])
def test_log_uniform_spectrum(N, p):
    run_case(f"spectrum N={N} p={p}", spd_spectrum(6 * N, p, np.random.default_rng(100 * N + p)), N + p)


@pytest.mark.parametrize("N,K", [(8, 0), (32, 0), (32, 1), (32, 3), (80, 4), (80, 9)])
@pytest.mark.parametrize("c", [8, 11, 13])
def test_ill_conditioned_pivot_block(N, K, c):
    """the factorization succeeds wherever LAPACK's does, and matches its accuracy"""
    run_case(f"pivot block {K} of N={N}, cond 1e{c}", spd_bad_pivot(6 * N, K, c, np.random.default_rng(7 * N + K + c)), c)


@pytest.mark.parametrize("N", [8, 80])
def test_graded_matrix(N):
    run_case(f"graded D A D N={N}", spd_graded(6 * N, np.random.default_rng(N)), N)


@pytest.mark.parametrize("N,p", [(n, p) for n in (1, 7, 9, 17) for p in (0, 8, 12, 14)] + [(n, p) for n in (639, 640) for p in (0, 12)])
def test_tile_edges(N, p):
    """orders 6 N that end inside a tile (all but 640) and the 640-pose cap of 80 full tile columns"""
    run_case(f"tile edge N={N} p={p}", spd_spectrum(6 * N, p, np.random.default_rng(N * 31 + p)), N)


@pytest.mark.parametrize("N", [1, 9, 32])
def test_indefinite_matrix_sets_dflag(N):
    n = 6 * N
    rng = np.random.default_rng(N)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    ev = 10.0 ** (-6 * rng.random(n))
    ev[0] = 1.0
    ev[n // 2] = -1e-3 * np.linalg.norm(ev)
    S = (Q * ev) @ Q.T
    S = 0.5 * (S + S.T)
    assert not lapack_factors(S)
    _, _, flag = factor_on_gpu(S, rng.standard_normal(n))
    assert flag == 1
    # the next factorization clears the flag
    S = spd_spectrum(n, 4, rng)
    _, _, flag = factor_on_gpu(S, rng.standard_normal(n))
    assert flag == 0


# ---------------------------------------------------------------- team shapes
@pytest.mark.parametrize("N", [17, 640])
def test_bit_identical_across_team_shapes(N):
    """L and x of every team shape equal the one-CTA run bit for bit (odd sizes move the look-ahead owner dtile(d, d) % T and
    the row ownership; team sizes over the SM count are cut to the device)"""
    n = 6 * N
    rng = np.random.default_rng(N)
    S, b = spd_spectrum(n, 12, rng), rng.standard_normal(n)
    L1, x1, f1 = factor_on_gpu(S, b, team=1)
    assert f1 == 0
    for team in (1, 2, 3, 5, 16, 33, 1 << 20):
        for cluster in (True, False):
            L, x, flag = factor_on_gpu(S, b, team=team, cluster=cluster)
            assert flag == 0
            assert np.array_equal(L, L1), (team, cluster)
            assert np.array_equal(x, x1), (team, cluster)


# ---------------------------------------------------------------- graphs through the assembly (stages 4, 1, 2)
def _ut_row(k, n=6):
    return sum(n - r for r in range(k))


def weak_stretch(g, s, dofs, f, keep_planes):
    """poses s .. s+7 observe only `keep_planes`, and the odometry factors that touch them carry sqrt-information rows
    `dofs` (xyzypr in the pose frame) scaled by f: the stretch can move in directions only those rows constrain"""
    g.odo_sqrtinf = g.odo_sqrtinf.copy()
    for e in range(max(0, s - 1), min(g.n_odometry, s + 8)):
        for d in dofs:
            g.odo_sqrtinf[e, _ut_row(d):_ut_row(d + 1)] *= f
    inside = (g.pp_pose >= s) & (g.pp_pose < s + 8)
    ok = ~inside | np.isin(g.pp_plane, keep_planes)
    for k in ("pp_pose", "pp_plane", "pp_meas", "pp_sqrtinf"):
        setattr(g, k, getattr(g, k)[ok])
    return g


# Camera-frame poses: x lateral, y down, z forward; pitch turns about the vertical.  The ground plane constrains height,
# roll and tilt only.
GRAPHS = {
    # config 2: poses 120-127 see only the ground plane; their odometry constrains lateral, forward and heading 1e-8 as strongly
    "config2_ground_only_stretch": lambda: weak_stretch(gg.make_config(2, seed=0), 120, (0, 2, 4), 1e-4, [0]),
    # a 64-pose corridor: poses 24-31 see the ground and one side wall, whose normals leave the forward direction unobserved;
    # their odometry constrains it (and lateral / heading) 1e-8 as strongly
    "corridor64_one_wall_stretch": lambda: weak_stretch(gg.make_config(2, seed=1, n_poses=64, n_planes=16), 24, (0, 2, 4), 1e-4,
                                                        [0, 4]),
}


@pytest.mark.parametrize("name", list(GRAPHS))
def test_ill_conditioned_graph(name):
    g = GRAPHS[name]()
    N, M, n = g.n_poses, g.n_planes, 6 * g.n_poses
    gpu = GpuGraphAPI()
    gpu.set_linear_solver(True)
    gg.build_bulk(gpu, g)
    gg.configure(gpu, g)
    gpu.upload()
    gpu.debug_run_stage(4, 0.0)
    Sl = gpu.debug_fetch("Sdir", n * n).reshape(n, n)
    S = Sl + np.tril(Sl, -1).T
    ev = np.linalg.eigvalsh(S)
    cf = sla.cho_factor(S, lower=True)
    piv = max(np.linalg.cond(np.tril(cf[0])[k:k + 48, k:k + 48]) ** 2 for k in range(0, n, 48))
    print(f"{name}: cond(S) {ev[-1] / ev[0]:.2e}, largest pivot-block cond of the Schur complements {piv:.2e}")
    assert ev[0] > 0 and ev[-1] / ev[0] >= 1e10
    # S entrywise against the oracle's Schur complement, each entry against the size of its own terms.  The two linearise
    # with their own closed-form Jacobians, and an entry of Hpp that cancels keeps their rounding: hence 1e-8, not 1e-15
    orc = OracleAPI()
    orc.set_jacobian_mode(1)
    gg.build_bulk(orc, g)
    gg.configure(orc, g)
    A = orc.normal_equations(0.0)[0].toarray()
    App, Apl, All = A[:n, :n], A[:n, n:], A[n:, n:]
    Y = np.linalg.solve(All, Apl.T).T
    S_o = App - Y @ Apl.T
    scale = np.abs(App) + np.abs(Y) @ np.abs(Apl).T
    lo = np.tril_indices(n)
    e_s = float(np.max(np.abs(S - S_o)[lo] / np.maximum(scale[lo], 1e-300)))
    print(f"{name}: S against the oracle, entrywise relative to |Hpp| + |Y| |W|^T: {e_s:.1e}")
    assert e_s <= 1e-8
    # the step of stage 2 against the refined solve of the GPU's own S and b
    gpu.debug_run_stage(2, 0.0)
    assert int(gpu.debug_fetch("dflag", 1)[0]) == 0
    L = gpu.debug_fetch("Ldir", n * n).reshape(n, n)
    b = gpu.debug_fetch("b", n)
    x = gpu.debug_fetch("delta", n + 3 * M)[:n]
    check(name, S, b, L, x)


def test_debug_hooks_refuse_misuse():
    g = gg.make_config(2, seed=1, n_poses=8, n_planes=4)
    a = GpuGraphAPI()
    a.set_linear_solver(True)
    gg.build_bulk(a, g)
    gg.configure(a, g)
    a.upload()
    with pytest.raises(Exception, match="Sdir"):
        a.debug_store("Sdir", np.eye(47))
    p = GpuGraphAPI()
    gg.build_bulk(p, g)
    gg.configure(p, g)
    p.upload()
    with pytest.raises(Exception, match="direct"):
        p.debug_store("Sdir", np.eye(48))
    with pytest.raises(Exception, match="direct"):
        p.debug_run_stage(5)
    with pytest.raises(Exception, match="direct"):
        p.debug_fetch("dflag", 1)
