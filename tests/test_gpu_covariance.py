"""Marginal covariances from the nested-dissection factor (pus_marginal_covariances / pus_covariance_blocks, DESIGN.md
section 5.4): every node's own block and cross blocks in and out of L's pattern against an inverse of J^T J formed from
pus_jacobian at the same estimate, bit-identity across team shapes, barrier kinds and repeated calls, the invalidation of the
stored Sigma, the absence of side effects on a later solve, the refusals, a 20 000-pose map, the reference's own
Covariances and the façade's isam::Covariances.

Reference: H = J^T J from the exported Jacobian.  For graphs up to a few thousand columns, LAPACK's float64 inverse refined
twice with residuals I - H X formed in long double is the reference; the worst block's relative error must be within 20
times LAPACK's unrefined worst against it (check_blocks says why 20).  The reference's own Covariances (tests/golden/ref_covariances.npz, pinned to the
live reference by tests/test_covariance_reference.py) is compared in reference-Jacobian mode.  Larger graphs are checked by
sparse column solves, and the 20 000-pose map by H Sigma_{.x} = E_x for whole columns of Sigma."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI
from test_gpu_band_solve import build_graph

pytestmark = pytest.mark.gpu
LD = np.longdouble
HERE = os.path.dirname(os.path.abspath(__file__))


def cov_api(kind=2, order=1):
    a = GpuGraphAPI()
    a.set_linear_solver(kind)
    a.set_direct_ordering(order)
    return a


CASES = {
    "config1": lambda: gg.make_config(1, seed=0),
    "config2": lambda: gg.make_config(2, seed=0),
    "huber600": lambda: gg.make_config(3, seed=0, n_poses=600, n_planes=60),
    "revisit600": lambda: gg.make_revisit(seed=0, n_poses=600, n_planes=100),
    "revisit2000": lambda: gg.make_revisit(seed=0, n_poses=2000, n_planes=100),
}


def build(case, api=None, solve=True):
    api = api or cov_api()
    if case == "sphere400":
        info, _, _ = build_graph(api, case)
    else:
        g = CASES[case]()
        info = gg.build_bulk(api, g)
        gg.configure(api, g, max_iterations=3)
    if solve:
        api.batch_optimize()
    return api, info


def node_ids(info):
    return [int(i) for i in info["pose_ids"]] + [int(i) for i in info["plane_ids"]]


def hessian(api):
    J, _ = api.jacobian()
    return (J.T @ J).tocsc()


def cols(api, i):
    s = api.node_start(i)
    return slice(s, s + api.node_dim(i))


def ld_residual(H, X):
    """I - H X with the products and sums in long double (H sparse, one row at a time)"""
    H = H.tocsr()
    Xl = X.astype(LD)
    R = np.empty(X.shape, dtype=LD)
    for i in range(H.shape[0]):
        s, e = H.indptr[i], H.indptr[i + 1]
        R[i] = -(H.data[s:e].astype(LD)[:, None] * Xl[H.indices[s:e]]).sum(axis=0)
        R[i, i] += 1
    return R


def dense_reference(H):
    """(LAPACK's float64 inverse refined twice with long-double residuals, LAPACK's unrefined inverse)"""
    n = H.shape[0]
    cf = sla.cho_factor(H.toarray(), lower=True)
    X0 = sla.cho_solve(cf, np.eye(n))
    X = X0.astype(LD)
    for _ in range(2):
        X = X + sla.cho_solve(cf, ld_residual(H, X.astype(np.float64)).astype(np.float64)).astype(LD)
    return X.astype(np.float64), X0


def block_err(B, R):
    return np.abs(B - R).max() / max(np.abs(R).max(), 1e-300)


def check_blocks(name, blocks, refs, laps):
    """per block: relative error against the refined reference; the bar is calibrated on the graph, as
    test_gpu_direct_accuracy.py does per matrix: the worst block's error within 20 x LAPACK's worst (floor 1e-15).  Unlike
    that test, which hands both sides the same stored S, the device forms J^T J and the reduced system itself, in its own
    summation order, so its input differs from the host's H by rounding; that alone is an error of the order of LAPACK's.
    (Measured: 0.3 to 13 x LAPACK's worst on these graphs.)"""
    e = [block_err(B, R) for B, R in zip(blocks, refs)]
    el = [block_err(Lb, R) for Lb, R in zip(laps, refs)]
    print(f"{name}: {len(blocks)} blocks, worst relative error {max(e):.1e} (LAPACK's {max(el):.1e})")
    assert max(e) <= 20 * max(max(el), 1e-15), (name, int(np.argmax(e)), max(e), max(el))


@pytest.mark.parametrize("case", ["config1", "config2", "sphere400", "huber600", "revisit600"])
def test_marginals_match_inverse(case):
    api, info = build(case)
    ids = node_ids(info)
    M = api.marginal_covariances(ids)
    X, X0 = dense_reference(hessian(api))
    check_blocks(case, M, [X[cols(api, i), cols(api, i)] for i in ids], [X0[cols(api, i), cols(api, i)] for i in ids])
    for B in M:
        assert np.array_equal(B, B.T)


def test_marginals_match_sparse_columns_revisited():
    api, info = build("revisit2000")
    ids = node_ids(info)
    M = api.marginal_covariances(ids)
    H = hessian(api)
    lu = spl.splu(H, permc_spec="MMD_AT_PLUS_A")
    rng = np.random.default_rng(1)
    for k in rng.choice(len(ids), 40, replace=False):
        c = cols(api, ids[k])
        E = np.zeros((H.shape[0], c.stop - c.start))
        E[np.arange(c.start, c.stop), np.arange(c.stop - c.start)] = 1.0
        R = lu.solve(E)[c]
        assert block_err(M[k], R) <= 1e-8, (k, block_err(M[k], R))


def test_cross_blocks_in_and_out_of_pattern():
    api, info = build("revisit600")
    P, L = [int(i) for i in info["pose_ids"]], [int(i) for i in info["plane_ids"]]
    border = set(api.debug_fetch("bborder", 1 << 16).astype(int).tolist())
    plane_node = api.debug_fetch("plane_node", 1 << 16).astype(int)
    bordered = [int(plane_node[l]) for l in sorted(border)]
    eliminated = [int(plane_node[l]) for l in range(len(plane_node)) if l not in border]
    X, X0 = dense_reference(hessian(api))
    # a plane that pose 0 never co-observes
    seen = {int(f) for f in api.node_factors(P[0])}
    far_plane = next(l for l in eliminated if not (set(int(f) for f in api.node_factors(l)) & seen))
    pairs = [(P[0], P[1]), (P[1], P[0]), (P[0], P[-1]), (P[-1], P[3]), (P[5], far_plane), (far_plane, P[5]),
             (eliminated[0], eliminated[-1]), (eliminated[2], eliminated[2]), (P[7], eliminated[1])]
    pairs += [(P[0], b) for b in bordered] + [(b, P[-2]) for b in bordered] + [(b, b) for b in bordered]
    got = api.covariance_blocks(pairs)
    check_blocks("revisit600 pairs", got, [X[cols(api, a), cols(api, b)] for a, b in pairs],
                 [X0[cols(api, a), cols(api, b)] for a, b in pairs])
    # the joint marginal of a list, assembled from its blocks, is symmetric positive definite
    lst = [P[0], P[-1], eliminated[0], far_plane]
    J = np.block([[B for B in api.covariance_blocks([(a, b) for b in lst])] for a in lst])
    assert np.allclose(J, J.T, rtol=0, atol=1e-12 * np.abs(J).max())
    assert np.linalg.eigvalsh(0.5 * (J + J.T)).min() > 0


def run_with(case, team, cluster):
    a, info = build(case)
    o = a.get_solver_options()
    o.team_ctas = team
    o.reserved[2] = 0 if cluster else (1 << 16)   # bit 16: global-memory barrier team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    ids = node_ids(info)
    P = [int(i) for i in info["pose_ids"]]
    M = np.concatenate([B.ravel() for B in a.marginal_covariances(ids)])
    X = np.concatenate([B.ravel() for B in a.covariance_blocks([(P[0], P[-1]), (ids[-1], P[2])])])
    return a, ids, M, X


def test_bit_identical_across_team_shapes_and_calls():
    ref = None
    for team in (1, 2, 3, 16, 10_000):
        for cluster in (True, False):
            a, ids, M, X = run_with("config2", team, cluster)
            M2 = np.concatenate([B.ravel() for B in a.marginal_covariances(ids)])
            assert np.array_equal(M, M2), (team, cluster)
            if ref is None:
                ref = (M, X)
                continue
            assert np.array_equal(M, ref[0]), (team, cluster)
            assert np.array_equal(X, ref[1]), (team, cluster)


def flat(api, ids):
    return np.concatenate([B.ravel() for B in api.marginal_covariances(ids)])


def test_cache_invalidation_matches_fresh_handle():
    """Huber weights: a pose-plane measurement moved far past the threshold changes J at a fixed estimate"""
    g = gg.make_config(3, seed=0, n_poses=160, n_planes=30)

    def fresh(edit):
        a = cov_api()
        info = gg.build_bulk(a, g)
        gg.configure(a, g, max_iterations=3)
        edit(a, info)
        return a, info

    def solve(a, info):
        a.batch_optimize()

    def init(a, info):
        a.init_pose(int(info["pose_ids"][5]), a.get_pose(int(info["pose_ids"][5])) + np.array([0.01, 0, 0, 0, 0, 0, 0]))

    def meas(a, info):
        m = np.array(g.pp_meas[7], dtype=float)
        m[3] += 0.5
        a.set_measurement(int(info["pp_fids"][7]), m)

    def remove(a, info):
        a.remove_factor(int(info["pp_fids"][7]))

    for name, edit in [("solve", solve), ("init_pose", init), ("set_measurement", meas), ("remove_factor", remove)]:
        a, info = fresh(lambda a, i: None)
        ids = node_ids(info)
        before = flat(a, ids)
        edit(a, info)
        after = flat(a, ids)
        b, _ = fresh(edit)
        assert np.array_equal(after, flat(b, ids)), name
        assert not np.array_equal(after, before), name


def test_no_side_effects_on_a_later_solve():
    g = CASES["config2"]()
    out = []
    for with_cov in (False, True):
        a = cov_api()
        info = gg.build_bulk(a, g)
        gg.configure(a, g, max_iterations=5)
        if with_cov:
            a.marginal_covariances(node_ids(info))
            a.covariance_blocks([(int(info["pose_ids"][0]), int(info["pose_ids"][-1]))])
        a.batch_optimize()
        out.append((a.get_poses(info["pose_ids"]), a.get_planes(info["plane_ids"]), a.trace(), a.chi2()))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    for k in out[0][2]:
        assert np.array_equal(np.asarray(out[0][2][k]), np.asarray(out[1][2][k])), k
    assert out[0][3] == out[1][3]


@pytest.mark.parametrize("kind,order", [(0, 0), (1, 0), (2, 0), (0, 1)])
def test_refusals_name_the_two_calls(kind, order):
    a = cov_api(kind, order)
    g = CASES["config1"]()
    info = gg.build_bulk(a, g)
    gg.configure(a, g)
    for call in (lambda: a.marginal_covariances(node_ids(info)), lambda: a.covariance_blocks([(node_ids(info)[0],) * 2])):
        with pytest.raises(capi.ApiError) as e:
            call()
        assert "pus_set_linear_solver(h, 2)" in str(e.value) and "pus_set_direct_ordering(h, 1)" in str(e.value)


def test_unconstrained_pose_fails_and_stores_nothing():
    """a pose no factor touches leaves its block of J^T J zero: a zero pivot whatever the order"""
    g = CASES["config1"]()
    a = cov_api()
    info = gg.build_bulk(a, g)
    gg.configure(a, g)
    a.add_pose(g.poses_init[0])
    ids = node_ids(info)
    with pytest.raises(capi.ApiError) as e:
        a.marginal_covariances(ids)
    assert "non-positive pivot" in str(e.value)
    with pytest.raises(capi.ApiError):   # nothing was kept: the next call computes again and fails again
        a.marginal_covariances(ids[:1])


def test_large_revisited_map_all_pose_marginals():
    """20 000 poses driven twice over: every pose's marginal in one call within the budget.  For 8 random poses and planes x,
    the whole column block Sigma_{.x} (pus_covariance_blocks against every live node) satisfies H Sigma_{.x} = E_x with the
    sparse H = J^T J of pus_jacobian, and its own block equals the marginal; 50 random nodes asked again give the bits of
    the all-pose call."""
    g = gg.make_revisit(seed=0, n_poses=20000, n_planes=1000)
    a = cov_api()
    info = gg.build_bulk(a, g)
    gg.configure(a, g)
    P = [int(i) for i in info["pose_ids"]]
    M = a.marginal_covariances(P)
    assert len(M) == len(P)
    ids = P + [int(i) for i in info["plane_ids"]]
    rng = np.random.default_rng(2)
    pick = rng.choice(len(ids), 50, replace=False)
    got = a.marginal_covariances([ids[k] for k in pick])
    for k, B in zip(pick, got):
        assert np.array_equal(B, B.T) and np.linalg.eigvalsh(B).min() > 0, k
        if k < len(P):
            assert np.array_equal(B, M[k])
    H = hessian(a).tocsr()
    start = np.array([a.node_start(i) for i in ids])
    order = np.argsort(start)
    worst = 0.0
    for k in list(rng.choice(len(P), 5, replace=False)) + list(len(P) + rng.choice(len(ids) - len(P), 3, replace=False)):
        x = ids[k]
        d = a.node_dim(x)
        blocks = a.covariance_blocks([(ids[y], x) for y in order])
        C = np.concatenate(blocks, axis=0)              # rows in column order of the stacked system
        E = np.zeros_like(C)
        E[start[k] + np.arange(d), np.arange(d)] = 1.0
        res = np.abs(H @ C - E).max() / (abs(H).sum(axis=1).max() * np.abs(C).max())
        worst = max(worst, res)
        assert res <= 1e-12, (k, res)
        own = a.marginal_covariances([x])[0]
        assert np.allclose(C[start[k]:start[k] + d], own, rtol=0, atol=1e-10 * np.abs(own).max())
    print(f"revisited 20000: {len(M)} pose marginals, {a.debug_fetch('covbytes', 1)[0] / 2**30:.2f} GiB of Sigma and lists, "
          f"worst |H Sigma - E| / (|H|_inf |Sigma|_max) {worst:.1e}")


def test_against_the_reference_covariances():
    """pus_set_jacobian_mode(h, 1) (the reference's numerical differences), the generator's initial estimate: the same Sigma
    as the reference's own Covariances::access after one Slam::update() (tests/golden/ref_covariances.npz)"""
    from cov_golden import CASES as RC, GOLDEN, build as rbuild
    if not os.path.exists(GOLDEN):
        pytest.skip("no reference covariance fixture")
    want = np.load(GOLDEN)
    for case in RC:
        a = cov_api()
        a.set_jacobian_mode(0)
        pairs, dims = rbuild(a, case)
        got = a.covariance_blocks(pairs)
        ref = want[case]
        o, worst = 0, 0.0
        for B, (r, c) in zip(got, dims):
            R = ref[o:o + r * c].reshape(r, c)
            o += r * c
            worst = max(worst, np.abs(B - R).max() / np.abs(R).max())
        print(f"{case}: {len(pairs)} blocks against the reference's Covariances, worst relative difference {worst:.1e}")
        assert worst <= 2e-8, (case, worst)   # (measured: 2e-11 to 4e-9; the numerical Jacobians' round trip differs)


def test_facade_covariances_replay(tmp_path):
    """tests/facade_cov_replay.cpp: Slam::covariances().marginal / marginals / access of a band ND façade after a replay,
    each block in its place of an inverse of the façade's own J^T J; joint marginals exactly symmetric, as iSAM's"""
    from test_facade import write_frames
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "facade_cov_replay")
    libdir = os.path.join(root, "pop_up_slam_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", exe, os.path.join(HERE, "facade_cov_replay.cpp"),
                           "-L" + libdir, "-lpopup_gpu", "-Wl,-rpath," + libdir])
    g = gg.make_config(2, seed=6, n_poses=150, n_planes=30, sigma_mode="reference")
    path = tmp_path / "frames.txt"
    write_frames(g, path, (1.0 / g.pp_sqrtinf[:, 0]).tolist())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, check=True).stdout.splitlines()
    k = next(i for i, t in enumerate(out) if t.startswith("J "))
    rows, ncol, nnz = (int(x) for x in out[k].split()[1:])
    J = sp.csr_matrix((np.array(out[k + 3].split(), dtype=float), np.array(out[k + 2].split(), dtype=int),
                       np.array(out[k + 1].split(), dtype=int)), shape=(rows, ncol))
    X, _ = dense_reference((J.T @ J).tocsc())
    nodes = [tuple(int(x) for x in t.split()[1:]) for t in out if t.startswith("node ")]
    start = dict(zip([n for n, _ in nodes], np.cumsum([0] + [d for _, d in nodes])[:-1]))
    dim = dict(nodes)
    ids = [n for n, _ in nodes]

    def mat(t):
        v = t.split()
        return np.array(v[3:], dtype=float).reshape(int(v[1]), int(v[2]))

    def ref(lst_a, lst_b):
        ra = np.concatenate([start[i] + np.arange(dim[i]) for i in lst_a])
        rb = np.concatenate([start[i] + np.arange(dim[i]) for i in lst_b])
        return X[np.ix_(ra, rb)]

    def close(A, R):
        return np.abs(A - R).max() <= 1e-9 * np.abs(R).max()

    marg = [mat(t) for t in out if t.startswith("marginal ")]
    assert len(marg) == len(ids)
    for i, m in zip(ids, marg):
        assert close(m, ref([i], [i])), i
    joints = [mat(t) for t in out if t.startswith("joint ")]
    lists = [[ids[0], ids[-1], ids[1]], [ids[len(ids) // 2], ids[2]]]
    assert len(joints) == 2
    for m, lst in zip(joints, lists):
        assert np.array_equal(m, m.T)
        assert close(m, ref(lst, lst)), lst
    acc = [mat(t) for t in out if t.startswith("access ")]
    for m, (a, b) in zip(acc, [(ids[0], ids[-1]), (ids[-1], ids[1]), (ids[3], ids[3])]):
        assert m.shape == (dim[a], dim[b]) and close(m, ref([a], [b])), (a, b)
