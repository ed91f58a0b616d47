"""GPU solves of dense-plane graphs (graphgen.make_dense): 16-pose blocks with more than 256 distinct planes or more than 64
(tile, pose) runs, whose PCG pose phase keeps its per-block vectors in the global overflow scratch instead of shared memory.
Every path such a graph can take matches the oracle at BASELINE's bar (final chi2, poses and planes within 1e-4 relative, the
same accept / reject sequence): closed-form and reference Jacobians, forced two / three preconditioner levels, bulk-copy-staged
tiles, cluster and global-barrier teams, a batch that mixes dense and in-limit graphs, one graph spanning two emulated ranks,
and repeated device-resident solves."""
import ctypes
import functools

import numpy as np
import pytest

from oracle_api import OracleAPI
from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

pytestmark = pytest.mark.gpu
TOL = 1e-4
CASES = sorted(gg.DENSE_CASES)


def dense(case, **kw):
    return gg.make_dense(seed=3, **dict(gg.DENSE_CASES[case], **kw))


def compare(gpu, orc, ig, io, tol=TOL):
    c_g, c_o = gpu.chi2(), orc.chi2()
    assert abs(c_g - c_o) <= tol * max(abs(c_o), 1e-9), (c_g, c_o)
    P_g, P_o = gpu.get_poses(ig["pose_ids"]), orc.get_poses(io["pose_ids"])
    scale = max(1.0, np.abs(P_o[:, :3]).max())
    assert np.abs(P_g[:, :3] - P_o[:, :3]).max() <= tol * scale
    sq = np.sign(np.sum(P_g[:, 3:] * P_o[:, 3:], axis=1))[:, None]
    assert np.abs(P_g[:, 3:] * sq - P_o[:, 3:]).max() <= tol
    L_g, L_o = gpu.get_planes(ig["plane_ids"]), orc.get_planes(io["plane_ids"])
    sl = np.sign(np.sum(L_g * L_o, axis=1))[:, None]
    assert np.abs(L_g * sl - L_o).max() <= tol


@functools.lru_cache(maxsize=None)
def oracle(case, jac):
    g = dense(case)
    orc = OracleAPI()
    orc.set_jacobian_mode(jac)
    io = gg.build_bulk(orc, g)
    gg.configure(orc, g)
    it = orc.batch_optimize()
    return orc, io, it, orc.trace()


def gpu_graph(g, flags=0, team=0, jac=1):
    a = GpuGraphAPI()
    ids = gg.build_bulk(a, g)
    gg.configure(a, g)
    a.set_jacobian_mode(jac)
    o = a.get_solver_options()
    o.reserved[2] = flags
    o.team_ctas = team
    a._chk(a.lib.pus_set_solver_options(a.h, ctypes.byref(o)))
    return a, ids


def uses_overflow(a):
    nblk = int(a.debug_fetch("dims", 12)[6])
    return int((a.debug_fetch("blk_ovf", nblk) >= 0).sum())


def check_against_oracle(a, ig, case, jac, it):
    orc, io, it_o, tr_o = oracle(case, jac)
    assert it == it_o
    tr = a.trace()
    assert np.array_equal(tr["accepted"], tr_o["accepted"])
    assert np.allclose(tr["chi2_new"], tr_o["chi2_new"], rtol=TOL)
    compare(a, orc, ig, io)


@pytest.mark.parametrize("jac", [1, 0])
@pytest.mark.parametrize("case", CASES)
def test_dense_graph_matches_oracle(case, jac):
    """closed-form (jac=1) and reference-Jacobian (jac=0, numerical differences as in the reference) modes"""
    a, ig = gpu_graph(dense(case), jac=jac)
    it = a.batch_optimize()
    assert uses_overflow(a) >= (2 if case == "mixed" else 3)
    check_against_oracle(a, ig, case, jac, it)


@pytest.mark.parametrize("flags", [16, 8, 2, 8 | 2])
@pytest.mark.parametrize("case", CASES)
def test_dense_graph_levels_and_bulk_copy_tiles(case, flags):
    """solver option reserved[2]: bit 4 forces two preconditioner levels, bit 3 three, bit 1 the bulk-copy-staged W / Wt tiles"""
    a, ig = gpu_graph(dense(case), flags=flags)
    it = a.batch_optimize()
    assert int(a.debug_fetch("dims", 18)[14]) == (3 if flags & 8 else 2)
    check_against_oracle(a, ig, case, 1, it)


@pytest.mark.parametrize("team", [0, 2])
@pytest.mark.parametrize("case", CASES)
def test_dense_graph_cluster_and_global_barrier_teams(case, team):
    """reserved[2] bit 16 keeps the global-memory team barrier instead of a thread-block cluster: same trace and answer"""
    g = dense(case)
    res = []
    for flags in (0, 1 << 16):
        a, ig = gpu_graph(g, flags=flags, team=team)
        it = a.batch_optimize()
        check_against_oracle(a, ig, case, 1, it)
        res.append((it, a.trace()["accepted"].tolist(), a.chi2(), a.get_poses(ig["pose_ids"]), a.get_planes(ig["plane_ids"])))
    (it_c, acc_c, chi_c, P_c, L_c), (it_g, acc_g, chi_g, P_g, L_g) = res
    assert it_c == it_g and acc_c == acc_g
    assert abs(chi_c - chi_g) <= 1e-9 * abs(chi_g)
    assert np.abs(P_c - P_g).max() < 1e-8 and np.abs(L_c - L_g).max() < 1e-8


def test_batch_mixing_dense_and_in_limit_graphs():
    """one batched launch (pus_batch_optimize_many) over dense and in-limit graphs gives each graph the answer of its own solve"""
    graphs = [dense(c) for c in CASES] + [gg.make_config(2, seed=s, n_poses=120, n_planes=24) for s in range(3)]
    many = [gpu_graph(g) for g in graphs]
    its = capi.batch_optimize_many([a for a, _ in many])
    for g, (a, ids), it in zip(graphs, many, its):
        b, idb = gpu_graph(g)
        assert b.batch_optimize() == it
        assert np.array_equal(a.trace()["accepted"], b.trace()["accepted"])
        assert abs(a.chi2() - b.chi2()) <= 1e-9 * abs(b.chi2())
        assert np.abs(a.get_poses(ids["pose_ids"]) - b.get_poses(idb["pose_ids"])).max() < 1e-8
        assert np.abs(a.get_planes(ids["plane_ids"]) - b.get_planes(idb["plane_ids"])).max() < 1e-8
    for (a, ig), case in zip(many[:len(CASES)], CASES):
        assert uses_overflow(a) > 0
        check_against_oracle(a, ig, case, 1, its[CASES.index(case)])


@pytest.mark.parametrize("flags", [0, 2])
@pytest.mark.parametrize("case", CASES)
def test_dense_graph_spanning_two_ranks_emulated(case, flags):
    """one graph split over two emulated ranks (global ownership of tiles / blocks, mirrored PCG vectors, cross-rank barrier),
    with and without the bulk-copy data path: same trace as the single-team solve and as the oracle, ranks bit-identical"""
    g = dense(case)
    one, i1 = gpu_graph(g, flags=flags)
    it1 = one.batch_optimize()
    apis = [gpu_graph(g, flags=flags) for _ in range(2)]
    its = capi.span_emulate_optimize([a for a, _ in apis])
    assert its == it1
    P1 = one.get_poses(i1["pose_ids"])
    acc = one.trace()["accepted"] == 1
    for a, info in apis:
        assert np.array_equal(a.trace()["accepted"], one.trace()["accepted"])
        assert np.allclose(a.trace()["chi2_new"][acc], one.trace()["chi2_new"][acc], rtol=1e-7)
        assert np.abs(a.get_poses(info["pose_ids"]) - P1).max() <= 1e-6
        check_against_oracle(a, info, case, 1, its)
    (a0, i0), (a1, i1b) = apis
    assert np.array_equal(a0.get_poses(i0["pose_ids"]), a1.get_poses(i1b["pose_ids"]))
    assert np.array_equal(a0.get_planes(i0["plane_ids"]), a1.get_planes(i1b["plane_ids"]))


@pytest.mark.parametrize("case", CASES)
def test_dense_resident_solve_is_repeatable(case):
    """repeated device-resident solves of the uploaded graph and a batch solve give the same bits (fixed-order sums, no atomics)"""
    g = dense(case)
    a, ids = gpu_graph(g)
    a.upload()
    its = [a.solve_resident() for _ in range(3)]
    a.download()
    P, L = a.get_poses(ids["pose_ids"]), a.get_planes(ids["plane_ids"])
    b, idb = gpu_graph(g)
    assert b.batch_optimize() == its[0] == its[1] == its[2]
    assert np.array_equal(P, b.get_poses(idb["pose_ids"]))
    assert np.array_equal(L, b.get_planes(idb["plane_ids"]))
