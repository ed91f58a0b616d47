"""CPU tests of the export's yardstick: the oracle's stacked exports (orc_weighted_errors, orc_jacobian, orc_normalized_chi2,
orc_local_chi2; tests/export_oracle_ext.cpp) against the UNMODIFIED reference's own Slam::weighted_errors, Slam::jacobian(),
normalized_chi2 and local_chi2 (ref_*; tests/export_ref_ext.cpp), on the graphs the GPU export tests use.

Slam::jacobian() has two branches (Slam.cpp:379-389) and both are pinned:
  - jacobian_partial (default): Factor::jacobian per factor, zeros stored, rhs = Jacobian::rhs() = -residual.  The oracle's
    numeric mode, and the product's mode 1, reproduce it entry for entry.
  - jacobian_numerical_columnwise (Properties::force_numerical_jacobian): the same central differences, but it omits entries
    that are exactly 0 (Slam.cpp:365) and its rhs is weighted_errors(LINPOINT), i.e. +residual (Slam.cpp:375).  Compared
    as such: same values wherever it stores one, exact zeros where it omits one, rhs of the opposite sign.
Skipped without the reference checkout and the objects `make -C oracle ref` leaves in oracle/_ref/obj."""
import numpy as np
import pytest

import export_api as X
from pop_up_slam_b200 import geometry as geo, graphgen as gg

pytestmark = pytest.mark.skipif(X.ref_objects() is None, reason="needs the reference checkout and oracle/_ref/obj")


def _factor2(api, g):
    """as tests/test_reference_build.py builds it: rays as precompute_edge_ray forms them from float32 pixels, (x, y, 1)"""
    pose_ids, plane_ids = api.add_poses(g.poses_init), api.add_planes(g.planes_init)
    api.add_pose_prior(pose_ids[g.prior_pose], g.prior_meas, g.prior_sqrtinf)
    api.add_odometry_bulk(pose_ids[g.odo_i], pose_ids[g.odo_j], g.odo_meas, g.odo_sqrtinf)
    api.add_plane_prior(plane_ids[g.ground_plane], g.ground_meas, g.ground_sqrtinf)
    n2 = 0
    for e in range(g.n_pose_plane):
        p, k = int(g.pp_pose[e]), int(g.pp_plane[e])
        rays = gg.rays_from_measurement(geo.pose7_to_T(g.poses_truth[p]), g.pp_meas[e])
        if k != g.ground_plane and abs(rays[2]) > 0.05 and abs(rays[5]) > 0.05:
            rays = np.concatenate([rays[:3] / rays[2], rays[3:] / rays[5]]).astype(np.float32).astype(np.float64)
            api.add_pose_plane2(pose_ids[p], plane_ids[k], g.pp_meas[e], rays, g.pp_sqrtinf[e])
            n2 += 1
        else:
            api.add_pose_plane(pose_ids[p], plane_ids[k], g.pp_meas[e], g.pp_sqrtinf[e])
    assert n2 > 100


def _loopclose(api, g):
    from test_reference_build import _loopclose_scenario
    ids = _loopclose_scenario(api, g)
    for k, dup in ids["dup_ids"].items():
        for f, e in ids["dup_facs"][k]:
            api.add_pose_plane(ids["pose_ids"][int(g.pp_pose[e])], ids["plane_ids"][k], api.get_measurement(f, 4), g.pp_sqrtinf[e])
            api.remove_factor(f)
    for k, dup in ids["dup_ids"].items():
        api.remove_node(dup)


CASES = {
    "config1": (lambda: gg.make_config(1, seed=0), gg.build_interleaved, None),
    "config2": (lambda: gg.make_config(2, seed=0), gg.build_interleaved, None),
    "huber_corridor": (lambda: gg.make_config(3, seed=0, n_poses=600, n_planes=60), gg.build_bulk, None),
    "pseudo_huber": (lambda: gg.make_config(3, seed=1, n_poses=300, n_planes=40), gg.build_bulk, (2, 0.5)),
    "factor2": (lambda: gg.make_config(2, seed=6, n_poses=60, n_planes=20), _factor2, None),
    "loopclose": (lambda: gg.make_config(2, seed=5, n_poses=160, n_planes=30), _loopclose, None),
}


def _build(name):
    make, build, robust = CASES[name]
    g = make()
    orc, ref, col = X.OracleExportAPI(), X.RefExportAPI(), X.RefExportAPI(columnwise=True)
    for api in (orc, ref, col):
        build(api, g)
        gg.configure(api, g)
        if robust:
            api.set_robust(*robust)
    orc.set_jacobian_mode(0)
    return orc, ref, col


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_export_matches_the_reference(name):
    orc, ref, col = _build(name)
    assert orc.jacobian_dims() == ref.jacobian_dims()
    e_o, e_r = orc.weighted_errors(), ref.weighted_errors()
    assert np.abs(e_o - e_r).max() <= 1e-12 * max(1.0, np.abs(e_r).max())
    fids = orc.live_fids()[::7]
    assert np.abs(orc.factor_errors(fids) - ref.factor_errors(fids)).max() <= 1e-12 * max(1.0, np.abs(e_r).max())
    # jacobian_partial: identical structure, values to rounding of the central differences, rhs = -errors
    (J_o, rhs_o), (J_r, rhs_r) = orc.jacobian(), ref.jacobian()
    assert J_o.shape == J_r.shape
    assert np.array_equal(J_o.indptr, J_r.indptr) and np.array_equal(J_o.indices, J_r.indices)
    scale = max(1.0, np.abs(J_r.data).max())
    assert np.abs(J_o.data - J_r.data).max() <= 1e-11 * scale
    assert np.abs(rhs_o - rhs_r).max() <= 1e-12 * max(1.0, np.abs(rhs_r).max())
    assert np.abs(rhs_r + e_r).max() <= 1e-9 * max(1.0, np.abs(e_r).max())   # (LINPOINT after the Euler round trip)
    # jacobian_numerical_columnwise: the same values wherever it stores one, zeros omitted, rhs = +residual
    J_c, rhs_c = col.jacobian()
    assert J_c.shape == J_r.shape and J_c.nnz <= J_r.nnz
    D = (J_o - J_c).tocsr()
    assert np.abs(D.data).max(initial=0.0) <= 1e-11 * scale
    omitted = J_o.copy()
    omitted.data = np.ones_like(omitted.data)
    kept = J_c.copy()
    kept.data = np.ones_like(kept.data)
    assert (omitted - kept).min() >= 0                                          # columnwise stores a subset of the pattern
    assert np.abs(rhs_c + rhs_o).max() <= 1e-12 * max(1.0, np.abs(rhs_o).max())
    # normalized_chi2 = chi2 / (_dim_measure - _dim_nodes); local_chi2 walks the factor list backwards
    assert abs(orc.normalized_chi2() - ref.normalized_chi2()) <= 1e-10 * ref.normalized_chi2()
    nlive = len(orc.live_fids())
    for n in (0, 1, 9, nlive // 3, nlive, nlive + 7):
        lo, lr = orc.local_chi2(n), ref.local_chi2(n)
        assert abs(lo - lr) <= 1e-10 * max(lr, 1e-12 * ref.normalized_chi2()), (n, lo, lr)
