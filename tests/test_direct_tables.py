"""Host tables of the exact direct solve (pus_set_linear_solver(h, 1)), without a GPU: every (pose pair, plane) product and
every pose-pose factor block of the reduced system is listed exactly once, under the pose pair whose entries it feeds, in
plane-ascending / factor order; and a direct-mode solve fails without a device instead of falling back to the CPU."""
import numpy as np
import pytest

from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI


def fetch_ints(api, name):
    return api.debug_fetch(name, 1 << 22).astype(int)


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


def compiled(g, dup=None):
    api = GpuGraphAPI()
    api.set_linear_solver(True)
    info = gg.build_bulk(api, g)
    if dup is not None:
        for e in dup:
            m = g.pp_meas[e].copy()
            m[3] += 0.01
            api.add_pose_plane(int(info["pose_ids"][g.pp_pose[e]]), int(info["plane_ids"][g.pp_plane[e]]), m / np.linalg.norm(m),
                               g.pp_sqrtinf[e])
    api._chk(api.lib.pus_debug_compile(api.h))
    return api


def check_tables(api):
    f = lambda nm: fetch_ints(api, nm)
    dims = api.debug_fetch("dims", 12)
    N = int(dims[0])
    pl_ptr, pl_pose = f("pl_ptr"), f("pl_pose")
    M = len(pl_ptr) - 1
    inc_pose, inc_plane, inc_lo, inc_hi = f("dinc_pose"), f("dinc_plane"), f("dinc_lo"), f("dinc_hi")
    # incidences: one per distinct (pose, plane), covering exactly that pair's plane-major slots
    want = []
    for l in range(M):
        poses = pl_pose[pl_ptr[l]:pl_ptr[l + 1]]
        for p in sorted(set(poses.tolist())):
            s = np.nonzero(poses == p)[0] + pl_ptr[l]
            want.append((l, p, s[0], s[-1] + 1))
            assert s[-1] + 1 - s[0] == len(s)
    assert list(zip(inc_plane, inc_pose, inc_lo, inc_hi)) == want
    # plane products: for every pair a >= b and every plane both observe, one record, plane-ascending
    lp_ptr, lp_a, lp_b = f("dlp_ptr"), f("dlp_a"), f("dlp_b")
    npair = N * (N + 1) // 2
    assert len(lp_ptr) == npair + 1
    exp = {}
    for l in range(M):
        ids = [i for i in range(len(inc_plane)) if inc_plane[i] == l]
        for i in ids:
            for j in ids:
                a, b = inc_pose[i], inc_pose[j]
                if a >= b:
                    exp.setdefault(a * (a + 1) // 2 + b, []).append((i, j))
    for q in range(npair):
        got = list(zip(lp_a[lp_ptr[q]:lp_ptr[q + 1]], lp_b[lp_ptr[q]:lp_ptr[q + 1]]))
        assert got == exp.get(q, []), q
    # pose-pose factor blocks: each odometry factor once, under (max, min) of its poses, side 1 when its second pose is larger
    fp_ptr, fp_f = f("dfp_ptr"), f("dfp_f")
    pf_i, pf_j = f("pf_i"), f("pf_j")
    expf = {}
    for k in range(len(pf_i)):
        if pf_j[k] < 0:
            continue
        a, b = max(pf_i[k], pf_j[k]), min(pf_i[k], pf_j[k])
        expf.setdefault(a * (a + 1) // 2 + b, []).append(2 * k + (1 if pf_j[k] > pf_i[k] else 0))
    for q in range(npair):
        assert list(fp_f[fp_ptr[q]:fp_ptr[q + 1]]) == expf.get(q, []), q
    return N


@pytest.mark.parametrize("cfg", [1, 2])
def test_direct_tables_configs(cfg):
    check_tables(compiled(gg.make_config(cfg, seed=0)))


def test_direct_tables_dense_planes():
    check_tables(compiled(gg.make_dense(seed=0)))


def test_direct_tables_repeated_observation():
    g = gg.make_config(2, seed=4, n_poses=60, n_planes=15)
    dup = np.random.default_rng(0).choice(len(g.pp_pose), size=25, replace=False)
    api = compiled(g, dup)
    check_tables(api)
    lo, hi = fetch_ints(api, "dinc_lo"), fetch_ints(api, "dinc_hi")
    assert np.sum(hi - lo == 2) == len(set((int(g.pp_pose[e]), int(g.pp_plane[e])) for e in dup))


def test_direct_mode_refuses_graphs_over_the_cap():
    g = gg.make_corridor(seed=0, n_poses=641, n_planes=40, obs_per_pose=4)
    api = GpuGraphAPI()
    gg.build_bulk(api, g)
    api._chk(api.lib.pus_debug_compile(api.h))   # PCG mode: fine
    api.set_linear_solver(True)
    assert api.linear_solver_is_direct()
    with pytest.raises(capi.ApiError, match="at most 640"):
        api._chk(api.lib.pus_debug_compile(api.h))


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_direct_mode_has_no_cpu_fallback_without_a_gpu():
    g = gg.make_config(1, seed=0)
    api = GpuGraphAPI()
    api.set_linear_solver(True)
    gg.build_interleaved(api, g)
    gg.configure(api, g)
    with pytest.raises(capi.ApiError, match="no CUDA device available"):
        api.batch_optimize()
