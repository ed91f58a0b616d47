"""Host tables of the band direct solve (pus_set_linear_solver(h, 2)), without a GPU, against a Python restatement: the
bordered planes follow the span rule, every tile row's first coupled column is right, the device byte count matches, and
every (pose pair, plane) product and pose-pose factor block inside the envelope is listed exactly once; the refusals (a graph
over the memory budget, bad kinds) and no CPU fallback."""
import json
import os
import sys

import numpy as np
import pytest

from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

HERE = os.path.dirname(os.path.abspath(__file__))
TILE_BYTES = 48 * 52 * 8
BUDGET = 8 << 30


def ints(api, name):
    return api.debug_fetch(name, 1 << 24).astype(np.int64)


def compiled(build, kind=2):
    api = GpuGraphAPI()
    api.set_linear_solver(kind)
    info = build(api)
    api._chk(api.lib.pus_debug_compile(api.h))
    return api, info


def incidences(pl_ptr, pl_pose):
    """per plane: its distinct observing poses, ascending (one incidence each)"""
    return [sorted(set(pl_pose[pl_ptr[l]:pl_ptr[l + 1]].tolist())) for l in range(len(pl_ptr) - 1)]


def layout(N, inc, pf, border):
    """(first tile column per tile row, device bytes) of the layout that borders `border`"""
    nbp = max(1, (6 * N + 47) // 48)
    nb = nbp + (3 * len(border) + 47) // 48
    slot = {l: k for k, l in enumerate(sorted(border))}
    mp = list(range(N))
    for i, j in pf:
        mp[max(i, j)] = min(mp[max(i, j)], min(i, j))
    first = list(range(nb))
    lp = 0
    for l, poses in enumerate(inc):
        if not poses:
            continue
        if l in slot:
            t = nbp + 3 * slot[l] // 48
            first[t] = min(first[t], poses[0] // 8)
        else:
            lp += len(poses) * (len(poses) + 1) // 2
            for a in poses:
                mp[a] = min(mp[a], poses[0])
    for a in range(N):
        first[a // 8] = min(first[a // 8], mp[a] // 8)
    tiles = sum(i - first[i] + 1 for i in range(nb))
    npair = sum(a - 8 * first[a // 8] + 1 for a in range(N))
    ninc = sum(len(p) for p in inc)
    n_int = 2 * (npair + 1) + 2 * lp + len(pf) + 3 * ninc + nb + (nb + 1) + N + (nb + 1) + (tiles - nb) + 3 * len(border)
    return first, (tiles + 3 * nb) * TILE_BYTES + 8 * (2 * 48 * nb + 36 * ninc + 3 * len(border)) + 4 * n_int


def restate(N, inc, pf):
    """the bordering rule: planes by observer span descending (ties: index), the k = 0 .. min(M, 64) widest, fewest bytes"""
    span = [p[-1] - p[0] if p else 0 for p in inc]
    order = sorted(range(len(inc)), key=lambda l: (-span[l], l))
    best = None
    for k in range(min(len(inc), 64) + 1):
        b = layout(N, inc, pf, order[:k])[1]
        if best is None or b < best[0]:
            best = (b, k)
    border = sorted(order[:best[1]])
    first, nbytes = layout(N, inc, pf, border)
    return border, first, nbytes


def check_band(api):
    N = int(api.debug_fetch("dims", 12)[0])
    pl_ptr, pl_pose = ints(api, "pl_ptr"), ints(api, "pl_pose")
    pf_i, pf_j = ints(api, "pf_i"), ints(api, "pf_j")
    inc = incidences(pl_ptr, pl_pose)
    pf = [(int(i), int(j)) for i, j in zip(pf_i, pf_j) if j >= 0]
    border, first, nbytes = restate(N, inc, pf)
    assert ints(api, "bborder").tolist() == border
    assert ints(api, "bfirst").tolist() == first
    assert int(api.debug_fetch("bbytes", 1)[0]) == nbytes
    # envelope pair lists: pair (a, b), a >= b >= 8 first[a / 8], at poff[a] + b - 8 first[a / 8]
    poff = np.concatenate([[0], np.cumsum([a - 8 * first[a // 8] + 1 for a in range(N)])]).astype(int)
    pair = lambda a, b: poff[a] + b - 8 * first[a // 8]
    inc_pose, inc_plane = ints(api, "dinc_pose"), ints(api, "dinc_plane")
    lp_ptr, lp_a, lp_b = ints(api, "dlp_ptr"), ints(api, "dlp_a"), ints(api, "dlp_b")
    assert len(lp_ptr) == poff[N] + 1
    exp = {}
    for l in range(len(inc)):
        if l in border:
            continue
        ids = [i for i in range(len(inc_plane)) if inc_plane[i] == l]
        for i in ids:
            for j in ids:
                a, b = inc_pose[i], inc_pose[j]
                if a >= b:
                    assert b >= 8 * first[a // 8]
                    exp.setdefault(pair(a, b), []).append((i, j))
    got = {}
    for q in range(poff[N]):
        if lp_ptr[q + 1] > lp_ptr[q]:
            got[q] = list(zip(lp_a[lp_ptr[q]:lp_ptr[q + 1]].tolist(), lp_b[lp_ptr[q]:lp_ptr[q + 1]].tolist()))
    assert got == exp
    fp_ptr, fp_f = ints(api, "dfp_ptr"), ints(api, "dfp_f")
    expf = {}
    for k in range(len(pf_i)):
        if pf_j[k] < 0:
            continue
        a, b = max(pf_i[k], pf_j[k]), min(pf_i[k], pf_j[k])
        expf.setdefault(pair(a, b), []).append(2 * k + (1 if pf_j[k] > pf_i[k] else 0))
    gotf = {q: fp_f[fp_ptr[q]:fp_ptr[q + 1]].tolist() for q in range(poff[N]) if fp_ptr[q + 1] > fp_ptr[q]}
    assert gotf == expf
    return border, first


def bulk(g, dup=None):
    def build(api):
        info = gg.build_bulk(api, g)
        for e in (dup if dup is not None else []):
            m = g.pp_meas[e].copy()
            m[3] += 0.01
            api.add_pose_plane(int(info["pose_ids"][g.pp_pose[e]]), int(info["plane_ids"][g.pp_plane[e]]), m / np.linalg.norm(m),
                               g.pp_sqrtinf[e])
        return info
    return build


@pytest.mark.parametrize("cfg", [1, 2])
def test_band_tables_configs(cfg):
    g = gg.make_config(cfg, seed=0)
    check_band(compiled(bulk(g))[0])


def test_band_tables_dense_planes():
    check_band(compiled(bulk(gg.make_dense(seed=0)))[0])


def test_band_tables_repeated_observation():
    g = gg.make_config(2, seed=4, n_poses=60, n_planes=15)
    dup = np.random.default_rng(0).choice(len(g.pp_pose), size=25, replace=False)
    check_band(compiled(bulk(g, dup))[0])


def test_band_tables_corridor_borders_the_ground_plane():
    g = gg.make_config(3, seed=0, n_poses=1200, n_planes=120)
    border, first = check_band(compiled(bulk(g))[0])
    assert g.ground_plane in border
    nbp = (6 * 1200 + 47) // 48
    assert max(i - first[i] for i in range(nbp)) < 20   # a narrow envelope once the ground plane is bordered


def test_band_tables_sphere400():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    from make_sphere_golden import build
    fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
    edges = [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]]
    border, _ = check_band(compiled(lambda api: build(api, edges))[0])
    assert border == []


def test_dense_kind_keeps_its_layout():
    """kind 1 is the band layout with no bordered plane and first = 0"""
    api, _ = compiled(bulk(gg.make_config(2, seed=0)), kind=1)
    N = int(api.debug_fetch("dims", 12)[0])
    assert ints(api, "bborder").tolist() == []
    assert ints(api, "bfirst").tolist() == [0] * ((6 * N + 47) // 48)
    assert api.linear_solver_kind() == 1 and api.linear_solver_is_direct()


def test_band_refuses_a_graph_over_the_budget():
    """20 000 poses, each with an odometry edge to pose 0: every tile row couples to column 0, a dense system of ~58 GB"""
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    ut = gg.diag_ut([1.0] * 6)
    ids = [api.add_pose(None)]
    api.add_pose_prior(ids[0], [0, 0, 0, 0, 0, 0], ut)
    for i in range(1, 20000):
        ids.append(api.add_pose(None))
        api.add_odometry(ids[0], ids[i], [0.1 * i, 0, 0, 0, 0, 0], ut)
    with pytest.raises(capi.ApiError, match=r"band linear solver: the graph needs \d+ bytes of device memory") as e:
        api._chk(api.lib.pus_debug_compile(api.h))
    need = int(str(e.value).split("needs ")[1].split(" bytes")[0])
    assert need > BUDGET
    assert api.linear_solver_kind() == 2 and not api.linear_solver_is_direct()


def test_bad_kinds_are_refused():
    api = GpuGraphAPI()
    for kind in (-1, 3):
        assert api.lib.pus_set_linear_solver(api.h, kind) < 0
        assert b"bad linear solver kind" in api.lib.pus_last_error()
        with pytest.raises(ValueError):
            api.set_linear_solver(kind)
    assert api.linear_solver_kind() == 0
    api.set_linear_solver(True)
    assert api.linear_solver_kind() == 1
    api.set_linear_solver(False)
    assert api.linear_solver_kind() == 0


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_band_mode_has_no_cpu_fallback_without_a_gpu():
    g = gg.make_config(1, seed=0)
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    gg.build_interleaved(api, g)
    gg.configure(api, g)
    with pytest.raises(capi.ApiError, match="no CUDA device available"):
        api.batch_optimize()
