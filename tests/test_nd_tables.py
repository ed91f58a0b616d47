"""Host tables of the band direct solve in nested-dissection order (pus_set_direct_ordering(h, 1)), without a GPU, against a
Python restatement: the tile order, the bordered planes, the elimination tree, L's tile pattern, the levels, the update lists,
the device byte count and the per-pose-pair assembly lists; the refusals (a graph over the budget, bad order values) and no
CPU fallback."""
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
LEAF = 4
ND_HDR = 14


def ints(api, name):
    return api.debug_fetch(name, 1 << 26).astype(np.int64)


def compiled(build, order=1):
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    api.set_direct_ordering(order)
    info = build(api)
    api._chk(api.lib.pus_debug_compile(api.h))
    return api, info


def incidences(pl_ptr, pl_pose):
    return [sorted(set(pl_pose[pl_ptr[l]:pl_ptr[l + 1]].tolist())) for l in range(len(pl_ptr) - 1)]


# ---------------------------------------------------------------- the restatement
def bfs(adj, r, S):
    """BFS level structure from r inside S: the levels (each ascending) and every tile's level"""
    lev, levels = {r: 0}, [[r]]
    while True:
        nxt = sorted({u for v in levels[-1] for u in adj[v] if u in S and u not in lev})
        if not nxt:
            return levels, lev
        for u in nxt:
            lev[u] = len(levels)
        levels.append(nxt)


def nd_order(adj):
    out = []

    def dissect(S):
        if len(S) <= LEAF:
            out.extend(S)
            return
        Sset, done, comps = set(S), set(), []
        for t in S:
            if t not in done:
                c = sorted(x for L in bfs(adj, t, Sset)[0] for x in L)
                done |= set(c)
                comps.append(c)
        if len(comps) > 1:
            for c in comps:
                dissect(c)
            return
        v = S[0]
        levels, lev = bfs(adj, v, Sset)
        while True:   # pseudo-peripheral: the lowest tile of the last level while the depth grows
            l2, lv2 = bfs(adj, levels[-1][0], Sset)
            if len(l2) <= len(levels):
                break
            levels, lev = l2, lv2
        h = len(levels)
        if h <= 2:
            out.extend(S)
            return
        cum, m = 0, 0
        for m, L in enumerate(levels):
            cum += len(L)
            if 2 * cum >= len(S):
                break
        m = max(1, min(h - 2, m))
        sep = [t for t in levels[m] if any(lev.get(u) == m + 1 for u in adj[t] if u in Sset)]
        A = sorted([x for L in levels[:m] for x in L] + [t for t in levels[m] if t not in sep])
        B = sorted(x for L in levels[m + 1:] for x in L)
        dissect(A)
        dissect(B)
        out.extend(sep)

    dissect(list(range(len(adj))))
    return out


def symbolic(nb, alow):
    """column patterns (ascending, diagonal first), parents, levels"""
    cols, parent, level, kids = [], [-1] * nb, [0] * nb, [[] for _ in range(nb)]
    for j in range(nb):
        col = {j} | alow[j]
        for c in kids[j]:
            col |= set(cols[c]) - {c}
            level[j] = max(level[j], level[c] + 1)
        col = sorted(col)
        cols.append(col)
        if len(col) > 1:
            parent[j] = col[1]
            kids[col[1]].append(j)
    return cols, parent, level


def layout(N, inc, pf, border, perm=None):
    """the ND layout that borders `border`: tile order, patterns, parents, levels, device bytes"""
    nbp = max(1, (6 * N + 47) // 48)
    nb = nbp + (3 * len(border) + 47) // 48
    slot = {l: k for k, l in enumerate(sorted(border))}
    adj = [set() for _ in range(nbp)]
    bt = [set() for _ in range(nb)]
    lp = 0
    for i, j in pf:
        if i // 8 != j // 8:
            adj[i // 8].add(j // 8)
            adj[j // 8].add(i // 8)
    for l, poses in enumerate(inc):
        if not poses:
            continue
        tl = sorted({p // 8 for p in poses})
        if l in slot:
            bt[nbp + 3 * slot[l] // 48] |= set(tl)
            continue
        lp += len(poses) * (len(poses) + 1) // 2
        for u in tl:
            adj[u] |= set(tl) - {u}
    adj = [sorted(a) for a in adj]
    if perm is None:
        perm = nd_order(adj) + list(range(nbp, nb))
    pos = {t: k for k, t in enumerate(perm)}
    alow = [set() for _ in range(nb)]
    for u in range(nbp):
        for v in adj[u]:
            alow[min(pos[u], pos[v])].add(max(pos[u], pos[v]))
    for t in range(nbp, nb):
        for u in bt[t]:
            alow[min(pos[u], pos[t])].add(max(pos[u], pos[t]))
    cols, parent, level = symbolic(nb, alow)
    T = sum(len(c) for c in cols)
    nupd = sum((len(c) - 1) * len(c) // 2 for c in cols)
    nlev = max(level) + 1
    ninc = sum(len(p) for p in inc)
    n_int = 5 * nb + 2 * nlev + 132 * T + 2 * nupd + 2 * lp + len(pf) + 3 * ninc + 3 * len(border) + 7 + ND_HDR
    nbytes = (T + nb) * TILE_BYTES + 8 * (2 * 48 * nb + 36 * ninc + 3 * len(border)) + 4 * n_int
    return dict(perm=perm, cols=cols, parent=parent, level=level, bytes=nbytes, nb=nb, nbp=nbp, nupd=nupd)


def restate(N, inc, pf):
    """the bordering rule: planes by the number of distinct observing pose tiles, descending (ties: index), fewest bytes"""
    ntile = [len({p // 8 for p in poses}) for poses in inc]
    order = sorted(range(len(inc)), key=lambda l: (-ntile[l], l))
    best = None
    for k in range(min(len(inc), 64) + 1):
        b = layout(N, inc, pf, order[:k])["bytes"]
        if best is None or b < best[0]:
            best = (b, k)
    return sorted(order[:best[1]])


def check_nd(api, restate_border=True):
    N = int(api.debug_fetch("dims", 12)[0])
    pl_ptr, pl_pose = ints(api, "pl_ptr"), ints(api, "pl_pose")
    pf_i, pf_j = ints(api, "pf_i"), ints(api, "pf_j")
    inc = incidences(pl_ptr, pl_pose)
    pf = [(int(i), int(j)) for i, j in zip(pf_i, pf_j) if j >= 0]
    border = ints(api, "bborder").tolist()
    if restate_border:
        assert border == restate(N, inc, pf)
    perm = ints(api, "ndtile").tolist()
    nbp = max(1, (6 * N + 47) // 48)
    nb = nbp + (3 * len(border) + 47) // 48
    assert sorted(perm) == list(range(nb)) and perm[nbp:] == list(range(nbp, nb))   # bordered tiles last
    ref = layout(N, inc, pf, border)
    assert perm == ref["perm"]
    given = layout(N, inc, pf, border, perm)
    assert ints(api, "ndparent").tolist() == given["parent"]
    assert ints(api, "ndlevel").tolist() == given["level"]
    cptr, crow = ints(api, "ndcptr"), ints(api, "ndcrow")
    cols = [crow[cptr[j]:cptr[j + 1]].tolist() for j in range(nb)]
    assert cols == given["cols"]
    assert int(api.debug_fetch("bbytes", 1)[0]) == given["bytes"]
    # tile storage: level by level, columns ascending inside a level, each column's tiles row-ascending
    toff, trow, tcol = ints(api, "ndtoff"), ints(api, "ndtrow"), ints(api, "ndtcol")
    lv = given["level"]
    order = sorted(range(nb), key=lambda j: (lv[j], j))
    t = 0
    for j in order:
        assert toff[j] == t
        assert trow[t:t + len(cols[j])].tolist() == cols[j] and set(tcol[t:t + len(cols[j])].tolist()) == {j}
        t += len(cols[j])
    assert t == len(trow)
    tile = {(int(trow[k]), int(tcol[k])): k for k in range(len(trow))}
    # update lists: tile (i, j) gets (L_iK, L_jK) for every K < j with i and j both in K's pattern, K ascending
    uptr, upd = ints(api, "nduptr"), ints(api, "ndupd")
    exp = {k: [] for k in range(len(trow))}
    for K in range(nb):
        rows = cols[K][1:]
        for a, i in enumerate(rows):
            for j in rows[:a + 1]:
                exp[tile[(i, j)]].append((tile[(i, K)], tile[(j, K)]))
    for k in range(len(trow)):
        got = [(int(upd[2 * u]), int(upd[2 * u + 1])) for u in range(uptr[k], uptr[k + 1])]
        assert got == exp[k]
    assert uptr[-1] == given["nupd"]
    # per-pose-pair lists of the stored tiles: every (pose pair, plane) product and pose-pose factor block exactly once,
    # in the original orientation a >= b, at 64 t + 8 (a % 8) + b % 8 of the tile t that holds the pair
    pos = {tt: k for k, tt in enumerate(perm)}

    def pair(a, b):
        i, j = pos[a // 8], pos[b // 8]
        return 64 * tile[(max(i, j), min(i, j))] + 8 * (a % 8) + b % 8
    inc_pose, inc_plane = ints(api, "dinc_pose"), ints(api, "dinc_plane")
    lp_ptr, lp_a, lp_b = ints(api, "dlp_ptr"), ints(api, "dlp_a"), ints(api, "dlp_b")
    assert len(lp_ptr) == 64 * len(trow) + 1
    expl = {}
    for l in range(len(inc)):
        if l in border:
            continue
        ids = [i for i in np.nonzero(inc_plane == l)[0]]
        for i in ids:
            for j in ids:
                if inc_pose[i] >= inc_pose[j] and j <= i:
                    expl.setdefault(pair(inc_pose[i], inc_pose[j]), []).append((int(i), int(j)))
    nz = np.nonzero(np.diff(lp_ptr))[0]
    gotl = {int(q): list(zip(lp_a[lp_ptr[q]:lp_ptr[q + 1]].tolist(), lp_b[lp_ptr[q]:lp_ptr[q + 1]].tolist())) for q in nz}
    assert gotl == expl
    fp_ptr, fp_f = ints(api, "dfp_ptr"), ints(api, "dfp_f")
    expf = {}
    for k in range(len(pf_i)):
        if pf_j[k] < 0:
            continue
        a, b = max(pf_i[k], pf_j[k]), min(pf_i[k], pf_j[k])
        expf.setdefault(pair(a, b), []).append(2 * k + (1 if pf_j[k] > pf_i[k] else 0))
    nz = np.nonzero(np.diff(fp_ptr))[0]
    assert {int(q): fp_f[fp_ptr[q]:fp_ptr[q + 1]].tolist() for q in nz} == expf
    # a second compile gives the same layout
    api._chk(api.lib.pus_debug_compile(api.h))
    assert ints(api, "ndtile").tolist() == perm and ints(api, "bborder").tolist() == border
    return dict(border=border, perm=perm, nb=nb, nbp=nbp, tiles=len(trow), levels=max(lv) + 1, nupd=given["nupd"])


def bulk(g, extra=()):
    def build(api):
        info = gg.build_bulk(api, g)
        for p, l in extra:
            e = int(np.nonzero(g.pp_plane == l)[0][0])
            api.add_pose_plane(int(info["pose_ids"][p]), int(info["plane_ids"][l]), g.pp_meas[e], g.pp_sqrtinf[e])
        return info
    return build


def sphere(name):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    from make_sphere_golden import build, load_edge3
    if name == "sphere400":
        fx = json.load(open(os.path.join(HERE, "golden", "sphere400.json")))
        edges = [(int(e[0]), int(e[1]), e[2:8], e[8:29]) for e in fx["edges"]]
    else:
        edges = load_edge3(os.path.join(HERE, "golden", "sphere2500.txt.xz"))
    return lambda api: build(api, edges)


# ---------------------------------------------------------------- the graphs
@pytest.mark.parametrize("cfg", [1, 2, 3])
def test_nd_tables_configs(cfg):
    g = gg.make_config(cfg, seed=0)
    r = check_nd(compiled(bulk(g))[0])
    if cfg == 3:
        assert g.ground_plane in r["border"]


@pytest.mark.parametrize("name", ["sphere400", "sphere2500"])
def test_nd_tables_sphere(name):
    r = check_nd(compiled(sphere(name))[0])
    assert r["border"] == []


def test_nd_tables_several_walls():
    """a corridor whose ground plane and three more planes are seen from every other pose"""
    g = gg.make_config(3, seed=2, n_poses=400, n_planes=60)
    r = check_nd(compiled(bulk(g, [(p, l) for l in (1, 2, 3) for p in range(0, 400, 2)]))[0])
    assert len(r["border"]) >= 4


def test_nd_tables_revisited_corridor():
    """the second pass re-observes the first pass's planes: insertion order has a wide envelope, ND keeps the fill low"""
    g = gg.make_revisit(seed=0, n_poses=2000, n_planes=100)
    api, _ = compiled(bulk(g))
    r = check_nd(api)
    band, _ = compiled(bulk(g), order=0)
    assert band.direct_ordering() == 0
    first = ints(band, "bfirst")
    band_tiles = int(sum(i - first[i] + 1 for i in range(len(first))))
    print(f"revisit 2000: ND {r['tiles']} tiles, {r['nupd']} products, {r['levels']} levels; insertion order {band_tiles} tiles")
    assert r["tiles"] < band_tiles / 2


def test_nd_tables_after_removals():
    g = gg.make_config(2, seed=3)
    def build(api):
        info = gg.build_bulk(api, g)
        for p in (17, 90, 91, 200):
            api.remove_node(int(info["pose_ids"][p]))
        for e in range(0, len(g.pp_pose), 37):
            if g.pp_pose[e] not in (17, 90, 91, 200):
                api.remove_factor(int(info["pp_fids"][e]))
        api.remove_node(int(info["plane_ids"][7]))
        return info
    check_nd(compiled(build)[0])


# ---------------------------------------------------------------- refusals
def revisit_api(n, order):
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    api.set_direct_ordering(order)
    gg.build_bulk(api, gg.make_revisit(seed=0, n_poses=n, n_planes=n // 20))
    return api


def test_revisited_map_over_the_band_budget_fits_in_nd_order():
    """20 000 poses driven twice over: the insertion-order envelope needs more than 8 GiB, the ND pattern a fraction of it"""
    band = revisit_api(20000, 0)
    with pytest.raises(capi.ApiError, match=r"band linear solver: the graph needs \d+ bytes") as e:
        band._chk(band.lib.pus_debug_compile(band.h))
    need = int(str(e.value).split("needs ")[1].split(" bytes")[0])
    assert need > BUDGET
    nd = revisit_api(20000, 1)
    nd._chk(nd.lib.pus_debug_compile(nd.h))
    got = int(nd.debug_fetch("bbytes", 1)[0])
    print(f"revisit 20000: insertion order {need / 2**30:.2f} GiB, nested dissection {got / 2**30:.2f} GiB")
    assert got < BUDGET / 2


def test_nd_refuses_a_graph_over_the_budget():
    """20 000 poses, each joined to its predecessor and to a random earlier pose: a random graph has no small separators,
    so its fill is close to dense in any order (a star, by contrast, has no fill at all once its hub is ordered last)"""
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    api.set_direct_ordering(1)
    ut = gg.diag_ut([1.0] * 6)
    rng = np.random.default_rng(0)
    ids = [api.add_pose(None)]
    api.add_pose_prior(ids[0], [0, 0, 0, 0, 0, 0], ut)
    for i in range(1, 20000):
        ids.append(api.add_pose(None))
        api.add_odometry(ids[i - 1], ids[i], [0.1, 0, 0, 0, 0, 0], ut)
        j = int(rng.integers(0, i))
        if j != i - 1:
            api.add_odometry(ids[j], ids[i], [0.1 * (i - j), 0, 0, 0, 0, 0], ut)
    with pytest.raises(capi.ApiError, match=r"band linear solver \(nested-dissection order\): the graph needs \d+ bytes") as e:
        api._chk(api.lib.pus_debug_compile(api.h))
    assert int(str(e.value).split("needs ")[1].split(" bytes")[0]) > BUDGET


def test_bad_orders_are_refused():
    api = GpuGraphAPI()
    for order in (-1, 2):
        assert api.lib.pus_set_direct_ordering(api.h, order) < 0
        assert b"bad direct ordering" in api.lib.pus_last_error()
        with pytest.raises(ValueError):
            api.set_direct_ordering(order)
    with pytest.raises(ValueError):
        api.set_direct_ordering(True)
    assert api.direct_ordering() == 0
    api.set_direct_ordering(1)
    assert api.direct_ordering() == 1 and api.linear_solver_kind() == 0   # accepted at any time; used by kind 2 only


def test_order_does_not_touch_other_kinds():
    g = gg.make_config(2, seed=0)
    for kind in (0, 1):
        api = GpuGraphAPI()
        api.set_linear_solver(kind)
        api.set_direct_ordering(1)
        gg.build_bulk(api, g)
        api._chk(api.lib.pus_debug_compile(api.h))
        assert ints(api, "ndtile").tolist() == []


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_nd_order_has_no_cpu_fallback_without_a_gpu():
    g = gg.make_config(1, seed=0)
    api = GpuGraphAPI()
    api.set_linear_solver(2)
    api.set_direct_ordering(1)
    gg.build_interleaved(api, g)
    gg.configure(api, g)
    with pytest.raises(capi.ApiError, match="no CUDA device available"):
        api.batch_optimize()
