"""Host tables of the marginal covariances (DESIGN.md section 5.4), without a GPU: the selected-inversion list of every stored
tile and the eliminated planes' observer-pair lists, restated in Python from the nested-dissection tables, on a corridor, the
revisited corridor and sphere2500.  Checks that every Sigma tile a list names is stored, that the lists are k-ascending and
cover R_j, and that each plane's pair list covers all its observer pairs."""
import numpy as np
import pytest

from pop_up_slam_b200 import graphgen as gg
from test_nd_tables import bulk, compiled, ints, sphere

LD = 52
TILE_BYTES = 48 * LD * 8


def check_cov(api):
    cptr, crow = ints(api, "ndcptr"), ints(api, "ndcrow")
    toff, trow, tcol = ints(api, "ndtoff"), ints(api, "ndtrow"), ints(api, "ndtcol")
    pos = np.argsort(ints(api, "ndtile"))
    nb, T = len(cptr) - 1, int(cptr[-1])
    stored = {(int(trow[t]), int(tcol[t])): t for t in range(T)}
    sptr, sel = ints(api, "covsptr"), ints(api, "covsel").reshape(-1, 2)
    assert len(sptr) == T + 1
    for t in range(T):
        i, j = int(trow[t]), int(tcol[t])
        lst = sel[sptr[t]:sptr[t + 1]]
        R = [int(k) for k in crow[cptr[j] + 1:cptr[j + 1]]]
        if i == j:
            assert len(lst) == 0
            continue
        assert len(lst) == len(R)
        assert np.all(np.diff(lst[:, 1]) == 1)   # the L tiles (k, j) in storage order: k ascending
        for (code, lt), k in zip(lst, R):
            hi, lo = max(i, k), min(i, k)
            assert code >> 1 == stored[(hi, lo)], (t, k)       # the Sigma tile is stored
            assert code & 1 == (1 if i < k else 0)
            assert int(trow[lt]) == k and int(tcol[lt]) == j   # the L tile (k, j)
    # the eliminated planes' observer pairs
    border = set(ints(api, "bborder").tolist())
    inc_pose, inc_plane = ints(api, "dinc_pose"), ints(api, "dinc_plane")
    iptr, pptr, pair = ints(api, "covincptr"), ints(api, "covpptr"), ints(api, "covpair").reshape(-1, 4)
    M = len(iptr) - 1
    assert np.array_equal(iptr, np.searchsorted(inc_plane, np.arange(M + 1)))
    npair = 0
    for l in range(M):
        lst = pair[pptr[l]:pptr[l + 1]]
        if l in border:
            assert len(lst) == 0
            continue
        want = [(qa, qb) for qa in range(iptr[l], iptr[l + 1]) for qb in range(iptr[l], qa + 1)]
        assert [(int(a), int(b)) for a, b, _, _ in lst] == want, l
        npair += len(want)
        for qa, qb, tile, code in lst:
            a, b = int(inc_pose[qa]), int(inc_pose[qb])
            ti, tj = int(pos[6 * a // 48]), int(pos[6 * b // 48])
            assert tile == stored[(max(ti, tj), min(ti, tj))]
            er, ec = 6 * a % 48, 6 * b % 48
            flag = 1 if ti < tj else 0
            assert code == 2 * (ec * LD + er if flag else er * LD + ec) + flag
    m = np.diff(cptr) - 1
    nsel = int(np.sum(m * m))
    want_bytes = T * TILE_BYTES + 8 * nsel + 4 * (T + 1) + 16 * npair + 4 * (M + 1) + 16
    assert int(api.debug_fetch("covbytes", 1)[0]) == want_bytes
    return dict(T=T, nsel=nsel, npair=npair, nupd=int(np.sum(m * (m + 1) // 2)))


def report(name, r):
    print(f"{name}: {r['T']} tiles, {r['nsel']} selected-inversion entries ({r['nsel'] / max(r['nupd'], 1):.2f} x nupd), "
          f"{r['npair']} plane pairs")


def test_cov_tables_corridor():
    report("config 2", check_cov(compiled(bulk(gg.make_config(2, seed=0)))[0]))


def test_cov_tables_revisited_corridor():
    report("revisited 2000", check_cov(compiled(bulk(gg.make_revisit(seed=0, n_poses=2000, n_planes=100)))[0]))


def test_cov_tables_sphere2500():
    report("sphere2500", check_cov(compiled(sphere("sphere2500"))[0]))


def test_cov_tables_refuse_insertion_order():
    api, _ = compiled(bulk(gg.make_config(1, seed=0)), order=0)
    with pytest.raises(Exception, match="not a nested-dissection layout"):
        api.debug_fetch("covsptr", 1 << 20)
