"""The plane map's rules on the host (tests/map_oracle.cpp: pus_map.cuh compiled for the host) against an independent
line-by-line Python restatement of Mapping.cpp:112-126, 256-460, Map_plane.cpp and main_3d.cpp:366-385: seeded corridors
under both presets and one crafted case per branch.  No GPU needed."""
import math

import numpy as np
import pytest

import map_native as M
from pop_up_slam_b200 import capi


def cfg(preset, **over):
    return capi.map_config(preset, M.INVK, **over)


def check_against_python(c, counts):
    def check(seq, P, lm, lw, alive, r):
        wTo, oTw = M.pose_T(r["est"])
        py = M.py_associate(c, seq, wTo, oTw, P, lm, lw, alive)
        for k in ("id", "assoc", "status"):
            assert list(py[k]) == list(r[k]), (seq, k)
        assert py["n_new"] == r["n_new"]
        for a, b in zip(py["err"], r["err"]):
            assert (math.isnan(a) and math.isnan(b)) or a == b, seq
        for a, b in zip(py["aerr"], r["aerr"]):
            assert (math.isnan(a) and math.isnan(b)) or a == b, seq
        for s in r["status"]:
            counts[int(s)] = counts.get(int(s), 0) + 1
    return check


@pytest.mark.parametrize("preset", ["tum_far", "mapping_h"])
def test_corridor_oracle_equals_python(preset):
    c = cfg(preset)
    counts = {}
    lm = M.replay(c, M.corridor(7, 300), check_against_python(c, counts))
    assert counts.get(0, 0) > 300 and counts.get(2, 0) > 10            # both matches and new landmarks occur
    assert lm["being_tracked_times"].sum() == sum(counts.values())      # copy_plane once per observation


def _plane(ind, local, v2, v3, dist=4.0):
    return dict(planes_sensor=[local], dist=[dist], plane_indice=[ind], bound=[v2], world=[v3])


def _lm(**kw):
    L = np.zeros(1, M.LANDMARK)
    for k, v in kw.items():
        L[k] = v
    return L[0]


ID7 = [0, 0, 0, 1, 0, 0, 0]
WALL = [0.0, -1.0, 0.0, 2.0]   # y = 2 in the camera frame (identity estimate: the world too)
V2 = [[100, 400], [300, 400]]
V3 = [[0, 2, 0], [3, 2, 0]]


def pair(c, P, L, lw, seq=10):
    p = M.planes_array(P)[0]
    err = M.C.c_double(0)
    code = M.oracle_lib().orc_map_pair(M.C.byref(c), seq, M._p(np.array([p])), M._p(np.array(ID7, float)), M._p(np.array([L])),
                                       M._p(np.array(lw, float)) if lw is not None else None, M.C.byref(err))
    wTo, oTw = M.pose_T(ID7)
    kind, e = M.py_pair(c, seq, p, wTo, oTw, L, lw)
    return code, err.value, kind, e


def wall_lm(**kw):
    base = dict(frame_plane_indice=1, frame_seq_id=9, n_bound2d=2, n_world3d=2, bound2d=V2, world3d=V3)
    base.update(kw)
    return _lm(**base)


def test_branches():
    c = cfg("mapping_h")
    P = _plane(1, WALL, V2, V3)
    assert pair(c, P, wall_lm(), WALL)[:1] == (9,) and pair(c, P, wall_lm(), WALL)[2] == "cand"
    assert pair(c, P, wall_lm(), None)[0] == 0                                           # deleted
    assert pair(c, P, wall_lm(frame_plane_indice=0), WALL)[0] == 2                       # wall against ground
    assert pair(c, P, wall_lm(n_world3d=1), WALL)[0] == 3                                # short landmark
    assert pair(c, P, wall_lm(frame_seq_id=4), WALL, seq=10)[0] == 4                     # the window (10 - 4 > 5)
    assert pair(c, P, wall_lm(frame_seq_id=5), WALL, seq=10)[0] == 9                     # 10 - 5 = 5 stays in
    tilted = [math.sin(math.radians(70)), -math.cos(math.radians(70)), 0, 2.0]
    assert pair(c, P, wall_lm(), tilted)[0] == 5                                         # 70 deg > 60
    assert pair(c, P, wall_lm(), [0.0, -1.0, 0.0, 6.5])[0] == 6                          # plane distance 4.5 > 4
    assert pair(c, P, wall_lm(bound2d=[[400, 100], [600, 100]]), WALL)[0] == 7           # 2-D end points
    assert pair(c, P, wall_lm(world3d=[[10, 2, 0], [12, 2, 0]]), WALL)[0] == 8           # no covering
    for a in (5.0, 20.0, 30.0):                                                          # <= 10, < 25 and the default rule
        r = math.radians(a)
        code, e, kind, pe = pair(c, P, wall_lm(), [math.sin(r), -math.cos(r), 0, 2.0])
        assert code == 9 and kind == "cand" and e == pe
    # the covering threshold (0.25 under 10 deg) is halved below a plane distance of 1.5: 0.2 passes at 0.1 m, not at 2 m
    half = wall_lm(world3d=[[0, 2, 0], [0.6, 2, 0]])
    assert pair(c, P, half, [0.0, -1.0, 0.0, 2.1])[0] == 9
    assert pair(c, P, half, [0.0, -1.0, 0.0, 4.0])[0] == 8
    # a degenerate old segment: point_proj_to_lineseg returns a distance, not a parameter
    assert M.oracle_lib().orc_map_proj(M._p(np.array([0, 0], np.float32)), M._p(np.array([0.0005, 0], np.float32)),
                                       M._p(np.array([3, 4], np.float32))) == 5.0
    assert M.proj_to_lineseg([0, 0], [0.0005, 0], [3, 4]) == 5.0


def _assoc(c, frame, lm, lw, seq=1):
    P = M.planes_array(frame)
    alive = np.array([0 if np.isnan(w).any() else 1 for w in lw], np.int32)
    lw = np.nan_to_num(np.asarray(lw, float))
    r = M.oracle_associate(c, seq, 1, ID7, ID7, P, lm, lw, alive)
    wTo, oTw = M.pose_T(r["est"])
    py = M.py_associate(c, seq, wTo, oTw, P, lm, lw, alive)
    assert list(py["assoc"]) == list(r["assoc"]) and list(py["status"]) == list(r["status"])
    return r


def test_ground_first_and_deleted_ground():
    c = cfg("mapping_h")
    g = _lm(frame_plane_indice=0, frame_seq_id=-100)   # outside the window: ground ignores it
    lm = np.array([wall_lm(), g, g, g])
    G = [0, 0, -1, 1.0]
    frame = _plane(0, G, V2, [])
    assert list(_assoc(c, frame, lm, [WALL, G, G, G])["assoc"]) == [1]
    assert list(_assoc(c, frame, lm, [WALL, [np.nan] * 4, G, G])["assoc"]) == [2]   # removed first ground


def test_dual_matches_and_numbering():
    c = cfg("tum_far")
    lm = np.array([wall_lm()])
    short, long_ = [[100, 400], [150, 400]], [[100, 400], [400, 400]]
    two = lambda a, b: dict(planes_sensor=[WALL, WALL], dist=[4, 4], plane_indice=[1, 2], bound=[a, b], world=[V3, V3])
    r = _assoc(c, two(short, long_), lm, [WALL])       # the later, longer one keeps it: the first loses with -1
    assert list(r["assoc"]) == [1, 0] and list(r["status"]) == [3, 0] and r["aerr"][0] == -1
    r = _assoc(c, two(long_, short), lm, [WALL])       # the earlier one keeps it: the second is new with 0
    assert list(r["assoc"]) == [0, 1] and list(r["status"]) == [0, 3] and r["aerr"][1] == 0
    # plane 1 has no candidate (new 1), then plane 2 takes landmark 0 from plane 0, which is numbered 2: out of plane order
    far = [[0.0, -1.0, 0.0, 9.0]]
    three = dict(planes_sensor=[WALL, far[0], WALL], dist=[4, 4, 4], plane_indice=[1, 2, 3], bound=[short, long_, long_],
                 world=[V3, V3, V3])
    r = _assoc(c, three, lm, [WALL])
    assert list(r["assoc"]) == [2, 1, 0] and list(r["status"]) == [3, 2, 0] and r["n_new"] == 2


def test_nan_first_and_later():
    c = cfg("tum_far")
    # a NaN angle passes the gate (NaN > thr is false) and gives a NaN error; the normals' dot exceeds 1 by rounding
    n = [0.1602141559123993, -0.8181289434432983, 0.5522648692131042, 0.0]
    P = M.planes_array(_plane(1, n, V2, V3))[0]
    wTo, oTw = M.pose_T(ID7)
    cw = M._plane_T(oTw, [float(x) for x in P["local"]])
    d = M._dot3(M._normal(cw), M._normal(cw))
    assert d > 1.0
    good = [cw[0] + 0.01, cw[1], cw[2], cw[3]]
    lm = np.array([wall_lm(), wall_lm()])
    r = _assoc(c, _plane(1, n, V2, V3), lm, [cw, good])            # NaN first: it wins and nothing replaces it
    assert r["assoc"][0] == 0 and math.isnan(r["err"][0])
    r = _assoc(c, _plane(1, n, V2, V3), lm, [good, cw])            # NaN later: ignored
    assert r["assoc"][0] == 0 and not math.isnan(r["err"][0])


def test_short_polygons_and_first_frame_identity():
    c = cfg("mapping_h")
    lm = np.array([wall_lm()])
    r = _assoc(c, _plane(1, WALL, [[100, 400]], V3), lm, [WALL])
    assert list(r["status"]) == [1] and list(r["assoc"]) == [1]
    P = M.planes_array(_plane(1, WALL, V2, V3))
    r = M.oracle_associate(c, 0, 0, np.zeros(7), [5, 6, 7, 0, 1, 0, 0], P, np.zeros(0, M.LANDMARK), np.zeros((0, 4)), [])
    assert list(r["est"]) == ID7                                     # estimate_pose is the identity on the first frame


def test_predict_pose_and_sigma():
    init = capi.TUM_FAR_INIT_WTO
    odom, pred, T = M.oracle_predict(0, None, None, init)
    assert np.array_equal(odom, pred) and np.array_equal(odom, M.T_to_pose(np.array(init).reshape(4, 4)))
    a = M.T_to_pose(M.corridor(1, 2)[0]["T"])
    b = M.T_to_pose(M.corridor(1, 2)[1]["T"])
    odom, pred, T = M.oracle_predict(1, b, None, init)
    assert list(odom) == ID7
    odom, pred, T = M.oracle_predict(2, b, a, init)
    assert np.array_equal(odom, M.ominus(b, a))
    wTo, _ = M.pose_T(pred)
    assert np.array_equal(T, np.array(wTo, np.float32))
    try:
        import ref_api as R
        if R.available():
            assert np.array_equal(odom, R.pose_ominus(b, a))
            # the library renormalises oplus's quaternion (pus_math.cuh, T_to_pose); the reference does not
            assert np.abs(pred - R.pose_oplus(b, odom)).max() <= 1e-15
    except ImportError:
        pass
    for d in (0.5, 3.0, 5.5, 8.0, 20.0):
        assert M.oracle_lib().orc_map_plane_sigma(d, 2.0) == M.py_sigma(d, 2.0)


KIND = {5: "angle", 6: "planedist", 7: "2d", 8: "cover", 9: "cand"}


def _rot(a_deg, d=4.2):
    r = math.radians(a_deg)
    return [math.sin(r), -math.cos(r), 0.0, d]   # plane distance to WALL about 1.6-2.2 m: no halving of the covering


def test_gate_boundaries_flip():
    """each threshold rule flips a pair on its own side of the boundary: the covering threshold (0.25 at <= 10 deg, 0.167
    below 25 deg, 0.5 above) against a covering of 0.2, and the 2-D threshold (x 1.5 below 25 deg) against 60 px"""
    c = cfg("mapping_h")
    P = _plane(1, WALL, V2, V3)
    cover02 = wall_lm(world3d=[[0, 2, 0], [0.6, 2, 0]])
    for a, want in ((5.0, 8), (9.9, 8), (10.1, 9), (20.0, 9), (24.9, 9), (25.1, 8), (30.0, 8)):
        code, e, kind, pe = pair(c, P, cover02, _rot(a))
        assert code == want and kind == KIND[want], a
        assert code != 9 or e == pe
    far2d = wall_lm(bound2d=[[160, 400], [360, 400]])
    for a, want in ((20.0, 9), (24.9, 9), (25.1, 7), (30.0, 7)):
        code, e, kind, pe = pair(c, P, far2d, _rot(a))
        assert code == want and kind == KIND[want], a


def test_predict_restated_on_independent_pose_arithmetic():
    """main_3d.cpp:366-385 restated in Python over the host oracle's own Pose3d (oracle/oracle_math.hpp), against the map's
    pus_math prediction; the float cast of wTo is compared too"""
    import oracle_api as O
    init = capi.TUM_FAR_INIT_WTO
    fr = M.corridor(4, 3)
    a, b = M.T_to_pose(fr[0]["T"]), M.T_to_pose(fr[1]["T"])
    for n, last, prev in ((0, None, None), (1, b, None), (2, b, a)):
        odom, pred, T = M.oracle_predict(n, last, prev, init)
        r_odom, r_pred, r_T = M.py_predict(n, last, prev, init, O.pose_from_mat4, O.pose_ominus, O.pose_oplus, O.pose_wTo)
        assert np.abs(odom - r_odom).max() <= 1e-15 and np.abs(pred - r_pred).max() <= 1e-15, n
        assert np.array_equal(T, r_T) or np.abs(T - r_T).max() <= 1e-6, n
        try:
            import ref_api as R
            if R.available():
                assert np.array_equal(np.asarray(R.pose_wTo(pred), np.float64).astype(np.float32), T)
        except ImportError:
            pass
