"""The plane map (pus_map_*) on the device against the host oracle (tests/map_oracle.cpp) on top of the same graph:
seeded corridors under both presets, the pose prediction, host and device inputs, refusals and repeatability."""
import math

import numpy as np
import pytest

import map_native as M
from pop_up_slam_b200 import capi

pytestmark = pytest.mark.gpu


def new_map(preset, **over):
    api = capi.GpuGraphAPI()
    p = api.get_properties()
    api.set_properties(method=1, mod_batch=1, epsilon2=p["epsilon2"] * 0.1, epsilon_abs=p["epsilon_abs"] * 0.1,
                       epsilon_rel=p["epsilon_rel"] * 0.1)   # Mapping.cpp:31-43
    cfg = capi.map_config(preset, M.INVK, **over)   # (init_wTo: the corridor's first camera, passed in `over`)
    return api, capi.PlaneMap(api, cfg), cfg


def close_err(a, b):
    """match errors agree bit for bit except through acos, where CUDA's and glibc's may differ by an ulp or two; an angle
    error of 2 ulp of pi moves the error by far less than 1e-12 relative"""
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    return a == b or abs(a - b) <= 1e-12 * max(1.0, abs(a))


def run(preset, frames, check=True, **over):
    """maps the frames with main_3d's loop: the odometry is the map's own constant-motion prediction"""
    api, pm, cfg = new_map(preset, init_wTo=frames[0]["T"], **over)
    poses, history = [], []
    for seq, fr in enumerate(frames):
        lm = pm.landmarks()
        alive = np.array([0 if l["deleted"] else 1 for l in lm], np.int32)
        lw = np.array([api.get_plane(l["node"]) if a else [1, 0, 0, 0] for l, a in zip(lm, alive)]).reshape(-1, 4)
        T, odom = pm.predict_pose()
        last = api.get_pose(poses[-1]) if poses else None
        prev = api.get_pose(poses[-2]) if len(poses) > 1 else None
        o_odom, _, o_T = M.oracle_predict(len(poses), last, prev, cfg.init_wTo)
        assert np.array_equal(odom, o_odom) and np.array_equal(T, o_T), seq
        n_nodes, n_fac = api.num_nodes(), api.num_factors()
        r = pm.process_frame(seq, planes=fr)
        if check:
            P = M.planes_array(fr)
            o = M.oracle_associate(cfg, seq, len(poses), last if last is not None else np.zeros(7), odom, P,
                                   lm.view(M.LANDMARK) if len(lm) else np.zeros(0, M.LANDMARK), lw, alive)
            assert list(r["landmark"]) == list(o["assoc"]) and list(r["status"]) == list(o["status"]), seq
            assert all(close_err(a, b) for a, b in zip(r["error"], o["aerr"])), seq
            assert r["pose_node"] == n_nodes and list(r["new_nodes"]) == list(range(n_nodes + 1, n_nodes + 1 + o["n_new"]))
            n_ground_new = sum(1 for i in range(len(P)) if o["assoc"][i] >= len(lm) and P[i]["ind"] == 0)
            assert r["factor"][0] == n_fac + 1 + n_ground_new * (P[0]["ind"] == 0) and api.num_factors() == n_fac + 1 + len(P) + n_ground_new
            want = M.oracle_apply(seq, P, o["assoc"], lm.view(M.LANDMARK) if len(lm) else np.zeros(0, M.LANDMARK), o["n_new"], r["new_nodes"])
            lw1 = np.array([api.get_plane(n) for n in want["node"]]).reshape(-1, 4)
            want = M.oracle_reproject(want, lw1, np.ones(len(want), np.int32))
            got = pm.landmarks().view(M.LANDMARK)
            assert got.tobytes() == want.tobytes(), seq
        poses.append(r["pose_node"])
        history.append(r)
        assert np.isfinite(api.get_pose(r["pose_node"])).all(), seq
    chi2 = api.chi2()
    assert np.isfinite(chi2)
    out = dict(lm=pm.landmarks().tobytes(), poses=np.array([api.get_pose(p) for p in poses]).tobytes(),
               chi2=chi2, meas=[api.get_measurement(f).tobytes() for r in history for f in r["factor"]])
    return api, pm, out, history


@pytest.mark.parametrize("preset", ["tum_far", "mapping_h"])
def test_corridor_against_oracle(preset):
    frames = M.corridor(3, 40)
    _, _, a, hist = run(preset, frames)
    statuses = np.concatenate([h["status"] for h in hist])
    assert (statuses == 0).sum() > 40 and (statuses == 2).sum() > 5
    _, _, b, _ = run(preset, frames, check=False)            # a fresh map repeats the bytes
    assert a == b


def test_device_inputs_equal_host_inputs():
    torch = pytest.importorskip("torch")
    frames = M.corridor(5, 12)
    _, _, host, _ = run("tum_far", frames, check=False)
    api, pm, cfg = new_map("tum_far", init_wTo=frames[0]["T"])
    for seq, fr in enumerate(frames):
        T = torch.zeros(16, dtype=torch.float32, device="cuda")
        pm.predict_pose(T)                                      # the prediction lands in device memory
        Th, _ = capi.PlaneMap.predict_pose(pm)
        assert np.array_equal(T.cpu().numpy().reshape(4, 4), Th)
        arrs = capi.PlaneMap._arrays(fr)
        dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in arrs.items()}
        torch.cuda.synchronize()
        pm.process_frame(seq, planes=dev)
    assert pm.landmarks().tobytes() == host["lm"]


def test_refusal_leaves_map_and_handle_unchanged():
    frames = M.corridor(9, 6)
    api, pm, cfg = new_map("mapping_h")
    for seq in range(3):
        pm.predict_pose()
        pm.process_frame(seq, planes=frames[seq])
    before = (api.num_nodes(), api.num_factors(), pm.landmarks().tobytes())
    bad = dict(frames[3])
    bad["planes_sensor"] = bad["planes_sensor"].copy()
    bad["planes_sensor"][1, 2] = np.nan
    with pytest.raises(capi.ApiError, match="not finite"):
        pm.process_frame(3, planes=bad)
    two_grounds = dict(frames[3], plane_indice=np.zeros(len(frames[3]["dist"]), np.int32))
    with pytest.raises(capi.ApiError, match="ground"):
        pm.process_frame(3, planes=two_grounds)
    assert (api.num_nodes(), api.num_factors(), pm.landmarks().tobytes()) == before
    pm.process_frame(3, planes=frames[3])                      # still usable
    assert api.num_nodes() > before[0]


def test_removed_landmark_is_deleted_and_skipped():
    frames = M.corridor(11, 8)
    api, pm, cfg = new_map("tum_far")
    for seq in range(4):
        pm.predict_pose()
        pm.process_frame(seq, planes=frames[seq])
    lm = pm.landmarks()
    victim = int(lm[1]["node"])
    api.remove_node(victim)
    assert pm.landmarks()[1]["deleted"] == 1
    for seq in range(4, 8):
        pm.predict_pose()
        r = pm.process_frame(seq, planes=frames[seq])
        assert 1 not in list(r["landmark"])
    assert pm.landmarks()[1].tobytes()[-40:] == lm[1].tobytes()[-40:]   # never re-projected again


def test_session_form_equals_array_form():
    import popup_frames_native as NF
    imgs, labs, Ts = NF.rooms(3, 6, 640, 480)
    cfg = NF.config(640, 480)
    sess = capi.PopupFrames(capi.load_library(), cfg)
    out = sess.run(imgs, labs, Ts)
    ident = np.array([0, 0, 0, 1, 0, 0, 0], float)
    maps = [new_map("tum_far", init_wTo=Ts[0].astype(float)) for _ in range(2)]
    mapped = 0
    for f in range(len(Ts)):
        g0, g1 = out["good_ptr"][f], out["good_ptr"][f + 1]
        rows_in = out["good_rows"][g0:g1]
        o0, o1 = out["open_ptr"][f], out["open_ptr"][f + 1]
        rows = o0 + f + rows_in
        bound = [out["bound2d"][out["bound_ptr"][r]:out["bound_ptr"][r + 1]] for r in rows]
        world = [out["world3d"][out["world_ptr"][r]:out["world_ptr"][r + 1]] for r in rows]
        planes = dict(planes_sensor=out["planes_sensor"][rows], dist=out["dist"][rows], plane_indice=rows_in, bound=bound,
                      world=world, segs=out["open_segs"][o0:o1])
        a = maps[0][1].process_frame(f, planes=planes, odom7=ident)
        b = maps[1][1].process_frame(f, session=(sess, f), odom7=ident)
        for k in ("landmark", "status", "factor", "error", "new_nodes"):
            assert np.array_equal(a[k], b[k]), (f, k)
        mapped += a["n_planes"] > 0
    assert mapped >= 3
    assert maps[0][1].landmarks().tobytes() == maps[1][1].landmarks().tobytes()
    n = maps[0][0].num_nodes()
    assert n == maps[1][0].num_nodes() and n > 0
    for i in range(n):
        try:
            pa, pb = maps[0][0].get_pose(i), maps[1][0].get_pose(i)
        except capi.ApiError:
            pa, pb = maps[0][0].get_plane(i), maps[1][0].get_plane(i)
        assert pa.tobytes() == pb.tobytes()


def _path_ab(preset, frames_iter, init_wTo, invK):
    """Path A: a session run on the map's own prediction (a device T16) -> pus_map_process_frame in the session form.
    Path B: the same session outputs downloaded -> host-oracle association -> capi add calls on a second handle -> the same
    solves -> pus_refresh_bind / run -> pus_project_to_planes.  After every frame the two graphs and tables are compared."""
    torch = pytest.importorskip("torch")
    import oracle_api as O
    apiA, pmA, cfg = new_map(preset, init_wTo=init_wTo)
    cfg.invK[:] = [float(x) for x in np.asarray(invK, np.float32).reshape(9)]
    pmA.close()
    pmA = capi.PlaneMap(apiA, cfg)
    apiB, pmB_unused, _ = new_map(preset, init_wTo=init_wTo)
    pmB_unused.close()
    B = M.PathB(apiB, cfg)
    mapped = 0
    for seq, (sess, img, lab) in enumerate(frames_iter):
        T = torch.zeros(16, dtype=torch.float32, device="cuda")
        _, odom = pmA.predict_pose(T)
        o_odom, o_pred, o_T = B.predict()
        assert np.array_equal(odom, o_odom) and np.array_equal(T.cpu().numpy().reshape(4, 4), o_T), seq
        # main_3d's pose arithmetic restated on the independent oracle poses (the library renormalises oplus)
        r_odom, r_pred, r_T = M.py_predict(len(B.frame_pose), apiB.get_pose(B.frame_pose[-1]) if B.frame_pose else None,
                                           apiB.get_pose(B.frame_pose[-2]) if len(B.frame_pose) > 1 else None, list(cfg.init_wTo),
                                           O.pose_from_mat4, O.pose_ominus, O.pose_oplus, O.pose_wTo)
        assert np.abs(odom - r_odom).max() <= 1e-12 and np.abs(T.cpu().numpy().reshape(4, 4) - r_T).max() <= 1e-5
        out = sess.run(torch.from_numpy(img).cuda(), torch.from_numpy(lab).cuda(), T.reshape(1, 4, 4))
        host = {k: v.cpu().numpy() for k, v in out.items()}
        a = pmA.process_frame(seq, session=(sess, 0), odom7=odom)
        b = B.frame(seq, M.session_frame(host, 0), odom)
        if b is None:
            assert a["n_planes"] == 0
            continue
        mapped += 1
        for k in ("landmark", "status", "factor", "new_nodes", "pose_node"):
            assert np.array_equal(a[k], b[k]), (seq, k)
        assert apiA.num_nodes() == apiB.num_nodes() and apiA.num_factors() == apiB.num_factors()
        poses = B.frame_pose
        assert apiA.get_poses(poses).tobytes() == apiB.get_poses(poses).tobytes(), seq
        nodes = [int(n) for n in B.lm["node"]]
        assert apiA.get_planes(nodes).tobytes() == apiB.get_planes(nodes).tobytes(), seq
        for f in B.map_fid:
            assert apiA.get_measurement(f).tobytes() == apiB.get_measurement(f).tobytes(), (seq, f)
        assert apiA.chi2() == apiB.chi2()
        assert pmA.landmarks().view(M.LANDMARK).tobytes() == B.lm.tobytes(), seq
    return mapped


@pytest.mark.parametrize("preset", ["tum_far", "mapping_h"])
def test_path_a_equals_path_b_moving_room(preset):
    import popup_frames_native as NF
    import popup_polygon_native as NP
    K = NP.camera_K(640, 480).astype(np.float64)
    imgs, labs, Ts = M.moving_room(17, 24, 640, 480, K)
    sess = capi.PopupFrames(capi.load_library(), NF.config(640, 480))
    invK = np.linalg.inv(K).astype(np.float32)
    assert _path_ab(preset, ((sess, imgs[i:i + 1], labs[i:i + 1]) for i in range(len(imgs))), Ts[0], invK) >= 12


@pytest.mark.parametrize("preset", ["tum_far", "mapping_h"])
def test_path_a_equals_path_b_sample_frames(preset):
    import popup_frames_native as NF
    samples = NF.samples()
    frames = []
    for img, lab, Ts in samples:
        h, w = lab.shape[1:]
        frames.append((capi.PopupFrames(capi.load_library(), NF.config(w, h)), img, lab))
    h, w = samples[0][1].shape[1:]
    invK = NF.config(w, h)["invK"]
    assert _path_ab(preset, iter(frames), samples[0][2][0].astype(np.float64), invK) >= 2


def test_two_maps_in_turn_on_one_handle():
    """a destroyed map gives the refresh tables up: the next map on the handle starts its own"""
    frames = M.corridor(13, 20)
    api, pm, cfg = new_map("tum_far", init_wTo=frames[0]["T"])
    for seq in range(18):   # past the tables' first growth
        pm.predict_pose()
        pm.process_frame(seq, planes=frames[seq])
    pm.close()
    n0 = api.num_nodes()
    for seq in range(n0):   # the first map's nodes go: the second map must not re-pop their frames
        api.remove_node(seq)
    pm2 = capi.PlaneMap(api, cfg)
    for seq in range(18, 20):
        pm2.predict_pose()
        r = pm2.process_frame(seq, planes=frames[seq])
        assert r["n_planes"] > 0
    assert len(pm2.landmarks()) > 0


_CAM = M.camera(np.array([0.0, 0.0, 1.0]), 0.0, math.radians(12))   # 1 m up, looking along +x, pitched down


def _wall(x, y0, y1):
    """the wall x = const between y0 and y1 (world), as the pop-up gives it: its plane in the camera frame, its ground line
    in pixels as the 2-D bound's first two vertices and the open segment, its ground end points as the world polygon"""
    Tinv = np.linalg.inv(_CAM)
    px = []
    for y in (y0, y1):
        c = Tinv[:3, :3] @ np.array([x, y, 0.0]) + Tinv[:3, 3]
        q = M.K @ c
        px.append([q[0] / q[2], q[1] / q[2]])
    return (M._plane_T(_CAM.tolist(), [-1.0, 0.0, 0.0, float(x)]), px + [[px[1][0], 0.0], [px[0][0], 0.0]],
            [[x, y0, 0.0], [x, y1, 0.0]], float(x))


def _frame(planes):
    ps = [M._plane_T(_CAM.tolist(), [0.0, 0.0, -1.0, 0.0])] + [p[0] for p in planes]
    bound = [[[0, 479], [639, 479], [639, 300], [0, 300]]] + [p[1] for p in planes]
    world = [[]] + [p[2] for p in planes]
    dist = [1.0] + [p[3] for p in planes]
    segs = [[b[0][0], b[0][1], b[1][0], b[1][1]] for b in (p[1] for p in planes)]
    return dict(planes_sensor=np.array(ps, np.float32), dist=np.array(dist, np.float32),
                plane_indice=np.arange(len(ps), dtype=np.int32), bound=bound, world=world,
                segs=np.array(segs, np.float32).reshape(-1, 4), T=_CAM)


def test_crafted_frames_against_oracle():
    """ground first, ties, dual matches both ways and a chain numbered out of plane order, on the device against the
    oracle (run() compares every frame)"""
    long_, short_ = _wall(5.0, -1.0, 2.0), _wall(5.0, 0.0, 0.5)
    far = _wall(40.0, -1.0, 2.0)
    # two more short walls that have no landmark of their own when they first meet the long one's (a short wall that loses
    # a dual match becomes a landmark, and the next sight of that same wall matches it)
    short2, short3 = _wall(5.0, -1.0, 1.5), _wall(5.0, 0.5, 2.0)
    ground_only = dict(_frame([long_]), planes_sensor=_frame([])["planes_sensor"], dist=np.array([1.0], np.float32),
                       plane_indice=np.array([0], np.int32), bound=_frame([])["bound"], world=[[]])
    frames = [
        ground_only,                     # the first frame's planes are initialised through the identity: no walls there
        _frame([long_, long_]),          # two identical walls: two landmarks, a tie later
        _frame([long_]),                 # the tie: the earlier landmark wins
        _frame([short_, long_]),         # dual: the later, longer one keeps it
        _frame([long_, short2]),         # dual: the earlier one keeps it
        _frame([short3, far, long_]),    # the chain: the far wall is new first, the short one is numbered after it
    ]
    _, _, _, hist = run("tum_far", frames)
    st = [list(h["status"]) for h in hist][1:]
    lm = [list(h["landmark"]) for h in hist][1:]
    assert lm[1][1] == 1                                                  # the tie: the earlier landmark
    assert st[2][1:] == [3, 0] and st[3][1:] == [0, 3] and st[4][1:] == [3, 2, 0]
    assert lm[4][1] > lm[4][2]                                            # numbered out of plane order
    assert all(h["landmark"][0] == 0 for h in hist[1:])                   # the ground takes the first ground landmark
