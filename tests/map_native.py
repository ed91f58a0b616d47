"""Test-side helpers for the plane map (pus_map_*): the host oracle (tests/map_oracle.cpp, pus_map.cuh compiled for the
host), an independent line-by-line Python restatement of findClosestPlane / the one-to-one rule / copy_plane
(pop_planar_slam/src/Mapping.cpp:112-126, 256-460, Map_plane.cpp:11-29), and seeded synthetic corridors.
Test infrastructure only."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np

from pop_up_slam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PI = 3.14159265358979323846   # isam::PI (util.h:40)
f32 = np.float32

PLANE = np.dtype([("local", "<f8", 4), ("dist", "<f4"), ("ind", "<i4"), ("good", "<i4"), ("n2", "<i4"), ("n3", "<i4"),
                  ("v2", "<f4", 4), ("v3", "<f4", 6)], align=True)
LANDMARK = np.dtype([(k, "<i4") for k in ("node", "deleted", "frame_seq_id", "frame_plane_indice", "good_plane_indice",
                                          "being_tracked_times")] + [
    ("plane_dist_cam", "<f8"), ("n_bound2d", "<i4"), ("n_world3d", "<i4"), ("bound2d", "<f4", (2, 2)), ("world3d", "<f4", (2, 3))],
    align=True)

_lib = None


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="map_oracle_"), "liborc_map.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               "-I/usr/local/cuda/include", os.path.join(ROOT, "tests", "map_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_map_plane_sigma.restype = C.c_double
        _lib.orc_map_plane_sigma.argtypes = [C.c_double, C.c_double]
        _lib.orc_map_proj.restype = C.c_float
        assert _lib.orc_map_plane_size() == PLANE.itemsize and _lib.orc_map_landmark_size() == LANDMARK.itemsize
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def planes_array(fr):
    """a frame dict (planes_sensor, dist, plane_indice, bound, world) -> PLANE records through the oracle"""
    n = len(fr["dist"])
    n2 = np.array([min(len(b), 2) for b in fr["bound"]], np.int32)
    n3 = np.array([min(len(w), 2) for w in fr["world"]], np.int32)
    v2 = np.zeros((n, 4), f32)
    v3 = np.zeros((n, 6), f32)
    for i in range(n):
        v2[i, :2 * n2[i]] = np.asarray(fr["bound"][i], f32).reshape(-1)[:2 * n2[i]]
        v3[i, :3 * n3[i]] = np.asarray(fr["world"][i], f32).reshape(-1)[:3 * n3[i]]
    out = np.zeros(n, PLANE)
    oracle_lib().orc_map_planes(n, _p(np.ascontiguousarray(fr["planes_sensor"], f32)), _p(np.ascontiguousarray(fr["dist"], f32)),
                                _p(np.ascontiguousarray(fr["plane_indice"], np.int32)), _p(n2), _p(n3), _p(v2), _p(v3), _p(out))
    return out


def oracle_associate(cfg, seq, n_mapped, last7, odom7, P, lm, lw, alive):
    n, L = len(P), len(lm)
    est = np.zeros(7)
    idv, assoc, status = (np.zeros(max(n, 1), np.int32) for _ in range(3))
    err, aerr = np.zeros(max(n, 1)), np.zeros(max(n, 1))
    lw = np.ascontiguousarray(lw, np.float64).reshape(-1, 4) if L else np.zeros((1, 4))
    alive = np.ascontiguousarray(alive, np.int32) if L else np.zeros(1, np.int32)
    lm_ = lm if L else np.zeros(1, LANDMARK)
    nn = oracle_lib().orc_map_associate(C.byref(cfg), int(seq), int(n_mapped), _p(np.asarray(last7, float)), _p(np.asarray(odom7, float)),
                                        n, _p(P), L, _p(lm_), _p(lw), _p(alive), _p(est), _p(idv), _p(err), _p(assoc), _p(aerr),
                                        _p(status))
    return dict(est=est, id=idv[:n], err=err[:n], assoc=assoc[:n], aerr=aerr[:n], status=status[:n], n_new=nn)


def oracle_apply(seq, P, assoc, lm, n_new, nodes):
    L0 = len(lm)
    out = np.concatenate([lm, np.zeros(n_new, LANDMARK)])
    oracle_lib().orc_map_apply(int(seq), len(P), _p(P), _p(np.ascontiguousarray(assoc, np.int32)), L0, int(n_new),
                               _p(np.ascontiguousarray(nodes, np.int32) if n_new else np.zeros(1, np.int32)), _p(out))
    return out


def oracle_reproject(lm, lw, alive):
    out = lm.copy()
    if len(out):
        oracle_lib().orc_map_reproject(len(out), _p(out), _p(np.ascontiguousarray(lw, np.float64)), _p(np.ascontiguousarray(alive, np.int32)))
    return out


def oracle_predict(n_mapped, last7, prev7, init_wTo):
    odom, pred, T = np.zeros(7), np.zeros(7), np.zeros(16, f32)
    z = np.zeros(7)
    oracle_lib().orc_map_predict(int(n_mapped), _p(np.asarray(last7 if last7 is not None else z, float)),
                                 _p(np.asarray(prev7 if prev7 is not None else z, float)), _p(np.asarray(init_wTo, float)),
                                 _p(odom), _p(pred), _p(T))
    return odom, pred, T.reshape(4, 4)


# ---- Python restatement (plain floats; float32 where the reference uses float) ---------------------------------------
def _norm3(v): return math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
def _normal(v): z = _norm3(v); return [v[0] / z, v[1] / z, v[2] / z]
def _dot3(a, b): return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _plane_T(T, p):                       # Plane3d(T^T * p), normalised
    r = []
    for i in range(4):
        s = 0.0
        for j in range(4):
            s += T[j][i] * p[j]
        r.append(s)
    z = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]
    n = math.sqrt(z)
    return [x / n for x in r]


def _n2f(a, b):                          # (Vector2f a - b).norm()
    x, y = f32(a[0]) - f32(b[0]), f32(a[1]) - f32(b[1])
    return f32(np.sqrt(f32(x * x + y * y)))


def _min2f(a, b): return b if b < a else a


def proj_to_lineseg(b, e, q):            # Mapping.cpp:112-126
    length = _n2f(e, b)
    if float(length) < 0.001:
        return _n2f(q, b)
    t = f32(f32(f32(f32(q[0]) - f32(b[0])) * f32(f32(e[0]) - f32(b[0]))) + f32(f32(f32(q[1]) - f32(b[1])) * f32(f32(e[1]) - f32(b[1]))))
    t = f32(f32(t / length) / length)
    if float(t) > 1.0:
        return f32(1.0)
    if float(t) < 0.0:
        return f32(0.0)
    return t


def py_pair(cfg, seq, p, est_wTo, est_oTw, L, lw):
    """findClosestPlane's body for one landmark: ("skip", branch) or ("cand", error)"""
    if lw is None:
        return "deleted", None
    if p["ind"] == 0 and L["frame_plane_indice"] == 0:
        return "ground", -1.0
    if (p["ind"] == 0 and L["frame_plane_indice"] >= 1) or (p["ind"] >= 1 and L["frame_plane_indice"] == 0):
        return "kind", None
    if L["n_bound2d"] < 2 or L["n_world3d"] < 2:
        return "short", None
    if seq - int(L["frame_seq_id"]) > cfg.assoc_near_frames:
        return "window", None
    local = [float(x) for x in p["local"]]
    cw = _plane_T(est_oTw, local)
    d = _dot3(_normal(cw), _normal(list(lw)))
    angle = (math.acos(d) if -1.0 <= d <= 1.0 else math.nan) * 180.0 / PI   # acos of |d| > 1 is NaN, as in C
    if angle > cfg.edge_asso_angle:
        return "angle", None
    thr2d, cover = cfg.edge_asso_2ddist, cfg.edge_asso_proj
    if angle < 25.0:
        cover = cfg.edge_asso_proj / 3
        thr2d = cfg.edge_asso_2ddist * 1.5
        if angle <= 10.0:
            cover = cfg.edge_asso_proj / 2
    old_local = _plane_T(est_wTo, list(lw))
    n_c = _normal(local)
    d_c = -local[3] / _norm3(local)
    d_o = -old_local[3] / _norm3(old_local)
    n_o = _normal(old_local)
    q = [d_o * n_o[k] for k in range(3)]
    q0 = [d_c * n_c[k] for k in range(3)]
    plane_dist = abs(_dot3(n_c, [q[k] - q0[k] for k in range(3)]))
    if plane_dist > cfg.edge_asso_planedist:
        return "planedist", None
    if plane_dist < 1.5:
        cover = cover / 2
    c2, o2 = p["v2"].reshape(2, 2), L["bound2d"]
    poly = f32(0)
    for i in range(2):
        poly = f32(poly + _min2f(_n2f(c2[i], o2[0]), _n2f(c2[i], o2[1])))
    poly = f32(poly / f32(2))
    cross = f32(0)
    for i in range(2):
        cross = f32(cross + _min2f(_n2f(c2[0], o2[i]), _n2f(c2[1], o2[i])))
    cross = f32(cross / f32(2))
    if float(poly) > thr2d or float(cross) > thr2d:
        return "2d", None
    c3, o3 = p["v3"].reshape(2, 3), L["world3d"]
    on = f32(abs(f32(proj_to_lineseg(c3[0], c3[1], o3[0]) - proj_to_lineseg(c3[0], c3[1], o3[1]))))
    no = f32(abs(f32(proj_to_lineseg(o3[0], o3[1], c3[0]) - proj_to_lineseg(o3[0], o3[1], c3[1]))))
    if float(on) < cover or float(no) < cover:
        return "cover", None
    total = angle / cfg.edge_asso_angle * 3 + float(f32(f32(1) - on)) + float(f32(f32(1) - no))
    total += float(cross if poly < cross else poly) / thr2d + plane_dist / 4
    return "cand", total


def py_associate(cfg, seq, est_wTo, est_oTw, P, lm, lw, alive):
    """findClosestPlane per plane and the one-to-one rule (Mapping.cpp:423-460)"""
    n, L = len(P), len(lm)
    ids, errs = [], []
    for i in range(n):
        p = P[i]
        best, best_err, num = -1, -1.0, 0
        if not (p["ind"] != 0 and (p["n2"] < 2 or p["n3"] < 2)):
            for c in range(L):
                kind, e = py_pair(cfg, seq, p, est_wTo, est_oTw, lm[c], lw[c] if alive[c] else None)
                if kind == "ground":
                    num += 1
                    best = c
                    break
                if kind != "cand":
                    continue
                num += 1
                if num == 1 or e < best_err:
                    best, best_err = c, e
        ids.append(best)
        errs.append(best_err)
    assoc, aerr, status = [0] * n, [0.0] * n, [0] * n
    num_new = 0
    for i in range(n):
        if ids[i] > -1:
            conflict = False
            for j in range(i):
                if assoc[j] == ids[i]:
                    raw = float(_n2f(P[j]["v2"][0:2], P[j]["v2"][2:4]))
                    new = float(_n2f(P[i]["v2"][0:2], P[i]["v2"][2:4]))
                    if new > raw:
                        assoc[j] = L + num_new; num_new += 1; aerr[j] = -1.0; status[j] = 3
                        assoc[i] = ids[i]; aerr[i] = errs[i]; status[i] = 0
                    else:
                        assoc[i] = L + num_new; num_new += 1; aerr[i] = 0.0; status[i] = 3
                    conflict = True
                    break
            if not conflict:
                assoc[i], aerr[i], status[i] = ids[i], errs[i], 0
        else:
            assoc[i] = L + num_new
            num_new += 1
            status[i] = 1 if (P[i]["ind"] != 0 and (P[i]["n2"] < 2 or P[i]["n3"] < 2)) else 2
    return dict(id=np.array(ids), err=np.array(errs), assoc=np.array(assoc), aerr=np.array(aerr), status=np.array(status), n_new=num_new)


def py_sigma(d, mul):
    d = 3 if d < 3 else d
    d = 8 if d > 8 else d
    return (d - 1) * mul + 5


# ---- seeded synthetic corridors ----------------------------------------------------------------------------------------
K = np.array([[537.96, 0, 320.0], [0, 537.96, 240.0], [0, 0, 1]])
INVK = np.linalg.inv(K).astype(np.float32)


def _look(pos, yaw):
    """camera-to-world: camera z forward along yaw in the xy plane, camera y down"""
    f = np.array([math.cos(yaw), math.sin(yaw), 0.0])
    down = np.array([0.0, 0.0, -1.0])
    right = np.cross(down, f)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, f, pos
    return T


def corridor(seed, n_frames, width=2.0, height=1.0, seg=3.0):
    """a camera walking down a corridor of wall pieces `seg` long on both sides, one frame per 0.25 m, with a little
    heading noise; per frame the pieces in front of it within 6 m as good planes (plane_indice 1..), plus the ground"""
    rng = np.random.default_rng(seed)
    frames = []
    for t in range(n_frames):
        x = 0.25 * t
        yaw = 0.05 * math.sin(0.3 * t) + rng.normal(0, 0.01)
        T = _look(np.array([x, 0.1 * math.sin(0.1 * t), height]), yaw)
        Tinv = np.linalg.inv(T)
        planes, dist, ind, bound, world, clean = [], [], [], [], [], []
        g = _plane_T(T.tolist(), [0.0, 0.0, -1.0, 0.0])
        planes.append(g); dist.append(0.0); ind.append(0)
        bound.append([[0, 479], [639, 479], [639, 300], [0, 300]]); world.append([])
        for side in (-1, 1):
            k0 = int(math.floor(x / seg))
            for k in range(k0, k0 + 3):
                a, b = np.array([k * seg, side * width, 0.0]), np.array([(k + 1) * seg, side * width, 0.0])
                ca, cb = Tinv[:3, :3] @ a + Tinv[:3, 3], Tinv[:3, :3] @ b + Tinv[:3, 3]
                if ca[2] < 0.3 and cb[2] < 0.3:
                    continue
                ca = ca if ca[2] >= 0.3 else ca + (cb - ca) * (0.3 - ca[2]) / (cb[2] - ca[2])
                cb = cb if cb[2] >= 0.3 else cb + (ca - cb) * (0.3 - cb[2]) / (ca[2] - cb[2])
                if min(ca[2], cb[2]) > 6:
                    continue
                pa, pb = K @ ca, K @ cb
                pa, pb = pa[:2] / pa[2], pb[:2] / pb[2]
                wa, wb = T[:3, :3] @ ca + T[:3, 3], T[:3, :3] @ cb + T[:3, 3]
                n_w = np.array([0.0, -side, 0.0])
                pl_w = [n_w[0], n_w[1], n_w[2], -float(n_w @ wa)]
                planes.append(_plane_T(T.tolist(), pl_w))
                dist.append(float(0.5 * (ca[2] + cb[2]) + rng.normal(0, 0.05)))
                ind.append(len(ind))
                clean.append([pa[0], pa[1], pb[0], pb[1]])
                noise = rng.normal(0, 0.5, 4)
                bound.append([[pa[0] + noise[0], pa[1] + noise[1]], [pb[0] + noise[2], pb[1] + noise[3]], [pb[0], 0], [pa[0], 0]])
                world.append([list(wa + rng.normal(0, 0.02, 3)), list(wb + rng.normal(0, 0.02, 3)),
                              list(wb + [0, 0, 2]), list(wa + [0, 0, 2])])
        ps = np.array(planes, np.float32) + rng.normal(0, 2e-3, (len(planes), 4)).astype(np.float32)
        n_segs = len(ind) - 1
        segs = np.array(clean, np.float32).reshape(-1, 4)   # the walls' ground lines, as the refresh re-pops them
        frames.append(dict(T=T, planes_sensor=ps, dist=np.array(dist, np.float32), plane_indice=np.array(ind, np.int32),
                           bound=bound, world=world, segs=segs, n_segs=n_segs))
    return frames


def pose_T(p7):
    wTo, oTw = np.zeros(16), np.zeros(16)
    oracle_lib().orc_map_pose_T(_p(np.asarray(p7, float)), _p(wTo), _p(oTw))
    return wTo.reshape(4, 4).tolist(), oTw.reshape(4, 4).tolist()


def T_to_pose(T):
    out = np.zeros(7)
    oracle_lib().orc_map_T_to_pose(_p(np.ascontiguousarray(T, float).reshape(16)), _p(out))
    return out


def ominus(a7, b7):
    out = np.zeros(7)
    oracle_lib().orc_map_ominus(_p(np.asarray(a7, float)), _p(np.asarray(b7, float)), _p(out))
    return out


def replay(cfg, frames, check=None):
    """Runs a corridor through the oracle with ground-truth poses as the solver's estimates and each landmark's plane at
    its first-sight initial value; check(seq, P, lm, lw, alive, est, result) sees every frame.  Returns the table."""
    lm = np.zeros(0, LANDMARK)
    lw = np.zeros((0, 4))
    poses = []
    for seq, fr in enumerate(frames):
        P = planes_array(fr)
        gt = T_to_pose(fr["T"])
        n_mapped = len(poses)
        last = poses[-1] if poses else np.zeros(7)
        odom = ominus(gt, last) if poses else gt
        alive = np.ones(len(lm), np.int32)
        r = oracle_associate(cfg, seq, n_mapped, last, odom, P, lm, lw, alive)
        if check:
            check(seq, P, lm, lw, alive, r)
        _, oTw = pose_T(r["est"])
        new_lw = np.zeros((r["n_new"], 4))
        for i in range(len(P)):
            if r["assoc"][i] >= len(lm):
                new_lw[r["assoc"][i] - len(lm)] = _plane_T(oTw, [float(x) for x in P[i]["local"]])
        lm = oracle_apply(seq, P, r["assoc"], lm, r["n_new"], np.arange(len(lm), len(lm) + r["n_new"]))
        lw = np.concatenate([lw, new_lw])
        poses.append(gt)
    return lm


# ---- main_3d's pose guess restated (main_3d.cpp:366-385, keyed on mapped frames) ----------------------------------------
def py_predict(n_mapped, last7, prev7, init_wTo, pose_from_mat4, ominus, oplus, wTo):
    """the reference's arithmetic through the given pose functions: (odom7, pred7, float32 wTo)"""
    if n_mapped == 0:
        odom = pose_from_mat4(np.asarray(init_wTo, float).reshape(4, 4))
        pred = odom
    else:
        odom = np.array([0, 0, 0, 1, 0, 0, 0], float) if n_mapped == 1 else ominus(last7, prev7)
        pred = oplus(last7, odom)
    return odom, pred, np.asarray(wTo(pred), np.float64).astype(np.float32).reshape(4, 4)


# ---- path B: main_3d's mapping step chained on the host -----------------------------------------------------------------
def sqrtinf_diag(sigmas):
    """isam::Covariance(diag(sigma^2)) as the C-ABI's packed upper sqrt-information: sqrt(1 / sigma^2) on the diagonal"""
    n = len(sigmas)
    U = np.zeros((n, n))
    for i, s in enumerate(sigmas):
        U[i, i] = math.sqrt(1.0 / (s * s))
    return np.array([U[r, c] for r in range(n) for c in range(r, n)])


def session_frame(out, f):
    """frame f of a pop-up session's downloaded outputs as the map's array form"""
    g0, g1 = out["good_ptr"][f], out["good_ptr"][f + 1]
    rows_in = out["good_rows"][g0:g1]
    o0, o1 = out["open_ptr"][f], out["open_ptr"][f + 1]
    rows = o0 + f + rows_in
    return dict(planes_sensor=out["planes_sensor"][rows], dist=out["dist"][rows], plane_indice=rows_in,
                bound=[out["bound2d"][out["bound_ptr"][r]:out["bound_ptr"][r + 1]] for r in rows],
                world=[out["world3d"][out["world_ptr"][r]:out["world_ptr"][r + 1]] for r in rows],
                segs=out["open_segs"][o0:o1])


class PathB:
    """Mapper_mono::processFrame + update_plane_measurement + reproj_to_newplane chained on the host over the C-ABI:
    host-oracle association, capi add calls in the reference's order, the same solve calls, pus_refresh_bind / run over
    every mapped frame and pus_project_to_planes.  `times` keeps (association + edits, solve, refresh + projection) per
    frame, host-clocked (every call returns synchronised)."""

    def __init__(self, api, cfg):
        import oracle_api as O
        self.O, self.api, self.cfg = O, api, cfg
        self.lm = np.zeros(0, LANDMARK)
        self.frame_pose, self.segs, self.map_fid, self.map_frame, self.map_row = [], [], [], [], []
        self.pose_sinf = sqrtinf_diag(list(cfg.pose_sigmas))
        self.plane_sinf = sqrtinf_diag(list(cfg.plane_sigmas))
        self.times = []

    def predict(self):
        nf = len(self.frame_pose)
        last = self.api.get_pose(self.frame_pose[-1]) if nf else None
        prev = self.api.get_pose(self.frame_pose[-2]) if nf > 1 else None
        return oracle_predict(nf, last, prev, list(self.cfg.init_wTo))

    def frame(self, seq, fr, odom7):
        import time
        api, cfg = self.api, self.cfg
        if len(fr["dist"]) == 0:
            return None
        t0 = time.perf_counter()
        P = planes_array(fr)
        nf, L = len(self.frame_pose), len(self.lm)
        last = api.get_pose(self.frame_pose[-1]) if nf else np.zeros(7)
        lw = np.array([api.get_plane(int(n)) for n in self.lm["node"]]).reshape(-1, 4)
        r = oracle_associate(cfg, seq, nf, last, odom7, P, self.lm, lw, np.ones(L, np.int32))
        pose = api.add_pose(r["est"] if nf else None)
        m6 = self.O.pose_vector(odom7)
        if nf == 0:
            api.add_pose_prior(pose, m6, self.pose_sinf)
        else:
            api.add_odometry(self.frame_pose[-1], pose, m6, self.pose_sinf)
        _, oTw = pose_T(r["est"])
        nodes = [int(n) for n in self.lm["node"]]
        new_nodes = []
        for k in range(r["n_new"]):
            i = [j for j in range(len(P)) if r["assoc"][j] == L + k][0]
            new_nodes.append(api.add_plane(_plane_T(oTw, [float(x) for x in P[i]["local"]])))
        nodes += new_nodes
        fids = []
        for i in range(len(P)):
            node = nodes[r["assoc"][i]]
            if r["assoc"][i] >= L and P[i]["ind"] == 0:
                api.add_plane_prior(node, [0.0, 0.0, -1.0, 0.0], self.plane_sinf)
            s = py_sigma(float(P[i]["dist"]), cfg.plane_sigma_dist_mul)
            fids.append(api.add_pose_plane(pose, node, [float(x) for x in P[i]["local"]], sqrtinf_diag([s, s, s])))
        self.frame_pose.append(pose)
        self.segs.append(np.asarray(fr["segs"], np.float32).reshape(-1, 4))
        self.map_fid += fids
        self.map_frame += [nf] * len(P)
        self.map_row += [int(x) for x in P["ind"]]
        t1 = time.perf_counter()
        if seq % 5 == 0:
            api.batch_optimize()
        else:
            api.update()
        t2 = time.perf_counter()
        seg_ptr = np.concatenate([[0], np.cumsum([len(s) for s in self.segs])])
        api.refresh_bind(self.frame_pose, seg_ptr, np.concatenate(self.segs), np.asarray(cfg.invK, np.float32).reshape(3, 3),
                         self.map_fid, self.map_frame, self.map_row)
        api.refresh_run()
        self.lm = oracle_apply(seq, P, r["assoc"], self.lm, r["n_new"], new_nodes)
        ids, pts, where = [], [], []
        for c in range(len(self.lm)):
            for k in range(int(self.lm[c]["n_world3d"])):
                ids.append(int(self.lm[c]["node"]))
                pts.append(self.lm[c]["world3d"][k])
                where.append((c, k))
        if ids:
            new = api.project_to_planes(ids, np.array(pts, np.float32))
            for (c, k), v in zip(where, new):
                self.lm[c]["world3d"][k] = v
        self.times.append((t1 - t0, t2 - t1, time.perf_counter() - t2))
        return dict(landmark=r["assoc"], status=r["status"], factor=np.array(fids), new_nodes=np.array(new_nodes), pose_node=pose)


# ---- one rendered room seen from a moving camera ------------------------------------------------------------------------
def camera(pos, yaw, pitch):
    """camera-to-world: x right, y down, z forward along yaw, pitched down by `pitch`"""
    f = np.array([math.cos(yaw) * math.cos(pitch), math.sin(yaw) * math.cos(pitch), -math.sin(pitch)])
    right = np.array([math.sin(yaw), -math.cos(yaw), 0.0])
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, np.cross(f, right), f, pos
    return T


def moving_room(seed, n, width=640, height=480, K=None):
    """a box room 8 x 6 m with a colour per wall, seen by a camera 1 m up, pitched 12 deg down, walking and turning slowly;
    label 255 where the pixel's ray meets the floor inside the room (popup_frames_native.room's colouring)"""
    rng = np.random.default_rng(seed)
    x0, x1, y0, y1 = 0.0, 8.0, 0.0, 6.0
    iK = np.linalg.inv(K)
    xs, ys = np.meshgrid(np.arange(width, dtype=np.float64), np.arange(height, dtype=np.float64))
    rays = np.stack([xs, ys, np.ones_like(xs)], -1) @ iK.T
    walls = rng.integers(60, 230, (4, 3))
    floor = rng.integers(20, 120, 3)
    imgs, labs, Ts = [], [], []
    for t in range(n):
        T = camera(np.array([2.0 + 0.08 * t, 2.5 + 0.3 * math.sin(0.2 * t), 1.0]), 0.35 * math.sin(0.15 * t), math.radians(12))
        d = rays @ T[:3, :3].T
        c = T[:3, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            tf = np.where(d[..., 2] < 0, -c[2] / d[..., 2], np.inf)
            px, py = c[0] + tf * d[..., 0], c[1] + tf * d[..., 1]
            ground = (d[..., 2] < 0) & (px >= x0) & (px <= x1) & (py >= y0) & (py <= y1)
            tx = np.where(d[..., 0] > 0, (x1 - c[0]) / d[..., 0], (x0 - c[0]) / d[..., 0])
            ty = np.where(d[..., 1] > 0, (y1 - c[1]) / d[..., 1], (y0 - c[1]) / d[..., 1])
        wall = np.where(tx < ty, np.where(d[..., 0] > 0, 1, 3), np.where(d[..., 1] > 0, 2, 0))
        img = walls[wall].astype(np.int16)
        img[ground] = floor
        img += rng.integers(-8, 9, img.shape).astype(np.int16)
        imgs.append(np.clip(img, 0, 255).astype(np.uint8))
        labs.append(np.where(ground, 255, 0).astype(np.uint8))
        Ts.append(T)
    return np.array(imgs), np.array(labs), np.array(Ts)
