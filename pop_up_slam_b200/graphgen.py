"""Synthetic pose-plane factor graphs for BASELINE.json's configs (SURVEY.md 8d).

Every graph follows the factor / vertex mix that pop_planar_slam's Mapper_mono::processFrame
builds (pop_planar_slam/src/Mapping.cpp:464-530): one Pose3d prior on the first pose, an
odometry chain, one ground plane (observed by every frame, with a Plane3d prior, :500-504) and
wall planes observed by the frames near them.  sigma_mode "reference" uses the sigmas of
Mapping.cpp:64-67,507-512 / params/plane_3d_tum_far.yaml; "consistent" uses the injected noise
so chi2 ~ dof and the LM iterations do real work (SURVEY.md 8d).

Host-side product code (bench.py / tests use it); no oracle dependency.
"""
from dataclasses import dataclass, field
import numpy as np

from . import geometry as geo

# camera-to-body base rotation: camera z forward along world +x, x right, y down.
# Euler (yaw, pitch, roll) = (-90deg, 0, -90deg): far from the pitch = +-90deg singularity of the
# reference's Euler-difference residuals (slam3d.h:174-191).
R_BASE = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])


@dataclass
class SyntheticGraph:
    name: str
    seed: int
    poses_truth: np.ndarray
    planes_truth: np.ndarray
    poses_init: np.ndarray
    planes_init: np.ndarray
    prior_pose: int
    prior_meas: np.ndarray
    prior_sqrtinf: np.ndarray
    odo_i: np.ndarray
    odo_j: np.ndarray
    odo_meas: np.ndarray
    odo_sqrtinf: np.ndarray
    pp_pose: np.ndarray
    pp_plane: np.ndarray
    pp_meas: np.ndarray
    pp_sqrtinf: np.ndarray
    ground_plane: int
    ground_meas: np.ndarray
    ground_sqrtinf: np.ndarray
    robust_kind: int = 0
    robust_b: float = 1.0
    properties: dict = field(default_factory=dict)

    @property
    def n_poses(self):
        return len(self.poses_truth)

    @property
    def n_planes(self):
        return len(self.planes_truth)

    @property
    def n_pose_plane(self):
        return len(self.pp_pose)

    @property
    def n_odometry(self):
        return len(self.odo_i)

    def dims(self):
        return dict(N=self.n_poses, M=self.n_planes, E_pl=self.n_pose_plane, E_od=self.n_odometry + 1,
                    state_dim=6 * self.n_poses + 3 * self.n_planes,
                    rows=3 * self.n_pose_plane + 6 * (self.n_odometry + 1) + (3 if self.ground_plane >= 0 else 0))


def diag_ut(d):
    """Packed upper-triangular (row-major) of diag(d)."""
    d = np.asarray(d, dtype=np.float64)
    n = len(d)
    out = []
    for r in range(n):
        for c in range(r, n):
            out.append(d[r] if r == c else 0.0)
    return np.array(out)


# PPS/src/Mapping.cpp:31-43 applied to the defaults of Properties.h:86-109
PPS_PROPERTIES = dict(method=1, epsilon2=1e-3, epsilon_abs=1e-4, epsilon_rel=1e-6, max_iterations=500,
                      lm_lambda0=1e-6, lm_lambda_factor=10.0, mod_update=1, mod_batch=1, mod_solve=1)


def _batch_quat_mul(a, b):
    aw, ax, ay, az = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    bw, bx, by, bz = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    return np.stack([
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by + ay * bw + az * bx - ax * bz,
        aw * bz + az * bw + ax * by - ay * bx], axis=1)


def _batch_plane_exmap(p, d):
    th = np.linalg.norm(d, axis=1)
    s = np.where(th < 1e-12, 0.5, np.sin(0.5 * th) / np.maximum(th, 1e-300))
    dq = np.concatenate([np.cos(0.5 * th)[:, None], s[:, None] * d], axis=1)
    qp = np.stack([p[:, 3], p[:, 0], p[:, 1], p[:, 2]], axis=1)
    q = _batch_quat_mul(dq, qp)
    out = np.stack([q[:, 1], q[:, 2], q[:, 3], q[:, 0]], axis=1)
    return out / np.linalg.norm(out, axis=1, keepdims=True)


def _finish(name, seed, T_truth, planes, obs_pose, obs_plane, plane_dist, rng, sigma_mode, plane_noise, odo_noise,
            outlier_frac, outlier_mag, robust_kind, robust_b, max_iterations, init_mode="dead_reckoning"):
    n = len(T_truth)
    T_truth = np.asarray(T_truth)
    # ---- pose-plane measurements: normalize(wTo^T pi) (+) noise  (isam_plane3d.h:180-182) ----
    local = np.einsum("eji,ej->ei", T_truth[obs_pose], planes[obs_plane])
    local /= np.linalg.norm(local, axis=1, keepdims=True)
    E = len(obs_pose)
    meas = _batch_plane_exmap(local, rng.normal(0.0, plane_noise, size=(E, 3)))
    if outlier_frac > 0:
        # mis-associated walls: the measurement is rotated by a large but bounded tangent step (20..100 sigma),
        # kept away from the +-pi wrap of the log map where the reference's central differences break down
        out = rng.random(E) < outlier_frac
        dirs = rng.normal(size=(E, 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        mag = rng.uniform(outlier_mag[0], outlier_mag[1], size=(E, 1))
        meas[out] = _batch_plane_exmap(meas, dirs * mag)[out]
    if sigma_mode == "reference":
        dist = np.clip(plane_dist, 3.0, 8.0)
        sig = (dist - 1.0) * 2.0 + 5.0  # Mapping.cpp:507-512, plane_sigma_dist_mul = 2
        pose_sig = np.full(6, 2.0)      # plane_3d_tum_far.yaml:16-21
    else:
        sig = np.full(E, plane_noise)
        pose_sig = np.array([odo_noise[0]] * 3 + [odo_noise[1]] * 3)
    pp_sqrtinf = np.zeros((E, 6))
    pp_sqrtinf[:, 0] = pp_sqrtinf[:, 3] = pp_sqrtinf[:, 5] = 1.0 / sig
    # ---- odometry chain ----
    odo_meas = np.zeros((n - 1, 6))
    for i in range(n - 1):
        rel = geo.inv_T(T_truth[i]) @ T_truth[i + 1]
        odo_meas[i] = geo.T_to_xyzypr(rel)
    odo_meas[:, :3] += rng.normal(0.0, odo_noise[0], size=(n - 1, 3))
    odo_meas[:, 3:] += rng.normal(0.0, odo_noise[1], size=(n - 1, 3))
    pose_ut = diag_ut(1.0 / pose_sig)
    odo_sqrtinf = np.tile(pose_ut, (n - 1, 1))
    # ---- initial estimates: dead-reckoned odometry (Pose3d_Pose3d_Factor::initialize, slam3d.h:133-137)
    T_init = [T_truth[0].copy()]
    for i in range(n - 1):
        if init_mode == "truth":
            T_init.append(T_truth[i + 1].copy())
        elif isinstance(init_mode, tuple):
            # ("perturbed", sigma_t, sigma_r): truth (+) independent noise per pose -- the state of a map that was
            # optimised a few frames ago (the reference re-solves every 5th frame, Mapping.cpp:550-554)
            d = np.concatenate([rng.normal(0, init_mode[1], 3), rng.normal(0, init_mode[2], 3)])
            Tn = T_truth[i + 1].copy()
            Tn[:3, 3] += d[:3]
            Tn[:3, :3] = Tn[:3, :3] @ geo.quat_to_R(geo.delta3_to_quat(d[3:]))
            T_init.append(Tn)
        else:
            T_init.append(T_init[-1] @ geo.xyzypr_to_T(odo_meas[i]))
    poses_init = np.array([geo.T_to_pose7(T) for T in T_init])
    poses_truth = np.array([geo.T_to_pose7(T) for T in T_truth])
    # plane init from the first observation: meas.transform_from(pose.oTw())  (isam_plane3d.h:252-264)
    m = len(planes)
    planes_init = np.array(planes, dtype=np.float64).copy()
    seen = np.zeros(m, dtype=bool)
    for e in range(E):
        k = obs_plane[e]
        if not seen[k]:
            seen[k] = True
            planes_init[k] = geo.plane_to_global(T_init[obs_pose[e]], meas[e])
    props = dict(PPS_PROPERTIES)
    props["max_iterations"] = max_iterations
    return SyntheticGraph(
        name=name, seed=seed, poses_truth=poses_truth, planes_truth=np.asarray(planes, dtype=np.float64),
        poses_init=poses_init, planes_init=planes_init,
        prior_pose=0, prior_meas=geo.T_to_xyzypr(T_truth[0]), prior_sqrtinf=pose_ut,
        odo_i=np.arange(0, n - 1, dtype=np.int32), odo_j=np.arange(1, n, dtype=np.int32),
        odo_meas=odo_meas, odo_sqrtinf=odo_sqrtinf,
        pp_pose=np.asarray(obs_pose, dtype=np.int32), pp_plane=np.asarray(obs_plane, dtype=np.int32),
        pp_meas=meas, pp_sqrtinf=pp_sqrtinf,
        ground_plane=0, ground_meas=np.array([0.0, 0.0, -1.0, 0.0]), ground_sqrtinf=diag_ut([1 / 0.05] * 3),
        robust_kind=robust_kind, robust_b=robust_b, properties=props)


def make_room(seed=0, n_poses=10, n_planes=20, obs_per_pose=10, sigma_mode="reference", plane_noise=0.01,
              odo_noise=(0.01, 0.005), max_iterations=500):
    """BASELINE config 1 "tiny room": poses on a 2 m circle at 1 m height facing inward, ground + vertical
    walls (cos phi, sin phi, 0, -rho), each pose observes `obs_per_pose` random planes."""
    rng = np.random.default_rng(seed)
    T = []
    for i in range(n_poses):
        ang = 2 * np.pi * i / n_poses
        pos = np.array([2 * np.cos(ang), 2 * np.sin(ang), 1.0])
        heading = ang + np.pi  # facing the centre
        R = geo.euler_to_R(heading, 0.02 * np.sin(3 * ang), 0.02 * np.cos(2 * ang)) @ R_BASE
        Ti = np.eye(4)
        Ti[:3, :3] = R
        Ti[:3, 3] = pos
        T.append(Ti)
    planes = [np.array([0.0, 0.0, -1.0, 0.0])]
    anchors = [np.zeros(3)]
    for _ in range(n_planes - 1):
        phi = rng.uniform(0, 2 * np.pi)
        rho = rng.uniform(3.0, 6.0)
        planes.append(geo.plane_normalize([np.cos(phi), np.sin(phi), 0.0, -rho]))
        anchors.append(np.array([rho * np.cos(phi), rho * np.sin(phi), 0.0]))
    planes = np.array(planes)
    obs_pose, obs_plane, dist = [], [], []
    for i in range(n_poses):
        ks = np.sort(rng.choice(n_planes, size=obs_per_pose, replace=False))
        for k in ks:
            obs_pose.append(i)
            obs_plane.append(int(k))
            dist.append(T[i][2, 3] if k == 0 else np.linalg.norm(anchors[k][:2] - T[i][:2, 3]))
    return _finish("room", seed, T, planes, np.array(obs_pose), np.array(obs_plane), np.array(dist), rng, sigma_mode,
                   plane_noise, odo_noise, 0.0, (0.2, 1.0), 0, 1.0, max_iterations)


def _serpentine(s, aisle, radius):
    """Position / heading at arclength s of a serpentine corridor: straight aisles of length `aisle`
    along +-x joined by semicircular U-turns of radius `radius` (aisle spacing 2*radius)."""
    per = aisle + np.pi * radius
    j = int(np.floor(s / per))
    u = s - j * per
    d = 1.0 if j % 2 == 0 else -1.0
    yj = j * 2.0 * radius
    if u <= aisle:
        return np.array([d * (-aisle / 2 + u), yj]), (0.0 if d > 0 else np.pi)
    phi = (u - aisle) / radius
    c = np.array([d * aisle / 2, yj + radius])
    if d > 0:
        return c + radius * np.array([np.sin(phi), -np.cos(phi)]), phi
    return c + radius * np.array([-np.sin(phi), -np.cos(phi)]), np.pi - phi


def make_corridor(seed=0, n_poses=5000, n_planes=500, obs_per_pose=10, step=0.1, sigma_mode="consistent",
                  plane_noise=0.01, odo_noise=(0.005, 0.0005), outlier_frac=0.0, outlier_mag=(0.2, 1.0),
                  robust_kind=0, robust_b=1.0, max_iterations=20, name="corridor", init_mode="dead_reckoning",
                  aisle=40.0, radius=2.5):
    """Corridor family (BASELINE configs 2, 3, 5): a camera walking a serpentine corridor (so the map stays
    within a few tens of metres of the origin -- the reference's unit-4-vector plane chart and its
    eps=1e-4 numerical differences degrade when |d|/|n| is large), the ground plane seen by every
    pose, and wall / door-frame planes anchored every L/(M-1) metres of path on alternating sides; each pose
    observes the ground plus the obs_per_pose-1 nearest anchors (by arclength)."""
    rng = np.random.default_rng(seed)
    T, planes, obs_pose, obs_plane, dist = _corridor_geometry(rng, n_poses, n_planes, obs_per_pose, step, aisle, radius)
    return _finish(name, seed, T, planes, obs_pose, obs_plane, dist, rng, sigma_mode, plane_noise, odo_noise,
                   outlier_frac, outlier_mag, robust_kind, robust_b, max_iterations, init_mode)


def _corridor_geometry(rng, n_poses, n_planes, obs_per_pose, step, aisle, radius):
    """truth poses, planes and observations of make_corridor"""
    L = n_poses * step
    n_aisles = int(np.floor(L / (aisle + np.pi * radius))) + 1
    centre = np.array([0.0, (n_aisles - 1) * radius])

    def frame_at(s):
        pxy, heading = _serpentine(s, aisle, radius)
        return pxy - centre, heading

    T = np.zeros((n_poses, 4, 4))
    for i in range(n_poses):
        s = i * step
        pxy, heading = frame_at(s)
        lat = np.array([-np.sin(heading), np.cos(heading)])
        pxy = pxy + 0.3 * np.sin(2 * np.pi * s / 25.0) * lat
        hd = heading + 0.1 * np.sin(2 * np.pi * s / 30.0)
        R = geo.euler_to_R(hd, 0.03 * np.sin(2 * np.pi * s / 17.0), 0.03 * np.cos(2 * np.pi * s / 23.0)) @ R_BASE
        T[i, :3, :3] = R
        T[i, :3, 3] = [pxy[0], pxy[1], 1.0 + 0.05 * np.sin(2 * np.pi * s / 40.0)]
        T[i, 3, 3] = 1.0
    m_walls = n_planes - 1
    spacing = L / m_walls
    planes = np.zeros((n_planes, 4))
    planes[0] = [0.0, 0.0, -1.0, 0.0]
    anchors = np.zeros((n_planes, 3))
    for k in range(1, n_planes):
        pxy, heading = frame_at((k - 0.5) * spacing)
        side = 1.0 if k % 2 == 0 else -1.0
        if k % 4 == 3:  # door frame / cross plane: normal along the path tangent
            psi = heading + rng.uniform(-0.4, 0.4)
            nrm = geo.euler_to_R(psi, rng.uniform(-0.1, 0.1), 0.0) @ np.array([1.0, 0.0, 0.0])
            a = np.array([pxy[0], pxy[1], 0.0])
        else:           # side wall: normal along the path lateral direction, pointing away from the path
            psi = heading + rng.uniform(-0.5, 0.5)
            nrm = geo.euler_to_R(psi, 0.0, rng.uniform(-0.1, 0.1)) @ np.array([0.0, side, 0.0])
            off = side * rng.uniform(1.5, 3.0)
            a = np.array([pxy[0] - np.sin(heading) * off, pxy[1] + np.cos(heading) * off, 0.0])
        planes[k] = geo.plane_normalize([nrm[0], nrm[1], nrm[2], -float(nrm @ a)])
        anchors[k] = a
    w = min(obs_per_pose - 1, m_walls)
    sarr = np.arange(n_poses) * step
    start = np.clip(np.round(sarr / spacing - w / 2.0).astype(np.int64), 0, m_walls - w)
    obs_pose = np.repeat(np.arange(n_poses), w + 1)
    obs_plane = np.zeros((n_poses, w + 1), dtype=np.int64)
    obs_plane[:, 1:] = 1 + start[:, None] + np.arange(w)[None, :]
    obs_plane = obs_plane.reshape(-1)
    cam = T[obs_pose, :3, 3]
    dist = np.where(obs_plane == 0, cam[:, 2], np.linalg.norm(anchors[obs_plane][:, :2] - cam[:, :2], axis=1))
    return T, planes, obs_pose, obs_plane, dist


def make_revisit(seed=0, n_poses=2000, n_planes=100, obs_per_pose=10, step=0.1, sigma_mode="consistent", plane_noise=0.01,
                 odo_noise=(0.003, 0.0002), outlier_frac=0.0, outlier_mag=(0.05, 0.3), robust_kind=0, robust_b=1.0,
                 max_iterations=20, name="revisit", init_mode="dead_reckoning", aisle=40.0, radius=2.5, offset=0.2):
    """A corridor driven twice: the first n_poses - n_poses // 2 poses walk the make_corridor path with n_planes planes, the
    rest walk it again from the start, `offset` metres to the side.  The odometry chain continues across the turn-back, and
    the second pass re-observes the first pass's planes with fresh noise -- the graph a loop closure that merges a revisit's
    planes into the first visit's (Mapper_mono::loopclose_merge, Mapping.cpp:637-704) leaves behind: pose a and pose
    a + n_poses // 2 share planes for every a."""
    rng = np.random.default_rng(seed)
    n1 = n_poses - n_poses // 2
    T1, planes, op1, ol1, dist1 = _corridor_geometry(rng, n1, n_planes, obs_per_pose, step, aisle, radius)
    n2 = n_poses - n1
    T2 = T1[:n2].copy()
    T2[:, :3, 3] += offset * T2[:, :3, 0]   # (R_BASE: the camera x axis points across the path)
    keep = op1 < n2
    T = np.concatenate([T1, T2])
    obs_pose = np.concatenate([op1, op1[keep] + n1])
    obs_plane = np.concatenate([ol1, ol1[keep]])
    dist = np.concatenate([dist1, dist1[keep]])
    return _finish(name, seed, T, planes, obs_pose, obs_plane, dist, rng, sigma_mode, plane_noise, odo_noise,
                   outlier_frac, outlier_mag, robust_kind, robust_b, max_iterations, init_mode)


def make_dense(seed=0, n_poses=48, walls=40, advance=20, dense_blocks=None, sparse_walls=6, sparse_advance=3,
               sigma_mode="consistent", plane_noise=0.01, odo_noise=(0.01, 0.005), max_iterations=10, name="dense"):
    """Dense plane observations, as front ends give them that extract 20-40 planes per RGB-D frame, that add a new landmark
    for every observation (no data association) or that take key-frames at a high rate while the camera turns on the spot.
    Poses on the 2 m circle of make_room; each observes the ground plane plus `walls` consecutive vertical walls of a running
    sequence that advances by `advance` walls per pose, so every wall is seen from about walls / advance poses.  With
    `dense_blocks` (16-pose block numbers) only those blocks observe that densely; the other poses see `sparse_walls` walls
    advancing by `sparse_advance`.
    A dense 16-pose block observes about 15 advance + walls + 1 distinct planes in about 16 (walls + 1) / 32 + 16 (tile, pose)
    runs: walls=40, advance=20 passes 256 distinct planes per block (with about 37 runs); walls=110, advance=6 passes 64 runs
    (with about 200 distinct planes)."""
    rng = np.random.default_rng(seed)
    T = []
    for i in range(n_poses):
        ang = 2 * np.pi * i / n_poses
        R = geo.euler_to_R(ang + np.pi, 0.02 * np.sin(3 * ang), 0.02 * np.cos(2 * ang)) @ R_BASE
        Ti = np.eye(4)
        Ti[:3, :3] = R
        Ti[:3, 3] = [2 * np.cos(ang), 2 * np.sin(ang), 1.0]
        T.append(Ti)
    dense = [dense_blocks is None or (i // 16) in dense_blocks for i in range(n_poses)]
    start, s = [], 0
    for i in range(n_poses):
        start.append(s)
        s += advance if dense[i] else sparse_advance
    n_walls = max(start[i] + (walls if dense[i] else sparse_walls) for i in range(n_poses))
    planes = [np.array([0.0, 0.0, -1.0, 0.0])]
    anchors = [np.zeros(3)]
    for _ in range(n_walls):
        phi = rng.uniform(0, 2 * np.pi)
        rho = rng.uniform(3.0, 6.0)
        planes.append(geo.plane_normalize([np.cos(phi), np.sin(phi), 0.0, -rho]))
        anchors.append(np.array([rho * np.cos(phi), rho * np.sin(phi), 0.0]))
    planes = np.array(planes)
    obs_pose, obs_plane, dist = [], [], []
    for i in range(n_poses):
        for k in [0] + list(range(1 + start[i], 1 + start[i] + (walls if dense[i] else sparse_walls))):
            obs_pose.append(i)
            obs_plane.append(k)
            dist.append(T[i][2, 3] if k == 0 else np.linalg.norm(anchors[k][:2] - T[i][:2, 3]))
    return _finish(name, seed, T, planes, np.array(obs_pose), np.array(obs_plane), np.array(dist), rng, sigma_mode,
                   plane_noise, odo_noise, 0.0, (0.2, 1.0), 0, 1.0, max_iterations)


# dense-plane graphs over each per-block limit of the fused PCG pose phase (DESIGN.md section 6), and a mix
DENSE_CASES = {
    "planes": dict(n_poses=48, walls=40, advance=20),                          # > 256 distinct planes in every block
    "runs": dict(n_poses=48, walls=110, advance=6),                            # > 64 (tile, pose) runs, < 256 planes
    "mixed": dict(n_poses=96, walls=40, advance=20, dense_blocks=(1, 4)),      # two of six blocks over a limit
}


def make_config(config, seed=0, **kw):
    """BASELINE.json configs by number (SURVEY.md 8, table of sizes)."""
    if config == 1:   # 10 poses, 20 planes, 100 edges
        return make_room(seed=seed, **kw)
    if config == 2:   # ~300 poses, ~60 planes, ~2k edges, 20 LM iters
        args = dict(n_poses=300, n_planes=60, obs_per_pose=7, step=10.0 / 300, sigma_mode="consistent",
                    max_iterations=20, name="tum_scale")
        args.update(kw)
        return make_corridor(seed=seed, **args)
    if config == 3:   # 5k poses, 500 planes, 50k + 5k edges, Huber
        args = dict(n_poses=5000, n_planes=500, obs_per_pose=10, step=0.1, sigma_mode="consistent",
                    odo_noise=(0.003, 0.0002), outlier_frac=0.05, outlier_mag=(0.05, 0.3), robust_kind=1,
                    robust_b=1.0, max_iterations=20, name="corridor")
        args.update(kw)
        return make_corridor(seed=seed, **args)
    if config == 5:   # 50k poses, 5k planes, 1M edges, 50 LM iters
        args = dict(n_poses=50000, n_planes=5000, obs_per_pose=20, step=0.02, sigma_mode="consistent",
                    max_iterations=50, name="stress", aisle=100.0, radius=2.0, odo_noise=(0.001, 0.0001))
        args.update(kw)
        return make_corridor(seed=seed, **args)
    raise ValueError("config must be 1, 2, 3 or 5 (4 = 64 x config 2)")


# ------------------------------------------------------------------------------------------------
# builders: push a SyntheticGraph through a GraphAPI (pus_* or orc_*)
# ------------------------------------------------------------------------------------------------
def build_interleaved(api, g):
    """Insertion order of Mapper_mono::processFrame (Mapping.cpp:464-530): pose node, prior | odometry,
    new plane nodes, then per observation [ground prior] + pose-plane factor.  Nodes are left
    uninitialised so the factors' initialize() paths run."""
    n, m = g.n_poses, g.n_planes
    pose_ids = np.full(n, -1, dtype=np.int32)
    plane_ids = np.full(m, -1, dtype=np.int32)
    pp_fids = np.full(g.n_pose_plane, -1, dtype=np.int32)
    odo_fids = np.full(g.n_odometry, -1, dtype=np.int32)
    order = np.argsort(g.pp_pose, kind="stable")
    ptr = np.searchsorted(g.pp_pose[order], np.arange(n + 1))
    odo_of = {int(j): e for e, j in enumerate(g.odo_j)}
    extra = {}
    for i in range(n):
        pose_ids[i] = api.add_pose(None)
        if i == g.prior_pose:
            extra["prior_fid"] = api.add_pose_prior(pose_ids[i], g.prior_meas, g.prior_sqrtinf)
        if i in odo_of:
            e = odo_of[i]
            odo_fids[e] = api.add_odometry(pose_ids[g.odo_i[e]], pose_ids[i], g.odo_meas[e], g.odo_sqrtinf[e])
        es = order[ptr[i]:ptr[i + 1]]
        new = [k for k in g.pp_plane[es] if plane_ids[k] < 0]
        for k in new:
            plane_ids[k] = api.add_plane(None)
        for e in es:
            k = g.pp_plane[e]
            if k in new and k == g.ground_plane:
                # Mapping.cpp:497-504: init the plane, then the ground prior, then the measurement factor
                api.init_plane(plane_ids[k], geo.plane_to_global(geo.pose7_to_T(api.get_pose(pose_ids[i])), g.pp_meas[e]))
                extra["ground_fid"] = api.add_plane_prior(plane_ids[k], g.ground_meas, g.ground_sqrtinf)
            pp_fids[e] = api.add_pose_plane(pose_ids[i], plane_ids[k], g.pp_meas[e], g.pp_sqrtinf[e])
    return dict(pose_ids=pose_ids, plane_ids=plane_ids, pp_fids=pp_fids, odo_fids=odo_fids, **extra)


def build_bulk(api, g):
    """Poses, planes, prior, odometry, ground prior, pose-plane edges -- each through one bulk call,
    with the generator's dead-reckoned initial values."""
    pose_ids = api.add_poses(g.poses_init)
    plane_ids = api.add_planes(g.planes_init)
    extra = {}
    extra["prior_fid"] = api.add_pose_prior(pose_ids[g.prior_pose], g.prior_meas, g.prior_sqrtinf)
    odo_fids = api.add_odometry_bulk(pose_ids[g.odo_i], pose_ids[g.odo_j], g.odo_meas, g.odo_sqrtinf)
    if g.ground_plane >= 0:
        extra["ground_fid"] = api.add_plane_prior(plane_ids[g.ground_plane], g.ground_meas, g.ground_sqrtinf)
    pp_fids = api.add_pose_plane_bulk(pose_ids[g.pp_pose], plane_ids[g.pp_plane], g.pp_meas, g.pp_sqrtinf)
    return dict(pose_ids=pose_ids, plane_ids=plane_ids, pp_fids=pp_fids, odo_fids=odo_fids, **extra)


def configure(api, g, **overrides):
    props = dict(g.properties)
    props.update(overrides)
    api.set_properties(**props)
    api.set_robust(g.robust_kind, g.robust_b)


def rays_from_measurement(T_pose, meas):
    """Two ground-edge rays (sensor frame) for a Pose3d_Plane3d_Factor2: points on the intersection line of the
    measured wall plane `meas` (sensor frame) with the ground plane z = 0 as seen from the camera pose `T_pose`
    (what invK * (x, y, 1) of the wall's ground edge would give, up to scale)."""
    gs = T_pose.T @ np.array([0.0, 0.0, -1.0, 0.0])
    nm, dm = np.asarray(meas[:3], dtype=float), float(meas[3])
    u = np.cross(nm, gs[:3])
    p0 = (-dm * np.cross(gs[:3], u) - gs[3] * np.cross(u, nm)) / (u @ u)
    return np.concatenate([p0 - 0.7 * u / np.linalg.norm(u), p0 + 0.9 * u / np.linalg.norm(u)])
