"""Test-side helpers for the closed wall and ground polygons (pus_popup_polygons): the CPU oracle
tests/popup_polygon_oracle.cpp compiled once per session into a temporary directory (the tree is not written), and a
generator of synthetic frames.  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None
fp = C.POINTER(C.c_float)
ip = C.POINTER(C.c_int)


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="popup_polygon_"), "liborc_polygon.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               os.path.join(ROOT, "tests", "popup_polygon_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_convex_hull.argtypes = [fp, C.c_int, fp]
        _lib.orc_point_polygon_test.argtypes = [fp, C.c_int, C.c_float, C.c_float]
        _lib.orc_popup_polygon_codes.argtypes = [C.c_int, ip, fp, fp, fp, fp, C.c_int, C.c_int, C.c_float, C.c_float, ip]
    return _lib


def hull(points):
    """the oracle's cv::convexHull(points) [m, 2]"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 2)
    out = np.zeros((max(len(p), 1), 2), np.float32)
    m = oracle_lib().orc_convex_hull(p.ctypes.data_as(fp), len(p), out.ctypes.data_as(fp))
    return out[:m]


def point_polygon_test(contour, pt):
    c = np.ascontiguousarray(contour, np.float32).reshape(-1, 2)
    return oracle_lib().orc_point_polygon_test(c.ctypes.data_as(fp), len(c), float(pt[0]), float(pt[1]))


def codes(b):
    """the oracle's per-row branch codes [n_rows, 4] of a batch (see orc_popup_polygon_codes)"""
    seg_ptr = np.ascontiguousarray(b["seg_ptr"], np.int32)
    n_rows = int(seg_ptr[-1]) + len(seg_ptr) - 1
    out = np.zeros((n_rows, 4), np.int32)
    a = [np.ascontiguousarray(b[k], np.float32) for k in ("segs", "K", "invK", "Ts")]
    oracle_lib().orc_popup_polygon_codes(len(seg_ptr) - 1, seg_ptr.ctypes.data_as(ip), *[x.ctypes.data_as(fp) for x in a],
                                         int(b["width"]), int(b["height"]), float(b["ceiling_threshold"]),
                                         float(b["walllength_threshold"]), out.ctypes.data_as(ip))
    return out


def camera_K(width, height):
    f = 0.8 * width
    return np.array([[f, 0, width / 2], [0, f, height / 2], [0, 0, 1]], np.float32)


def random_frame(rng, width, height, n_seg=None, snap=0.35, roll_deg=4.0):
    """one frame: a camera 0.8-1.6 m above the floor pitched 5-25 degrees down with a small roll, and a connected ground
    polyline of 1-8 segments below the horizon, left to right; endpoints land exactly on x = 0, x = w-1 or y = h-1 with
    probability snap each.  A roll of 20 degrees or more moves the nadir's image column past the border, so downward image
    directions can leave through a side (the ground polygon's border cases).  Returns (segs [n, 4] float32, T [4, 4]
    float32)."""
    K = camera_K(width, height).astype(np.float64)
    pitch, roll, yaw = np.radians(rng.uniform(5, 25)), np.radians(rng.uniform(-roll_deg, roll_deg)), rng.uniform(0, 2 * np.pi)
    c, s = np.cos(-pitch), np.sin(-pitch)
    Rx = np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    c, s = np.cos(roll), np.sin(roll)
    Rr = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    c, s = np.cos(yaw), np.sin(yaw)
    Rz = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    R = Rz @ np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]) @ Rx @ Rr
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = [rng.uniform(-2, 2), rng.uniform(-2, 2), rng.uniform(0.8, 1.6)]
    iK = np.linalg.inv(K)

    def lowest_ok(x):   # the smallest image row at column x whose ray clearly hits the floor
        for y in range(height):
            d = R @ iK @ [x, y, 1.0]
            if d[2] < -0.08 * np.linalg.norm(d):
                return y
        return height - 1

    n = int(rng.integers(1, 9)) if n_seg is None else n_seg
    xs = np.sort(rng.uniform(0, width - 1, n + 1))
    if rng.random() < snap:
        xs[0] = 0.0
    if rng.random() < snap:
        xs[-1] = width - 1.0
    pts = []
    for i, x in enumerate(xs):
        y0 = min(lowest_ok(x) + 10, height - 1)
        y = rng.uniform(y0, height - 1)
        if rng.random() < snap * (0.6 if 0 < i < n else 1.0):
            y = height - 1.0
        pts.append((x, y))
    pts = np.array(pts, np.float32)
    segs = np.concatenate([pts[:-1], pts[1:]], axis=1)
    return segs.astype(np.float32), T.astype(np.float32)


def corner_frame(rng, width, height):
    """a frame with a strong roll (up to 35 degrees) whose 1-2 segments are squeezed into a bottom corner: the downward
    image directions there can leave through a side border, so the ground polygon's border cases occur"""
    segs, T = random_frame(rng, width, height, n_seg=int(rng.integers(1, 3)), snap=0.0, roll_deg=35.0)
    x = segs[:, [0, 2]]
    segs[:, [0, 2]] = (width - 1 - (width - 1 - x) * 0.05) if rng.random() < 0.5 else x * 0.05
    segs[:, [1, 3]] = height - 1 - (height - 1 - segs[:, [1, 3]]) * 0.1
    return segs.astype(np.float32), T


def batch(frames, width, height, ceiling_threshold, walllength_threshold):
    """the keyword arguments of capi.popup_polygons for a list of (segs, T)"""
    seg_ptr = np.concatenate([[0], np.cumsum([len(s) for s, _ in frames])]).astype(np.int32)
    segs = np.concatenate([s for s, _ in frames]).astype(np.float32) if frames else np.zeros((0, 4), np.float32)
    K = camera_K(width, height)
    return dict(seg_ptr=seg_ptr, segs=segs, K=K, invK=np.linalg.inv(K.astype(np.float64)).astype(np.float32),
                Ts=np.array([T for _, T in frames], np.float32).reshape(-1, 4, 4), width=width, height=height,
                ceiling_threshold=ceiling_threshold, walllength_threshold=walllength_threshold)


def random_batch(seed, n_frames, width, height, ceiling_threshold, walllength_threshold):
    rng = np.random.default_rng(seed)
    return batch([random_frame(rng, width, height) for _ in range(n_frames)], width, height, ceiling_threshold,
                 walllength_threshold)


# the settings every test sweeps: both image sizes, the three wall-length modes, both ceilings
SETTINGS = [((w, h), c, l) for (w, h) in ((640, 480), (960, 540)) for l in (-1.0, 3.0, 0.5) for c in (2.5, 5.0)]
