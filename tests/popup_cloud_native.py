"""Test-side helpers for the dense plane clouds (pus_popup_clouds): the CPU oracle tests/popup_cloud_oracle.cpp compiled
once per session into a temporary directory (the tree is not written), the synthetic BGR image every fixture and test
uses, and a generator of random frames.  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="popup_cloud_"), "liborc_cloud.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               os.path.join(ROOT, "tests", "popup_cloud_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_popup_polygon_pixels.restype = C.c_longlong
        _lib.orc_popup_polygon_pixels.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.POINTER(C.c_int), C.c_longlong]
    return _lib


def oracle_pixels(poly, downsample):
    """the oracle's pixel list [m, 2] (x, y) of one polygon, in findNonZero order"""
    lib = oracle_lib()
    poly = np.ascontiguousarray(poly, dtype=np.float32).reshape(-1, 2)
    fp = poly.ctypes.data_as(C.POINTER(C.c_float))
    m = lib.orc_popup_polygon_pixels(fp, len(poly), int(downsample), None, 0)
    out = np.zeros((m, 2), np.int32)
    lib.orc_popup_polygon_pixels(fp, len(poly), int(downsample), out.ctypes.data_as(C.POINTER(C.c_int)), m)
    return out


def fixture_pixels(boxes, masks, downsample):
    """the pixel lists [m, 2] (x, y) of a fixture case, one per polygon: each box mask's nonzero pixels in row-major order
    (findNonZero's) plus the box offset, doubled when downsampling"""
    bits = np.unpackbits(masks)
    out, at = [], 0
    for bx, by, bw, bh in boxes:
        m = bits[at:at + bw * bh].reshape(bh, bw)
        at += bw * bh
        out.append(((np.argwhere(m)[:, ::-1] + [bx, by]) * (2 if downsample else 1)).astype(np.int32).reshape(-1, 2))
    return out


def image(frame, width, height):
    """the synthetic BGR image of a frame: a fixed function of (frame, row, column)"""
    y, x = np.mgrid[0:height, 0:width]
    return np.stack([(x * 7 + y * 3 + frame) % 256, (x * 5 + y * 11 + 3 * frame) % 256, (x + y * 13 + 7 * frame) % 256],
                    axis=-1).astype(np.uint8)


def _polygon(rng, kind, w, h):
    if kind == "convex":
        c = rng.uniform([0, 0], [w, h])
        r = rng.uniform(5, min(w, h) / 3)
        a = np.sort(rng.uniform(0, 2 * np.pi, int(rng.integers(3, 9))))
        return c + r * np.stack([np.cos(a), np.sin(a)], 1)
    if kind == "nonconvex":
        return rng.uniform([-0.1 * w, -0.1 * h], [1.1 * w, 1.1 * h], size=(int(rng.integers(4, 9)), 2))
    if kind == "offimage":
        c = rng.uniform([-0.3 * w, -0.3 * h], [1.3 * w, 1.3 * h])
        return c + rng.uniform(-w / 3, w / 3, size=(int(rng.integers(3, 7)), 2))
    if kind == "degenerate":
        n = int(rng.integers(0, 3))
        return rng.uniform([0, 0], [w, h], size=(n, 2))
    if kind == "collinear":
        p, d = rng.uniform([0, 0], [w, h]), rng.normal(size=2)
        return p + np.outer(rng.uniform(-100, 100, int(rng.integers(3, 6))), d)
    raise ValueError(kind)


KINDS = ("convex", "nonconvex", "offimage", "degenerate", "collinear")


def random_frame(rng, width, height, n_walls, kinds=KINDS, extent=1.0):
    """one frame: the ground plane and n_walls walls, each with a random polygon drawn in a random window of extent times
    the image size; returns (polys list, planes [n, 4], T)"""
    pitch, yaw = rng.uniform(-0.4, 0.1), rng.uniform(0, 2 * np.pi)   # a camera looking roughly horizontally, tilted down
    Rx = np.array([[1, 0, 0], [0, np.cos(pitch), -np.sin(pitch)], [0, np.sin(pitch), np.cos(pitch)]])
    Rz = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    R = Rz @ np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]) @ Rx
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = [rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(0.5, 1.5)]
    planes_w = [np.array([0.0, 0.0, -1.0, 0.0])]
    for _ in range(n_walls):
        a = rng.uniform(0, 2 * np.pi)
        planes_w.append(np.array([np.cos(a), np.sin(a), 0.0, rng.uniform(-4, 4)]))
    planes = np.array([T.T @ p for p in planes_w], np.float32)
    polys = []
    for i in range(n_walls + 1):
        poly = _polygon(rng, "convex" if i == 0 else kinds[int(rng.integers(len(kinds)))], extent * width, extent * height)
        poly = np.asarray(poly).reshape(-1, 2) + rng.uniform([0, 0], [(1 - extent) * width + 1e-9, (1 - extent) * height + 1e-9])
        polys.append(poly.astype(np.float32))
    return polys, planes, T.astype(np.float32)


def invK(width, height):
    f = 0.8 * width
    K = np.array([[f, 0, width / 2], [0, f, height / 2], [0, 0, 1]])
    return np.linalg.inv(K).astype(np.float32)


def batch(frames):
    """CSR arrays of a list of (polys, planes, T): plane_ptr, poly_ptr, polys, planes, Ts"""
    plane_ptr, poly_ptr, P, L, Ts = [0], [0], [], [], []
    for polys, planes, T in frames:
        for p in polys:
            P.append(p)
            poly_ptr.append(poly_ptr[-1] + len(p))
        L.append(planes)
        Ts.append(T)
        plane_ptr.append(plane_ptr[-1] + len(polys))
    return (np.array(plane_ptr, np.int32), np.array(poly_ptr, np.int32), np.concatenate(P).reshape(-1, 2).astype(np.float32),
            np.concatenate(L).astype(np.float32), np.array(Ts, np.float32))
