"""Test-side helpers for the pop-up depth map (pus_popup_depth): the CPU oracle tests/popup_depth_oracle.cpp compiled once
per session into a temporary directory (the tree is not written), its per-pixel source codes and resize chain, and seeded
random batches.  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import popup_cloud_native as NC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None
fp = C.POINTER(C.c_float)
ip = C.POINTER(C.c_int)

# per-pixel source codes of orc_popup_depth_codes: low 16 bits 0 untouched or 1 + the plane's index in its frame, and flags
CEILING, KEPT_AFTER_SKIP, OVERWRITTEN, DEPTH_SKIP, CEILING_SKIP = (1 << k for k in range(16, 21))


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="popup_depth_"), "liborc_depth.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               os.path.join(ROOT, "tests", "popup_depth_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_popup_depth_codes.restype = C.c_longlong
        _lib.orc_popup_depth_codes.argtypes = [C.c_int, ip, ip, fp, fp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_float, ip]
        _lib.orc_popup_depth_resize.argtypes = [fp, C.c_int, C.c_int]
    return _lib


def codes(b):
    """(codes [n_frames, height, width] int32, number of polygon pixels off the image) of a batch (popup_depth kwargs)"""
    a = {k: np.ascontiguousarray(b[k], np.int32) for k in ("plane_ptr", "poly_ptr")}
    a.update({k: np.ascontiguousarray(b[k], np.float32) for k in ("polys", "planes_sensor", "Ts", "invK")})
    nf = len(a["plane_ptr"]) - 1
    out = np.zeros((nf, b["height"], b["width"]), np.int32)
    off = oracle_lib().orc_popup_depth_codes(nf, a["plane_ptr"].ctypes.data_as(ip), a["poly_ptr"].ctypes.data_as(ip),
                                             *[a[k].ctypes.data_as(fp) for k in ("polys", "planes_sensor", "Ts", "invK")],
                                             int(b["width"]), int(b["height"]), int(bool(b["downsample"])),
                                             float(b["ceiling_threshold"]), out.ctypes.data_as(ip))
    return out, off


def resize_chain(m):
    """the oracle's 0.5x / x4 / 2x chain of an even-sized float32 map"""
    m = np.array(m, np.float32, order="C")
    oracle_lib().orc_popup_depth_resize(m.ctypes.data_as(fp), m.shape[1], m.shape[0])
    return m


def random_batch(seed, n_frames, width, height, downsample, ceiling_threshold):
    """popup_depth kwargs of n_frames random frames (popup_cloud_native.random_frame: the ground and 1-5 walls with random
    polygons) plus one frame without planes"""
    rng = np.random.default_rng(seed)
    frames = [NC.random_frame(rng, width, height, int(rng.integers(1, 6))) for _ in range(n_frames)]
    frames.append(([], np.zeros((0, 4), np.float32), np.eye(4, dtype=np.float32)))
    return batch(frames, width, height, downsample, ceiling_threshold)


def batch(frames, width, height, downsample, ceiling_threshold):
    """popup_depth kwargs of a list of (polys, planes, T)"""
    plane_ptr, poly_ptr, P, L, Ts = [0], [0], [np.zeros((0, 2), np.float32)], [np.zeros((0, 4), np.float32)], []
    for polys, planes, T in frames:
        for p in polys:
            P.append(np.asarray(p, np.float32).reshape(-1, 2))
            poly_ptr.append(poly_ptr[-1] + len(P[-1]))
        L.append(np.asarray(planes, np.float32).reshape(-1, 4))
        Ts.append(T)
        plane_ptr.append(plane_ptr[-1] + len(polys))
    return dict(plane_ptr=np.array(plane_ptr, np.int32), poly_ptr=np.array(poly_ptr, np.int32), polys=np.concatenate(P),
                planes_sensor=np.concatenate(L), Ts=np.array(Ts, np.float32).reshape(-1, 4, 4), invK=NC.invK(width, height),
                width=width, height=height, downsample=downsample, ceiling_threshold=ceiling_threshold)
