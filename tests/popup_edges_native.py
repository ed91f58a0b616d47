"""Test-side helpers for the ground edges (pus_popup_edges): the CPU oracle tests/popup_edges_oracle.cpp compiled once per
session into a temporary directory (the tree is not written), its stage entry points, the fixture's batches and seeded
random batches.  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_popup_edge_golden as G  # noqa: E402
from pop_up_slam_b200 import capi  # noqa: E402

_lib = None
fp = C.POINTER(C.c_float)
ip = C.POINTER(C.c_int)
up = C.POINTER(C.c_ubyte)


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="popup_edges_"), "liborc_edges.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               os.path.join(ROOT, "tests", "popup_edges_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_edges_preprocess.argtypes = [up, C.c_int, C.c_int, C.POINTER(capi.EdgeParams), up]
        _lib.orc_edges_contour.argtypes = [up, C.c_int, C.c_int, C.c_int, fp, C.c_int]
        _lib.orc_popup_edges_codes.argtypes = [C.c_int, up, C.c_int, C.c_int, ip, fp, C.POINTER(capi.EdgeParams), ip]
    return _lib


def params(**over):
    return capi.EdgeParams(**dict(capi.EDGE_DEFAULTS, **over))


def preprocess(lab, **over):
    lab = np.ascontiguousarray(lab, np.uint8)
    out = np.zeros(lab.size, np.uint8)
    r = oracle_lib().orc_edges_preprocess(lab.ctypes.data_as(up), lab.shape[1], lab.shape[0], C.byref(params(**over)),
                                          out.ctypes.data_as(up))
    w, h = r >> 16, r & 0xffff
    return out[:w * h].reshape(h, w)


def contour(m, scale=1):
    """the oracle's kept contour points of a preprocessed map, or None"""
    m = np.ascontiguousarray(m, np.uint8)
    pts = np.zeros((m.size + 8, 2), np.float32)
    n = oracle_lib().orc_edges_contour(m.ctypes.data_as(up), m.shape[1], m.shape[0], scale, pts.ctypes.data_as(fp), len(pts))
    return None if n < 0 else pts[:n]


def codes(b):
    lab = np.ascontiguousarray(b["labels"], np.uint8)
    ptr, lines = np.ascontiguousarray(b["line_ptr"], np.int32), np.ascontiguousarray(b["lines"], np.float32)
    out = np.zeros(lab.shape[0], np.int32)
    oracle_lib().orc_popup_edges_codes(lab.shape[0], lab.ctypes.data_as(up), lab.shape[2], lab.shape[1], ptr.ctypes.data_as(ip),
                                       lines.ctypes.data_as(fp), C.byref(params(**b["params"])), out.ctypes.data_as(ip))
    return out


def fixture():
    """[(batch kwargs of capi.popup_edges, expected dict)] of tests/golden/popup_edges.npz"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "popup_edges.npz"))
    out = []
    for ci in range(len(G.CONFIGS)):
        p = z[f"c{ci}_params"]
        prm = {k: (int(v) if k in ("dilation_distance", "erosion_distance", "downsample_contour") else float(v))
               for k, v in zip(capi.EDGE_DEFAULTS, p)}
        b = dict(labels=z[f"c{ci}_labels"], line_ptr=z[f"c{ci}_line_ptr"], lines=z[f"c{ci}_lines"], params=prm)
        want = {k: z[f"c{ci}_{k}"] for k in ("status", "bits", "open_counts", "connect_counts", "open", "connect",
                                             "open_in_connect")}
        out.append((b, want))
    return out


def random_batch(seed, n_frames, width, height, downsample):
    """popup_edges kwargs of n_frames generator frames (tools/make_popup_edge_golden.frame) plus the crafted ones"""
    import cv2
    rng = np.random.default_rng(seed)
    frames = [G.frame(cv2, rng, width, height) for _ in range(n_frames)] + G.crafted(width, height)
    ptr = np.concatenate([[0], np.cumsum([len(L) for _, L in frames])]).astype(np.int32)
    return dict(labels=np.array([f[0] for f in frames]), line_ptr=ptr,
                lines=np.concatenate([np.asarray(L, np.float32).reshape(-1, 4) for _, L in frames]),
                params=dict(downsample_contour=int(downsample)))
