"""Test-side helpers for the line detection (pus_popup_lines): the CPU oracle tests/popup_lines_oracle.cpp compiled once
per session into a temporary directory (the tree is not written), its stage entry points, the fixture's batches and
seeded random batches.  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_popup_line_golden as G  # noqa: E402

_lib = None
vp = C.c_void_p
UNCOVERED = {"ZERO_GRAD"}   # a line of zero mean gradient: no crafted frame reaches it (see DESIGN.md 5.9)


def oracle_lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="popup_lines_"), "liborc_lines.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               os.path.join(ROOT, "tests", "popup_lines_oracle.cpp"), "-o", out])
        _lib = C.CDLL(out)
        _lib.orc_lines_contrast.restype = C.c_int
        _lib.orc_lines_chains.restype = C.c_int
        _lib.orc_lines_chains.argtypes = [vp, C.c_int, C.c_int, vp, C.c_longlong, vp, C.c_longlong]
    return _lib


def _p(a):
    return a.ctypes.data_as(vp)


def grey(img):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.zeros(img.shape[:2], np.uint8)
    oracle_lib().orc_lines_grey(_p(img), img.shape[1], img.shape[0], 3 if img.ndim == 3 else 1, _p(out))
    return out


def contrast(g):
    g = np.ascontiguousarray(g, np.uint8)
    out = np.zeros_like(g)
    bits = oracle_lib().orc_lines_contrast(_p(g), g.shape[1], g.shape[0], _p(out))
    return out, bits


def halve(g):
    g = np.ascontiguousarray(g, np.uint8)
    out = np.zeros((g.shape[0] // 2, g.shape[1] // 2), np.uint8)
    oracle_lib().orc_lines_halve(_p(g), g.shape[1], g.shape[0], _p(out))
    return out


def blur(g):
    g = np.ascontiguousarray(g, np.uint8)
    out = np.zeros_like(g)
    oracle_lib().orc_lines_blur(_p(g), g.shape[1], g.shape[0], _p(out))
    return out


def gradient(b):
    b = np.ascontiguousarray(b, np.uint8)
    dx, dy, g = (np.zeros(b.shape, np.int16) for _ in range(3))
    d = np.zeros(b.shape, np.uint8)
    oracle_lib().orc_lines_gradient(_p(b), b.shape[1], b.shape[0], _p(dx), _p(dy), _p(g), _p(d))
    return dx, dy, g, d


def chains(b):
    """the oracle's chains of a blurred image as lists of (x, y), or the status"""
    b = np.ascontiguousarray(b, np.uint8)
    px, sid = np.zeros(b.size, np.int32), np.zeros(b.size // 16 + 2, np.int32)
    n = oracle_lib().orc_lines_chains(_p(b), b.shape[1], b.shape[0], _p(px), px.size, _p(sid), sid.size)
    if n < 0:
        return n
    w = b.shape[1]
    return [[(int(p) % w, int(p) // w) for p in px[sid[c]:sid[c + 1]]] for c in range(n)]


def bits(images, downsample):
    images = np.ascontiguousarray(images, np.uint8)
    out = np.zeros(images.shape[0], np.uint32)
    ch = 3 if images.ndim == 4 else 1
    oracle_lib().orc_popup_lines_bits(images.shape[0], _p(images), images.shape[2], images.shape[1], ch, int(downsample),
                                      _p(out))
    return out


def fixture(path=None):
    """[(key, images, downsample, expected dict)] of tests/golden/popup_lines.npz"""
    z = np.load(path or os.path.join(ROOT, "tests", "golden", "popup_lines.npz"))
    cv2 = G.cv()
    return [(str(k), z[f"{k}_images"] if f"{k}_images" in z else np.asarray(G.frames(cv2, str(k).replace("_ds", ""))),
             int(z[f"{k}_downsample"]), {n: z[f"{k}_{n}"] for n in ("status", "counts", "lines", "bits")})
            for k in z["keys"]]


def random_batch(seed, n_frames, width, height, channels):
    import cv2
    G.cv()
    rng = np.random.default_rng(seed)
    return np.array([G.room(cv2, rng, width, height, channels) for _ in range(n_frames)])
