"""A malformed seg_ptr (NULL, not starting at 0, decreasing, or more rows than an int counts) is refused with a message
naming it, before any device work: by pus_popup_fit_frames and by both measurement-refresh calls.  pus_popup_polygons
refuses a frame above PUS_POPUP_MAX_SEGMENTS before it builds any row table.  These run with or without a GPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

BAD = [[0, 5, 1], [1, 2]]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_P = C.POINTER(C.c_int)


def _last_error(lib):
    lib.pus_last_error.restype = C.c_char_p
    return lib.pus_last_error()


def _fit(lib, seg_ptr):
    nf = len(seg_ptr) - 1
    segs = np.zeros((8, 4), np.float32)
    Ts = np.eye(4, dtype=np.float32)[None].repeat(nf, 0)
    return capi.popup_fit_frames(lib, seg_ptr, segs, np.eye(3, dtype=np.float32), Ts)


@pytest.mark.parametrize("seg_ptr", BAD)
def test_fit_frames_refuses(seg_ptr):
    lib = capi.load_library()
    with pytest.raises(capi.ApiError):
        _fit(lib, seg_ptr)
    assert b"seg_ptr" in _last_error(lib)


def test_fit_frames_refuses_null():
    lib = capi.load_library()
    fn = lib.pus_popup_fit_frames
    rc = fn(C.c_int(0), C.c_int(1), None, None, None, None, C.c_float(10.0), C.c_int(0), None, None, None, None)
    assert rc < 0 and b"seg_ptr" in _last_error(lib)


def test_fit_frames_refuses_more_rows_than_an_int_counts():
    lib = capi.load_library()
    seg_ptr = np.array([0, 2**31 - 1], np.int32)
    fn = lib.pus_popup_fit_frames
    rc = fn(C.c_int(0), C.c_int(1), seg_ptr.ctypes.data_as(INT_P), None, None, None, C.c_float(10.0), C.c_int(0), None, None,
            None, None)
    assert rc < 0 and b"seg_ptr" in _last_error(lib)


@pytest.mark.parametrize("call", ["refresh_plane_measurements", "refresh_bind"])
@pytest.mark.parametrize("seg_ptr", BAD)
def test_refresh_refuses(call, seg_ptr):
    a = GpuGraphAPI()
    ids = gg.build_bulk(a, gg.make_config(1, seed=0))
    nf = len(seg_ptr) - 1
    segs = np.zeros((8, 4), np.float32)
    with pytest.raises(capi.ApiError, match="seg_ptr"):
        getattr(a, call)(ids["pose_ids"][:nf], seg_ptr, segs, np.eye(3), ids["pp_fids"][:1], [0], [0])


@pytest.mark.parametrize("call", ["refresh_plane_measurements", "refresh_bind"])
def test_refresh_refuses_null(call):
    a = GpuGraphAPI()
    ids = gg.build_bulk(a, gg.make_config(1, seed=0))
    frame_pose = np.ascontiguousarray(ids["pose_ids"][:1], np.int32)
    fid = np.ascontiguousarray(ids["pp_fids"][:1], np.int32)
    zero = np.zeros(1, np.int32)
    segs = np.zeros((1, 4), np.float32)
    invK = np.eye(3, dtype=np.float32)
    float_p = C.POINTER(C.c_float)
    args = [a.h, C.c_int(1), frame_pose.ctypes.data_as(INT_P), None, segs.ctypes.data_as(float_p),
            invK.ctypes.data_as(float_p), C.c_int(1), fid.ctypes.data_as(INT_P), zero.ctypes.data_as(INT_P),
            zero.ctypes.data_as(INT_P)]
    fn = getattr(a.lib, "pus_" + call)
    rc = fn(*(args + [None] if call == "refresh_plane_measurements" else args))
    assert rc < 0 and b"seg_ptr" in _last_error(a.lib)


_POLYGONS = r"""
import ctypes as C, resource, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from pop_up_slam_b200 import capi
lib = capi.load_library()
lib.pus_last_error.restype = C.c_char_p
seg_ptr = np.array([int(v) for v in sys.argv[2].split(",")], np.int32)
counts = np.zeros(4, np.int32)
ip = counts.ctypes.data_as(C.POINTER(C.c_int))
before = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
rc = lib.pus_popup_polygons(C.c_int(0), C.c_int(len(seg_ptr) - 1), seg_ptr.ctypes.data_as(C.POINTER(C.c_int)), None, None,
                            None, None, C.c_int(640), C.c_int(480), C.c_float(2.5), C.c_float(3.0), ip, ip, ip, None, None,
                            None, C.c_longlong(0), C.c_longlong(0), C.c_longlong(0))
grown = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss - before
print(rc, grown, lib.pus_last_error().decode())
"""


@pytest.mark.parametrize("seg_ptr", ["0,268435456", "0,300,299", "0,2147483647"])
def test_polygons_refuses_a_long_frame_before_building_rows(seg_ptr):
    """each frame's order and segment cap are checked in turn, before the row table is sized; a fresh process, so that its
    peak resident size shows what the refusal allocated"""
    out = subprocess.run([sys.executable, "-c", _POLYGONS, ROOT, seg_ptr], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    rc, grown_kb, why = out.stdout.strip().split(" ", 2)
    assert int(rc) < 0 and "PUS_POPUP_MAX_SEGMENTS" in why
    assert int(grown_kb) < 64 * 1024
