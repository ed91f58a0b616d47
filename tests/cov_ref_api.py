"""Test-side binding of tests/cov_ref_ext.cpp: the reference driver plus ref_covariance_blocks over the unmodified
reference's own Slam::covariances().access (Covariances.cpp / covariance.cpp, compiled against the CHOLMOD stand-in's R in
oracle/ref_shim).  Compiled once per session into a temporary directory from the reference objects in oracle/_ref/obj;
it needs the reference checkout's headers, so it is only available where that checkout is.  Test infrastructure only."""
import ctypes as C
import os

import numpy as np

from export_api import ISAM, PPS, ROOT, _compile, ref_objects
from pop_up_slam_b200.capi import GraphAPI, _dp, _i32, _ip, c_double_p, c_int_p

_lib = []


def available():
    return ref_objects() is not None


def cov_ref_lib():
    if not _lib:
        objs = ref_objects()
        if objs is None:
            raise RuntimeError("the reference checkout and oracle/_ref/obj are needed (make -C oracle ref)")
        sh = os.path.join(ROOT, "oracle", "ref_shim")
        path = _compile("libref_cov.so", ["g++", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++14", "-fPIC", "-shared", "-w",
                                          "-I" + sh, "-I" + os.path.join(ISAM, "include"), "-I" + PPS,
                                          os.path.join(ROOT, "tests", "cov_ref_ext.cpp")] + objs)
        lib = C.CDLL(path)
        lib.ref_covariance_blocks.restype = C.c_longlong
        lib.ref_covariance_blocks.argtypes = [C.c_void_p, C.c_int, c_int_p, c_double_p]
        lib.ref_standard_rad.restype = C.c_double
        lib.ref_standard_rad.argtypes = [C.c_double]
        _lib.append(lib)
    return _lib[0]


class RefCovAPI(GraphAPI):
    """isam::Slam of the reference with Covariances::access."""

    def __init__(self):
        super().__init__(cov_ref_lib(), "ref_", 0)

    def covariance_blocks(self, pairs, dims):
        p = _i32(np.asarray(pairs).reshape(-1))
        out = np.zeros(max(1, sum(a * b for a, b in dims)))
        self._chk(self.lib.ref_covariance_blocks(self.h, len(dims), _ip(p), _dp(out)))
        res, o = [], 0
        for a, b in dims:
            res.append(out[o:o + a * b].reshape(a, b).copy())
            o += a * b
        return res
