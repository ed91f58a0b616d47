"""Test-side bindings for the parity tests of the error / Jacobian export (pus_weighted_errors, pus_factor_errors,
pus_jacobian, pus_normalized_chi2, pus_local_chi2): the oracle and the reference build with the same method names as
GpuGraphAPI, through native entry points of the same shapes.

  tests/export_oracle_ext.cpp  the oracle (oracle/oracle_capi.cpp, included unmodified) + orc_weighted_errors, orc_factor_errors,
                               orc_jacobian, orc_normalized_chi2, orc_local_chi2 over its restatement of the Slam methods;
  tests/export_ref_ext.cpp     the reference driver (oracle/ref_driver.cpp, included unmodified) + ref_* entries over the
                               reference's own Slam::weighted_errors, Slam::jacobian() (both branches), normalized_chi2 and
                               local_chi2, linked against the reference objects in oracle/_ref/obj.

Both are compiled once per test session into a temporary directory (the tree is not written).  Test infrastructure only."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import numpy as np
import scipy.sparse as sp

from oracle_api import OracleAPI
from pop_up_slam_b200.capi import GraphAPI, _dp, _i32, _ip, c_double_p, c_int_p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = "/root/reference"
ISAM = os.path.join(REFERENCE, "pop_planar_slam", "Thirdparty", "isam")
PPS = os.path.join(REFERENCE, "pop_planar_slam", "src")
_TMP = tempfile.mkdtemp(prefix="export_native_")
_libs = {}


def _compile(name, cmd):
    out = os.path.join(_TMP, name)
    subprocess.check_call(cmd + ["-o", out])
    return out


def oracle_ext():
    if "orc" not in _libs:
        path = _compile("liborc_export.so", ["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                                             "-w", os.path.join(ROOT, "tests", "export_oracle_ext.cpp")])
        _libs["orc"] = _bind(C.CDLL(path), "orc_")
    return _libs["orc"]


def ref_objects():
    objs = [o for o in glob.glob(os.path.join(ROOT, "oracle", "_ref", "obj", "*.o")) if not o.endswith("ref_driver.o")]
    return objs if len(objs) > 5 and os.path.isdir(ISAM) else None


def ref_ext():
    if "ref" not in _libs:
        objs = ref_objects()
        if objs is None:
            raise RuntimeError("the reference checkout and oracle/_ref/obj are needed (make -C oracle ref)")
        sh = os.path.join(ROOT, "oracle", "ref_shim")
        path = _compile("libref_export.so", ["g++", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++14", "-fPIC", "-shared", "-w",
                                             "-I" + sh, "-I" + os.path.join(ISAM, "include"), "-I" + PPS,
                                             os.path.join(ROOT, "tests", "export_ref_ext.cpp")] + objs)
        lib = _bind(C.CDLL(path), "ref_")
        lib.ref_standard_rad.restype = C.c_double
        lib.ref_standard_rad.argtypes = [C.c_double]
        _libs["ref"] = lib
    return _libs["ref"]


def _bind(lib, p):
    getattr(lib, p + "weighted_errors").restype = C.c_longlong
    getattr(lib, p + "weighted_errors").argtypes = [C.c_void_p, c_double_p, C.c_longlong]
    getattr(lib, p + "factor_errors").argtypes = [C.c_void_p, C.c_int, c_int_p, c_double_p]
    getattr(lib, p + "jacobian").restype = C.c_longlong
    getattr(lib, p + "jacobian_dims").argtypes = [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    getattr(lib, p + "local_chi2").argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double)]
    return lib


class ExportMixin:
    """weighted_errors / factor_errors / jacobian / normalized_chi2 / local_chi2 / jacobian_dims over <prefix>_* entries."""

    def jacobian_dims(self):
        r, c = C.c_longlong(0), C.c_longlong(0)
        self._chk(self._f("jacobian_dims")(self.h, C.byref(r), C.byref(c)))
        return r.value, c.value

    def weighted_errors(self):
        fn = self._f("weighted_errors")
        rows = self._chk(fn(self.h, None, 0))
        out = np.zeros(rows)
        self._chk(fn(self.h, _dp(out), rows))
        return out

    def factor_errors(self, fids):
        fids = _i32(np.atleast_1d(fids))
        out = np.zeros(6 * len(fids))
        n = self._chk(self._f("factor_errors")(self.h, len(fids), _ip(fids), _dp(out)))
        return out[:n].copy()

    def _jacobian_call(self, *args):
        return self._f("jacobian")(self.h, *args)

    def jacobian(self):
        rows, cols = self.jacobian_dims()
        nnz = self._chk(self._jacobian_call(None, None, None, None, C.c_longlong(0)))
        row_ptr, col_idx = np.zeros(rows + 1, dtype=np.int32), np.zeros(max(nnz, 1), dtype=np.int32)
        vals, rhs = np.zeros(max(nnz, 1)), np.zeros(rows)
        self._chk(self._jacobian_call(_ip(row_ptr), _ip(col_idx), _dp(vals), _dp(rhs), C.c_longlong(nnz)))
        return sp.csr_matrix((vals[:nnz], col_idx[:nnz], row_ptr), shape=(rows, cols)), rhs

    def normalized_chi2(self):
        out = C.c_double(0)
        self._chk(self._f("normalized_chi2")(self.h, C.byref(out)))
        return out.value

    def local_chi2(self, last_n):
        out = C.c_double(0)
        self._chk(self._f("local_chi2")(self.h, int(last_n), C.byref(out)))
        return out.value


class OracleExportAPI(ExportMixin, OracleAPI):
    """The oracle (its own handle in the extended library) with the export's names.  Jacobian mode as
    OracleAPI.set_jacobian_mode: 0 = the reference's central differences, 1 = the analytic blocks."""

    def __init__(self):
        GraphAPI.__init__(self, oracle_ext(), "orc_", 0)

    def live_fids(self, n_ids=None):
        """live factor ids, ascending (factor_nodes refuses a removed or unknown id)"""
        out, f, buf = [], 0, np.zeros(2, dtype=np.int32)
        n = self.lib.orc_num_factors(self.h)
        while len(out) < n:
            if self.lib.orc_factor_nodes(self.h, f, _ip(buf)) >= 0:
                out.append(f)
            f += 1
        return out


class RefExportAPI(ExportMixin, GraphAPI):
    """The reference build with the export's names; columnwise=True sets Properties::force_numerical_jacobian for
    Slam::jacobian() (jacobian_numerical_columnwise), else Slam::jacobian() runs jacobian_partial over each factor's
    numericalDiff."""

    def __init__(self, columnwise=False):
        GraphAPI.__init__(self, ref_ext(), "ref_", 0)
        self.columnwise = columnwise

    def _jacobian_call(self, *args):
        return self.lib.ref_jacobian(self.h, int(self.columnwise), *args)
