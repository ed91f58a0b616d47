"""ctypes binding of the C-ABI declared in include/popup_gpu.h.

`GraphAPI` is a thin, prefix-generic wrapper: the product binds it to libpopup_gpu.so with the
`pus_` prefix (see `load_library` / `Solver` in slam.py); the test-suite binds the same class to the CPU
oracle's `orc_` entry points, so parity tests drive both through identical calls.  Nothing here
imports or loads anything under oracle/.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpopup_gpu.so")

c_double_p = C.POINTER(C.c_double)
c_int_p = C.POINTER(C.c_int)
c_float_p = C.POINTER(C.c_float)


class Properties(C.Structure):
    """pus_properties (isam::Properties, Properties.h:37-110)."""
    _fields_ = [("method", C.c_int), ("epsilon2", C.c_double), ("epsilon_abs", C.c_double),
                ("epsilon_rel", C.c_double), ("max_iterations", C.c_int), ("lm_lambda0", C.c_double),
                ("lm_lambda_factor", C.c_double), ("mod_update", C.c_int), ("mod_batch", C.c_int),
                ("mod_solve", C.c_int)]


class SolverOptions(C.Structure):
    _fields_ = [("pcg_rel_tol", C.c_double), ("pcg_max_iter", C.c_int), ("ctas_per_sm", C.c_int),
                ("team_ctas", C.c_int), ("reserved", C.c_int * 4)]


class Stats(C.Structure):
    _fields_ = [("lm_iterations", C.c_int), ("accepted", C.c_int), ("relinearizations", C.c_int),
                ("chi2_evals", C.c_int), ("pcg_iterations", C.c_longlong), ("chi2_initial", C.c_double),
                ("chi2_final", C.c_double), ("kernel_ms", C.c_double), ("h2d_ms", C.c_double),
                ("d2h_ms", C.c_double), ("h2d_bytes", C.c_longlong), ("d2h_bytes", C.c_longlong),
                ("n_poses", C.c_int), ("n_planes", C.c_int), ("n_pose_plane", C.c_int), ("n_odometry", C.c_int),
                ("n_pose_prior", C.c_int), ("n_plane_prior", C.c_int), ("gpu_launches", C.c_int),
                ("grid_ctas", C.c_int), ("block_threads", C.c_int), ("phase_ms", C.c_double * 24)]

    def as_dict(self):
        d = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            d[name] = list(v) if hasattr(v, "__len__") else v
        return d


def _dp(a):
    return a.ctypes.data_as(c_double_p)


def _ip(a):
    return a.ctypes.data_as(c_int_p)


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None:
        assert a.shape == shape, (a.shape, shape)
    return a


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class ApiError(RuntimeError):
    pass


def load_library(path=None):
    """Load libpopup_gpu.so. Fails loudly when the CUDA library has not been built -- there is no
    CPU fallback behind this ABI."""
    path = path or os.environ.get("PUS_LIBRARY", LIB_PATH)   # (PUS_LIBRARY: A/B builds of the same ABI)
    if not os.path.exists(path):
        raise ApiError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a). There is no CPU fallback.")
    return C.CDLL(path)


class GraphAPI:
    """One solver handle behind the C-ABI (prefix `pus_` = CUDA library, `orc_` = test oracle)."""

    def __init__(self, lib, prefix="pus_", device=0):
        self.lib = lib
        self.prefix = prefix
        self._bind()
        h = C.c_void_p()
        self._chk(self._f("create")(int(device), C.byref(h)))
        self.h = h

    # -- plumbing --
    def _f(self, name):
        return getattr(self.lib, self.prefix + name)

    def _bind(self):
        f = self._f
        f("last_error").restype = C.c_char_p
        for name in ("debug_fetch", "debug_store", "normal_equations"):
            if hasattr(self.lib, self.prefix + name):
                f(name).restype = C.c_longlong
        if hasattr(self.lib, self.prefix + "set_robust"):
            f("set_robust").argtypes = [C.c_void_p, C.c_int, C.c_double]
        if hasattr(self.lib, self.prefix + "debug_run_stage"):
            f("debug_run_stage").argtypes = [C.c_void_p, C.c_int, C.c_double]

    def _chk(self, rc):
        if rc < 0:
            msg = self._f("last_error")()
            raise ApiError((msg or b"?").decode())
        return rc

    def close(self):
        if self.h is not None:
            self._f("destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- vertices --
    def add_pose(self, init7=None):
        p = _dp(_f64(init7, (7,))) if init7 is not None else None
        return self._chk(self._f("add_pose")(self.h, p))

    def add_plane(self, abcd=None):
        p = _dp(_f64(abcd, (4,))) if abcd is not None else None
        return self._chk(self._f("add_plane")(self.h, p))

    def add_poses(self, init7s):
        v = _f64(init7s)
        ids = np.empty(len(v), dtype=np.int32)
        self._chk(self._f("add_poses")(self.h, len(v), _dp(v), _ip(ids)))
        return ids

    def add_planes(self, abcds):
        v = _f64(abcds)
        ids = np.empty(len(v), dtype=np.int32)
        self._chk(self._f("add_planes")(self.h, len(v), _dp(v), _ip(ids)))
        return ids

    def init_pose(self, id_, init7):
        self._chk(self._f("init_pose")(self.h, int(id_), _dp(_f64(init7, (7,)))))

    def init_plane(self, id_, abcd):
        self._chk(self._f("init_plane")(self.h, int(id_), _dp(_f64(abcd, (4,)))))

    def init_poses(self, ids, init7s):
        ids, v = _i32(ids), _f64(init7s, (len(ids), 7))
        self._chk(self._f("init_poses")(self.h, len(ids), _ip(ids), _dp(v)))

    def init_planes(self, ids, abcds):
        ids, v = _i32(ids), _f64(abcds, (len(ids), 4))
        self._chk(self._f("init_planes")(self.h, len(ids), _ip(ids), _dp(v)))

    def get_pose(self, id_):
        out = np.empty(7)
        self._chk(self._f("get_pose")(self.h, int(id_), _dp(out)))
        return out

    def get_plane(self, id_):
        out = np.empty(4)
        self._chk(self._f("get_plane")(self.h, int(id_), _dp(out)))
        return out

    def get_poses(self, ids):
        ids = _i32(ids)
        out = np.empty((len(ids), 7))
        self._chk(self._f("get_poses")(self.h, len(ids), _ip(ids), _dp(out)))
        return out

    def get_planes(self, ids):
        ids = _i32(ids)
        out = np.empty((len(ids), 4))
        self._chk(self._f("get_planes")(self.h, len(ids), _ip(ids), _dp(out)))
        return out

    # -- edges --
    def add_pose_prior(self, pose, xyzypr, sqrtinf21):
        return self._chk(self._f("add_pose_prior")(self.h, int(pose), _dp(_f64(xyzypr, (6,))), _dp(_f64(sqrtinf21, (21,)))))

    def add_odometry(self, p1, p2, xyzypr, sqrtinf21):
        return self._chk(self._f("add_odometry")(self.h, int(p1), int(p2), _dp(_f64(xyzypr, (6,))), _dp(_f64(sqrtinf21, (21,)))))

    def add_pose_plane(self, pose, plane, meas4, sqrtinf6):
        return self._chk(self._f("add_pose_plane")(self.h, int(pose), int(plane), _dp(_f64(meas4, (4,))), _dp(_f64(sqrtinf6, (6,)))))

    def add_pose_plane2(self, pose, plane, meas4, rays6, sqrtinf6):
        """Pose3d_Plane3d_Factor2: measurement re-popped from two ground-edge rays inside the residual."""
        fn = self._f("add_pose_plane2")
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p]
        return self._chk(fn(self.h, int(pose), int(plane), _dp(_f64(meas4, (4,))), _dp(_f64(rays6, (6,))), _dp(_f64(sqrtinf6, (6,)))))

    def add_plane_prior(self, plane, abcd, sqrtinf6):
        return self._chk(self._f("add_plane_prior")(self.h, int(plane), _dp(_f64(abcd, (4,))), _dp(_f64(sqrtinf6, (6,)))))

    def add_odometry_bulk(self, p1, p2, xyzypr, sqrtinf21):
        p1, p2 = _i32(p1), _i32(p2)
        m, s = _f64(xyzypr, (len(p1), 6)), _f64(sqrtinf21, (len(p1), 21))
        out = np.empty(len(p1), dtype=np.int32)
        if len(p1):
            self._chk(self._f("add_odometry_bulk")(self.h, len(p1), _ip(p1), _ip(p2), _dp(m), _dp(s), _ip(out)))
        return out

    def add_pose_plane_bulk(self, pose, plane, meas4, sqrtinf6):
        pose, plane = _i32(pose), _i32(plane)
        m, s = _f64(meas4, (len(pose), 4)), _f64(sqrtinf6, (len(pose), 6))
        out = np.empty(len(pose), dtype=np.int32)
        if len(pose):
            self._chk(self._f("add_pose_plane_bulk")(self.h, len(pose), _ip(pose), _ip(plane), _dp(m), _dp(s), _ip(out)))
        return out

    def set_measurement(self, fid, meas):
        self._chk(self._f("set_measurement")(self.h, int(fid), _dp(_f64(meas))))

    def get_measurement(self, fid, n=4):
        out = np.zeros(6)
        self._chk(self._f("get_measurement")(self.h, int(fid), _dp(out)))
        return out[:n]

    def remove_factor(self, fid):
        self._chk(self._f("remove_factor")(self.h, int(fid)))

    def remove_node(self, id_):
        self._chk(self._f("remove_node")(self.h, int(id_)))

    def num_nodes(self):
        return self._chk(self._f("num_nodes")(self.h))

    def num_factors(self):
        return self._chk(self._f("num_factors")(self.h))

    def factor_nodes(self, fid):
        out = np.zeros(2, dtype=np.int32)
        n = self._chk(self._f("factor_nodes")(self.h, int(fid), _ip(out)))
        return out[:n].tolist()

    def node_factors(self, id_, cap=1 << 16):
        out = np.zeros(cap, dtype=np.int32)
        n = self._chk(self._f("node_factors")(self.h, int(id_), _ip(out), cap))
        return out[:min(n, cap)].tolist()

    def node_start(self, id_):
        return self._f("node_start")(self.h, int(id_))

    def factor_row(self, fid):
        return self._f("factor_row")(self.h, int(fid))

    # -- configuration --
    def get_properties(self):
        p = Properties()
        self._chk(self._f("get_properties")(self.h, C.byref(p)))
        return {n: getattr(p, n) for n, _ in Properties._fields_}

    def set_properties(self, **kw):
        p = Properties()
        self._chk(self._f("get_properties")(self.h, C.byref(p)))
        for k, v in kw.items():
            if not hasattr(p, k):
                raise KeyError(k)
            setattr(p, k, v)
        self._chk(self._f("set_properties")(self.h, C.byref(p)))

    def set_robust(self, kind, b):
        self._chk(self._f("set_robust")(self.h, int(kind), float(b)))

    # -- optimisation --
    def batch_optimize(self):
        it = C.c_int(0)
        self._chk(self._f("batch_optimize")(self.h, C.byref(it)))
        return it.value

    def update(self):
        self._chk(self._f("update")(self.h))

    def chi2(self):
        out = C.c_double(0)
        self._chk(self._f("chi2")(self.h, C.byref(out)))
        return out.value

    def trace(self, cap=4096):
        lam, en, eb, dn = (np.zeros(cap) for _ in range(4))
        acc, pcg = np.zeros(cap, dtype=np.int32), np.zeros(cap, dtype=np.int32)
        n = self._chk(self._f("get_trace")(self.h, cap, _dp(lam), _dp(en), _dp(eb), _dp(dn), _ip(acc), _ip(pcg)))
        n = min(n, cap)
        return dict(lam=lam[:n], chi2_new=en[:n], chi2_before=eb[:n], delta_norm=dn[:n], accepted=acc[:n], pcg=pcg[:n])

    def save_graph(self, path, precision=0):
        """Slam::save text format (include/popup_gpu.h); host only."""
        fn = self._f("save_graph")
        fn.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        self._chk(fn(self.h, str(path).encode(), int(precision)))

    def load_isam_dataset(self, path):
        """3-D part of the iSAM dataset grammar (EDGE3, POSE3D_INIT); returns (poses added, factors added)."""
        fn = self._f("load_isam_dataset")
        fn.argtypes = [C.c_void_p, C.c_char_p, c_int_p, c_int_p]
        a, b = C.c_int(0), C.c_int(0)
        self._chk(fn(self.h, str(path).encode(), C.byref(a), C.byref(b)))
        return a.value, b.value

    def refresh_plane_measurements(self, frame_pose, seg_ptr, segs, invK, map_fid, map_frame, map_row):
        """Mapper_mono::update_plane_measurement on the resident estimates (include/popup_gpu.h); returns the new
        measurements [n_map, 4]."""
        frame_pose, seg_ptr = _i32(frame_pose), _i32(seg_ptr)
        map_fid, map_frame, map_row = _i32(map_fid), _i32(map_frame), _i32(map_row)
        segs = np.ascontiguousarray(segs, dtype=np.float32).reshape(-1, 4)
        invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
        out = np.zeros((len(map_fid), 4))
        fn = self._f("refresh_plane_measurements")
        fn.argtypes = [C.c_void_p, C.c_int, c_int_p, c_int_p, c_float_p, c_float_p, C.c_int, c_int_p, c_int_p, c_int_p, c_double_p]
        self._chk(fn(self.h, len(frame_pose), _ip(frame_pose), _ip(seg_ptr), segs.ctypes.data_as(c_float_p),
                     invK.ctypes.data_as(c_float_p), len(map_fid), _ip(map_fid), _ip(map_frame), _ip(map_row), _dp(out)))
        return out

    def refresh_bind(self, frame_pose, seg_ptr, segs, invK, map_fid, map_frame, map_row):
        """pus_refresh_bind: keep the frames' segment lists / invK / factor map resident on the device."""
        frame_pose, seg_ptr = _i32(frame_pose), _i32(seg_ptr)
        segs = np.ascontiguousarray(segs, dtype=np.float32).reshape(-1, 4)
        invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
        map_fid, map_frame, map_row = _i32(map_fid), _i32(map_frame), _i32(map_row)
        self._n_map = len(map_fid)
        self._chk(self._f("refresh_bind")(self.h, len(frame_pose), _ip(frame_pose), _ip(seg_ptr), segs.ctypes.data_as(c_float_p),
                                          invK.ctypes.data_as(c_float_p), len(map_fid), _ip(map_fid), _ip(map_frame), _ip(map_row)))

    def refresh_run(self, want_output=False):
        """pus_refresh_run: re-pop every bound frame from the resident pose estimates; new measurements stay on the device unless
        `want_output`."""
        out = np.zeros((self._n_map, 4)) if want_output else None
        self._chk(self._f("refresh_run")(self.h, _dp(out) if want_output else None))
        return out

    def project_to_planes(self, plane_ids, pts):
        """Plane3d::project_to_plane of float points onto the current plane estimates (include/popup_gpu.h)."""
        plane_ids = _i32(plane_ids)
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        out = np.zeros_like(pts)
        fn = self._f("project_to_planes")
        fn.argtypes = [C.c_void_p, C.c_int, c_int_p, c_float_p, c_float_p]
        self._chk(fn(self.h, len(plane_ids), _ip(plane_ids), pts.ctypes.data_as(c_float_p), out.ctypes.data_as(c_float_p)))
        return out


class GpuGraphAPI(GraphAPI):
    """GraphAPI plus the entry points only the CUDA library has (solver options, split
    upload/solve/download, stats, debug hooks)."""

    def __init__(self, lib=None, device=0):
        super().__init__(lib if lib is not None else load_library(), "pus_", device)

    def set_stream(self, cuda_stream_ptr):
        self._chk(self.lib.pus_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))

    def set_jacobian_mode(self, mode):
        """Same convention as the oracle binding: 0 = the reference's numerical differences (numericalDiff, eps = 1e-4), 1 = closed
        forms (the default of the CUDA library)."""
        self._chk(self.lib.pus_set_jacobian_mode(self.h, 1 if int(mode) == 0 else 0))

    def set_linear_solver(self, direct):
        """direct=True or 1: solve the reduced pose system exactly (dense Cholesky on the device, graphs of at most 640 poses);
        2: exactly, by a band Cholesky of the bordered system (any graph within its device-memory budget);
        direct=False or 0: block-preconditioned CG (the default)."""
        if isinstance(direct, bool):
            kind = 1 if direct else 0
        elif isinstance(direct, (int, np.integer)) and int(direct) in (0, 1, 2):
            kind = int(direct)
        else:
            raise ValueError(f"linear solver: expected True / False or a kind 0, 1 or 2, got {direct!r}")
        self._chk(self.lib.pus_set_linear_solver(self.h, kind))

    def linear_solver_kind(self):
        """0 = PCG, 1 = dense direct, 2 = band direct."""
        return self._chk(self.lib.pus_get_linear_solver(self.h))

    def linear_solver_is_direct(self):
        return self.linear_solver_kind() == 1

    def set_direct_ordering(self, order):
        """Order of the band solve's pose tiles (kind 2 only): 0 insertion order (the default), 1 nested dissection."""
        if not isinstance(order, (int, np.integer)) or isinstance(order, bool) or int(order) not in (0, 1):
            raise ValueError(f"direct ordering: expected 0 (insertion order) or 1 (nested dissection), got {order!r}")
        self._chk(self.lib.pus_set_direct_ordering(self.h, int(order)))

    def direct_ordering(self):
        """0 = insertion order, 1 = nested dissection."""
        return self._chk(self.lib.pus_get_direct_ordering(self.h))

    def get_solver_options(self):
        o = SolverOptions()
        self._chk(self.lib.pus_get_solver_options(self.h, C.byref(o)))
        return o

    def set_solver_options(self, **kw):
        o = self.get_solver_options()
        for k, v in kw.items():
            if not hasattr(o, k):
                raise KeyError(k)
            setattr(o, k, v)
        self._chk(self.lib.pus_set_solver_options(self.h, C.byref(o)))

    def upload(self):
        self._chk(self.lib.pus_upload(self.h))

    def solve_resident(self):
        it = C.c_int(0)
        self._chk(self.lib.pus_solve_resident(self.h, C.byref(it)))
        return it.value

    def download(self):
        self._chk(self.lib.pus_download(self.h))

    def stats(self):
        s = Stats()
        self._chk(self.lib.pus_get_stats(self.h, C.byref(s)))
        return s.as_dict()

    def span_export(self):
        buf = C.create_string_buffer(64)
        fn = self.lib.pus_span_export
        fn.argtypes = [C.c_void_p, C.c_void_p]
        self._chk(fn(self.h, buf))
        return bytes(buf.raw)

    def span_connect(self, rank, world, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        fn = self.lib.pus_span_connect
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
        self._chk(fn(self.h, int(rank), int(world), blob))

    def span_optimize(self):
        it = C.c_int(0)
        fn = self.lib.pus_span_optimize
        fn.argtypes = [C.c_void_p, c_int_p]
        self._chk(fn(self.h, C.byref(it)))
        return it.value

    def span_disconnect(self):
        fn = self.lib.pus_span_disconnect
        fn.argtypes = [C.c_void_p]
        self._chk(fn(self.h))

    # -- weighted errors / stacked Jacobian at the current estimate (evaluated on the device) --
    def jacobian_dims(self):
        """(rows, columns) of the stacked system: the live factors' dims and the live nodes' dims."""
        r, c = C.c_longlong(0), C.c_longlong(0)
        self._chk(self.lib.pus_jacobian_dims(self.h, C.byref(r), C.byref(c)))
        return r.value, c.value

    def weighted_errors(self):
        """Slam::weighted_errors(): Factor::error of every live factor, stacked in factor order (numpy, float64)."""
        fn = self.lib.pus_weighted_errors
        fn.restype = C.c_longlong
        fn.argtypes = [C.c_void_p, c_double_p, C.c_longlong]
        rows = self._chk(fn(self.h, None, 0))
        out = np.zeros(rows)
        self._chk(fn(self.h, _dp(out), rows))
        return out

    def factor_errors(self, fids):
        """Factor::error of the given factors, their rows concatenated in the order of fids."""
        fids = _i32(np.atleast_1d(fids))
        out = np.zeros(6 * len(fids))
        fn = self.lib.pus_factor_errors
        fn.argtypes = [C.c_void_p, C.c_int, c_int_p, c_double_p]
        n = self._chk(fn(self.h, len(fids), _ip(fids), _dp(out)))
        return out[:n].copy()

    def jacobian(self):
        """Slam::jacobian() at the current estimate, in the handle's Jacobian mode: (scipy.sparse.csr_matrix, rhs), with
        rhs = Jacobian::rhs() = minus the residual rows."""
        import scipy.sparse as sp
        fn = self.lib.pus_jacobian
        fn.restype = C.c_longlong
        fn.argtypes = [C.c_void_p, c_int_p, c_int_p, c_double_p, c_double_p, C.c_longlong]
        rows, cols = self.jacobian_dims()
        nnz = self._chk(fn(self.h, None, None, None, None, 0))
        row_ptr = np.zeros(rows + 1, dtype=np.int32)
        col_idx = np.zeros(max(nnz, 1), dtype=np.int32)
        vals = np.zeros(max(nnz, 1))
        rhs = np.zeros(rows)
        self._chk(fn(self.h, _ip(row_ptr), _ip(col_idx), _dp(vals), _dp(rhs), nnz))
        return sp.csr_matrix((vals[:nnz], col_idx[:nnz], row_ptr), shape=(rows, cols)), rhs

    def normalized_chi2(self):
        out = C.c_double(0)
        self._chk(self.lib.pus_normalized_chi2(self.h, C.byref(out)))
        return out.value

    def local_chi2(self, last_n):
        out = C.c_double(0)
        self._chk(self.lib.pus_local_chi2(self.h, int(last_n), C.byref(out)))
        return out.value

    # -- marginal covariances at the current estimate (band solver in nested-dissection order only) --
    def marginal_covariances(self, ids):
        """Each node's own block of (J^T J)^-1 (6 x 6 per pose, 3 x 3 per plane), as a list of numpy arrays in ids order."""
        ids = _i32(np.atleast_1d(ids))
        dims = [self.node_dim(int(i)) for i in ids]
        out = np.zeros(max(1, sum(d * d for d in dims)))
        fn = self.lib.pus_marginal_covariances
        fn.argtypes = [C.c_void_p, C.c_int, c_int_p, c_double_p]
        self._chk(fn(self.h, len(ids), _ip(ids), _dp(out)))
        res, o = [], 0
        for d in dims:
            res.append(out[o:o + d * d].reshape(d, d).copy())
            o += d * d
        return res

    def covariance_blocks(self, pairs):
        """The cross blocks Sigma_ab of the (a, b) node pairs, as a list of dim(a) x dim(b) numpy arrays."""
        p = _i32(np.asarray(pairs).reshape(-1, 2))
        dims = [(self.node_dim(int(a)), self.node_dim(int(b))) for a, b in p]
        out = np.zeros(max(1, sum(a * b for a, b in dims)))
        fn = self.lib.pus_covariance_blocks
        fn.restype = C.c_longlong
        fn.argtypes = [C.c_void_p, C.c_int, c_int_p, c_double_p]
        self._chk(fn(self.h, len(p), _ip(np.ascontiguousarray(p.reshape(-1))), _dp(out)))
        res, o = [], 0
        for a, b in dims:
            res.append(out[o:o + a * b].reshape(a, b).copy())
            o += a * b
        return res

    def node_dim(self, id_):
        """6 for a live pose, 3 for a live plane."""
        buf = np.zeros(7)
        if self.lib.pus_get_pose(self.h, int(id_), _dp(buf)) >= 0:
            return 6
        if self.lib.pus_get_plane(self.h, int(id_), _dp(buf)) >= 0:
            return 3
        raise ApiError(f"bad node id {id_}")

    def debug_fetch(self, name, cap):
        out = np.zeros(int(cap))
        n = self.lib.pus_debug_fetch(self.h, name.encode(), _dp(out), C.c_longlong(int(cap)))
        if n < 0:
            raise ApiError((self.lib.pus_last_error() or b"?").decode())
        return out[:n]

    def debug_store(self, name, arr):
        a = _f64(arr).reshape(-1)
        n = self.lib.pus_debug_store(self.h, name.encode(), _dp(a), C.c_longlong(len(a)))
        if n < 0:
            raise ApiError((self.lib.pus_last_error() or b"?").decode())

    def debug_run_stage(self, stage, lam=0.0):
        self._chk(self.lib.pus_debug_run_stage(self.h, int(stage), float(lam)))

    PATH_BITS = ("resident", "tma", "tma_ring", "apply_smem", "apply_l2", "l3_local", "cluster", "res_listed_heavy",
                 "res_unlisted_heavy", "res_pose_pose_tail", "res_wide_block", "coarse_tail")

    def pcg_path(self):
        """The branches the kernel reported for the linear solve of the last debug launch: a dict of the PathBit flags
        (pus_kernels.cuh) plus the team size, the preconditioner levels, the hat spacing SP and the most pose blocks a CTA owns."""
        v = self.debug_fetch("path", 5).astype(int)
        d = {name: bool(v[0] >> i & 1) for i, name in enumerate(self.PATH_BITS)}
        d.update(team=int(v[1]), levels=int(v[2]), SP=int(v[3]), owned=int(v[4]))
        return d


def _handles(apis):
    arr = (C.c_void_p * len(apis))(*[a.h for a in apis])
    return arr


def batch_optimize_many(apis):
    lib = apis[0].lib
    its = np.zeros(len(apis), dtype=np.int32)
    rc = lib.pus_batch_optimize_many(_handles(apis), len(apis), _ip(its))
    if rc < 0:
        raise ApiError((lib.pus_last_error() or b"?").decode())
    return its


def span_emulate_optimize(apis):
    """one graph spanning len(apis) "ranks" emulated on one device (include/popup_gpu.h); every api holds the same graph"""
    lib = apis[0].lib
    it = C.c_int(0)
    rc = lib.pus_span_emulate_optimize(_handles(apis), len(apis), C.byref(it))
    if rc < 0:
        raise ApiError((lib.pus_last_error() or b"?").decode())
    return it.value


def upload_many(apis):
    rc = apis[0].lib.pus_upload_many(_handles(apis), len(apis))
    if rc < 0:
        raise ApiError((apis[0].lib.pus_last_error() or b"?").decode())


def solve_resident_many(apis):
    lib = apis[0].lib
    its = np.zeros(len(apis), dtype=np.int32)
    rc = lib.pus_solve_resident_many(_handles(apis), len(apis), _ip(its))
    if rc < 0:
        raise ApiError((lib.pus_last_error() or b"?").decode())
    return its


def download_many(apis):
    rc = apis[0].lib.pus_download_many(_handles(apis), len(apis))
    if rc < 0:
        raise ApiError((apis[0].lib.pus_last_error() or b"?").decode())


def popup_fit_frames(lib, seg_ptr, segs, invK, Ts, dist_thre=10.0, mode=0, prefix="pus_", device=0):
    """popup_plane::get_plane_equation batched over frames (include/popup_gpu.h)."""
    seg_ptr = _i32(seg_ptr)
    nf = len(seg_ptr) - 1
    segs = np.ascontiguousarray(segs, dtype=np.float32).reshape(-1, 4)
    invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
    Ts = np.ascontiguousarray(Ts, dtype=np.float32).reshape(nf, 4, 4)
    rows = int(seg_ptr[-1]) + nf
    pw = np.zeros((rows, 4), dtype=np.float32)
    ps = np.zeros((rows, 4), dtype=np.float32)
    dist = np.zeros(rows, dtype=np.float32)
    good = np.zeros(rows, dtype=np.int32)
    fn = getattr(lib, prefix + "popup_fit_frames")
    fn.argtypes = [C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_float_p, C.c_float, C.c_int, c_float_p,
                   c_float_p, c_float_p, c_int_p]
    rc = fn(device, nf, _ip(seg_ptr), segs.ctypes.data_as(c_float_p), invK.ctypes.data_as(c_float_p),
            Ts.ctypes.data_as(c_float_p), float(dist_thre), int(mode), pw.ctypes.data_as(c_float_p),
            ps.ctypes.data_as(c_float_p), dist.ctypes.data_as(c_float_p), _ip(good))
    if rc < 0:
        raise ApiError("popup_fit_frames failed")
    return pw, ps, dist, good


def popup_clouds(lib, plane_ptr, poly_ptr, polys, planes_sensor, Ts, invK, width, height, images=None, downsample=True,
                 depth_thre=5.0, ceiling_threshold=2.8, labels=False, points=True, capacity=None, prefix="pus_", device=0):
    """popup_plane::generate_cloud batched over frames and their planes (pus_popup_clouds, include/popup_gpu.h).

    plane_ptr [n_frames+1] and poly_ptr [n_planes+1] are CSR offsets; polys [n_vertices, 2] float pixels; planes_sensor
    [n_planes, 4]; Ts [n_frames, 4, 4] camera-to-world; images [n_frames, height, width, 3] uint8 BGR or None.
    Returns a dict: counts [n_planes] int32, offsets [n_planes] int64, xyz [total, 3] float32 and rgb [total, 3] uint8
    (absent with points=False: a size query), labels [n_frames, height, width] uint8 (with labels=True).  Without a
    capacity (in points) a size query runs first; with one, a single call fills buffers of that size."""
    plane_ptr = _i32(plane_ptr)
    nf = len(plane_ptr) - 1
    npl = int(plane_ptr[-1])
    poly_ptr = _i32(poly_ptr)
    polys = np.ascontiguousarray(polys, dtype=np.float32).reshape(-1, 2)
    planes_sensor = np.ascontiguousarray(planes_sensor, dtype=np.float32).reshape(-1, 4)
    Ts = np.ascontiguousarray(Ts, dtype=np.float32).reshape(nf, 4, 4)
    invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
    u8p = C.POINTER(C.c_ubyte)
    img = None if images is None else np.ascontiguousarray(images, dtype=np.uint8).reshape(nf, height, width, 3)
    counts = np.zeros(npl, np.int32)
    offsets = np.zeros(npl, np.int64)
    lab = np.zeros((nf, height, width), np.uint8) if labels else None
    fn = getattr(lib, prefix + "popup_clouds")
    fn.restype = C.c_longlong
    fn.argtypes = [C.c_int, C.c_int, c_int_p, c_int_p, c_float_p, c_float_p, c_float_p, c_float_p, u8p, C.c_int, C.c_int,
                   C.c_int, C.c_float, C.c_float, c_int_p, C.POINTER(C.c_longlong), c_float_p, u8p, C.c_longlong, u8p]
    err = getattr(lib, prefix + "last_error", None) or getattr(lib, prefix + "popup_last_error")
    err.restype = C.c_char_p

    def call(xyz, rgb, cap):
        n = fn(device, nf, _ip(plane_ptr), _ip(poly_ptr), polys.ctypes.data_as(c_float_p),
               planes_sensor.ctypes.data_as(c_float_p), Ts.ctypes.data_as(c_float_p), invK.ctypes.data_as(c_float_p),
               None if img is None else img.ctypes.data_as(u8p), int(width), int(height), int(bool(downsample)),
               float(depth_thre), float(ceiling_threshold), _ip(counts), offsets.ctypes.data_as(C.POINTER(C.c_longlong)),
               None if xyz is None else xyz.ctypes.data_as(c_float_p), None if rgb is None else rgb.ctypes.data_as(u8p),
               int(cap), None if lab is None else lab.ctypes.data_as(u8p))
        if n < 0:
            raise ApiError((err() or b"?").decode())
        return n

    out = {"counts": counts, "offsets": offsets}
    if not points:
        total = call(None, None, 0)
    else:
        cap = call(None, None, 0) if capacity is None else int(capacity)
        xyz, rgb = np.empty((cap, 3), np.float32), np.empty((cap, 3), np.uint8)
        total = call(xyz, rgb, cap)
        out.update(xyz=xyz[:total], rgb=rgb[:total])
    out["total"] = total
    if labels:
        out["labels"] = lab
    return out


def popup_polygons(lib, seg_ptr, segs, K, invK, Ts, width, height, ceiling_threshold=2.5, walllength_threshold=3.0,
                   vertices=True, capacity=None, prefix="pus_", device=0):
    """popup_plane::find_2d_3d_closed_polygon batched over frames (pus_popup_polygons, include/popup_gpu.h).

    seg_ptr [n_frames+1] CSR offsets, segs [n_seg, 4] float pixels, K and invK [3, 3], Ts [n_frames, 4, 4]
    camera-to-world.  Rows as popup_fit_frames'.  Returns a dict with, for each of "bound" (2-D, to the image border),
    "cut" (2-D, the cut polygon projected back) and "world" (3-D, cut, on the wall): <name>_counts [n_rows] int32,
    <name>_ptr [n_rows+1] int32 CSR offsets and, unless vertices=False (a size query), <name> [total, 2 or 3] float32.
    bound_ptr / bound or cut_ptr / cut are the poly_ptr / polys of popup_clouds.  capacity = (bound, cut, world) in
    vertices fills buffers of that size instead of the queried ones."""
    seg_ptr = _i32(seg_ptr)
    nf = len(seg_ptr) - 1
    n_rows = int(seg_ptr[-1]) + nf
    segs = np.ascontiguousarray(segs, dtype=np.float32).reshape(-1, 4)
    K = np.ascontiguousarray(K, dtype=np.float32).reshape(3, 3)
    invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
    Ts = np.ascontiguousarray(Ts, dtype=np.float32).reshape(nf, 4, 4)
    cnt = {k: np.zeros(n_rows, np.int32) for k in ("bound", "cut", "world")}
    fn = getattr(lib, prefix + "popup_polygons")
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_float,
                   C.c_float, c_int_p, c_int_p, c_int_p, c_float_p, c_float_p, c_float_p, C.c_longlong, C.c_longlong,
                   C.c_longlong]
    err = getattr(lib, prefix + "last_error", None) or getattr(lib, prefix + "popup_last_error")
    err.restype = C.c_char_p

    def call(out, caps):
        rc = fn(device, nf, _ip(seg_ptr), segs.ctypes.data_as(c_float_p), K.ctypes.data_as(c_float_p),
                invK.ctypes.data_as(c_float_p), Ts.ctypes.data_as(c_float_p), int(width), int(height),
                float(ceiling_threshold), float(walllength_threshold), _ip(cnt["bound"]), _ip(cnt["cut"]), _ip(cnt["world"]),
                *[None if o is None else o.ctypes.data_as(c_float_p) for o in out], *[int(c) for c in caps])
        if rc < 0:
            raise ApiError((err() or b"?").decode())

    call((None, None, None), (0, 0, 0))
    res = {}
    for k in cnt:
        res[k + "_counts"] = cnt[k].copy()
        res[k + "_ptr"] = np.concatenate([[0], np.cumsum(cnt[k])]).astype(np.int32)
    if vertices:
        tot = [int(res[k + "_ptr"][-1]) for k in cnt]
        cap = tot if capacity is None else [int(c) for c in capacity]
        out = (np.empty((cap[0], 2), np.float32), np.empty((cap[1], 2), np.float32), np.empty((cap[2], 3), np.float32))
        call(out, cap)
        res.update(bound=out[0][:tot[0]], cut=out[1][:tot[1]], world=out[2][:tot[2]])
    return res


def popup_depth(lib, plane_ptr, poly_ptr, polys, planes_sensor, Ts, invK, width, height, downsample=True,
                ceiling_threshold=2.8, prefix="pus_", device=0):
    """popup_plane::get_depth_map_good batched over frames (pus_popup_depth, include/popup_gpu.h).

    The inputs are popup_clouds': plane_ptr [n_frames+1] and poly_ptr [n_planes+1] CSR offsets, polys [n_vertices, 2] the
    planes' closed 2-D bound polygons (popup_polygons' bound_ptr / bound of the good rows), planes_sensor [n_planes, 4],
    Ts [n_frames, 4, 4] camera-to-world, invK [3, 3].  Returns the depth maps [n_frames, height, width] float32."""
    plane_ptr = _i32(plane_ptr)
    nf = len(plane_ptr) - 1
    poly_ptr = _i32(poly_ptr)
    polys = np.ascontiguousarray(polys, dtype=np.float32).reshape(-1, 2)
    planes_sensor = np.ascontiguousarray(planes_sensor, dtype=np.float32).reshape(-1, 4)
    Ts = np.ascontiguousarray(Ts, dtype=np.float32).reshape(nf, 4, 4)
    invK = np.ascontiguousarray(invK, dtype=np.float32).reshape(3, 3)
    out = np.empty((nf, int(height), int(width)), np.float32)
    fn = getattr(lib, prefix + "popup_depth")
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, c_int_p, c_int_p, c_float_p, c_float_p, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                   C.c_float, c_float_p]
    err = getattr(lib, prefix + "last_error", None) or getattr(lib, prefix + "popup_last_error")
    err.restype = C.c_char_p
    rc = fn(device, nf, _ip(plane_ptr), _ip(poly_ptr), polys.ctypes.data_as(c_float_p), planes_sensor.ctypes.data_as(c_float_p),
            Ts.ctypes.data_as(c_float_p), invK.ctypes.data_as(c_float_p), int(width), int(height), int(bool(downsample)),
            float(ceiling_threshold), out.ctypes.data_as(c_float_p))
    if rc < 0:
        raise ApiError((err() or b"?").decode())
    return out


class EdgeParams(C.Structure):
    """pus_edge_params (include/popup_gpu.h)"""
    _fields_ = [("dilation_distance", C.c_int), ("erosion_distance", C.c_int), ("downsample_contour", C.c_int)] + [
        (k, C.c_double) for k in (
            "pre_vertical_thre", "pre_minium_len", "pre_boundary_thre", "pre_contour_close_thre", "pre_merge_angle_thre",
            "pre_merge_dist_thre", "pre_proj_angle_thre", "pre_proj_cover_thre", "pre_proj_cover_large_thre",
            "pre_proj_dist_thre", "interval_overlap_thre", "post_short_thre", "post_bind_dist_thre", "post_merge_dist_thre",
            "post_merge_angle_thre", "post_extend_thre")]


# popup_plane's member defaults (popup_plane.h:178-200, popup_plane.cpp:32-33) with popup_param.yaml's downsample_contour.
# main_3d loads popup_param.yaml over the members, which changes four of them: post_short_thre 20, post_bind_dist_thre 15,
# post_merge_dist_thre 10, post_extend_thre 50 (popup_tum_far.yaml: downsample_contour off, pre_contour_close_thre 400,
# post_bind_dist_thre 30, post_merge_dist_thre 50, post_merge_angle_thre 20, post_extend_thre 0).  Pass those as params to
# follow a launch file.
EDGE_DEFAULTS = dict(dilation_distance=11, erosion_distance=11, downsample_contour=1, pre_vertical_thre=15.0,
                     pre_minium_len=15.0, pre_boundary_thre=5.0, pre_contour_close_thre=50.0, pre_merge_angle_thre=10.0,
                     pre_merge_dist_thre=10.0, pre_proj_angle_thre=20.0, pre_proj_cover_thre=0.6,
                     pre_proj_cover_large_thre=0.8, pre_proj_dist_thre=100.0, interval_overlap_thre=20.0,
                     post_short_thre=30.0, post_bind_dist_thre=10.0, post_merge_dist_thre=20.0, post_merge_angle_thre=10.0,
                     post_extend_thre=15.0)


def popup_edges(lib, labels, line_ptr, lines, params=None, segments=True, capacity=None, prefix="pus_", device=0):
    """popup_plane::edge_get_polygons batched over frames (pus_popup_edges, include/popup_gpu.h).

    labels [n_frames, height, width] uint8 (ground 255), line_ptr [n_frames+1] CSR offsets, lines [n, 4] float pixels,
    params a dict over EDGE_DEFAULTS (None: the defaults).  Returns a dict: status, open_counts, connect_counts [n_frames]
    int32, open_ptr / connect_ptr [n_frames+1] and, unless segments=False (a size query), open [.., 4], connect [.., 4]
    float32 and open_in_connect int32.  open_ptr / open are the seg_ptr / segs of popup_fit_frames and popup_polygons.
    capacity = (open, connect) in rows fills buffers of that size instead of the queried ones."""
    labels = np.ascontiguousarray(labels, dtype=np.uint8)
    nf, h, w = labels.shape
    line_ptr = _i32(line_ptr)
    lines = np.ascontiguousarray(lines, dtype=np.float32).reshape(-1, 4)
    P = EdgeParams(**dict(EDGE_DEFAULTS, **(params or {})))
    st, oc, cc = (np.zeros(nf, np.int32) for _ in range(3))
    fn = getattr(lib, prefix + "popup_edges")
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, c_int_p, c_float_p, C.POINTER(EdgeParams), c_int_p,
                   c_int_p, c_int_p, c_float_p, c_float_p, c_int_p, C.c_longlong, C.c_longlong]
    err = getattr(lib, prefix + "last_error", None) or getattr(lib, prefix + "popup_last_error")
    err.restype = C.c_char_p

    def call(o, c, i, caps):
        rc = fn(device, nf, labels.ctypes.data, w, h, _ip(line_ptr), lines.ctypes.data_as(c_float_p), C.byref(P), _ip(st),
                _ip(oc), _ip(cc), *[None if a is None else a.ctypes.data_as(c_float_p) for a in (o, c)],
                None if i is None else _ip(i), *[int(x) for x in caps])
        if rc < 0:
            raise ApiError((err() or b"?").decode())

    call(None, None, None, (0, 0))
    res = dict(status=st.copy(), open_counts=oc.copy(), connect_counts=cc.copy(),
               open_ptr=np.concatenate([[0], np.cumsum(oc)]).astype(np.int32),
               connect_ptr=np.concatenate([[0], np.cumsum(cc)]).astype(np.int32))
    if segments:
        tot = (int(res["open_ptr"][-1]), int(res["connect_ptr"][-1]))
        cap = tot if capacity is None else [int(c) for c in capacity]
        o, c, i = np.empty((cap[0], 4), np.float32), np.empty((cap[1], 4), np.float32), np.empty(max(cap[0], 0), np.int32)
        call(o, c, i, cap)
        res.update(open=o[:tot[0]], connect=c[:tot[1]], open_in_connect=i[:tot[0]])
    return res


def popup_lines(lib, images, downsample=False, lines=True, capacity=None, prefix="pus_", device=0):
    """popup_plane::get_ground_edges' line detection (grey, contrast, EDLines) batched over frames (pus_popup_lines,
    include/popup_gpu.h).

    images [n_frames, height, width, 3] uint8 BGR or [n_frames, height, width] grey.  Returns a dict: status, counts
    [n_frames] int32, line_ptr [n_frames+1] and, unless lines=False (a size query), lines [total, 4] float32 -- line_ptr
    and lines are popup_edges' arguments as they are.  capacity (rows) fills a buffer of that size instead."""
    images = np.ascontiguousarray(images, dtype=np.uint8)
    if images.ndim not in (3, 4):
        raise ValueError("images must be [n, h, w] or [n, h, w, c]")
    nf, h, w = images.shape[:3]
    ch = 1 if images.ndim == 3 else images.shape[3]
    st, cnt = np.zeros(nf, np.int32), np.zeros(nf, np.int32)
    fn = getattr(lib, prefix + "popup_lines")
    fn.restype = C.c_longlong
    fn.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, c_int_p, c_int_p, c_float_p,
                   C.c_longlong]
    err = getattr(lib, prefix + "last_error", None) or getattr(lib, prefix + "popup_last_error")
    err.restype = C.c_char_p

    def call(out, cap):
        rc = fn(device, nf, images.ctypes.data if images.size else None, w, h, ch, int(bool(downsample)), _ip(st),
                _ip(cnt), None if out is None else out.ctypes.data_as(c_float_p), int(cap))
        if rc < 0:
            raise ApiError((err() or b"?").decode())
        return rc

    total = call(None, 0)
    res = dict(status=st.copy(), counts=cnt.copy(), line_ptr=np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32))
    if lines:
        cap = total if capacity is None else int(capacity)
        out = np.empty((max(cap, 0), 4), np.float32)
        call(out, cap)
        res["lines"] = out[:total]
    return res


class PopupConfig(C.Structure):
    """pus_popup_config (include/popup_gpu.h)"""
    _fields_ = [("K", C.c_float * 9), ("invK", C.c_float * 9), ("width", C.c_int), ("height", C.c_int),
                ("channels", C.c_int), ("fast_edges", C.c_int), ("edges", EdgeParams), ("plane_cam_dist_thre", C.c_float),
                ("ceiling_threshold", C.c_float), ("walllength_threshold", C.c_float), ("downsample_poly", C.c_int),
                ("depth_thre", C.c_float), ("want_rgb", C.c_int), ("want_labels", C.c_int), ("want_depth", C.c_int)]


# (field, dtype, per-element shape, length as a function of the result's counts)
_FRAME_OUTPUTS = [
    ("status", np.int32, (), "n"), ("line_status", np.int32, (), "n"), ("line_counts", np.int32, (), "n"),
    ("edge_status", np.int32, (), "n"), ("open_ptr", np.int32, (), "n1"), ("connect_ptr", np.int32, (), "n1"),
    ("open_segs", np.float32, (4,), "n_open"), ("connect_segs", np.float32, (4,), "n_connect"),
    ("open_in_connect", np.int32, (), "n_open"), ("planes_world", np.float32, (4,), "n_rows"),
    ("planes_sensor", np.float32, (4,), "n_rows"), ("dist", np.float32, (), "n_rows"), ("good", np.int32, (), "n_rows"),
    ("bound_ptr", np.int32, (), "rows1"), ("cut_ptr", np.int32, (), "rows1"), ("world_ptr", np.int32, (), "rows1"),
    ("bound2d", np.float32, (2,), "n_bound"), ("cut2d", np.float32, (2,), "n_cut"), ("world3d", np.float32, (3,), "n_world"),
    ("good_ptr", np.int32, (), "n1"), ("good_rows", np.int32, (), "n_good"), ("plane_status", np.int32, (), "n_good"),
    ("cloud_counts", np.int32, (), "n_good"), ("cloud_offsets", np.int64, (), "n_good"),
    ("xyz", np.float32, (3,), "n_points"), ("rgb", np.uint8, (3,), "n_points"), ("labels", np.uint8, ("h", "w"), "n"),
    ("depth", np.float32, ("h", "w"), "n")]
_CT = {np.int32: C.c_int, np.float32: C.c_float, np.int64: C.c_longlong, np.uint8: C.c_ubyte}


class PopupFrameResult(C.Structure):
    """pus_popup_frames (include/popup_gpu.h)"""
    _fields_ = [("n_frames", C.c_int), ("n_rows", C.c_int), ("n_good", C.c_int)] + [
        (k, C.c_longlong) for k in ("n_open", "n_connect", "n_bound", "n_cut", "n_world", "n_points")] + [
        (k, C.POINTER(_CT[t])) for k, t, _, _ in _FRAME_OUTPUTS]


def popup_config(config):
    """a PopupConfig from a dict (see PopupFrames)"""
    c = dict(fast_edges=0, edges=None, plane_cam_dist_thre=10.0, ceiling_threshold=5.0, walllength_threshold=3.0,
             downsample_poly=1, depth_thre=10.0, want_rgb=None, want_labels=0, want_depth=0)
    c.update(config)
    if c["want_rgb"] is None:
        c["want_rgb"] = int(c["channels"] == 3)
    cfg = PopupConfig()
    cfg.K[:] = [float(v) for v in np.asarray(c["K"], np.float32).ravel()]
    cfg.invK[:] = [float(v) for v in np.asarray(c["invK"], np.float32).ravel()]
    for k in ("width", "height", "channels", "fast_edges", "downsample_poly", "want_rgb", "want_labels", "want_depth"):
        setattr(cfg, k, int(c[k]))
    for k in ("plane_cam_dist_thre", "ceiling_threshold", "walllength_threshold", "depth_thre"):
        setattr(cfg, k, float(c[k]))
    cfg.edges = EdgeParams(**dict(EDGE_DEFAULTS, **(c["edges"] or {})))
    return cfg


class PopupFrames:
    """A pop-up session (pus_popup_session_*, include/popup_gpu.h): main_3d's per-frame pop-up over batches of frames.

    config: K, invK [3, 3], width, height, channels (3 BGR, 1 grey) and optionally fast_edges, edges (a dict over
    EDGE_DEFAULTS), plane_cam_dist_thre (10), ceiling_threshold (5), walllength_threshold (3), downsample_poly (True),
    depth_thre (10), want_rgb (True with BGR), want_labels, want_depth (False).  run(images, labels, Ts) takes numpy arrays
    and returns a dict of numpy arrays, or torch CUDA tensors and returns torch CUDA tensors, ordered on torch's current
    stream."""

    def __init__(self, lib, config, device=0):
        self.lib = lib
        cfg = popup_config(config)
        self.config = cfg
        vp = C.c_void_p
        lib.pus_popup_session_create.argtypes = [C.c_int, C.POINTER(PopupConfig), C.POINTER(vp)]
        lib.pus_popup_session_destroy.argtypes = [vp]
        lib.pus_popup_session_set_stream.argtypes = [vp, vp]
        lib.pus_popup_session_run.argtypes = [vp, C.c_int, vp, vp, vp]
        lib.pus_popup_session_result.argtypes = [vp, C.POINTER(PopupFrameResult)]
        lib.pus_popup_session_download.argtypes = [vp, C.POINTER(PopupFrameResult)]
        lib.pus_popup_session_memory.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
        lib.pus_last_error.restype = C.c_char_p
        self.h = vp()
        self._check(lib.pus_popup_session_create(int(device), C.byref(cfg), C.byref(self.h)))

    def _check(self, rc):
        if rc < 0:
            raise ApiError((self.lib.pus_last_error() or b"?").decode())
        return rc

    def close(self):
        if self.h:
            self.lib.pus_popup_session_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def memory(self):
        """(allocations made so far, bytes reserved) of the session's device and pinned buffers"""
        a, b = C.c_longlong(), C.c_longlong()
        self._check(self.lib.pus_popup_session_memory(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def _check_shapes(self, img, lab, T):
        """the library reads n frames of the configured size from each input: refuse arrays of another shape"""
        c, n = self.config, img[0] if len(img) else -1
        want = (n, c.height, c.width) + ((c.channels,) if c.channels == 3 else ())
        if tuple(img) != want and not (c.channels == 1 and tuple(img) == want + (1,)):
            raise ValueError(f"images must be {want}, not {tuple(img)}")
        if tuple(lab) != (n, c.height, c.width):
            raise ValueError(f"labels must be {(n, c.height, c.width)}, not {tuple(lab)}")
        if tuple(T) not in ((n, 4, 4), (n, 16)):
            raise ValueError(f"Ts must be ({n}, 4, 4), not {tuple(T)}")

    def run(self, images, labels, Ts):
        torch_in = type(images).__module__.startswith("torch")
        if torch_in:
            import torch
            for t in (images, labels, Ts):
                if not (t.is_cuda and t.is_contiguous()):
                    raise ValueError("torch inputs must be contiguous CUDA tensors")
            if images.dtype != torch.uint8 or labels.dtype != torch.uint8 or Ts.dtype != torch.float32:
                raise ValueError("images and labels must be uint8, Ts float32")
            n = images.shape[0]
            self._check_shapes(tuple(images.shape), tuple(labels.shape), tuple(Ts.shape))
            self._check(self.lib.pus_popup_session_set_stream(self.h, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            ptrs = [t.data_ptr() or None for t in (images, labels, Ts)]
        else:
            images = np.ascontiguousarray(images, np.uint8)
            labels = np.ascontiguousarray(labels, np.uint8)
            Ts = np.ascontiguousarray(Ts, np.float32)
            n = images.shape[0]
            self._check_shapes(images.shape, labels.shape, Ts.shape)
            self._check(self.lib.pus_popup_session_set_stream(self.h, None))
            ptrs = [a.ctypes.data if a.size else None for a in (images, labels, Ts)]
        self._check(self.lib.pus_popup_session_run(self.h, int(n), *ptrs))
        res = PopupFrameResult()
        self._check(self.lib.pus_popup_session_result(self.h, C.byref(res)))
        cfg = self.config
        size = dict(n=res.n_frames, n1=res.n_frames + 1, rows1=res.n_rows + 1, n_rows=res.n_rows, n_good=res.n_good,
                    n_open=res.n_open, n_connect=res.n_connect, n_bound=res.n_bound, n_cut=res.n_cut, n_world=res.n_world,
                    n_points=res.n_points, h=cfg.height, w=cfg.width)
        dst, out = PopupFrameResult(), {}
        for k, t, shape, count in _FRAME_OUTPUTS:
            if not getattr(res, k):
                continue
            shp = (int(size[count]),) + tuple(int(size[s]) if isinstance(s, str) else s for s in shape)
            if torch_in:
                a = torch.empty(shp, dtype=getattr(torch, np.dtype(t).name), device=images.device)
                p = a.data_ptr()
            else:
                a = np.empty(shp, t)
                p = a.ctypes.data
            if a.numel() if torch_in else a.size:
                setattr(dst, k, C.cast(C.c_void_p(p), C.POINTER(_CT[t])))
            out[k] = a
        self._check(self.lib.pus_popup_session_download(self.h, C.byref(dst)))
        return out


# ---- plane map (pus_map_*, include/popup_gpu.h) ------------------------------------------------------------------------
class MapConfig(C.Structure):
    """pus_map_config (include/popup_gpu.h)"""
    _fields_ = [("edge_asso_2ddist", C.c_double), ("edge_asso_proj", C.c_double), ("edge_asso_angle", C.c_double),
                ("edge_asso_planedist", C.c_double), ("assoc_near_frames", C.c_int), ("pose_sigmas", C.c_double * 6),
                ("plane_sigmas", C.c_double * 3), ("plane_sigma_dist_mul", C.c_double), ("init_wTo", C.c_double * 16),
                ("invK", C.c_float * 9)]


class MapLandmark(C.Structure):
    """pus_map_landmark (include/popup_gpu.h)"""
    _fields_ = [(k, C.c_int) for k in ("node", "deleted", "frame_seq_id", "frame_plane_indice", "good_plane_indice",
                                       "being_tracked_times")] + [
        ("plane_dist_cam", C.c_double), ("n_bound2d", C.c_int), ("n_world3d", C.c_int),
        ("bound2d", (C.c_float * 2) * 2), ("world3d", (C.c_float * 3) * 2)]


class MapFrame(C.Structure):
    """pus_map_frame (include/popup_gpu.h)"""
    _fields_ = [("seq_id", C.c_int), ("odom7", C.c_void_p), ("session", C.c_void_p), ("frame", C.c_int), ("n_planes", C.c_int),
                ("planes_sensor", C.c_void_p), ("dist", C.c_void_p), ("plane_indice", C.c_void_p), ("bound_ptr", C.c_void_p),
                ("bound2d", C.c_void_p), ("world_ptr", C.c_void_p), ("world3d", C.c_void_p), ("n_segs", C.c_int),
                ("segs", C.c_void_p)]


class MapResult(C.Structure):
    """pus_map_result (include/popup_gpu.h)"""
    _fields_ = [("capacity", C.c_int), ("n_planes", C.c_int), ("pose_node", C.c_int), ("n_new", C.c_int),
                ("lm_iterations", C.c_int)] + [(k, C.POINTER(C.c_int)) for k in ("landmark", "status", "factor", "new_nodes")] + [
        ("error", C.POINTER(C.c_double))]


# main_3d.cpp:368-376: the TUM fr3 "no texture far" first pose from ground truth (camera-to-world)
TUM_FAR_INIT_WTO = [-0.4563, 0.2444, -0.8556, -1.2432, 0.8898, 0.1249, -0.4388, 1.9219, -0.0004, -0.9616, -0.2745, 1.0547,
                    0, 0, 0, 1]
# pop_planar_slam/params/plane_3d_tum_far.yaml: the covering and 2-D gates disabled
MAP_PRESET_TUM_FAR = dict(edge_asso_2ddist=10000.0, edge_asso_proj=-1.0, edge_asso_angle=35.0, edge_asso_planedist=2.0,
                          assoc_near_frames=1000, pose_sigmas=[2.0] * 6, plane_sigmas=[0.05] * 3, plane_sigma_dist_mul=2.0)
# pop_planar_slam/src/Mapping.h:72-94: the in-class values, every gate enabled
MAP_PRESET_MAPPING_H = dict(edge_asso_2ddist=50.0, edge_asso_proj=0.5, edge_asso_angle=60.0, edge_asso_planedist=4.0,
                            assoc_near_frames=5, pose_sigmas=[0.001, 0.001, 0.001, 0.01, 0.01, 0.01], plane_sigmas=[0.001] * 3,
                            plane_sigma_dist_mul=3.0)
MAP_PRESETS = {"tum_far": MAP_PRESET_TUM_FAR, "mapping_h": MAP_PRESET_MAPPING_H}


def map_config(preset, invK, init_wTo=TUM_FAR_INIT_WTO, **over):
    """A pus_map_config from a preset name ("tum_far" or "mapping_h"), the camera's invK and the first pose; keyword
    arguments replace preset values."""
    v = dict(MAP_PRESETS[preset], **over)
    c = MapConfig()
    for k in ("edge_asso_2ddist", "edge_asso_proj", "edge_asso_angle", "edge_asso_planedist", "plane_sigma_dist_mul"):
        setattr(c, k, float(v[k]))
    c.assoc_near_frames = int(v["assoc_near_frames"])
    c.pose_sigmas[:] = [float(x) for x in v["pose_sigmas"]]
    c.plane_sigmas[:] = [float(x) for x in v["plane_sigmas"]]
    c.init_wTo[:] = [float(x) for x in np.asarray(init_wTo, np.float64).reshape(16)]
    c.invK[:] = [float(x) for x in np.asarray(invK, np.float32).reshape(9)]
    return c


class PlaneMap:
    """A plane map (pus_map_*): Mapper_mono::processFrame on the device, bound to a GpuGraphAPI handle.

    config: a MapConfig (map_config(preset, invK)).  predict_pose() -> (T [4, 4] float32, odom7); process_frame(seq_id,
    planes=dict(planes_sensor [n, 4], dist [n], plane_indice [n], bound [list of [k, 2]], world [list of [k, 3]],
    segs [m, 4]) or session=(PopupFrames, frame), odom7=None) -> dict of the per-plane and per-frame results;
    landmarks() -> a numpy structured array of the table."""

    def __init__(self, api, config):
        self.api, self.lib = api, api.lib
        self.lib.pus_map_create.argtypes = [C.c_void_p, C.POINTER(MapConfig), C.POINTER(C.c_void_p)]
        self.lib.pus_map_destroy.argtypes = [C.c_void_p]
        self.lib.pus_map_predict_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.pus_map_process_frame.argtypes = [C.c_void_p, C.POINTER(MapFrame), C.POINTER(MapResult)]
        self.lib.pus_map_landmarks.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.config = config
        h = C.c_void_p()
        self._check(self.lib.pus_map_create(api.h, C.byref(config), C.byref(h)))
        self.h = h

    def _check(self, rc):
        if rc < 0:
            raise ApiError(self.lib.pus_last_error().decode())
        return rc

    def close(self):
        if getattr(self, "h", None):
            self.lib.pus_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict_pose(self, T_out=None):
        """T_out: None (a host array is returned) or a torch CUDA tensor of 16 float32 written in place"""
        odom = np.zeros(7)
        if T_out is not None:
            self._check(self.lib.pus_map_predict_pose(self.h, C.c_void_p(T_out.data_ptr()), odom.ctypes.data))
            return T_out, odom
        T = np.zeros(16, np.float32)
        self._check(self.lib.pus_map_predict_pose(self.h, T.ctypes.data, odom.ctypes.data))
        return T.reshape(4, 4), odom

    @staticmethod
    def _ptr(a):
        if a is None:
            return None
        return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data

    def process_frame(self, seq_id, planes=None, session=None, odom7=None, capacity=None):
        f = MapFrame()
        f.seq_id = int(seq_id)
        keep = []
        if odom7 is not None:
            o = np.ascontiguousarray(odom7, np.float64)
            keep.append(o)
            f.odom7 = o.ctypes.data
        if session is not None:
            sess, frame = session
            f.session, f.frame = sess.h, int(frame)
            n_cap = capacity or 1024
        else:
            arrs = self._arrays(planes)
            keep.append(arrs)
            f.n_planes = int(len(arrs["planes_sensor"]))
            f.n_segs = int(len(arrs["segs"]))
            for k in ("planes_sensor", "dist", "plane_indice", "bound_ptr", "bound2d", "world_ptr", "world3d", "segs"):
                setattr(f, k, self._ptr(arrs[k]))
            n_cap = capacity or max(f.n_planes, 1)
        out = {k: np.zeros(n_cap, np.int32) for k in ("landmark", "status", "factor", "new_nodes")}
        out["error"] = np.zeros(n_cap)
        r = MapResult()
        r.capacity = n_cap
        for k in ("landmark", "status", "factor", "new_nodes"):
            setattr(r, k, out[k].ctypes.data_as(C.POINTER(C.c_int)))
        r.error = out["error"].ctypes.data_as(C.POINTER(C.c_double))
        self._check(self.lib.pus_map_process_frame(self.h, C.byref(f), C.byref(r)))
        n = r.n_planes
        res = {k: out[k][:n].copy() for k in ("landmark", "status", "factor", "error")}
        res.update(new_nodes=out["new_nodes"][:r.n_new].copy(), n_planes=n, pose_node=r.pose_node, n_new=r.n_new,
                   lm_iterations=r.lm_iterations)
        return res

    @staticmethod
    def _arrays(p):
        """numpy (host) or torch CUDA (device) arrays of one frame's planes, CSR-packed"""
        if "bound_ptr" in p:
            return p
        lens = lambda polys: np.concatenate([[0], np.cumsum([len(x) for x in polys])]).astype(np.int32)
        cat = lambda polys, d: (np.concatenate([np.asarray(x, np.float32).reshape(-1, d) for x in polys])
                                if sum(len(x) for x in polys) else np.zeros((0, d), np.float32))
        return dict(planes_sensor=np.ascontiguousarray(p["planes_sensor"], np.float32).reshape(-1, 4),
                    dist=np.ascontiguousarray(p["dist"], np.float32), plane_indice=np.ascontiguousarray(p["plane_indice"], np.int32),
                    bound_ptr=lens(p["bound"]), bound2d=np.ascontiguousarray(cat(p["bound"], 2)),
                    world_ptr=lens(p["world"]), world3d=np.ascontiguousarray(cat(p["world"], 3)),
                    segs=np.ascontiguousarray(p["segs"], np.float32).reshape(-1, 4))

    def landmarks(self):
        n = self._check(self.lib.pus_map_landmarks(self.h, 0, None))
        buf = (MapLandmark * max(n, 1))()
        self._check(self.lib.pus_map_landmarks(self.h, n, buf))
        return np.ctypeslib.as_array(buf)[:n].copy()
