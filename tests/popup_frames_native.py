"""Test-side helpers for the pop-up session (pus_popup_session_*): main_3d's per-frame chain composed from the stage calls
with the glue restated in Python (the rule of INTEGRATION.md), seeded rendered rooms, and the reference's sample frames.
Test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import oracle_api
import popup_depth_native as ND
import popup_edges_native as NE
import popup_lines_native as NL
import popup_polygon_native as NP
from pop_up_slam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_LINES, MAX_SEGMENTS = 512, 250

# main_3d's settings (main_3d.cpp:417-454, popup_plane's members)
MAIN_3D = dict(plane_cam_dist_thre=10.0, ceiling_threshold=5.0, walllength_threshold=3.0, downsample_poly=1, depth_thre=10.0)


_lib = None


def oracle_lib():
    """tests/popup_frames_oracle.cpp (the session's glue header compiled for the host) linked against the stage oracles,
    built once per session into a temporary directory"""
    global _lib
    if _lib is None:
        stages = [NL.oracle_lib(), NE.oracle_lib(), oracle_api.oracle_lib(), NP.oracle_lib(), ND.oracle_lib()]
        out = os.path.join(tempfile.mkdtemp(prefix="popup_frames_"), "liborc_frames.so")
        subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-Wall",
                               "-I/usr/local/cuda/include", os.path.join(ROOT, "tests", "popup_frames_oracle.cpp"), "-o", out]
                              + [os.path.abspath(lib._name) for lib in stages])
        _lib = C.CDLL(out)
        _lib.orc_popup_frames_run.argtypes = [C.POINTER(capi.PopupConfig), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_popup_frames_result.argtypes = [C.POINTER(capi.PopupFrameResult)]
        _lib.orc_popup_frames_last_error.restype = C.c_char_p
    return _lib


def oracle_run(cfg, images, labels, Ts):
    """the whole run through the host oracle: a dict shaped as capi.PopupFrames.run's"""
    lib = oracle_lib()
    pc = capi.popup_config(cfg)
    images, labels = np.ascontiguousarray(images, np.uint8), np.ascontiguousarray(labels, np.uint8)
    Ts = np.ascontiguousarray(Ts, np.float32)
    if lib.orc_popup_frames_run(C.byref(pc), len(labels), images.ctypes.data, labels.ctypes.data, Ts.ctypes.data) < 0:
        raise capi.ApiError(lib.orc_popup_frames_last_error().decode())
    r = capi.PopupFrameResult()
    lib.orc_popup_frames_result(C.byref(r))
    size = dict(n=r.n_frames, n1=r.n_frames + 1, rows1=r.n_rows + 1, n_rows=r.n_rows, n_good=r.n_good, n_open=r.n_open,
                n_connect=r.n_connect, n_bound=r.n_bound, n_cut=r.n_cut, n_world=r.n_world, n_points=r.n_points,
                h=pc.height, w=pc.width)
    optional = dict(rgb=pc.want_rgb, labels=pc.want_labels, depth=pc.want_depth)
    out = {}
    for k, t, shape, count in capi._FRAME_OUTPUTS:
        if not optional.get(k, 1):
            continue
        shp = (int(size[count]),) + tuple(int(size[x]) if isinstance(x, str) else x for x in shape)
        ptr = getattr(r, k)
        out[k] = (np.ctypeslib.as_array(ptr, shape=shp).copy() if ptr and int(np.prod(shp)) else np.zeros(shp, t))
    return out


def config(width, height, channels=3, **over):
    K = NP.camera_K(width, height)
    c = dict(K=K, invK=np.linalg.inv(K.astype(np.float64)).astype(np.float32), width=width, height=height,
             channels=channels, fast_edges=0, edges=None, want_rgb=int(channels == 3), want_labels=0, want_depth=0,
             **MAIN_3D)
    c.update(over)
    return c


def room(rng, width, height, dark=False):
    """a rendered room: the camera and ground polyline of popup_polygon_native.random_frame, a label map of 255 on and
    below the polyline, and a textured BGR image with a floor colour below it and a colour per wall above it"""
    segs, T = NP.random_frame(rng, width, height)
    xs = np.arange(width, dtype=np.float64)
    yline = np.full(width, np.nan)
    for x1, y1, x2, y2 in segs.astype(np.float64):
        m = (xs >= min(x1, x2)) & (xs <= max(x1, x2))
        yline[m] = y1 + (y2 - y1) * (xs[m] - x1) / max(x2 - x1, 1e-9)
    x0, x1 = segs[0, 0], segs[-1, 2]
    yline[xs < x0] = segs[0, 1]
    yline[xs > x1] = segs[-1, 3]
    ys = np.arange(height, dtype=np.float64)[:, None]
    ground = ys >= yline[None, :]
    lab = np.where(ground, 255, 0).astype(np.uint8)
    img = np.empty((height, width, 3), np.int16)
    wall_of = np.searchsorted(segs[:, 2], xs)   # the wall above each column
    colours = rng.integers(60, 230, (len(segs) + 1, 3))
    img[:] = colours[np.minimum(wall_of, len(segs))][None, :, :]
    img[ground] = rng.integers(20, 120, 3)
    img += rng.integers(-8, 9, img.shape).astype(np.int16)
    img = np.clip(img, 0, 255).astype(np.uint8)
    if dark:
        img = (img * 0.4).astype(np.uint8)   # below a mean of 90: the equalizeHist branch
    return img, lab, T


def rooms(seed, n, width, height):
    rng = np.random.default_rng(seed)
    out = [room(rng, width, height, dark=(i % 5 == 3)) for i in range(n)]
    return (np.array([o[0] for o in out]), np.array([o[1] for o in out]),
            np.array([o[2] for o in out], np.float32).reshape(n, 4, 4))


def samples():
    """the reference's four sample frames, each [1, h, w, 3] BGR, [1, h, w] label map and [1, 4, 4] seeded pose (their sizes
    differ)"""
    import cv2
    d = os.path.join(ROOT, "tests", "golden", "popup_lines_frames")
    out = []
    for i, k in enumerate(NL.G.SAMPLES):
        img = cv2.imread(os.path.join(d, f"rgb_{k}.png"))
        lab = cv2.imread(os.path.join(d, f"label_{k}.png"), cv2.IMREAD_GRAYSCALE)
        Ts = NP.random_batch(21 + i, 1, img.shape[1], img.shape[0], 5.0, 3.0)["Ts"]
        out.append((img[None], lab[None], Ts))
    return out


def actual_filter(good, open_ptr, open_in_connect):
    """get_plane_equation's filter (popup_plane.cpp:629-635) with actual_plane_indices_inall = {0} u
    {open_in_connect + 1} (:792-794): open wall s of a frame stays good only when s is one of its open_in_connect values"""
    good = good.copy()
    for f in range(len(open_ptr) - 1):
        o0, o1 = int(open_ptr[f]), int(open_ptr[f + 1])
        inc = set(int(v) for v in open_in_connect[o0:o1])
        for s in range(o1 - o0):
            if s not in inc:
                good[o0 + f + 1 + s] = 0
    return good


def chain(libs, images, labels, Ts, cfg, prefix="pus_"):
    """the session's outputs composed from the stage calls (libs: lines, edges, fit, polygons, clouds, depth)"""
    ll, el, fl, pl, cl, dl = libs
    n, h, w = labels.shape
    L = capi.popup_lines(ll, images, downsample=bool(cfg["fast_edges"]), prefix=prefix)
    cnt, lines = L["counts"], L["lines"].reshape(-1, 4)
    ptr = L["line_ptr"]
    status = np.zeros(n, np.int32)
    for f in range(n):
        if cnt[f] > MAX_LINES or not np.isfinite(lines[ptr[f]:ptr[f + 1]]).all():
            status[f] = 1
    ecnt = np.where(status == 0, cnt, 0)
    elines = np.concatenate([lines[ptr[f]:ptr[f + 1]] for f in range(n) if status[f] == 0] + [np.zeros((0, 4), np.float32)])
    e = capi.popup_edges(el, labels, np.concatenate([[0], np.cumsum(ecnt)]).astype(np.int32), elines,
                         params=cfg.get("edges"), prefix=prefix)
    edge_status = np.where(status == 1, -1, e["status"]).astype(np.int32)
    status[(status == 0) & (e["open_counts"] > MAX_SEGMENTS)] = 2
    keep = status == 0
    op, cp = e["open_ptr"], e["connect_ptr"]
    pick = lambda a, p: np.concatenate([a[p[f]:p[f + 1]] for f in range(n) if keep[f]] + [a[:0]])   # noqa: E731
    oc, cc = np.where(keep, e["open_counts"], 0), np.where(keep, e["connect_counts"], 0)
    open_ptr = np.concatenate([[0], np.cumsum(oc)]).astype(np.int32)
    out = dict(status=status, line_status=L["status"], line_counts=cnt, edge_status=edge_status, open_ptr=open_ptr,
               connect_ptr=np.concatenate([[0], np.cumsum(cc)]).astype(np.int32), open_segs=pick(e["open"], op),
               connect_segs=pick(e["connect"], cp), open_in_connect=pick(e["open_in_connect"], op))
    K, invK = cfg["K"], cfg["invK"]
    pw, ps, dist, good = capi.popup_fit_frames(fl, open_ptr, out["open_segs"], invK, Ts, cfg["plane_cam_dist_thre"], 0,
                                               prefix=prefix)
    good = actual_filter(good, open_ptr, out["open_in_connect"])
    out.update(planes_world=pw, planes_sensor=ps, dist=dist, good=good)
    poly = capi.popup_polygons(pl, open_ptr, out["open_segs"], K, invK, Ts, w, h, cfg["ceiling_threshold"],
                               cfg["walllength_threshold"], prefix=prefix)
    out.update(bound_ptr=poly["bound_ptr"], cut_ptr=poly["cut_ptr"], world_ptr=poly["world_ptr"], bound2d=poly["bound"],
               cut2d=poly["cut"], world3d=poly["world"])
    src = "cut" if cfg["walllength_threshold"] > 0 else "bound"
    good_ptr, good_rows, rows = [0], [], []
    for f in range(n):
        r0 = open_ptr[f] + f
        g = [j for j in range(open_ptr[f + 1] - open_ptr[f] + 1) if good[r0 + j]] if oc[f] > 0 else []
        good_rows += g
        rows += [r0 + j for j in g]
        good_ptr.append(len(good_rows))
    out.update(good_ptr=np.array(good_ptr, np.int32), good_rows=np.array(good_rows, np.int32),
               plane_status=np.zeros(len(rows), np.int32))

    def polys(kind):
        p, v = poly[kind + "_ptr"], poly[kind]
        return (np.concatenate([[0], np.cumsum([p[r + 1] - p[r] for r in rows])]).astype(np.int32),
                np.concatenate([v[p[r]:p[r + 1]] for r in rows] + [np.zeros((0, 2), np.float32)]))

    planes = ps[rows].reshape(-1, 4)
    cptr, cpoly = polys(src)
    cl_ = capi.popup_clouds(cl, good_ptr, cptr, cpoly, planes, Ts, invK, w, h, images=images if images.ndim == 4 else None,
                            downsample=bool(cfg["downsample_poly"]), depth_thre=cfg["depth_thre"],
                            ceiling_threshold=cfg["ceiling_threshold"], labels=bool(cfg["want_labels"]), prefix=prefix)
    out.update(cloud_counts=cl_["counts"], cloud_offsets=cl_["offsets"], xyz=cl_["xyz"])
    if cfg["want_rgb"]:
        out["rgb"] = cl_["rgb"]
    if cfg["want_labels"]:
        out["labels"] = cl_["labels"]
    if cfg["want_depth"]:
        bptr, bpoly = polys("bound")
        out["depth"] = capi.popup_depth(dl, good_ptr, bptr, bpoly, planes, Ts, invK, w, h,
                                        downsample=bool(cfg["downsample_poly"]), ceiling_threshold=cfg["ceiling_threshold"],
                                        prefix=prefix)
    return out


def assert_same(got, want, keys=None, where=""):
    for k in keys or want:
        a, b = np.ascontiguousarray(np.asarray(got[k])), np.ascontiguousarray(np.asarray(want[k]))
        assert a.shape == b.shape and a.dtype == b.dtype, (where, k, a.shape, b.shape, a.dtype, b.dtype)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (where, k)
