"""CPU tests of the closed wall and ground polygons (pus_popup_polygons): the oracle tests/popup_polygon_oracle.cpp
against the fixture tests/golden/popup_polygons.npz, which a separately written numpy + live-cv2 restatement
(tools/make_popup_polygon_golden.py) made, bit for bit; the oracle's convex hull and point-in-polygon test against live
cv2; the fixture's branch coverage; the geometry of the oracle's output checked in float64 against the fitted planes; and
the C-ABI's refusals, which need no GPU."""
import os

import numpy as np
import pytest

import popup_polygon_native as N
from pop_up_slam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def point_set(rng, t):
    n = int(rng.integers(1, 35))
    kind = t % 5
    if kind == 0:
        p = rng.uniform(-50, 50, (n, 2))
    elif kind == 1:   # integer grid: duplicates, collinear runs, points on edges
        p = rng.integers(-4, 5, (n, 2)).astype(float)
    elif kind == 2:   # a duplicated half
        p = rng.integers(-3, 4, (n, 2)).astype(float)
        p[: n // 2] = p[0]
    elif kind == 3:   # an exactly collinear run
        p = np.outer(rng.integers(-5, 6, n), rng.integers(-3, 4, 2) / 4.0) + rng.integers(-4, 4, 2)
    else:             # a box with points on its edges and crossings, as the cut sees them
        x0, x1, c = -1.0, float(rng.integers(1, 8)), float(rng.integers(1, 5))
        e = [(x0, -1), (x1, -1), (x1, c), (x0, c)]
        e += [(rng.uniform(x0, x1), -1.0) for _ in range(n // 3)] + [(x1, rng.uniform(-1, c)) for _ in range(n // 3)]
        e += list(rng.uniform([x0, -1], [x1, c], (n // 3, 2)))
        p = np.array(e, float)
    return p.astype(np.float32)


def test_oracle_hull_and_point_test_equal_live_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    for t in range(3000):
        p = point_set(rng, t)
        want = cv2.convexHull(p.reshape(-1, 1, 2)).reshape(-1, 2)
        np.testing.assert_array_equal(N.hull(p).view(np.uint32), want.view(np.uint32), err_msg=f"{t} {p.tolist()}")
        contour = np.concatenate([p, p[:1]]) if t % 2 else p
        for q in (p[int(rng.integers(len(p)))], (p[0] + p[-1]) / 2, rng.uniform(-50, 50, 2)):
            q = np.asarray(q, np.float32)
            assert N.point_polygon_test(contour, q) == cv2.pointPolygonTest(contour.reshape(-1, 1, 2), (float(q[0]), float(q[1])),
                                                                            False), (t, contour.tolist(), q.tolist())


GOLDEN = os.path.join(ROOT, "tests", "golden", "popup_polygons.npz")


def fixture_cases():
    """(batch kwargs for capi.popup_polygons, expected dict) per setting of tests/golden/popup_polygons.npz"""
    g = np.load(GOLDEN)
    for c in range(int(g["n_cases"])):
        d = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(f"{c}/")}
        w, h, ceiling, walllength = d["setting"]
        b = dict(seg_ptr=d["seg_ptr"], segs=d["segs"], K=d["K"], invK=d["invK"], Ts=d["Ts"], width=int(w), height=int(h),
                 ceiling_threshold=float(ceiling), walllength_threshold=float(walllength))
        yield b, d


def test_oracle_equals_the_fixture():
    n = 0
    for b, d in fixture_cases():
        r = capi.popup_polygons(N.oracle_lib(), prefix="orc_", **b)
        for k in ("bound", "cut", "world"):
            np.testing.assert_array_equal(r[k + "_counts"], d[k + "_counts"], err_msg=f"{b['width']} {k}")
            # both are float32 with every operation rounded: identical bits
            np.testing.assert_array_equal(r[k].view(np.uint32), d[k].view(np.uint32), err_msg=f"{b['width']} {k}")
        n += len(b["seg_ptr"]) - 1
    assert n >= 72


def test_fixture_reaches_every_branch():
    seen = set()
    for b, _ in fixture_cases():
        seen |= set(map(tuple, N.codes(b).tolist()))
    for A in range(5):   # ground: both segments' five cases, the quirk branch (first segment, case 2) included
        assert any(c[0] == 0 and c[1] == A for c in seen), ("last", A)
        assert any(c[0] == 0 and c[2] == A for c in seen), ("first", A)
    for kind in (1, 3):   # leftmost and rightmost walls: both edge branches with every inner case, and the general split
        for outer in (0, 1):
            assert {0, 1, 2} <= {c[2] for c in seen if c[:2] == (kind, outer)}, (kind, outer)
        assert any(c[:2] == (kind, 2) for c in seen), kind
    assert {0, 1, 2, 3, 4} <= {c[2] for c in seen if c[0] > 0 and c[1] == 2}
    cut = {c[3] for c in seen if c[0] > 0}
    assert {0, 1, 2} <= {c % 4 for c in cut} and any(c >= 4 for c in cut), cut   # both modes, both ends, the fallback


def ground_ends64(b, f, s):
    """the world ground endpoints of segment s of frame f, in float64"""
    T = b["Ts"][f].astype(np.float64)
    out = []
    for k in range(2):
        r = T[:3, :3] @ np.linalg.inv(b["K"].astype(np.float64)) @ [*b["segs"][b["seg_ptr"][f] + s][2 * k:2 * k + 2], 1.0]
        p = T[:3, 3] + (-T[2, 3] / r[2]) * r
        out.append(np.array([p[0], p[1], 0.0]))
    return out


def test_oracle_geometry_in_float64():
    import oracle_api
    for i, ((w, h), c, l) in enumerate(N.SETTINGS):
        rng = np.random.default_rng(100 + i)
        b = N.batch([N.random_frame(rng, w, h) for _ in range(25)] + [N.corner_frame(rng, w, h) for _ in range(5)], w, h, c, l)
        r = capi.popup_polygons(N.oracle_lib(), prefix="orc_", **b)
        planes_world = capi.popup_fit_frames(oracle_api.oracle_lib(), b["seg_ptr"], b["segs"], b["invK"], b["Ts"],
                                             prefix="orc_")[0].astype(np.float64)
        K = b["K"].astype(np.float64)
        cds = N.codes(b)
        for f in range(len(b["seg_ptr"]) - 1):
            s0, s1 = b["seg_ptr"][f], b["seg_ptr"][f + 1]
            T = b["Ts"][f].astype(np.float64)
            for j in range(s1 - s0 + 1):
                row = s0 + f + j
                bd = r["bound"][r["bound_ptr"][row]:r["bound_ptr"][row + 1]].astype(np.float64)
                cut = r["cut"][r["cut_ptr"][row]:r["cut_ptr"][row + 1]].astype(np.float64)
                wd = r["world"][r["world_ptr"][row]:r["world_ptr"][row + 1]].astype(np.float64)
                assert len(bd) >= 3 and (bd[0] == bd[-1]).all()
                if j == 0:
                    assert len(wd) == 0 and np.array_equal(cut, bd)
                    continue
                seg = b["segs"][s0 + j - 1]
                assert (bd[0] == seg[:2]).all() and (bd[1] == seg[2:]).all()
                assert len(wd) == len(cut) >= 3
                scale = max(1.0, np.abs(wd).max())
                # every 3-D vertex lies on the row's fitted wall plane (the fallback's too)
                pl = planes_world[row]
                assert np.abs(wd @ pl[:3] + pl[3]).max() < 1e-4 * scale * np.linalg.norm(pl[:3]), row
                sensor = (wd - T[:3, 3]) @ T[:3, :3]
                proj = sensor @ K.T
                proj = proj[:, :2] / proj[:, 2:]
                np.testing.assert_allclose(cut, proj, rtol=1e-3, atol=1e-2)
                if cds[row, 3] >= 4:   # the uncut fallback: its closing vertex keeps the z the first one loses
                    continue
                assert (wd[0] == wd[-1]).all() and (cut[0] == cut[-1]).all()
                assert wd[:, 2].min() > -1e-4 * scale and wd[:, 2].max() < c + 1e-4 * scale
                if l >= 0:   # along the ground line from the nearer endpoint: [-1, l] ahead of it, or [-l, 1] from the end
                    e0, e1 = ground_ends64(b, f, j - 1)
                    u = (e1 - e0) / np.linalg.norm(e1 - e0)
                    x = (wd - e0) @ u
                    lo, hi = (-1.0, l) if cds[row, 3] == 1 else ((e1 - e0) @ u - l, (e1 - e0) @ u + 1.0)
                    tol = 1e-4 * scale
                    assert x.min() > lo - tol and x.max() < hi + tol, (row, cds[row, 3], x, lo, hi)


def _args(**over):
    b = N.batch([(np.array([[0, 400, 300, 380], [300, 380, 639, 420]], np.float32), np.eye(4, dtype=np.float32))],
                640, 480, 2.5, 3.0)
    b.update(over)
    return b


@pytest.mark.parametrize("over,msg", [
    (dict(seg_ptr=[1, 2]), "seg_ptr"),
    (dict(seg_ptr=[0, 2, 1], Ts=np.eye(4, dtype=np.float32)[None].repeat(2, 0)), "not ascending"),
    (dict(segs=np.array([[0, 400, np.nan, 380], [300, 380, 639, 420]], np.float32)), "not finite"),
    (dict(segs=np.array([[0, 400, 5e6, 380], [300, 380, 639, 420]], np.float32)), "PUS_POPUP_MAX_COORD"),
    (dict(K=np.full((3, 3), np.inf, np.float32)), "K and invK"),
    (dict(invK=np.full((3, 3), np.nan, np.float32)), "K and invK"),
    (dict(Ts=np.full((1, 4, 4), np.nan, np.float32)), "Ts"),
    (dict(width=1), "at least 2"),
    (dict(height=0), "at least 2"),
    (dict(seg_ptr=[0, 251], segs=np.tile(np.array([[0, 400, 300, 380]], np.float32), (251, 1))), "PUS_POPUP_MAX_SEGMENTS"),
])
def test_bad_arguments_are_refused(over, msg):
    with pytest.raises(capi.ApiError, match=msg):
        capi.popup_polygons(capi.load_library(), **_args(**over))


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_no_cpu_fallback_without_a_gpu():
    with pytest.raises(capi.ApiError, match="no CUDA device"):
        capi.popup_polygons(capi.load_library(), **_args())
