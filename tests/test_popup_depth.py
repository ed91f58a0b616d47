"""CPU tests of the pop-up depth map (pus_popup_depth): the oracle tests/popup_depth_oracle.cpp against the fixture
tests/golden/popup_depth.npz (tools/make_popup_depth_golden.py, an independent numpy restatement on OpenCV's own fill and
resize), the fixture's branch coverage, the oracle's resize chain against live cv2, and the C-ABI's refusals, which need
no GPU."""
import os

import numpy as np
import pytest

import popup_cloud_native as NC
import popup_depth_native as N
from pop_up_slam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "popup_depth.npz")


def fixture_cases():
    """(popup_depth kwargs, expected maps) per setting of the fixture"""
    g = np.load(GOLDEN)
    for c in range(int(g["n_cases"])):
        w, h, ds, ceiling = g[f"{c}/setting"]
        b = {k: g[f"{c}/{k}"] for k in ("plane_ptr", "poly_ptr", "polys", "planes_sensor", "Ts", "invK")}
        b.update(width=int(w), height=int(h), downsample=bool(ds), ceiling_threshold=float(ceiling))
        yield b, g[f"{c}/depth"]


def same_bits(a, b, msg=""):
    assert a.shape == b.shape, msg
    nan = np.isnan(a)
    np.testing.assert_array_equal(nan, np.isnan(b), err_msg=msg)
    np.testing.assert_array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32), err_msg=msg)


def test_oracle_equals_the_fixture():
    for b, want in fixture_cases():
        same_bits(capi.popup_depth(N.oracle_lib(), prefix="orc_", **b), want, str((b["downsample"], b["ceiling_threshold"])))


def test_fixture_reaches_every_branch():
    seen, settings = {}, set()
    for b, want in fixture_cases():
        settings.add(b["downsample"])
        code, off = N.codes(b)
        src = code & 0xffff
        seen["plane"] = seen.get("plane", 0) + int(((src > 0) & ~(code & N.CEILING).astype(bool)).sum())
        seen["ceiling"] = seen.get("ceiling", 0) + int(((src > 0) & (code & N.CEILING).astype(bool)).sum())
        for name, flag in (("depth_skip_kept", N.DEPTH_SKIP | N.KEPT_AFTER_SKIP), ("ceiling_skip", N.CEILING_SKIP),
                           ("overwrite", N.OVERWRITTEN)):
            seen[name] = seen.get(name, 0) + int(((code & flag) == flag).sum())
        seen["untouched"] = seen.get("untouched", 0) + int((code == 0).sum())
        seen["off_image"] = seen.get("off_image", 0) + off
        n = np.diff(b["poly_ptr"])
        seen["empty_polygon"] = seen.get("empty_polygon", 0) + int((n == 0).sum())
        seen["no_planes"] = seen.get("no_planes", 0) + int((np.diff(b["plane_ptr"]) == 0).sum())
        assert (want[np.diff(b["plane_ptr"]) == 0] == 0).all()
    assert settings == {True, False}
    assert all(v > 0 for v in seen.values()), seen


def _maps(rng, n, sparse):
    h, w = 2 * int(rng.integers(1, 70)), 2 * int(rng.integers(1, 90))
    m = np.zeros((h, w), np.float32)
    keep = rng.random((h, w)) < (0.5 if not sparse else 1.0)
    m[keep] = rng.uniform(-2, 12, keep.sum()).astype(np.float32)
    special = rng.random((h, w))
    for lo, v in ((0.0, np.inf), (0.02, np.nan), (0.04, -0.0), (0.06, np.float32(1e-41)), (0.08, -np.inf)):
        m[(special >= lo) & (special < lo + 0.02)] = v
    if sparse:   # downsample mode: only even pixels are written
        e = np.zeros_like(m)
        e[0::2, 0::2] = m[0::2, 0::2]
        m = e
    return m


def test_oracle_resize_chain_equals_live_opencv():
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        rng = np.random.default_rng(11)
        for t in range(200):
            m = _maps(rng, t, sparse=bool(t % 2))
            want = cv2.resize(cv2.resize(m, None, fx=0.5, fy=0.5) * np.float32(4) + np.float32(0), None, fx=2, fy=2)
            same_bits(N.resize_chain(m), want, f"map {t} {m.shape}")
    finally:
        cv2.ipp.setUseIPP(ipp)


def _args(**over):
    a = dict(plane_ptr=[0, 1], poly_ptr=[0, 3], polys=np.array([[10, 10], [50, 10], [30, 40]], np.float32),
             planes_sensor=np.array([[0, -1, 0, 1]], np.float32), Ts=np.eye(4, dtype=np.float32)[None], invK=NC.invK(640, 480),
             width=640, height=480)
    a.update(over)
    return a


@pytest.mark.parametrize("over,msg", [
    (dict(width=0), "width and height"),
    (dict(plane_ptr=[1, 1]), "plane_ptr"),
    (dict(plane_ptr=[0, 2, 1], Ts=np.stack([np.eye(4, dtype=np.float32)] * 2)), "plane_ptr is not ascending"),
    (dict(poly_ptr=[0, 300], polys=np.zeros((300, 2), np.float32)), "PUS_POPUP_MAX_VERTICES"),
    (dict(polys=np.array([[10, 10], [np.nan, 10], [30, 40]], np.float32)), "not finite"),
    (dict(polys=np.array([[10, 10], [5e6, 10], [30, 40]], np.float32)), "PUS_POPUP_MAX_COORD"),
    (dict(width=641), "even width"),
    (dict(height=479), "even width"),
])
def test_bad_arguments_are_refused(over, msg):
    with pytest.raises(capi.ApiError, match=msg):
        capi.popup_depth(capi.load_library(), **_args(**over))


def test_odd_sizes_are_accepted_without_downsample():
    try:
        capi.popup_depth(capi.load_library(), downsample=False, **_args(width=641, height=479))
    except capi.ApiError as e:
        assert "no CUDA device" in str(e)


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_no_cpu_fallback_without_a_gpu():
    with pytest.raises(capi.ApiError, match="no CUDA device"):
        capi.popup_depth(capi.load_library(), **_args())
