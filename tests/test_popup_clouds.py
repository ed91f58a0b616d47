"""CPU tests of the dense plane clouds (pus_popup_clouds): the oracle tests/popup_cloud_oracle.cpp against the OpenCV-made
fixture tests/golden/popup_clouds.npz (tools/make_popup_cloud_golden.py) and, where cv2 imports, against a live
cv2.fillConvexPoly / findNonZero run; and the C-ABI's refusals, which need no GPU."""
import os

import numpy as np
import pytest

import popup_cloud_native as N
from pop_up_slam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "popup_clouds.npz")


def cases():
    g = np.load(GOLDEN)
    for c in range(int(g["n_cases"])):
        yield c, {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(f"{c}/")}, g


def run_case(lib, d, g, prefix, device=0, **kw):
    w, h, ds, with_img = (int(v) for v in d["size"])
    frame = int(kw.pop("frame", 0))
    img = N.image(frame, w, h)[None] if with_img else None
    return capi.popup_clouds(lib, [0, len(d["planes"])], d["poly_ptr"], d["polys"], d["planes"], d["T"][None], d["invK"], w, h,
                             images=img, downsample=bool(ds), depth_thre=float(g["depth_thre"]),
                             ceiling_threshold=float(g["ceiling_threshold"]), labels=True, prefix=prefix, device=device, **kw)


def test_oracle_pixel_lists_equal_the_opencv_fixture():
    n = 0
    for c, d, _ in cases():
        ds = bool(d["size"][2])
        for p, want in enumerate(N.fixture_pixels(d["boxes"], d["masks"], ds)):
            got = N.oracle_pixels(d["polys"][d["poly_ptr"][p]:d["poly_ptr"][p + 1]], ds)
            np.testing.assert_array_equal(got, want, err_msg=f"case {c} plane {p}")
            n += len(want)
    assert n > 20000


def test_oracle_pixel_lists_equal_live_opencv():
    cv2 = pytest.importorskip("cv2")
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_popup_cloud_golden", os.path.join(ROOT, "tools", "make_popup_cloud_golden.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    rng = np.random.default_rng(7)
    for t in range(3000):
        w, h = (640, 480) if t % 2 else (960, 540)
        kind = N.KINDS[t % len(N.KINDS)]
        poly = np.asarray(N._polygon(rng, kind, w, h), np.float32).reshape(-1, 2)
        if t % 7 == 0:   # small boxes with fractional, negative and integral corners
            poly = (rng.integers(-20, 20, size=poly.shape) + rng.choice([0, 0.5, -0.5, 0.999], size=poly.shape)).astype(np.float32)
        ds = bool(t % 3)
        np.testing.assert_array_equal(N.oracle_pixels(poly, ds), tool.cv_pixels(poly, ds), err_msg=f"{t} {kind} {poly.tolist()}")
    assert cv2.__version__


def test_oracle_points_labels_equal_the_fixture():
    orc = N.oracle_lib()
    for c, d, g in cases():
        r = run_case(orc, d, g, "orc_", frame=c)
        np.testing.assert_array_equal(r["counts"], d["counts"], err_msg=f"case {c}")
        np.testing.assert_array_equal(r["offsets"], np.cumsum(np.r_[0, d["counts"][:-1]]))
        # both are float32 with every operation rounded (no contraction): identical bits
        np.testing.assert_array_equal(r["xyz"].view(np.uint32), d["xyz"].view(np.uint32), err_msg=f"case {c}")
        np.testing.assert_array_equal(r["rgb"], d["rgb"], err_msg=f"case {c}")
        np.testing.assert_array_equal(r["labels"][0], d["labels"], err_msg=f"case {c}")


def _args(**over):
    a = dict(plane_ptr=[0, 1], poly_ptr=[0, 3], polys=np.array([[10, 10], [50, 10], [30, 40]], np.float32),
             planes_sensor=np.array([[0, -1, 0, 1]], np.float32), Ts=np.eye(4, dtype=np.float32)[None], invK=N.invK(640, 480),
             width=640, height=480)
    a.update(over)
    return a


@pytest.mark.parametrize("over,msg", [
    (dict(width=0), "width and height"),
    (dict(plane_ptr=[1, 1]), "plane_ptr"),
    (dict(poly_ptr=[0, 300], polys=np.zeros((300, 2), np.float32)), "PUS_POPUP_MAX_VERTICES"),
    (dict(polys=np.array([[10, 10], [np.nan, 10], [30, 40]], np.float32)), "not finite"),
    (dict(polys=np.array([[10, 10], [5e6, 10], [30, 40]], np.float32)), "PUS_POPUP_MAX_COORD"),
    (dict(width=641, labels=True), "even width"),
])
def test_bad_arguments_are_refused(over, msg):
    lib = capi.load_library()
    kw = _args(**over)
    labels = kw.pop("labels", False)
    with pytest.raises(capi.ApiError, match=msg):
        capi.popup_clouds(lib, labels=labels, **kw)


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_no_cpu_fallback_without_a_gpu():
    with pytest.raises(capi.ApiError, match="no CUDA device"):
        capi.popup_clouds(capi.load_library(), **_args())
