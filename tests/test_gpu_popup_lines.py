"""pus_popup_lines on the device against the CPU oracle (tests/popup_lines_oracle.cpp): the fixture frames, seeded
64-frame batches at 640x480 and 960x540 with 1 and 3 channels and downsampling on and off, batch against frame-by-frame
calls, repeated calls, size queries, capacities and refusals, the >512-line frame, and the sample frames' chain
images + labels -> lines -> edges -> fit -> polygons.  Comparisons are on bit patterns."""
import os

import numpy as np
import pytest

import oracle_api
import popup_edges_native as NE
import popup_lines_native as N
import popup_polygon_native as NP
from pop_up_slam_b200 import capi
from test_popup_lines import same

pytestmark = pytest.mark.gpu


def test_fixture_frames_match():
    lib = capi.load_library()
    for key, imgs, ds, want in N.fixture():
        same(capi.popup_lines(lib, imgs, downsample=ds), want, key)


@pytest.mark.parametrize("size", [(640, 480), (960, 540)])
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("down", [0, 1])
def test_random_batches_match_the_oracle(size, channels, down):
    lib, orc = capi.load_library(), N.oracle_lib()
    imgs = N.random_batch(size[0] + 10 * channels + down, 64, *size, channels)
    got = capi.popup_lines(lib, imgs, downsample=down)
    same(got, capi.popup_lines(orc, imgs, downsample=down, prefix="orc_"), (size, channels, down))
    assert got["counts"].sum() > 64


def test_batch_equals_frame_by_frame_and_repeats():
    lib = capi.load_library()
    imgs = N.random_batch(5, 10, 640, 480, 3)
    whole = capi.popup_lines(lib, imgs)
    same(capi.popup_lines(lib, imgs), whole, "repeat")
    for f in range(len(imgs)):
        one = capi.popup_lines(lib, imgs[f:f + 1])
        a, b = whole["line_ptr"][f], whole["line_ptr"][f + 1]
        assert one["status"][0] == whole["status"][f]
        assert np.array_equal(one["lines"].view(np.uint32), whole["lines"][a:b].view(np.uint32))
    half = [capi.popup_lines(lib, imgs[:4]), capi.popup_lines(lib, imgs[4:])]
    assert np.array_equal(np.concatenate([h["lines"] for h in half]).view(np.uint32), whole["lines"].view(np.uint32))


def test_size_query_capacity_and_refusals():
    lib = capi.load_library()
    imgs = N.random_batch(6, 4, 640, 480, 1)
    q = capi.popup_lines(lib, imgs, lines=False)
    full = capi.popup_lines(lib, imgs)
    assert np.array_equal(q["counts"], full["counts"]) and "lines" not in q
    same(capi.popup_lines(lib, imgs, capacity=len(full["lines"]) + 7), full)
    with pytest.raises(capi.ApiError, match="capacity"):
        capi.popup_lines(lib, imgs, capacity=len(full["lines"]) - 1)
    with pytest.raises(capi.ApiError, match="channels"):
        capi.popup_lines(lib, np.zeros((1, 8, 8, 4), np.uint8))
    with pytest.raises(capi.ApiError, match="even"):
        capi.popup_lines(lib, np.zeros((1, 9, 8), np.uint8), downsample=True)
    with pytest.raises(capi.ApiError, match="3 x 3"):
        capi.popup_lines(lib, np.zeros((1, 4, 8), np.uint8), downsample=True)


def test_many_lines_come_back_whole_and_edges_still_refuse_them():
    lib = capi.load_library()
    key, imgs, ds, want = [f for f in N.fixture() if f[0] == "crafted_many"][0]
    got = capi.popup_lines(lib, imgs, downsample=ds)
    same(got, want)
    assert got["counts"][0] > 512   # PUS_POPUP_MAX_LINES
    lab = np.zeros((1,) + imgs.shape[1:3], np.uint8)
    with pytest.raises(capi.ApiError):
        capi.popup_edges(lib, lab, got["line_ptr"], got["lines"])


def test_sample_chain_lines_edges_fit_polygons():
    """the reference's four sample frames from image and label map: lines -> edges -> fit -> polygons on the device, and
    the same chain through the oracles (each stage fed by its own side's previous stage)"""
    import cv2
    lib = capi.load_library()
    orcs = (N.oracle_lib(), NE.oracle_lib(), oracle_api.oracle_lib(), NP.oracle_lib())
    pb = NP.random_batch(21, 1, 640, 480, 2.5, 3.0)
    d = os.path.join(N.ROOT, "tests", "golden", "popup_lines_frames")
    opened = 0
    for n in N.G.SAMPLES:
        img = cv2.imread(os.path.join(d, f"rgb_{n}.png"))
        lab = cv2.imread(os.path.join(d, f"label_{n}.png"), cv2.IMREAD_GRAYSCALE)
        h, w = lab.shape
        assert img.shape[:2] == (h, w)
        outs = []
        for (ll, el, fl, pl), pre in (((lib,) * 4, "pus_"), (orcs, "orc_")):
            L = capi.popup_lines(ll, img[None], prefix=pre)
            assert L["status"][0] == 0 and 0 < L["counts"][0] <= 512, n
            e = capi.popup_edges(el, lab[None], L["line_ptr"], L["lines"], prefix=pre)
            fit = capi.popup_fit_frames(fl, e["open_ptr"], e["open"], pb["invK"], pb["Ts"][:1], 10.0, 0, prefix=pre)
            poly = capi.popup_polygons(pl, e["connect_ptr"], e["connect"], pb["K"], pb["invK"], pb["Ts"][:1], w, h,
                                       prefix=pre)
            outs.append((L, e, fit, poly))
        (L, e, fit, poly), (L2, e2, fit2, poly2) = outs
        same(L, L2, n)
        for k in ("status", "open_counts", "connect_counts", "open", "connect", "open_in_connect"):
            assert np.array_equal(np.asarray(e[k]).view(np.uint8), np.asarray(e2[k]).view(np.uint8)), (n, k)
        for a, c in zip(fit, fit2):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(c).view(np.uint8)), n
        for k in ("bound_counts", "bound"):
            assert np.array_equal(poly[k].view(np.uint8), poly2[k].view(np.uint8)), n
        if e["status"][0] == 0 and len(e["open"]):
            opened += 1
    assert opened >= 3
