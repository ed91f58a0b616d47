"""pus_popup_lines' CPU oracle (tests/popup_lines_oracle.cpp) against the fixture written by the separate restatement
tools/make_popup_line_golden.py (live cv2 per-pixel stages, Python walk / fits / nfa), bit for bit; each stage entry
point against live cv2; the branch-bit union; the generator's reproducibility; the refusals."""
import math
import os

import numpy as np
import pytest

import popup_lines_native as N
from pop_up_slam_b200 import capi

G = N.G


def same(got, want, tag=""):
    assert np.array_equal(got["status"], want["status"]), tag
    assert np.array_equal(got["counts"], want["counts"]), tag
    assert np.array_equal(np.asarray(got["lines"], np.float32).view(np.uint32), want["lines"].view(np.uint32)), tag


def test_oracle_equals_the_fixture():
    orc = N.oracle_lib()
    for key, imgs, ds, want in N.fixture():
        same(capi.popup_lines(orc, imgs, downsample=ds, prefix="orc_"), want, key)
        assert np.array_equal(N.bits(imgs, ds), want["bits"]), key


def test_branch_bits_cover_every_branch():
    union = 0
    for _, _, _, want in N.fixture():
        for b in want["bits"]:
            union |= int(b)
    missing = {k for k in G.BITS if not union & G.B[k]}
    assert missing == N.UNCOVERED, missing
    statuses = {int(s) for _, _, _, w in N.fixture() for s in w["status"]}
    assert statuses == {0, 1}


def test_decision_margins_are_reported():
    z = np.load(os.path.join(N.ROOT, "tests", "golden", "popup_lines.npz"))
    print(f"smallest margin: angle test {float(z['margin_angle']):.3g} rad, nfa {float(z['margin_nfa']):.3g}")
    assert float(z["margin_angle"]) > 0 and float(z["margin_nfa"]) > 0


def test_generator_reproduces_the_fixture(tmp_path):
    out = tmp_path / "g.npz"
    G.main(str(out))
    a, b = np.load(out), np.load(os.path.join(N.ROOT, "tests", "golden", "popup_lines.npz"))
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].tobytes() == b[k].tobytes(), k


def _images():
    rng = np.random.default_rng(3)
    out = [rng.integers(0, 256, (h, w), dtype=np.uint8) for h, w in ((3, 3), (4, 4), (3, 7), (5, 4), (31, 17), (480, 640))]
    out += [np.zeros((9, 11), np.uint8), np.full((6, 6), 255, np.uint8), np.tile(np.uint8([0, 255]), (7, 5))]
    for _, imgs, _, _ in N.fixture()[:4]:
        out.append(np.asarray(imgs[0]))
    return out


def test_stages_equal_cv2():
    cv2 = G.cv()
    for im in _images():
        g = cv2.cvtColor(im, cv2.COLOR_BGR2GRAY) if im.ndim == 3 else im
        assert np.array_equal(N.grey(im), g)
        eq = cv2.equalizeHist(g) if cv2.mean(g)[0] < 90 else g
        assert np.array_equal(N.contrast(g)[0], eq)
        if g.shape[0] % 2 == 0 and g.shape[1] % 2 == 0 and min(g.shape) >= 6:
            assert np.array_equal(N.halve(g), cv2.resize(g, None, fx=0.5, fy=0.5))
        b = cv2.GaussianBlur(g, (5, 5), 1)
        assert np.array_equal(N.blur(g), b), g.shape
        dx, dy, gg, d = N.gradient(b)
        wdx, wdy, wg, wh = G.gradient(cv2, b)
        assert np.array_equal(dx, wdx) and np.array_equal(dy, wdy) and np.array_equal(gg, wg)
        assert np.array_equal(d == 255, wh)


def test_contrast_at_the_mean_90_boundary():
    cv2 = G.cv()
    g = np.full((10, 10), 90, np.uint8)
    g[0, :2] = (89, 91)                      # sum exactly 90 N: not below 90
    assert cv2.mean(g)[0] == 90.0 and N.contrast(g)[1] == 0
    g[0, 1] = 90                             # one below: equalized
    out, bits = N.contrast(g)
    assert bits & G.B["EQUALIZED"] and np.array_equal(out, cv2.equalizeHist(g))
    u = np.full((5, 7), 33, np.uint8)        # one bin: every pixel keeps its value
    out, bits = N.contrast(u)
    assert bits & G.B["ONE_BIN"] and np.array_equal(out, u) and np.array_equal(cv2.equalizeHist(u), u)


def test_gradient_rounds_half_to_even():
    cv2 = G.cv()
    t = np.array([[82, 86, 90, 81, 84]], np.int16)
    assert cv2.multiply(t, 0.25).tolist() == [[20, 22, 22, 20, 21]]


def test_chains_equal_the_restatement():
    cv2 = G.cv()
    for _, imgs, ds, _ in N.fixture():
        b, _ = G.prepare(cv2, np.asarray(imgs[0]), ds)
        dx, dy, g, hz = G.gradient(cv2, b)
        st, want, _ = G.chains(b, dx, dy, g, hz, 0)
        got = N.chains(b)
        assert (got == -1) if st else (got == want)


def test_refusals():
    orc = N.oracle_lib()
    img = np.zeros((2, 8, 8, 3), np.uint8)
    with pytest.raises(capi.ApiError, match="channels"):
        capi.popup_lines(orc, np.zeros((1, 8, 8, 2), np.uint8), prefix="orc_")
    with pytest.raises(capi.ApiError, match="even"):
        capi.popup_lines(orc, np.zeros((1, 8, 7), np.uint8), downsample=True, prefix="orc_")
    with pytest.raises(capi.ApiError, match="3 x 3"):
        capi.popup_lines(orc, np.zeros((1, 4, 8), np.uint8), downsample=True, prefix="orc_")
    with pytest.raises(capi.ApiError, match="3 x 3"):
        capi.popup_lines(orc, np.zeros((1, 2, 8), np.uint8), prefix="orc_")
    r = capi.popup_lines(orc, img, prefix="orc_")
    assert r["lines"].shape == (0, 4) and list(r["status"]) == [0, 0]


def test_no_gpu_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = capi.load_library()
    with pytest.raises(capi.ApiError, match="no CPU fallback"):
        capi.popup_lines(lib, np.zeros((1, 8, 8), np.uint8))
