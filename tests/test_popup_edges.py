"""CPU tests of the ground edges (pus_popup_edges): the oracle (tests/popup_edges_oracle.cpp, the device's frame code
compiled for the host) against the separately written Python restatement of tools/make_popup_edge_golden.py -- its
fixture bit for bit, its stage 0 through live cv2 and its scikit-image 0.14 contour assembly on crafted maps -- plus the
refusals and the missing-GPU error."""
import os
import subprocess

import numpy as np
import pytest

import popup_edges_native as N
from pop_up_slam_b200 import capi

G = N.G
KEYS = ("status", "open_counts", "connect_counts", "open", "connect", "open_in_connect")


def same(got, want, what=""):
    for k in KEYS:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), (what, k)


def test_oracle_equals_the_fixture_bit_for_bit():
    orc = N.oracle_lib()
    for b, want in N.fixture():
        same(capi.popup_edges(orc, prefix="orc_", **b), want, b["params"])
        assert np.array_equal(N.codes(b), want["bits"])


def test_fixture_reaches_every_status_and_the_selection_branches():
    st, bits = set(), 0
    for _, want in N.fixture():
        st |= set(want["status"].tolist())
        bits |= int(np.bitwise_or.reduce(want["bits"]))
    assert st == {0, 1, 2, 3, 4}
    # the shared-point branches (STALE, MATERIALIZE) come from the crafted maps of the contour test below
    missing = [k for k in G.BITS if not bits & G.B[k] and k not in ("STALE", "MATERIALIZE")]
    assert not missing, missing


@pytest.mark.parametrize("down", [1, 0])
def test_preprocessing_equals_cv2(down):
    cv2 = pytest.importorskip("cv2")
    cv2.setUseOptimized(False)
    rng = np.random.default_rng(7 + down)
    for h, w in ((48, 64), (37, 51), (5, 4), (120, 161)):
        for k in ((11, 11), (3, 8), (1, 1)):
            lab = rng.choice(np.array([0, 127, 255], np.uint8), (h, w), p=[0.5, 0.2, 0.3])
            P = dict(capi.EDGE_DEFAULTS, downsample_contour=down, dilation_distance=k[0], erosion_distance=k[1])
            assert np.array_equal(N.preprocess(lab, **P), G.preprocess(cv2, lab, P)), (h, w, k, down)


def crafted_maps():
    rng = np.random.default_rng(3)
    maps = [np.zeros((9, 9), np.uint8), np.full((9, 9), 255, np.uint8)]
    m = np.full((20, 30), 255, np.uint8)
    m[10:, :] = 0
    m[2, 3:20] = 0        # a 1-pixel ground line
    m[2:10, 12] = 0       # touching the region
    m[5, 25] = 0          # an isolated pixel
    maps.append(m)
    m = np.full((16, 16), 255, np.uint8)
    m[::2, ::2] = 0       # a checkerboard of ground pixels: saddles everywhere
    maps.append(m)
    m = np.full((12, 12), 255, np.uint8)
    m[0, :] = 0
    m[:, 0] = 0           # ground along the border
    maps.append(m)
    # speckle with 10-15 % or 85-90 % ground pixels: most maps assemble, and many reuse a stale dict entry.  Near 50 %
    # most maps end in the assembly's KeyError (a pop of a key never stored), which the 40 maps of that kind check.
    for dens in [0.1, 0.15, 0.85, 0.9] * 40 + [0.5] * 40:
        h, w = int(rng.integers(8, 40)), int(rng.integers(8, 40))
        maps.append(np.where(rng.random((h, w)) < dens, 0, 255).astype(np.uint8))
    return maps


def test_contour_assembly_equals_the_restatement_on_crafted_maps():
    bits, compared, stale_compared = 0, 0, 0
    for m in crafted_maps():
        b = [0]
        want, got = G.ground_contour(m, 2, b), N.contour(m, 2)
        bits |= b[0]
        assert (want is None) == (got is None)
        if want is not None:
            assert np.array_equal(want, got)
            compared += 1
            stale_compared += bool(b[0] & G.B["STALE"])
    assert compared >= 100 and stale_compared >= 20, (compared, stale_compared)   # 106 and 49 of the 205 maps
    assert bits & G.B["CLOSE"] and bits & G.B["JOIN_APPEND"] and bits & G.B["JOIN_PREPEND"]


def pileup_frame(n=154, w=960, h=540):
    """a half-ground map and n 16 px lines on the boundary, 6 px apart: with the angle thresholds at 0 nothing is merged or
    deleted, the greedy pass keeps every line, and split_overlaps leaves more pieces than the 100 merge passes can join --
    more output rows than input lines"""
    lab = np.zeros((h, w), np.uint8)
    lab[h // 2:] = 255
    lines = np.array([[10 + 6 * i, h / 2, 26 + 6 * i, h / 2] for i in range(n)], np.float32)
    prm = dict(pre_merge_angle_thre=0.0, pre_proj_angle_thre=0.0, post_short_thre=1.0, post_merge_angle_thre=0.0,
               post_bind_dist_thre=0.0)
    return lab, lines, prm


def test_more_output_rows_than_input_lines():
    cv2 = pytest.importorskip("cv2")
    lab, lines, prm = pileup_frame()
    P = dict(capi.EDGE_DEFAULTS, **prm)
    st, o, c, inc, _ = G.edges(cv2, lab, lines, P)
    assert st == 0 and len(o) > len(lines)
    # the frame between two others, so that rows written past a frame's slots would show in its neighbours
    labs = np.stack([lab, lab, lab])
    ptr = [0, 3, 3 + len(lines), 6 + len(lines)]
    L = np.concatenate([lines[:3], lines, lines[:3]])
    got = capi.popup_edges(N.oracle_lib(), labs, ptr, L, prm, prefix="orc_")
    assert got["status"][1] == 0
    o0, o1 = got["open_ptr"][1], got["open_ptr"][2]
    assert np.array_equal(got["open"][o0:o1].view(np.uint8), o.view(np.uint8))
    c0, c1 = got["connect_ptr"][1], got["connect_ptr"][2]
    assert np.array_equal(got["connect"][c0:c1].view(np.uint8), c.view(np.uint8))
    assert np.array_equal(got["open_in_connect"][o0:o1], inc)
    single = capi.popup_edges(N.oracle_lib(), labs[:1], [0, 3], lines[:3], prm, prefix="orc_")
    for f in (0, 2):
        a0, a1 = got["open_ptr"][f], got["open_ptr"][f + 1]
        assert np.array_equal(got["open"][a0:a1].view(np.uint8), single["open"].view(np.uint8))


ASAN_MAIN = r"""
#include "popup_edges_oracle.cpp"
int main() {
  const int w = 960, h = 540, n = 154;
  std::vector<unsigned char> lab((size_t)w * h, 0);
  for (int y = h / 2; y < h; y++) for (int x = 0; x < w; x++) lab[(size_t)y * w + x] = 255;
  std::vector<float> L;
  for (int i = 0; i < n; i++) { L.push_back(10 + 6.f * i); L.push_back(h / 2.f); L.push_back(26 + 6.f * i); L.push_back(h / 2.f); }
  int ptr[2] = {0, n};
  pus_edge_params P = {11, 11, 1, 15, 15, 5, 50, 0, 10, 0, 0.6, 0.8, 100, 20, 1, 0, 20, 0, 15};
  int st, oc, cc;
  std::vector<float> o(4 * 4 * n), c(4 * 4 * n);
  std::vector<int> inc(4 * n);
  int r = orc_popup_edges(0, 1, lab.data(), w, h, ptr, L.data(), &P, &st, &oc, &cc, o.data(), c.data(), inc.data(), 4 * n, 4 * n);
  return (r == 1 && st == 0 && oc > n) ? 0 : 1;
}
"""


def test_frame_code_stays_in_its_rows_under_address_sanitizer(tmp_path):
    """the frame code's work and output rows are sized by the documented bound (pus_edges.cuh, Sel): the pile-up frame
    under AddressSanitizer, whose buffers in the oracle are exactly that size"""
    src = tmp_path / "asan_main.cpp"
    src.write_text(ASAN_MAIN)
    exe = tmp_path / "asan_main"
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run(["g++", "-g", "-O1", "-fsanitize=address", "-ffp-contract=off", "-std=c++17", "-I", tests, str(src),
                        "-o", str(exe)], capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr:
        pytest.skip("no AddressSanitizer runtime: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert run.returncode == 0, run.stderr[-2000:]


def test_refusals():
    orc = N.oracle_lib()
    lab = np.zeros((1, 32, 32), np.uint8)
    ok = dict(labels=lab, line_ptr=[0, 1], lines=[[1, 2, 20, 3]])
    capi.popup_edges(orc, prefix="orc_", **ok)
    bad = [dict(ok, line_ptr=[1, 1]), dict(ok, line_ptr=[0, -1]), dict(ok, lines=[[1, np.nan, 2, 3]]),
           dict(ok, line_ptr=[0, N_MAX + 1], lines=np.zeros((N_MAX + 1, 4))), dict(ok, labels=np.zeros((1, 3, 32), np.uint8)),
           dict(ok, params=dict(downsample_contour=0, dilation_distance=0))]
    for b in bad:
        with pytest.raises(capi.ApiError):
            capi.popup_edges(orc, prefix="orc_", **b)


N_MAX = 512   # PUS_POPUP_MAX_LINES


def test_no_gpu_is_an_error():
    if os.path.exists("/dev/nvidia0"):
        pytest.skip("a GPU is present")
    try:
        lib = capi.load_library()
    except capi.ApiError:
        return
    with pytest.raises(capi.ApiError, match="no CPU fallback"):
        capi.popup_edges(lib, np.zeros((1, 32, 32), np.uint8), [0, 0], np.zeros((0, 4)))
