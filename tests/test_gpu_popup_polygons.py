"""pus_popup_polygons on the device against the CPU oracle (tests/popup_polygon_oracle.cpp, orc_popup_polygons) on seeded
the fixture frames of tests/golden/popup_polygons.npz and seeded synthetic batches of both image sizes, every wall-length mode and both ceilings.  Counts are exact and vertices
bit-identical, NaN positions included: both sides evaluate the same float32 expressions in the same order with every
operation rounded (the device code is built with --fmad=false, the oracle with -ffp-contract=off)."""
import numpy as np
import pytest

import oracle_api
import popup_cloud_native as NC
import popup_polygon_native as N
from pop_up_slam_b200 import capi
from test_popup_polygons import fixture_cases

pytestmark = pytest.mark.gpu
SETS = ("bound", "cut", "world")


def same(a, b, msg=""):
    for k in SETS:
        np.testing.assert_array_equal(a[k + "_counts"], b[k + "_counts"], err_msg=f"{msg} {k}")
        nan = np.isnan(a[k])
        np.testing.assert_array_equal(nan, np.isnan(b[k]), err_msg=f"{msg} {k}")
        np.testing.assert_array_equal(a[k][~nan].view(np.uint32), b[k][~nan].view(np.uint32), err_msg=f"{msg} {k}")


def test_fixture_frames_match_the_oracle():
    lib, orc = capi.load_library(), N.oracle_lib()
    for b, _ in fixture_cases():
        same(capi.popup_polygons(lib, **b), capi.popup_polygons(orc, prefix="orc_", **b), str(b["width"]))


@pytest.mark.parametrize("size,ceiling,walllength", N.SETTINGS)
def test_random_batches_match_the_oracle(size, ceiling, walllength):
    lib, orc = capi.load_library(), N.oracle_lib()
    b = N.random_batch(int(size[0] + 10 * ceiling + 7 * walllength), 64, *size, ceiling, walllength)
    same(capi.popup_polygons(lib, **b), capi.popup_polygons(orc, prefix="orc_", **b), str((size, ceiling, walllength)))


def test_batch_equals_frame_by_frame_and_repeats_bit_identically():
    lib = capi.load_library()
    rng = np.random.default_rng(3)
    frames = [N.random_frame(rng, 960, 540) for _ in range(12)] + [(np.zeros((0, 4), np.float32), np.eye(4, dtype=np.float32))]
    b = N.batch(frames, 960, 540, 2.5, 3.0)
    whole = capi.popup_polygons(lib, **b)
    same(whole, capi.popup_polygons(lib, **b), "repeat")
    parts = [capi.popup_polygons(lib, **N.batch([fr], 960, 540, 2.5, 3.0)) for fr in frames]
    assert parts[-1]["bound_counts"].tolist() == [0]
    for k in SETS:
        np.testing.assert_array_equal(np.concatenate([p[k + "_counts"] for p in parts]), whole[k + "_counts"])
        np.testing.assert_array_equal(np.concatenate([p[k] for p in parts]).view(np.uint32), whole[k].view(np.uint32))


def test_size_query_agrees_with_the_filled_call_and_a_short_capacity_is_refused():
    lib = capi.load_library()
    b = N.random_batch(4, 20, 640, 480, 5.0, 0.5)
    q = capi.popup_polygons(lib, vertices=False, **b)
    full = capi.popup_polygons(lib, **b)
    tot = [int(q[k + "_ptr"][-1]) for k in SETS]
    for k, t in zip(SETS, tot):
        np.testing.assert_array_equal(q[k + "_counts"], full[k + "_counts"])
        assert len(full[k]) == t
    same(full, capi.popup_polygons(lib, capacity=[t + 3 for t in tot], **b), "roomy")
    for i in range(3):
        cap = list(tot)
        cap[i] -= 1
        with pytest.raises(capi.ApiError, match="capacity"):
            capi.popup_polygons(lib, capacity=cap, **b)


@pytest.mark.parametrize("seed,size", [(21, (640, 480)), (22, (960, 540))])
def test_fit_polygons_clouds_chain_matches_the_oracles(seed, size):
    """main_3d's per-frame geometry: the fit, the polygons, and the clouds of the good rows from the cut polygons"""
    lib, orc, corc, forc = capi.load_library(), N.oracle_lib(), NC.oracle_lib(), oracle_api.oracle_lib()
    b = N.random_batch(seed, 16, *size, 2.5, 3.0)
    w, h = size
    nf = len(b["seg_ptr"]) - 1
    outs = []
    for fit_lib, poly_lib, cloud_lib, pre in ((lib, lib, lib, "pus_"), (forc, orc, corc, "orc_")):
        fit = capi.popup_fit_frames(fit_lib, b["seg_ptr"], b["segs"], b["invK"], b["Ts"], 10.0, 0, prefix=pre)
        poly = capi.popup_polygons(poly_lib, prefix=pre, **b)
        good = np.flatnonzero(fit[3])
        plane_ptr = np.zeros(nf + 1, np.int32)
        for f in range(nf):
            r0, r1 = b["seg_ptr"][f] + f, b["seg_ptr"][f + 1] + f + 1
            plane_ptr[f + 1] = plane_ptr[f] + int(np.sum((good >= r0) & (good < r1)))
        cnt = poly["cut_counts"][good]
        polys = np.concatenate([poly["cut"][poly["cut_ptr"][r]:poly["cut_ptr"][r + 1]] for r in good])
        cl = capi.popup_clouds(cloud_lib, plane_ptr, np.concatenate([[0], np.cumsum(cnt)]), polys, fit[1][good], b["Ts"],
                               b["invK"], w, h, images=np.stack([NC.image(f, w, h) for f in range(nf)]), prefix=pre)
        outs.append((poly, cl))
    same(outs[0][0], outs[1][0], "polygons")
    g, o = outs[0][1], outs[1][1]
    np.testing.assert_array_equal(g["counts"], o["counts"])
    assert g["total"] > 1000
    nan = np.isnan(g["xyz"])
    np.testing.assert_array_equal(nan, np.isnan(o["xyz"]))
    np.testing.assert_array_equal(g["xyz"][~nan].view(np.uint32), o["xyz"][~nan].view(np.uint32))
    np.testing.assert_array_equal(g["rgb"], o["rgb"])
