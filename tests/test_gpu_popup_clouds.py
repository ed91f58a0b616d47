"""pus_popup_clouds on the device against the CPU oracle (tests/popup_cloud_oracle.cpp, orc_popup_clouds): the fixture
frames of tests/golden/popup_clouds.npz and random batches.  Pixel order, counts, offsets, colours, labels and the filter
decisions are exact, and xyz is bit-identical: both sides evaluate the same float32 expressions in the same order with every
operation rounded (the device code is built with --fmad=false, the oracle with -ffp-contract=off; float division is IEEE
on both).  NaN points (a ray parallel to its plane) compare as NaN on both sides."""
import numpy as np
import pytest

import popup_cloud_native as N
from pop_up_slam_b200 import capi
from test_popup_clouds import cases, run_case

pytestmark = pytest.mark.gpu


def same(a, b, msg=""):
    np.testing.assert_array_equal(a["counts"], b["counts"], err_msg=msg)
    np.testing.assert_array_equal(a["offsets"], b["offsets"], err_msg=msg)
    assert a["xyz"].shape == b["xyz"].shape, msg
    nan = np.isnan(a["xyz"])
    np.testing.assert_array_equal(nan, np.isnan(b["xyz"]), err_msg=msg)
    np.testing.assert_array_equal(a["xyz"][~nan].view(np.uint32), b["xyz"][~nan].view(np.uint32), err_msg=msg)
    np.testing.assert_array_equal(a["rgb"], b["rgb"], err_msg=msg)
    if "labels" in a or "labels" in b:
        np.testing.assert_array_equal(a["labels"], b["labels"], err_msg=msg)


def test_fixture_frames_match_the_oracle():
    lib, orc = capi.load_library(), N.oracle_lib()
    for c, d, g in cases():
        same(run_case(lib, d, g, "pus_", frame=c), run_case(orc, d, g, "orc_", frame=c), f"case {c}")


def random_batch(seed, n_frames, width, height, downsample, with_images=True):
    rng = np.random.default_rng(seed)
    frames = [N.random_frame(rng, width, height, int(rng.integers(1, 6))) for _ in range(n_frames)]
    plane_ptr, poly_ptr, polys, planes, Ts = N.batch(frames)
    imgs = np.stack([N.image(f, width, height) for f in range(n_frames)]) if with_images else None
    return dict(plane_ptr=plane_ptr, poly_ptr=poly_ptr, polys=polys, planes_sensor=planes, Ts=Ts, invK=N.invK(width, height),
                width=width, height=height, images=imgs, downsample=downsample)


@pytest.mark.parametrize("seed,size,downsample,with_images", [(1, (640, 480), True, True), (2, (640, 480), False, True),
                                                              (3, (960, 540), True, True), (4, (960, 540), False, False)])
def test_random_batches_match_the_oracle(seed, size, downsample, with_images):
    lib, orc = capi.load_library(), N.oracle_lib()
    b = random_batch(seed, 12, *size, downsample, with_images)
    got = capi.popup_clouds(lib, labels=True, **b)
    same(got, capi.popup_clouds(orc, labels=True, prefix="orc_", **b), f"seed {seed}")
    assert got["total"] > 1000


def test_batch_equals_frame_by_frame_and_repeats_bit_identically():
    lib = capi.load_library()
    b = random_batch(5, 10, 640, 480, True)
    whole = capi.popup_clouds(lib, labels=True, **b)
    again = capi.popup_clouds(lib, labels=True, **b)
    same(whole, again, "repeat")
    parts = []
    for f in range(10):
        p0, p1 = b["plane_ptr"][f], b["plane_ptr"][f + 1]
        v0, v1 = b["poly_ptr"][p0], b["poly_ptr"][p1]
        one = dict(b, plane_ptr=[0, p1 - p0], poly_ptr=b["poly_ptr"][p0:p1 + 1] - v0, polys=b["polys"][v0:v1],
                   planes_sensor=b["planes_sensor"][p0:p1], Ts=b["Ts"][f:f + 1], images=b["images"][f:f + 1])
        parts.append(capi.popup_clouds(lib, labels=True, **one))
    np.testing.assert_array_equal(np.concatenate([p["counts"] for p in parts]), whole["counts"])
    np.testing.assert_array_equal(np.concatenate([p["xyz"] for p in parts]).view(np.uint32), whole["xyz"].view(np.uint32))
    np.testing.assert_array_equal(np.concatenate([p["rgb"] for p in parts]), whole["rgb"])
    np.testing.assert_array_equal(np.concatenate([p["labels"] for p in parts]), whole["labels"])


def test_size_query_agrees_with_the_filled_call_and_a_short_capacity_is_refused():
    lib = capi.load_library()
    b = random_batch(6, 6, 960, 540, True)
    q = capi.popup_clouds(lib, points=False, **b)
    full = capi.popup_clouds(lib, capacity=q["total"] + 5, **b)
    assert q["total"] == full["total"] == len(full["xyz"]) == q["counts"].sum()
    np.testing.assert_array_equal(q["counts"], full["counts"])
    np.testing.assert_array_equal(q["offsets"], full["offsets"])
    with pytest.raises(capi.ApiError, match="capacity"):
        capi.popup_clouds(lib, capacity=q["total"] - 1, **b)
