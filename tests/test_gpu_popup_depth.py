"""pus_popup_depth on the device against the CPU oracle (tests/popup_depth_oracle.cpp, orc_popup_depth): the fixture frames
of tests/golden/popup_depth.npz, seeded batches of both image sizes, downsample on and off and three ceilings (one below
every camera), and the fit -> polygons -> depth chain.  Every comparison is on float32 bit patterns, NaN compared as NaN:
both sides evaluate the same float32 expressions in the same order with every operation rounded (the device code is built
with --fmad=false, the oracle with -ffp-contract=off)."""
import numpy as np
import pytest

import oracle_api
import popup_depth_native as N
import popup_polygon_native as NP
from pop_up_slam_b200 import capi
from test_popup_depth import fixture_cases, same_bits

pytestmark = pytest.mark.gpu


def test_fixture_frames_match_the_oracle():
    lib, orc = capi.load_library(), N.oracle_lib()
    for b, want in fixture_cases():
        got = capi.popup_depth(lib, **b)
        same_bits(got, capi.popup_depth(orc, prefix="orc_", **b))
        same_bits(got, want)


@pytest.mark.parametrize("size", [(640, 480), (960, 540)])
@pytest.mark.parametrize("downsample", [True, False])
@pytest.mark.parametrize("ceiling", [2.5, 5.0, 0.4])
def test_random_batches_match_the_oracle(size, downsample, ceiling):
    lib, orc = capi.load_library(), N.oracle_lib()
    b = N.random_batch(int(size[0] + 10 * ceiling + downsample), 12, *size, downsample, ceiling)
    got = capi.popup_depth(lib, **b)
    same_bits(got, capi.popup_depth(orc, prefix="orc_", **b), str((size, downsample, ceiling)))
    assert (got[:-1] != 0).sum() > 10000 and not got[-1].any()


def test_batch_equals_frame_by_frame_and_repeats_bit_identically():
    lib = capi.load_library()
    b = N.random_batch(5, 10, 640, 480, True, 2.5)
    whole = capi.popup_depth(lib, **b)
    same_bits(whole, capi.popup_depth(lib, **b), "repeat")
    for f in range(len(b["plane_ptr"]) - 1):
        p0, p1 = b["plane_ptr"][f], b["plane_ptr"][f + 1]
        v0, v1 = b["poly_ptr"][p0], b["poly_ptr"][p1]
        one = dict(b, plane_ptr=[0, p1 - p0], poly_ptr=b["poly_ptr"][p0:p1 + 1] - v0, polys=b["polys"][v0:v1],
                   planes_sensor=b["planes_sensor"][p0:p1], Ts=b["Ts"][f:f + 1])
        same_bits(capi.popup_depth(lib, **one)[0], whole[f], f"frame {f}")


@pytest.mark.parametrize("seed,size,downsample", [(31, (640, 480), True), (32, (960, 540), False)])
def test_fit_polygons_depth_chain_matches_the_oracles(seed, size, downsample):
    """get_depth_map_good after get_plane_equation and find_2d_3d_closed_polygon: the good rows' bound polygons and planes"""
    lib, orc, porc, forc = capi.load_library(), N.oracle_lib(), NP.oracle_lib(), oracle_api.oracle_lib()
    b = NP.random_batch(seed, 16, *size, 2.5, 3.0)
    nf = len(b["seg_ptr"]) - 1
    outs = []
    for fit_lib, poly_lib, depth_lib, pre in ((lib, lib, lib, "pus_"), (forc, porc, orc, "orc_")):
        fit = capi.popup_fit_frames(fit_lib, b["seg_ptr"], b["segs"], b["invK"], b["Ts"], 10.0, 0, prefix=pre)
        poly = capi.popup_polygons(poly_lib, prefix=pre, **b)
        good = np.flatnonzero(fit[3])
        plane_ptr = np.zeros(nf + 1, np.int32)
        for f in range(nf):
            r0, r1 = b["seg_ptr"][f] + f, b["seg_ptr"][f + 1] + f + 1
            plane_ptr[f + 1] = plane_ptr[f] + int(np.sum((good >= r0) & (good < r1)))
        cnt = poly["bound_counts"][good]
        polys = np.concatenate([poly["bound"][poly["bound_ptr"][r]:poly["bound_ptr"][r + 1]] for r in good])
        outs.append(capi.popup_depth(depth_lib, plane_ptr, np.concatenate([[0], np.cumsum(cnt)]), polys, fit[1][good], b["Ts"],
                                     b["invK"], *size, downsample=downsample, ceiling_threshold=2.5, prefix=pre))
    same_bits(outs[0], outs[1])
    assert (outs[0] != 0).sum() > 100000
