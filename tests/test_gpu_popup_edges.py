"""pus_popup_edges on the device against the CPU oracle (tests/popup_edges_oracle.cpp): the fixture frames, seeded 64-frame
batches at 640x480 and 960x540 with downsample_contour on and off, batch against frame-by-frame calls, repeated calls,
size queries and capacities, and the labels + lines -> edges -> fit -> polygons chain.  Comparisons are on bit patterns
(the device code is built with --fmad=false, the oracle with -ffp-contract=off)."""
import numpy as np
import pytest

import oracle_api
import popup_edges_native as N
import popup_polygon_native as NP
from pop_up_slam_b200 import capi
from test_popup_edges import KEYS, same

pytestmark = pytest.mark.gpu


def test_fixture_frames_match_the_oracle():
    lib = capi.load_library()
    for b, want in N.fixture():
        same(capi.popup_edges(lib, **b), want, b["params"])


@pytest.mark.parametrize("size", [(640, 480), (960, 540)])
@pytest.mark.parametrize("down", [1, 0])
def test_random_batches_match_the_oracle(size, down):
    lib, orc = capi.load_library(), N.oracle_lib()
    b = N.random_batch(size[0] + down, 64, *size, down)
    got = capi.popup_edges(lib, **b)
    same(got, capi.popup_edges(orc, prefix="orc_", **b), (size, down))
    assert (got["status"] == 0).sum() > 20


def test_batch_equals_frame_by_frame_and_repeats():
    lib = capi.load_library()
    b = N.random_batch(11, 12, 640, 480, 1)
    whole = capi.popup_edges(lib, **b)
    same(capi.popup_edges(lib, **b), whole, "repeat")
    for f in range(len(b["line_ptr"]) - 1):
        l0, l1 = b["line_ptr"][f], b["line_ptr"][f + 1]
        one = capi.popup_edges(lib, b["labels"][f:f + 1], [0, l1 - l0], b["lines"][l0:l1], b["params"])
        o0, o1 = whole["open_ptr"][f], whole["open_ptr"][f + 1]
        c0, c1 = whole["connect_ptr"][f], whole["connect_ptr"][f + 1]
        assert one["status"][0] == whole["status"][f]
        assert np.array_equal(one["open"].view(np.uint8), whole["open"][o0:o1].view(np.uint8))
        assert np.array_equal(one["connect"].view(np.uint8), whole["connect"][c0:c1].view(np.uint8))
        assert np.array_equal(one["open_in_connect"], whole["open_in_connect"][o0:o1])


def test_size_query_and_capacities():
    lib = capi.load_library()
    b = N.random_batch(12, 8, 640, 480, 1)
    q = capi.popup_edges(lib, segments=False, **b)
    full = capi.popup_edges(lib, **b)
    for k in ("status", "open_counts", "connect_counts"):
        assert np.array_equal(q[k], full[k])
    big = capi.popup_edges(lib, capacity=(len(full["open"]) + 5, len(full["connect"]) + 5), **b)
    same(big, full)
    if len(full["open"]):
        with pytest.raises(capi.ApiError, match="capacity"):
            capi.popup_edges(lib, capacity=(len(full["open"]) - 1, len(full["connect"])), **b)


def test_edges_fit_polygons_chain_matches_the_oracles():
    """main_3d's order: edges, then get_plane_equation on the open segments, with good walls filtered by the connected-list
    indices of the open segments (open_in_connect), then the closed polygons of the connected segments"""
    lib, orc, porc, forc = capi.load_library(), N.oracle_lib(), NP.oracle_lib(), oracle_api.oracle_lib()
    b = N.random_batch(21, 16, 640, 480, 1)
    pb = NP.random_batch(21, 1, 640, 480, 2.5, 3.0)
    outs = []
    for el, fl, pl, pre in ((lib, lib, lib, "pus_"), (orc, forc, porc, "orc_")):
        e = capi.popup_edges(el, prefix=pre, **b)
        nf = len(e["status"])
        Ts = np.repeat(pb["Ts"][:1], nf, axis=0)
        fit = capi.popup_fit_frames(fl, e["open_ptr"], e["open"], pb["invK"], Ts, 10.0, 0, prefix=pre)
        poly = capi.popup_polygons(pl, e["connect_ptr"], e["connect"], pb["K"], pb["invK"], Ts, 640, 480, prefix=pre)
        outs.append((e, fit, poly))
    (e, fit, poly), (e2, fit2, poly2) = outs
    same(e, e2)
    for a, c in zip(fit, fit2):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(c).view(np.uint8))
    for k in ("bound_counts", "bound"):
        assert np.array_equal(poly[k].view(np.uint8), poly2[k].view(np.uint8))
    # get_plane_equation's filter (popup_plane.cpp:629-635, 792-794): wall row seg + 1 of a frame stays good only if seg + 1
    # is in actual_plane_indices_inall = {0} u {open_in_connect + 1}
    filtered = []
    for ed, ft in ((e, fit), (e2, fit2)):
        g = np.asarray(ft[3]).copy()
        for f in range(len(ed["status"])):
            o0, o1 = ed["open_ptr"][f], ed["open_ptr"][f + 1]
            actual = {0} | {int(i) + 1 for i in ed["open_in_connect"][o0:o1]}
            for seg in range(o1 - o0):
                r = o0 + f + 1 + seg
                g[r] = g[r] if (seg + 1) in actual else 0
        filtered.append(g)
    assert np.array_equal(filtered[0], filtered[1])
    # the filter acts: some frame has connectors, so some good wall of it is dropped
    assert (filtered[0] != np.asarray(fit[3])).any()


def test_more_output_rows_than_input_lines():
    """the pile-up frame of test_popup_edges between two others: more open rows than input lines, no row outside its slot"""
    from test_popup_edges import pileup_frame
    lib, orc = capi.load_library(), N.oracle_lib()
    lab, lines, prm = pileup_frame()
    labs = np.stack([lab, lab, lab])
    L = np.concatenate([lines[:3], lines, lines[:3]])
    b = dict(labels=labs, line_ptr=[0, 3, 3 + len(lines), 6 + len(lines)], lines=L, params=prm)
    got = capi.popup_edges(lib, **b)
    same(got, capi.popup_edges(orc, prefix="orc_", **b))
    assert got["status"][1] == 0 and got["open_counts"][1] > len(lines)
