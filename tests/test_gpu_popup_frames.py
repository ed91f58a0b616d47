"""The pop-up session (pus_popup_session_*) on the device against the device stage calls with main_3d's glue between them
and against the host oracle of the whole run (tests/popup_frames_oracle.cpp), bit for bit."""
import numpy as np
import pytest

import oracle_api
import popup_cloud_native as NC
import popup_depth_native as ND
import popup_edges_native as NE
import popup_frames_native as NF
import popup_lines_native as NL
import popup_polygon_native as NP
from pop_up_slam_b200 import capi

pytestmark = pytest.mark.gpu


def _libs(prefix):
    if prefix == "pus_":
        return (capi.load_library(),) * 6
    return (NL.oracle_lib(), NE.oracle_lib(), oracle_api.oracle_lib(), NP.oracle_lib(), NC.oracle_lib(), ND.oracle_lib())


def _check(imgs, labs, Ts, cfg, prefixes=("pus_", "orc_"), where=""):
    s = capi.PopupFrames(capi.load_library(), cfg)
    got = s.run(imgs, labs, Ts)
    for pre in prefixes:
        want = NF.chain(_libs(pre), imgs, labs, Ts, cfg) if pre == "pus_" else NF.oracle_run(cfg, imgs, labs, Ts)
        NF.assert_same(got, want, where=f"{where} {pre}")
    return got


@pytest.mark.parametrize("fast", [0, 1])
@pytest.mark.parametrize("dsc", [0, 1])
def test_sample_frames_equal_the_stage_chain_and_the_oracles(fast, dsc):
    planes = dropped = 0
    lib = capi.load_library()
    for i, (imgs, labs, Ts) in enumerate(NF.samples()):
        h, w = labs.shape[1:]
        cfg = NF.config(w, h, fast_edges=fast, edges=dict(downsample_contour=dsc), want_labels=1, want_depth=1)
        got = _check(imgs, labs, Ts, cfg, where=f"sample {i} fast={fast} dsc={dsc}")
        planes += got["good_ptr"][-1]
        raw = capi.popup_fit_frames(lib, got["open_ptr"], got["open_segs"], cfg["invK"], Ts, cfg["plane_cam_dist_thre"])[3]
        dropped += int(((raw == 1) & (got["good"] == 0)).sum())   # walls the actual-index filter drops
    assert planes > 4
    if (fast, dsc) == (0, 1):
        assert dropped > 0


@pytest.mark.parametrize("size", [(640, 480), (960, 540)])
def test_seeded_room_batches_equal_the_stage_chain(size):
    w, h = size
    imgs, labs, Ts = NF.rooms(5 + w, 64, w, h)
    cfg = NF.config(w, h, want_labels=1, want_depth=1)
    got = _check(imgs, labs, Ts, cfg, prefixes=("pus_",), where=f"rooms {size}")
    assert (got["status"] == 0).all() and got["good_ptr"][-1] > 64 and len(got["xyz"]) > 0


def test_seeded_rooms_equal_the_oracles():
    imgs, labs, Ts = NF.rooms(3, 6, 640, 480)
    _check(imgs, labs, Ts, NF.config(640, 480, want_labels=1, want_depth=1), prefixes=("orc_",), where="rooms orc")


def test_crafted_frames():
    """no ground, a uniform image, and walls that all fail plane_cam_dist_thre"""
    w, h = 640, 480
    imgs, labs, Ts = NF.rooms(17, 8, w, h)
    labs[0] = 0                   # no ground
    imgs[1] = 90                  # uniform image: no lines
    got = _check(imgs, labs, Ts, NF.config(w, h, want_labels=1, want_depth=1), where="crafted")
    assert got["good_ptr"][2] == 0   # neither frame has open segments, so neither has good planes
    got = _check(imgs, labs, Ts, NF.config(w, h, plane_cam_dist_thre=0.01), prefixes=("pus_",), where="far walls")
    assert (got["good_rows"] == 0).all()   # every wall fails the distance threshold: only the grounds stay good


def test_over_limit_frame_gets_its_status_and_leaves_its_neighbours_alone():
    key, many, ds, want = [f for f in NL.fixture() if f[0] == "crafted_many"][0]
    h, w = many.shape[1:3]
    imgs, labs, Ts = NF.rooms(8, 4, w, h)
    grey = np.array([img.mean(axis=2).astype(np.uint8) for img in imgs])
    cfg = NF.config(w, h, channels=1, want_labels=1, want_depth=1)
    batch = np.concatenate([grey[:2], many.reshape(1, h, w), grey[2:]])
    blab = np.concatenate([labs[:2], labs[:1], labs[2:]])
    bT = np.concatenate([Ts[:2], Ts[:1], Ts[2:]])
    s = capi.PopupFrames(capi.load_library(), cfg)
    got = s.run(batch, blab, bT)
    assert got["status"].tolist() == [0, 0, 1, 0, 0] and got["edge_status"][2] == -1
    assert got["line_counts"][2] > 512
    assert got["open_ptr"][3] == got["open_ptr"][2] and got["good_ptr"][3] == got["good_ptr"][2]
    NF.assert_same(got, NF.chain(_libs("pus_"), batch, blab, bT, cfg), where="over limit")
    NF.assert_same(got, NF.oracle_run(cfg, batch, blab, bT), where="over limit orc")
    without = s.run(grey, labs, Ts)

    def cloud(r, f):   # frame f's mixed cloud: its good planes' points back to back
        g0, g1 = r["good_ptr"][f], r["good_ptr"][f + 1]
        if g1 == g0:
            return r["xyz"][:0]
        p0 = r["cloud_offsets"][g0]
        return r["xyz"][p0:p0 + r["cloud_counts"][g0:g1].sum()]

    for f_with, f_without in ((0, 0), (1, 1), (3, 2), (4, 3)):
        for k, ptr in (("good_rows", "good_ptr"), ("open_segs", "open_ptr"), ("cloud_counts", "good_ptr")):
            a = got[k][got[ptr][f_with]:got[ptr][f_with + 1]]
            b = without[k][without[ptr][f_without]:without[ptr][f_without + 1]]
            assert np.array_equal(a, b), (k, f_with)
        assert np.array_equal(cloud(got, f_with).view(np.uint8), cloud(without, f_without).view(np.uint8)), f_with
        assert np.array_equal(got["depth"][f_with], without["depth"][f_without])
        assert np.array_equal(got["labels"][f_with], without["labels"][f_without])


def test_grey_960_wide_frames_take_no_border_rule():
    """grey images give the clouds no images, so the 960-wide x < 4 || y < 4 rule is not applied, as in the stage call"""
    imgs, labs, Ts = NF.rooms(61, 6, 960, 540)
    grey = np.array([img.mean(axis=2).astype(np.uint8) for img in imgs])
    got = _check(grey, labs, Ts, NF.config(960, 540, channels=1), where="grey 960")
    assert len(got["xyz"]) > 0


def test_batch_equals_frames_repeats_and_reuse_across_sizes():
    w, h = 640, 480
    imgs, labs, Ts = NF.rooms(23, 64, w, h)
    cfg = NF.config(w, h, want_labels=1, want_depth=1)
    lib = capi.load_library()
    s = capi.PopupFrames(lib, cfg)
    one = s.run(imgs[:1], labs[:1], Ts[:1])
    full = s.run(imgs, labs, Ts)
    three = s.run(imgs[5:8], labs[5:8], Ts[5:8])
    NF.assert_same(one, capi.PopupFrames(lib, cfg).run(imgs[:1], labs[:1], Ts[:1]), where="1")
    NF.assert_same(three, capi.PopupFrames(lib, cfg).run(imgs[5:8], labs[5:8], Ts[5:8]), where="3")
    fresh = capi.PopupFrames(lib, cfg)
    NF.assert_same(full, fresh.run(imgs, labs, Ts), where="64")
    allocs = fresh.memory()[0]
    again = fresh.run(imgs, labs, Ts)
    NF.assert_same(again, full, where="repeat")
    assert fresh.memory()[0] == allocs
    import torch   # device inputs take the same buffers: alternating them with host inputs allocates nothing either
    d_in = [torch.from_numpy(x).cuda() for x in (imgs, labs, Ts)]
    fresh.run(*d_in)
    allocs = fresh.memory()[0]
    fresh.run(imgs, labs, Ts)
    fresh.run(*d_in)
    assert fresh.memory()[0] == allocs
    for f in (0, 6, 63):   # frame by frame
        single = fresh.run(imgs[f:f + 1], labs[f:f + 1], Ts[f:f + 1])
        g0, g1 = full["good_ptr"][f], full["good_ptr"][f + 1]
        assert np.array_equal(single["good_rows"], full["good_rows"][g0:g1])
        assert np.array_equal(single["cloud_counts"], full["cloud_counts"][g0:g1])
        p0 = full["cloud_offsets"][g0] if g1 > g0 else 0
        assert np.array_equal(single["xyz"], full["xyz"][p0:p0 + single["xyz"].shape[0]])
        assert np.array_equal(single["depth"][0], full["depth"][f])


def test_device_inputs_equal_host_inputs():
    import torch
    w, h = 640, 480
    imgs, labs, Ts = NF.rooms(31, 8, w, h)
    cfg = NF.config(w, h, want_labels=1, want_depth=1)
    s = capi.PopupFrames(capi.load_library(), cfg)
    host = s.run(imgs, labs, Ts)
    dev = s.run(torch.from_numpy(imgs).cuda(), torch.from_numpy(labs).cuda(), torch.from_numpy(Ts).cuda())
    assert all(t.is_cuda for t in dev.values())
    NF.assert_same({k: v.cpu().numpy() for k, v in dev.items()}, host, where="device")


def test_refused_run_then_good_run():
    w, h = 640, 480
    imgs, labs, Ts = NF.rooms(41, 3, w, h)
    cfg = NF.config(w, h)
    lib = capi.load_library()
    s = capi.PopupFrames(lib, cfg)
    assert lib.pus_popup_session_run(s.h, -1, None, None, None) < 0 and b"n_frames" in lib.pus_last_error()
    assert lib.pus_popup_session_run(s.h, 2, None, None, None) < 0 and b"must be given" in lib.pus_last_error()
    NF.assert_same(s.run(imgs, labs, Ts), capi.PopupFrames(lib, cfg).run(imgs, labs, Ts), where="after refusal")
