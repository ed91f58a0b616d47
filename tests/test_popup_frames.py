"""The pop-up session's host side: config and argument refusals, the missing-device error, and the glue rule the GPU tests
restate."""
import numpy as np
import pytest

import popup_frames_native as NF
from pop_up_slam_b200 import capi


def _lib():
    try:
        return capi.load_library()
    except Exception as e:   # the library is built by build()
        pytest.skip(str(e))


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.parametrize("over,why", [
    (dict(channels=2), "channels"), (dict(width=3), "at least 4"), (dict(fast_edges=1, width=641), "even"),
    (dict(edges=dict(downsample_contour=0, dilation_distance=0)), "dilation_distance"),
    (dict(want_depth=1, height=481), "even"), (dict(channels=1, want_rgb=1), "want_rgb"),
])
def test_config_refusals(over, why):
    lib = _lib()
    cfg = NF.config(640, 480, **{k: v for k, v in over.items() if k not in ("width", "height")})
    cfg.update({k: v for k, v in over.items() if k in ("width", "height")})
    with pytest.raises(capi.ApiError, match=why):
        capi.PopupFrames(lib, cfg)


def test_non_finite_camera_is_refused():
    cfg = NF.config(640, 480)
    cfg["invK"] = np.full((3, 3), np.nan, np.float32)
    with pytest.raises(capi.ApiError, match="finite"):
        capi.PopupFrames(_lib(), cfg)


@pytest.mark.skipif(_has_gpu(), reason="checks the error without a device")
def test_no_device_is_an_error():
    with pytest.raises(capi.ApiError, match="no CUDA device"):
        capi.PopupFrames(_lib(), NF.config(640, 480))


def test_null_session_calls_are_refused():
    lib = _lib()
    with pytest.raises(capi.ApiError):
        capi.PopupFrames(lib, NF.config(640, 480, channels=2))
    assert lib.pus_popup_session_run(None, 1, None, None, None) < 0
    assert lib.pus_popup_session_destroy(None) < 0
    assert b"NULL" in lib.pus_last_error()


def test_actual_filter_keeps_the_open_walls_named_by_open_in_connect():
    # one frame, 3 open segments, connected list with 2 connectors: open_in_connect = [0, 2, 4] keeps open walls 0 and 2
    good = np.array([1, 1, 1, 1], np.int32)
    out = NF.actual_filter(good, np.array([0, 3]), np.array([0, 2, 4]))
    assert out.tolist() == [1, 1, 0, 1]
    # without connectors nothing is dropped; the ground row is never touched
    out = NF.actual_filter(np.array([1, 0, 1], np.int32), np.array([0, 2]), np.array([0, 1]))
    assert out.tolist() == [1, 0, 1]


def test_rendered_rooms_are_seeded_and_labelled_below_the_polyline():
    a, b = NF.rooms(2, 3, 160, 120), NF.rooms(2, 3, 160, 120)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    imgs, labs, Ts = a
    assert imgs.shape == (3, 120, 160, 3) and labs.shape == (3, 120, 160) and Ts.shape == (3, 4, 4)
    assert set(np.unique(labs).tolist()) <= {0, 255} and (labs[:, -1] == 255).all()


# ---- the host oracle of the whole run (the session's glue header compiled for the host, linked to the stage oracles)
# against the stage oracles composed with the glue restated in Python ----

def _orcs():
    import oracle_api
    import popup_cloud_native as NC
    import popup_depth_native as ND
    import popup_edges_native as NE
    import popup_lines_native as NL
    import popup_polygon_native as NP
    return (NL.oracle_lib(), NE.oracle_lib(), oracle_api.oracle_lib(), NP.oracle_lib(), NC.oracle_lib(), ND.oracle_lib())


def _same(cfg, imgs, labs, Ts, where):
    got = NF.oracle_run(cfg, imgs, labs, Ts)
    NF.assert_same(got, NF.chain(_orcs(), imgs, labs, Ts, cfg, prefix="orc_"), where=where)
    return got


@pytest.mark.parametrize("fast", [0, 1])
@pytest.mark.parametrize("dsc", [0, 1])
def test_oracle_run_on_the_sample_frames(fast, dsc):
    dropped = 0
    for i, (imgs, labs, Ts) in enumerate(NF.samples()):
        h, w = labs.shape[1:]
        cfg = NF.config(w, h, fast_edges=fast, edges=dict(downsample_contour=dsc), want_labels=1, want_depth=1)
        got = _same(cfg, imgs, labs, Ts, f"sample {i}")
        raw = capi.popup_fit_frames(_orcs()[2], got["open_ptr"], got["open_segs"], cfg["invK"], Ts,
                                    cfg["plane_cam_dist_thre"], prefix="orc_")[3]
        dropped += int(((raw == 1) & (got["good"] == 0)).sum())
    if (fast, dsc) == (0, 1):
        assert dropped > 0   # connectors make open_in_connect skip a wall the fit finds good


@pytest.mark.parametrize("size,channels", [((640, 480), 3), ((960, 540), 3), ((960, 540), 1)])
def test_oracle_run_on_rendered_rooms(size, channels):
    w, h = size
    imgs, labs, Ts = NF.rooms(5 + w + channels, 5, w, h)   # frame 3 is dark: the equalizeHist branch
    if channels == 1:
        imgs = np.array([img.mean(axis=2).astype(np.uint8) for img in imgs])
    got = _same(NF.config(w, h, channels=channels, want_labels=1, want_depth=1), imgs, labs, Ts, f"rooms {size} {channels}")
    assert (got["status"] == 0).all() and len(got["xyz"]) > 0


def test_oracle_run_on_crafted_frames():
    w, h = 640, 480
    imgs, labs, Ts = NF.rooms(17, 4, w, h)
    labs[0] = 0                   # no ground
    imgs[1] = 90                  # uniform image: no lines
    got = _same(NF.config(w, h, want_labels=1, want_depth=1), imgs, labs, Ts, "crafted")
    assert got["good_ptr"][2] == 0
    got = _same(NF.config(w, h, plane_cam_dist_thre=0.01), imgs, labs, Ts, "far walls")
    assert (got["good_rows"] == 0).all()


def test_oracle_run_gives_the_over_limit_frame_its_status():
    import popup_lines_native as NL
    _, many, _, _ = [f for f in NL.fixture() if f[0] == "crafted_many"][0]
    h, w = many.shape[1:3]
    imgs, labs, Ts = NF.rooms(8, 3, w, h)
    grey = np.array([img.mean(axis=2).astype(np.uint8) for img in imgs])
    batch = np.concatenate([grey[:1], many.reshape(1, h, w), grey[1:]])
    got = _same(NF.config(w, h, channels=1, want_labels=1, want_depth=1), batch, np.concatenate([labs[:1], labs]),
                np.concatenate([Ts[:1], Ts]), "over limit")
    assert got["status"].tolist() == [0, 1, 0, 0] and got["edge_status"][1] == -1
    assert got["good_ptr"][2] == got["good_ptr"][1]


def test_run_refuses_inputs_of_another_shape():
    lib = _lib()
    if not _has_gpu():
        pytest.skip("needs a session")
    s = capi.PopupFrames(lib, NF.config(64, 48))
    imgs, labs, Ts = NF.rooms(1, 2, 64, 48)
    with pytest.raises(ValueError, match="images"):
        s.run(imgs[:, :, :32], labs, Ts)
    with pytest.raises(ValueError, match="labels"):
        s.run(imgs, labs[:1], Ts)
    with pytest.raises(ValueError, match="Ts"):
        s.run(imgs, labs, Ts[:1])
