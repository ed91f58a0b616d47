"""Writes tests/golden/popup_depth.npz, the fixture of the pop-up depth map (pus_popup_depth).

A second restatement of popup_plane::get_depth_map_good (pop_up_wall/libs/popup_plane.cpp:866-921), written separately from
the oracle tests/popup_depth_oracle.cpp: numpy float32 arrays (every operation rounded), with the pixel lists from OpenCV
itself (cv2 4.13: truncation, boundingRect, fillConvexPoly and findNonZero, as tools/make_popup_cloud_golden.py runs them)
and the resize from live cv2.resize with Intel IPP switched off (cv2.ipp.setUseIPP(False)), which is OpenCV's own code.
convertTo(-1, 4) is not exposed to Python; it is x * 4 + 0 in float32.

Frames are 160x120 with a matching K: random frames (tests/popup_cloud_native.random_frame: the ground and 1-5 walls with
random, partly off-image polygons) and realistic ones, whose bound polygons and planes come from the polygon fixture's
restatement (tools/make_popup_polygon_golden.py) on synthetic ground lines.  Four settings: downsample on and off, ceilings
2.5, 5.0 and 0.4 (below every camera).  Frames are added until every branch has been taken: a plane's depth written, a
depth < 0 skipped over an earlier value, a ceiling depth written, a ceiling behind the camera skipped, a later plane
overwriting an earlier one, pixels off the image; every setting also has an empty polygon and a frame without planes.

    python tools/make_popup_depth_golden.py [out.npz]
"""
import importlib.util
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import popup_cloud_native as NC  # noqa: E402
import popup_depth_native as ND  # noqa: E402
import popup_polygon_native as NP  # noqa: E402

f32 = np.float32
W, H = 160, 120
SETTINGS = [(True, 2.5), (False, 5.0), (True, 0.4), (False, 0.4)]   # (downsample, ceiling)
BRANCHES = ("plane", "kept_after_depth_skip", "ceiling", "ceiling_skip", "overwrite", "off_image")


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


CLOUD, POLY = tool("make_popup_cloud_golden"), tool("make_popup_polygon_golden")


def depth_map(polys, planes, T, iK, ds, ceiling):
    """(map [H, W] float32 before the resize, branches taken)"""
    m = np.zeros((H, W), f32)
    src = np.zeros((H, W), np.int32)   # 0 untouched, else 1 + the writing plane
    taken = set()
    cw = np.array([0, 0, -1, ceiling], f32)
    cs = [T[0, i] * cw[0] + T[1, i] * cw[1] + T[2, i] * cw[2] + T[3, i] * cw[3] for i in range(4)]
    for k, (poly, pl) in enumerate(zip(polys, planes)):
        if len(poly) == 0:
            continue
        px = CLOUD.cv_pixels(poly, ds)
        ok = (px[:, 0] >= 0) & (px[:, 0] < W) & (px[:, 1] >= 0) & (px[:, 1] < H)
        if not ok.all():
            taken.add("off_image")
        px = px[ok]
        x, y = px[:, 0].astype(f32), px[:, 1].astype(f32)
        ray = [iK[i, 0] * x + iK[i, 1] * y + iK[i, 2] * f32(1) for i in range(3)]
        frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2])
        ps = [frac * r for r in ray]
        height = T[2, 0] * ps[0] + T[2, 1] * ps[1] + T[2, 2] * ps[2] + T[2, 3]
        cz = (-cs[3] / (cs[0] * ray[0] + cs[1] * ray[1] + cs[2] * ray[2])) * ray[2]
        low = height < ceiling
        write = np.where(low, ~(ps[2] < 0), ~(cz < 0))
        had = src[px[:, 1], px[:, 0]] > 0
        if (low & ~write & had).any():
            taken.add("kept_after_depth_skip")
        if (~low & ~write).any():
            taken.add("ceiling_skip")
        if (write & low).any():
            taken.add("plane")
        if (write & ~low).any():
            taken.add("ceiling")
        if (write & had).any():
            taken.add("overwrite")
        v = np.where(low, ps[2], cz).astype(f32)
        m[px[write, 1], px[write, 0]] = v[write]
        src[px[write, 1], px[write, 0]] = k + 1
    return m, taken


def resize_chain(m):
    h = cv2.resize(m, None, fx=0.5, fy=0.5)
    return cv2.resize(h * f32(4) + f32(0), None, fx=2, fy=2)


def realistic_frame(rng, ceiling):
    K = NP.camera_K(W, H)
    iK = np.linalg.inv(K.astype(np.float64)).astype(f32)
    segs, T = NP.random_frame(rng, W, H)
    bound, _, _, _, planes = POLY.frame(cv2, segs, K, iK, T, W, H, f32(ceiling), f32(-1))
    polys = [np.array(p, f32).reshape(-1, 2) for p in bound]
    if not all(np.isfinite(p).all() for p in polys):
        raise POLY.NearCollinear
    return polys, np.array(planes, f32), T


def main(out):
    cv2.ipp.setUseIPP(False)
    rng = np.random.default_rng(20261018)
    iK = NC.invK(W, H)
    cases, have, tries = [], set(), 0
    for ds, ceiling in SETTINGS:
        frames = []
        while len(frames) < 3 or (len(frames) < 6 and set(BRANCHES) - have):
            tries += 1
            try:
                with np.errstate(all="ignore"):
                    fr = realistic_frame(rng, ceiling) if len(frames) % 3 == 1 else \
                        NC.random_frame(rng, W, H, int(rng.integers(1, 5)), extent=0.6)
                    if len(frames) == 0:   # an empty polygon in the middle of the frame
                        fr = (fr[0][:1] + [np.zeros((0, 2), f32)] + fr[0][1:], np.insert(fr[1], 1, fr[1][0], 0), fr[2])
                    m, taken = depth_map(fr[0], fr[1], fr[2], iK, ds, f32(ceiling))
            except POLY.NearCollinear:
                continue
            if len(frames) >= 3 and not (taken - have):
                continue
            have |= taken
            frames.append(fr)
        frames.append(([], np.zeros((0, 4), f32), np.eye(4, dtype=f32)))   # a frame without planes
        b = ND.batch(frames, W, H, ds, ceiling)
        maps = []
        with np.errstate(all="ignore"):
            for polys, planes, T in frames:
                m, _ = depth_map(polys, planes, T, iK, ds, f32(ceiling))
                maps.append(resize_chain(m) if ds and len(polys) else m)
        cases.append((b, np.stack(maps)))
        print(f"downsample={ds} ceiling={ceiling}: {len(frames)} frames")
    missing = set(BRANCHES) - have
    if missing:
        raise SystemExit(f"branches not reached: {sorted(missing)}")
    d = {"cv2_version": np.array(cv2.__version__), "n_cases": np.array(len(cases))}
    for c, (b, maps) in enumerate(cases):
        for k in ("plane_ptr", "poly_ptr", "polys", "planes_sensor", "Ts", "invK"):
            d[f"{c}/{k}"] = b[k]
        d[f"{c}/setting"] = np.array([W, H, int(b["downsample"]), b["ceiling_threshold"]], np.float64)
        d[f"{c}/depth"] = maps
    np.savez_compressed(out, **d)
    print(out, os.path.getsize(out), "bytes,", tries, "frames drawn")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "popup_depth.npz"))
