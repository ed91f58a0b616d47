"""Writes tests/golden/popup_clouds.npz, the fixture of the dense plane clouds (pus_popup_clouds).

The pixel sets and label images come from OpenCV itself (the cv2 module, 4.13): the polygon truncated to cv::Point, its
boundingRect, fillConvexPoly on the box and findNonZero, as popup_plane::closed_polygons_homo_pts does
(pop_up_wall/libs/popup_plane.cpp:81-116), and the label image with its INTER_NEAREST 0.5x / 2x resize (:840-855).  The
points are a float32 numpy restatement of steps 2-3 (ray_plane_interact, the rigid transform, matrixToCloud's filters and
colours, :925-985), each operation rounded to float32 as the device's --fmad=false code rounds it.  cv2 is needed only here.
A polygon's pixel set is stored as its boundingRect and the filled box mask (packed bits): findNonZero's list is the
mask's nonzero pixels in row-major order plus the box offset.  The polygons are kept small so the file stays small.

    python tools/make_popup_cloud_golden.py [out.npz]
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import popup_cloud_native as N  # noqa: E402

DEPTH_THRE, CEILING = np.float32(5.0), np.float32(2.8)


def cv_fill(poly, downsample):
    """closed_polygons_homo_pts through OpenCV up to findNonZero: the boundingRect (x, y, w, h) and the filled box mask"""
    poly = np.asarray(poly, np.float32).reshape(-1, 2)
    if len(poly) == 0:
        return (0, 0, 0, 0), np.zeros((0, 0), np.uint8)
    f = poly / np.float32(2) if downsample else poly
    ip = np.trunc(f).astype(np.int32)
    bx, by, bw, bh = cv2.boundingRect(ip)
    sh = np.trunc(f - np.array([bx, by], np.float32)).astype(np.int32)
    img = np.zeros((bh, bw), np.uint8)
    cv2.fillConvexPoly(img, sh, 255)
    return (bx, by, bw, bh), img


def cv_pixels(poly, downsample):
    """[m, 2] int32 (x, y) image pixels in findNonZero order, with the box offset added back (doubled when downsampling)"""
    (bx, by, _, _), img = cv_fill(poly, downsample)
    nz = cv2.findNonZero(img) if img.size else None
    px = np.zeros((0, 2), np.int32) if nz is None else nz.reshape(-1, 2).astype(np.int32) + [bx, by]
    return px * (2 if downsample else 1)


def points(px, plane, T, K, img, width):
    """steps 2-3 in float32: (xyz [k, 3], rgb [k, 3]) of the kept pixels"""
    f32 = np.float32
    x, y = px[:, 0].astype(f32), px[:, 1].astype(f32)
    ray = [K[i, 0] * x + K[i, 1] * y + K[i, 2] * f32(1) for i in range(3)]
    frac = -plane[3] / (plane[0] * ray[0] + plane[1] * ray[1] + plane[2] * ray[2])
    ps = [frac * r for r in ray]
    pw = [T[i, 0] * ps[0] + T[i, 1] * ps[1] + T[i, 2] * ps[2] + T[i, 3] for i in range(3)]
    with np.errstate(invalid="ignore"):
        keep = ~((ps[2] < 0) | (ps[2] > DEPTH_THRE) | (pw[2].astype(np.float64) < -0.2))
    if img is not None and width == 960:
        keep &= ~((px[:, 0] < 4) | (px[:, 1] < 4))
    z = np.where(pw[2] < CEILING, pw[2], CEILING)
    xyz = np.stack([pw[0], pw[1], z], 1)[keep].astype(f32)
    h = img.shape[0] if img is not None else 0
    inside = (px[:, 0] >= 0) & (px[:, 0] < width) & (px[:, 1] >= 0) & (px[:, 1] < h)
    rgb = np.zeros((len(px), 3), np.uint8)
    if img is not None:
        rgb[inside] = img[px[inside, 1], px[inside, 0]][:, ::-1]
    return xyz, rgb[keep]


def label_image(pxs, width, height, downsample):
    lab = np.full((height, width), 127, np.uint8)
    for i, px in enumerate(pxs):
        ok = (px[:, 0] >= 0) & (px[:, 0] < width) & (px[:, 1] >= 0) & (px[:, 1] < height)
        lab[px[ok, 1], px[ok, 0]] = 255 if i == 0 else 0
    if downsample:
        lab = cv2.resize(lab, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_NEAREST)
        lab = cv2.resize(lab, None, fx=2, fy=2, interpolation=cv2.INTER_NEAREST)
    return lab


# (width, height, downsample, with image, number of walls, polygon extent)
CASES = [(640, 480, True, True, 4, 0.3), (640, 480, False, True, 3, 0.12), (960, 540, True, True, 4, 0.25),
         (960, 540, False, True, 3, 0.1), (640, 480, True, False, 4, 0.3), (960, 540, True, True, 5, 0.25),
         (640, 480, False, False, 2, 0.1), (640, 480, True, True, 6, 0.3)]


def straddling(rng, w, h):
    """a small polygon across a random image border or corner, so part of its pixels lie outside the image"""
    c = [[0, rng.uniform(0, h)], [w - 1, rng.uniform(0, h)], [rng.uniform(0, w), 0], [rng.uniform(0, w), h - 1], [0, 0],
         [w - 1, h - 1]][int(rng.integers(6))]
    a = np.sort(rng.uniform(0, 2 * np.pi, int(rng.integers(3, 7))))
    return (np.array(c) + rng.uniform(10, 30) * np.stack([np.cos(a), np.sin(a)], 1)).astype(np.float32)


def main(out):
    rng = np.random.default_rng(20261017)
    d = {"cv2_version": np.array(cv2.__version__), "depth_thre": DEPTH_THRE, "ceiling_threshold": CEILING}
    for c, (w, h, ds, with_img, nw, ext) in enumerate(CASES):
        polys, planes, T = N.random_frame(rng, w, h, nw, extent=ext)
        polys[-1] = straddling(rng, w, h)
        K = N.invK(w, h)
        img = N.image(c, w, h) if with_img else None
        fills = [cv_fill(p, ds) for p in polys]
        pxs = [cv_pixels(p, ds) for p in polys]
        pts = [points(px, planes[i], T, K, img, w) for i, px in enumerate(pxs)]
        d.update({f"{c}/size": np.array([w, h, int(ds), int(with_img)]), f"{c}/poly_ptr": np.cumsum([0] + [len(p) for p in polys]),
                  f"{c}/polys": np.concatenate(polys).reshape(-1, 2), f"{c}/planes": planes, f"{c}/T": T, f"{c}/invK": K,
                  f"{c}/boxes": np.array([b for b, _ in fills], np.int32).reshape(-1, 4),
                  f"{c}/masks": np.packbits(np.concatenate([m.reshape(-1) > 0 for _, m in fills])),
                  f"{c}/counts": np.array([len(x) for x, _ in pts], np.int32), f"{c}/xyz": np.concatenate([x for x, _ in pts]),
                  f"{c}/rgb": np.concatenate([r for _, r in pts]), f"{c}/labels": label_image(pxs, w, h, ds)})
        off = sum(int(((p < 0) | (p >= [w, h])).any(1).sum()) for p in pxs)
        print(f"case {c}: {w}x{h} downsample={ds} image={with_img} pixels={[len(p) for p in pxs]} off-image={off} "
              f"kept={d[f'{c}/counts'].tolist()}")
    d["n_cases"] = np.array(len(CASES))
    np.savez_compressed(out, **d)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "popup_clouds.npz"))
