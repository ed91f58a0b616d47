"""Writes tests/golden/popup_polygons.npz, the fixture of pus_popup_polygons' CPU oracle (tests/popup_polygon_oracle.cpp).

A second restatement of popup_plane::find_2d_3d_closed_polygon (popup_plane.cpp:120-406; matrix_utils.cpp:229-270,
506-713), written separately from the oracle: numpy float32 scalars (every operation rounded, sums left to right, as
Eigen's small products and the scalar code evaluate them), float64 where the reference computes in double, and live
OpenCV (cv2 4.13) for convexHull and pointPolygonTest.  Frames are synthetic (tests/popup_polygon_native.py): cameras
0.8-1.6 m high, pitched 5-25 degrees down with a small roll, 1-8 connected ground segments below the horizon with
endpoints snapped onto x = 0, x = w-1 and y = h-1, plus strong-roll frames squeezed into a bottom corner for the ground
polygon's border cases; 640x480 and 960x540; walllength -1, 3.0 and 0.5; ceiling 2.5 and 5.0.  Frames are added until
every branch of the ground, wall and cut splits has been taken.  A frame is left out when a vertex is not finite, or when
a hull input has three distinct points collinear only up to float rounding (neither on one row nor one column): OpenCV's
hull there depends on how its build rounds the orientation test, which pus_popup_polygons does not pin.

    python tools/make_popup_polygon_golden.py [out.npz]
"""
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import popup_polygon_native as N  # noqa: E402

f32 = np.float32
INT_MIN = -2 ** 31


class NearCollinear(Exception):
    pass


def cvtt(v):
    """(int)v as x86 cvttss2si computes it"""
    v = float(v)
    return int(v) if -2147483648.0 <= v < 2147483648.0 else INT_MIN


def mat_vec4(A, p):   # A (p, 1) with p a 3-vector, four terms left to right per row
    return [A[i, 0] * p[0] + A[i, 1] * p[1] + A[i, 2] * p[2] + A[i, 3] * f32(1) for i in range(4)]


def to_world(A, p):
    h = mat_vec4(A, p)
    return np.array([h[0] / h[3], h[1] / h[3], h[2] / h[3]], f32)


def to_image(K, p):
    q = [K[i, 0] * p[0] + K[i, 1] * p[1] + K[i, 2] * p[2] for i in range(3)]
    return np.array([q[0] / q[2], q[1] / q[2]], f32)


def ray(iK, x, y):
    return [iK[i, 0] * x + iK[i, 1] * y + iK[i, 2] * f32(1) for i in range(3)]


def hits(pt, d, w, h):
    """direction_hit_boundary(pt, d, w, h, nobottom = false); its lambdas are double, rounded to float"""
    for axis, cond, num in ((1, d[1] < 0, lambda: 0.0 - float(pt[1])), (1, d[1] > 0, lambda: h - 1.0 - float(pt[1])),
                            (0, d[0] > 0, lambda: w - 1.0 - float(pt[0])), (0, d[0] < 0, lambda: 0.0 - float(pt[0]))):
        if not cond:
            continue
        lam = f32(num() / float(d[axis]))
        if lam >= 0:
            q = np.array([pt[0] + lam * d[0], pt[1] + lam * d[1]], f32)
            other, lim = (0, w - 1) if axis == 1 else (1, h - 1)
            if 0 <= cvtt(q[other]) <= lim:
                return q
    return np.array([-1, -1], f32)


def check_hull_input(pts):
    p = np.asarray(pts, np.float64)
    for a, b, c in itertools.combinations(range(len(p)), 3):
        A, B, C = p[a], p[b], p[c]
        if (A == B).all() or (B == C).all() or (A == C).all():
            continue
        if A[0] == B[0] == C[0] or A[1] == B[1] == C[1]:
            continue
        u, v = B - A, C - A
        if abs(u[0] * v[1] - u[1] * v[0]) <= 1e-5 * np.linalg.norm(u) * np.linalg.norm(v):
            raise NearCollinear()


def overlap(cv2, a, b):
    """polygon_overlap_func: the hull of the shared corners and the edge crossings (lineSegmentIntersect_f2)"""
    sect = []
    with np.errstate(all="ignore"):
        for i in range(len(a) - 1):
            for j in range(len(b) - 1):
                d21, d43, d13 = a[i + 1] - a[i], b[j + 1] - b[j], a[i] - b[j]
                den = d43[1] * d21[0] - d43[0] * d21[1]
                ua = (d43[0] * d13[1] - d43[1] * d13[0]) / den
                ub = (d21[0] * d13[1] - d21[1] * d13[0]) / den
                if 0 <= ua <= 1 and 0 <= ub <= 1:
                    sect.append(np.array([a[i][0] + d21[0] * ua, a[i][1] + d21[1] * ua], f32) * f32(1))
    ca, cb = np.asarray(a, f32).reshape(-1, 1, 2), np.asarray(b, f32).reshape(-1, 1, 2)
    inside = [c for c in list(a[:-1]) + list(b[:-1])
              if cv2.pointPolygonTest(ca, (float(c[0]), float(c[1])), False) >= 0
              and cv2.pointPolygonTest(cb, (float(c[0]), float(c[1])), False) >= 0]
    inside += sect
    if not inside:
        return np.zeros((0, 2), f32)
    check_hull_input(inside)
    return cv2.convexHull(np.array(inside, f32).reshape(-1, 1, 2)).reshape(-1, 2)


def ground_sequence(q, originkept):
    """find_correct_ground_seq; None where it finds none (or would index past the hull)"""
    n = len(q)
    first = second = -1
    for i in range(n):
        if float(abs(q[i][1])) < 1e-3:
            if originkept:
                if float(abs(q[i][0])) < 1e-3:
                    first = i
                else:
                    second = i
            elif first == -1:
                first = i
            else:
                second = i
    if abs(first - second) not in (1, n - 1):
        return None
    inc = second - first
    if first == 0 and second == n - 1:
        inc = -1
    if first == n - 1 and second == 0:
        inc = 1
    out = []
    for j in range(n + 1):
        cur = first + j * inc
        cur = cur - n if cur > n - 1 else cur + n if cur < 0 else cur
        if not 0 <= cur < n:
            return None
        out.append(cur)
    return out


def cut_wall(cv2, P, ceiling, wl, cam):
    d = P[1] - P[0]
    z = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    u = d / np.sqrt(z) if z > 0 else d
    L = np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    flat = [np.array([(p - P[0])[0] * u[0] + (p - P[0])[1] * u[1] + (p - P[0])[2] * u[2], p[2]], f32) for p in P]
    height_only = wl < 0
    x0, x1, code = f32(-1), L + f32(1), 0
    if not height_only:
        def dist(p):
            e = cam - p
            return np.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
        if dist(P[0]) < dist(P[1]):
            x1, code = wl, 1
        else:
            x0, x1, code = flat[1][0] - wl, flat[1][0] + f32(1), 2
    box = [np.array(v, f32) for v in ((x0, -1), (x1, -1), (x1, ceiling), (x0, ceiling), (x0, -1))]
    hull = overlap(cv2, flat, box)
    seq = ground_sequence(hull, height_only)
    if seq is None:
        return [p.copy() for p in P], code + 4
    return [np.array([(P[0][k] + hull[i][0] * u[k]) + hull[i][1] * f32(k == 2) for k in range(3)], f32) for i in seq], code


def frame(cv2, segs, K, iK, T, w, h, ceiling, wl):
    """the three polygon lists of one frame, its branch cases {(kind, A, B, cut)} and its sensor-frame planes (row order)"""
    n = len(segs)
    gw = [f32(0), f32(0), f32(-1), f32(0)]
    gs = [T[0, i] * gw[0] + T[1, i] * gw[1] + T[2, i] * gw[2] + T[3, i] * gw[3] for i in range(4)]
    ends, planes = [], [gs]
    for s in range(n):
        e = []
        for k in range(2):
            r = ray(iK, segs[s, 2 * k], segs[s, 2 * k + 1])
            fr = -gs[3] / (gs[0] * r[0] + gs[1] * r[1] + gs[2] * r[2])
            p = to_world(T, [fr * r[0], fr * r[1], fr * r[2]])
            p[2] = 0
            e.append(p)
        t1 = e[1] - e[0]
        nv = [t1[1] * gw[2] - t1[2] * gw[1], t1[2] * gw[0] - t1[0] * gw[2], t1[0] * gw[1] - t1[1] * gw[0]]
        pw = nv + [-(nv[0] * e[0][0] + nv[1] * e[0][1] + nv[2] * e[0][2])]
        planes.append([T[0, i] * pw[0] + T[1, i] * pw[1] + T[2, i] * pw[2] + T[3, i] * pw[3] for i in range(4)])
        ends.append(e)
    iT = np.zeros((4, 4), f32)
    iT[:3, :3] = T[:3, :3].T
    for i in range(3):
        iT[i, 3] = -(T[0, i] * T[0, 3] + T[1, i] * T[1, 3] + T[2, i] * T[2, 3])
    iT[3, 3] = 1

    def up(s, k):
        v0 = ends[s][k]
        v1 = np.array([v0[0] + f32(0), v0[1] + f32(0), v0[2] + f32(2)], f32)
        dv = to_image(K, to_world(iT, v1)) - to_image(K, to_world(iT, v0))
        return -dv if dv[1] > 0 else dv

    W1, H1 = f32(w - 1), f32(h - 1)
    pt = lambda s, k: segs[s, 2 * k:2 * k + 2]   # noqa: E731
    cases = set()
    # ground
    g = [pt(s, 0) for s in range(n)] + [pt(n - 1, 1)]
    last = segs[n - 1]
    if last[3] == H1 and last[2] < W1:
        a = 0
    elif last[2] == W1 and last[3] <= H1:
        g.append(np.array([W1, H1], f32)); a = 1
    else:
        eh = hits(pt(n - 1, 1), -up(n - 1, 1), w, h)
        a = 2 if eh[0] == W1 else 3 if 0 <= eh[0] < W1 else 4
        g += [eh, np.array([W1, H1], f32)] if a == 2 else [eh] if a == 3 else []
    first = segs[0]
    if first[1] == H1 and first[0] > 0:
        b = 0
    elif first[0] == 0 and first[1] <= H1:
        g.append(np.array([0, H1], f32)); b = 1
    else:
        bh, eh = hits(pt(0, 0), -up(0, 0), w, h), hits(pt(0, 1), -up(0, 1), w, h)
        b = 2 if bh[0] == W1 else 3 if 0 <= bh[0] < W1 else 4
        g += [np.array([0, H1], f32), eh] if b == 2 else [eh] if b == 3 else []
    g.append(g[0])
    bound, cut, world = [g], [g], [[]]
    cases.add((0, a, b, -1))
    corner = {"TR": np.array([W1, 0], f32), "TL": np.array([0, 0], f32), "BR": np.array([W1, H1], f32),
              "BL": np.array([0, H1], f32)}
    for s in range(n):
        bh, eh = hits(pt(s, 0), up(s, 0), w, h), hits(pt(s, 1), up(s, 1), w, h)
        inner = lambda x: 0 < x < W1   # noqa: E731
        general = [(bh[0] == W1 and eh[0] == W1, [eh, bh]), (inner(bh[0]) and eh[0] == W1, [eh, corner["TR"], bh]),
                   (inner(bh[0]) and inner(eh[0]), [eh, bh]), (bh[0] == 0 and inner(eh[0]), [eh, corner["TL"], bh]),
                   (bh[0] == 0 and eh[0] == 0, [eh, bh])]
        right = [(bh[0] == W1, [bh]), (inner(bh[0]), [corner["TR"], bh]), (bh[0] == 0, [corner["TR"], corner["TL"], bh])]
        left = [(eh[0] == W1, [eh, corner["TR"], corner["TL"]]), (inner(eh[0]), [eh, corner["TL"]]), (eh[0] == 0, [eh])]

        def take(options):
            hit = [i for i, (c, _) in enumerate(options) if c]
            return (hit[0], options[hit[0]][1]) if hit else (len(options), [])

        sg = segs[s]
        if s == n - 1:
            kind = 3
            if sg[3] == H1 and sg[2] < W1:
                outer, (inner_c, extra) = 0, take(right)
                extra = [corner["BR"]] + extra
            elif sg[2] == W1 and sg[3] <= H1:
                outer, (inner_c, extra) = 1, take(right)
            else:
                outer, (inner_c, extra) = 2, take(general)
        elif 0 < s < n - 1:
            kind, outer, (inner_c, extra) = 2, 2, take(general)
        else:
            kind = 1
            if sg[1] == H1 and sg[0] > 0:
                outer, (inner_c, extra) = 0, take(left)
                extra = extra + [corner["BL"]]
            elif sg[0] == 0 and sg[1] <= H1:
                outer, (inner_c, extra) = 1, take(left)
            else:
                outer, (inner_c, extra) = 2, take(general)
        poly = [pt(s, 0), pt(s, 1)] + extra + [pt(s, 0)]
        pl = planes[s + 1]
        Q = []
        for v in poly:
            r = ray(iK, v[0], v[1])
            fr = -pl[3] / (pl[0] * r[0] + pl[1] * r[1] + pl[2] * r[2])
            Q.append(to_world(T, [fr * r[0], fr * r[1], fr * r[2]]))
        Q[0][2] = 0
        Q[1][2] = 0
        wd, code = cut_wall(cv2, Q, ceiling, wl, np.array([T[0, 3], T[1, 3], T[2, 3]], f32))
        bound.append(poly)
        world.append(wd)
        cut.append([to_image(K, to_world(iT, p)) for p in wd])
        cases.add((kind, outer, inner_c, code))
    return bound, cut, world, cases, planes


def required(cases):
    """the branches the fixture must take: every ground case, every wall split and inner case, every cut mode and the
    fallback"""
    need = {("g_last", a) for a in range(5)} | {("g_first", b) for b in range(5)}
    need |= {("wall", k, o, i) for k in (1, 3) for o in (0, 1) for i in range(3)}
    need |= {("general", i) for i in range(5)} | {("cut", c) for c in range(3)} | {("fallback",)}
    have = set()
    for k, a, b, c in cases:
        if k == 0:
            have |= {("g_last", a), ("g_first", b)}
            continue
        if a < 2:
            have.add(("wall", k, a, b))
        else:
            have.add(("general", b))
        have |= {("cut", c % 4)} | ({("fallback",)} if c >= 4 else set())
    return need - have


def main():
    import cv2
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "popup_polygons.npz")
    rng = np.random.default_rng(2024)
    groups = {s: [] for s in N.SETTINGS}
    cases, skipped, tries = set(), 0, 0
    while True:
        for setting in N.SETTINGS:
            (w, h), c, wl = setting
            fr = N.corner_frame(rng, w, h) if tries % 3 == 2 else N.random_frame(rng, w, h)
            tries += 1
            b = N.batch([fr], w, h, c, wl)
            K, iK, T = b["K"], b["invK"], b["Ts"][0]
            try:
                with np.errstate(all="ignore"):
                    bound, cut, world, cs, _ = frame(cv2, fr[0], K, iK, T, w, h, f32(c), f32(wl))
            except NearCollinear:
                skipped += 1
                continue
            if not all(np.isfinite(np.asarray(v, np.float64)).all() for P in (bound, cut, world) for v in P if len(v)):
                skipped += 1
                continue
            new = required(cases) - required(cases | cs)
            if len(groups[setting]) < 6 or new:
                groups[setting].append((fr, bound, cut, world))
                cases |= cs
        if all(len(g) >= 6 for g in groups.values()) and not required(cases):
            break
        if tries > 200000:
            raise SystemExit(f"branches not reached: {sorted(required(cases))}")
    data = {"n_cases": len(N.SETTINGS)}
    for ci, (setting, frames) in enumerate(groups.items()):
        (w, h), c, wl = setting
        b = N.batch([f[0] for f in frames], w, h, c, wl)
        data[f"{ci}/setting"] = np.array([w, h, c, wl], np.float64)
        for k in ("seg_ptr", "segs", "K", "invK", "Ts"):
            data[f"{ci}/{k}"] = b[k]
        for name, idx, dim in (("bound", 1, 2), ("cut", 2, 2), ("world", 3, 3)):
            polys = [p for f in frames for p in f[idx]]
            data[f"{ci}/{name}_counts"] = np.array([len(p) for p in polys], np.int32)
            data[f"{ci}/{name}"] = np.array([v for p in polys for v in p], np.float32).reshape(-1, dim)
    np.savez_compressed(out, **data)
    print(f"wrote {out}: {sum(len(g) for g in groups.values())} frames, {skipped} left out, {tries} drawn")


if __name__ == "__main__":
    main()
