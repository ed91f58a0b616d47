"""Writes tests/golden/popup_edges.npz, the fixture of pus_popup_edges' CPU oracle (tests/popup_edges_oracle.cpp).

A second restatement of popup_plane::edge_get_polygons (select_edge.cpp:66-406) and of the Python it calls
(pop_up_fun.py:85-205), written separately from pus_edges.cuh:
  - stage 0 with live OpenCV (cv2 4.13): cv2.resize 0.5x INTER_NEAREST, cv2.dilate / cv2.erode with a ones kernel, 255 - v;
  - stage 1 with scikit-image 0.14's find_contours restated in Python: its marching-squares case table and its
    _assemble_contours, dicts and deques included, so points shared by several chains behave as they did there;
  - stages 2-4 in numpy float32 scalars, float64 where the reference computes in double;
  - the interval stage with intervaltree 2.x's semantics on Python objects, with NumPy 1.x's promotion made explicit
    (a float32 scalar with a Python number gave float64).
Frames: 640x480 and 960x540 label maps, downsample_contour on and off, with a ground region under a random polyline,
noise blobs and thin ground structures; the lines are the boundary's pieces split and jittered plus vertical, short, far,
duplicated and overlapping distractors (the generator's own polyline ground, not make_popup_polygon_golden.frame());
crafted frames reach every status.  A fixed number of frames is drawn per setting (seeded); the tests check that together
they take every branch bit of pus_edges.cuh except the two of points shared by several chains (STALE, MATERIALIZE), which
the crafted-map tests of tests/test_popup_edges.py reach.

    python tools/make_popup_edge_golden.py [out.npz]
"""
import math
import os
import sys
from collections import deque

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pop_up_slam_b200.capi import EDGE_DEFAULTS  # noqa: E402

f32 = np.float32
PI = 3.14159265
BITS = ["JOIN_APPEND", "JOIN_PREPEND", "CLOSE", "STALE", "MERGE_END", "MERGE_BEGIN", "DELETE_COVER", "DELETE_CONTOUR",
        "SPLIT", "DUPLICATE", "PIECE_MERGE", "REFINE", "SHORT", "BIND", "POST_MERGE", "EXTEND_KEPT", "EXTEND_REVERTED",
        "CONNECT", "MATERIALIZE"]
B = {k: 1 << i for i, k in enumerate(BITS)}


class Status(Exception):
    pass


# ---- stage 0 ------------------------------------------------------------------------------------------------------------
def preprocess(cv2, lab, P):
    if P["downsample_contour"]:
        m = cv2.resize(lab, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_NEAREST)
        m = cv2.erode(cv2.dilate(m, np.ones((8, 8), np.uint8)), np.ones((8, 8), np.uint8))
    else:
        m = cv2.dilate(lab, np.ones((P["dilation_distance"],) * 2, np.uint8))
        m = cv2.erode(m, np.ones((P["erosion_distance"],) * 2, np.uint8))
    return (255 - m.astype(np.int32)).astype(np.uint8)


# ---- stage 1: skimage 0.14 find_contours(map, 0) --------------------------------------------------------------------------
def _frac(a, b):
    return 0.0 if b == a else (0.0 - a) / (b - a)


def marching_squares(m):
    a = m.astype(np.float64)
    out = []
    cs = (a[:-1, :-1] > 0) * 1 + (a[:-1, 1:] > 0) * 2 + (a[1:, :-1] > 0) * 4 + (a[1:, 1:] > 0) * 8
    for r0, c0 in zip(*np.nonzero((cs != 0) & (cs != 15))):
        r0, c0 = int(r0), int(c0)
        r1, c1 = r0 + 1, c0 + 1
        ul, ur, ll, lr = a[r0, c0], a[r0, c1], a[r1, c0], a[r1, c1]
        top, bottom = (r0, c0 + _frac(ul, ur)), (r1, c0 + _frac(ll, lr))
        left, right = (r0 + _frac(ul, ll), c0), (r0 + _frac(ur, lr), c1)
        s = cs[r0, c0]
        seq = {1: [top, left], 2: [right, top], 3: [right, left], 4: [left, bottom], 5: [top, bottom],
               6: [right, top, left, bottom], 7: [right, bottom], 8: [bottom, right], 9: [top, left, bottom, right],
               10: [bottom, top], 11: [bottom, left], 12: [left, right], 13: [top, right], 14: [left, top]}[s]
        out += seq
    return out


def assemble(points, bits):
    current_index = 0
    contours, starts, ends = {}, {}, {}
    joined = set()   # ids of deques absorbed by a join (for the STALE bit only)
    it = iter(points)
    for from_point, to_point in zip(it, it):
        if from_point == to_point:
            continue
        tail_data, head_data = starts.get(to_point), ends.get(from_point)
        if tail_data is not None and head_data is not None:
            tail, tail_num = tail_data
            head, head_num = head_data
            if id(tail) in joined or id(head) in joined or tail_num not in contours or head_num not in contours:
                bits[0] |= B["STALE"]
            if tail is head:
                bits[0] |= B["CLOSE"]
                head.append(to_point)
            elif tail_num > head_num:
                bits[0] |= B["JOIN_APPEND"]
                head.extend(tail)
                joined.add(id(tail))
                ends.pop(tail[-1])
                contours.pop(tail_num, None)
                starts[head[0]] = (head, head_num)
                ends[head[-1]] = (head, head_num)
            else:
                bits[0] |= B["JOIN_PREPEND"]
                tail.extendleft(reversed(head))
                joined.add(id(head))
                starts.pop(head[0])
                contours.pop(head_num, None)
                starts[tail[0]] = (tail, tail_num)
                ends[tail[-1]] = (tail, tail_num)
        elif tail_data is None and head_data is None:
            current_index += 1
            new_contour = deque((from_point, to_point))
            contours[current_index] = new_contour
            starts[from_point] = (new_contour, current_index)
            ends[to_point] = (new_contour, current_index)
        elif tail_data is not None:
            tail, tail_num = tail_data
            if id(tail) in joined or tail_num not in contours:
                bits[0] |= B["STALE"]
            tail.appendleft(from_point)
            starts[from_point] = (tail, tail_num)
        else:
            head, head_num = head_data
            if id(head) in joined or head_num not in contours:
                bits[0] |= B["STALE"]
            head.append(to_point)
            ends[to_point] = (head, head_num)
    return [np.array(c) for _, c in sorted(contours.items())]


def ground_contour(m, scale, bits=None):
    """python_get_contours on a preprocessed map, times scale, as float32 (x, y); None without a contour"""
    bits = bits if bits is not None else [0]
    try:
        contours = assemble(marching_squares(m), bits)
    except KeyError:
        return None
    if not contours:
        return None
    lengths = np.array([np.linalg.norm(c[0, :] - c[-1, :]) for c in contours])
    c = contours[int(np.argmax(lengths))]
    g = c[:, ::-1][0:-1:20]
    return (g * scale).astype(f32)


# ---- stages 2-4 ---------------------------------------------------------------------------------------------------------
def norm(x, y):
    return f32(np.sqrt(f32(f32(x * x) + f32(y * y))))


def angle(dx, dy):
    a = f32(math.atan2(float(dy), float(dx)))
    ang = f32(float(a) / PI * 180.0)
    return f32(ang - f32(180)) if ang > 90 else (f32(ang + f32(180)) if ang < -90 else ang)


def adiff(a, b):
    d = f32(abs(f32(a - b)))
    e = f32(f32(180) - d)
    return e if e < d else d


def cdist(l, C):
    mx = None
    for k in range(10):
        s = f32(k / 10.0)
        px, py = f32(l[0] + f32(s * f32(l[2] - l[0]))), f32(l[1] + f32(s * f32(l[3] - l[1])))
        dx, dy = C[:, 0] - px, C[:, 1] - py
        mn = np.sqrt(dx * dx + dy * dy).astype(f32).min()
        mx = mn if mx is None or mn > mx else mx
    return mx


def distproj(b0, b1, e0, e1, q0, q1):
    ln = norm(e0 - b0, e1 - b1)
    if float(ln) < 0.001:
        return norm(q0 - b0, q1 - b1), f32(-1)
    t = f32(f32(f32(f32((q0 - b0) * (e0 - b0)) + f32((q1 - b1) * (e1 - b1))) / ln) / ln)
    px, py = f32(b0 + f32(t * f32(e0 - b0))), f32(b1 + f32(t * f32(e1 - b1)))
    return norm(q0 - px, q1 - py), f32(1) if t > 1 else (f32(0) if t < 0 else t)


def dist_line(b, e, q):
    ln = norm(e[0] - b[0], e[1] - b[1])
    if float(ln) < 0.001:
        return norm(q[0] - b[0], q[1] - b[1])
    t = f32(f32(f32(f32((q[0] - b[0]) * (e[0] - b[0])) + f32((q[1] - b[1]) * (e[1] - b[1]))) / ln) / ln)
    return norm(q[0] - f32(b[0] + f32(t * f32(e[0] - b[0]))), q[1] - f32(b[1] + f32(t * f32(e[1] - b[1]))))


def trunc(v):
    v = float(v)
    return int(v) if -2147483648.0 <= v < 2147483648.0 else -2 ** 31


def hit(pt, d, w, h):
    px, py, dx, dy = (f32(v) for v in (*pt, *d))
    for cond, num, den, axis, lim in ((dy < 0, -float(py), dy, 0, w), (dy > 0, h - 1.0 - float(py), dy, 0, w),
                                      (dx > 0, w - 1.0 - float(px), dx, 1, h), (dx < 0, -float(px), dx, 1, h)):
        if cond:
            lam = f32(num / float(den))
            if lam >= 0:
                q = (f32(px + f32(lam * dx)), f32(py + f32(lam * dy)))
                if 0 <= trunc(q[axis]) <= lim - 1:
                    return q
    return (f32(-1), f32(-1))


def intervals(G, P, bits):
    """interval_tree_optimization with intervaltree 2.x semantics; G rows of float32"""
    lens = [norm(g[2] - g[0], g[3] - g[1]) for g in G]
    data = [tuple(float(v) for v in g) for g in G]
    tree = set()

    def add(i):
        b, e = G[i][0], G[i][2]
        iv = (b, e, data[i])
        if iv in tree:
            return
        if not b < e:
            raise Status(3)
        tree.add(iv)

    def inter(i):
        q0, q1 = G[i][0], G[i][2]
        if not q0 < q1:
            return 0
        s = 0
        for b, e, _ in sorted(iv for iv in tree if iv[0] < q1 and iv[1] > q0):
            s = float(s) + float(min(f32(q1 - b), f32(e - q0), f32(abs(f32(q1 - q0))), f32(e - b)))
        return s

    open_list = list(range(len(G)))
    best = int(np.argmax([lens[i] for i in open_list]))
    add(open_list.pop(best))
    while open_list:
        pot = [k for k, i in enumerate(open_list) if inter(i) < P["interval_overlap_thre"]]
        if not pot:
            break
        bb = int(np.argmax([lens[open_list[k]] for k in pot]))
        add(open_list.pop(pot[bb]))
    raw = len(tree)
    bounds = sorted({iv[0] for iv in tree} | {iv[1] for iv in tree})
    if len(bounds) > 2:
        tree = {(lb, ub, iv[2]) for lb, ub in zip(bounds[:-1], bounds[1:]) for iv in tree if iv[0] <= lb < iv[1]}
    post = len(tree) != raw
    if post:
        bits[0] |= B["SPLIT"]
        al = sorted(tree)
        dele = set()
        for i in range(len(al)):
            for j in range(i + 1, len(al)):
                if al[i][0] == al[j][0] and al[i][1] == al[j][1]:
                    dele.add(al[i] if (al[i][2][2] - al[i][2][0]) < (al[j][2][2] - al[j][2][0]) else al[j])
        if dele:
            bits[0] |= B["DUPLICATE"]
        tree -= dele
        for _ in range(100):
            al, hitm = sorted(tree), False
            for i in range(len(al)):
                for j in range(i + 1, len(al)):
                    if (al[i][0] == al[j][1] or al[i][1] == al[j][0]) and al[i][2] == al[j][2]:
                        tree -= {al[i], al[j]}
                        tree.add((min(al[i][0], al[j][0]), max(al[i][1], al[j][1]), al[j][2]))
                        hitm = True
                        break
                if hitm:
                    break
            if not hitm:
                break
            bits[0] |= B["PIECE_MERGE"]
    out = []
    for b, e, d in sorted(tree):
        if post and (float(b) != d[0] or float(e) != d[2]):
            bits[0] |= B["REFINE"]
            f1 = (float(b) - d[0]) / (d[2] - d[0])   # np.float32 - float was float64 under NumPy 1.x
            f2 = (float(e) - d[0]) / (d[2] - d[0])
            out.append([b, f32(int(f1 * (d[3] - d[1]) + d[1])), e, f32(int(f2 * (d[3] - d[1]) + d[1]))])
        else:
            out.append([f32(v) for v in d])
    return out


def select(P, width, height, lines, C, bits):
    G = []
    for l in lines:
        l = [f32(v) for v in l]
        vx, vy = f32(l[2] - l[0]), f32(l[3] - l[1])
        if float(norm(vx, vy)) < P["pre_minium_len"]:
            continue
        bt = P["pre_boundary_thre"]
        if (l[0] < bt and l[2] < bt) or (l[0] > width - bt and l[2] > width - bt) or (l[1] < bt and l[3] < bt) or \
                (l[1] > height - bt and l[3] > height - bt):
            continue
        if not float(abs(f32(abs(angle(vx, vy)) - f32(90)))) > P["pre_vertical_thre"]:
            continue
        if not float(cdist(l, C)) < P["pre_contour_close_thre"]:
            continue
        G.append(l if l[0] <= l[2] else [l[2], l[3], l[0], l[1]])
    ang = lambda g: angle(f32(g[2] - g[0]), f32(g[3] - g[1]))  # noqa: E731
    for _ in range(100):
        done = False
        for s1 in range(len(G)):
            for s2 in range(s1 + 1, len(G)):
                if not float(adiff(ang(G[s1]), ang(G[s2]))) < P["pre_merge_angle_thre"]:
                    continue
                if float(norm(G[s1][2] - G[s2][0], G[s1][3] - G[s2][1])) < P["pre_merge_dist_thre"]:
                    G[s1] = G[s1][:2] + G[s2][2:]
                    bits[0] |= B["MERGE_END"]
                elif float(norm(G[s2][2] - G[s1][0], G[s2][3] - G[s1][1])) < P["pre_merge_dist_thre"]:
                    G[s1] = G[s2][:2] + G[s1][2:]
                    bits[0] |= B["MERGE_BEGIN"]
                else:
                    continue
                del G[s2]
                done = True
                break
            if done:
                break
        if not done:
            break
    for _ in range(100):
        done = False
        for s1 in range(len(G)):
            for s2 in range(s1 + 1, len(G)):
                a, b = G[s1], G[s2]
                if not float(adiff(ang(a), ang(b))) < P["pre_proj_angle_thre"]:
                    continue
                d1b, p1b = distproj(*b, a[0], a[1])
                d1e, p1e = distproj(*b, a[2], a[3])
                d2b, p2b = distproj(*a, b[0], b[1])
                d2e, p2e = distproj(*a, b[2], b[3])
                dt = P["pre_proj_dist_thre"]
                if not all(float(d) < dt for d in (d1b, d1e, d2b, d2e)):
                    continue
                c12, c21 = f32(abs(f32(p1b - p1e))), f32(abs(f32(p2b - p2e)))
                if not (float(c12) > P["pre_proj_cover_thre"] or float(c21) > P["pre_proj_cover_thre"]):
                    continue
                if float(min(c12, c21)) < P["pre_proj_cover_large_thre"]:
                    de = s2 if c12 > c21 else s1
                    bits[0] |= B["DELETE_COVER"]
                else:
                    de = s1 if cdist(a, C) > cdist(b, C) else s2
                    bits[0] |= B["DELETE_CONTOUR"]
                del G[de]
                done = True
                break
            if done:
                break
        if not done:
            break
    if not G:
        raise Status(2)
    O = intervals(G, P, bits)
    n0 = len(O)
    O = [o for o in O if float(norm(o[2] - o[0], o[3] - o[1])) > P["post_short_thre"]]
    if len(O) < n0:
        bits[0] |= B["SHORT"]
    if not O:
        raise Status(4)
    for _ in range(100):
        hb = False
        for s in range(len(O) - 1):
            if O[s][2] != O[s + 1][0] or O[s][3] != O[s + 1][1]:
                if float(norm(O[s][2] - O[s + 1][0], O[s][3] - O[s + 1][1])) < P["post_bind_dist_thre"]:
                    mx = f32(trunc(f32(f32(O[s][2] + O[s + 1][0]) / f32(2))))
                    my = f32(trunc(f32(f32(O[s][3] + O[s + 1][1]) / f32(2))))
                    O[s] = [O[s][0], O[s][1], mx, my]
                    O[s + 1] = [mx, my, O[s + 1][2], O[s + 1][3]]
                    bits[0] |= B["BIND"]
                    hb = True
        if not hb:
            break
    for _ in range(100):
        hm = False
        for s in range(len(O) - 1):
            a, b = O[s], O[s + 1]
            if not float(adiff(ang(a), ang(b))) < P["post_merge_angle_thre"]:
                continue
            t = P["post_merge_dist_thre"]
            c1, c2 = float(dist_line(b[:2], b[2:], a[:2])) < t, float(dist_line(b[:2], b[2:], a[2:])) < t
            c3, c4 = float(dist_line(a[:2], a[2:], b[:2])) < t, float(dist_line(a[:2], a[2:], b[2:])) < t
            if (c1 and c2) or (c3 and c4):
                O[s] = a[:2] + b[2:]
                del O[s + 1]
                bits[0] |= B["POST_MERGE"]
                hm = True
                break
        if not hm:
            break
    f, l = O[0], O[-1]
    os_, oe = f[:2], l[2:]
    ns = hit(f[2:], (f32(f[0] - f[2]), f32(f[1] - f[3])), width, height)
    ne = hit(l[:2], (f32(l[2] - l[0]), f32(l[3] - l[1])), width, height)
    O[0] = [f32(trunc(ns[0])), f32(trunc(ns[1]))] + O[0][2:]
    O[-1] = O[-1][:2] + [f32(trunc(ne[0])), f32(trunc(ne[1]))]
    bd0, bd1 = cdist(O[0], C), cdist(O[-1], C)
    for bd, first in ((bd0, True), (bd1, False)):
        if float(bd) > P["post_extend_thre"]:
            bits[0] |= B["EXTEND_REVERTED"]
            if first:
                O[0] = os_ + O[0][2:]
            else:
                O[-1] = O[-1][:2] + oe
        else:
            bits[0] |= B["EXTEND_KEPT"]
    conn, inc = [], []
    for s in range(len(O)):
        if s > 0 and (O[s - 1][2] != O[s][0] or O[s - 1][3] != O[s][1]):
            conn.append(O[s - 1][2:] + O[s][:2])
            bits[0] |= B["CONNECT"]
        inc.append(len(conn))
        conn.append(O[s])
    return np.array(O, f32).reshape(-1, 4), np.array(conn, f32).reshape(-1, 4), np.array(inc, np.int32)


def edges(cv2, lab, lines, P):
    """(status, open, connect, open_in_connect, bits) of one frame"""
    h, w = lab.shape
    bits = [0]
    m = preprocess(cv2, lab, P)
    C = ground_contour(m, 2 if P["downsample_contour"] else 1, bits)
    empty = (np.zeros((0, 4), f32), np.zeros((0, 4), f32), np.zeros(0, np.int32))
    if C is None or len(C) == 0:
        return (1, *empty, bits[0])
    try:
        return (0, *select(P, w, h, np.asarray(lines, f32).reshape(-1, 4), C, bits), bits[0])
    except Status as s:
        return (s.args[0], *empty, bits[0])


# ---- frames -------------------------------------------------------------------------------------------------------------
def frame(cv2, rng, w, h):
    """a label map with a ground region under a random polyline, blobs and thin structures, and its detected lines"""
    lab = np.zeros((h, w), np.uint8)
    k = int(rng.integers(2, 6))
    xs = np.sort(np.concatenate([[0, w - 1], rng.uniform(0.1, 0.9, k - 1) * w]))
    ys = rng.uniform(0.45, 0.8, len(xs)) * h
    poly = np.concatenate([np.stack([xs, ys], 1), [[w - 1, h - 1], [0, h - 1]]]).astype(np.int32)
    cv2.fillPoly(lab, [poly], 255)
    for _ in range(int(rng.integers(0, 5))):
        c = (int(rng.integers(0, w)), int(rng.integers(0, h)))
        cv2.circle(lab, c, int(rng.integers(2, 25)), int(rng.choice([0, 255, 127])), -1)
    for _ in range(int(rng.integers(0, 3))):   # thin ground lines that survive the closing
        p0 = (int(rng.integers(0, w)), int(rng.integers(0, h // 2)))
        cv2.line(lab, p0, (p0[0] + int(rng.integers(-80, 80)), p0[1] + int(rng.integers(20, 80))), 255, 1)
    L = []
    for i in range(len(xs) - 1):
        a, b = np.array([xs[i], ys[i]]), np.array([xs[i + 1], ys[i + 1]])
        cuts = np.sort(rng.uniform(0, 1, int(rng.integers(0, 3))))
        ts = np.concatenate([[0], cuts, [1]])
        for t0, t1 in zip(ts[:-1], ts[1:]):
            p, q = a + (b - a) * (t0 + 0.02), a + (b - a) * (t1 - 0.02)
            L.append(np.concatenate([p, q]) + rng.normal(0, 1.5, 4))
            if rng.random() < 0.3:
                L.append(L[-1][[2, 3, 0, 1]])               # reversed duplicate
            if rng.random() < 0.3:
                L.append(L[-1] + np.array([8, 2, 12, 2]) * rng.normal(1, 0.3))   # overlapping
    for _ in range(int(rng.integers(2, 10))):
        x, y = rng.uniform(0, w), rng.uniform(0, h)
        kind = rng.integers(0, 4)
        if kind == 0:
            L.append([x, y, x + rng.normal(0, 3), y + rng.uniform(30, 100)])   # vertical
        elif kind == 1:
            L.append([x, y, x + rng.uniform(2, 12), y + rng.uniform(-3, 3)])   # short
        elif kind == 2:
            L.append([x, rng.uniform(0, 0.3) * h, x + rng.uniform(30, 150), rng.uniform(0, 0.3) * h])   # far
        else:
            L.append([x, y, x + rng.uniform(-150, 150), y + rng.uniform(-40, 40)])
    L = np.array(L, np.float64)
    rng.shuffle(L)
    return lab, np.round(L * 4) / 4   # quarter pixels, as a sub-pixel detector's float output


def crafted(w, h):
    """(labels, lines) reaching statuses 1-4"""
    out = []
    out.append((np.zeros((h, w), np.uint8), np.array([[10, 300, 200, 310]], np.float64)))            # 1: all wall
    out.append((np.full((h, w), 255, np.uint8), np.array([[10, 300, 200, 310]], np.float64)))        # 1: all ground
    lab = np.zeros((h, w), np.uint8)
    lab[h // 2:] = 255
    out.append((lab, np.array([[100, 20, 300, 22]], np.float64)))                                     # 2: far from it
    out.append((lab, np.array([[100, h / 2, 300, h / 2 + 1], [150, h / 2 - 1, 400, h / 2 - 1],
                               [420, h / 2 + 2, 430, h / 2 - 30]], np.float64)))                       # merges
    out.append((lab, np.array([[100, h / 2, 118, h / 2]], np.float64)))                                # 4: too short
    out.append((lab, np.array([[200, h / 2 - 10, 120, h / 2 + 10], [200, h / 2 - 10, 230, h / 2 + 10],
                               [215, h / 2 - 10, 215.5, h / 2 + 30]], np.float64)))                    # merges
    out.append((lab, np.array([[300, h / 2 - 20, 300, h / 2 + 20]], np.float64)))                     # 3 where vertical
    return out                                                                                         # lines pass


CONFIGS = [((640, 480), dict(downsample_contour=1)), ((640, 480), dict(downsample_contour=0)),
           ((960, 540), dict(downsample_contour=1)), ((960, 540), dict(downsample_contour=0, dilation_distance=7,
                                                                          erosion_distance=13, post_extend_thre=50.0,
                                                                          pre_contour_close_thre=400.0,
                                                                          pre_vertical_thre=-1.0))]


def main():
    import cv2
    cv2.setUseOptimized(False)
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "popup_edges.npz")
    rng = np.random.default_rng(20261018)
    rec = {}
    seen_bits, seen_status = 0, set()
    for ci, ((w, h), over) in enumerate(CONFIGS):
        P = dict(EDGE_DEFAULTS, **over)
        frames = crafted(w, h)
        for _ in range(6):
            frames.append(frame(cv2, rng, w, h))
        labs, ptr, lines, res = [], [0], [], []
        for lab, L in frames:
            r = edges(cv2, lab, L, P)
            seen_bits |= r[4]
            seen_status.add(r[0])
            labs.append(lab)
            lines.append(np.asarray(L, np.float32).reshape(-1, 4))
            ptr.append(ptr[-1] + len(lines[-1]))
            res.append(r)
        rec[f"c{ci}_labels"] = np.array(labs)
        rec[f"c{ci}_line_ptr"] = np.array(ptr, np.int32)
        rec[f"c{ci}_lines"] = np.concatenate(lines)
        rec[f"c{ci}_params"] = np.array([P[k] for k in EDGE_DEFAULTS], np.float64)
        rec[f"c{ci}_status"] = np.array([r[0] for r in res], np.int32)
        rec[f"c{ci}_bits"] = np.array([r[4] for r in res], np.int64)
        rec[f"c{ci}_open_counts"] = np.array([len(r[1]) for r in res], np.int32)
        rec[f"c{ci}_connect_counts"] = np.array([len(r[2]) for r in res], np.int32)
        rec[f"c{ci}_open"] = np.concatenate([r[1] for r in res])
        rec[f"c{ci}_connect"] = np.concatenate([r[2] for r in res])
        rec[f"c{ci}_open_in_connect"] = np.concatenate([r[3] for r in res])
    missing = [k for k in BITS if not seen_bits & B[k]]
    print("statuses", sorted(seen_status), "branches not taken:", missing)
    # labels compress well: store them packed
    np.savez_compressed(out, **rec)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
