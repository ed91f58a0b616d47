"""Writes tests/golden/popup_lines.npz: the expected output of pus_popup_lines (include/popup_gpu.h) on the reference's
four sample frames, seeded synthetic rooms and crafted frames, from a restatement written apart from the library's frame
code.  The per-pixel stages are live cv2 (4.13, Intel IPP switched off): cvtColor, mean, equalizeHist, resize,
GaussianBlur, Sobel, and gemm for the line fits' products; the walk, the fits' solves, the validation, nfa and the
orientation are restated here in Python.  Per-frame branch bits (the B_* values of pus_lines.cuh) are recorded, and the
crafted frames are there so that their union covers every bit.

    python tools/make_popup_line_golden.py [out.npz]
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAMES = os.path.join(ROOT, "tests", "golden", "popup_lines_frames")
SAMPLES = ["0050", "0115", "0185", "0700"]
MAX_LINES = 512   # PUS_POPUP_MAX_LINES

BITS = ["EQUALIZED", "ONE_BIN", "TURN", "BORDER", "SHORT", "BLOCKED", "FIT_FAIL", "FIT_NAN", "POPBACK",
        "TRYCAP", "BORDER_LINE", "NFA_REJECT", "NFA_NK", "NFA_ZERO", "ZERO_GRAD", "SWAP_Q0", "SWAP_Q1", "SWAP_Q2",
        "SWAP_Q3", "FLOAT_PI", "OVER_ANCHORS", "OVER_CHAINS", "OVER_PIXELS", "LINE_H", "LINE_V", "MANY", "HALVED"]
B = {k: 1 << i for i, k in enumerate(BITS)}
ALL_BITS = (1 << len(BITS)) - 1
UP, RIGHT, DOWN, LEFT = 1, 2, 3, 4


def cv():
    import cv2
    cv2.ipp.setUseIPP(False)
    return cv2


def prepare(cv2, img, ds):
    """grey, contrast, optional halving, blur (popup_plane.cpp:759-768, line_lbd_allclass.cpp:171-185, :811-812)"""
    bits = 0
    g = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if img.ndim == 3 else img.copy()
    if cv2.mean(g)[0] < 90:
        bits |= B["EQUALIZED"]
        if len(np.unique(g)) == 1:
            bits |= B["ONE_BIN"]
        g = cv2.equalizeHist(g)
    if ds:
        bits |= B["HALVED"]
        g = cv2.resize(g, None, fx=0.5, fy=0.5)
    return cv2.GaussianBlur(g, (5, 5), 1), bits


def gradient(cv2, b):
    dx = cv2.Sobel(b, cv2.CV_16S, 1, 0, ksize=3)
    dy = cv2.Sobel(b, cv2.CV_16S, 0, 1, ksize=3)
    s = cv2.add(np.abs(dx), np.abs(dy))
    _, t = cv2.threshold(s, 81, 255, cv2.THRESH_TOZERO)
    g = cv2.multiply(t, 0.25)          # saturate_cast<short>(v * 0.25f)
    return dx, dy, g, np.abs(dx) < np.abs(dy)


def chains(b, dx, dy, g, horiz, bits):
    """EdgeDrawing (binary_descriptor.cpp:1579-2377); returns (status, [chain pixel lists of (x, y)])"""
    h, w = g.shape
    n = w * h
    plim, clim = n // 5, (n // 5) // 20
    G = g.astype(np.int64).ravel().tolist()
    Hz = horiz.ravel().tolist()
    anchors = []
    for x in range(1, w - 1, 2):
        for y in range(1, h - 1, 2):
            i = y * w + x
            v = G[i]
            if Hz[i]:
                ok = v >= G[i - w] + 8 and v >= G[i + w] + 8
            else:
                ok = v >= G[i - 1] + 8 and v >= G[i + 1] + 8
            if ok:
                anchors.append((x, y))
    if len(anchors) > plim:
        return 1, [], bits | B["OVER_ANCHORS"]
    mark = [0] * n          # 1 marked, 2 marked by a dropped chain
    state = {"lx": 0, "ly": 0, "bits": bits}

    def walk(x, y, last):
        out = []
        while True:
            i = y * w + x
            if G[i] <= 0:
                break
            if mark[i]:
                if mark[i] == 2:
                    state["bits"] |= B["BLOCKED"]
                break
            mark[i] = 1
            out.append((x, y))
            if Hz[i]:
                should = 0
                if last in (UP, DOWN):
                    should = RIGHT if x > state["lx"] else LEFT
                    state["bits"] |= B["TURN"]
                state["lx"], state["ly"] = x, y
                if last == RIGHT or should == RIGHT:
                    if x == w - 1 or y == 0 or y == h - 1:
                        state["bits"] |= B["BORDER"]
                        break
                    nb = [(x + 1, y - 1), (x + 1, y), (x + 1, y + 1)]
                    last = RIGHT
                else:
                    if x == 0 or y == 0 or y == h - 1:
                        state["bits"] |= B["BORDER"]
                        break
                    nb = [(x - 1, y - 1), (x - 1, y), (x - 1, y + 1)]
                    last = LEFT
            else:
                should = 0
                if last in (RIGHT, LEFT):
                    should = DOWN if y > state["ly"] else UP
                    state["bits"] |= B["TURN"]
                state["lx"], state["ly"] = x, y
                if last == DOWN or should == DOWN:
                    if x == 0 or x == w - 1 or y == h - 1:
                        state["bits"] |= B["BORDER"]
                        break
                    nb = [(x + 1, y + 1), (x, y + 1), (x - 1, y + 1)]
                    last = DOWN
                else:
                    if x == 0 or x == w - 1 or y == 0:
                        state["bits"] |= B["BORDER"]
                        break
                    nb = [(x + 1, y - 1), (x, y - 1), (x - 1, y - 1)]
                    last = UP
            v1, v2, v3 = [G[q * w + p] & 0xff for p, q in nb]   # (unsigned char) of the short
            if v1 >= v2 and v1 >= v3:
                x, y = nb[0]
            elif v3 >= v2 and v3 >= v1:
                x, y = nb[2]
            else:
                x, y = nb[1]
        return out

    kept, n1, n2 = [], 0, 0
    for x, y in anchors:
        if mark[y * w + x]:
            continue
        first = walk(x, y, RIGHT if Hz[y * w + x] else DOWN)
        mark[y * w + x] = 0
        second = walk(x, y, LEFT if Hz[y * w + x] else UP)
        if len(first) + len(second) < 16:
            state["bits"] |= B["SHORT"]
            for p, q in first + second:
                mark[q * w + p] = 2
            continue
        n1 += len(first)
        n2 += len(second)
        if n1 > plim or n2 > plim:
            return 1, [], state["bits"] | B["OVER_PIXELS"]
        kept.append(first[::-1] + second[1:])
        if len(kept) > clim:
            return 1, [], state["bits"] | B["OVER_CHAINS"]
    return 0, kept, state["bits"]


def log_gamma(x):
    if x > 15.0:
        return 0.918938533204673 + (x - 0.5) * math.log(x) - x + 0.5 * x * math.log(
            x * math.sinh(1 / x) + 1 / (810.0 * math.pow(x, 6.0)))
    q = [75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511]
    a = (x + 0.5) * math.log(x + 5.5) - (x + 5.5)
    b = 0.0
    for n in range(7):
        a -= math.log(x + n)
        b += q[n] * math.pow(x, float(n))
    return a + math.log(b)


def nfa(n, k, p, logNT, st):
    """descriptor.hpp:763-844"""
    if n == 0 or k == 0:
        return -logNT
    if n == k:
        st["bits"] |= B["NFA_NK"]
        return -logNT - n * math.log10(p)
    p_term = p / (1.0 - p)
    log1term = (log_gamma(n + 1.0) - log_gamma(k + 1.0) - log_gamma((n - k) + 1.0) + k * math.log(p)
                + (n - k) * math.log(1.0 - p))
    term = math.exp(log1term)
    if term == 0.0 or abs(term) / max(abs(term), 2.2250738585072014e-308) <= 100.0 * 2.220446049250313e-16:
        st["bits"] |= B["NFA_ZERO"]
        return -log1term / 2.30258509299404568402 - logNT if k > n * p else -logNT
    bin_tail = term
    for i in range(k + 1, n + 1):
        bin_term = (n - i + 1) / i
        mult_term = bin_term * p_term
        term *= mult_term
        bin_tail += term
        if bin_term < 1.0:
            err = term * ((1.0 - math.pow(mult_term, float(n - i + 1))) / (1.0 - mult_term) - 1.0)
            if err < 0.1 * abs(-math.log10(bin_tail) - logNT) * bin_tail:
                break
    return -math.log10(bin_tail) - logNT


def products(cv2, X, Y):
    """fitMatT * fitMatT.t() and fitMatT * vec with live cv2.gemm on Mat_<float> (fitMatT = [X; 1])"""
    m = np.vstack([np.asarray(X, np.float32), np.ones(len(X), np.float32)])
    A = cv2.gemm(m, m, 1, None, 0, flags=cv2.GEMM_2_T)
    V = cv2.gemm(m, np.asarray(Y, np.float32).reshape(-1, 1), 1, None, 0)
    return A.astype(np.float32).ravel(), V.astype(np.float32).ravel()


def solve(A, V):
    """the 2 x 2 solve in double (a singular ATA gives inf / NaN as in C)"""
    A = [np.float64(v) for v in A]
    V = [np.float64(v) for v in V]
    with np.errstate(all="ignore"):
        coef = np.float64(1.0) / (A[0] * A[3] - A[1] * A[2])
        return coef * (A[3] * V[0] - A[1] * V[1]), coef * (A[0] * V[1] - A[2] * V[0])


def xy(horiz, p):
    return (p[0], p[1]) if horiz else (p[1], p[0])


def chain_lines(cv2, px, dx, dy, Hz, w, h, scale, st, margins):
    """EDline's loop body over one chain (binary_descriptor.cpp:2423-2619) and OctaveKeyLines' orientation"""
    logNT = 2.0 * (math.log10(w) + math.log10(h))
    n, S, out = len(px), 0, []
    err = 0.0
    while n > S + 15:
        while n > S + 15:
            hz = Hz[px[S][1]][px[S][0]]
            pts = [xy(hz, p) for p in px[S:S + 15]]
            A, V = products(cv2, [p[0] for p in pts], [p[1] for p in pts])
            a, b = solve(A, V)
            with np.errstate(all="ignore"):
                e2 = np.float64(0.0)
                for X, Y in pts:
                    c = (np.float64(Y) - np.float64(X) * a) - b
                    e2 += c * c
                err = float(np.sqrt(e2))
            if err <= 1.6:
                break
            st["bits"] |= B["FIT_NAN"] if math.isnan(err) else B["FIT_FAIL"]
            S += 2
        if not err <= 1.6:
            break
        l0 = S
        hz = bool(Hz[px[l0][1]][px[l0][0]])
        l, tries, first = l0, 0, True
        while True:
            tries += 1
            if first:
                first = False
                l += 15
                S += 15
            else:
                pts = [xy(hz, p) for p in px[new_s:l]]
                A2, V2 = products(cv2, [p[0] for p in pts], [p[1] for p in pts])
                A = (A + A2).astype(np.float32)
                V = (V + V2).astype(np.float32)
                a, b = solve(A, V)
            with np.errstate(all="ignore"):
                coef1 = float(1 / np.sqrt(a * a + 1) if hz else 1 / np.sqrt(1 + a * a))
            a, b = float(a), float(b)
            outl, new_s = 0, l
            while n > S:
                X, Y = px[S]
                d = abs((a * X - Y) + b) * coef1 if hz else abs((X - a * Y) - b) * coef1
                S += 1
                l += 1
                if d > 1.6:
                    outl += 1
                    if outl > 3:
                        break
                else:
                    outl = 0
            if outl:
                st["bits"] |= B["POPBACK"]
            l -= outl
            S -= outl
            if l - new_s > 0 and tries < 6:
                continue
            if l - new_s > 0:
                st["bits"] |= B["TRYCAP"]
            break
        eq = [a * coef1, -1 * coef1, b * coef1] if hz else [1 * coef1, -a * coef1, -b * coef1]
        line = px[l0:l]
        mgx = sum(int(dx[q][p]) for p, q in line)
        mgy = sum(int(dy[q][p]) for p, q in line)
        ax, ay = abs(eq[1]), abs(eq[0])
        if mgx == 0 and mgy == 0:
            st["bits"] |= B["ZERO_GRAD"]
            continue
        if mgx > 0 and mgy >= 0:
            dr = math.atan2(-ay, ax)
        elif mgx <= 0 and mgy > 0:
            dr = math.atan2(ay, ax)
        elif mgx < 0 and mgy <= 0:
            dr = math.atan2(ay, -ax)
        else:
            dr = math.atan2(-ay, -ax)
        direction = float(np.float32(dr))
        ad = abs(direction)
        if ad < 0.15 or math.pi - ad < 0.15:
            if abs(eq[2]) < 10 or abs(h - abs(eq[2])) < 10:
                st["bits"] |= B["BORDER_LINE"]
                continue
        if abs(ad - math.pi * 0.5) < 0.15:
            if abs(eq[2]) < 10 or abs(w - abs(eq[2])) < 10:
                st["bits"] |= B["BORDER_LINE"]
                continue
        k = 0
        for p, q in line:
            dis = abs(direction - math.atan2(-float(dx[q][p]), float(dy[q][p])))
            m = min(abs(abs(2 * math.pi - dis) - 0.392699), abs(dis - 0.392699))
            margins["angle"] = min(margins["angle"], m)
            if abs(2 * math.pi - dis) < 0.392699 or dis < 0.392699:
                k += 1
        r = nfa(len(line), k, 0.125, logNT, st)
        margins["nfa"] = min(margins["nfa"], abs(r))
        if not r > 0:
            st["bits"] |= B["NFA_REJECT"]
            continue
        st["bits"] |= B["LINE_H"] if hz else B["LINE_V"]
        a1, a2, a3, a4, a5 = eq[1] * eq[1], eq[0] * eq[0], eq[0] * eq[1], eq[2] * eq[0], eq[2] * eq[1]
        (P0x, P0y), (P1x, P1y) = line[0], line[-1]
        s1, s2 = np.float32(a1 * P0x - a3 * P0y - a4), np.float32(a2 * P0y - a3 * P0x - a5)
        e1, e2 = np.float32(a1 * P1x - a3 * P1y - a4), np.float32(a2 * P1y - a3 * P1x - a5)
        ddx, ddy = np.float32(e1 - s1), np.float32(e2 - s2)
        pi, swap = math.pi, False
        for lo, hi, cond, bit in ((-0.75 * pi, -0.25 * pi, ddy > 0, "SWAP_Q0"), (-0.25 * pi, 0.25 * pi, ddx < 0, "SWAP_Q1"),
                                  (0.25 * pi, 0.75 * pi, ddy < 0, "SWAP_Q2")):
            if lo <= direction < hi and cond:
                swap = True
                st["bits"] |= B[bit]
        if ((0.75 * pi <= direction < pi) or (-pi <= direction < -0.75 * pi)) and ddx > 0:
            swap = True
            st["bits"] |= B["SWAP_Q3"]
        if direction >= pi or direction < -pi:
            st["bits"] |= B["FLOAT_PI"]
        row = (e1, e2, s1, s2) if swap else (s1, s2, e1, e2)
        out.append([np.float32(np.float32(1) * v) * np.float32(scale) for v in row])
    return out


def detect(cv2, img, ds, margins=None):
    """one frame: (status, lines [n, 4] float32, bits)"""
    margins = margins if margins is not None else {"angle": math.inf, "nfa": math.inf}
    b, bits = prepare(cv2, img, ds)
    dx, dy, g, horiz = gradient(cv2, b)
    h, w = b.shape
    status, chs, bits = chains(b, dx, dy, g, horiz, bits)
    if status:
        return status, np.zeros((0, 4), np.float32), bits
    st = {"bits": bits}
    Hz, DX, DY = horiz.tolist(), dx.tolist(), dy.tolist()
    out = []
    for c in chs:
        out += chain_lines(cv2, c, DX, DY, Hz, w, h, 2.0 if ds else 1.0, st, margins)
    if len(out) > MAX_LINES:
        st["bits"] |= B["MANY"]
    return 0, np.asarray(out, np.float32).reshape(-1, 4), st["bits"]


# ---- frames ------------------------------------------------------------------------------------------------------------
def room(cv2, rng, w, h, channels):
    """a seeded room-like frame: a floor, walls, a few boxes and doors, noise"""
    img = np.zeros((h, w, 3), np.uint8)
    horizon = int(rng.integers(h // 3, 2 * h // 3))
    img[:horizon] = rng.integers(60, 200, 3)
    img[horizon:] = rng.integers(30, 160, 3)
    xs = sorted(rng.integers(0, w, 3).tolist())
    for x0, x1 in zip([0] + xs, xs + [w]):
        dy = int(rng.integers(-h // 10, h // 10))
        pts = np.array([[x0, 0], [x1, 0], [x1, horizon + dy], [x0, horizon - dy]], np.int32)
        cv2.fillPoly(img, [pts], tuple(int(v) for v in rng.integers(40, 230, 3)))
    for _ in range(int(rng.integers(3, 8))):
        x, y = int(rng.integers(0, w - 20)), int(rng.integers(0, h - 20))
        cv2.rectangle(img, (x, y), (x + int(rng.integers(10, w // 4)), y + int(rng.integers(10, h // 4))),
                      tuple(int(v) for v in rng.integers(0, 256, 3)), -1)
    for _ in range(int(rng.integers(2, 6))):
        p = rng.integers(0, [w, h], (2, 2))
        cv2.line(img, tuple(int(v) for v in p[0]), tuple(int(v) for v in p[1]),
                 tuple(int(v) for v in rng.integers(0, 256, 3)), int(rng.integers(1, 4)))
    img = np.clip(img.astype(np.int16) + rng.integers(-6, 7, img.shape), 0, 255).astype(np.uint8)
    if rng.random() < 0.3:
        img = (img * 0.55).astype(np.uint8)   # dark: the equalizeHist branch
    return img if channels == 3 else cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)


def crafted(cv2, w=160, h=120):
    """grey frames that take the rarer branches (their bits are asserted by the tests through the union)"""
    rng = np.random.default_rng(7)
    out = {}
    out["uniform"] = np.full((h, w), 40, np.uint8)
    m = np.full((h, w), 90, np.uint8)            # sum exactly 90 N: not below 90, no equalizeHist
    m[h // 4:h // 2, w // 4:w // 2] = 140
    m[h // 2:3 * h // 4, w // 2:3 * w // 4] = 40
    out["mean90"] = m
    out["noise"] = rng.integers(0, 256, (h, w), dtype=np.uint8)
    c = np.zeros((h, w), np.uint8)               # circles and diagonals: turns, swaps in every quadrant
    for r in range(10, min(w, h) // 2, 9):
        cv2.circle(c, (w // 2, h // 2), r, 255 if r % 2 else 120, 2)
    out["circles"] = c
    t = np.full((h, w), 200, np.uint8)           # lines hugging the border, exact horizontals and verticals
    t[:4] = 20
    t[:, -5:] = 20
    t[h // 2:, w // 3] = 20
    t[2 * h // 3, :] = 60
    out["border"] = t
    q = np.full((h, w), 128, np.uint8)           # four half-planes: each orientation of a step edge
    q[: h // 2, : w // 2] = 30
    q[h // 2:, w // 2:] = 230
    q[20:24, 20:w - 20] = 250
    q[h - 30:h - 26, 20:w - 20] = 10
    q[20:h - 20, 30:33] = 250
    q[20:h - 20, w - 40:w - 37] = 10
    out["steps"] = q
    k = rng.integers(0, 2, (h // 2, w // 2), dtype=np.uint8) * 255   # checkerboard noise: overflows
    out["checker"] = np.kron(k, np.ones((2, 2), np.uint8))
    out["fine"] = (np.indices((h, w)).sum(0) % 2 * 255).astype(np.uint8)
    a = np.zeros((100, 100), np.uint8)           # every scanned position an anchor: more than N / 5
    a[:, 2::4] = 255
    out["anchors"] = a
    p = np.zeros((400, 100), np.uint8)           # 30 full-height lines: more than N / 5 pixels in the first halves
    p[:, 2:60:4] = 255
    out["pixels"] = p
    c = np.zeros((400, 100), np.uint8)           # 1-pixel segments, two chains each: more than N / 100 chains
    for y in range(4, 380, 20):
        c[y:y + 16, 4:96:6] = 255
    out["chains"] = c
    big = np.zeros((480, 640), np.uint8)         # many short straight strokes: more than 512 lines
    for y in range(8, 472, 10):
        for x in range(8, 620, 40):
            cv2.line(big, (x, y), (x + 28, y + int(rng.integers(-3, 4))), 255, 2)
    out["many"] = big
    return out


CONFIGS = [  # (name, width, height, channels, downsample)
    ("room640", 640, 480, 3, 0), ("room640g", 640, 480, 1, 1), ("room960", 960, 540, 3, 1), ("room960g", 960, 540, 1, 0)]


def frames(cv2, key):
    """the images of a sample or room batch (not stored in the fixture): the sample PNGs, or two seeded rooms"""
    if key.startswith("sample"):
        return [cv2.imread(os.path.join(FRAMES, f"rgb_{key[6:10]}.png"))]
    ci = [c[0] for c in CONFIGS].index(key)
    _, w, h, ch, _ = CONFIGS[ci]
    rng = np.random.default_rng(100 + ci)
    return [room(cv2, rng, w, h, ch) for _ in range(2)]


def main(out_path):
    cv2 = cv()
    data, union = {}, 0
    margins = {"angle": math.inf, "nfa": math.inf}

    def put(key, imgs, ds):
        nonlocal union
        st, cnt, L, bits = [], [], [], []
        for im in imgs:
            s, lines, b = detect(cv2, im, ds, margins)
            st.append(s)
            cnt.append(len(lines))
            L.append(lines)
            bits.append(b)
            union |= b
        if key.startswith("crafted"):   # the sample frames and rooms are rebuilt by frames()
            data[f"{key}_images"] = np.asarray(imgs)
        data[f"{key}_downsample"] = np.int32(ds)
        data[f"{key}_status"] = np.asarray(st, np.int32)
        data[f"{key}_counts"] = np.asarray(cnt, np.int32)
        data[f"{key}_lines"] = np.concatenate(L).astype(np.float32).reshape(-1, 4)
        data[f"{key}_bits"] = np.asarray(bits, np.uint32)

    for n in SAMPLES:
        put(f"sample{n}", frames(cv2, f"sample{n}"), 0)
        put(f"sample{n}_ds", frames(cv2, f"sample{n}"), 1)
    for name, w, h, ch, ds in CONFIGS:
        put(name, frames(cv2, name), ds)
    for name, im in crafted(cv2).items():
        put(f"crafted_{name}", [im], 0)
        if im.shape[0] % 2 == 0 and im.shape[1] % 2 == 0 and name in ("circles", "checker"):
            put(f"crafted_{name}_ds", [im], 1)
    data["keys"] = np.array(sorted({k.rsplit("_", 1)[0] for k in data if k.endswith("_status")}))
    data["margin_angle"] = np.float64(margins["angle"])
    data["margin_nfa"] = np.float64(margins["nfa"])
    np.savez_compressed(out_path, **data)
    missing = [k for k in BITS if not union & B[k]]
    print(f"wrote {out_path}: {len(data['keys'])} batches, margins angle {margins['angle']:.3g} nfa {margins['nfa']:.3g}, "
          f"bits not taken: {missing}")
    return missing


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "popup_lines.npz"))
