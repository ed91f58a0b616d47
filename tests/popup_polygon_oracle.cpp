// TEST INFRASTRUCTURE ONLY.  Scalar CPU restatement of popup_plane::find_2d_3d_closed_polygon for the device's
// pus_popup_polygons (include/popup_gpu.h), exported as orc_popup_polygons with the same argument list.  Compiled by the
// tests into a temporary library (tests/popup_polygon_native.py); nothing in the product links it.  Build with
// -ffp-contract=off so no FMA contraction changes the float32 rounding.
//
// Reference (relative to the reference checkout):
//   pop_up_wall/libs/popup_plane.cpp:551-579   get_plane_equation (world ground endpoints, sensor-frame planes)
//   pop_up_wall/libs/popup_plane.cpp:120-406   popup_plane::find_2d_3d_closed_polygon
//   pop_up_wall/libs/matrix_utils.cpp:229-270  direction_hit_boundary (nobottom = false)
//   pop_up_wall/libs/matrix_utils.cpp:506-568  lineSegmentIntersect_f2, polygon_overlap_func
//   pop_up_wall/libs/matrix_utils.cpp:596-713  find_correct_ground_seq, cut_wall_polygons
// plus OpenCV 4.13's cv::convexHull (Sklansky, Point2f, clockwise = false) and cv::pointPolygonTest (measureDist = false).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace {
thread_local std::string g_err;

struct P2 { float x, y; };
struct P3 { float x, y, z; };

// x86 cvttss2si: NaN or out of range gives INT_MIN
int trunc_i(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }
template <class T> int sgn(T a) { return (a > 0) - (a < 0); }

// ---- cv::convexHull (modules/imgproc/src/convhull.cpp) on Point2f, returnPoints, clockwise = false ---------------------
int sklansky(const P2* p, const int* ord, int start, int end, int* stack, int nsign, int sign2) {
  const int incr = end > start ? 1 : -1;
  int pprev = start, pcur = pprev + incr, pnext = pcur + incr;
  int stacksize = 3;
  if (start == end || (p[ord[start]].x == p[ord[end]].x && p[ord[start]].y == p[ord[end]].y)) {
    stack[0] = start;
    return 1;
  }
  stack[0] = pprev;
  stack[1] = pcur;
  stack[2] = pnext;
  end += incr;
  while (pnext != end) {
    const float cury = p[ord[pcur]].y, nexty = p[ord[pnext]].y, by = nexty - cury;
    if (sgn(by) != nsign) {
      const float ax = p[ord[pcur]].x - p[ord[pprev]].x, bx = p[ord[pnext]].x - p[ord[pcur]].x, ay = cury - p[ord[pprev]].y;
      // float, as for Point2f; the two chains' values are then exact negatives, so no point is kept by both
      const float convexity = ay * bx - ax * by;
      if (sgn(convexity) == sign2 && (ax != 0 || ay != 0)) {
        pprev = pcur;
        pcur = pnext;
        pnext += incr;
        stack[stacksize] = pnext;
        stacksize++;
      } else if (pprev == start) {
        pcur = pnext;
        stack[1] = pcur;
        pnext += incr;
        stack[2] = pnext;
      } else {
        stack[stacksize - 2] = pnext;
        pcur = pprev;
        pprev = stack[stacksize - 4];
        stacksize--;
      }
    } else {
      pnext += incr;
      stack[stacksize - 1] = pnext;
    }
  }
  return --stacksize;
}

// hull of p[0..n) into out (original points, OpenCV's order); returns the hull's size
int convex_hull(const P2* p, int n, P2* out) {
  if (n <= 0) return 0;
  std::vector<int> ord(n), stack(n + 2), hull(n);
  for (int i = 0; i < n; i++) ord[i] = i;
  // std::sort with CHullCmpPoints (x, then y, then address) is a total order on distinct addresses: any sort agrees
  for (int i = 1; i < n; i++) {
    const int k = ord[i];
    int j = i - 1;
    while (j >= 0) {
      const P2 a = p[ord[j]], b = p[k];
      const bool greater = a.x != b.x ? b.x < a.x : a.y != b.y ? b.y < a.y : k < ord[j];
      if (!greater) break;
      ord[j + 1] = ord[j];
      j--;
    }
    ord[j + 1] = k;
  }
  int miny = 0, maxy = 0;
  for (int i = 1; i < n; i++) {
    const float y = p[ord[i]].y;
    if (p[ord[miny]].y > y) miny = i;
    if (p[ord[maxy]].y < y) maxy = i;
  }
  int nout = 0;
  if (p[ord[0]].x == p[ord[n - 1]].x && p[ord[0]].y == p[ord[n - 1]].y) {
    hull[nout++] = ord[0];
  } else {
    int* tl = stack.data();
    int tlc = sklansky(p, ord.data(), 0, maxy, tl, -1, 1);
    int* tr = stack.data() + tlc;
    int trc = sklansky(p, ord.data(), n - 1, maxy, tr, -1, -1);
    std::swap(tl, tr);   // !clockwise
    std::swap(tlc, trc);
    for (int i = 0; i < tlc - 1; i++) hull[nout++] = ord[tl[i]];
    for (int i = trc - 1; i > 0; i--) hull[nout++] = ord[tr[i]];
    const int stop = trc > 2 ? tr[1] : tlc > 2 ? tl[tlc - 2] : -1;
    int* bl = stack.data();
    int blc = sklansky(p, ord.data(), 0, miny, bl, 1, -1);
    int* br = stack.data() + blc;
    int brc = sklansky(p, ord.data(), n - 1, miny, br, 1, 1);
    if (stop >= 0) {
      const int check = blc > 2 ? bl[1] : blc + brc > 2 ? br[2 - blc] : -1;
      if (check == stop || (check >= 0 && p[ord[check]].x == p[ord[stop]].x && p[ord[check]].y == p[ord[stop]].y)) {
        blc = std::min(blc, 2);
        brc = std::min(brc, 2);
      }
    }
    for (int i = 0; i < blc - 1; i++) hull[nout++] = ord[bl[i]];
    for (int i = brc - 1; i > 0; i--) hull[nout++] = ord[br[i]];
    // the cyclic shift that makes the hull's indices ascending or descending where one exists
    if (nout >= 3) {
      int min_idx = 0, max_idx = 0, lt = 0;
      for (int i = 1; i < nout; i++) {
        const int idx = hull[i];
        lt += hull[i - 1] < idx;
        if (lt > 1 && lt <= i - 2) break;
        if (idx < hull[min_idx]) min_idx = i;
        if (idx > hull[max_idx]) max_idx = i;
      }
      const int mmdist = std::abs(max_idx - min_idx);
      if ((mmdist == 1 || mmdist == nout - 1) && (lt <= 1 || lt >= nout - 2)) {
        const int ascending = (max_idx + 1) % nout == min_idx;
        const int i0 = ascending ? min_idx : max_idx;
        int j = i0;
        if (i0 > 0) {
          int i;
          for (i = 0; i < nout; i++) {
            const int cur = stack[i] = hull[j];
            const int next = hull[j + 1 < nout ? j + 1 : 0];
            if (i < nout - 1 && (ascending != (cur < next))) break;
            if (++j >= nout) j = 0;
          }
          if (i == nout) std::copy(stack.begin(), stack.begin() + nout, hull.begin());
        }
      }
    }
  }
  for (int i = 0; i < nout; i++) out[i] = p[hull[i]];
  return nout;
}

// cv::pointPolygonTest (modules/imgproc/src/geometry.cpp), Point2f contour, measureDist = false: 1 in, 0 on, -1 out
int point_polygon_test(const P2* c, int n, P2 pt) {
  if (n == 0) return -1;
  int counter = 0;
  P2 v = c[n - 1];
  for (int i = 0; i < n; i++) {
    const P2 v0 = v;
    v = c[i];
    if ((v0.y <= pt.y && v.y <= pt.y) || (v0.y > pt.y && v.y > pt.y) || (v0.x < pt.x && v.x < pt.x)) {
      if (pt.y == v.y && (pt.x == v.x || (pt.y == v0.y && ((v0.x <= pt.x && pt.x <= v.x) || (v.x <= pt.x && pt.x <= v0.x)))))
        return 0;
      continue;
    }
    double dist = (double)(pt.y - v0.y) * (v.x - v0.x) - (double)(pt.x - v0.x) * (v.y - v0.y);
    if (dist == 0) return 0;
    if (v.y < v0.y) dist = -dist;
    counter += dist > 0;
  }
  return counter % 2 == 0 ? -1 : 1;
}

// ---- the reference's geometry --------------------------------------------------------------------------------------
P2 hit_boundary(P2 pt, P2 d, int w, int h) {   // direction_hit_boundary, nobottom = false
  if (d.y < 0) {
    const float l = (float)((0.0 - pt.y) / d.y);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.x) && trunc_i(q.x) <= w - 1) return q;
    }
  }
  if (d.y > 0) {
    const float l = (float)(((double)h - 1.0 - pt.y) / d.y);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.x) && trunc_i(q.x) <= w - 1) return q;
    }
  }
  if (d.x > 0) {
    const float l = (float)(((double)w - 1.0 - pt.x) / d.x);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.y) && trunc_i(q.y) <= h - 1) return q;
    }
  }
  if (d.x < 0) {
    const float l = (float)((0.0 - pt.x) / d.x);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.y) && trunc_i(q.y) <= h - 1) return q;
    }
  }
  return P2{-1.f, -1.f};
}

// A = [R | t] (row-major 4x4) times (p, 1), divided by the fourth row (homo_to_real_coord)
P3 xform(const float* A, P3 p) {
  float h[4];
  for (int i = 0; i < 4; i++) h[i] = A[i * 4 + 0] * p.x + A[i * 4 + 1] * p.y + A[i * 4 + 2] * p.z + A[i * 4 + 3] * 1.0f;
  return P3{h[0] / h[3], h[1] / h[3], h[2] / h[3]};
}
P2 project(const float* K, P3 p) {
  float q[3];
  for (int i = 0; i < 3; i++) q[i] = K[i * 3 + 0] * p.x + K[i * 3 + 1] * p.y + K[i * 3 + 2] * p.z;
  return P2{q[0] / q[2], q[1] / q[2]};
}
float norm3(P3 a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }

// lineSegmentIntersect_f2 + polygon_overlap_func's hull of the common part of two closed polygons
int overlap(const P2* a, int na, const P2* b, int nb, P2* out) {
  std::vector<P2> sect, inside;
  for (int i = 0; i + 1 < na; i++)
    for (int j = 0; j + 1 < nb; j++) {
      const float X2_X1 = a[i + 1].x - a[i].x, Y2_Y1 = a[i + 1].y - a[i].y;
      const float X4_X3 = b[j + 1].x - b[j].x, Y4_Y3 = b[j + 1].y - b[j].y;
      const float X1_X3 = a[i].x - b[j].x, Y1_Y3 = a[i].y - b[j].y;
      const float ua = (X4_X3 * Y1_Y3 - Y4_Y3 * X1_X3) / (Y4_Y3 * X2_X1 - X4_X3 * Y2_Y1);
      const float ub = (X2_X1 * Y1_Y3 - Y2_Y1 * X1_X3) / (Y4_Y3 * X2_X1 - X4_X3 * Y2_Y1);
      const float ix = a[i].x + X2_X1 * ua, iy = a[i].y + Y2_Y1 * ua;
      const float ib = (float)((ua >= 0) && (ua <= 1) && (ub >= 0) && (ub <= 1));
      if ((ua >= 0) && (ua <= 1) && (ub >= 0) && (ub <= 1)) sect.push_back(P2{ix * ib, iy * ib});
    }
  std::vector<P2> corners(a, a + (na > 0 ? na - 1 : 0));
  corners.insert(corners.end(), b, b + (nb > 0 ? nb - 1 : 0));
  for (const P2& c : corners)
    if (point_polygon_test(a, na, c) >= 0 && point_polygon_test(b, nb, c) >= 0) inside.push_back(c);
  inside.insert(inside.end(), sect.begin(), sect.end());
  return convex_hull(inside.data(), (int)inside.size(), out);
}

// find_correct_ground_seq; returns the sequence length (0: none).  An index the reference would read past its hull with
// (one of the two ground vertices missing) also gives 0.
int ground_seq(const P2* q, int n, bool originkept, int* seq) {
  int first = -1, second = -1;
  for (int i = 0; i < n; i++)
    if ((double)std::fabs(q[i].y) < 1e-3) {
      if (originkept) {
        if ((double)std::fabs(q[i].x) < 1e-3) first = i;
        else second = i;
      } else {
        if (first == -1) first = i;
        else second = i;
      }
    }
  if (!(std::abs(first - second) == 1 || std::abs(first - second) == n - 1)) return 0;
  int inc = second - first;
  if (first == 0 && second == n - 1) inc = -1;
  if (first == n - 1 && second == 0) inc = 1;
  for (int j = 0; j < n + 1; j++) {
    int cur = first + j * inc;
    if (cur > n - 1) cur -= n;
    if (cur < 0) cur += n;
    if (cur < 0 || cur > n - 1) return 0;
    seq[j] = cur;
  }
  return n + 1;
}

// a wall polygon has at most 7 vertices: 6 x 4 edge crossings + 10 corners go into the hull
constexpr int kHullMax = 34;
constexpr int kCutMax = kHullMax + 1;

// cut_wall_polygons; returns the cut polygon's size; *code = 0 height only, 1 / 2 length from the start / end vertex,
// + 4 when the uncut polygon is returned
int cut_wall(const P3* P, int m, float ceiling, float walllength, P3 cam, P3* out, int* code) {
  const P3 d{P[1].x - P[0].x, P[1].y - P[0].y, P[1].z - P[0].z};
  const float z = d.x * d.x + d.y * d.y + d.z * d.z;
  P3 dir = d;
  if (z > 0) {
    const float s = std::sqrt(z);
    dir = P3{d.x / s, d.y / s, d.z / s};
  }
  const float L = norm3(d);
  std::vector<P2> poly(m);
  for (int i = 0; i < m; i++) {
    const P3 r{P[i].x - P[0].x, P[i].y - P[0].y, P[i].z - P[0].z};
    poly[i] = P2{r.x * dir.x + r.y * dir.y + r.z * dir.z, P[i].z};
  }
  const bool height_only = walllength < 0;
  float x0 = -1.f, x1 = L + 1;
  *code = 0;
  if (!height_only) {
    const float s0 = norm3(P3{cam.x - P[0].x, cam.y - P[0].y, cam.z - P[0].z});
    const float s1 = norm3(P3{cam.x - P[1].x, cam.y - P[1].y, cam.z - P[1].z});
    if (s0 < s1) {
      x1 = walllength;
      *code = 1;
    } else {
      x0 = poly[1].x - walllength;
      x1 = poly[1].x + 1;
      *code = 2;
    }
  }
  const P2 box[5] = {{x0, -1.f}, {x1, -1.f}, {x1, ceiling}, {x0, ceiling}, {x0, -1.f}};
  P2 hull[kHullMax];
  const int nh = overlap(poly.data(), m, box, 5, hull);
  int seq[kCutMax + 1];
  const int ns = ground_seq(hull, nh, height_only, seq);
  if (ns == 0) {
    *code += 4;
    std::copy(P, P + m, out);
    return m;
  }
  for (int i = 0; i < ns; i++) {
    const P2 h = hull[seq[i]];
    out[i] = P3{(P[0].x + h.x * dir.x) + h.y * 0.f, (P[0].y + h.x * dir.y) + h.y * 0.f, (P[0].z + h.x * dir.z) + h.y * 1.f};
  }
  return ns;
}

struct FrameOut {
  std::vector<std::vector<P2>> bound, cut;
  std::vector<std::vector<P3>> world;
  std::vector<int> codes;   // 4 per row, see orc_popup_polygon_codes
};

void frame_polygons(const float* segs, int n, const float* K, const float* invK, const float* T, int w, int h, float ceiling,
                    float walllength, FrameOut& o) {
  o.bound.assign(n + 1, {});
  o.cut.assign(n + 1, {});
  o.world.assign(n + 1, {});
  o.codes.assign(4 * (n + 1), -1);
  if (n <= 0) return;
  // get_plane_equation: ground plane in the sensor frame, world ground endpoints (z = 0), wall planes
  const float gw[4] = {0.f, 0.f, -1.f, 0.f};
  float gs[4];
  for (int i = 0; i < 4; i++) gs[i] = T[0 * 4 + i] * gw[0] + T[1 * 4 + i] * gw[1] + T[2 * 4 + i] * gw[2] + T[3 * 4 + i] * gw[3];
  std::vector<float> planes(4 * (n + 1));
  for (int i = 0; i < 4; i++) planes[i] = gs[i];
  std::vector<P3> Pw(2 * n);
  for (int s = 0; s < n; s++) {
    for (int k = 0; k < 2; k++) {
      const float x = segs[4 * s + 2 * k], y = segs[4 * s + 2 * k + 1];
      float ray[3];
      for (int i = 0; i < 3; i++) ray[i] = invK[i * 3 + 0] * x + invK[i * 3 + 1] * y + invK[i * 3 + 2] * 1.0f;
      const float frac = -gs[3] / (gs[0] * ray[0] + gs[1] * ray[1] + gs[2] * ray[2]);
      Pw[2 * s + k] = xform(T, P3{frac * ray[0], frac * ray[1], frac * ray[2]});
      Pw[2 * s + k].z = 0.f;
    }
    const P3 a = Pw[2 * s], b = Pw[2 * s + 1];
    const float t1[3] = {b.x - a.x, b.y - a.y, b.z - a.z};
    const float nrm[3] = {t1[1] * gw[2] - t1[2] * gw[1], t1[2] * gw[0] - t1[0] * gw[2], t1[0] * gw[1] - t1[1] * gw[0]};
    const float pw[4] = {nrm[0], nrm[1], nrm[2], -(nrm[0] * a.x + nrm[1] * a.y + nrm[2] * a.z)};
    for (int i = 0; i < 4; i++)
      planes[4 * (s + 1) + i] = T[0 * 4 + i] * pw[0] + T[1 * 4 + i] * pw[1] + T[2 * 4 + i] * pw[2] + T[3 * 4 + i] * pw[3];
  }
  // the camera inverse [R^T | -R^T t]
  float iT[16];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) iT[i * 4 + j] = T[j * 4 + i];
    iT[i * 4 + 3] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
  iT[12] = 0.f; iT[13] = 0.f; iT[14] = 0.f; iT[15] = 1.f;
  // up / down image directions of a world vertical at every endpoint and where they leave the image
  std::vector<P2> up(2 * n), down(2 * n);
  for (int e = 0; e < 2 * n; e++) {
    const P3 v0 = Pw[e], v1{Pw[e].x + 0.f, Pw[e].y + 0.f, Pw[e].z + 2.f};
    const P2 i0 = project(K, xform(iT, v0)), i1 = project(K, xform(iT, v1));
    P2 dir{i1.x - i0.x, i1.y - i0.y};
    if (dir.y > 0) dir = P2{-dir.x, -dir.y};
    const P2 pt{segs[2 * e], segs[2 * e + 1]};
    up[e] = hit_boundary(pt, dir, w, h);
    down[e] = hit_boundary(pt, P2{-dir.x, -dir.y}, w, h);
  }
  const float W1 = (float)(w - 1), H1 = (float)(h - 1);
  auto S = [&](int s, int c) { return segs[4 * s + c]; };
  // ground polygon (popup_plane.cpp:158-196)
  {
    std::vector<P2>& g = o.bound[0];
    for (int s = 0; s < n; s++) g.push_back(P2{S(s, 0), S(s, 1)});
    g.push_back(P2{S(n - 1, 2), S(n - 1, 3)});
    int s = n - 1;
    P2 eh = down[2 * s + 1];
    int c1, c2;
    if (S(s, 3) == H1 && S(s, 2) < W1) c1 = 0;
    else if (S(s, 2) == W1 && S(s, 3) <= H1) { g.push_back(P2{W1, H1}); c1 = 1; }
    else {
      c1 = 4;
      if (eh.x == W1) { g.push_back(eh); g.push_back(P2{W1, H1}); c1 = 2; }
      if (0 <= eh.x && eh.x < W1) { g.push_back(eh); c1 = 3; }
    }
    s = 0;
    const P2 bh = down[0];
    eh = down[1];
    if (S(s, 1) == H1 && S(s, 0) > 0) c2 = 0;
    else if (S(s, 0) == 0 && S(s, 1) <= H1) { g.push_back(P2{0.f, H1}); c2 = 1; }
    else {
      c2 = 4;
      if (bh.x == W1) { g.push_back(P2{0.f, H1}); g.push_back(eh); c2 = 2; }
      if (0 <= bh.x && bh.x < W1) { g.push_back(eh); c2 = 3; }
    }
    g.push_back(g[0]);
    o.codes[0] = 0; o.codes[1] = c1; o.codes[2] = c2;
    o.cut[0] = g;
  }
  // wall polygons (popup_plane.cpp:198-344)
  for (int s = 0; s < n; s++) {
    std::vector<P2>& p = o.bound[s + 1];
    p.push_back(P2{S(s, 0), S(s, 1)});
    p.push_back(P2{S(s, 2), S(s, 3)});
    const P2 bh = up[2 * s], eh = up[2 * s + 1];
    int kind, outer = 2, inner = 5;
    auto general = [&]() {
      if (bh.x == W1 && eh.x == W1) { p.push_back(eh); p.push_back(bh); inner = 0; }
      if (0 < bh.x && bh.x < W1 && eh.x == W1) { p.push_back(eh); p.push_back(P2{W1, 0.f}); p.push_back(bh); inner = 1; }
      if (0 < bh.x && bh.x < W1 && 0 < eh.x && eh.x < W1) { p.push_back(eh); p.push_back(bh); inner = 2; }
      if (bh.x == 0 && 0 < eh.x && eh.x < W1) { p.push_back(eh); p.push_back(P2{0.f, 0.f}); p.push_back(bh); inner = 3; }
      if (bh.x == 0 && eh.x == 0) { p.push_back(eh); p.push_back(bh); inner = 4; }
    };
    auto right_begin = [&]() {
      inner = 3;
      if (bh.x == W1) { p.push_back(bh); inner = 0; }
      if (0 < bh.x && bh.x < W1) { p.push_back(P2{W1, 0.f}); p.push_back(bh); inner = 1; }
      if (bh.x == 0) { p.push_back(P2{W1, 0.f}); p.push_back(P2{0.f, 0.f}); p.push_back(bh); inner = 2; }
    };
    auto left_end = [&]() {
      inner = 3;
      if (eh.x == W1) { p.push_back(eh); p.push_back(P2{W1, 0.f}); p.push_back(P2{0.f, 0.f}); inner = 0; }
      if (0 < eh.x && eh.x < W1) { p.push_back(eh); p.push_back(P2{0.f, 0.f}); inner = 1; }
      if (eh.x == 0) { p.push_back(eh); inner = 2; }
    };
    if (s == n - 1) {
      kind = 3;
      if (S(s, 3) == H1 && S(s, 2) < W1) { p.push_back(P2{W1, H1}); right_begin(); outer = 0; }
      else if (S(s, 2) == W1 && S(s, 3) <= H1) { right_begin(); outer = 1; }
      else general();
    } else if (0 < s && s < n - 1) {
      kind = 2;
      general();
    } else {
      kind = 1;
      if (S(s, 1) == H1 && S(s, 0) > 0) { left_end(); p.push_back(P2{0.f, H1}); outer = 0; }
      else if (S(s, 0) == 0 && S(s, 1) <= H1) { left_end(); outer = 1; }
      else general();
    }
    p.push_back(P2{S(s, 0), S(s, 1)});
    int* c = &o.codes[4 * (s + 1)];
    c[0] = kind; c[1] = outer; c[2] = inner;
  }
  // 3-D polygons on the walls, cut, and projected back (popup_plane.cpp:346-404)
  const P3 cam{T[3], T[7], T[11]};
  for (int r = 1; r <= n; r++) {
    const std::vector<P2>& p = o.bound[r];
    const int m = (int)p.size();
    const float* pl = &planes[4 * r];
    std::vector<P3> Q(m);
    for (int i = 0; i < m; i++) {
      float ray[3];
      for (int k = 0; k < 3; k++) ray[k] = invK[k * 3 + 0] * p[i].x + invK[k * 3 + 1] * p[i].y + invK[k * 3 + 2] * 1.0f;
      const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
      Q[i] = xform(T, P3{frac * ray[0], frac * ray[1], frac * ray[2]});
    }
    Q[0].z = 0.f;
    Q[1].z = 0.f;
    P3 cut[kCutMax];
    const int nc = cut_wall(Q.data(), m, ceiling, walllength, cam, cut, &o.codes[4 * r + 3]);
    o.world[r].assign(cut, cut + nc);
    for (int i = 0; i < nc; i++) o.cut[r].push_back(project(K, xform(iT, cut[i])));
  }
}

bool finite_all(const float* a, int n) {
  for (int i = 0; i < n; i++)
    if (!std::isfinite(a[i])) return false;
  return true;
}
}  // namespace

extern "C" {

const char* orc_popup_last_error(void) { return g_err.c_str(); }

// cv::convexHull of n points (2 floats each) into out; returns the hull's size
int orc_convex_hull(const float* pts, int n, float* out) {
  std::vector<P2> p(n > 0 ? n : 0), h(n > 0 ? n : 0);
  for (int i = 0; i < n; i++) p[i] = P2{pts[2 * i], pts[2 * i + 1]};
  const int m = convex_hull(p.data(), n, h.data());
  for (int i = 0; i < m; i++) { out[2 * i] = h[i].x; out[2 * i + 1] = h[i].y; }
  return m;
}

// cv::pointPolygonTest(contour, (x, y), false)
int orc_point_polygon_test(const float* contour, int n, float x, float y) {
  std::vector<P2> c(n > 0 ? n : 0);
  for (int i = 0; i < n; i++) c[i] = P2{contour[2 * i], contour[2 * i + 1]};
  return point_polygon_test(c.data(), n, P2{x, y});
}

// same arguments and outputs as pus_popup_polygons (the argument checks are the device library's; here only the shape)
int orc_popup_polygons(int, int n_frames, const int* seg_ptr, const float* segs, const float* K, const float* invK,
                       const float* Ts, int width, int height, float ceiling_threshold, float walllength_threshold,
                       int* bound_counts, int* cut_counts, int* world_counts, float* bound2d, float* cut2d, float* world3d,
                       long long bound_capacity, long long cut_capacity, long long world_capacity) {
  if (n_frames < 0 || !seg_ptr || !finite_all(K, 9) || !finite_all(invK, 9)) { g_err = "orc_popup_polygons: bad arguments"; return -1; }
  long long nb = 0, nc = 0, nw = 0;
  std::vector<float> B, Cc, Wd;
  FrameOut o;
  for (int f = 0; f < n_frames; f++) {
    const int n = seg_ptr[f + 1] - seg_ptr[f];
    frame_polygons(segs + 4 * (size_t)seg_ptr[f], n, K, invK, Ts + 16 * (size_t)f, width, height, ceiling_threshold,
                   walllength_threshold, o);
    for (int r = 0; r <= n; r++) {
      const int row = seg_ptr[f] + f + r;
      if (bound_counts) bound_counts[row] = (int)o.bound[r].size();
      if (cut_counts) cut_counts[row] = (int)o.cut[r].size();
      if (world_counts) world_counts[row] = (int)o.world[r].size();
      for (const P2& q : o.bound[r]) { B.push_back(q.x); B.push_back(q.y); }
      for (const P2& q : o.cut[r]) { Cc.push_back(q.x); Cc.push_back(q.y); }
      for (const P3& q : o.world[r]) { Wd.push_back(q.x); Wd.push_back(q.y); Wd.push_back(q.z); }
    }
  }
  nb = (long long)B.size() / 2; nc = (long long)Cc.size() / 2; nw = (long long)Wd.size() / 3;
  if ((bound2d && bound_capacity < nb) || (cut2d && cut_capacity < nc) || (world3d && world_capacity < nw)) {
    g_err = "orc_popup_polygons: capacity too small";
    return -1;
  }
  if (bound2d) std::memcpy(bound2d, B.data(), B.size() * sizeof(float));
  if (cut2d) std::memcpy(cut2d, Cc.data(), Cc.size() * sizeof(float));
  if (world3d) std::memcpy(world3d, Wd.data(), Wd.size() * sizeof(float));
  return 0;
}

// per row 4 ints: [kind, A, B, cut].  kind 0 ground, 1 leftmost, 2 middle, 3 rightmost wall.
//   ground: A = last segment's case (0 end on the bottom edge, 1 end on the right edge, 2 down hit on the right border,
//           3 down hit inside [0, w-1), 4 none of these), B = the first segment's (0 start on the bottom edge, 1 start on
//           the left edge, 2 down hit x == w-1, 3 down hit inside, 4 none); cut = -1
//   walls:  A = outer branch (0 on the bottom edge, 1 on the side edge, 2 the general split), B = the inner branch taken
//           (general: 0..4 in source order, 5 none; rightmost / leftmost edge branches: 0 hit x == w-1, 1 inside, 2 x == 0,
//           3 none), cut = 0 height only / 1 length from the start / 2 from the end, + 4 when the uncut polygon is kept
int orc_popup_polygon_codes(int n_frames, const int* seg_ptr, const float* segs, const float* K, const float* invK,
                            const float* Ts, int width, int height, float ceiling_threshold, float walllength_threshold,
                            int* codes) {
  FrameOut o;
  for (int f = 0; f < n_frames; f++) {
    const int n = seg_ptr[f + 1] - seg_ptr[f];
    frame_polygons(segs + 4 * (size_t)seg_ptr[f], n, K, invK, Ts + 16 * (size_t)f, width, height, ceiling_threshold,
                   walllength_threshold, o);
    std::copy(o.codes.begin(), o.codes.end(), codes + 4 * (size_t)(seg_ptr[f] + f));
  }
  return 0;
}

}  // extern "C"
