// TEST INFRASTRUCTURE ONLY.  Scalar CPU restatement of popup_plane::generate_cloud for the device's pus_popup_clouds
// (include/popup_gpu.h), exported as orc_popup_clouds with the same argument list.  Compiled by the tests into a temporary
// library (tests/popup_cloud_native.py); nothing in the product links it.  Build with -ffp-contract=off so no FMA
// contraction changes the float32 rounding.
//
// Reference (relative to the reference checkout):
//   pop_up_wall/libs/popup_plane.cpp:807-863  popup_plane::generate_cloud
//   pop_up_wall/libs/popup_plane.cpp:81-116   popup_plane::closed_polygons_homo_pts
//   pop_up_wall/libs/popup_plane.cpp:925-985  popup_plane::matrixToCloud
//   pop_up_wall/libs/matrix_utils.cpp:48-53   matrix_to_points (float -> cv::Point truncation)
//   pop_up_wall/libs/matrix_utils.cpp:189-193 ray_plane_interact
// The pixel set is OpenCV 4.13's cv::fillConvexPoly (LINE_8, shift 0) + cv::findNonZero, restated below as the scalar walk
// OpenCV runs: the outline drawn edge by edge with the 8-connected line iterator (clipped to the image), then the two-edge
// scanline fill.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {
thread_local std::string g_err;

// the line clip of cv::LineIterator (imgproc drawing): Cohen-Sutherland against [0, w) x [0, h) with truncating divisions
bool clip_line(int64_t w, int64_t h, int64_t& x1, int64_t& y1, int64_t& x2, int64_t& y2) {
  const int64_t right = w - 1, bottom = h - 1;
  if (w <= 0 || h <= 0) return false;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    int64_t a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (int64_t)((double)(a - y1) * (x2 - x1) / (y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (int64_t)((double)(a - y2) * (x2 - x1) / (y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (int64_t)((double)(a - x1) * (y2 - y1) / (x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (int64_t)((double)(a - x2) * (y2 - y1) / (x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// 8-connected line, iterated left to right (cv::LineIterator with leftToRight = true)
void draw_line(std::vector<uint8_t>& img, int w, int h, int x1, int y1, int x2, int y2) {
  if (x1 < 0 || x1 >= w || x2 < 0 || x2 >= w || y1 < 0 || y1 >= h || y2 < 0 || y2 >= h) {
    int64_t a = x1, b = y1, c = x2, d = y2;
    if (!clip_line(w, h, a, b, c, d)) return;
    x1 = (int)a; y1 = (int)b; x2 = (int)c; y2 = (int)d;
  }
  int dx = x2 - x1, dy = y2 - y1;
  if (dx < 0) { dx = -dx; dy = -dy; std::swap(x1, x2); std::swap(y1, y2); }
  int sy = 1;
  if (dy < 0) { dy = -dy; sy = -1; }
  const bool vert = dy > dx;
  if (vert) std::swap(dx, dy);
  int err = dx - 2 * dy;
  int x = x1, y = y1;
  for (int i = 0; i <= dx; i++) {
    img[(size_t)y * w + x] = 255;
    const bool minor = err < 0;
    err += -2 * dy + (minor ? 2 * dx : 0);
    if (vert) { y += sy; if (minor) x += 1; }
    else { x += 1; if (minor) y += sy; }
  }
}

// cv::fillConvexPoly(img, v, n, 255, LINE_8, 0)
void fill_convex_poly(std::vector<uint8_t>& img, int w, int h, const int* v, int n) {
  int px = v[2 * (n - 1)], py = v[2 * (n - 1) + 1];
  int xmin = v[0], xmax = v[0], ymin = v[1], ymax = v[1], imin = 0;
  for (int i = 0; i < n; i++) {
    const int x = v[2 * i], y = v[2 * i + 1];
    if (y < ymin) { ymin = y; imin = i; }
    ymax = std::max(ymax, y); xmax = std::max(xmax, x); xmin = std::min(xmin, x);
    draw_line(img, w, h, px, py, x, y);
    px = x; py = y;
  }
  if (n < 3 || xmax < 0 || ymax < 0 || xmin >= w || ymin >= h) return;
  ymax = std::min(ymax, h - 1);
  constexpr int SH = 16;
  struct { int idx, di; int64_t x, dx; int ye; } e[2];
  e[0].idx = e[1].idx = imin;
  e[0].ye = e[1].ye = ymin;
  e[0].di = 1; e[1].di = n - 1;
  e[0].x = e[1].x = -((int64_t)1 << SH);
  e[0].dx = e[1].dx = 0;
  int edges = n, y = ymin;
  do {
    for (int i = 0; i < 2; i++) {
      if (y < e[i].ye) continue;
      int idx0 = e[i].idx, di = e[i].di, idx = idx0 + di;
      if (idx >= n) idx -= n;
      for (; edges-- > 0;) {
        const int ty = v[2 * idx + 1];
        if (ty > y) {
          const int64_t xs = (int64_t)v[2 * idx0] << SH, xe = (int64_t)v[2 * idx] << SH;
          e[i].ye = ty;
          e[i].dx = ((xe - xs) * 2 + ((int64_t)ty - y)) / (2 * ((int64_t)ty - y));
          e[i].x = xs;
          e[i].idx = idx;
          break;
        }
        idx0 = idx;
        idx += di;
        if (idx >= n) idx -= n;
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int l = e[0].x > e[1].x ? 1 : 0, r = 1 - l;
      int x1 = (int)((e[l].x + (1 << (SH - 1))) >> SH), x2 = (int)((e[r].x + (1 << (SH - 1))) >> SH);
      if (x2 >= 0 && x1 < w) {
        if (x1 < 0) x1 = 0;
        if (x2 >= w) x2 = w - 1;
        std::memset(&img[(size_t)y * w + x1], 255, (size_t)(x2 - x1 + 1));
      }
    }
    e[0].x += e[0].dx;
    e[1].x += e[1].dx;
  } while (++y <= ymax);
}

struct Box { int x, y, w, h; };

// closed_polygons_homo_pts up to findNonZero: the pixel list (image coordinates) of one polygon, in findNonZero order
void polygon_pixels(const float* poly, int n, bool downsample, std::vector<int>& px) {
  px.clear();
  if (n <= 0) return;
  std::vector<float> f(2 * (size_t)n);
  std::vector<int> ip(2 * (size_t)n), sh(2 * (size_t)n);
  for (int i = 0; i < 2 * n; i++) f[i] = downsample ? poly[i] / 2.f : poly[i];
  for (int i = 0; i < 2 * n; i++) ip[i] = (int)f[i];
  Box b{ip[0], ip[1], 0, 0};
  int xmax = ip[0], ymax = ip[1];
  for (int i = 0; i < n; i++) {
    b.x = std::min(b.x, ip[2 * i]); xmax = std::max(xmax, ip[2 * i]);
    b.y = std::min(b.y, ip[2 * i + 1]); ymax = std::max(ymax, ip[2 * i + 1]);
  }
  b.w = xmax - b.x + 1;
  b.h = ymax - b.y + 1;
  for (int i = 0; i < n; i++) {
    sh[2 * i] = (int)(f[2 * i] - (float)b.x);
    sh[2 * i + 1] = (int)(f[2 * i + 1] - (float)b.y);
  }
  std::vector<uint8_t> img((size_t)b.w * b.h, 0);
  fill_convex_poly(img, b.w, b.h, sh.data(), n);
  const int s = downsample ? 2 : 1;
  for (int y = 0; y < b.h; y++)
    for (int x = 0; x < b.w; x++)
      if (img[(size_t)y * b.w + x]) { px.push_back((x + b.x) * s); px.push_back((y + b.y) * s); }
}
}  // namespace

extern "C" {

const char* orc_popup_last_error(void) { return g_err.c_str(); }

// pixel list of one polygon (2 ints per pixel); returns the pixel count, out = NULL or too small a capacity only counts
long long orc_popup_polygon_pixels(const float* poly, int n, int downsample, int* out, long long capacity) {
  std::vector<int> px;
  polygon_pixels(poly, n, downsample != 0, px);
  const long long m = (long long)px.size() / 2;
  if (out && capacity >= m) std::memcpy(out, px.data(), px.size() * sizeof(int));
  return m;
}

// same arguments and outputs as pus_popup_clouds
long long orc_popup_clouds(int, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                           const float* planes_sensor, const float* Ts, const float* invK, const unsigned char* images,
                           int width, int height, int downsample, float depth_thre, float ceiling_threshold, int* counts,
                           long long* offsets, float* xyz, unsigned char* rgb, long long capacity, unsigned char* labels) {
  if (n_frames < 0 || !plane_ptr || width <= 0 || height <= 0) { g_err = "orc_popup_clouds: bad arguments"; return -1; }
  const int n_planes = plane_ptr[n_frames];
  std::vector<long long> cnt(n_planes, 0);
  std::vector<float> P;   // xyz of every kept point
  std::vector<unsigned char> C;
  std::vector<int> px;
  const size_t wh = (size_t)width * height;
  std::vector<uint8_t> lab(labels ? wh : 0);
  for (int f = 0; f < n_frames; f++) {
    const float* T = Ts + 16 * (size_t)f;
    const unsigned char* img = images ? images + 3 * wh * f : nullptr;
    if (labels) std::fill(lab.begin(), lab.end(), 127);
    for (int p = plane_ptr[f]; p < plane_ptr[f + 1]; p++) {
      polygon_pixels(polys + 2 * (size_t)poly_ptr[p], poly_ptr[p + 1] - poly_ptr[p], downsample != 0, px);
      const float* pl = planes_sensor + 4 * (size_t)p;
      const int m = (int)px.size() / 2;
      for (int k = 0; k < m; k++) {
        const int x = px[2 * k], y = px[2 * k + 1];
        const bool inside = x >= 0 && x < width && y >= 0 && y < height;
        if (labels && inside) lab[(size_t)y * width + x] = p == plane_ptr[f] ? 255 : 0;   // popup_plane.cpp:840-847
        const float fx = (float)x, fy = (float)y;
        float ray[3];
        for (int i = 0; i < 3; i++) ray[i] = invK[i * 3 + 0] * fx + invK[i * 3 + 1] * fy + invK[i * 3 + 2] * 1.0f;
        const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
        float ps[3], pw[3];
        for (int i = 0; i < 3; i++) ps[i] = frac * ray[i];
        for (int i = 0; i < 3; i++) pw[i] = T[i * 4 + 0] * ps[0] + T[i * 4 + 1] * ps[1] + T[i * 4 + 2] * ps[2] + T[i * 4 + 3];
        // matrixToCloud, popup_plane.cpp:951-977
        if (ps[2] < 0 || ps[2] > depth_thre || (double)pw[2] < -0.2) continue;
        if (img && width == 960 && (x < 4 || y < 4)) continue;
        P.push_back(pw[0]);
        P.push_back(pw[1]);
        P.push_back(pw[2] < ceiling_threshold ? pw[2] : ceiling_threshold);
        const unsigned char* c = (img && inside) ? img + 3 * ((size_t)y * width + x) : nullptr;
        C.push_back(c ? c[2] : 0);
        C.push_back(c ? c[1] : 0);
        C.push_back(c ? c[0] : 0);
        cnt[p]++;
      }
    }
    if (labels) {
      unsigned char* out = labels + wh * f;
      if (downsample) {   // cv::resize 0.5x then 2x, INTER_NEAREST (popup_plane.cpp:852-855), even sizes
        for (int y = 0; y < height; y++)
          for (int x = 0; x < width; x++) out[(size_t)y * width + x] = lab[(size_t)(y / 2 * 2) * width + x / 2 * 2];
      } else {
        std::memcpy(out, lab.data(), wh);
      }
    }
  }
  const long long total = (long long)C.size() / 3;
  long long off = 0;
  for (int p = 0; p < n_planes; p++) {
    if (counts) counts[p] = (int)cnt[p];
    if (offsets) offsets[p] = off;
    off += cnt[p];
  }
  if ((xyz || rgb) && capacity < total) { g_err = "orc_popup_clouds: capacity too small"; return -1; }
  if (xyz) std::memcpy(xyz, P.data(), P.size() * sizeof(float));
  if (rgb) std::memcpy(rgb, C.data(), C.size());
  return total;
}

}  // extern "C"
