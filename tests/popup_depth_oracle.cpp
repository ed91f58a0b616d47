// TEST INFRASTRUCTURE ONLY.  Scalar CPU restatement of popup_plane::get_depth_map_good for the device's pus_popup_depth
// (include/popup_gpu.h), exported as orc_popup_depth with the same argument list.  The pixel lists come from the clouds
// oracle's fill (tests/popup_cloud_oracle.cpp, compiled into this translation unit), so both oracles share one restatement of
// cv::fillConvexPoly + cv::findNonZero.  Compiled by the tests into a temporary library (tests/popup_depth_native.py); nothing
// in the product links it.  Build with -ffp-contract=off so no FMA contraction changes the float32 rounding.
//
// Reference (relative to the reference checkout):
//   pop_up_wall/libs/popup_plane.cpp:866-921  popup_plane::get_depth_map_good
//   pop_up_wall/libs/popup_plane.cpp:602-603  ceiling_plane_sensor = T^T (0, 0, -1, ceiling_threshold)
//   pop_up_wall/libs/matrix_utils.cpp:189-193 ray_plane_interact
// The resize chain (:912-916) is OpenCV 4.13's own code (IPP off): cv::resize 0.5x INTER_LINEAR, which OpenCV runs as its
// area fast path, ((s00 + s01) + (s10 + s11)) * 0.25f; convertTo(-1, 4), x * 4 + 0; cv::resize 2x INTER_LINEAR, separable,
// horizontal pass first, a * w0 + b * w1 per pass, with OpenCV's border handling (see resize2x).
#include "popup_cloud_oracle.cpp"

namespace {
// source codes of orc_popup_depth_codes (per pixel of the map before the resize)
constexpr int kCeiling = 1 << 16;      // the value came from the ceiling branch
constexpr int kKeptAfterSkip = 1 << 17;   // a later plane skipped the pixel (depth < 0 or ceiling behind) and it kept its value
constexpr int kOverwritten = 1 << 18;  // a later plane overwrote an earlier plane's value
constexpr int kDepthSkip = 1 << 19;    // some plane skipped it with depth < 0
constexpr int kCeilingSkip = 1 << 20;  // some plane skipped it with the ceiling behind the camera

// the map of one frame before the resize; codes (optional): low 16 bits 0 untouched or 1 + the plane's index in the frame,
// plus the flags above.  Returns the number of pixels that fell outside the image.
long long depth_frame(const int* pp, const int* poly_ptr, const float* polys, const float* planes, const float* T,
                      const float* invK, int width, int height, bool downsample, float ceiling, float* map, int* codes) {
  const float cw[4] = {0.f, 0.f, -1.f, ceiling};
  float cs[4];
  for (int i = 0; i < 4; i++) cs[i] = T[0 * 4 + i] * cw[0] + T[1 * 4 + i] * cw[1] + T[2 * 4 + i] * cw[2] + T[3 * 4 + i] * cw[3];
  std::vector<int> px;
  long long off = 0;
  for (int p = pp[0]; p < pp[1]; p++) {
    const int n = poly_ptr[p + 1] - poly_ptr[p];
    if (n == 0) continue;
    polygon_pixels(polys + 2 * (size_t)poly_ptr[p], n, downsample, px);
    const float* pl = planes + 4 * (size_t)p;
    for (size_t k = 0; k < px.size() / 2; k++) {
      const int x = px[2 * k], y = px[2 * k + 1];
      const float fx = (float)x, fy = (float)y;
      float ray[3], ps[3], pw[3];
      for (int i = 0; i < 3; i++) ray[i] = invK[i * 3 + 0] * fx + invK[i * 3 + 1] * fy + invK[i * 3 + 2] * 1.0f;
      const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
      for (int i = 0; i < 3; i++) ps[i] = frac * ray[i];
      for (int i = 0; i < 3; i++) pw[i] = T[i * 4 + 0] * ps[0] + T[i * 4 + 1] * ps[1] + T[i * 4 + 2] * ps[2] + T[i * 4 + 3];
      if (x < 0 || x >= width || y < 0 || y >= height) { off++; continue; }
      const size_t at = (size_t)y * width + x;
      int* c = codes ? codes + at : nullptr;
      float v;
      bool ceil_branch = false;
      if (pw[2] < ceiling) {
        if (ps[2] < 0) {
          if (c) *c |= kDepthSkip | ((*c & 0xffff) ? kKeptAfterSkip : 0);
          continue;
        }
        v = ps[2];
      } else {
        const float cf = -cs[3] / (cs[0] * ray[0] + cs[1] * ray[1] + cs[2] * ray[2]);
        v = cf * ray[2];
        if (v < 0) {
          if (c) *c |= kCeilingSkip | ((*c & 0xffff) ? kKeptAfterSkip : 0);
          continue;
        }
        ceil_branch = true;
      }
      map[at] = v;
      if (c) {
        const int flags = (*c & ~0xffff & ~kCeiling) | ((*c & 0xffff) ? kOverwritten : 0) | (ceil_branch ? kCeiling : 0);
        *c = flags | (p - pp[0] + 1);
      }
    }
  }
  return off;
}

// the half-size image after convertTo, at (r, c).  OpenCV's area fast path sums the 2 x 2 block pairwise in its 4-lane SIMD
// loop and left to right onto 0 in the scalar loop that finishes the last width % 4 columns; the two agree when three of the
// four pixels are +0, as in the depth map.
float quarter(const float* m, int w, int r, int c) {
  const float a = m[(size_t)(2 * r) * w + 2 * c], b = m[(size_t)(2 * r) * w + 2 * c + 1];
  const float d = m[(size_t)(2 * r + 1) * w + 2 * c], e = m[(size_t)(2 * r + 1) * w + 2 * c + 1];
  const int hw = w / 2;
  const float s = (c < hw / 4 * 4 ? (a + b) + (d + e) : 0.f + (((a + b) + d) + e)) * 0.25f;
  return s * 4.f + 0.f;
}

// OpenCV's 2x INTER_LINEAR on src [sh][sw]: source column of output column d is floor((d + 0.5) / 2 - 0.5) with weights
// (0.75, 0.25) or (0.25, 0.75).  Column borders: below 0 it is S[0] * 1 + S[1] * 0; at or past the last column S[last] * 1
// alone (a one-column source has only the latter).  Row borders take one row: R[0] * 1 or R[last] * 1.
void resize2x(const std::vector<float>& src, int sw, int sh, float* out) {
  const int w = 2 * sw;
  std::vector<float> hb((size_t)sh * w);
  for (int r = 0; r < sh; r++)
    for (int d = 0; d < w; d++) {
      const float* S = &src[(size_t)r * sw];
      float v;
      if (d == w - 1 || sw == 1) v = S[sw - 1] * 1.f;
      else if (d == 0) v = S[0] * 1.f + S[1] * 0.f;
      else {
        const int sx = (d & 1) ? d / 2 : d / 2 - 1;
        v = S[sx] * ((d & 1) ? 0.75f : 0.25f) + S[sx + 1] * ((d & 1) ? 0.25f : 0.75f);
      }
      hb[(size_t)r * w + d] = v;
    }
  for (int d = 0; d < 2 * sh; d++) {
    float* O = out + (size_t)d * w;
    if (d == 0 || d == 2 * sh - 1) {
      const float* R = &hb[(size_t)(d == 0 ? 0 : sh - 1) * w];
      for (int x = 0; x < w; x++) O[x] = R[x] * 1.f;
      continue;
    }
    const int sy = (d & 1) ? d / 2 : d / 2 - 1;
    const float w0 = (d & 1) ? 0.75f : 0.25f, w1 = (d & 1) ? 0.25f : 0.75f;
    for (int x = 0; x < w; x++) O[x] = hb[(size_t)sy * w + x] * w0 + hb[(size_t)(sy + 1) * w + x] * w1;
  }
}

// popup_plane.cpp:912-916 on an even-sized map, in place
void resize_chain(float* map, int width, int height) {
  const int hw = width / 2, hh = height / 2;
  std::vector<float> q((size_t)hw * hh);
  for (int r = 0; r < hh; r++)
    for (int c = 0; c < hw; c++) q[(size_t)r * hw + c] = quarter(map, width, r, c);
  resize2x(q, hw, hh, map);
}
}  // namespace

extern "C" {

// same arguments and output as pus_popup_depth
int orc_popup_depth(int, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys, const float* planes_sensor,
                    const float* Ts, const float* invK, int width, int height, int downsample, float ceiling_threshold,
                    float* depth) {
  if (n_frames < 0 || !plane_ptr || width <= 0 || height <= 0 || !depth || (downsample && ((width | height) & 1))) {
    g_err = "orc_popup_depth: bad arguments";
    return -1;
  }
  const size_t wh = (size_t)width * height;
  for (int f = 0; f < n_frames; f++) {
    float* map = depth + wh * f;
    std::fill(map, map + wh, 0.f);
    if (plane_ptr[f + 1] == plane_ptr[f]) continue;   // no good planes: all zero, not resized
    depth_frame(plane_ptr + f, poly_ptr, polys, planes_sensor, Ts + 16 * (size_t)f, invK, width, height, downsample != 0,
                ceiling_threshold, map, nullptr);
    if (downsample) resize_chain(map, width, height);
  }
  return 0;
}

// per-pixel source codes [n_frames][height][width] of the maps before the resize (see depth_frame); returns the number of
// polygon pixels outside the image
long long orc_popup_depth_codes(int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                                const float* planes_sensor, const float* Ts, const float* invK, int width, int height,
                                int downsample, float ceiling_threshold, int* codes) {
  const size_t wh = (size_t)width * height;
  std::vector<float> map(wh);
  long long off = 0;
  for (int f = 0; f < n_frames; f++) {
    std::fill(codes + wh * f, codes + wh * (f + 1), 0);
    off += depth_frame(plane_ptr + f, poly_ptr, polys, planes_sensor, Ts + 16 * (size_t)f, invK, width, height,
                       downsample != 0, ceiling_threshold, map.data(), codes + wh * f);
  }
  return off;
}

// the resize chain alone, in place on an even-sized map [height][width]
void orc_popup_depth_resize(float* map, int width, int height) { resize_chain(map, width, height); }

}  // extern "C"
