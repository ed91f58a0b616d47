// pus_popup.cu -- per-frame ground-polyline -> wall-plane "pop-up" fit on the GPU (float32), batched
// over frames: one thread per (frame, plane) output row.  Reproduces
//   popup_plane::get_plane_equation              pop_up_wall/libs/popup_plane.cpp:551-652   (mode 0)
//   popup_plane::update_plane_equation_from_seg  pop_up_wall/libs/popup_plane.cpp:654-705   (mode 0)
//   popup_plane::update_plane_equation_from_seg_fast  popup_plane.cpp:708-749               (mode 1)
//   ray_plane_interact / point_dist_lineseg      pop_up_wall/libs/matrix_utils.cpp:189-193, 290-303
// and, for pus_popup_clouds, the dense plane clouds of
//   popup_plane::generate_cloud / closed_polygons_homo_pts / matrixToCloud  popup_plane.cpp:807-863, 81-116, 925-985
// Compiled with --fmad=false so the float32 arithmetic rounds like the reference's scalar code.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"

namespace pus {
extern thread_local std::string g_err;

__device__ __forceinline__ float seg_dist(const float* b, const float* e, const float* q) {
  float dx = e[0] - b[0], dy = e[1] - b[1];
  float length = sqrtf(dx * dx + dy * dy);
  float qx = q[0] - b[0], qy = q[1] - b[1];
  if (length < 0.001f) return sqrtf(qx * qx + qy * qy);
  float t = (qx * dx + qy * dy) / length / length;
  if (t < 0.0f) return sqrtf(qx * qx + qy * qy);
  else if (t > 1.0f) { float ex = q[0] - e[0], ey = q[1] - e[1]; return sqrtf(ex * ex + ey * ey); }
  float px = b[0] + t * dx, py = b[1] + t * dy;
  float rx = q[0] - px, ry = q[1] - py;
  return sqrtf(rx * rx + ry * ry);
}

__global__ void popup_kernel(int n_frames, const int* __restrict__ seg_ptr, const int* __restrict__ row_frame,
                             int n_rows, const float* __restrict__ segs, const float* __restrict__ invK,
                             const float* __restrict__ Ts, float dist_thre, int mode, float* planes_world,
                             float* planes_sensor, float* dist, int* good) {
  int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n_rows) return;
  const int f = row_frame[row];
  const int s0 = seg_ptr[f];
  const int n = seg_ptr[f + 1] - s0;
  const int j = row - (s0 + f);  // 0 = ground, 1.. = segments
  if (n <= 0) return;
  float T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Ts[(size_t)f * 16 + i];
  const float gw[4] = {0.f, 0.f, -1.f, 0.f};
  float gs[4];
#pragma unroll
  for (int i = 0; i < 4; i++) gs[i] = T[0 * 4 + i] * gw[0] + T[1 * 4 + i] * gw[1] + T[2 * 4 + i] * gw[2] + T[3 * 4 + i] * gw[3];
  if (j == 0) {
    if (planes_sensor) for (int i = 0; i < 4; i++) planes_sensor[(size_t)row * 4 + i] = gs[i];
    if (mode == 0) {
      if (planes_world) for (int i = 0; i < 4; i++) planes_world[(size_t)row * 4 + i] = gw[i];
      if (dist) dist[row] = T[2 * 4 + 3];
      if (good) good[row] = 1;
    }
    return;
  }
  const int s = s0 + j - 1;
  float K[9];
#pragma unroll
  for (int i = 0; i < 9; i++) K[i] = invK[i];
  float Ps[2][3], Pw[2][3];
#pragma unroll
  for (int k = 0; k < 2; k++) {
    float x = segs[(size_t)s * 4 + 2 * k], y = segs[(size_t)s * 4 + 2 * k + 1];
    float ray[3];
    for (int i = 0; i < 3; i++) ray[i] = K[i * 3 + 0] * x + K[i * 3 + 1] * y + K[i * 3 + 2] * 1.0f;
    float den = gs[0] * ray[0] + gs[1] * ray[1] + gs[2] * ray[2];
    float frac = -gs[3] / den;
    for (int i = 0; i < 3; i++) Ps[k][i] = frac * ray[i];
    if (mode == 0) {
      float h[4];
      for (int i = 0; i < 4; i++) h[i] = T[i * 4 + 0] * Ps[k][0] + T[i * 4 + 1] * Ps[k][1] + T[i * 4 + 2] * Ps[k][2] + T[i * 4 + 3] * 1.0f;
      for (int i = 0; i < 3; i++) Pw[k][i] = h[i] / h[3];
    }
  }
  if (mode == 0) {
    Pw[0][2] = 0.f; Pw[1][2] = 0.f;
    float t1[3] = {Pw[1][0] - Pw[0][0], Pw[1][1] - Pw[0][1], Pw[1][2] - Pw[0][2]};
    float t2[3] = {gw[0], gw[1], gw[2]};
    float nrm[3] = {t1[1] * t2[2] - t1[2] * t2[1], t1[2] * t2[0] - t1[0] * t2[2], t1[0] * t2[1] - t1[1] * t2[0]};
    float d = -(nrm[0] * Pw[0][0] + nrm[1] * Pw[0][1] + nrm[2] * Pw[0][2]);
    float pw[4] = {nrm[0], nrm[1], nrm[2], d};
    if (planes_world) for (int i = 0; i < 4; i++) planes_world[(size_t)row * 4 + i] = pw[i];
    if (planes_sensor)
      for (int i = 0; i < 4; i++)
        planes_sensor[(size_t)row * 4 + i] = T[0 * 4 + i] * pw[0] + T[1 * 4 + i] * pw[1] + T[2 * 4 + i] * pw[2] + T[3 * 4 + i] * pw[3];
    float cam[2] = {T[0 * 4 + 3], T[1 * 4 + 3]};
    float dd = seg_dist(Pw[0], Pw[1], cam);
    if (dist) dist[row] = dd;
    if (good) good[row] = ((Ps[0][2] > 0) && (Ps[1][2] > 0) && (dd < dist_thre)) ? 1 : 0;
  } else {
    float t1[3] = {Ps[1][0] - Ps[0][0], Ps[1][1] - Ps[0][1], Ps[1][2] - Ps[0][2]};
    float t2[3] = {gs[0], gs[1], gs[2]};
    float nrm[3] = {t1[1] * t2[2] - t1[2] * t2[1], t1[2] * t2[0] - t1[0] * t2[2], t1[0] * t2[1] - t1[1] * t2[0]};
    float d = -(nrm[0] * Ps[0][0] + nrm[1] * Ps[0][1] + nrm[2] * Ps[0][2]);
    if (planes_sensor) {
      planes_sensor[(size_t)row * 4 + 0] = nrm[0]; planes_sensor[(size_t)row * 4 + 1] = nrm[1];
      planes_sensor[(size_t)row * 4 + 2] = nrm[2]; planes_sensor[(size_t)row * 4 + 3] = d;
    }
  }
}
// ---- device-resident refresh (pus_refresh_plane_measurements) -------------------------------------------
// Pose3d::wTo (Pose3d.h:188-194) of the frame's pose estimate, cast to float as Mapping.cpp:598-599 does
__global__ void frame_pose_kernel(int n_frames, const int* __restrict__ frame_pose, const double* pose7, float* Ts) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const double* p = pose7 + (size_t)frame_pose[f] * 7;
  const double qw = p[3], qx = p[4], qy = p[5], qz = p[6];
  // Eigen toRotationMatrix, no normalisation (Rot3d.h:96-98)
  const double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  float* T = Ts + (size_t)f * 16;
  T[0] = (float)(1 - (tyy + tzz)); T[1] = (float)(txy - twz);       T[2] = (float)(txz + twy);        T[3] = (float)p[0];
  T[4] = (float)(txy + twz);       T[5] = (float)(1 - (txx + tzz)); T[6] = (float)(tyz - twx);        T[7] = (float)p[1];
  T[8] = (float)(txz - twy);       T[9] = (float)(tyz + twx);       T[10] = (float)(1 - (txx + tyy)); T[11] = (float)p[2];
  T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
}

// Plane3d(row.cast<double>()) (normalised 4-vector) -> the factor's measurement slot and the host copy
__global__ void store_meas_kernel(int n_map, const int* __restrict__ map_row, const int* __restrict__ map_slot,
                                  const float* __restrict__ planes_sensor, double* pp_meas, double* out) {
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_map) return;
  const float* r = planes_sensor + (size_t)map_row[m] * 4;
  double v[4] = {(double)r[0], (double)r[1], (double)r[2], (double)r[3]};
  const double z = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
  if (z > 0) {
    const double n = sqrt(z);
    v[0] /= n; v[1] /= n; v[2] /= n; v[3] /= n;
  }
  double* dst = pp_meas + (size_t)map_slot[m] * 4;
  for (int i = 0; i < 4; i++) { dst[i] = v[i]; out[(size_t)m * 4 + i] = v[i]; }
}

// Plane3d::project_to_plane (isam_plane3d.h:172-177): normal() = abc/|abc|, d() = -d/|abc|
__global__ void project_kernel(int n, const int* __restrict__ plane_idx, const double* plane4, const float* __restrict__ in, float* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* pl = plane4 + (size_t)plane_idx[i] * 4;
  const double nn = sqrt(pl[0] * pl[0] + pl[1] * pl[1] + pl[2] * pl[2]);
  const double nx = pl[0] / nn, ny = pl[1] / nn, nz = pl[2] / nn;
  const double dd = -pl[3] / nn;
  const double px = in[(size_t)i * 3], py = in[(size_t)i * 3 + 1], pz = in[(size_t)i * 3 + 2];
  const double t = (nx * px + ny * py + nz * pz) - dd;
  out[(size_t)i * 3] = (float)(px - nx * t);
  out[(size_t)i * 3 + 1] = (float)(py - ny * t);
  out[(size_t)i * 3 + 2] = (float)(pz - nz * t);
}

// launchers used by pus_engine.cu (all pointers are device pointers)
cudaError_t launch_refresh(cudaStream_t st, int n_frames, const int* d_frame_pose, const double* d_pose7, const int* d_seg_ptr,
                           const int* d_row_frame, int n_rows, const float* d_segs, const float* d_invK, float* d_Ts,
                           float* d_planes_sensor, int n_map, const int* d_map_row, const int* d_map_slot, double* d_pp_meas,
                           double* d_out) {
  frame_pose_kernel<<<(n_frames + 127) / 128, 128, 0, st>>>(n_frames, d_frame_pose, d_pose7, d_Ts);
  popup_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(n_frames, d_seg_ptr, d_row_frame, n_rows, d_segs, d_invK, d_Ts, 0.f, 0, nullptr,
                                                      d_planes_sensor, nullptr, nullptr);
  if (n_map > 0) store_meas_kernel<<<(n_map + 255) / 256, 256, 0, st>>>(n_map, d_map_row, d_map_slot, d_planes_sensor, d_pp_meas, d_out);
  return cudaGetLastError();
}
cudaError_t launch_project(cudaStream_t st, int n, const int* d_plane_idx, const double* d_plane4, const float* d_in, float* d_out) {
  project_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, d_plane_idx, d_plane4, d_in, d_out);
  return cudaGetLastError();
}
}  // namespace pus

using namespace pus;

#define PCHK(call)                                                                  \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) { g_err = std::string(#call) + ": " + cudaGetErrorString(e__); rc = -1; goto done; } \
  } while (0)

extern "C" int pus_popup_fit_frames(int device, int n_frames, const int* seg_ptr, const float* segs, const float* invK,
                                    const float* Ts, float dist_thre, int mode, float* planes_world, float* planes_sensor,
                                    float* dist, int* good) {
  int rc = 0;
  if (n_frames <= 0) return 0;
  const int n_seg = seg_ptr[n_frames];
  const int n_rows = n_seg + n_frames;
  int *d_ptr = nullptr, *d_rf = nullptr, *d_good = nullptr;
  float *d_segs = nullptr, *d_K = nullptr, *d_T = nullptr, *d_pw = nullptr, *d_ps = nullptr, *d_dist = nullptr;
  int* rf = new int[n_rows];
  for (int f = 0; f < n_frames; f++)
    for (int r = seg_ptr[f] + f; r < seg_ptr[f + 1] + f + 1; r++) rf[r] = f;
  {
    int ndev = 0;
    cudaError_t de = cudaGetDeviceCount(&ndev);
    if (de != cudaSuccess || ndev <= 0 || device >= ndev) {
      g_err = "pus_popup_fit_frames: no usable CUDA device; libpopup_gpu has no CPU fallback";
      delete[] rf;
      return -1;
    }
  }
  PCHK(cudaSetDevice(device));
  PCHK(cudaMalloc(&d_ptr, (n_frames + 1) * sizeof(int)));
  PCHK(cudaMalloc(&d_rf, n_rows * sizeof(int)));
  PCHK(cudaMalloc(&d_segs, (size_t)(n_seg > 0 ? n_seg : 1) * 4 * sizeof(float)));
  PCHK(cudaMalloc(&d_K, 9 * sizeof(float)));
  PCHK(cudaMalloc(&d_T, (size_t)n_frames * 16 * sizeof(float)));
  PCHK(cudaMalloc(&d_pw, (size_t)n_rows * 4 * sizeof(float)));
  PCHK(cudaMalloc(&d_ps, (size_t)n_rows * 4 * sizeof(float)));
  PCHK(cudaMalloc(&d_dist, (size_t)n_rows * sizeof(float)));
  PCHK(cudaMalloc(&d_good, (size_t)n_rows * sizeof(int)));
  PCHK(cudaMemcpy(d_ptr, seg_ptr, (n_frames + 1) * sizeof(int), cudaMemcpyHostToDevice));
  PCHK(cudaMemcpy(d_rf, rf, n_rows * sizeof(int), cudaMemcpyHostToDevice));
  if (n_seg > 0) PCHK(cudaMemcpy(d_segs, segs, (size_t)n_seg * 4 * sizeof(float), cudaMemcpyHostToDevice));
  PCHK(cudaMemcpy(d_K, invK, 9 * sizeof(float), cudaMemcpyHostToDevice));
  PCHK(cudaMemcpy(d_T, Ts, (size_t)n_frames * 16 * sizeof(float), cudaMemcpyHostToDevice));
  PCHK(cudaMemset(d_pw, 0, (size_t)n_rows * 4 * sizeof(float)));
  PCHK(cudaMemset(d_ps, 0, (size_t)n_rows * 4 * sizeof(float)));
  PCHK(cudaMemset(d_dist, 0, (size_t)n_rows * sizeof(float)));
  PCHK(cudaMemset(d_good, 0, (size_t)n_rows * sizeof(int)));
  popup_kernel<<<(n_rows + 255) / 256, 256>>>(n_frames, d_ptr, d_rf, n_rows, d_segs, d_K, d_T, dist_thre, mode, d_pw, d_ps, d_dist, d_good);
  PCHK(cudaGetLastError());
  PCHK(cudaDeviceSynchronize());
  if (planes_world) PCHK(cudaMemcpy(planes_world, d_pw, (size_t)n_rows * 4 * sizeof(float), cudaMemcpyDeviceToHost));
  if (planes_sensor) PCHK(cudaMemcpy(planes_sensor, d_ps, (size_t)n_rows * 4 * sizeof(float), cudaMemcpyDeviceToHost));
  if (dist) PCHK(cudaMemcpy(dist, d_dist, (size_t)n_rows * sizeof(float), cudaMemcpyDeviceToHost));
  if (good) PCHK(cudaMemcpy(good, d_good, (size_t)n_rows * sizeof(int), cudaMemcpyDeviceToHost));
done:
  delete[] rf;
  cudaFree(d_ptr); cudaFree(d_rf); cudaFree(d_segs); cudaFree(d_K); cudaFree(d_T); cudaFree(d_pw); cudaFree(d_ps); cudaFree(d_dist); cudaFree(d_good);
  return rc;
}

// ---- dense plane clouds (pus_popup_clouds) ------------------------------------------------------------------------------
// The pixel set of a polygon is cv::fillConvexPoly (OpenCV 4.13, LINE_8, shift 0) on its bounding box: the outline drawn edge
// by edge with the 8-connected line iterator, plus the two-edge scanline fill.  Here both are per-row closed forms, so the
// pixels of a row are the union of one scanline span and one run per edge, and every row can be enumerated on its own in
// findNonZero order (row-major).  The scanline walk is sequential in OpenCV (it tracks two edge chains and a budget of edges,
// which decides its result on non-convex polygons), so one thread per plane replays it into a span table first.
namespace pus {
namespace cloud {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct Job { int frame, v0, n, bx, by, bw, bh, row0; };   // per plane: polygon in vtx[v0 .. v0+n), box, first span row
struct Edge { int x1, y1, major, minor, sy, vert, valid; };

// cv::LineIterator's clip against [0, w) x [0, h): Cohen-Sutherland with truncating divisions in double
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)(__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1)));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)(__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1)));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)(__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1)));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)(__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1)));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// edge i of the outline runs from vertex i-1 (cyclically) to vertex i, drawn left to right
__device__ Edge make_edge(const int2* v, int n, int i, int w, int h) {
  const int2 a = v[(i + n - 1) % n], b = v[i];
  long long x1 = a.x, y1 = a.y, x2 = b.x, y2 = b.y;
  Edge e{};
  e.valid = 1;
  if (x1 < 0 || x1 >= w || x2 < 0 || x2 >= w || y1 < 0 || y1 >= h || y2 < 0 || y2 >= h) e.valid = clip_line(w, h, x1, y1, x2, y2);
  if (x2 < x1) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
  const int dx = (int)(x2 - x1);
  int dy = (int)(y2 - y1);
  e.sy = dy < 0 ? -1 : 1;
  dy = dy < 0 ? -dy : dy;
  e.vert = dy > dx;
  e.major = e.vert ? dy : dx;
  e.minor = e.vert ? dx : dy;
  e.x1 = (int)x1;
  e.y1 = (int)y1;
  return e;
}

__device__ __forceinline__ long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// the run of edge e's pixels on box row y (lo > hi: none).  Pixel i of the iterator sits at major offset i and minor offset
// ceil((2*minor*i - major) / (2*major)), the closed form of its error recurrence.
__device__ int2 edge_run(const Edge& e, int y) {
  if (!e.valid) return make_int2(1, 0);
  const long long t = (long long)(y - e.y1) * e.sy;
  if (e.vert) {
    if (t < 0 || t > e.major) return make_int2(1, 0);
    const int x = e.x1 + (int)(-floor_div(-(2LL * e.minor * t - e.major), 2LL * e.major));
    return make_int2(x, x);
  }
  if (t < 0 || t > e.minor) return make_int2(1, 0);
  long long lo = 0, hi = e.major;
  if (e.minor > 0) {
    lo = max(0LL, floor_div(2LL * e.major * t - e.major, 2LL * e.minor) + 1);
    hi = min((long long)e.major, floor_div(2LL * e.major * t + e.major, 2LL * e.minor));
  }
  return make_int2(e.x1 + (int)lo, e.x1 + (int)hi);
}

// cv::fillConvexPoly's scanline walk (the filled span of every box row; rows it never reaches stay empty)
__device__ void scan_spans(const int2* v, int n, int w, int h, int2* span) {
  int xmin = v[0].x, xmax = v[0].x, ymin = v[0].y, ymax = v[0].y, imin = 0;
  for (int i = 0; i < n; i++) {
    if (v[i].y < ymin) { ymin = v[i].y; imin = i; }
    ymax = max(ymax, v[i].y); xmax = max(xmax, v[i].x); xmin = min(xmin, v[i].x);
  }
  if (n < 3 || xmax < 0 || ymax < 0 || xmin >= w || ymin >= h) return;
  ymax = min(ymax, h - 1);
  int idx_[2] = {imin, imin}, ye[2] = {ymin, ymin};
  const int di[2] = {1, n - 1};
  long long ex[2] = {-(1LL << 16), -(1LL << 16)}, edx[2] = {0, 0};
  int edges = n, y = ymin;
  do {
#pragma unroll
    for (int i = 0; i < 2; i++) {
      if (y < ye[i]) continue;
      int idx0 = idx_[i], idx = idx0 + di[i];
      if (idx >= n) idx -= n;
      for (; edges-- > 0;) {
        const int ty = v[idx].y;
        if (ty > y) {
          const long long xs = (long long)v[idx0].x << 16, xe = (long long)v[idx].x << 16;
          ye[i] = ty;
          edx[i] = ((xe - xs) * 2 + ((long long)ty - y)) / (2 * ((long long)ty - y));
          ex[i] = xs;
          idx_[i] = idx;
          break;
        }
        idx0 = idx;
        idx += di[i];
        if (idx >= n) idx -= n;
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int l = ex[0] > ex[1] ? 1 : 0;
      int x1 = (int)((ex[l] + (1 << 15)) >> 16), x2 = (int)((ex[1 - l] + (1 << 15)) >> 16);
      if (x2 >= 0 && x1 < w) span[y] = make_int2(max(x1, 0), min(x2, w - 1));
    }
    ex[0] += edx[0];
    ex[1] += edx[1];
  } while (++y <= ymax);
}

struct Params {
  const Job* jobs;
  const int2* vtx;
  const float* planes;   // [n_planes][4] sensor frame
  const float* Ts;       // [n_frames][16]
  const float* invK;
  const unsigned char* images;   // uploaded only when colours are written
  int width, height, scale, border;   // border: images were given and are 960 wide (matrixToCloud's x < 4 || y < 4 rule)
  float depth_thre, ceiling;
  int2* span;            // [rows]
  int* row_count;        // [rows]
  const long long* row_off;
  float* xyz;
  unsigned char* rgb;
};

// the warp's pixel range of box row y, and its edge runs in runs[] (lanes over edges)
__device__ __forceinline__ int2 row_setup(const Edge* E, int n, int2 sp, int y, int2* runs, int lane) {
  int lo = sp.x <= sp.y ? sp.x : INT_MAX, hi = sp.x <= sp.y ? sp.y : INT_MIN;
  for (int e = lane; e < n; e += 32) {
    const int2 r = edge_run(E[e], y);
    runs[e] = r;
    if (r.x <= r.y) { lo = min(lo, r.x); hi = max(hi, r.y); }
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __syncwarp();
  return make_int2(lo, hi);
}

__device__ __forceinline__ bool member(int x, int2 sp, const int2* runs, int n) {
  if (x >= sp.x && x <= sp.y) return true;
  for (int e = 0; e < n; e++)
    if (x >= runs[e].x && x <= runs[e].y) return true;
  return false;
}

// COUNT: replay the scanline walk into span[], then count the kept points of every box row.
// WRITE: write the kept points of every row at row_off[row] in pixel order.
template <bool WRITE>
__global__ void __launch_bounds__(kThreads) cloud_kernel(Params P) {
  __shared__ Edge E[PUS_POPUP_MAX_VERTICES];
  __shared__ int2 runs[kWarps][PUS_POPUP_MAX_VERTICES];
  const Job J = P.jobs[blockIdx.x];
  if (J.n <= 0) return;
  const int2* v = P.vtx + J.v0;
  for (int i = threadIdx.x; i < J.n; i += kThreads) E[i] = make_edge(v, J.n, i, J.bw, J.bh);
  if (!WRITE) {
    for (int y = threadIdx.x; y < J.bh; y += kThreads) P.span[J.row0 + y] = make_int2(1, 0);
    __syncthreads();
    if (threadIdx.x == 0) scan_spans(v, J.n, J.bw, J.bh, P.span + J.row0);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float T[12], K[9], pl[4];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = P.Ts[(size_t)J.frame * 16 + i];
#pragma unroll
  for (int i = 0; i < 9; i++) K[i] = P.invK[i];
#pragma unroll
  for (int i = 0; i < 4; i++) pl[i] = P.planes[(size_t)blockIdx.x * 4 + i];
  const unsigned char* img = P.images ? P.images + (size_t)J.frame * P.width * P.height * 3 : nullptr;
  int2* wr = runs[warp];
  for (int y = warp; y < J.bh; y += kWarps) {
    const int2 sp = P.span[J.row0 + y];
    const int2 range = row_setup(E, J.n, sp, y, wr, lane);
    long long base = WRITE ? P.row_off[J.row0 + y] : 0;
    int kept = 0;
    for (int x0 = range.x; x0 <= range.y; x0 += 32) {
      const int x = x0 + lane;
      bool keep = x <= range.y && member(x, sp, wr, J.n);
      float pw[3] = {0.f, 0.f, 0.f};
      const int X = (J.bx + x) * P.scale, Y = (J.by + y) * P.scale;
      if (keep) {
        const float fx = (float)X, fy = (float)Y;
        float ray[3];
#pragma unroll
        for (int i = 0; i < 3; i++) ray[i] = K[i * 3 + 0] * fx + K[i * 3 + 1] * fy + K[i * 3 + 2] * 1.0f;
        const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
        float ps[3];
#pragma unroll
        for (int i = 0; i < 3; i++) ps[i] = frac * ray[i];
#pragma unroll
        for (int i = 0; i < 3; i++) pw[i] = T[i * 4 + 0] * ps[0] + T[i * 4 + 1] * ps[1] + T[i * 4 + 2] * ps[2] + T[i * 4 + 3];
        // matrixToCloud's filters, popup_plane.cpp:951-977 (-0.2 is a double literal there)
        keep = !(ps[2] < 0.f || ps[2] > P.depth_thre || (double)pw[2] < -0.2) && !(P.border && (X < 4 || Y < 4));
      }
      const unsigned mask = __ballot_sync(0xffffffffu, keep);
      if (WRITE && keep) {
        const long long o = base + __popc(mask & ((1u << lane) - 1u));
        if (P.xyz) {
          P.xyz[o * 3 + 0] = pw[0];
          P.xyz[o * 3 + 1] = pw[1];
          P.xyz[o * 3 + 2] = pw[2] < P.ceiling ? pw[2] : P.ceiling;
        }
        if (P.rgb) {
          const bool inside = X >= 0 && X < P.width && Y >= 0 && Y < P.height;
          const unsigned char* c = inside && img ? img + ((size_t)Y * P.width + X) * 3 : nullptr;
          P.rgb[o * 3 + 0] = c ? c[2] : 0;
          P.rgb[o * 3 + 1] = c ? c[1] : 0;
          P.rgb[o * 3 + 2] = c ? c[0] : 0;
        }
      }
      base += __popc(mask);
      kept += __popc(mask);
    }
    if (!WRITE && lane == 0) P.row_count[J.row0 + y] = kept;
    __syncwarp();
  }
}

// exclusive prefix sum of the row counts in one CTA (row_off[rows] = total), then every plane's count and offset
__global__ void __launch_bounds__(1024) cloud_scan_kernel(int rows, const int* row_count, long long* row_off, int n_planes,
                                                          const Job* jobs, int* counts, long long* offsets) {
  __shared__ long long s[1024];
  const int t = threadIdx.x;
  const int chunk = (rows + 1023) / 1024;
  const int r0 = min(rows, t * chunk), r1 = min(rows, r0 + chunk);
  long long sum = 0;
  for (int r = r0; r < r1; r++) sum += row_count[r];
  s[t] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const long long add = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += add;
    __syncthreads();
  }
  long long run = s[t] - sum;
  for (int r = r0; r < r1; r++) { row_off[r] = run; run += row_count[r]; }
  if (t == 1023) row_off[rows] = s[1023];
  __syncthreads();
  for (int p = t; p < n_planes; p += 1024) {
    const long long a = row_off[jobs[p].row0], b = row_off[jobs[p].row0 + jobs[p].bh];
    counts[p] = (int)(b - a);
    offsets[p] = a;
  }
}

// popup_plane.cpp:815-847 label image, one CTA per frame, its planes in order (a later plane overwrites an earlier one).
// Downsampled pixels sit on even coordinates, so the nearest-neighbour 0.5x / 2x resize (:852-855) is the 2x2 block of each.
__global__ void __launch_bounds__(kThreads) cloud_label_kernel(const int* plane_ptr, const Job* jobs, const int2* vtx,
                                                               const int2* spans, int width, int height, int scale,
                                                               unsigned char* labels) {
  __shared__ Edge E[PUS_POPUP_MAX_VERTICES];
  __shared__ int2 runs[kWarps][PUS_POPUP_MAX_VERTICES];
  const int f = blockIdx.x;
  unsigned char* L = labels + (size_t)f * width * height;   // already 127 (void) everywhere
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = plane_ptr[f]; p < plane_ptr[f + 1]; p++) {
    const Job J = jobs[p];
    const unsigned char value = p == plane_ptr[f] ? 255 : 0;
    __syncthreads();
    for (int i = threadIdx.x; i < J.n; i += kThreads) E[i] = make_edge(vtx + J.v0, J.n, i, J.bw, J.bh);
    __syncthreads();
    for (int y = warp; y < J.bh; y += kWarps) {
      const int2 sp = spans[J.row0 + y];
      const int2 range = row_setup(E, J.n, sp, y, runs[warp], lane);
      const int Y = (J.by + y) * scale;
      for (int x0 = range.x; x0 <= range.y; x0 += 32) {
        const int x = x0 + lane;
        const int X = (J.bx + x) * scale;
        if (x <= range.y && X >= 0 && X < width && Y >= 0 && Y < height && member(x, sp, runs[warp], J.n))
          for (int dy = 0; dy < scale; dy++)
            for (int dx = 0; dx < scale; dx++) L[(size_t)(Y + dy) * width + X + dx] = value;
      }
      __syncwarp();
    }
  }
}
}  // namespace cloud
}  // namespace pus

namespace {
template <class T>
struct DevBuf {   // a device allocation freed on every return path
  T* p = nullptr;
  ~DevBuf() { cudaFree(p); }
  cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n > 0 ? n : 1) * sizeof(T)); }
};
}  // namespace

#define CCHK(call)                                                                                        \
  do {                                                                                                    \
    cudaError_t e__ = (call);                                                                             \
    if (e__ != cudaSuccess) { g_err = std::string("pus_popup_clouds: ") + #call + ": " + cudaGetErrorString(e__); return -1; } \
  } while (0)

extern "C" long long pus_popup_clouds(int device, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                                      const float* planes_sensor, const float* Ts, const float* invK,
                                      const unsigned char* images, int width, int height, int downsample, float depth_thre,
                                      float ceiling_threshold, int* counts, long long* offsets, float* xyz, unsigned char* rgb,
                                      long long capacity, unsigned char* labels) {
  using namespace pus::cloud;
  auto refuse = [](const char* why) { g_err = std::string("pus_popup_clouds: ") + why; return -1LL; };
  if (n_frames < 0) return refuse("n_frames < 0");
  if (!plane_ptr || plane_ptr[0] != 0) return refuse("plane_ptr must be given and start at 0");
  if (width <= 0 || height <= 0) return refuse("width and height must be positive");
  if (labels && downsample && ((width | height) & 1)) return refuse("label images in downsample mode need an even width and height");
  for (int f = 0; f < n_frames; f++)
    if (plane_ptr[f + 1] < plane_ptr[f]) return refuse("plane_ptr is not ascending");
  const int n_planes = plane_ptr[n_frames];
  if (n_planes > 0 && (!poly_ptr || poly_ptr[0] != 0)) return refuse("poly_ptr must be given and start at 0");
  if (n_frames > 0 && (!Ts || !invK)) return refuse("Ts and invK must be given");
  if (n_planes > 0 && !planes_sensor) return refuse("planes_sensor must be given");
  for (int p = 0; p < n_planes; p++) {
    const int n = poly_ptr[p + 1] - poly_ptr[p];
    if (n < 0) return refuse("poly_ptr is not ascending");
    if (n > PUS_POPUP_MAX_VERTICES) return refuse("a polygon has more than PUS_POPUP_MAX_VERTICES vertices");
  }
  const int n_vtx = n_planes > 0 ? poly_ptr[n_planes] : 0;
  if (n_vtx > 0 && !polys) return refuse("polys must be given");
  for (int i = 0; i < 2 * n_vtx; i++)
    if (!(std::fabs(polys[i]) <= PUS_POPUP_MAX_COORD)) return refuse("a polygon coordinate is not finite or exceeds PUS_POPUP_MAX_COORD");

  // per polygon: matrix_to_points' truncation, boundingRect, and the box-shifted vertices (popup_plane.cpp:85-96)
  std::vector<Job> jobs(n_planes);
  std::vector<int2> vtx(n_vtx);
  long long rows = 0;
  for (int f = 0; f < n_frames; f++)
    for (int p = plane_ptr[f]; p < plane_ptr[f + 1]; p++) {
      Job& J = jobs[p];
      J = Job{f, poly_ptr[p], poly_ptr[p + 1] - poly_ptr[p], 0, 0, 0, 0, (int)rows};
      if (J.n == 0) continue;
      const float* q = polys + 2 * (size_t)J.v0;
      auto at = [&](int i) { return downsample ? q[i] / 2.f : q[i]; };
      int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
      for (int i = 0; i < J.n; i++) {
        const int x = (int)at(2 * i), y = (int)at(2 * i + 1);
        xmin = std::min(xmin, x); xmax = std::max(xmax, x); ymin = std::min(ymin, y); ymax = std::max(ymax, y);
      }
      J.bx = xmin; J.by = ymin; J.bw = xmax - xmin + 1; J.bh = ymax - ymin + 1;
      for (int i = 0; i < J.n; i++)
        vtx[J.v0 + i] = make_int2((int)(at(2 * i) - (float)J.bx), (int)(at(2 * i + 1) - (float)J.by));
      rows += J.bh;
      if (rows > INT_MAX / 2) return refuse("the polygons' bounding boxes have too many rows in all");
    }
  {
    int ndev = 0;
    cudaError_t de = cudaGetDeviceCount(&ndev);
    if (de != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev)
      return refuse("no CUDA device usable; libpopup_gpu has no CPU fallback");
  }
  CCHK(cudaSetDevice(device));
  DevBuf<Job> d_jobs;
  DevBuf<int2> d_vtx, d_span;
  DevBuf<float> d_planes, d_T, d_K, d_xyz;
  DevBuf<unsigned char> d_img, d_rgb, d_lab;
  DevBuf<int> d_rowcnt, d_cnt, d_ptr;
  DevBuf<long long> d_rowoff, d_off;
  const size_t img_bytes = (size_t)n_frames * width * height * 3;
  CCHK(d_jobs.alloc(n_planes));
  CCHK(d_vtx.alloc(n_vtx));
  CCHK(d_span.alloc(rows));
  CCHK(d_planes.alloc((size_t)n_planes * 4));
  CCHK(d_T.alloc((size_t)n_frames * 16));
  CCHK(d_K.alloc(9));
  CCHK(d_rowcnt.alloc(rows));
  CCHK(d_rowoff.alloc(rows + 1));
  CCHK(d_cnt.alloc(n_planes));
  CCHK(d_off.alloc(n_planes));
  if (n_planes > 0) {
    CCHK(cudaMemcpy(d_jobs.p, jobs.data(), n_planes * sizeof(Job), cudaMemcpyHostToDevice));
    CCHK(cudaMemcpy(d_planes.p, planes_sensor, (size_t)n_planes * 4 * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (n_vtx > 0) CCHK(cudaMemcpy(d_vtx.p, vtx.data(), n_vtx * sizeof(int2), cudaMemcpyHostToDevice));
  if (n_frames > 0) {
    CCHK(cudaMemcpy(d_T.p, Ts, (size_t)n_frames * 16 * sizeof(float), cudaMemcpyHostToDevice));
    CCHK(cudaMemcpy(d_K.p, invK, 9 * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (images && rgb) {
    CCHK(d_img.alloc(img_bytes));
    CCHK(cudaMemcpy(d_img.p, images, img_bytes, cudaMemcpyHostToDevice));
  }
  Params P{d_jobs.p, d_vtx.p, d_planes.p, d_T.p, d_K.p, d_img.p, width, height, downsample ? 2 : 1, images && width == 960, depth_thre,
           ceiling_threshold, d_span.p, d_rowcnt.p, d_rowoff.p, nullptr, nullptr};
  if (n_planes > 0) cloud_kernel<false><<<n_planes, kThreads>>>(P);
  CCHK(cudaGetLastError());
  cloud_scan_kernel<<<1, 1024>>>((int)rows, d_rowcnt.p, d_rowoff.p, n_planes, d_jobs.p, d_cnt.p, d_off.p);
  CCHK(cudaGetLastError());
  long long total = 0;
  CCHK(cudaMemcpy(&total, d_rowoff.p + rows, sizeof(long long), cudaMemcpyDeviceToHost));
  if (counts && n_planes > 0) CCHK(cudaMemcpy(counts, d_cnt.p, n_planes * sizeof(int), cudaMemcpyDeviceToHost));
  if (offsets && n_planes > 0) CCHK(cudaMemcpy(offsets, d_off.p, n_planes * sizeof(long long), cudaMemcpyDeviceToHost));
  if ((xyz || rgb) && capacity < total) return refuse("capacity is smaller than the number of points");
  if ((xyz || rgb) && total > 0) {
    if (xyz) CCHK(d_xyz.alloc((size_t)total * 3));
    if (rgb) CCHK(d_rgb.alloc((size_t)total * 3));
    P.xyz = d_xyz.p;
    P.rgb = d_rgb.p;
    cloud_kernel<true><<<n_planes, kThreads>>>(P);
    CCHK(cudaGetLastError());
    if (xyz) CCHK(cudaMemcpy(xyz, d_xyz.p, (size_t)total * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    if (rgb) CCHK(cudaMemcpy(rgb, d_rgb.p, (size_t)total * 3, cudaMemcpyDeviceToHost));
  }
  if (labels && n_frames > 0) {
    CCHK(d_lab.alloc((size_t)n_frames * width * height));
    CCHK(d_ptr.alloc(n_frames + 1));
    CCHK(cudaMemcpy(d_ptr.p, plane_ptr, (n_frames + 1) * sizeof(int), cudaMemcpyHostToDevice));
    CCHK(cudaMemset(d_lab.p, 127, (size_t)n_frames * width * height));
    cloud_label_kernel<<<n_frames, kThreads>>>(d_ptr.p, d_jobs.p, d_vtx.p, d_span.p, width, height, downsample ? 2 : 1, d_lab.p);
    CCHK(cudaGetLastError());
    CCHK(cudaMemcpy(labels, d_lab.p, (size_t)n_frames * width * height, cudaMemcpyDeviceToHost));
  }
  CCHK(cudaDeviceSynchronize());
  return total;
}
