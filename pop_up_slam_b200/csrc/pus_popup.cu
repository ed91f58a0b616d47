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
#include <cstring>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"
#include "pus_edges.cuh"
#include "pus_frames.cuh"
#include "pus_stages.cuh"

namespace pus {
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
                             float* planes_sensor, float* dist, int* good, float* ends_world = nullptr) {
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
    if (ends_world)   // the world ground endpoints (get_plane_equation's ground_seg3d_lines_world row)
      for (int k = 0; k < 2; k++)
        for (int i = 0; i < 3; i++) ends_world[(size_t)row * 6 + 3 * k + i] = Pw[k][i];
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
  for (int i = 0; i < 4; i++) out[(size_t)m * 4 + i] = v[i];
  if (map_slot[m] < 0) return;   // (a plane map's entry whose factor the caller removed)
  double* dst = pp_meas + (size_t)map_slot[m] * 4;
  for (int i = 0; i < 4; i++) dst[i] = v[i];
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
cudaError_t launch_fit(cudaStream_t st, int n_frames, const int* d_seg_ptr, const int* d_row_frame, int n_rows,
                       const float* d_segs, const float* d_invK, const float* d_Ts, float dist_thre, int mode, float* d_pw,
                       float* d_ps, float* d_dist, int* d_good, float* d_ends) {
  if (n_rows > 0)
    popup_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(n_frames, d_seg_ptr, d_row_frame, n_rows, d_segs, d_invK, d_Ts, dist_thre,
                                                        mode, d_pw, d_ps, d_dist, d_good, d_ends);
  return cudaGetLastError();
}
cudaError_t launch_project(cudaStream_t st, int n, const int* d_plane_idx, const double* d_plane4, const float* d_in, float* d_out) {
  project_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, d_plane_idx, d_plane4, d_in, d_out);
  return cudaGetLastError();
}
}  // namespace pus

using namespace pus;

extern "C" int pus_popup_fit_frames(int device, int n_frames, const int* seg_ptr, const float* segs, const float* invK,
                                    const float* Ts, float dist_thre, int mode, float* planes_world, float* planes_sensor,
                                    float* dist, int* good) {
  const Call C{"pus_popup_fit_frames"};
  if (n_frames <= 0) return 0;
  std::vector<int> rf;
  if (const char* why = row_frames(n_frames, seg_ptr, rf)) return C.refuse(why);
  const int n_seg = seg_ptr[n_frames];
  const int n_rows = n_seg + n_frames;
  if (C.check_device(device) < 0) return -1;
  PUS_CALL_OK(C, cudaSetDevice(device));
  TempAlloc A;
  int *d_ptr = nullptr, *d_rf = nullptr, *d_good = nullptr;
  float *d_segs = nullptr, *d_K = nullptr, *d_T = nullptr, *d_pw = nullptr, *d_ps = nullptr, *d_dist = nullptr;
  PUS_CALL_OK(C, A.upload(d_ptr, seg_ptr, n_frames + 1));
  PUS_CALL_OK(C, A.upload(d_rf, rf.data(), n_rows));
  PUS_CALL_OK(C, A.upload(d_segs, segs, (size_t)n_seg * 4));
  PUS_CALL_OK(C, A.upload(d_K, invK, 9));
  PUS_CALL_OK(C, A.upload(d_T, Ts, (size_t)n_frames * 16));
  PUS_CALL_OK(C, A.get(d_pw, (size_t)n_rows * 4));
  PUS_CALL_OK(C, A.get(d_ps, (size_t)n_rows * 4));
  PUS_CALL_OK(C, A.get(d_dist, n_rows));
  PUS_CALL_OK(C, A.get(d_good, n_rows));
  PUS_CALL_OK(C, cudaMemset(d_pw, 0, (size_t)n_rows * 4 * sizeof(float)));
  PUS_CALL_OK(C, cudaMemset(d_ps, 0, (size_t)n_rows * 4 * sizeof(float)));
  PUS_CALL_OK(C, cudaMemset(d_dist, 0, (size_t)n_rows * sizeof(float)));
  PUS_CALL_OK(C, cudaMemset(d_good, 0, (size_t)n_rows * sizeof(int)));
  PUS_CALL_OK(C, launch_fit(0, n_frames, d_ptr, d_rf, n_rows, d_segs, d_K, d_T, dist_thre, mode, d_pw, d_ps, d_dist, d_good,
                            nullptr));
  PUS_CALL_OK(C, cudaDeviceSynchronize());
  if (planes_world) PUS_CALL_OK(C, download(planes_world, d_pw, (size_t)n_rows * 4));
  if (planes_sensor) PUS_CALL_OK(C, download(planes_sensor, d_ps, (size_t)n_rows * 4));
  if (dist) PUS_CALL_OK(C, download(dist, d_dist, n_rows));
  if (good) PUS_CALL_OK(C, download(good, d_good, n_rows));
  return 0;
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

// pixel (fx, fy) on plane pl: ray = invK (x, y, 1), p_s = -d / (n . ray) ray (ray_plane_interact), p_w = R p_s + t
__device__ __forceinline__ void pixel_on_plane(const float* K, const float* T, const float* pl, float fx, float fy, float* ray,
                                               float* ps, float* pw) {
#pragma unroll
  for (int i = 0; i < 3; i++) ray[i] = K[i * 3 + 0] * fx + K[i * 3 + 1] * fy + K[i * 3 + 2] * 1.0f;
  const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
#pragma unroll
  for (int i = 0; i < 3; i++) ps[i] = frac * ray[i];
#pragma unroll
  for (int i = 0; i < 3; i++) pw[i] = T[i * 4 + 0] * ps[0] + T[i * 4 + 1] * ps[1] + T[i * 4 + 2] * ps[2] + T[i * 4 + 3];
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
        float ray[3], ps[3];
        pixel_on_plane(K, T, pl, (float)X, (float)Y, ray, ps, pw);
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

// ---- pop-up depth map (pus_popup_depth) ----
// per plane: its outline edges (into edges[v0 ..]) and the scanline walk into span[]
__global__ void __launch_bounds__(128) depth_span_kernel(const Job* jobs, const int2* vtx, Edge* edges, int2* span) {
  const Job J = jobs[blockIdx.x];
  if (J.n <= 0) return;
  for (int i = threadIdx.x; i < J.n; i += blockDim.x) edges[J.v0 + i] = make_edge(vtx + J.v0, J.n, i, J.bw, J.bh);
  for (int y = threadIdx.x; y < J.bh; y += blockDim.x) span[J.row0 + y] = make_int2(1, 0);
  __syncthreads();
  if (threadIdx.x == 0) scan_spans(vtx + J.v0, J.n, J.bw, J.bh, span + J.row0);
}

constexpr int kChunk = 32 * 32;   // fill-space columns per pass of a warp: one bit per pixel in a lane's 32-bit mask

// popup_plane.cpp:891-910 on the fill grid (the image, or its even pixels in downsample mode: scale 2), one warp per
// (frame, fill row).  Last writer wins, so the warp walks the frame's planes from the last to the first and a pixel takes the
// first value that passes; every pixel of out is written exactly once.
__global__ void __launch_bounds__(kThreads) depth_kernel(int n_frames, const int* plane_ptr, const Job* jobs, const Edge* edges,
                                                         const int2* spans, const float* planes, const float* Ts,
                                                         const float* invK, int fw, int fh, int scale, float ceiling,
                                                         float* out) {
  __shared__ int2 runs[kWarps][PUS_POPUP_MAX_VERTICES];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * kWarps + warp;
  if (row >= (long long)n_frames * fh) return;
  const int f = (int)(row / fh), hy = (int)(row % fh);
  float T[12], K[9], cs[4];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = Ts[(size_t)f * 16 + i];
#pragma unroll
  for (int i = 0; i < 9; i++) K[i] = invK[i];
  // ceiling_plane_sensor = T^T (0, 0, -1, c) (popup_plane.cpp:602-603), the four terms as popup_kernel forms the ground
  const float cw[4] = {0.f, 0.f, -1.f, ceiling};
#pragma unroll
  for (int i = 0; i < 4; i++)
    cs[i] = T[0 * 4 + i] * cw[0] + T[1 * 4 + i] * cw[1] + T[2 * 4 + i] * cw[2] + Ts[(size_t)f * 16 + 12 + i] * cw[3];
  float* o = out + row * fw;
  const int p0 = plane_ptr[f], p1 = plane_ptr[f + 1];
  const float fY = (float)(hy * scale);
  for (int c0 = 0; c0 < fw; c0 += kChunk) {
    const int c1 = min(fw, c0 + kChunk);
    const int nk = c1 - c0 - lane > 0 ? (c1 - c0 - lane + 31) >> 5 : 0;   // this lane's pixels in the chunk
    const unsigned full = nk >= 32 ? 0xffffffffu : (1u << nk) - 1u;
    unsigned taken = 0;
    for (int p = p1 - 1; p >= p0 && !__all_sync(0xffffffffu, taken == full); p--) {
      const Job J = jobs[p];
      const int y = hy - J.by;
      if (J.n <= 0 || y < 0 || y >= J.bh || J.bx >= c1 || J.bx + J.bw <= c0) continue;
      const int2 sp = spans[J.row0 + y];
      const int2 range = row_setup(edges + J.v0, J.n, sp, y, runs[warp], lane);
      if (range.x > range.y) continue;
      const int lo = max(range.x + J.bx, c0), hi = min(range.y + J.bx, c1 - 1);
      float pl[4];
#pragma unroll
      for (int i = 0; i < 4; i++) pl[i] = planes[(size_t)p * 4 + i];
      for (int x0 = c0 + ((lo - c0) & ~31); x0 <= hi; x0 += 32) {
        const int x = x0 + lane;
        const unsigned bit = 1u << ((x0 - c0) >> 5);
        if (x < lo || x > hi || (taken & bit) || !member(x - J.bx, sp, runs[warp], J.n)) continue;
        float ray[3], ps[3], pw[3];
        pixel_on_plane(K, T, pl, (float)(x * scale), fY, ray, ps, pw);
        float v;
        if (pw[2] < ceiling) {
          if (ps[2] < 0) continue;
          v = ps[2];
        } else {   // ray_plane_interact(ray, ceiling_plane_sensor), its z
          v = -cs[3] / (cs[0] * ray[0] + cs[1] * ray[1] + cs[2] * ray[2]) * ray[2];
          if (v < 0) continue;
        }
        o[x] = v;
        taken |= bit;
      }
      __syncwarp();
    }
    for (int k = 0; k < nk; k++)
      if (!(taken & (1u << k))) o[c0 + lane + 32 * k] = 0.f;
  }
}

// downsample mode (popup_plane.cpp:912-916): cv::resize 0.5x (INTER_LINEAR at 0.5 is OpenCV's area fast path), convertTo x4,
// cv::resize 2x INTER_LINEAR, as OpenCV 4.13's own code computes them (not the IPP build).  half holds the full map's even
// pixels; its odd pixels are 0, as no written pixel is odd (so the area path's pairwise SIMD sum and its left-to-right scalar
// tail agree).  One thread per output pixel; each recomputes the horizontal pass of its two source rows, so the result is
// the separable one.
__device__ __forceinline__ float depth_quarter(const float* half, int hw, int r, int c) {
  const float s = ((half[(size_t)r * hw + c] + 0.f) + (0.f + 0.f)) * 0.25f;
  return s * 4.f + 0.f;
}

// the horizontal 2x pass at output column dx of half-size row r: left border (1 - 0) x S[0] + 0 x S[1], right border S[w-1]
// (a one-column source has only the single-term border)
__device__ __forceinline__ float depth_hpass(const float* half, int hw, int r, int dx) {
  const int j = dx >> 1;
  if (dx == 2 * hw - 1 || hw == 1) return depth_quarter(half, hw, r, hw - 1) * 1.f;
  if (dx == 0) return depth_quarter(half, hw, r, 0) * 1.f + depth_quarter(half, hw, r, 1) * 0.f;
  const int sx = (dx & 1) ? j : j - 1;
  const float w0 = (dx & 1) ? 0.75f : 0.25f, w1 = (dx & 1) ? 0.25f : 0.75f;
  return depth_quarter(half, hw, r, sx) * w0 + depth_quarter(half, hw, r, sx + 1) * w1;
}

__global__ void depth_resize_kernel(int n_frames, const float* half, int width, int height, float* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long wh = (long long)width * height;
  if (i >= (long long)n_frames * wh) return;
  const int f = (int)(i / wh), Y = (int)(i % wh / width), X = (int)(i % width);
  const int hw = width / 2, hh = height / 2;
  const float* H = half + (size_t)f * hw * hh;
  float v;
  if (Y == 0 || Y == height - 1) {   // the border rows take one source row
    v = depth_hpass(H, hw, Y == 0 ? 0 : hh - 1, X) * 1.f;
  } else {
    const int sy = (Y & 1) ? Y >> 1 : (Y >> 1) - 1;
    const float w0 = (Y & 1) ? 0.75f : 0.25f, w1 = (Y & 1) ? 0.25f : 0.75f;
    v = depth_hpass(H, hw, sy, X) * w0 + depth_hpass(H, hw, sy + 1, X) * w1;
  }
  out[i] = v;
}

cudaError_t launch_count(cudaStream_t st, int n_planes, long long rows, const Params& P, long long* d_row_off, int* d_counts,
                         long long* d_offsets) {
  if (n_planes > 0) cloud_kernel<false><<<n_planes, kThreads, 0, st>>>(P);
  cloud_scan_kernel<<<1, 1024, 0, st>>>((int)rows, P.row_count, d_row_off, n_planes, P.jobs, d_counts, d_offsets);
  return cudaGetLastError();
}
cudaError_t launch_write(cudaStream_t st, int n_planes, const Params& P) {
  if (n_planes > 0) cloud_kernel<true><<<n_planes, kThreads, 0, st>>>(P);
  return cudaGetLastError();
}
cudaError_t launch_labels(cudaStream_t st, int n_frames, const int* d_plane_ptr, const Params& P, unsigned char* d_labels) {
  if (n_frames > 0)
    cloud_label_kernel<<<n_frames, kThreads, 0, st>>>(d_plane_ptr, P.jobs, P.vtx, P.span, P.width, P.height, P.scale, d_labels);
  return cudaGetLastError();
}
cudaError_t launch_depth(cudaStream_t st, int n_frames, int n_planes, const int* d_plane_ptr, const Job* d_jobs,
                         const int2* d_vtx, Edge* d_edges, int2* d_span, const float* d_planes, const float* d_Ts,
                         const float* d_invK, int width, int height, int downsample, float ceiling, float* d_fill,
                         float* d_out) {
  if (n_frames == 0) return cudaSuccess;
  const int scale = downsample ? 2 : 1, fw = width / scale, fh = height / scale;
  if (n_planes > 0) depth_span_kernel<<<n_planes, 128, 0, st>>>(d_jobs, d_vtx, d_edges, d_span);
  const long long fill_rows = (long long)n_frames * fh;
  depth_kernel<<<(unsigned)((fill_rows + kWarps - 1) / kWarps), kThreads, 0, st>>>(n_frames, d_plane_ptr, d_jobs, d_edges, d_span,
                                                                                   d_planes, d_Ts, d_invK, fw, fh, scale,
                                                                                   ceiling, d_fill);
  if (downsample) {
    const size_t out_n = (size_t)n_frames * width * height;
    depth_resize_kernel<<<(unsigned)((out_n + 255) / 256), 256, 0, st>>>(n_frames, d_fill, width, height, d_out);
  }
  return cudaGetLastError();
}
}  // namespace cloud
}  // namespace pus

namespace {
// The planes' polygon arguments of pus_popup_clouds and pus_popup_depth, checked, and per polygon matrix_to_points'
// truncation, boundingRect and the box-shifted vertices (popup_plane.cpp:85-96).  Returns the number of box rows in all, or
// -1 refused through C.
long long plane_jobs(const Call& C, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                     const float* planes_sensor, const float* Ts, const float* invK, int downsample,
                     std::vector<pus::cloud::Job>& jobs, std::vector<int2>& vtx) {
  using pus::cloud::Job;
  auto refuse = [&](const char* why) { return (long long)C.refuse(why); };
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
  jobs.assign(n_planes, Job{});
  vtx.assign(n_vtx, int2{});
  long long rows = 0;
  for (int f = 0; f < n_frames; f++)
    for (int p = plane_ptr[f]; p < plane_ptr[f + 1]; p++) {
      Job& J = jobs[p];
      J = Job{f, poly_ptr[p], poly_ptr[p + 1] - poly_ptr[p], 0, 0, 0, 0, (int)rows};
      if (J.n == 0) continue;
      pus::glue::polygon_box(polys + 2 * (size_t)J.v0, J.n, downsample, J, vtx.data() + J.v0);
      rows += J.bh;
      if (rows > INT_MAX / 2) return refuse("the polygons' bounding boxes have too many rows in all");
    }
  return rows;
}
}  // namespace

extern "C" long long pus_popup_clouds(int device, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                                      const float* planes_sensor, const float* Ts, const float* invK,
                                      const unsigned char* images, int width, int height, int downsample, float depth_thre,
                                      float ceiling_threshold, int* counts, long long* offsets, float* xyz, unsigned char* rgb,
                                      long long capacity, unsigned char* labels) {
  using namespace pus::cloud;
  const Call C{"pus_popup_clouds"};
  if (n_frames < 0) return C.refuse("n_frames < 0");
  if (!plane_ptr || plane_ptr[0] != 0) return C.refuse("plane_ptr must be given and start at 0");
  if (width <= 0 || height <= 0) return C.refuse("width and height must be positive");
  if (labels && downsample && ((width | height) & 1)) return C.refuse("label images in downsample mode need an even width and height");
  std::vector<Job> jobs;
  std::vector<int2> vtx;
  const long long rows = plane_jobs(C, n_frames, plane_ptr, poly_ptr, polys, planes_sensor, Ts, invK, downsample, jobs, vtx);
  if (rows < 0) return -1;
  const int n_planes = (int)jobs.size(), n_vtx = (int)vtx.size();
  if (C.check_device(device) < 0) return -1;
  PUS_CALL_OK(C, cudaSetDevice(device));
  TempAlloc A;
  Job* d_jobs = nullptr;
  int2 *d_vtx = nullptr, *d_span = nullptr;
  float *d_planes = nullptr, *d_T = nullptr, *d_K = nullptr, *d_xyz = nullptr;
  unsigned char *d_img = nullptr, *d_rgb = nullptr, *d_lab = nullptr;
  int *d_rowcnt = nullptr, *d_cnt = nullptr, *d_ptr = nullptr;
  long long *d_rowoff = nullptr, *d_off = nullptr;
  const size_t img_bytes = (size_t)n_frames * width * height * 3;
  PUS_CALL_OK(C, A.upload(d_jobs, jobs.data(), n_planes));
  PUS_CALL_OK(C, A.upload(d_planes, planes_sensor, (size_t)n_planes * 4));
  PUS_CALL_OK(C, A.upload(d_vtx, vtx.data(), n_vtx));
  PUS_CALL_OK(C, A.upload(d_T, Ts, (size_t)n_frames * 16));
  PUS_CALL_OK(C, A.upload(d_K, invK, n_frames > 0 ? 9 : 0));
  PUS_CALL_OK(C, A.get(d_span, rows));
  PUS_CALL_OK(C, A.get(d_rowcnt, rows));
  PUS_CALL_OK(C, A.get(d_rowoff, rows + 1));
  PUS_CALL_OK(C, A.get(d_cnt, n_planes));
  PUS_CALL_OK(C, A.get(d_off, n_planes));
  if (images && rgb) PUS_CALL_OK(C, A.upload(d_img, images, img_bytes));
  Params P{d_jobs, d_vtx, d_planes, d_T, d_K, d_img, width, height, downsample ? 2 : 1, images && width == 960, depth_thre,
           ceiling_threshold, d_span, d_rowcnt, d_rowoff, nullptr, nullptr};
  PUS_CALL_OK(C, launch_count(0, n_planes, rows, P, d_rowoff, d_cnt, d_off));
  long long total = 0;
  PUS_CALL_OK(C, download(&total, d_rowoff + rows, 1));
  if (counts) PUS_CALL_OK(C, download(counts, d_cnt, n_planes));
  if (offsets) PUS_CALL_OK(C, download(offsets, d_off, n_planes));
  if ((xyz || rgb) && capacity < total) return C.refuse("capacity is smaller than the number of points");
  if ((xyz || rgb) && total > 0) {
    if (xyz) PUS_CALL_OK(C, A.get(d_xyz, (size_t)total * 3));
    if (rgb) PUS_CALL_OK(C, A.get(d_rgb, (size_t)total * 3));
    P.xyz = d_xyz;
    P.rgb = d_rgb;
    PUS_CALL_OK(C, launch_write(0, n_planes, P));
    if (xyz) PUS_CALL_OK(C, download(xyz, d_xyz, (size_t)total * 3));
    if (rgb) PUS_CALL_OK(C, download(rgb, d_rgb, (size_t)total * 3));
  }
  if (labels && n_frames > 0) {
    PUS_CALL_OK(C, A.get(d_lab, (size_t)n_frames * width * height));
    PUS_CALL_OK(C, A.upload(d_ptr, plane_ptr, n_frames + 1));
    PUS_CALL_OK(C, cudaMemset(d_lab, 127, (size_t)n_frames * width * height));
    PUS_CALL_OK(C, launch_labels(0, n_frames, d_ptr, P, d_lab));
    PUS_CALL_OK(C, download(labels, d_lab, (size_t)n_frames * width * height));
  }
  PUS_CALL_OK(C, cudaDeviceSynchronize());
  return total;
}

extern "C" int pus_popup_depth(int device, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                               const float* planes_sensor, const float* Ts, const float* invK, int width, int height,
                               int downsample, float ceiling_threshold, float* depth) {
  using namespace pus::cloud;
  const Call C{"pus_popup_depth"};
  if (n_frames < 0) return C.refuse("n_frames < 0");
  if (!plane_ptr || plane_ptr[0] != 0) return C.refuse("plane_ptr must be given and start at 0");
  if (width <= 0 || height <= 0) return C.refuse("width and height must be positive");
  if (downsample && ((width | height) & 1)) return C.refuse("downsample mode needs an even width and height");
  if (!depth) return C.refuse("depth must be given");
  std::vector<Job> jobs;
  std::vector<int2> vtx;
  const long long rows = plane_jobs(C, n_frames, plane_ptr, poly_ptr, polys, planes_sensor, Ts, invK, downsample, jobs, vtx);
  if (rows < 0) return -1;
  const int n_planes = (int)jobs.size(), n_vtx = (int)vtx.size();
  if (C.check_device(device) < 0) return -1;
  if (n_frames == 0) return 0;
  PUS_CALL_OK(C, cudaSetDevice(device));
  const int scale = downsample ? 2 : 1, fw = width / scale, fh = height / scale;
  const size_t out_n = (size_t)n_frames * width * height, fill_n = (size_t)n_frames * fw * fh;
  TempAlloc A;
  Job* d_jobs = nullptr;
  int2 *d_vtx = nullptr, *d_span = nullptr;
  Edge* d_edges = nullptr;
  float *d_planes = nullptr, *d_T = nullptr, *d_K = nullptr, *d_fill = nullptr, *d_out = nullptr;
  int* d_ptr = nullptr;
  PUS_CALL_OK(C, A.upload(d_jobs, jobs.data(), n_planes));
  PUS_CALL_OK(C, A.upload(d_planes, planes_sensor, (size_t)n_planes * 4));
  PUS_CALL_OK(C, A.upload(d_vtx, vtx.data(), n_vtx));
  PUS_CALL_OK(C, A.upload(d_T, Ts, (size_t)n_frames * 16));
  PUS_CALL_OK(C, A.upload(d_K, invK, 9));
  PUS_CALL_OK(C, A.upload(d_ptr, plane_ptr, n_frames + 1));
  PUS_CALL_OK(C, A.get(d_edges, n_vtx));
  PUS_CALL_OK(C, A.get(d_span, rows));
  PUS_CALL_OK(C, A.get(d_fill, fill_n));
  if (downsample) PUS_CALL_OK(C, A.get(d_out, out_n));
  PUS_CALL_OK(C, launch_depth(0, n_frames, n_planes, d_ptr, d_jobs, d_vtx, d_edges, d_span, d_planes, d_T, d_K, width,
                              height, downsample, ceiling_threshold, d_fill, d_out));
  PUS_CALL_OK(C, download(depth, downsample ? d_out : d_fill, out_n));
  return 0;
}

// ---- closed wall and ground polygons (pus_popup_polygons) -------------------------------------------------------------
// popup_plane::find_2d_3d_closed_polygon (popup_plane.cpp:120-406) with direction_hit_boundary, polygon_overlap_func,
// find_correct_ground_seq and cut_wall_polygons (matrix_utils.cpp:229-270, 506-713), and OpenCV 4.13's cv::convexHull and
// cv::pointPolygonTest on Point2f.  One thread per (frame, plane) row; the polygons go to fixed per-row slots, and a second
// pass packs the slots in row order at offsets scanned from the counts.
namespace pus {
namespace poly {
struct P3 { float x, y, z; };

// P2, trunc_i and hit_boundary (direction_hit_boundary) are in pus_edges.cuh, shared with pus_popup_edges
__device__ __forceinline__ int sgnf(float a) { return (a > 0.f) - (a < 0.f); }

__device__ int sklansky(const P2* p, const int* ord, int start, int end, int* stack, int nsign, int sign2) {
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
    if (sgnf(by) != nsign) {
      const float ax = p[ord[pcur]].x - p[ord[pprev]].x, bx = p[ord[pnext]].x - p[ord[pcur]].x, ay = cury - p[ord[pprev]].y;
      const float convexity = ay * bx - ax * by;
      if (sgnf(convexity) == sign2 && (ax != 0 || ay != 0)) {
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

// cv::convexHull(points, hull, clockwise = false, returnPoints = true); n <= kHullMax.  The sort is an insertion sort on
// OpenCV's order (x, y, then position), a total order, so it gives std::sort's result.
__device__ int convex_hull(const P2* p, int n, P2* out) {
  if (n <= 0) return 0;
  int ord[kHullMax], stack[kHullMax + 2], hull[kHullMax];
  for (int i = 0; i < n; i++) ord[i] = i;
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
    // upper half, right chain first (clockwise = false)
    int tlc = sklansky(p, ord, 0, maxy, stack, -1, 1);
    int* tr = stack;
    int* tl = stack + tlc;
    int trc = tlc;
    tlc = sklansky(p, ord, n - 1, maxy, tl, -1, -1);
    for (int i = 0; i < tlc - 1; i++) hull[nout++] = ord[tl[i]];
    for (int i = trc - 1; i > 0; i--) hull[nout++] = ord[tr[i]];
    const int stop = trc > 2 ? tr[1] : tlc > 2 ? tl[tlc - 2] : -1;
    int* bl = stack;
    int blc = sklansky(p, ord, 0, miny, bl, 1, -1);
    int* br = stack + blc;
    int brc = sklansky(p, ord, n - 1, miny, br, 1, 1);
    if (stop >= 0) {
      const int check = blc > 2 ? bl[1] : blc + brc > 2 ? br[2 - blc] : -1;
      if (check == stop || (check >= 0 && p[ord[check]].x == p[ord[stop]].x && p[ord[check]].y == p[ord[stop]].y)) {
        blc = min(blc, 2);
        brc = min(brc, 2);
      }
    }
    for (int i = 0; i < blc - 1; i++) hull[nout++] = ord[bl[i]];
    for (int i = brc - 1; i > 0; i--) hull[nout++] = ord[br[i]];
    if (nout >= 3) {   // the cyclic shift that makes the indices ascending or descending where one exists
      int min_idx = 0, max_idx = 0, lt = 0;
      for (int i = 1; i < nout; i++) {
        const int idx = hull[i];
        lt += hull[i - 1] < idx;
        if (lt > 1 && lt <= i - 2) break;
        if (idx < hull[min_idx]) min_idx = i;
        if (idx > hull[max_idx]) max_idx = i;
      }
      const int mmdist = abs(max_idx - min_idx);
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
          if (i == nout)
            for (int k = 0; k < nout; k++) hull[k] = stack[k];
        }
      }
    }
  }
  for (int i = 0; i < nout; i++) out[i] = p[hull[i]];
  return nout;
}

// cv::pointPolygonTest(contour, pt, measureDist = false): 1 inside, 0 on the outline, -1 outside
__device__ int point_polygon_test(const P2* c, int n, P2 pt) {
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
    // products of two floats are exact in double, so only the difference rounds
    double dist = (double)(pt.y - v0.y) * (double)(v.x - v0.x) - (double)(pt.x - v0.x) * (double)(v.y - v0.y);
    if (dist == 0) return 0;
    if (v.y < v0.y) dist = -dist;
    counter += dist > 0;
  }
  return counter % 2 == 0 ? -1 : 1;
}

// A (p, 1) for a row-major 4x4 A, divided by its fourth component (homo_to_real_coord)
__device__ __forceinline__ P3 xform(const float* A, P3 p) {
  float h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = A[i * 4 + 0] * p.x + A[i * 4 + 1] * p.y + A[i * 4 + 2] * p.z + A[i * 4 + 3] * 1.0f;
  return P3{h[0] / h[3], h[1] / h[3], h[2] / h[3]};
}
__device__ __forceinline__ P2 project(const float* K, P3 p) {
  float q[3];
#pragma unroll
  for (int i = 0; i < 3; i++) q[i] = K[i * 3 + 0] * p.x + K[i * 3 + 1] * p.y + K[i * 3 + 2] * p.z;
  return P2{q[0] / q[2], q[1] / q[2]};
}
__device__ __forceinline__ float norm3(P3 a) { return sqrtf(a.x * a.x + a.y * a.y + a.z * a.z); }

// polygon_overlap_func: the hull of the corners inside both closed polygons and of their edges' crossings
// (lineSegmentIntersect_f2); a has at most kWallMax vertices, b is the 5-vertex cut box
__device__ int overlap(const P2* a, int na, const P2* b, int nb, P2* out) {
  P2 sect[kHullMax], inside[kHullMax];
  int ns = 0, ni = 0;
  for (int i = 0; i + 1 < na; i++)
    for (int j = 0; j + 1 < nb; j++) {
      const float X2_X1 = a[i + 1].x - a[i].x, Y2_Y1 = a[i + 1].y - a[i].y;
      const float X4_X3 = b[j + 1].x - b[j].x, Y4_Y3 = b[j + 1].y - b[j].y;
      const float X1_X3 = a[i].x - b[j].x, Y1_Y3 = a[i].y - b[j].y;
      const float ua = (X4_X3 * Y1_Y3 - Y4_Y3 * X1_X3) / (Y4_Y3 * X2_X1 - X4_X3 * Y2_Y1);
      const float ub = (X2_X1 * Y1_Y3 - Y2_Y1 * X1_X3) / (Y4_Y3 * X2_X1 - X4_X3 * Y2_Y1);
      const float ix = a[i].x + X2_X1 * ua, iy = a[i].y + Y2_Y1 * ua;
      const float ib = (float)((ua >= 0) && (ua <= 1) && (ub >= 0) && (ub <= 1));
      if ((ua >= 0) && (ua <= 1) && (ub >= 0) && (ub <= 1)) sect[ns++] = P2{ix * ib, iy * ib};
    }
  for (int k = 0; k < (na - 1) + (nb - 1); k++) {
    const P2 c = k < na - 1 ? a[k] : b[k - (na - 1)];
    if (point_polygon_test(a, na, c) >= 0 && point_polygon_test(b, nb, c) >= 0) inside[ni++] = c;
  }
  for (int k = 0; k < ns; k++) inside[ni++] = sect[k];
  return convex_hull(inside, ni, out);
}

// find_correct_ground_seq; 0 = none.  Where the reference would index past its hull (one of the two ground vertices
// missing and the other not next to the wrap) this also returns 0, i.e. the uncut polygon.
__device__ int ground_seq(const P2* q, int n, bool originkept, int* seq) {
  int first = -1, second = -1;
  for (int i = 0; i < n; i++)
    if ((double)fabsf(q[i].y) < 1e-3) {
      if (originkept) {
        if ((double)fabsf(q[i].x) < 1e-3) first = i;
        else second = i;
      } else {
        if (first == -1) first = i;
        else second = i;
      }
    }
  if (!(abs(first - second) == 1 || abs(first - second) == n - 1)) return 0;
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

// cut_wall_polygons (matrix_utils.cpp:642-713): the wall polygon P (world frame, closed) cut to the box of height
// [-1, ceiling] and, with walllength >= 0, of that length from the ground endpoint nearer the camera
__device__ int cut_wall(const P3* P, int m, float ceiling, float walllength, P3 cam, P3* out) {
  const P3 d{P[1].x - P[0].x, P[1].y - P[0].y, P[1].z - P[0].z};
  const float z = d.x * d.x + d.y * d.y + d.z * d.z;
  P3 dir = d;
  if (z > 0) {   // Eigen's normalized()
    const float s = sqrtf(z);
    dir = P3{d.x / s, d.y / s, d.z / s};
  }
  const float L = norm3(d);
  P2 poly[kWallMax];
  for (int i = 0; i < m; i++) {
    const P3 r{P[i].x - P[0].x, P[i].y - P[0].y, P[i].z - P[0].z};
    poly[i] = P2{r.x * dir.x + r.y * dir.y + r.z * dir.z, P[i].z};
  }
  const bool height_only = walllength < 0;
  float x0 = -1.f, x1 = L + 1;
  if (!height_only) {
    const float s0 = norm3(P3{cam.x - P[0].x, cam.y - P[0].y, cam.z - P[0].z});
    const float s1 = norm3(P3{cam.x - P[1].x, cam.y - P[1].y, cam.z - P[1].z});
    if (s0 < s1) {
      x1 = walllength;
    } else {
      x0 = poly[1].x - walllength;
      x1 = poly[1].x + 1;
    }
  }
  const P2 box[5] = {{x0, -1.f}, {x1, -1.f}, {x1, ceiling}, {x0, ceiling}, {x0, -1.f}};
  P2 hull[kHullMax];
  const int nh = overlap(poly, m, box, 5, hull);
  int seq[kCutSlot];
  const int ns = ground_seq(hull, nh, height_only, seq);
  if (ns == 0) {   // the reference prints "BAD cut_wall_polygons1" and keeps the uncut polygon
    for (int i = 0; i < m; i++) out[i] = P[i];
    return m;
  }
  for (int i = 0; i < ns; i++) {
    const P2 h = hull[seq[i]];
    out[i] = P3{(P[0].x + h.x * dir.x) + h.y * 0.f, (P[0].y + h.x * dir.y) + h.y * 0.f, (P[0].z + h.x * dir.z) + h.y * 1.f};
  }
  return ns;
}

// the up image direction of a world vertical at ground endpoint k of the frame's segment s (popup_plane.cpp:127-143)
__device__ P2 up_direction(const Params& P, const float* K, const float* iT, int row_of_seg, int k) {
  const float* e = P.ends + (size_t)row_of_seg * 6 + 3 * k;
  const P3 v0{e[0], e[1], e[2]}, v1{e[0] + 0.f, e[1] + 0.f, e[2] + 2.f};
  const P2 i0 = project(K, xform(iT, v0)), i1 = project(K, xform(iT, v1));
  P2 dir{i1.x - i0.x, i1.y - i0.y};
  if (dir.y > 0) dir = P2{-dir.x, -dir.y};
  return dir;
}

__global__ void polygon_kernel(Params P) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= P.n_rows) return;
  const int f = P.row_frame[row];
  const int s0 = P.seg_ptr[f];
  const int n = P.seg_ptr[f + 1] - s0;
  const int j = row - (s0 + f);
  int* cnt = P.counts;
  if (n <= 0) {
    cnt[row] = cnt[P.n_rows + row] = cnt[2 * P.n_rows + row] = 0;
    return;
  }
  float T[16], K[9], iT[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = P.Ts[(size_t)f * 16 + i];
#pragma unroll
  for (int i = 0; i < 9; i++) K[i] = P.K[i];
  // the camera inverse in closed form, [R^T | -R^T t]
#pragma unroll
  for (int i = 0; i < 3; i++) {
#pragma unroll
    for (int c = 0; c < 3; c++) iT[i * 4 + c] = T[c * 4 + i];
    iT[i * 4 + 3] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
  iT[12] = 0.f; iT[13] = 0.f; iT[14] = 0.f; iT[15] = 1.f;
  const float W1 = (float)(P.width - 1), H1 = (float)(P.height - 1);
  const float* S = P.segs + (size_t)s0 * 4;
  float* B = P.bound + (size_t)row * kBoundSlot * 2;
  int nb = 0;
  auto push = [&](P2 q) { B[2 * nb] = q.x; B[2 * nb + 1] = q.y; nb++; };
  if (j == 0) {   // ground polygon (popup_plane.cpp:158-196)
    for (int s = 0; s < n; s++) push(P2{S[4 * s], S[4 * s + 1]});
    const float* l = S + 4 * (n - 1);
    push(P2{l[2], l[3]});
    if (l[3] == H1 && l[2] < W1) {
    } else if (l[2] == W1 && l[3] <= H1) {
      push(P2{W1, H1});
    } else {
      const P2 u = up_direction(P, K, iT, s0 + f + n, 1);
      const P2 eh = hit_boundary(P2{l[2], l[3]}, P2{-u.x, -u.y}, P.width, P.height);
      if (eh.x == W1) { push(eh); push(P2{W1, H1}); }
      if (0 <= eh.x && eh.x < W1) push(eh);
    }
    const float* g = S;
    if (g[1] == H1 && g[0] > 0) {
    } else if (g[0] == 0 && g[1] <= H1) {
      push(P2{0.f, H1});
    } else {
      const P2 ub = up_direction(P, K, iT, s0 + f + 1, 0), ue = up_direction(P, K, iT, s0 + f + 1, 1);
      const P2 bh = hit_boundary(P2{g[0], g[1]}, P2{-ub.x, -ub.y}, P.width, P.height);
      const P2 eh = hit_boundary(P2{g[2], g[3]}, P2{-ue.x, -ue.y}, P.width, P.height);
      if (bh.x == W1) { push(P2{0.f, H1}); push(eh); }   // the reference pushes the end's hit in both cases
      if (0 <= bh.x && bh.x < W1) push(eh);
    }
    push(P2{B[0], B[1]});
    cnt[row] = nb;
    cnt[P.n_rows + row] = nb;   // the cut polygon of the ground is its bound polygon, packed from the bound slot
    cnt[2 * P.n_rows + row] = 0;
    return;
  }
  // wall polygon (popup_plane.cpp:198-344)
  const int s = j - 1;
  const float* g = S + 4 * s;
  P2 p[kWallMax];
  int m = 0;
  p[m++] = P2{g[0], g[1]};
  p[m++] = P2{g[2], g[3]};
  const P2 ub = up_direction(P, K, iT, row, 0), ue = up_direction(P, K, iT, row, 1);
  const P2 bh = hit_boundary(P2{g[0], g[1]}, ub, P.width, P.height);
  const P2 eh = hit_boundary(P2{g[2], g[3]}, ue, P.width, P.height);
  auto general = [&]() {
    if (bh.x == W1 && eh.x == W1) { p[m++] = eh; p[m++] = bh; }
    if (0 < bh.x && bh.x < W1 && eh.x == W1) { p[m++] = eh; p[m++] = P2{W1, 0.f}; p[m++] = bh; }
    if (0 < bh.x && bh.x < W1 && 0 < eh.x && eh.x < W1) { p[m++] = eh; p[m++] = bh; }
    if (bh.x == 0 && 0 < eh.x && eh.x < W1) { p[m++] = eh; p[m++] = P2{0.f, 0.f}; p[m++] = bh; }
    if (bh.x == 0 && eh.x == 0) { p[m++] = eh; p[m++] = bh; }
  };
  auto right_begin = [&]() {
    if (bh.x == W1) p[m++] = bh;
    if (0 < bh.x && bh.x < W1) { p[m++] = P2{W1, 0.f}; p[m++] = bh; }
    if (bh.x == 0) { p[m++] = P2{W1, 0.f}; p[m++] = P2{0.f, 0.f}; p[m++] = bh; }
  };
  auto left_end = [&]() {
    if (eh.x == W1) { p[m++] = eh; p[m++] = P2{W1, 0.f}; p[m++] = P2{0.f, 0.f}; }
    if (0 < eh.x && eh.x < W1) { p[m++] = eh; p[m++] = P2{0.f, 0.f}; }
    if (eh.x == 0) p[m++] = eh;
  };
  if (s == n - 1) {   // rightmost
    if (g[3] == H1 && g[2] < W1) { p[m++] = P2{W1, H1}; right_begin(); }
    else if (g[2] == W1 && g[3] <= H1) right_begin();
    else general();
  } else if (0 < s && s < n - 1) {
    general();
  } else {            // leftmost
    if (g[1] == H1 && g[0] > 0) { left_end(); p[m++] = P2{0.f, H1}; }
    else if (g[0] == 0 && g[1] <= H1) left_end();
    else general();
  }
  p[m++] = P2{g[0], g[1]};
  for (int i = 0; i < m; i++) push(p[i]);
  // onto the wall plane, to the world frame, cut, and back into the image (popup_plane.cpp:346-404)
  float invK[9], pl[4];
#pragma unroll
  for (int i = 0; i < 9; i++) invK[i] = P.invK[i];
#pragma unroll
  for (int i = 0; i < 4; i++) pl[i] = P.planes[(size_t)row * 4 + i];
  P3 Q[kWallMax];
  for (int i = 0; i < m; i++) {
    float ray[3];
#pragma unroll
    for (int k = 0; k < 3; k++) ray[k] = invK[k * 3 + 0] * p[i].x + invK[k * 3 + 1] * p[i].y + invK[k * 3 + 2] * 1.0f;
    const float frac = -pl[3] / (pl[0] * ray[0] + pl[1] * ray[1] + pl[2] * ray[2]);
    Q[i] = xform(T, P3{frac * ray[0], frac * ray[1], frac * ray[2]});
  }
  Q[0].z = 0.f;
  Q[1].z = 0.f;
  P3 out[kCutSlot];
  const int nc = cut_wall(Q, m, P.ceiling, P.walllength, P3{T[3], T[7], T[11]}, out);
  float* C = P.cut + (size_t)row * kCutSlot * 2;
  float* Wd = P.world + (size_t)row * kCutSlot * 3;
  for (int i = 0; i < nc; i++) {
    const P2 q = project(K, xform(iT, out[i]));
    C[2 * i] = q.x; C[2 * i + 1] = q.y;
    Wd[3 * i] = out[i].x; Wd[3 * i + 1] = out[i].y; Wd[3 * i + 2] = out[i].z;
  }
  cnt[row] = nb;
  cnt[P.n_rows + row] = nc;
  cnt[2 * P.n_rows + row] = nc;
}

// pack every row's slots at its offsets (off[3][n_rows], exclusive scans of the counts); the ground's cut polygon is its
// bound polygon
__global__ void pack_kernel(int n_rows, const int* row_frame, const int* seg_ptr, const int* counts, const long long* off,
                            const float* bound, const float* cut, const float* world, float* ob, float* oc, float* ow) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n_rows) return;
  const int f = row_frame[row];
  const bool ground = row == seg_ptr[f] + f;
  const float* b = bound + (size_t)row * kBoundSlot * 2;
  if (ob)
    for (int i = 0; i < 2 * counts[row]; i++) ob[2 * off[row] + i] = b[i];
  if (oc) {
    const float* c = ground ? b : cut + (size_t)row * kCutSlot * 2;
    for (int i = 0; i < 2 * counts[n_rows + row]; i++) oc[2 * off[n_rows + row] + i] = c[i];
  }
  if (ow)
    for (int i = 0; i < 3 * counts[2 * n_rows + row]; i++) ow[3 * off[2 * n_rows + row] + i] = world[(size_t)row * kCutSlot * 3 + i];
}

cudaError_t launch_rows(cudaStream_t st, const Params& P) {
  if (P.n_rows > 0) polygon_kernel<<<(P.n_rows + 127) / 128, 128, 0, st>>>(P);
  return cudaGetLastError();
}
cudaError_t launch_pack(cudaStream_t st, const Params& P, const long long* d_off, float* ob, float* oc, float* ow) {
  if (P.n_rows > 0)
    pack_kernel<<<(P.n_rows + 255) / 256, 256, 0, st>>>(P.n_rows, P.row_frame, P.seg_ptr, P.counts, d_off, P.bound, P.cut,
                                                        P.world, ob, oc, ow);
  return cudaGetLastError();
}
}  // namespace poly
}  // namespace pus

extern "C" int pus_popup_polygons(int device, int n_frames, const int* seg_ptr, const float* segs, const float* K,
                                  const float* invK, const float* Ts, int width, int height, float ceiling_threshold,
                                  float walllength_threshold, int* bound_counts, int* cut_counts, int* world_counts,
                                  float* bound2d, float* cut2d, float* world3d, long long bound_capacity,
                                  long long cut_capacity, long long world_capacity) {
  using namespace pus::poly;
  const Call C{"pus_popup_polygons"};
  auto finite = [](const float* a, size_t n) {
    for (size_t i = 0; i < n; i++)
      if (!std::isfinite(a[i])) return false;
    return true;
  };
  if (n_frames < 0) return C.refuse("n_frames < 0");
  std::vector<int> rf;
  if (const char* why = row_frames(n_frames, seg_ptr, rf, true)) return C.refuse(why);
  if (width < 2 || height < 2) return C.refuse("width and height must be at least 2");
  const int n_seg = seg_ptr[n_frames];
  const int n_rows = n_seg + n_frames;
  if (n_seg > 0 && !segs) return C.refuse("segs must be given");
  for (long long i = 0; i < 4LL * n_seg; i++)
    if (!(std::fabs(segs[i]) <= PUS_POPUP_MAX_COORD)) return C.refuse("a segment coordinate is not finite or exceeds PUS_POPUP_MAX_COORD");
  if (!K || !invK || !finite(K, 9) || !finite(invK, 9)) return C.refuse("K and invK must be given and finite");
  if (n_frames > 0 && (!Ts || !finite(Ts, (size_t)n_frames * 16))) return C.refuse("Ts must be given and finite");
  if (!bound_counts || !cut_counts || !world_counts) return C.refuse("the count arrays must be given");
  if (n_frames == 0) return 0;
  if (C.check_device(device) < 0) return -1;
  PUS_CALL_OK(C, cudaSetDevice(device));
  TempAlloc A;
  int *d_ptr = nullptr, *d_rf = nullptr, *d_cnt = nullptr;
  float *d_segs = nullptr, *d_K = nullptr, *d_iK = nullptr, *d_T = nullptr, *d_pl = nullptr, *d_ends = nullptr, *d_b = nullptr,
        *d_c = nullptr, *d_w = nullptr, *d_ob = nullptr, *d_oc = nullptr, *d_ow = nullptr;
  long long* d_off = nullptr;
  PUS_CALL_OK(C, A.upload(d_ptr, seg_ptr, n_frames + 1));
  PUS_CALL_OK(C, A.upload(d_rf, rf.data(), n_rows));
  PUS_CALL_OK(C, A.upload(d_segs, segs, (size_t)n_seg * 4));
  PUS_CALL_OK(C, A.upload(d_K, K, 9));
  PUS_CALL_OK(C, A.upload(d_iK, invK, 9));
  PUS_CALL_OK(C, A.upload(d_T, Ts, (size_t)n_frames * 16));
  PUS_CALL_OK(C, A.get(d_pl, (size_t)n_rows * 4));
  PUS_CALL_OK(C, A.get(d_ends, (size_t)n_rows * 6));
  PUS_CALL_OK(C, A.get(d_b, (size_t)n_rows * kBoundSlot * 2));
  PUS_CALL_OK(C, A.get(d_c, (size_t)n_rows * kCutSlot * 2));
  PUS_CALL_OK(C, A.get(d_w, (size_t)n_rows * kCutSlot * 3));
  PUS_CALL_OK(C, A.get(d_cnt, (size_t)n_rows * 3));
  // the planes and the world ground endpoints: get_plane_equation, as pus_popup_fit_frames runs it (mode 0)
  PUS_CALL_OK(C, launch_fit(0, n_frames, d_ptr, d_rf, n_rows, d_segs, d_iK, d_T, 0.f, 0, nullptr, d_pl, nullptr, nullptr,
                            d_ends));
  Params P{d_ptr, d_rf, n_rows, d_segs, d_K, d_iK, d_T, d_pl, d_ends, width, height, ceiling_threshold,
           walllength_threshold, d_b, d_c, d_w, d_cnt};
  PUS_CALL_OK(C, launch_rows(0, P));
  std::vector<int> cnt((size_t)n_rows * 3);
  PUS_CALL_OK(C, download(cnt.data(), d_cnt, cnt.size()));
  std::memcpy(bound_counts, cnt.data(), n_rows * sizeof(int));
  std::memcpy(cut_counts, cnt.data() + n_rows, n_rows * sizeof(int));
  std::memcpy(world_counts, cnt.data() + 2 * (size_t)n_rows, n_rows * sizeof(int));
  // row offsets of the packed outputs, in row order
  std::vector<long long> off((size_t)n_rows * 3);
  long long tot[3] = {0, 0, 0};
  for (int k = 0; k < 3; k++)
    for (int r = 0; r < n_rows; r++) {
      off[(size_t)k * n_rows + r] = tot[k];
      tot[k] += cnt[(size_t)k * n_rows + r];
    }
  if ((bound2d && bound_capacity < tot[0]) || (cut2d && cut_capacity < tot[1]) || (world3d && world_capacity < tot[2]))
    return C.refuse("a capacity is smaller than its number of vertices");
  if (!bound2d && !cut2d && !world3d) return 0;   // size query
  PUS_CALL_OK(C, A.upload(d_off, off.data(), off.size()));
  if (bound2d) PUS_CALL_OK(C, A.get(d_ob, (size_t)tot[0] * 2));
  if (cut2d) PUS_CALL_OK(C, A.get(d_oc, (size_t)tot[1] * 2));
  if (world3d) PUS_CALL_OK(C, A.get(d_ow, (size_t)tot[2] * 3));
  PUS_CALL_OK(C, launch_pack(0, P, d_off, d_ob, d_oc, d_ow));
  if (bound2d) PUS_CALL_OK(C, download(bound2d, d_ob, (size_t)tot[0] * 2));
  if (cut2d) PUS_CALL_OK(C, download(cut2d, d_oc, (size_t)tot[1] * 2));
  if (world3d) PUS_CALL_OK(C, download(world3d, d_ow, (size_t)tot[2] * 3));
  PUS_CALL_OK(C, cudaDeviceSynchronize());
  return 0;
}

// ---- ground edges (pus_popup_edges) ----------------------------------------------------------------------------------
// popup_plane::edge_get_polygons (select_edge.cpp:66-406) with pop_up_fun.python_get_contours and
// interval_tree_optimization.  The label preprocessing runs as four separable box passes, one thread per pixel; a per-cell
// kernel counts each frame's marching-squares segments (integer atomics: the count does not depend on their order) so the
// host can size the assembly scratch; then one thread per frame, each in a block of its own so that the frames' divergent
// sequential work does not serialise within a warp, replays the order-dependent part -- the dict-driven
// contour assembly in cell order and the restart loops of the selection -- with the shared code of pus_edges.cuh.
namespace pus {
namespace edges {
// one box pass over all frames; pass 0 reads the label maps (with the 0.5x pick), the last one writes 255 - v
__global__ void edge_box_kernel(int n_frames, const unsigned char* src, int sw, int sh, int ds, int w, int h, int k, int horiz,
                                int dilate, int invert, unsigned char* dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x, per = (long long)w * h;
  if (i >= per * n_frames) return;
  const int f = (int)(i / per), p = (int)(i % per);
  const unsigned char v = box_pass(src + (long long)f * sw * sh, sw, sh, ds, w, h, p % w, p / w, k, horiz, dilate);
  dst[i] = invert ? (unsigned char)(255 - v) : v;
}

__global__ void edge_count_kernel(int n_frames, const unsigned char* map, int w, int h, int* counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x, per = (long long)(w - 1) * (h - 1);
  if (i >= per * n_frames) return;
  const int f = (int)(i / per), p = (int)(i % per);
  const int c = cell_count(map + (long long)f * w * h, w, p / (w - 1), p % (w - 1));
  if (c) atomicAdd(counts + f, c);
}

__global__ void edge_frame_kernel(int n_frames, pus_edge_params P, int width, int height, const unsigned char* map, int w,
                                  int h, const Frame* fr, int* tab, int* nodes, int* objs, unsigned char* flags, float* cpts,
                                  const float* lines, Lin* rows, float* bounds, Ivl* ivl, float* open_slot, float* conn_slot,
                                  int* in_conn_slot, int* out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const Frame F = fr[f];
  const long long cells = (long long)w * h;
  Asm A{tab + F.tab, tab + F.tab + cells, nodes + 2 * F.node, nodes + 2 * F.node + F.node_cap, objs + 3 * F.obj,
        objs + 3 * F.obj + F.obj_cap, objs + 3 * F.obj + 2 * F.obj_cap, flags + 2 * F.obj, flags + 2 * F.obj + F.obj_cap,
        F.node_cap, F.obj_cap, 0, 0, 0u, false};
  Sel S{rows + 2 * F.line, 2 * F.n, ivl + 2 * F.ivl, ivl + 2 * F.ivl + F.ivl_cap, bounds + 2 * F.line, F.ivl_cap};
  int n_open = 0, n_conn = 0;
  unsigned bits = 0;
  const int st = frame_edges(P, width, height, map + (long long)f * cells, w, h, A, cpts + 2 * F.cpt, F.cpt_cap,
                             lines + 4 * (long long)F.l0, F.n, S, open_slot + 8 * (long long)F.l0,
                             conn_slot + 16 * (long long)F.l0, in_conn_slot + 2 * F.l0, n_open, n_conn, bits);
  out[4 * f] = st;
  out[4 * f + 1] = st ? 0 : n_open;
  out[4 * f + 2] = st ? 0 : n_conn;
  out[4 * f + 3] = (int)bits;
}

cudaError_t prep(cudaStream_t st, Alloc& A, int n_frames, const unsigned char* d_labels, int width, int height,
                 const pus_edge_params& P, Maps& M) {
  const int ds = P.downsample_contour ? 1 : 0;
  M.w = ds ? half_size(width) : width;
  M.h = ds ? half_size(height) : height;
  const int w = M.w, h = M.h, kd = ds ? 8 : P.dilation_distance, ke = ds ? 8 : P.erosion_distance;
  const size_t map_n = (size_t)n_frames * w * h;
  unsigned char* d_a = nullptr;
  cudaError_t e;
  if ((e = A.get(d_a, map_n)) != cudaSuccess || (e = A.get(M.map, map_n)) != cudaSuccess ||
      (e = A.get(M.seg_count, n_frames)) != cudaSuccess)
    return e;
  if (n_frames == 0) return cudaSuccess;
  if ((e = cudaMemsetAsync(M.seg_count, 0, n_frames * sizeof(int), st)) != cudaSuccess) return e;
  const unsigned gb = (unsigned)((map_n + 255) / 256);
  edge_box_kernel<<<gb, 256, 0, st>>>(n_frames, d_labels, width, height, ds, w, h, kd, 1, 1, 0, d_a);
  edge_box_kernel<<<gb, 256, 0, st>>>(n_frames, d_a, w, h, 0, w, h, kd, 0, 1, 0, M.map);
  edge_box_kernel<<<gb, 256, 0, st>>>(n_frames, M.map, w, h, 0, w, h, ke, 1, 0, 0, d_a);
  edge_box_kernel<<<gb, 256, 0, st>>>(n_frames, d_a, w, h, 0, w, h, ke, 0, 0, 1, M.map);
  const long long n_cells = (long long)n_frames * (w - 1) * (h - 1);
  edge_count_kernel<<<(unsigned)((n_cells + 255) / 256), 256, 0, st>>>(n_frames, M.map, w, h, M.seg_count);
  return cudaGetLastError();
}

cudaError_t select(cudaStream_t st, Alloc& A, int n_frames, const pus_edge_params& P, int width, int height, const Maps& M,
                   const Frame* d_fr, const long long tot[4], long long n_lines, const float* d_lines, float* d_open,
                   float* d_conn, int* d_inc, int* d_out) {
  const size_t map_n = (size_t)n_frames * M.w * M.h;
  int *d_tab = nullptr, *d_nodes = nullptr, *d_objs = nullptr;
  unsigned char* d_flags = nullptr;
  float *d_cpts = nullptr, *d_bounds = nullptr;
  Lin* d_rows = nullptr;
  Ivl* d_ivl = nullptr;
  cudaError_t e;
  // per frame of n lines: 2 n work and open rows, 4 n connected rows (Sel in pus_edges.cuh)
  if ((e = A.get(d_tab, 2 * map_n)) != cudaSuccess || (e = A.get(d_nodes, 2 * tot[0])) != cudaSuccess ||
      (e = A.get(d_objs, 3 * tot[1])) != cudaSuccess || (e = A.get(d_flags, 2 * tot[1])) != cudaSuccess ||
      (e = A.get(d_cpts, 2 * tot[2])) != cudaSuccess || (e = A.get(d_rows, 2 * n_lines)) != cudaSuccess ||
      (e = A.get(d_bounds, 2 * n_lines)) != cudaSuccess || (e = A.get(d_ivl, 2 * tot[3])) != cudaSuccess)
    return e;
  if (n_frames == 0) return cudaSuccess;
  if ((e = cudaMemsetAsync(d_tab, 0xff, 2 * map_n * sizeof(int), st)) != cudaSuccess) return e;
  edge_frame_kernel<<<n_frames, 1, 0, st>>>(n_frames, P, width, height, M.map, M.w, M.h, d_fr, d_tab, d_nodes, d_objs, d_flags,
                                            d_cpts, d_lines, d_rows, d_bounds, d_ivl, d_open, d_conn, d_inc, d_out);
  return cudaGetLastError();
}
}  // namespace edges
}  // namespace pus

extern "C" int pus_popup_edges(int device, int n_frames, const unsigned char* labels, int width, int height,
                               const int* line_ptr, const float* lines, const pus_edge_params* params, int* status,
                               int* open_counts, int* connect_counts, float* open_segs, float* connect_segs,
                               int* open_in_connect, long long open_capacity, long long connect_capacity) {
  using namespace pus::edges;
  const Call C{"pus_popup_edges"};
  const std::string why = args_error(n_frames, labels, width, height, line_ptr, lines, params, status, open_counts,
                                      connect_counts);
  if (!why.empty()) return C.refuse(why);
  if (C.check_device(device) < 0) return -1;
  if (n_frames == 0) return 0;
  PUS_CALL_OK(C, cudaSetDevice(device));
  const pus_edge_params P = *params;
  const long long n_lines = line_ptr[n_frames];
  TempAlloc A;
  unsigned char* d_lab = nullptr;
  PUS_CALL_OK(C, A.upload(d_lab, labels, (size_t)n_frames * width * height));
  Maps M;
  PUS_CALL_OK(C, prep(0, A, n_frames, d_lab, width, height, P, M));
  std::vector<int> cnt(n_frames);
  PUS_CALL_OK(C, download(cnt.data(), M.seg_count, n_frames));
  // scratch layout
  std::vector<Frame> fr(n_frames);
  long long tot[4] = {0, 0, 0, 0};
  for (int f = 0; f < n_frames; f++)
    pus::glue::edge_frame(f, cnt[f], line_ptr[f], line_ptr[f + 1] - line_ptr[f], (long long)M.w * M.h, tot, fr[f]);
  Frame* d_fr = nullptr;
  float *d_lines = nullptr, *d_open = nullptr, *d_conn = nullptr;
  int *d_inc = nullptr, *d_out = nullptr;
  PUS_CALL_OK(C, A.upload(d_fr, fr.data(), n_frames));
  PUS_CALL_OK(C, A.upload(d_lines, lines, 4 * n_lines));
  PUS_CALL_OK(C, A.get(d_open, 8 * n_lines));
  PUS_CALL_OK(C, A.get(d_conn, 16 * n_lines));
  PUS_CALL_OK(C, A.get(d_inc, 2 * n_lines));
  PUS_CALL_OK(C, A.get(d_out, 4 * (size_t)n_frames));
  PUS_CALL_OK(C, select(0, A, n_frames, P, width, height, M, d_fr, tot, n_lines, d_lines, d_open, d_conn, d_inc, d_out));
  std::vector<int> out(4 * (size_t)n_frames);
  PUS_CALL_OK(C, download(out.data(), d_out, out.size()));
  long long tot_open = 0, tot_conn = 0;
  int found = 0;
  for (int f = 0; f < n_frames; f++) {
    status[f] = out[4 * f];
    open_counts[f] = out[4 * f + 1];
    connect_counts[f] = out[4 * f + 2];
    tot_open += open_counts[f];
    tot_conn += connect_counts[f];
    found += status[f] == 0;
  }
  if ((open_segs && open_capacity < tot_open) || (connect_segs && connect_capacity < tot_conn))
    return C.refuse("a capacity is smaller than its number of segments");
  if (!open_segs && !connect_segs) return found;   // size query
  std::vector<float> os(8 * (size_t)n_lines), cs(16 * (size_t)n_lines);
  std::vector<int> inc(2 * (size_t)n_lines);
  PUS_CALL_OK(C, download(os.data(), d_open, os.size()));
  PUS_CALL_OK(C, download(cs.data(), d_conn, cs.size()));
  PUS_CALL_OK(C, download(inc.data(), d_inc, inc.size()));
  long long po = 0, pc = 0;
  for (int f = 0; f < n_frames; f++) {
    const long long l0 = line_ptr[f];
    if (open_segs) std::memcpy(open_segs + 4 * po, os.data() + 8 * l0, 4 * (size_t)open_counts[f] * sizeof(float));
    if (open_in_connect) std::memcpy(open_in_connect + po, inc.data() + 2 * l0, (size_t)open_counts[f] * sizeof(int));
    if (connect_segs) std::memcpy(connect_segs + 4 * pc, cs.data() + 16 * l0, 4 * (size_t)connect_counts[f] * sizeof(float));
    po += open_counts[f];
    pc += connect_counts[f];
  }
  return found;
}
