// pus_frames.cuh -- the glue between the pop-up stages as __host__ __device__ code: the stage calls run it on the host
// (pus_popup.cu), the pop-up session on the device (pus_frames.cu), so its arithmetic exists once.
#pragma once
#include <climits>
#include <cmath>

#include "pus_edges.cuh"
#include "pus_stages.cuh"

namespace pus {
namespace glue {

// frame f's entry of pus_popup_edges' scratch table: ns marching-squares segments, n lines from line row l0, cells per
// map; the running offsets advance past it
PUS_EHD inline void edge_frame(int f, long long ns, int l0, int n, long long cells, long long run[4], edges::Frame& F) {
  F.node_cap = (int)edges::node_cap_of(ns);
  F.obj_cap = (int)edges::obj_cap_of(ns);
  F.cpt_cap = (int)edges::cpt_cap_of(ns);
  F.n = n;
  F.ivl_cap = (int)edges::ivl_cap_of(n);
  F.l0 = l0;
  F.node = run[0]; F.obj = run[1]; F.cpt = run[2]; F.ivl = run[3]; F.line = l0; F.tab = 2 * cells * f;
  run[0] += F.node_cap; run[1] += F.obj_cap; run[2] += F.cpt_cap; run[3] += F.ivl_cap;
}

// a frame's status after the lines (n of them, x1 y1 x2 y2 each): 1 when pus_popup_edges would refuse them (more than
// PUS_POPUP_MAX_LINES, a coordinate not finite), else 0
PUS_EHD inline int lines_status(const float* lines, int n) {
  if (n > PUS_POPUP_MAX_LINES) return 1;
  for (int i = 0; i < 4 * n; i++)
    if (!isfinite(lines[i])) return 1;
  return 0;
}

// a frame's status after the edges: 2 when a frame with status 0 has more open segments than the polygons take
PUS_EHD inline int edges_status(int status, int n_open) {
  return status == 0 && n_open > PUS_POPUP_MAX_SEGMENTS ? 2 : status;
}

// a polygon of n vertices (q: x y pairs) the clouds and the depth map can take: at most PUS_POPUP_MAX_VERTICES vertices,
// every coordinate finite and of magnitude at most PUS_POPUP_MAX_COORD
PUS_EHD inline bool polygon_ok(const float* q, int n) {
  if (n > PUS_POPUP_MAX_VERTICES) return false;
  for (int i = 0; i < 2 * n; i++)
    if (!(fabsf(q[i]) <= PUS_POPUP_MAX_COORD)) return false;
  return true;
}

// matrix_to_points' truncation, boundingRect and the box-shifted vertices (popup_plane.cpp:85-96) of a checked polygon
// (halved first when downsampling): J's box, vtx[0 .. n) the shifted vertices
PUS_EHD inline void polygon_box(const float* q, int n, int downsample, cloud::Job& J, int2* vtx) {
  int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
  for (int i = 0; i < n; i++) {
    const float fx = downsample ? q[2 * i] / 2.f : q[2 * i], fy = downsample ? q[2 * i + 1] / 2.f : q[2 * i + 1];
    const int x = poly::trunc_i(fx), y = poly::trunc_i(fy);
    xmin = x < xmin ? x : xmin; xmax = x > xmax ? x : xmax; ymin = y < ymin ? y : ymin; ymax = y > ymax ? y : ymax;
  }
  J.bx = xmin; J.by = ymin; J.bw = xmax - xmin + 1; J.bh = ymax - ymin + 1;
  for (int i = 0; i < n; i++) {
    const float fx = downsample ? q[2 * i] / 2.f : q[2 * i], fy = downsample ? q[2 * i + 1] / 2.f : q[2 * i + 1];
    vtx[i] = make_int2(poly::trunc_i(fx - (float)J.bx), poly::trunc_i(fy - (float)J.by));
  }
}

// get_plane_equation's filter (popup_plane.cpp:629-635) with get_ground_edges' actual_plane_indices_inall =
// {0} u {open_in_connect + 1} (:792-794): open wall s (row 1 + s) stays good only when s is one of the frame's
// open_in_connect values.  good[0 .. n_open] are the frame's rows; returns the number still good.
PUS_EHD inline int actual_filter(const int* open_in_connect, int n_open, int* good) {
  int kept = good[0] ? 1 : 0;
  for (int s = 0; s < n_open; s++) {
    bool actual = false;
    for (int i = 0; i < n_open && !actual; i++) actual = open_in_connect[i] == s;
    if (!actual) good[1 + s] = 0;
    kept += good[1 + s] ? 1 : 0;
  }
  return kept;
}
}  // namespace glue
}  // namespace pus
