// pus_map.cuh -- Mapper_mono::processFrame's rules (pop_planar_slam/src/Mapping.cpp:112-126, 256-530, Map_plane.cpp:11-29,
// main_3d.cpp:366-385) as __host__ __device__ functions: the plane map's kernels run them on the device (pus_map.cu), the
// host oracle (tests/map_oracle.cpp) on the host, so the arithmetic exists once.  Float and double are mixed operation by
// operation as the reference mixes them; both sides are compiled without FMA contraction.
#pragma once
#include <math.h>

#include "../../include/popup_gpu.h"
#include "pus_math.cuh"

namespace pus {
namespace map {

constexpr double kIsamPi = 3.14159265358979323846;   // isam::PI (util.h:40), which Mapping.cpp's PI resolves to

// A frame's good plane as the association reads it (main_3d.cpp:478-492): temp_value, plane_dist_cam, frame_plane_indice,
// good_plane_indice, and the first two vertices of its closed 2-D bound polygon and of its 3-D world polygon.
struct Plane {
  double local[4];   // Plane3d(planes_sensor row as double): normalised
  float dist;
  int ind, good;
  int n2, n3;        // stored vertices: min(polygon size, 2)
  float v2[4], v3[6];
};

// popup_gpu.h's pus_map_landmark is the landmark record on both sides.
typedef pus_map_landmark Landmark;

// Plane3d's accessors (isam_plane3d.h:149-170) on a 4-vector
PUS_HD double abc_norm(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
PUS_HD void normal(const double* v, double* n) {
  const double z = abc_norm(v);
  n[0] = v[0] / z; n[1] = v[1] / z; n[2] = v[2] / z;
}
PUS_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
// Plane3d::distance(point0 of `other`): fabs(normal . (point0(other) - point0(p)))
PUS_HD double plane_distance_to_point0(const double* p, const double* other) {
  double n[3], no[3], q[3], q0[3];
  normal(p, n);
  normal(other, no);
  const double d_other = -other[3] / abc_norm(other), d_p = -p[3] / abc_norm(p);
  for (int k = 0; k < 3; k++) { q[k] = d_other * no[k]; q0[k] = d_p * n[k]; }
  const double r[3] = {q[0] - q0[0], q[1] - q0[1], q[2] - q0[2]};
  return fabs(dot3(n, r));
}

// Vector2f::norm() of a - b
PUS_HD float dist2f(const float* a, const float* b) {
  const float x = a[0] - b[0], y = a[1] - b[1];
  return sqrtf(x * x + y * y);
}
// Vector2f::minCoeff() of (a, b): std::min(a, b)
PUS_HD float min2f(float a, float b) { return b < a ? b : a; }

// point_proj_to_lineseg (Mapping.cpp:112-126); points are x y pairs.  A segment shorter than 0.001 gives the query's
// DISTANCE to begin, not a parameter.
PUS_HD float point_proj_to_lineseg(const float* b, const float* e, const float* q) {
  const float length = dist2f(e, b);
  if ((double)length < 0.001) return dist2f(q, b);
  const float qx = q[0] - b[0], qy = q[1] - b[1], ex = e[0] - b[0], ey = e[1] - b[1];
  const float t = (qx * ex + qy * ey) / length / length;
  if ((double)t > 1.0) return 1.0f;
  if ((double)t < 0.0) return 0.0f;
  return t;
}

// which branch of findClosestPlane a (plane, landmark) pair took
enum PairCode {
  PAIR_DELETED = 0,   // the landmark's plane node was removed (deteted_by_merge)
  PAIR_GROUND = 1,    // both ground: a candidate with error -1; the first one ends the scan
  PAIR_KIND = 2,      // ground against wall
  PAIR_SHORT = 3,     // a wall landmark whose polygons have fewer than two vertices (never matched)
  PAIR_WINDOW = 4,    // older than assoc_near_frames
  PAIR_ANGLE = 5,
  PAIR_PLANEDIST = 6,
  PAIR_2D = 7,
  PAIR_COVER = 8,
  PAIR_MATCH = 9      // passed every gate: a candidate with error *err
};

// findClosestPlane's body (Mapping.cpp:274-380) for plane p of frame seq and landmark L.  cw = p's plane in the world
// (temp_value.transform_from(estimate.oTw())), wTo = estimate.wTo(), lw = the landmark's current plane estimate (NULL when
// its node was removed).  Returns the PairCode; *err is set for PAIR_GROUND and PAIR_MATCH.
PUS_HD int pair(const pus_map_config& cfg, int seq, const Plane& p, const double* cw, const double* wTo, const Landmark& L,
                const double* lw, double* err) {
  if (!lw) return PAIR_DELETED;
  if (p.ind == 0 && L.frame_plane_indice == 0) { *err = -1.0; return PAIR_GROUND; }
  if ((p.ind == 0 && L.frame_plane_indice >= 1) || (p.ind >= 1 && L.frame_plane_indice == 0)) return PAIR_KIND;
  if (L.n_bound2d < 2 || L.n_world3d < 2) return PAIR_SHORT;
  if (seq - L.frame_seq_id > cfg.assoc_near_frames) return PAIR_WINDOW;
  double nc[3], nl[3];
  normal(cw, nc);
  normal(lw, nl);
  const double angle = acos(dot3(nc, nl)) * 180.0 / kIsamPi;   // NaN when |dot| > 1 by rounding: passes the gate
  if (angle > cfg.edge_asso_angle) return PAIR_ANGLE;
  double thr2d = cfg.edge_asso_2ddist, cover = cfg.edge_asso_proj;
  if (angle < 25.0) {
    cover = cfg.edge_asso_proj / 3;
    thr2d = cfg.edge_asso_2ddist * 1.5;
    if (angle <= 10.0) cover = cfg.edge_asso_proj / 2;
  }
  double old_local[4];
  plane_transform_T(wTo, lw, old_local);   // Plane3d::transform_to(wTo)
  const double plane_dist = plane_distance_to_point0(p.local, old_local);
  if (plane_dist > cfg.edge_asso_planedist) return PAIR_PLANEDIST;
  if (plane_dist < 1.5) cover = cover / 2;
  float poly = 0;
  for (int i = 0; i < 2; i++) poly += min2f(dist2f(p.v2 + 2 * i, L.bound2d[0]), dist2f(p.v2 + 2 * i, L.bound2d[1]));
  poly = poly / 2;
  float cross = 0;
  for (int i = 0; i < 2; i++) cross += min2f(dist2f(p.v2, L.bound2d[i]), dist2f(p.v2 + 2, L.bound2d[i]));
  cross = cross / 2;
  if (poly > thr2d || cross > thr2d) return PAIR_2D;
  const float cb[2] = {p.v3[0], p.v3[1]}, ce[2] = {p.v3[3], p.v3[4]};
  const float ob[2] = {L.world3d[0][0], L.world3d[0][1]}, oe[2] = {L.world3d[1][0], L.world3d[1][1]};
  const float old_to_new = fabsf(point_proj_to_lineseg(cb, ce, ob) - point_proj_to_lineseg(cb, ce, oe));
  const float new_to_old = fabsf(point_proj_to_lineseg(ob, oe, cb) - point_proj_to_lineseg(ob, oe, ce));
  if (old_to_new < cover || new_to_old < cover) return PAIR_COVER;
  double total = angle / cfg.edge_asso_angle * 3 + (1 - old_to_new) + (1 - new_to_old);
  total += (poly < cross ? cross : poly) / thr2d + plane_dist / 4;   // std::max(poly, cross)
  *err = total;
  return PAIR_MATCH;
}

// findClosestPlane's selection (:374-377) as an order-free reduction.  Scanned in landmark order, the first candidate sets
// the best error and a later one replaces it only when strictly smaller; a NaN never compares smaller.  So the result is
// the first candidate when its error is NaN, and otherwise the earliest candidate of least non-NaN error -- which the
// state below gives whatever order its parts are merged in.  Ground candidates all carry -1: the first wins (the break).
struct Best {
  int first;  double first_err;   // earliest candidate
  int best;   double best_err;    // earliest candidate of least non-NaN error
};
PUS_HD Best best_none() { return Best{-1, 0.0, -1, 0.0}; }
PUS_HD void best_add(Best& b, int c, double e) {
  if (b.first < 0 || c < b.first) { b.first = c; b.first_err = e; }
  if (!isnan(e) && (b.best < 0 || e < b.best_err || (e == b.best_err && c < b.best))) { b.best = c; b.best_err = e; }
}
PUS_HD Best best_merge(Best a, const Best& b) {
  if (b.first >= 0) best_add(a, b.first, b.first_err);
  if (b.best >= 0) best_add(a, b.best, b.best_err);
  return a;
}
// (bestMatch, bestReprojError): (-1, -1) without a candidate
PUS_HD void best_result(const Best& b, int* id, double* err) {
  if (b.first < 0) { *id = -1; *err = -1.0; }
  else if (isnan(b.first_err)) { *id = b.first; *err = b.first_err; }
  else { *id = b.best; *err = b.best_err; }
}

// per-plane outcome of the association (pus_map_result.status)
enum PlaneStatus {
  ST_MATCHED = 0,     // joined an existing landmark
  ST_SHORT = 1,       // a wall whose bound or world polygon has fewer than two vertices: a new landmark, never matched later
  ST_NEW = 2,         // no candidate: a new landmark
  ST_DUAL_LOST = 3    // a candidate another plane of the frame kept (the one-to-one rule): a new landmark
};

// a wall that findClosestPlane would read past its polygons (.col(1)) for
PUS_HD bool is_short(const Plane& p) { return p.ind != 0 && (p.n2 < 2 || p.n3 < 2); }

// processFrame's one-to-one rule (Mapping.cpp:423-460), in plane order.  id / err are findClosestPlane's results (id -1
// for short planes); num_old landmarks exist.  Writes assoc, assoc_error (the reference's: 0 for a plane without a
// candidate and for the loser that comes second, -1 for the loser that came first) and status; returns numNewPlanes.
PUS_HD int one_to_one(int n, const Plane* P, const int* id, const double* err, int num_old, int* assoc, double* aerr, int* status) {
  int num_new = 0;
  for (int i = 0; i < n; i++) {
    aerr[i] = 0.0;
    if (id[i] > -1) {
      bool conflict = false;
      for (int j = 0; j < i; j++) {
        if (assoc[j] == id[i]) {
          const double raw_length = dist2f(P[j].v2, P[j].v2 + 2);
          const double new_length = dist2f(P[i].v2, P[i].v2 + 2);
          if (new_length > raw_length) {
            assoc[j] = num_old + num_new++;
            aerr[j] = -1;
            status[j] = ST_DUAL_LOST;
            assoc[i] = id[i];
            aerr[i] = err[i];
            status[i] = ST_MATCHED;
          } else {
            assoc[i] = num_old + num_new++;
            aerr[i] = 0.0;
            status[i] = ST_DUAL_LOST;
          }
          conflict = true;
          break;
        }
      }
      if (!conflict) { assoc[i] = id[i]; aerr[i] = err[i]; status[i] = ST_MATCHED; }
    } else {
      assoc[i] = num_old + num_new++;
      status[i] = is_short(P[i]) ? ST_SHORT : ST_NEW;
    }
  }
  return num_new;
}

// the pose-plane factor's sigma (Mapping.cpp:507-510), the same in all three axes
PUS_HD double plane_sigma(double plane_dist, double mul) {
  plane_dist = plane_dist < 3 ? 3 : plane_dist;
  plane_dist = plane_dist > 8 ? 8 : plane_dist;
  return (plane_dist - 1) * mul + 5;
}

// new Map_plane() with its plane node (Map_plane.h's in-class defaults)
PUS_HD void new_landmark(Landmark& L, int node) {
  L.node = node;
  L.deleted = 0;
  L.frame_seq_id = 0; L.frame_plane_indice = 0; L.good_plane_indice = 0; L.being_tracked_times = 0;
  L.plane_dist_cam = 0.0;
  L.n_bound2d = 0; L.n_world3d = 0;
  for (int k = 0; k < 2; k++) { L.bound2d[k][0] = L.bound2d[k][1] = 0.f; L.world3d[k][0] = L.world3d[k][1] = L.world3d[k][2] = 0.f; }
}
// copy_plane (Map_plane.cpp:11-29) from plane p of frame seq: the latest observation's descriptor, one more sighting
PUS_HD void copy_plane(Landmark& L, int seq, const Plane& p) {
  L.frame_seq_id = seq;
  L.frame_plane_indice = p.ind;
  L.good_plane_indice = p.good;
  L.plane_dist_cam = (double)p.dist;
  L.n_bound2d = p.n2; L.n_world3d = p.n3;
  for (int k = 0; k < 2; k++) {
    L.bound2d[k][0] = p.v2[2 * k]; L.bound2d[k][1] = p.v2[2 * k + 1];
    L.world3d[k][0] = p.v3[3 * k]; L.world3d[k][1] = p.v3[3 * k + 1]; L.world3d[k][2] = p.v3[3 * k + 2];
  }
  L.being_tracked_times += 1;
}

// main_3d.cpp:366-385 keyed on the number of mapped frames: none -> odometry and prediction are the initial pose; one ->
// zero odometry; more -> last.ominus(prev).  The prediction is last.oplus(odometry).
PUS_HD void predict_pose(int n_mapped, const double* last, const double* prev, const double* init7, double* odom7, double* pred7) {
  if (n_mapped == 0) {
    for (int k = 0; k < 7; k++) odom7[k] = pred7[k] = init7[k];
    return;
  }
  if (n_mapped == 1) {
    for (int k = 0; k < 7; k++) odom7[k] = 0.0;
    odom7[3] = 1.0;
  } else {
    pose_ominus(last, prev, odom7);
  }
  pose_oplus(last, odom7, pred7);
}
// processFrame's estimate_pose (Mapping.cpp:413-416): the identity until a frame is mapped, then last.oplus(odometry)
PUS_HD void estimate_pose(int n_mapped, const double* last, const double* odom7, double* est7) {
  if (n_mapped == 0) {
    for (int k = 0; k < 7; k++) est7[k] = 0.0;
    est7[3] = 1.0;
  } else {
    pose_oplus(last, odom7, est7);
  }
}
// Plane3d(planes_sensor row cast to double) (main_3d.cpp:478)
PUS_HD void plane_local(const float* ps, double* out) {
  for (int k = 0; k < 4; k++) out[k] = (double)ps[k];
  normalize4(out);
}

}  // namespace map
}  // namespace pus
