// Host oracle of the plane map: pus_map.cuh's rules compiled for the host (-ffp-contract=off), with findClosestPlane's
// selection written as the reference's sequential scan (Mapping.cpp:274-380), so that the device's order-free reduction
// is checked against it.  Test infrastructure only.
#include <cmath>
#include <cstring>

#include "../pop_up_slam_b200/csrc/pus_map.cuh"

using namespace pus;
using namespace pus::map;

extern "C" {
int orc_map_plane_size() { return (int)sizeof(Plane); }
int orc_map_landmark_size() { return (int)sizeof(Landmark); }

// Plane records from arrays: planes_sensor [n][4], dist, ind, n2 / n3 (stored vertices), v2 [n][4], v3 [n][6]
void orc_map_planes(int n, const float* ps, const float* dist, const int* ind, const int* n2, const int* n3, const float* v2,
                    const float* v3, Plane* out) {
  for (int i = 0; i < n; i++) {
    Plane& p = out[i];
    plane_local(ps + 4 * i, p.local);
    p.dist = dist[i]; p.ind = ind[i]; p.good = i; p.n2 = n2[i]; p.n3 = n3[i];
    std::memcpy(p.v2, v2 + 4 * i, sizeof(p.v2));
    std::memcpy(p.v3, v3 + 6 * i, sizeof(p.v3));
  }
}

// one pair: est7 the estimate; lw NULL for a removed landmark
int orc_map_pair(const pus_map_config* cfg, int seq, const Plane* p, const double* est7, const Landmark* L, const double* lw, double* err) {
  double wTo[16], oTw[16], cw[4];
  pose_to_T(est7, wTo);
  pose_to_Tinv(est7, oTw);
  plane_transform_T(oTw, p->local, cw);
  return pair(*cfg, seq, *p, cw, wTo, *L, lw, err);
}

// association of one frame: estimate, sequential findClosestPlane per plane, one-to-one rule.  lw [L][4] the landmarks'
// plane estimates, alive [L].  Writes est7, id / err (findClosestPlane), assoc / aerr / status; returns numNewPlanes.
int orc_map_associate(const pus_map_config* cfg, int seq, int n_mapped, const double* last7, const double* odom7, int n,
                      const Plane* P, int L, const Landmark* lm, const double* lw, const int* alive, double* est7, int* id,
                      double* err, int* assoc, double* aerr, int* status) {
  double wTo[16], oTw[16];
  estimate_pose(n_mapped, last7, odom7, est7);
  pose_to_T(est7, wTo);
  pose_to_Tinv(est7, oTw);
  for (int i = 0; i < n; i++) {
    int num = 0, best = -1;
    double best_err = -1;
    if (!is_short(P[i])) {
      double cw[4];
      plane_transform_T(oTw, P[i].local, cw);
      for (int c = 0; c < L; c++) {
        double e = 0;
        const int code = pair(*cfg, seq, P[i], cw, wTo, lm[c], alive[c] ? lw + 4 * c : nullptr, &e);
        if (code == PAIR_GROUND) { num++; best = c; break; }
        if (code != PAIR_MATCH) continue;
        num++;
        if (num == 1 || e < best_err) { best = c; best_err = e; }
      }
    }
    id[i] = best;
    err[i] = best_err;
  }
  return one_to_one(n, P, id, err, L, assoc, aerr, status);
}

// copy_plane of a frame (new landmarks [L0, L0 + n_new) first), then reproj_to_newplane's landmark part with the landmarks'
// plane estimates after the solve (lw [L][4], alive [L])
void orc_map_apply(int seq, int n, const Plane* P, const int* assoc, int L0, int n_new, const int* nodes, Landmark* lm) {
  for (int k = 0; k < n_new; k++) new_landmark(lm[L0 + k], nodes[k]);
  for (int i = 0; i < n; i++) copy_plane(lm[assoc[i]], seq, P[i]);
}
void orc_map_reproject(int L, Landmark* lm, const double* lw, const int* alive) {
  for (int c = 0; c < L; c++) {
    lm[c].deleted = !alive[c];
    if (!alive[c]) continue;
    const double* pl = lw + 4 * c;
    const double nn = std::sqrt(pl[0] * pl[0] + pl[1] * pl[1] + pl[2] * pl[2]);
    const double nx = pl[0] / nn, ny = pl[1] / nn, nz = pl[2] / nn, dd = -pl[3] / nn;
    for (int k = 0; k < lm[c].n_world3d; k++) {
      float* v = lm[c].world3d[k];
      const double px = v[0], py = v[1], pz = v[2];
      const double t = (nx * px + ny * py + nz * pz) - dd;
      v[0] = (float)(px - nx * t); v[1] = (float)(py - ny * t); v[2] = (float)(pz - nz * t);
    }
  }
}

// main_3d.cpp:366-385
void orc_map_predict(int n_mapped, const double* last7, const double* prev7, const double* init_wTo, double* odom7, double* pred7,
                     float* T16) {
  double init7[7], T[16];
  T_to_pose(init_wTo, init7);
  predict_pose(n_mapped, last7, prev7, init7, odom7, pred7);
  pose_to_T(pred7, T);
  for (int k = 0; k < 16; k++) T16[k] = (float)T[k];
}
void orc_map_pose_T(const double* p7, double* wTo, double* oTw) { pose_to_T(p7, wTo); pose_to_Tinv(p7, oTw); }
void orc_map_T_to_pose(const double* T16, double* p7) { T_to_pose(T16, p7); }
void orc_map_ominus(const double* a7, const double* b7, double* out7) { pose_ominus(a7, b7, out7); }
double orc_map_plane_sigma(double d, double mul) { return plane_sigma(d, mul); }
float orc_map_proj(const float* b, const float* e, const float* q) { return point_proj_to_lineseg(b, e, q); }
}
