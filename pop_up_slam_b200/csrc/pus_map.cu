// pus_map.cu -- the plane map (pus_map_* in include/popup_gpu.h): Mapper_mono::processFrame's association, landmark table
// and frame insertion on the device, bound to one solver handle.  The rules are pus_map.cuh's, shared with the host oracle;
// built with --fmad=false so that they round as the reference's float / double arithmetic does.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"
#include "../../include/popup_noise.hpp"
#include "pus_map.cuh"
#include "pus_stages.cuh"

namespace pus {
// what the map reads from its handle (pus_engine.cu)
int engine_sync(pus_handle h);
int engine_device(pus_handle h);
cudaStream_t engine_stream(pus_handle h);
const double* engine_pose_lin(pus_handle h);
const double* engine_plane_lin(pus_handle h);
int engine_node_index(pus_handle h, int id, int kind);
bool engine_node_alive(pus_handle h, int id, int kind);
int engine_iterations(pus_handle h);
int engine_refresh_append(pus_handle h, const void* owner, int pose_node, int n_segs, const float* d_segs, const float* invK,
                          int n_map, const int* fids, const int* rows);
bool engine_refresh_owned(pus_handle h, const void* owner);
void engine_refresh_release(pus_handle h, const void* owner);
cudaError_t launch_project(cudaStream_t st, int n, const int* d_plane_idx, const double* d_plane4, const float* d_in, float* d_out);

namespace map {

constexpr int kAssocThreads = 128;

// bad-input bits of a frame, raised by the kernels that read it
enum Bad { BAD_VALUE = 1, BAD_CSR = 2, BAD_INDICE = 4 };

// The frame's planes as pus_map.cuh's Plane.  Plane i reads row rows[i] (NULL: row i) of planes_sensor / dist / the CSR
// polygons; its plane_indice is inds[i].  Only the values read are checked (finite) and only within the CSR's range.
__global__ void pack_kernel(int n, const int* rows, const int* inds, const float* ps, const float* dist, const int* bptr,
                            const float* b2, const int* wptr, const float* w3, int n_segs, Plane* out, int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rows ? rows[i] : i;
  Plane p;
  p.ind = inds[i];
  p.good = i;
  p.dist = dist[r];
  int flags = 0;
  for (int k = 0; k < 4; k++) flags |= isfinite(ps[4 * (size_t)r + k]) ? 0 : BAD_VALUE;
  plane_local(ps + 4 * (size_t)r, p.local);
  if (!isfinite(p.dist)) flags |= BAD_VALUE;
  if (p.ind < 0 || p.ind > n_segs) flags |= BAD_INDICE;
  for (int k = 0; k < 4; k++) p.v2[k] = 0.f;
  for (int k = 0; k < 6; k++) p.v3[k] = 0.f;
  p.n2 = p.n3 = 0;
  const int b0 = bptr[r], b1 = bptr[r + 1], w0 = wptr[r], w1 = wptr[r + 1];
  const bool b_ok = (rows || bptr[0] == 0) && b0 >= 0 && b0 <= b1 && b1 <= bptr[rows ? r + 1 : n];
  const bool w_ok = (rows || wptr[0] == 0) && w0 >= 0 && w0 <= w1 && w1 <= wptr[rows ? r + 1 : n];
  if (!b_ok || !w_ok) flags |= BAD_CSR;
  if (b_ok) {
    p.n2 = min(b1 - b0, 2);
    for (int k = 0; k < 2 * p.n2; k++) p.v2[k] = b2[2 * (size_t)b0 + k];
  }
  if (w_ok) {
    p.n3 = min(w1 - w0, 2);
    for (int k = 0; k < 3 * p.n3; k++) p.v3[k] = w3[3 * (size_t)w0 + k];
  }
  for (int k = 0; k < 4; k++) flags |= isfinite(p.v2[k]) ? 0 : BAD_VALUE;
  for (int k = 0; k < 6; k++) flags |= isfinite(p.v3[k]) ? 0 : BAD_VALUE;
  out[i] = p;
  if (flags) atomicOr(bad, flags);
}

__global__ void finite_kernel(long long n, const float* v, int* bad) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n && !isfinite(v[i])) atomicOr(bad, BAD_VALUE);
}

// the session form: frame f's good planes -> their rows in the session's packing and their plane_indice
__global__ void gather_kernel(int f, const int* open_ptr, const int* good_ptr, const int* good_rows, int* rows, int* inds) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int g0 = good_ptr[f], n = good_ptr[f + 1] - g0;
  if (k >= n) return;
  inds[k] = good_rows[g0 + k];
  rows[k] = open_ptr[f] + f + good_rows[g0 + k];
}

// est = [est7 | wTo 16 | oTw 16] of processFrame's estimate_pose
__global__ void estimate_kernel(int n_mapped, int last_idx, const double* pose_lin, const double* odom7, double* est) {
  estimate_pose(n_mapped, n_mapped ? pose_lin + 7 * (size_t)last_idx : nullptr, odom7, est);
  pose_to_T(est, est + 7);
  pose_to_Tinv(est, est + 23);
}

// one block per plane: findClosestPlane over every landmark, reduced in a fixed tree (no atomics)
__global__ void __launch_bounds__(kAssocThreads) assoc_kernel(pus_map_config cfg, int seq, int n, const Plane* planes, int L,
                                                                const Landmark* lm, const int* lm_idx, const double* plane_lin,
                                                                const double* est, int* id, double* err) {
  __shared__ Best red[kAssocThreads];
  const int i = blockIdx.x;
  const Plane p = planes[i];
  Best b = best_none();
  if (!is_short(p)) {
    double cw[4];
    plane_transform_T(est + 23, p.local, cw);   // Plane3d::transform_from(oTw)
    for (int c = threadIdx.x; c < L; c += blockDim.x) {
      double e = 0.0;
      const int code = pair(cfg, seq, p, cw, est + 7, lm[c], lm_idx[c] >= 0 ? plane_lin + 4 * (size_t)lm_idx[c] : nullptr, &e);
      if (code == PAIR_GROUND || code == PAIR_MATCH) best_add(b, c, e);
    }
  }
  red[threadIdx.x] = b;
  __syncthreads();
  for (int w = kAssocThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] = best_merge(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) best_result(red[0], id + i, err + i);
}

// the one-to-one rule, in plane order on one thread; res = [assoc n | status n | num_new]
__global__ void one_to_one_kernel(int n, const Plane* planes, const int* id, const double* err, int L, int* res, double* aerr) {
  res[2 * n] = one_to_one(n, planes, id, err, L, res, aerr, res + n);
}

// landmarks [L0, L0 + n_new) are new (nodes[k]); then copy_plane in plane order
__global__ void apply_kernel(int seq, int n, const Plane* planes, const int* assoc, int L0, int n_new, const int* nodes, Landmark* lm) {
  for (int k = 0; k < n_new; k++) new_landmark(lm[L0 + k], nodes[k]);
  for (int i = 0; i < n; i++) copy_plane(lm[assoc[i]], seq, planes[i]);
}

// the landmarks' stored 3-D vertices as point lists for launch_project; a removed landmark's points take a live plane's
// index (fallback) and are not written back.  Also refreshes the deleted flags.
__global__ void lm_points_kernel(int L, Landmark* lm, const int* lm_idx, int fallback, int* pidx, float* pts) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * L) return;
  const int c = t / 2, k = t % 2;
  pidx[t] = lm_idx[c] >= 0 ? lm_idx[c] : fallback;
  for (int j = 0; j < 3; j++) pts[3 * (size_t)t + j] = lm[c].world3d[k][j];
  if (k == 0) lm[c].deleted = lm_idx[c] < 0;
}
__global__ void lm_store_kernel(int L, Landmark* lm, const int* lm_idx, const float* pts) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * L) return;
  const int c = t / 2, k = t % 2;
  if (lm_idx[c] < 0 || k >= lm[c].n_world3d) return;   // reproj_to_newplane: live landmarks, their polygon's vertices
  for (int j = 0; j < 3; j++) lm[c].world3d[k][j] = pts[3 * (size_t)t + j];
}

// main_3d.cpp:366-385: out = [odom7 | pred7], T16 = float(pred.wTo())
__global__ void predict_kernel(int n_mapped, int last_idx, int prev_idx, const double* pose_lin, pus_map_config cfg, double* out,
                               float* T16) {
  double init7[7], T[16];
  T_to_pose(cfg.init_wTo, init7);
  predict_pose(n_mapped, n_mapped ? pose_lin + 7 * (size_t)last_idx : nullptr, n_mapped > 1 ? pose_lin + 7 * (size_t)prev_idx : nullptr,
               init7, out, out + 7);
  pose_to_T(out + 7, T);
  for (int k = 0; k < 16; k++) T16[k] = (float)T[k];
}

// grow-only device buffer
template <class T>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    const size_t c = std::max(n, cap + cap / 2);
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, c * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p) { cudaStreamSynchronize(st); cudaFree(p); }
    p = q;
    cap = c;
    return cudaSuccess;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct Map {
  pus_handle h;
  pus_map_config cfg;
  std::vector<double> pose_sinf, plane_sinf;    // packed sqrt-information of the prior / odometry and the ground prior
  std::vector<int> frame_pose;                  // pose node of every mapped frame
  std::vector<int> lm_node;                     // plane node of every landmark
  double odom[7];                               // the last prediction's odometry
  bool has_odom = false;
  Buf<Landmark> lm;                             // the landmark table (lm_node.size() rows)
  Buf<Landmark> lm_next;                        // (growth)
  Buf<Plane> planes;
  Buf<int> rows, inds, id, res, lm_idx, pidx, nodes, bad;
  Buf<double> err, aerr, est, pred;
  Buf<float> pts, pts_out, T16;
  Buf<float> s_ps, s_dist, s_b2, s_w3, s_segs;   // staged host inputs
  Buf<int> s_pind, s_bptr, s_wptr;
};

const Call kMap{"pus_map"};

bool finite_config(const pus_map_config& c) {
  const double d[] = {c.edge_asso_2ddist, c.edge_asso_proj, c.edge_asso_angle, c.edge_asso_planedist, c.plane_sigma_dist_mul};
  for (double v : d) if (!std::isfinite(v)) return false;
  for (double v : c.pose_sigmas) if (!std::isfinite(v)) return false;
  for (double v : c.plane_sigmas) if (!std::isfinite(v)) return false;
  for (double v : c.init_wTo) if (!std::isfinite(v)) return false;
  for (float v : c.invK) if (!std::isfinite(v)) return false;
  return true;
}
// a sigma the noise model can take: its square and that square's inverse positive and finite
bool good_sigma(double s) {
  const double v = s * s;
  return v > 0 && std::isfinite(v) && 1.0 / v > 0 && std::isfinite(1.0 / v);
}

}  // namespace map
}  // namespace pus

using namespace pus;
using namespace pus::map;

#define MAP_OK(call) PUS_CALL_OK(kMap, call)

extern "C" int pus_map_create(pus_handle h, const pus_map_config* config, pus_map* out) {
  if (!h || !config || !out) return kMap.refuse("handle, config and out must be given");
  const pus_map_config& c = *config;
  if (!finite_config(c)) return kMap.refuse("the config holds a non-finite value");
  for (double s : c.pose_sigmas) if (!good_sigma(s)) return kMap.refuse("pose_sigmas must be positive, with a finite square and inverse square");
  for (double s : c.plane_sigmas) if (!good_sigma(s)) return kMap.refuse("plane_sigmas must be positive, with a finite square and inverse square");
  if (!good_sigma(plane_sigma(3.0, c.plane_sigma_dist_mul)) || !good_sigma(plane_sigma(8.0, c.plane_sigma_dist_mul)) ||
      plane_sigma(3.0, c.plane_sigma_dist_mul) <= 0 || plane_sigma(8.0, c.plane_sigma_dist_mul) <= 0)
    return kMap.refuse("plane_sigma_dist_mul makes a pose-plane sigma non-positive");
  if (c.init_wTo[15] == 0) return kMap.refuse("init_wTo[15] must not be 0");
  Map* m = new Map();
  m->h = h;
  m->cfg = c;
  m->pose_sinf = pus_noise::covariance_diag_packed(c.pose_sigmas, 6);
  m->plane_sinf = pus_noise::covariance_diag_packed(c.plane_sigmas, 3);
  *out = m;
  return 0;
}

extern "C" int pus_map_destroy(pus_map mp) {
  if (!mp) return kMap.refuse("map is NULL");
  Map* m = (Map*)mp;
  cudaSetDevice(engine_device(m->h));
  engine_refresh_release(m->h, m);   // a later map on the handle starts its tables afresh
  for (auto* b : {&m->lm, &m->lm_next}) b->release();
  m->planes.release();
  for (auto* b : {&m->rows, &m->inds, &m->id, &m->res, &m->lm_idx, &m->pidx, &m->nodes, &m->bad, &m->s_pind, &m->s_bptr, &m->s_wptr}) b->release();
  for (auto* b : {&m->err, &m->aerr, &m->est, &m->pred}) b->release();
  for (auto* b : {&m->pts, &m->pts_out, &m->T16, &m->s_ps, &m->s_dist, &m->s_b2, &m->s_w3, &m->s_segs}) b->release();
  delete m;
  return 0;
}

extern "C" int pus_map_predict_pose(pus_map mp, float* T16, double* odom7) {
  if (!mp || !T16) return kMap.refuse("map and T16 must be given");
  Map* m = (Map*)mp;
  const int nf = (int)m->frame_pose.size();
  if (nf > 0 && !engine_node_alive(m->h, m->frame_pose[nf - 1], 0)) return kMap.refuse("the last mapped frame's pose node was removed");
  if (nf > 1 && !engine_node_alive(m->h, m->frame_pose[nf - 2], 0)) return kMap.refuse("the previous mapped frame's pose node was removed");
  if (engine_sync(m->h) < 0) return -1;
  cudaStream_t st = engine_stream(m->h);
  const int last = nf ? engine_node_index(m->h, m->frame_pose[nf - 1], 0) : 0;
  const int prev = nf > 1 ? engine_node_index(m->h, m->frame_pose[nf - 2], 0) : 0;
  MAP_OK(m->pred.ensure(14, st));
  MAP_OK(m->T16.ensure(16, st));
  const bool dev = on_device(T16);
  predict_kernel<<<1, 1, 0, st>>>(nf, last, prev, engine_pose_lin(m->h), m->cfg, m->pred.p, dev ? T16 : m->T16.p);
  MAP_OK(cudaGetLastError());
  double host[14];
  MAP_OK(cudaMemcpyAsync(host, m->pred.p, sizeof(host), cudaMemcpyDeviceToHost, st));
  if (!dev) MAP_OK(cudaMemcpyAsync(T16, m->T16.p, 64, cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaStreamSynchronize(st));
  std::memcpy(m->odom, host, sizeof(m->odom));
  m->has_odom = true;
  if (odom7) std::memcpy(odom7, host, 7 * sizeof(double));
  return 0;
}

// stage host or device input on the device: device pointers are used in place
template <class T>
static cudaError_t stage(Buf<T>& b, const T*& p, size_t n, cudaStream_t st) {
  if (!p || n == 0 || on_device(p)) return cudaSuccess;
  cudaError_t e = b.ensure(n, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(b.p, p, n * sizeof(T), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) p = b.p;
  return e;
}

extern "C" int pus_map_process_frame(pus_map mp, const pus_map_frame* in, pus_map_result* out) {
  if (!mp || !in || !out) return kMap.refuse("map, in and out must be given");
  Map* m = (Map*)mp;
  pus_handle h = m->h;
  const pus_map_config& cfg = m->cfg;
  const int nf = (int)m->frame_pose.size(), L = (int)m->lm_node.size();
  out->n_planes = 0; out->n_new = 0; out->pose_node = -1; out->lm_iterations = 0;
  if (!in->odom7 && !m->has_odom) return kMap.refuse("no odometry: give odom7 or call pus_map_predict_pose first");
  if (in->odom7)
    for (int k = 0; k < 7; k++) if (!std::isfinite(in->odom7[k])) return kMap.refuse("odom7 is not finite");
  if (nf > 0 && !engine_node_alive(h, m->frame_pose[nf - 1], 0)) return kMap.refuse("the last mapped frame's pose node was removed");
  if (nf > 0 && !engine_refresh_owned(h, m)) return kMap.refuse("the handle's refresh tables were rebound (pus_refresh_bind)");
  if (kMap.check_device(engine_device(h)) < 0) return -1;
  if (engine_sync(h) < 0) return -1;
  cudaStream_t st = engine_stream(h);

  // ---- the frame's planes on the device ----
  int n = 0, n_segs = 0;
  const float *ps = nullptr, *dist = nullptr, *b2 = nullptr, *w3 = nullptr, *segs = nullptr;
  const int *pind = nullptr, *bptr = nullptr, *wptr = nullptr, *rows = nullptr;
  if (in->session) {
    pus_popup_frames R;
    if (pus_popup_session_result(in->session, &R) < 0) return -1;
    if (in->frame < 0 || in->frame >= R.n_frames) return kMap.refuse("frame out of the session's range");
    int gp[2], op[2];
    MAP_OK(cudaMemcpy(gp, R.good_ptr + in->frame, 8, cudaMemcpyDeviceToHost));
    MAP_OK(cudaMemcpy(op, R.open_ptr + in->frame, 8, cudaMemcpyDeviceToHost));
    n = gp[1] - gp[0];
    n_segs = op[1] - op[0];
    if (n > 0) {
      MAP_OK(m->rows.ensure(n, st));
      MAP_OK(m->inds.ensure(n, st));
      gather_kernel<<<(n + 127) / 128, 128, 0, st>>>(in->frame, R.open_ptr, R.good_ptr, R.good_rows, m->rows.p, m->inds.p);
      MAP_OK(cudaGetLastError());
    }
    rows = m->rows.p; pind = m->inds.p;
    ps = R.planes_sensor; dist = R.dist; bptr = R.bound_ptr; b2 = R.bound2d; wptr = R.world_ptr; w3 = R.world3d;
    segs = R.open_segs + 4 * (size_t)op[0];
  } else {
    n = in->n_planes; n_segs = in->n_segs;
    if (n < 0 || n_segs < 0) return kMap.refuse("n_planes and n_segs must not be negative");
    if (n > 0 && (!in->planes_sensor || !in->dist || !in->plane_indice || !in->bound_ptr || !in->bound2d || !in->world_ptr || !in->world3d))
      return kMap.refuse("every plane array must be given");
    if (n_segs > 0 && !in->segs) return kMap.refuse("segs must be given");
    ps = in->planes_sensor; dist = in->dist; pind = in->plane_indice; bptr = in->bound_ptr; wptr = in->world_ptr;
    b2 = in->bound2d; w3 = in->world3d; segs = in->segs;
    if (n > 0) {
      int nb = 0, nw = 0;   // the polygons' vertex totals: bound_ptr[n], world_ptr[n]
      if (on_device(bptr)) MAP_OK(cudaMemcpy(&nb, bptr + n, 4, cudaMemcpyDeviceToHost)); else nb = bptr[n];
      if (on_device(wptr)) MAP_OK(cudaMemcpy(&nw, wptr + n, 4, cudaMemcpyDeviceToHost)); else nw = wptr[n];
      if (nb < 0 || nw < 0) return kMap.refuse("malformed bound_ptr / world_ptr");
      MAP_OK(stage(m->s_ps, ps, 4 * (size_t)n, st));
      MAP_OK(stage(m->s_dist, dist, (size_t)n, st));
      MAP_OK(stage(m->s_pind, pind, (size_t)n, st));
      MAP_OK(stage(m->s_bptr, bptr, (size_t)n + 1, st));
      MAP_OK(stage(m->s_wptr, wptr, (size_t)n + 1, st));
      MAP_OK(stage(m->s_b2, b2, 2 * (size_t)nb, st));
      MAP_OK(stage(m->s_w3, w3, 3 * (size_t)nw, st));
    }
    MAP_OK(stage(m->s_segs, segs, 4 * (size_t)n_segs, st));
  }
  if (n == 0) return 0;   // main_3d maps no frame without good planes
  if (out->capacity < n) return kMap.refuse("the result's capacity is smaller than the frame's planes");

  // ---- checks, estimate, association, one-to-one rule ----
  MAP_OK(m->planes.ensure(n, st));
  MAP_OK(m->bad.ensure(1, st));
  MAP_OK(m->id.ensure(n, st));
  MAP_OK(m->err.ensure(n, st));
  MAP_OK(m->aerr.ensure(n, st));
  MAP_OK(m->res.ensure(2 * (size_t)n + 1, st));
  MAP_OK(m->est.ensure(46, st));   // est7 | wTo | oTw | odom7
  MAP_OK(m->lm_idx.ensure(std::max(L, 1), st));
  MAP_OK(cudaMemsetAsync(m->bad.p, 0, 4, st));
  pack_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, rows, pind, ps, dist, bptr, b2, wptr, w3, n_segs, m->planes.p, m->bad.p);
  if (n_segs) finite_kernel<<<(4 * n_segs + 255) / 256, 256, 0, st>>>(4LL * n_segs, segs, m->bad.p);
  std::vector<int> lm_idx(L);
  int fallback = -1;
  for (int c = 0; c < L; c++) {
    lm_idx[c] = engine_node_index(h, m->lm_node[c], 1);
    if (fallback < 0 && lm_idx[c] >= 0) fallback = lm_idx[c];
  }
  if (L) MAP_OK(cudaMemcpyAsync(m->lm_idx.p, lm_idx.data(), 4 * (size_t)L, cudaMemcpyHostToDevice, st));
  const double* odom = in->odom7 ? in->odom7 : m->odom;
  double odom_h[7];
  std::memcpy(odom_h, odom, sizeof(odom_h));
  MAP_OK(cudaMemcpyAsync(m->est.p + 39, odom_h, 56, cudaMemcpyHostToDevice, st));
  estimate_kernel<<<1, 1, 0, st>>>(nf, nf ? engine_node_index(h, m->frame_pose[nf - 1], 0) : 0, engine_pose_lin(h), m->est.p + 39, m->est.p);
  assoc_kernel<<<n, kAssocThreads, 0, st>>>(cfg, in->seq_id, n, m->planes.p, L, m->lm.p, m->lm_idx.p, engine_plane_lin(h), m->est.p,
                                            m->id.p, m->err.p);
  one_to_one_kernel<<<1, 1, 0, st>>>(n, m->planes.p, m->id.p, m->err.p, L, m->res.p, m->aerr.p);
  MAP_OK(cudaGetLastError());
  int bad = 0;
  std::vector<int> res(2 * (size_t)n + 1);
  std::vector<double> aerr(n), est(7);
  std::vector<Plane> planes(n);
  MAP_OK(cudaMemcpyAsync(&bad, m->bad.p, 4, cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaMemcpyAsync(res.data(), m->res.p, 4 * res.size(), cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaMemcpyAsync(aerr.data(), m->aerr.p, 8 * (size_t)n, cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaMemcpyAsync(est.data(), m->est.p, 56, cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaMemcpyAsync(planes.data(), m->planes.p, sizeof(Plane) * (size_t)n, cudaMemcpyDeviceToHost, st));
  MAP_OK(cudaStreamSynchronize(st));
  if (bad & BAD_VALUE) return kMap.refuse("a plane, dist, polygon vertex or segment value is not finite");
  if (bad & BAD_CSR) return kMap.refuse("malformed bound_ptr / world_ptr");
  if (bad & BAD_INDICE) return kMap.refuse("a plane_indice lies outside 0..n_segs");
  int grounds = 0;
  for (const Plane& p : planes) grounds += p.ind == 0;
  if (grounds > 1) return kMap.refuse("more than one ground plane (plane_indice 0)");
  if (n_segs == 0) return kMap.refuse("a frame with planes needs its open segments (n_segs >= 1), as pus_refresh_bind does");
  const int* assoc = res.data();
  const int* status = res.data() + n;
  const int n_new = res[2 * (size_t)n];

  // ---- graph edits (Mapping.cpp:463-530), ids in insertion order ----
  double meas6[6];
  meas6[0] = odom_h[0]; meas6[1] = odom_h[1]; meas6[2] = odom_h[2];
  quat_to_euler(odom_h + 3, meas6[3], meas6[4], meas6[5]);
  // The edits only add to a graph whose ids were all checked above, so none of them is expected to fail; should one fail
  // all the same, the nodes this frame added are removed again (with their factors) and the map stays as it was.
  std::vector<int> added;
  auto undo = [&]() {
    for (int id : added) pus_remove_node(h, id);
    return -1;
  };
  const int pose = pus_add_pose(h, nf ? est.data() : nullptr);
  if (pose < 0) return -1;
  added.push_back(pose);
  if (nf == 0) { if (pus_add_pose_prior(h, pose, meas6, m->pose_sinf.data()) < 0) return undo(); }
  else if (pus_add_odometry(h, m->frame_pose[nf - 1], pose, meas6, m->pose_sinf.data()) < 0) return undo();
  double oTw[16];
  pose_to_Tinv(est.data(), oTw);
  std::vector<int> owner(n_new, -1), nodes(n_new), lm_node = m->lm_node;
  for (int i = 0; i < n; i++) if (assoc[i] >= L) owner[assoc[i] - L] = i;
  for (int k = 0; k < n_new; k++) {
    double init[4];
    plane_transform_T(oTw, planes[owner[k]].local, init);   // measure.transform_from(estimate_pose.oTw())
    nodes[k] = pus_add_plane(h, init);
    if (nodes[k] < 0) return undo();
    added.push_back(nodes[k]);
    lm_node.push_back(nodes[k]);
  }
  std::vector<int> fids(n), rows_h(n);
  for (int i = 0; i < n; i++) {
    const int node = lm_node[assoc[i]];
    if (assoc[i] >= L && planes[i].ind == 0) {
      const double ground[4] = {0, 0, -1, 0};
      if (pus_add_plane_prior(h, node, ground, m->plane_sinf.data()) < 0) return undo();
    }
    const double sg = plane_sigma((double)planes[i].dist, cfg.plane_sigma_dist_mul);
    const double sig3[3] = {sg, sg, sg};
    const std::vector<double> si = pus_noise::covariance_diag_packed(sig3, 3);
    fids[i] = pus_add_pose_plane(h, pose, node, planes[i].local, si.data());
    if (fids[i] < 0) return undo();
    rows_h[i] = planes[i].ind;
  }
  m->lm_node.swap(lm_node);
  m->frame_pose.push_back(pose);

  // ---- copy_plane on the device table ----
  if (L + n_new > (int)m->lm.cap) {
    MAP_OK(m->lm_next.ensure(std::max<size_t>(L + n_new, m->lm.cap + m->lm.cap / 2), st));
    if (L) MAP_OK(cudaMemcpyAsync(m->lm_next.p, m->lm.p, sizeof(Landmark) * (size_t)L, cudaMemcpyDeviceToDevice, st));
    std::swap(m->lm, m->lm_next);
  }
  MAP_OK(m->nodes.ensure(std::max(n_new, 1), st));
  if (n_new) MAP_OK(cudaMemcpyAsync(m->nodes.p, nodes.data(), 4 * (size_t)n_new, cudaMemcpyHostToDevice, st));
  MAP_OK(cudaMemcpyAsync(m->res.p, assoc, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
  apply_kernel<<<1, 1, 0, st>>>(in->seq_id, n, m->planes.p, m->res.p, L, n_new, m->nodes.p, m->lm.p);
  MAP_OK(cudaGetLastError());
  if (engine_refresh_append(h, m, pose, n_segs, segs, cfg.invK, n, fids.data(), rows_h.data()) < 0) return -1;
  MAP_OK(cudaStreamSynchronize(st));   // (the staging vectors go out of scope)

  // ---- results before the solve, so that they are complete when it fails ----
  out->n_planes = n; out->pose_node = pose; out->n_new = n_new;
  for (int i = 0; i < n; i++) {
    if (out->landmark) out->landmark[i] = assoc[i];
    if (out->status) out->status[i] = status[i];
    if (out->factor) out->factor[i] = fids[i];
    if (out->error) out->error[i] = aerr[i];
  }
  if (out->new_nodes) for (int k = 0; k < n_new && k < out->capacity; k++) out->new_nodes[k] = nodes[k];

  // ---- the solve on main_3d's schedule, re-projection, measurement refresh ----
  int iters = 0;
  if (in->seq_id % 5 == 0) { if (pus_batch_optimize(h, &iters) < 0) return -1; }
  else if (pus_update(h) < 0) return -1;
  out->lm_iterations = engine_iterations(h);
  if (engine_sync(h) < 0) return -1;
  const int L1 = L + n_new;
  lm_idx.resize(L1);
  fallback = -1;
  for (int c = 0; c < L1; c++) {
    lm_idx[c] = engine_node_index(h, m->lm_node[c], 1);
    if (fallback < 0 && lm_idx[c] >= 0) fallback = lm_idx[c];
  }
  if (fallback >= 0) {
    MAP_OK(m->lm_idx.ensure(L1, st));
    MAP_OK(m->pidx.ensure(2 * (size_t)L1, st));
    MAP_OK(m->pts.ensure(6 * (size_t)L1, st));
    MAP_OK(m->pts_out.ensure(6 * (size_t)L1, st));
    MAP_OK(cudaMemcpyAsync(m->lm_idx.p, lm_idx.data(), 4 * (size_t)L1, cudaMemcpyHostToDevice, st));
    lm_points_kernel<<<(2 * L1 + 255) / 256, 256, 0, st>>>(L1, m->lm.p, m->lm_idx.p, fallback, m->pidx.p, m->pts.p);
    MAP_OK(launch_project(st, 2 * L1, m->pidx.p, engine_plane_lin(h), m->pts.p, m->pts_out.p));
    lm_store_kernel<<<(2 * L1 + 255) / 256, 256, 0, st>>>(L1, m->lm.p, m->lm_idx.p, m->pts_out.p);
    MAP_OK(cudaGetLastError());
    MAP_OK(cudaStreamSynchronize(st));   // (lm_idx goes out of scope)
  }
  return pus_refresh_run(h, nullptr);
}

extern "C" int pus_map_landmarks(pus_map mp, int capacity, pus_map_landmark* out) {
  if (!mp) return kMap.refuse("map is NULL");
  Map* m = (Map*)mp;
  const int L = (int)m->lm_node.size();
  if (!out) return L;
  if (capacity < L) return kMap.refuse("capacity is smaller than the number of landmarks");
  if (L) {
    cudaStream_t st = engine_stream(m->h);
    MAP_OK(cudaSetDevice(engine_device(m->h)));
    MAP_OK(cudaMemcpyAsync(out, m->lm.p, sizeof(Landmark) * (size_t)L, cudaMemcpyDeviceToHost, st));
    MAP_OK(cudaStreamSynchronize(st));
    for (int c = 0; c < L; c++) out[c].deleted = !engine_node_alive(m->h, m->lm_node[c], 1);
  }
  return L;
}
