// popup_frames_oracle.cpp -- the CPU oracle of the pop-up session (pus_popup_session_run): main_3d's per-frame chain through
// the stage oracles (orc_popup_lines, orc_popup_edges, orc_popup_fit_frames, orc_popup_polygons, orc_popup_clouds,
// orc_popup_depth), linked in from their own libraries, with the glue between them taken from the session's shared header
// pus_frames.cuh compiled for the host.  orc_popup_frames_run runs a batch; orc_popup_frames_result fills a
// pus_popup_frames with host pointers into the last run's outputs.  Test infrastructure only.
#include <cstring>
#include <string>
#include <vector>

#include "../pop_up_slam_b200/csrc/pus_frames.cuh"

extern "C" {
long long orc_popup_lines(int, int, const unsigned char*, int, int, int, int, int*, int*, float*, long long);
int orc_popup_edges(int, int, const unsigned char*, int, int, const int*, const float*, const pus_edge_params*, int*, int*,
                    int*, float*, float*, int*, long long, long long);
int orc_popup_fit_frames(int, int, const int*, const float*, const float*, const float*, float, int, float*, float*, float*,
                         int*);
int orc_popup_polygons(int, int, const int*, const float*, const float*, const float*, const float*, int, int, float, float,
                       int*, int*, int*, float*, float*, float*, long long, long long, long long);
long long orc_popup_clouds(int, int, const int*, const int*, const float*, const float*, const float*, const float*,
                           const unsigned char*, int, int, int, float, float, int*, long long*, float*, unsigned char*,
                           long long, unsigned char*);
int orc_popup_depth(int, int, const int*, const int*, const float*, const float*, const float*, const float*, int, int, int,
                    float, float*);
}

namespace {
std::string g_err;

struct Run {
  int n = 0, n_rows = 0, n_good = 0;
  std::vector<int> status, line_status, line_counts, edge_status, open_ptr, connect_ptr, inc, good, bound_ptr, cut_ptr,
      world_ptr, good_ptr, good_rows, plane_status, cloud_counts;
  std::vector<float> open, conn, pw, ps, dist, bound, cut, world, xyz, depth;
  std::vector<long long> cloud_offsets;
  std::vector<unsigned char> rgb, labels;
  bool rgb_on = false, labels_on = false, depth_on = false;
} R;

template <class T>
T* data(std::vector<T>& v) { return v.empty() ? nullptr : v.data(); }

int fail(const char* who) {
  g_err = std::string("orc_popup_frames_run: ") + who + " failed";
  R = Run{};
  return -1;
}

std::vector<int> offsets(const std::vector<int>& counts) {
  std::vector<int> p(counts.size() + 1, 0);
  for (size_t i = 0; i < counts.size(); i++) p[i + 1] = p[i] + counts[i];
  return p;
}
}  // namespace

extern "C" {
const char* orc_popup_frames_last_error(void) { return g_err.c_str(); }

int orc_popup_frames_run(const pus_popup_config* c, int n, const unsigned char* images, const unsigned char* labels,
                         const float* Ts) {
  using namespace pus::glue;
  R = Run{};
  if (!c || n < 0 || (n > 0 && (!images || !labels || !Ts))) { g_err = "orc_popup_frames_run: bad arguments"; return -1; }
  const int W = c->width, H = c->height;
  R.n = n;
  // 1. lines
  R.line_status.assign(n, 0);
  R.line_counts.assign(n, 0);
  long long nl = orc_popup_lines(0, n, images, W, H, c->channels, c->fast_edges, R.line_status.data(), R.line_counts.data(),
                                 nullptr, 0);
  if (nl < 0) return fail("lines");
  std::vector<float> lines(4 * (size_t)nl + 4);
  if (orc_popup_lines(0, n, images, W, H, c->channels, c->fast_edges, R.line_status.data(), R.line_counts.data(),
                      lines.data(), nl) < 0)
    return fail("lines");
  const std::vector<int> lptr = offsets(R.line_counts);
  // 2. edges, on the lines of the frames whose lines they take
  R.status.assign(n, 0);
  std::vector<int> ecnt(n, 0);
  std::vector<float> elines;
  for (int f = 0; f < n; f++) {
    R.status[f] = lines_status(lines.data() + 4 * (size_t)lptr[f], R.line_counts[f]);
    if (R.status[f]) continue;
    ecnt[f] = R.line_counts[f];
    elines.insert(elines.end(), lines.begin() + 4 * (size_t)lptr[f], lines.begin() + 4 * (size_t)lptr[f + 1]);
  }
  const std::vector<int> eptr = offsets(ecnt);
  std::vector<int> est(n), oc(n), cc(n);
  if (orc_popup_edges(0, n, labels, W, H, eptr.data(), data(elines), &c->edges, est.data(), oc.data(), cc.data(), nullptr,
                      nullptr, nullptr, 0, 0) < 0)
    return fail("edges");
  const std::vector<int> op = offsets(oc), cp = offsets(cc);
  std::vector<float> eo(4 * (size_t)op[n] + 4), ec(4 * (size_t)cp[n] + 4);
  std::vector<int> ei((size_t)op[n] + 1);
  if (orc_popup_edges(0, n, labels, W, H, eptr.data(), data(elines), &c->edges, est.data(), oc.data(), cc.data(), eo.data(),
                      ec.data(), ei.data(), op[n], cp[n]) < 0)
    return fail("edges");
  R.edge_status.assign(n, 0);
  std::vector<int> koc(n, 0), kcc(n, 0);
  for (int f = 0; f < n; f++) {
    R.edge_status[f] = R.status[f] == 1 ? -1 : est[f];
    R.status[f] = edges_status(R.status[f], oc[f]);
    if (R.status[f]) continue;
    koc[f] = oc[f];
    kcc[f] = cc[f];
    R.open.insert(R.open.end(), eo.begin() + 4 * (size_t)op[f], eo.begin() + 4 * (size_t)op[f + 1]);
    R.conn.insert(R.conn.end(), ec.begin() + 4 * (size_t)cp[f], ec.begin() + 4 * (size_t)cp[f + 1]);
    R.inc.insert(R.inc.end(), ei.begin() + op[f], ei.begin() + op[f + 1]);
  }
  R.open_ptr = offsets(koc);
  R.connect_ptr = offsets(kcc);
  // 3. fit on the open segments, 4. the actual-index filter
  const int rows = R.open_ptr[n] + n;
  R.n_rows = rows;
  R.pw.assign(4 * (size_t)rows, 0.f);
  R.ps.assign(4 * (size_t)rows, 0.f);
  R.dist.assign(rows, 0.f);
  R.good.assign(rows, 0);
  if (n > 0 && orc_popup_fit_frames(0, n, R.open_ptr.data(), data(R.open), c->invK, Ts, c->plane_cam_dist_thre, 0, R.pw.data(),
                                    R.ps.data(), R.dist.data(), R.good.data()) < 0)
    return fail("fit");
  std::vector<int> n_good(n, 0);
  for (int f = 0; f < n; f++) {
    const int o0 = R.open_ptr[f], no = R.open_ptr[f + 1] - o0;
    n_good[f] = no > 0 ? actual_filter(data(R.inc) + o0, no, R.good.data() + o0 + f) : 0;
  }
  R.good_ptr = offsets(n_good);
  // 5. polygons on the open segments
  std::vector<int> nb(rows), ncut(rows), nw(rows);
  if (orc_popup_polygons(0, n, R.open_ptr.data(), data(R.open), c->K, c->invK, Ts, W, H, c->ceiling_threshold,
                         c->walllength_threshold, nb.data(), ncut.data(), nw.data(), nullptr, nullptr, nullptr, 0, 0, 0) < 0)
    return fail("polygons");
  R.bound_ptr = offsets(nb);
  R.cut_ptr = offsets(ncut);
  R.world_ptr = offsets(nw);
  R.bound.assign(2 * (size_t)R.bound_ptr[rows], 0.f);
  R.cut.assign(2 * (size_t)R.cut_ptr[rows], 0.f);
  R.world.assign(3 * (size_t)R.world_ptr[rows], 0.f);
  if (orc_popup_polygons(0, n, R.open_ptr.data(), data(R.open), c->K, c->invK, Ts, W, H, c->ceiling_threshold,
                         c->walllength_threshold, nb.data(), ncut.data(), nw.data(), data(R.bound), data(R.cut),
                         data(R.world), R.bound_ptr[rows], R.cut_ptr[rows], R.world_ptr[rows]) < 0)
    return fail("polygons");
  // 6. / 7. the good rows' planes and polygons; a polygon the clouds or the depth map cannot take is passed empty
  const bool from_cut = c->walllength_threshold > 0;
  std::vector<float> planes, cpoly, dpoly;
  std::vector<int> cptr{0}, dptr{0};
  for (int f = 0; f < n; f++) {
    const int r0 = R.open_ptr[f] + f;
    if (n_good[f] == 0) continue;
    for (int j = 0; j <= R.open_ptr[f + 1] - R.open_ptr[f]; j++) {
      const int r = r0 + j;
      if (!R.good[r]) continue;
      R.good_rows.push_back(j);
      planes.insert(planes.end(), R.ps.begin() + 4 * (size_t)r, R.ps.begin() + 4 * (size_t)r + 4);
      int st = 0;
      for (int k = 0; k < 2; k++) {
        const bool cut = k == 0 && from_cut;
        const std::vector<int>& p = cut ? R.cut_ptr : R.bound_ptr;
        const float* q = (cut ? R.cut.data() : R.bound.data()) + 2 * (size_t)p[r];
        const int m = p[r + 1] - p[r];
        std::vector<float>& out = k == 0 ? cpoly : dpoly;
        if (polygon_ok(q, m)) out.insert(out.end(), q, q + 2 * m);
        else st |= 1 << k;
        (k == 0 ? cptr : dptr).push_back((int)out.size() / 2);
      }
      R.plane_status.push_back(st);
    }
  }
  R.n_good = R.good_ptr[n];
  R.cloud_counts.assign(R.n_good, 0);
  R.cloud_offsets.assign(R.n_good, 0);
  R.rgb_on = c->want_rgb;
  R.labels_on = c->want_labels;
  R.depth_on = c->want_depth;
  const unsigned char* bgr = c->channels == 3 ? images : nullptr;   // the clouds take BGR images only
  if (c->want_labels) R.labels.assign((size_t)n * W * H, 0);
  const long long np = orc_popup_clouds(0, n, R.good_ptr.data(), cptr.data(), data(cpoly), data(planes), Ts, c->invK, bgr, W, H,
                                        c->downsample_poly, c->depth_thre, c->ceiling_threshold, data(R.cloud_counts),
                                        data(R.cloud_offsets), nullptr, nullptr, 0, nullptr);
  if (np < 0) return fail("clouds");
  R.xyz.assign(3 * (size_t)np, 0.f);
  R.rgb.assign(3 * (size_t)np, 0);
  if (orc_popup_clouds(0, n, R.good_ptr.data(), cptr.data(), data(cpoly), data(planes), Ts, c->invK, bgr, W, H,
                       c->downsample_poly, c->depth_thre, c->ceiling_threshold, data(R.cloud_counts), data(R.cloud_offsets),
                       data(R.xyz), data(R.rgb), np, c->want_labels ? data(R.labels) : nullptr) < 0)
    return fail("clouds");
  if (c->want_depth) {
    R.depth.assign((size_t)n * W * H, 0.f);
    if (n > 0 && orc_popup_depth(0, n, R.good_ptr.data(), dptr.data(), data(dpoly), data(planes), Ts, c->invK, W, H,
                                 c->downsample_poly, c->ceiling_threshold, R.depth.data()) < 0)
      return fail("depth");
  }
  return 0;
}

int orc_popup_frames_result(pus_popup_frames* o) {
  if (!o) return -1;
  *o = pus_popup_frames{};
  o->n_frames = R.n;
  o->n_rows = R.n_rows;
  o->n_good = R.n_good;
  o->n_open = R.open_ptr.empty() ? 0 : R.open_ptr.back();
  o->n_connect = R.connect_ptr.empty() ? 0 : R.connect_ptr.back();
  o->n_bound = R.bound.size() / 2;
  o->n_cut = R.cut.size() / 2;
  o->n_world = R.world.size() / 3;
  o->n_points = R.xyz.size() / 3;
  o->status = data(R.status); o->line_status = data(R.line_status); o->line_counts = data(R.line_counts);
  o->edge_status = data(R.edge_status); o->open_ptr = data(R.open_ptr); o->connect_ptr = data(R.connect_ptr);
  o->open_segs = data(R.open); o->connect_segs = data(R.conn); o->open_in_connect = data(R.inc);
  o->planes_world = data(R.pw); o->planes_sensor = data(R.ps); o->dist = data(R.dist); o->good = data(R.good);
  o->bound_ptr = data(R.bound_ptr); o->cut_ptr = data(R.cut_ptr); o->world_ptr = data(R.world_ptr);
  o->bound2d = data(R.bound); o->cut2d = data(R.cut); o->world3d = data(R.world);
  o->good_ptr = data(R.good_ptr); o->good_rows = data(R.good_rows); o->plane_status = data(R.plane_status);
  o->cloud_counts = data(R.cloud_counts); o->cloud_offsets = data(R.cloud_offsets); o->xyz = data(R.xyz);
  o->rgb = R.rgb_on ? data(R.rgb) : nullptr;
  o->labels = R.labels_on ? data(R.labels) : nullptr;
  o->depth = R.depth_on ? data(R.depth) : nullptr;
  return 0;
}
}
