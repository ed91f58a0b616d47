// Host-only regression harness for compile_graph(): builds a random graph (loop closures, repeated observations,
// removed factors), compiles it twice into the same object and prints an FNV hash of every array of the device image.
// Use it to prove that a host-side refactor leaves the image bit-identical:
//   g++ -O2 -std=c++17 -DHDR='"<old checkout>/pop_up_slam_b200/csrc/pus_graph.hpp"' -x c++ tools/compile_graph_hash.cpp -o /tmp/h_old
//   g++ -O2 -std=c++17 -DHDR='"pop_up_slam_b200/csrc/pus_graph.hpp"'               -x c++ tools/compile_graph_hash.cpp -o /tmp/h_new
//   for a in "40 6 1" "300 8 2" "2000 12 3" "20000 20 5"; do /tmp/h_old $a; /tmp/h_new $a; done      (args: poses, edges/pose, seed [, force_levels])
// With `--file <graph.txt> [force_levels]` it reads the graph instead, one Graph call per line in insertion order (node ids
// are the running node count), so that generated or dataset graphs can be hashed too:
//   pose - | pose x y z qw qx qy qz          plane - | plane a b c d
//   prior <pose> m[6] sinf[21]   odo <pose> <pose> m[6] sinf[21]   pp <pose> <plane> m[4] sinf[6]   lprior <plane> m[4] sinf[6]
// With `--direct <kind> <order>` in front of either form it hashes the direct solve's host tables instead: build_direct, and
// build_cov for order 1 (or the refusal text of a layout that is refused), so that a refactor of the direct layouts can be
// checked the same way:
//   /tmp/h_old --direct 2 1 2000 12 3;  /tmp/h_new --direct 2 1 --file graph.txt
#include <chrono>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <random>
#include <sstream>
#include HDR
using namespace pus;
static uint64_t H = 1469598103934665603ull;
template <typename T> void hv(const std::vector<T>& v) { const unsigned char* p = (const unsigned char*)v.data(); for (size_t i = 0; i < v.size() * sizeof(T); i++) { H ^= p[i]; H *= 1099511628211ull; } H ^= v.size(); H *= 1099511628211ull; }
void hi(int x) { H ^= (uint64_t)(uint32_t)x; H *= 1099511628211ull; }
// the overflow scratch layout of over-limit pose blocks: hashed when the header has it and a block uses it, so the hash of
// a graph within the limits is the same as from a header that predates it
template <typename C> auto hash_overflow(const C& c, int) -> decltype(c.blk_ovf, void()) {
  if (!c.blk_ovf.empty()) { hv(c.blk_ovf); hi((int)c.n_ovf); hi(c.n_ovf_blk); }
}
template <typename C> void hash_overflow(const C&, long) {}
static uint64_t image_hash(const Compiled& c) {
  H = 1469598103934665603ull;
  for (int x : {c.N, c.M, c.Epl, c.Epf, c.Elp, c.SP, c.nc_pad, c.ntile, c.nslot, c.nblk, c.nc, c.n_upart, c.n_ypart, c.nce, c.ngrp, c.n_hv, c.n_heavy, c.n_huge, c.n_f2, c.ntile_pl}) hi(x);
  hv(c.pose_node); hv(c.plane_node); hv(c.node_idx); hv(c.pose_val); hv(c.plane_val);
  hv(c.pp_fid); hv(c.pp_pose); hv(c.pp_plane); hv(c.pp_ptr); hv(c.pm2pl); hv(c.pm_part); hv(c.ypart_ptr); hv(c.tile_ptr); hv(c.blk_part_ptr); hv(c.grp_of_slot);
  hv(c.pp_meas); hv(c.pp_sinf); hv(c.pp_rays); hv(c.pp_kind);
  hv(c.pl2pm); hv(c.pl_ptr); hv(c.pl_plane); hv(c.pl_pose); hv(c.pl_part); hv(c.upart_ptr); hv(c.pp_end); hv(c.heavy); hv(c.huge);
  hv(c.pf_fid); hv(c.pf_i); hv(c.pf_j); hv(c.pinc_ptr); hv(c.pinc); hv(c.pnbr); hv(c.pf_meas); hv(c.pf_sinf);
  hv(c.lp_fid); hv(c.lp_plane); hv(c.linc_ptr); hv(c.linc); hv(c.lp_meas); hv(c.lp_sinf);
  hv(c.blk_grp_ptr); hv(c.grp_plane); hv(c.grp_mem_ptr); hv(c.grp_mem); hv(c.blk_simple); hv(c.grp_info);
  hv(c.ce_ptr); hv(c.ce_node); hv(c.ce_plane); hv(c.ce_lo); hv(c.ce_hi); hv(c.n2ce_ptr); hv(c.n2ce);
  hv(c.hv_plane); hv(c.lp_ptr); hv(c.lp_cea); hv(c.lp_ceb); hv(c.fp_ptr); hv(c.fp_f);
  // (members added in round 2: resident-loop records, assembly tasks, the level-2 pairs of the three-level preconditioner)
  for (int x : {c.res_nt, c.res_ng, c.res_np, c.n_atask, c.n_asplit, c.levels, c.nc2, c.nce2, c.ng2}) hi(x);
  hv(c.grp_info2); hv(c.at_plane); hv(c.at_lo); hv(c.at_hi); hv(c.at_ptr); hv(c.as_plane);
  hv(c.ce2_ptr); hv(c.ce2_node); hv(c.ce2_plane); hv(c.ce2_lo); hv(c.ce2_hi); hv(c.g2_ptr); hv(c.g2_ce);
  hash_overflow(c, 0);
  return H;
}
// the per-plane incidence pointer of a covariance layout: a CovTables member in older headers, a DirectTables one since
template <typename C, typename D> auto inc_ptr_of(const C& cv, const D&, int) -> decltype((cv.inc_ptr)) { return cv.inc_ptr; }
template <typename C, typename D> auto inc_ptr_of(const C&, const D& d, long) -> decltype((d.inc_ptr)) { return d.inc_ptr; }
static void hll(long long x) { hi((int)(x & 0xffffffff)); hi((int)(x >> 32)); }
// FNV hash of every DirectTables (and, for order 1, CovTables) member; the refusal text instead when a layout is refused
static std::string direct_hash(const Compiled& c, int kind, int order) {
  DirectTables d; CovTables cv; std::string err;
  if (!build_direct(c, d, err, kind, order)) return "refused: " + err;
  H = 1469598103934665603ull;
  for (int x : {d.nb, d.nbp, d.order, d.nlev}) hi(x);
  hll(d.bytes); hll(d.nupd);
  hv(d.inc_pose); hv(d.inc_plane); hv(d.inc_lo); hv(d.inc_hi); hv(d.lp_ptr); hv(d.lp_a); hv(d.lp_b); hv(d.fp_ptr); hv(d.fp_f);
  hv(d.first); hv(d.toff); hv(d.poff); hv(d.col_ptr); hv(d.col_row); hv(d.border); hv(d.binc);
  hv(d.nd_perm); hv(d.nd_pos); hv(d.nd_parent); hv(d.nd_level); hv(d.nd_cptr); hv(d.nd_crow); hv(d.nd_toff); hv(d.nd_lptr);
  hv(d.nd_lcol); hv(d.nd_ltptr); hv(d.nd_trow); hv(d.nd_tcol); hv(d.nd_uptr); hv(d.nd_upd); hv(d.nd_rptr); hv(d.nd_rtile); hv(d.nd_dev);
  char buf[64];
  snprintf(buf, sizeof(buf), "tables=%016llx", (unsigned long long)H);
  std::string out = buf;
  if (order != 1) return out;
  if (!build_cov(c, d, cv, err)) return out + " cov refused: " + err;
  H = 1469598103934665603ull;
  hll((long long)cv.topo); hll(cv.nsel); hll(cv.bytes);
  hv(cv.sel_ptr); hv(cv.sel); hv(inc_ptr_of(cv, d, 0)); hv(cv.pair_ptr); hv(cv.pair); hv(cv.dev);
  snprintf(buf, sizeof(buf), " cov=%016llx", (unsigned long long)H);
  return out + buf;
}
static bool read_graph(const char* path, Graph& g) {
  std::ifstream in(path);
  std::string line, op;
  auto vals = [](std::istringstream& ss, double* v, int n) { for (int i = 0; i < n; i++) if (!(ss >> v[i])) return false; return true; };
  while (std::getline(in, line)) {
    std::istringstream ss(line);
    if (!(ss >> op)) continue;
    double v[27];
    int a = -1, b = -1, r = 0;
    if (op == "pose" || op == "plane") {
      const int n = op == "pose" ? 7 : 4;
      std::string first;
      if (!(ss >> first)) return false;
      const bool init = first != "-";
      if (init) { v[0] = std::stod(first); if (!vals(ss, v + 1, n - 1)) return false; }
      r = g.add_node(op == "pose" ? NODE_POSE : NODE_PLANE, init ? v : nullptr);
    } else if (op == "prior") { if (!(ss >> a) || !vals(ss, v, 27)) return false; r = g.add_pose_prior(a, v, v + 6); }
    else if (op == "odo") { if (!(ss >> a >> b) || !vals(ss, v, 27)) return false; r = g.add_odometry(a, b, v, v + 6); }
    else if (op == "pp") { if (!(ss >> a >> b) || !vals(ss, v, 10)) return false; r = g.add_pose_plane(a, b, v, v + 4); }
    else if (op == "lprior") { if (!(ss >> a) || !vals(ss, v, 10)) return false; r = g.add_plane_prior(a, v, v + 4); }
    else return false;
    if (r < 0) return false;
  }
  return true;
}

int main(int argc, char** argv) {
  int dkind = -1, dorder = 0;
  if (argc > 3 && !strcmp(argv[1], "--direct")) {
    dkind = atoi(argv[2]); dorder = atoi(argv[3]);
    argv += 3; argc -= 3;
  }
  if (argc > 2 && !strcmp(argv[1], "--file")) {
    Graph g;
    if (!read_graph(argv[2], g)) { printf("ok=0 cannot read %s: %s\n", argv[2], g.err.c_str()); return 1; }
    if (argc > 3) g.force_levels = atoi(argv[3]);
    Compiled c; std::string err;
    bool ok = compile_graph(g, c, err);
    const uint64_t h1 = ok ? image_hash(c) : 0;
    ok = compile_graph(g, c, err) && ok && image_hash(c) == h1;
    if (ok && dkind >= 0) {
      printf("file=%s direct kind=%d order=%d N=%d %s\n", argv[2], dkind, dorder, c.N, direct_hash(c, dkind, dorder).c_str());
      return 0;
    }
    printf("file=%s ok=%d E=%d hash=%016llx %s\n", argv[2], ok, c.Epl, (unsigned long long)H, err.c_str());
    return ok ? 0 : 1;
  }
  int N = atoi(argv[1]), per = atoi(argv[2]), seed = atoi(argv[3]);
  int M = std::max(3, N / 10);
  Graph g; std::mt19937 rng(seed);
  auto U = [&](double a, double b) { return std::uniform_real_distribution<double>(a, b)(rng); };
  double s21[21], s6[6] = {1, 0.1, 0, 2, 0, 1};
  int q = 0; for (int r = 0; r < 6; r++) for (int c = r; c < 6; c++) s21[q++] = r == c ? 1.0 + r : 0.0;
  std::vector<int> poses, planes;
  for (int i = 0; i < N; i++) {
    double p7[7] = {U(-5, 5), U(-5, 5), U(0.5, 2), 1, 0, 0, 0};
    poses.push_back(g.add_node(NODE_POSE, i == 0 ? p7 : nullptr));
    double m6[6] = {U(-1, 1), U(-1, 1), 0, U(-.2, .2), 0, 0};
    if (i == 0) g.add_pose_prior(poses[0], m6, s21); else g.add_odometry(poses[i - 1], poses[i], m6, s21);
    if (i > 20 && (rng() % 7) == 0) g.add_odometry(poses[rng() % (i - 10)], poses[i], m6, s21);   // loop closures
    int k = 1 + rng() % per;
    for (int j = 0; j < k; j++) {
      int l = (rng() % 3 == 0) ? 0 : (int)(rng() % M);
      while ((int)planes.size() <= l) { planes.push_back(g.add_node(NODE_PLANE, nullptr)); }
      double m4[4] = {U(-1, 1), U(-1, 1), U(-1, 1), U(-3, 3)};
      int f = g.add_pose_plane(poses[i], planes[l], m4, s6);
      if (rng() % 50 == 0) g.add_pose_plane(poses[i], planes[l], m4, s6);   // duplicate observation
      if (f > 0 && rng() % 97 == 0) g.remove_factor(f);
    }
  }
  if (!planes.empty()) { double m4[4] = {0, 0, 1, 0}; g.add_plane_prior(planes[0], m4, s6); }
  if (argc > 4) g.force_levels = atoi(argv[4]);
  Compiled c; std::string err;
  auto t0 = std::chrono::steady_clock::now();
  bool ok = compile_graph(g, c, err);
  double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  const uint64_t h1 = ok ? image_hash(c) : 0;
  auto t1 = std::chrono::steady_clock::now();
  ok = compile_graph(g, c, err) && ok;   // a second compile into the same object must give the same image
  const double ms2 = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
  const uint64_t h2 = image_hash(c);
  ok = ok && (h1 == h2);   // the re-compile into the same object gives the same image
  if (ok && dkind >= 0) {
    printf("N=%d per=%d seed=%d direct kind=%d order=%d %s\n", N, per, seed, dkind, dorder, direct_hash(c, dkind, dorder).c_str());
    return 0;
  }
  H = h2;
  printf("N=%d per=%d seed=%d ok=%d E=%d hash=%016llx  (%.2f ms, again %.2f ms) %s\n", N, per, seed, ok, c.Epl, (unsigned long long)H, ms, ms2, err.c_str());
}
