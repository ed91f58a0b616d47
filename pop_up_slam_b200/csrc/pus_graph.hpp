// pus_graph.hpp -- host side of the drop-in boundary: the factor-graph container that mirrors
// isam::Slam's graph bookkeeping, and the "compiler" that flattens it into the HBM layout the
// CUDA kernels sweep.  Pure C++ (no CUDA), so it is unit-tested on the CPU.
//
// Reference semantics reproduced (paths relative to the reference checkout;
// ISAM = pop_planar_slam/Thirdparty/isam, PPS = pop_planar_slam):
//   insertion-ordered ids / lists ...... ISAM/isamlib/Slam.cpp:47-48,91-126, ISAM/include/isam/Graph.h:40-133
//   column / row offsets ................ Slam::update_starts Slam.cpp:59-67, jacobian_partial Slam.cpp:395-432
//   factor initialisation of nodes ...... slam3d.h:75-80,123-137 ; PPS/src/isam_plane3d.h:252-264,443-448
//   measurement update .................. ISAM/include/isam/Factor.h:203-206
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "pus_math.cuh"

namespace pus {

enum NodeKind { NODE_POSE = 0, NODE_PLANE = 1 };
enum FactorKind { F_POSE_PRIOR = 0, F_ODOMETRY = 1, F_POSE_PLANE = 2, F_PLANE_PRIOR = 3 };

constexpr int kBlockPoses = 16;            // poses per dense preconditioner block
constexpr int kBlockDim = 6 * kBlockPoses; // 96
// Three-level additive preconditioner of the reduced pose system (DESIGN.md section 5):
//   level 1  exact inverses of the 16-pose diagonal blocks of S
//   level 2  piecewise-linear ("hat") trajectory modes with one node every kL2Spacing poses, solved by block-Jacobi in
//            groups of kGroupNodes nodes (96 x 96 blocks of P2^T S P2, same size as the level-1 blocks)
//   level 3  hat modes with one node every kCoarseSpacing poses, Galerkin operator inverted densely (<= 1920^2)
// Graphs of up to kL2Spacing * kMaxCoarseNodes = 5120 poses use two levels (1 + an exactly inverted hat level with a node
// every 16 poses: fewest PCG iterations, dense A_c^-1 <= 1920^2); larger graphs use all three, so the hat level with the
// fine spacing never has to be inverted (or applied) as a dense matrix and the iteration count stays flat in N.
constexpr int kL2Spacing = 16;             // = kBlockPoses: every pose block is exactly one level-2 interval
constexpr int kGroupNodes = 16;            // level-2 nodes per block-Jacobi group (6 * 16 = kBlockDim)
constexpr int kCoarseSpacing = 128;        // base spacing (poses) of the level-3 nodes; multiple of kBlockPoses
constexpr int kMaxCoarseNodes = 320;       // the level-3 spacing grows in steps of 128 so that the dense A_c stays <= 1920^2
constexpr int kHeavyCoarse = 16;           // planes touching more coarse nodes than this are dense rank-3 updates of A_c
constexpr int kPivotNodes = 8;             // coarse nodes per pivot block of the blocked Gauss-Jordan inversion (48 scalars)
constexpr int kTile = 32;                  // edges per warp tile
constexpr int kWStride = 18 * kTile;       // doubles per W tile
constexpr int kMaxGrp = 256;               // plane groups per 16-pose block held in shared memory (more: global overflow scratch)
constexpr int kMaxPart = 64;               // (tile, pose) partial sums per block held in shared memory (more: global overflow scratch)
constexpr int kAsmChunk = 128;             // plane-major edge slots per Hll / gl assembly task (one warp)

struct HNode {
  int kind = NODE_POSE;
  bool alive = true;
  bool initialized = false;
  double v[7] = {0, 0, 0, 1, 0, 0, 0};  // pose: x y z qw qx qy qz ; plane: a b c d
};

struct HFactor {
  int kind = F_POSE_PLANE;
  bool alive = true;
  int nodes[2] = {-1, -1};
  int n_nodes = 1;
  int dim = 3;
  double meas[6] = {0, 0, 0, 0, 0, 0};
  double sinf[21];  // packed upper-triangular
  bool has_rays = false;   // Pose3d_Plane3d_Factor2: the measured plane is re-popped from two ground-edge rays (sensor frame)
  double rays[6] = {0, 0, 0, 0, 0, 0};
};

struct Graph {
  std::vector<HNode> nodes;
  std::vector<HFactor> factors;
  std::string err;
  uint64_t topo_version = 1;  // bumped on any structural edit (node/factor add/remove)
  int force_levels = 0;       // 0: two or three preconditioner levels by graph size; 2 / 3: forced (tests, studies)

  bool ok_node(int id, int kind) const { return id >= 0 && id < (int)nodes.size() && nodes[id].alive && nodes[id].kind == kind; }
  bool ok_factor(int f) const { return f >= 0 && f < (int)factors.size() && factors[f].alive; }

  int add_node(int kind, const double* v) {
    HNode n;
    n.kind = kind;
    if (v) {
      if (kind == NODE_POSE) std::memcpy(n.v, v, 7 * sizeof(double));
      else { std::memcpy(n.v, v, 4 * sizeof(double)); normalize4(n.v); }
      n.initialized = true;
    } else if (kind == NODE_PLANE) { n.v[0] = 1; n.v[1] = n.v[2] = n.v[3] = 0; }
    nodes.push_back(n);
    topo_version++;
    return (int)nodes.size() - 1;
  }
  void init_node(int id, const double* v) {
    HNode& n = nodes[id];
    if (n.kind == NODE_POSE) std::memcpy(n.v, v, 7 * sizeof(double));
    else { std::memcpy(n.v, v, 4 * sizeof(double)); normalize4(n.v); }
    n.initialized = true;
  }

  int push_factor(HFactor& f) { factors.push_back(f); topo_version++; return (int)factors.size() - 1; }

  int add_pose_prior(int pose, const double* m, const double* si) {
    if (!ok_node(pose, NODE_POSE)) { err = "add_pose_prior: bad pose id"; return -1; }
    HFactor f; f.kind = F_POSE_PRIOR; f.n_nodes = 1; f.nodes[0] = pose; f.dim = 6;
    std::memcpy(f.meas, m, 6 * sizeof(double)); std::memcpy(f.sinf, si, 21 * sizeof(double));
    if (!nodes[pose].initialized) { double p[7]; pose_from_xyzypr(m, p); init_node(pose, p); }  // slam3d.h:75-80
    return push_factor(f);
  }
  int add_odometry(int a, int b, const double* m, const double* si) {
    if (!ok_node(a, NODE_POSE) || !ok_node(b, NODE_POSE)) { err = "add_odometry: bad pose id"; return -1; }
    if (!nodes[a].initialized && !nodes[b].initialized) {
      err = "slam3d: Pose3d_Pose3d_Factor requires pose1 or pose2 to be initialized";  // slam3d.h:124-125
      return -1;
    }
    HFactor f; f.kind = F_ODOMETRY; f.n_nodes = 2; f.nodes[0] = a; f.nodes[1] = b; f.dim = 6;
    std::memcpy(f.meas, m, 6 * sizeof(double)); std::memcpy(f.sinf, si, 21 * sizeof(double));
    double mp[7]; pose_from_xyzypr(m, mp);
    if (!nodes[a].initialized) {            // slam3d.h:127-132: p2.oplus(z.ominus(measure))
      double z[7] = {0, 0, 0, 1, 0, 0, 0}, inv[7], out[7];
      pose_ominus(z, mp, inv); pose_oplus(nodes[b].v, inv, out); init_node(a, out);
    } else if (!nodes[b].initialized) {     // slam3d.h:133-137: p1.oplus(measure)
      double out[7]; pose_oplus(nodes[a].v, mp, out); init_node(b, out);
    }
    return push_factor(f);
  }
  int add_pose_plane(int pose, int plane, const double* m, const double* si) {
    if (!ok_node(pose, NODE_POSE) || !ok_node(plane, NODE_PLANE)) { err = "add_pose_plane: bad node id"; return -1; }
    if (!nodes[pose].initialized) { err = "Plane3d: Pose3d_Plane3d_Factor requires pose to be initialized"; return -1; }
    HFactor f; f.kind = F_POSE_PLANE; f.n_nodes = 2; f.nodes[0] = pose; f.nodes[1] = plane; f.dim = 3;
    std::memcpy(f.meas, m, 4 * sizeof(double)); normalize4(f.meas);
    std::memcpy(f.sinf, si, 6 * sizeof(double));
    if (!nodes[plane].initialized) {        // isam_plane3d.h:256-262: measure.transform_from(p.oTw())
      double T[16], g[4]; pose_to_Tinv(nodes[pose].v, T); plane_transform_T(T, f.meas, g); init_node(plane, g);
    }
    return push_factor(f);
  }
  // Pose3d_Plane3d_Factor2 (isam_plane3d.h:314-424): same nodes / initialisation, plus the precomputed rays (:358-370)
  int add_pose_plane2(int pose, int plane, const double* m, const double* rays6, const double* si) {
    const int f = add_pose_plane(pose, plane, m, si);
    if (f < 0) return f;
    factors[f].has_rays = true;
    std::memcpy(factors[f].rays, rays6, 6 * sizeof(double));
    return f;
  }
  int add_plane_prior(int plane, const double* m, const double* si) {
    if (!ok_node(plane, NODE_PLANE)) { err = "add_plane_prior: bad plane id"; return -1; }
    HFactor f; f.kind = F_PLANE_PRIOR; f.n_nodes = 1; f.nodes[0] = plane; f.dim = 3;
    std::memcpy(f.meas, m, 4 * sizeof(double)); normalize4(f.meas);
    std::memcpy(f.sinf, si, 6 * sizeof(double));
    if (!nodes[plane].initialized) init_node(plane, f.meas);  // isam_plane3d.h:443-448
    return push_factor(f);
  }
  void remove_factor(int f) { factors[f].alive = false; topo_version++; }
  void remove_node(int id) {  // Slam::remove_node Slam.cpp:107-115: adjacent factors go too
    for (auto& f : factors) {
      if (!f.alive) continue;
      for (int k = 0; k < f.n_nodes; k++) if (f.nodes[k] == id) { f.alive = false; break; }
    }
    nodes[id].alive = false;
    topo_version++;
  }
  int num_nodes() const { int c = 0; for (auto& n : nodes) c += n.alive; return c; }
  int num_factors() const { int c = 0; for (auto& f : factors) c += f.alive; return c; }
  int node_start(int id) const {
    if (id < 0 || id >= (int)nodes.size() || !nodes[id].alive) return -1;
    int s = 0;
    for (int i = 0; i < id; i++) if (nodes[i].alive) s += nodes[i].kind == NODE_POSE ? 6 : 3;
    return s;
  }
  int factor_row(int fid) const {
    if (!ok_factor(fid)) return -1;
    int r = 0;
    for (int i = 0; i < fid; i++) if (factors[i].alive) r += factors[i].dim;
    return r;
  }
};

// ------------------------------------------------------------------------------------------------
// Flattened problem (host copy of what goes to HBM).  All index arrays are int32.
// ------------------------------------------------------------------------------------------------
struct Compiled {
  int N = 0, M = 0, Epl = 0, Epf = 0, Elp = 0;
  int SP = kCoarseSpacing;
  int nc_pad = 0;  // nc rounded up to whole pivot blocks; the padding nodes carry identity blocks
  int ntile = 0, nslot = 0, nblk = 0, nc = 0, n_upart = 0, n_ypart = 0, nce = 0, ngrp = 0, n_hv = 0, n_heavy = 0, n_huge = 0;
  std::vector<int> pose_node, plane_node;   // idx -> node id
  std::vector<int> node_idx;                // node id -> idx (pose idx or plane idx), -1 dead
  std::vector<double> pose_val, plane_val;  // [N*7], [M*4]
  // pose-plane edges, pose-major
  // (slot-indexed: every 16-pose block's edges are padded to whole 32-edge tiles; pad slots have pp_pose = -1)
  std::vector<int> pp_fid, pp_pose, pp_plane, pp_ptr, pm2pl, pm_part, ypart_ptr, tile_ptr, blk_part_ptr, grp_of_slot;
  std::vector<double> pp_meas, pp_sinf, pp_rays;   // pp_rays: [slots][6] when any edge is a Factor2 (else one dummy entry)
  std::vector<int> pp_kind;                        // 1 = Factor2 (uses pp_rays), else 0
  int n_f2 = 0;
  // plane-major view
  std::vector<int> pl2pm, pl_ptr, pl_plane, pl_pose, pl_part, upart_ptr, pp_end, heavy, huge;
  int ntile_pl = 0;
  // pose factors (prior / odometry)
  std::vector<int> pf_fid, pf_i, pf_j, pinc_ptr, pinc, pnbr;
  std::vector<double> pf_meas, pf_sinf;
  // plane priors
  std::vector<int> lp_fid, lp_plane, linc_ptr, linc;
  std::vector<double> lp_meas, lp_sinf;
  // dense-block groups: per pose block, its edges grouped by plane
  std::vector<int> blk_grp_ptr, grp_plane, grp_mem_ptr, grp_mem, blk_simple, grp_info;
  // block-resident PCG (small / medium graphs): the plane exchange is per (pose block, plane) instead of per plane-major tile
  // run -- grp_info2 = {plane, first slot of the plane's per-block partial sums, their number, this group's own slot};
  // res_* = largest tile / group / (tile, pose)-run count of any pose block (uniform shared-memory strides)
  std::vector<int> grp_info2;
  int res_nt = 0, res_ng = 0, res_np = 0;
  // fused PCG pose phase, blocks over kMaxGrp plane groups or kMaxPart (tile, pose) runs: per block the offset (doubles) of its
  // group vectors [ng][3] and run sums [npart][6] in the global overflow scratch, -1 for a block that keeps them in shared
  // memory.  Empty when no block is over a limit (n_ovf = total doubles of the scratch, n_ovf_blk = blocks over a limit).
  std::vector<int> blk_ovf;
  size_t n_ovf = 0;
  int n_ovf_blk = 0;
  // Hll / gl assembly tasks: the plane-major slots of every plane cut into chunks of kAsmChunk (a plane seen from thousands of
  // poses is gathered by many warps instead of one); at_* per task, at_ptr per plane, as_plane = planes with more than one task
  std::vector<int> at_plane, at_lo, at_hi, at_ptr, as_plane;
  int n_atask = 0, n_asplit = 0;
  // coarse (hat) space: (plane, coarse node) pairs
  std::vector<int> ce_ptr, ce_node, ce_plane, ce_lo, ce_hi, n2ce_ptr, n2ce;
  std::vector<int> hv_plane, lp_ptr, lp_cea, lp_ceb, fp_ptr, fp_f;   // coarse assembly: heavy planes, per node-pair lists
  // level 2: (plane, node) pairs at spacing kL2Spacing, and per block-Jacobi group its pairs sorted by (plane, node)
  int levels = 2;   // preconditioner levels in use (2: SP = 16 k hats inverted exactly; 3: level-2 block-Jacobi + level 3 at SP = 256 k)
  int nc2 = 0, nce2 = 0, ng2 = 0;
  std::vector<int> ce2_ptr, ce2_node, ce2_plane, ce2_lo, ce2_hi, g2_ptr, g2_ce;
};

inline int coarse_spacing(int N, int levels) {
  const int base = (levels == 3) ? kCoarseSpacing : kL2Spacing;
  return base * std::max(1, (N + base * kMaxCoarseNodes - 1) / (base * kMaxCoarseNodes));
}
inline int coarse_nodes(int N, int sp) { return N <= 1 ? 1 : (N - 1 + sp - 1) / sp + 1; }

inline bool compile_graph(const Graph& g, Compiled& c, std::string& err) {
  c = Compiled();
  const int nn = (int)g.nodes.size();
  c.node_idx.assign(nn, -1);
  for (int i = 0; i < nn; i++) {
    const HNode& n = g.nodes[i];
    if (!n.alive) continue;
    if (!n.initialized) { err = "node " + std::to_string(i) + " is not initialised"; return false; }
    if (n.kind == NODE_POSE) { c.node_idx[i] = (int)c.pose_node.size(); c.pose_node.push_back(i); }
    else { c.node_idx[i] = (int)c.plane_node.size(); c.plane_node.push_back(i); }
  }
  c.N = (int)c.pose_node.size(); c.M = (int)c.plane_node.size();
  const int N = c.N, M = c.M;
  c.pose_val.resize((size_t)N * 7); c.plane_val.resize((size_t)M * 4);
  for (int p = 0; p < N; p++) std::memcpy(&c.pose_val[(size_t)p * 7], g.nodes[c.pose_node[p]].v, 7 * sizeof(double));
  for (int l = 0; l < M; l++) std::memcpy(&c.plane_val[(size_t)l * 4], g.nodes[c.plane_node[l]].v, 4 * sizeof(double));

  // ---- split factors ----
  std::vector<int> ppf;  // pose-plane factor ids in insertion order
  {
    int npp = 0, npf = 0, nlp = 0;
    for (const HFactor& F : g.factors) {
      if (!F.alive) continue;
      if (F.kind == F_POSE_PLANE) npp++; else if (F.kind == F_PLANE_PRIOR) nlp++; else npf++;
    }
    ppf.reserve(npp);
    c.pf_fid.reserve(npf); c.pf_i.reserve(npf); c.pf_j.reserve(npf); c.pf_meas.reserve((size_t)npf * 6); c.pf_sinf.reserve((size_t)npf * 21);
    c.lp_fid.reserve(nlp); c.lp_plane.reserve(nlp); c.lp_meas.reserve((size_t)nlp * 4); c.lp_sinf.reserve((size_t)nlp * 6);
  }
  for (int f = 0; f < (int)g.factors.size(); f++) {
    const HFactor& F = g.factors[f];
    if (!F.alive) continue;
    switch (F.kind) {
      case F_POSE_PLANE: ppf.push_back(f); break;
      case F_POSE_PRIOR:
      case F_ODOMETRY:
        c.pf_fid.push_back(f);
        c.pf_i.push_back(c.node_idx[F.nodes[0]]);
        c.pf_j.push_back(F.kind == F_ODOMETRY ? c.node_idx[F.nodes[1]] : -1);
        c.pf_meas.insert(c.pf_meas.end(), F.meas, F.meas + 6);
        c.pf_sinf.insert(c.pf_sinf.end(), F.sinf, F.sinf + 21);
        break;
      case F_PLANE_PRIOR:
        c.lp_fid.push_back(f);
        c.lp_plane.push_back(c.node_idx[F.nodes[0]]);
        c.lp_meas.insert(c.lp_meas.end(), F.meas, F.meas + 4);
        c.lp_sinf.insert(c.lp_sinf.end(), F.sinf, F.sinf + 6);
        break;
    }
  }
  c.Epf = (int)c.pf_fid.size(); c.Elp = (int)c.lp_fid.size();
  // ---- pose-major ordering of the pose-plane edges (stable: insertion order within a pose), padded so that
  //      every 16-pose block owns whole 32-edge tiles ----
  c.Epl = (int)ppf.size();
  const int E = c.Epl;
  c.nblk = (N + kBlockPoses - 1) / kBlockPoses;
  // stable counting sort by pose index (keys gathered once: the comparison sort chased the factor records)
  std::vector<int> order(E), key(E);
  {
    std::vector<int> start(N + 1, 0);
    for (int i = 0; i < E; i++) { key[i] = c.node_idx[g.factors[ppf[i]].nodes[0]]; start[key[i] + 1]++; }
    for (int p = 0; p < N; p++) start[p + 1] += start[p];
    for (int i = 0; i < E; i++) order[start[key[i]]++] = i;
  }
  c.pp_ptr.assign(N + 1, 0);
  c.tile_ptr.assign(c.nblk + 1, 0);
  {
    // count edges per pose, then lay the slots out block by block
    std::vector<int> cnt(N, 0);
    for (int i = 0; i < E; i++) cnt[key[i]]++;   // (the keys gathered for the counting sort)
    int slot = 0;
    for (int k = 0; k < c.nblk; k++) {
      c.tile_ptr[k] = slot / kTile;
      int p0 = k * kBlockPoses, p1 = std::min(N, p0 + kBlockPoses);
      for (int p = p0; p < p1; p++) { c.pp_ptr[p] = slot; slot += cnt[p]; }
      slot = (slot + kTile - 1) / kTile * kTile;
    }
    c.pp_ptr[N] = slot;  // only used as the end of the last pose when it has no padding after it
    c.tile_ptr[c.nblk] = slot / kTile;
    c.nslot = slot;
    // end of pose p's range = start + cnt (pp_ptr[p+1] may include padding): keep an explicit end array in pp_ptr
    // by storing starts in pp_ptr[0..N) and ends in pose_end
    c.ntile = slot / kTile;
    const int slots = c.nslot;
    c.pp_fid.assign(slots, -1); c.pp_pose.assign(slots, -1); c.pp_plane.assign(slots, 0);
    c.pp_meas.assign((size_t)slots * 4, 0.0); c.pp_sinf.assign((size_t)slots * 6, 0.0);
    for (int s2 = 0; s2 < slots; s2++) c.pp_meas[(size_t)s2 * 4] = 1.0;
    c.pp_rays.assign(1, 0.0); c.pp_kind.assign(1, 0); c.n_f2 = 0;
    std::vector<int> fill(c.pp_ptr.begin(), c.pp_ptr.begin() + N);
    for (int i = 0; i < E; i++) {
      const HFactor& F = g.factors[ppf[order[i]]];
      int p = key[order[i]];
      int e = fill[p]++;
      c.pp_fid[e] = ppf[order[i]];
      c.pp_pose[e] = p;
      c.pp_plane[e] = c.node_idx[F.nodes[1]];
      std::memcpy(&c.pp_meas[(size_t)e * 4], F.meas, 4 * sizeof(double));
      if (F.has_rays) {
        if (c.pp_rays.size() < (size_t)slots * 6) { c.pp_rays.assign((size_t)slots * 6, 0.0); c.pp_kind.assign(slots, 0); }
        std::memcpy(&c.pp_rays[(size_t)e * 6], F.rays, 6 * sizeof(double));
        c.pp_kind[e] = 1; c.n_f2++;
      }
      std::memcpy(&c.pp_sinf[(size_t)e * 6], F.sinf, 6 * sizeof(double));
    }
    c.pp_end.assign(N, 0);
    for (int p = 0; p < N; p++) c.pp_end[p] = c.pp_ptr[p] + cnt[p];
  }
  const int slots = c.nslot;
  // partial slots for the pose-major sweep: one per (tile, pose) run, numbered in slot order (block-local ranges)
  c.pm_part.assign(slots, -1);
  c.ypart_ptr.assign(N + 1, 0);
  c.blk_part_ptr.assign(c.nblk + 1, 0);
  {
    int np = 0, prev = -1;
    for (int e = 0; e < slots; e++) {
      int p = c.pp_pose[e];
      if (p < 0) { prev = -1; continue; }
      bool head = (e % kTile == 0) || (p != prev);
      if (head) { np++; c.ypart_ptr[p + 1]++; }
      c.pm_part[e] = np - 1;
      prev = p;
    }
    c.n_ypart = np;
    for (int p = 0; p < N; p++) c.ypart_ptr[p + 1] += c.ypart_ptr[p];
    for (int k = 0; k <= c.nblk; k++) c.blk_part_ptr[k] = c.ypart_ptr[std::min(N, k * kBlockPoses)];
  }
  // ---- plane-major view (slots of its own: dense, E real entries then padding) ----
  const int pslots = (E + kTile - 1) / kTile * kTile;
  c.ntile_pl = pslots / kTile;
  std::vector<int> pord(E);   // live slots in slot order, stably counting-sorted by plane
  {
    std::vector<int> start(M + 1, 0);
    for (int e = 0; e < slots; e++) if (c.pp_pose[e] >= 0) start[c.pp_plane[e] + 1]++;
    for (int l = 0; l < M; l++) start[l + 1] += start[l];
    for (int e = 0; e < slots; e++) if (c.pp_pose[e] >= 0) pord[start[c.pp_plane[e]]++] = e;
  }
  c.pl2pm.assign(pslots, -1); c.pl_plane.assign(pslots, -1); c.pl_pose.assign(pslots, 0); c.pl_part.assign(pslots, -1);
  c.pm2pl.assign(slots, -1);
  c.pl_ptr.assign(M + 1, 0); c.upart_ptr.assign(M + 1, 0);
  {
    int np = 0;
    for (int s2 = 0; s2 < E; s2++) {
      int e = pord[s2];
      c.pl2pm[s2] = e; c.pm2pl[e] = s2;
      c.pl_plane[s2] = c.pp_plane[e]; c.pl_pose[s2] = c.pp_pose[e];
      c.pl_ptr[c.pp_plane[e] + 1]++;
      bool head = (s2 % kTile == 0) || (c.pl_plane[s2] != c.pl_plane[s2 - 1]);
      if (head) { np++; c.upart_ptr[c.pl_plane[s2] + 1]++; }
      c.pl_part[s2] = np - 1;
    }
    c.n_upart = np;
    for (int l = 0; l < M; l++) { c.pl_ptr[l + 1] += c.pl_ptr[l]; c.upart_ptr[l + 1] += c.upart_ptr[l]; }
    c.heavy.clear(); c.huge.clear();   // planes with more than 8 partial sums are summed by a warp, more than 512 by a CTA
    for (int l = 0; l < M; l++) {
      const int n = c.upart_ptr[l + 1] - c.upart_ptr[l];
      if (n > 512) c.huge.push_back(l);
      else if (n > 8) c.heavy.push_back(l);
    }
    c.n_heavy = (int)c.heavy.size(); c.n_huge = (int)c.huge.size();
    if (c.heavy.empty()) c.heavy.push_back(-1);
    if (c.huge.empty()) c.huge.push_back(-1);
  }
  // ---- Hll / gl assembly tasks ----
  c.at_plane.clear(); c.at_lo.clear(); c.at_hi.clear(); c.as_plane.clear();
  c.at_ptr.assign(M + 1, 0);
  for (int l = 0; l < M; l++) {
    const int s0 = c.pl_ptr[l], s1 = c.pl_ptr[l + 1];
    c.at_ptr[l] = (int)c.at_plane.size();
    int lo = s0;
    do {   // (a plane without edges still gets one empty task: its priors are added there)
      const int hi = std::min(s1, lo + kAsmChunk);
      c.at_plane.push_back(l); c.at_lo.push_back(lo); c.at_hi.push_back(hi);
      lo = hi;
    } while (lo < s1);
    if ((int)c.at_plane.size() - c.at_ptr[l] > 1) c.as_plane.push_back(l);
  }
  c.at_ptr[M] = (int)c.at_plane.size();
  c.n_atask = (int)c.at_plane.size();
  c.n_asplit = (int)c.as_plane.size();
  if (c.at_plane.empty()) { c.at_plane.push_back(0); c.at_lo.push_back(0); c.at_hi.push_back(0); }
  if (c.as_plane.empty()) c.as_plane.push_back(-1);
  // ---- incidence lists ----
  c.pinc_ptr.assign(N + 1, 0);
  for (int f = 0; f < c.Epf; f++) { c.pinc_ptr[c.pf_i[f] + 1]++; if (c.pf_j[f] >= 0) c.pinc_ptr[c.pf_j[f] + 1]++; }
  for (int p = 0; p < N; p++) c.pinc_ptr[p + 1] += c.pinc_ptr[p];
  c.pinc.assign(c.pinc_ptr[N], 0);
  {
    std::vector<int> fill(c.pinc_ptr.begin(), c.pinc_ptr.end() - 1);
    for (int f = 0; f < c.Epf; f++) {
      c.pinc[fill[c.pf_i[f]]++] = (f << 1) | 0;
      if (c.pf_j[f] >= 0) c.pinc[fill[c.pf_j[f]]++] = (f << 1) | 1;
    }
  }
  // per pose: its first two pose-pose neighbours resolved (factor*2+side, other pose) and where the generic
  // incidence loop resumes -- one 32-byte record instead of a four-level index chain in the PCG pose phase
  c.pnbr.assign((size_t)N * 8, -1);
  for (int p = 0; p < N; p++) {
    int nf = 0, kk = c.pinc_ptr[p];
    const int i1 = c.pinc_ptr[p + 1];
    for (; kk < i1 && nf < 2; kk++) {
      const int inc = c.pinc[kk], f = inc >> 1, side = inc & 1;
      if (c.pf_j[f] < 0) continue;
      c.pnbr[(size_t)p * 8 + 2 * nf] = inc;
      c.pnbr[(size_t)p * 8 + 2 * nf + 1] = side ? c.pf_i[f] : c.pf_j[f];
      nf++;
    }
    c.pnbr[(size_t)p * 8 + 4] = kk;
    c.pnbr[(size_t)p * 8 + 5] = i1;
  }
  c.linc_ptr.assign(M + 1, 0);
  for (int f = 0; f < c.Elp; f++) c.linc_ptr[c.lp_plane[f] + 1]++;
  for (int l = 0; l < M; l++) c.linc_ptr[l + 1] += c.linc_ptr[l];
  c.linc.assign(c.linc_ptr[M], 0);
  {
    std::vector<int> fill(c.linc_ptr.begin(), c.linc_ptr.end() - 1);
    for (int f = 0; f < c.Elp; f++) c.linc[fill[c.lp_plane[f]]++] = f;
  }
  // ---- dense-block groups: the edges of every pose block grouped by plane ----
  c.blk_grp_ptr.assign(c.nblk + 1, 0);
  c.blk_simple.assign(c.nblk, 0);
  c.grp_of_slot.assign(slots, 0);
  c.grp_mem_ptr.clear(); c.grp_mem.clear(); c.grp_plane.clear();
  c.grp_mem.reserve(E); c.grp_plane.reserve(E / 2 + 16); c.grp_mem_ptr.reserve(E / 2 + 16);
  std::vector<unsigned long long> ekey;
  std::vector<int> es;
  for (int k = 0; k < c.nblk; k++) {
    int e0 = c.tile_ptr[k] * kTile, e1 = c.tile_ptr[k + 1] * kTile;
    // (plane, slot) packed into one integer: an integer sort gives the order of a stable sort by plane over the slot order
    ekey.clear();
    for (int e = e0; e < e1; e++) if (c.pp_pose[e] >= 0) ekey.push_back(((unsigned long long)(unsigned)c.pp_plane[e] << 32) | (unsigned)e);
    std::sort(ekey.begin(), ekey.end());
    es.resize(ekey.size());
    for (size_t i = 0; i < ekey.size(); i++) es[i] = (int)(unsigned)(ekey[i] & 0xffffffffull);
    int g0 = (int)c.grp_plane.size();
    for (int i = 0; i < (int)es.size(); i++) {
      if (i == 0 || c.pp_plane[es[i]] != c.pp_plane[es[i - 1]]) {
        c.grp_plane.push_back(c.pp_plane[es[i]]);
        c.grp_mem_ptr.push_back((int)c.grp_mem.size());
      }
      c.grp_of_slot[es[i]] = (int)c.grp_plane.size() - 1 - g0;
      c.grp_mem.push_back(es[i]);
    }
    c.blk_grp_ptr[k + 1] = (int)c.grp_plane.size();
    {  // fast dense-block build: at most 16 tiles, 96 planes and no pose observing one plane twice
      bool simple = (c.tile_ptr[k + 1] - c.tile_ptr[k] <= 16) && ((int)c.grp_plane.size() - g0 <= 96);
      for (int i = 1; i < (int)es.size() && simple; i++)
        if (c.pp_plane[es[i]] == c.pp_plane[es[i - 1]] && c.pp_pose[es[i]] == c.pp_pose[es[i - 1]]) simple = false;
      c.blk_simple[k] = simple ? 1 : 0;
    }
    {  // a block over either shared-memory limit of the fused pose phase keeps its vectors in the overflow scratch
      const int ng = c.blk_grp_ptr[k + 1] - g0, npart = c.blk_part_ptr[k + 1] - c.blk_part_ptr[k];
      if (ng > kMaxGrp || npart > kMaxPart) {
        if (c.blk_ovf.empty()) c.blk_ovf.assign(c.nblk, -1);
        c.blk_ovf[k] = (int)c.n_ovf;
        c.n_ovf += (size_t)ng * 3 + (size_t)npart * 6;
        c.n_ovf_blk++;
      }
    }
  }
  c.grp_mem_ptr.push_back((int)c.grp_mem.size());
  c.ngrp = (int)c.grp_plane.size();
  c.grp_info.assign((size_t)std::max(1, c.ngrp) * 4, 0);   // {plane, first partial sum, number of partial sums, -}
  for (int g = 0; g < c.ngrp; g++) {
    const int l = c.grp_plane[g];
    c.grp_info[(size_t)g * 4] = l;
    c.grp_info[(size_t)g * 4 + 1] = c.upart_ptr[l];
    c.grp_info[(size_t)g * 4 + 2] = c.upart_ptr[l + 1] - c.upart_ptr[l];
  }
  {
    // per-block partial sums of the block-resident PCG: plane l owns slots [ub_ptr[l], ub_ptr[l+1]), one per observing pose
    // block in ascending block order (groups are numbered block by block, so a counting pass keeps that order)
    std::vector<int> ub_ptr(M + 1, 0);
    for (int g2 = 0; g2 < c.ngrp; g2++) ub_ptr[c.grp_plane[g2] + 1]++;
    for (int l = 0; l < M; l++) ub_ptr[l + 1] += ub_ptr[l];
    std::vector<int> fill(ub_ptr.begin(), ub_ptr.end() - 1);
    c.grp_info2.assign((size_t)std::max(1, c.ngrp) * 4, 0);
    for (int g2 = 0; g2 < c.ngrp; g2++) {
      const int l = c.grp_plane[g2];
      c.grp_info2[(size_t)g2 * 4] = l;
      c.grp_info2[(size_t)g2 * 4 + 1] = ub_ptr[l];
      c.grp_info2[(size_t)g2 * 4 + 2] = ub_ptr[l + 1] - ub_ptr[l];
      c.grp_info2[(size_t)g2 * 4 + 3] = fill[l]++;
    }
    c.res_nt = c.res_ng = c.res_np = 0;
    for (int k = 0; k < c.nblk; k++) {
      c.res_nt = std::max(c.res_nt, c.tile_ptr[k + 1] - c.tile_ptr[k]);
      c.res_ng = std::max(c.res_ng, c.blk_grp_ptr[k + 1] - c.blk_grp_ptr[k]);
      c.res_np = std::max(c.res_np, c.blk_part_ptr[k + 1] - c.blk_part_ptr[k]);
    }
  }
  // ---- (plane, node) pairs of the two hat levels ----
  auto build_pairs = [&](int SPx, std::vector<int>& ce_ptr, std::vector<int>& ce_node, std::vector<int>& ce_plane, std::vector<int>& ce_lo,
                         std::vector<int>& ce_hi) {
    ce_ptr.assign(M + 1, 0);
    ce_node.clear(); ce_plane.clear(); ce_lo.clear(); ce_hi.clear();
    for (int l = 0; l < M; l++) {
      int s0 = c.pl_ptr[l], s1 = c.pl_ptr[l + 1];
      int last = -1;
      for (int s = s0; s < s1; s++) {
        int p = c.pl_pose[s];
        int c0 = p / SPx;
        int cand[2] = {c0, (p % SPx) ? c0 + 1 : -1};
        for (int q = 0; q < 2; q++) {
          int nd = cand[q];
          if (nd < 0 || nd <= last) continue;
          // slots of plane l supporting node nd: poses in ((nd-1)*SP, (nd+1)*SP)
          // slots are pose-sorted within the plane: lo = first slot with pose > (nd-1)*SP, hi = first with pose >= (nd+1)*SP
          const int* pb = c.pl_pose.data();
          const int lo = (int)(std::upper_bound(pb + s0, pb + s1, (nd - 1) * SPx) - pb);
          const int hi = (int)(std::lower_bound(pb + lo, pb + s1, (nd + 1) * SPx) - pb);
          ce_node.push_back(nd); ce_plane.push_back(l); ce_lo.push_back(lo); ce_hi.push_back(hi);
          last = nd;
        }
      }
      ce_ptr[l + 1] = (int)ce_node.size();
    }
  };
  c.levels = g.force_levels ? g.force_levels : (N > kL2Spacing * kMaxCoarseNodes ? 3 : 2);
  c.SP = coarse_spacing(N, c.levels);
  const int SPc = c.SP;
  c.nc = coarse_nodes(N, SPc);
  c.nc_pad = (c.nc + kPivotNodes - 1) / kPivotNodes * kPivotNodes;
  build_pairs(SPc, c.ce_ptr, c.ce_node, c.ce_plane, c.ce_lo, c.ce_hi);
  c.nc2 = coarse_nodes(N, kL2Spacing);
  c.ng2 = (c.nc2 + kGroupNodes - 1) / kGroupNodes;
  if (c.levels == 3) build_pairs(kL2Spacing, c.ce2_ptr, c.ce2_node, c.ce2_plane, c.ce2_lo, c.ce2_hi);
  else { c.ce2_ptr.assign(M + 1, 0); c.ce2_node.assign(1, 0); c.ce2_plane.assign(1, 0); c.ce2_lo.assign(1, 0); c.ce2_hi.assign(1, 0); c.ng2 = 0; }
  c.nce2 = (c.levels == 3) ? (int)c.ce2_node.size() : 0;
  if (c.levels == 3) {
    // per group: its pairs in (plane, node) order = the order they already have, restricted to the group's nodes
    c.g2_ptr.assign(c.ng2 + 1, 0);
    for (int i = 0; i < c.nce2; i++) c.g2_ptr[c.ce2_node[i] / kGroupNodes + 1]++;
    for (int gq = 0; gq < c.ng2; gq++) c.g2_ptr[gq + 1] += c.g2_ptr[gq];
    c.g2_ce.assign(std::max(1, c.nce2), 0);
    std::vector<int> fill(c.g2_ptr.begin(), c.g2_ptr.end() - 1);
    for (int i = 0; i < c.nce2; i++) c.g2_ce[fill[c.ce2_node[i] / kGroupNodes]++] = i;
  } else {
    c.g2_ptr.assign(1, 0); c.g2_ce.assign(1, 0);
  }
  c.nce = (int)c.ce_node.size();
  c.n2ce_ptr.assign(c.nc + 1, 0);
  for (int i = 0; i < c.nce; i++) c.n2ce_ptr[c.ce_node[i] + 1]++;
  for (int a = 0; a < c.nc; a++) c.n2ce_ptr[a + 1] += c.n2ce_ptr[a];
  c.n2ce.assign(c.nce, 0);
  {
    std::vector<int> fill(c.n2ce_ptr.begin(), c.n2ce_ptr.end() - 1);
    for (int i = 0; i < c.nce; i++) c.n2ce[fill[c.ce_node[i]]++] = i;
  }
  // ---- output-stationary assembly of A_c = P^T S P: for every coarse node pair (a, b) the plane products
  // Wc[a,l] Hll^-1 Wc[b,l]^T of the light planes and the pose-pose factors coupling the two supports; planes that
  // touch more than kHeavyCoarse nodes (the ground plane touches all) are applied as dense rank-3 updates instead
  {
    const int nc = c.nc;
    const size_t np = (size_t)nc * nc;
    c.hv_plane.clear();
    std::vector<char> heavy(M, 0);
    for (int l = 0; l < M; l++)
      if (c.ce_ptr[l + 1] - c.ce_ptr[l] > kHeavyCoarse) { heavy[l] = 1; c.hv_plane.push_back(l); }
    c.n_hv = (int)c.hv_plane.size();
    if (c.hv_plane.empty()) c.hv_plane.push_back(-1);
    c.lp_ptr.assign(np + 1, 0);
    for (int l = 0; l < M; l++) {
      if (heavy[l]) continue;
      for (int i = c.ce_ptr[l]; i < c.ce_ptr[l + 1]; i++)
        for (int j = c.ce_ptr[l]; j < c.ce_ptr[l + 1]; j++) c.lp_ptr[(size_t)c.ce_node[i] * nc + c.ce_node[j] + 1]++;
    }
    for (size_t q = 0; q < np; q++) c.lp_ptr[q + 1] += c.lp_ptr[q];
    c.lp_cea.assign(std::max(1, c.lp_ptr[np]), 0);
    c.lp_ceb.assign(std::max(1, c.lp_ptr[np]), 0);
    {
      std::vector<int> fill(c.lp_ptr.begin(), c.lp_ptr.end() - 1);
      for (int l = 0; l < M; l++) {   // plane-ascending order inside every pair: fixed summation order
        if (heavy[l]) continue;
        for (int i = c.ce_ptr[l]; i < c.ce_ptr[l + 1]; i++)
          for (int j = c.ce_ptr[l]; j < c.ce_ptr[l + 1]; j++) {
            int at = fill[(size_t)c.ce_node[i] * nc + c.ce_node[j]]++;
            c.lp_cea[at] = i; c.lp_ceb[at] = j;
          }
      }
    }
    auto nodes_of = [&](int p, int* out) {   // coarse nodes whose hat function is non-zero at pose p
      int n = 0, c0 = p / SPc;
      if (c0 < nc) out[n++] = c0;
      if ((p % SPc) && c0 + 1 < nc) out[n++] = c0 + 1;
      return n;
    };
    c.fp_ptr.assign(np + 1, 0);
    for (int pass = 0; pass < 2; pass++) {
      std::vector<int> fill;
      if (pass == 1) {
        for (size_t q = 0; q < np; q++) c.fp_ptr[q + 1] += c.fp_ptr[q];
        c.fp_f.assign(std::max(1, c.fp_ptr[np]), 0);
        fill.assign(c.fp_ptr.begin(), c.fp_ptr.end() - 1);
      }
      for (int f = 0; f < c.Epf; f++) {
        if (c.pf_j[f] < 0) continue;
        for (int side = 0; side < 2; side++) {
          const int p = side ? c.pf_j[f] : c.pf_i[f], o = side ? c.pf_i[f] : c.pf_j[f];
          int na[2], nb[2];
          const int ka = nodes_of(p, na), kb = nodes_of(o, nb);
          for (int x = 0; x < ka; x++)
            for (int y = 0; y < kb; y++) {
              const size_t q = (size_t)na[x] * nc + nb[y];
              if (pass == 0) c.fp_ptr[q + 1]++;
              else c.fp_f[fill[q]++] = f * 2 + side;
            }
        }
      }
    }
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
// Tables of the exact direct solves (pus_set_linear_solver(h, 1) dense, (h, 2) band), built only for handles in those modes.
// The reduced system is assembled entry by entry; for every pose pair a >= b inside the envelope (index pair_index(a, b))
// the host lists what couples the two poses, in a fixed order:
//   dfp: pose-pose factors, f * 2 + side (side 1: the factor's second pose is a, its block enters transposed), factor order;
//   dlp: eliminated planes seen from both poses, as a pair of (pose, plane) incidences (the coarse assembly's lp lists with
//        P = I), plane-ascending.  An incidence covers every edge between its pose and plane (a pose that observes a plane
//        twice has one incidence with two edges), as a range of plane-major slots.
// Band layout (kind 2): the poses in insertion order, padded to a whole tile with identity, then 3 rows per bordered plane
// (plane-ascending), padded likewise.  A bordered plane stays an unknown of the reduced system instead of being eliminated:
// eliminating a plane couples every pair of its observers, so the few planes seen from most of the trajectory (the ground
// plane, a plane merged by a loop closure) would make the whole system dense.  Tile row i holds tiles first[i] .. i only
// (first[i]: the smallest tile column any of its rows couples to); a Cholesky factor has no fill outside that envelope.
// The dense solve (kind 1) is the same layout with no bordered plane and first = 0.
// ------------------------------------------------------------------------------------------------
constexpr int kDirectMaxPoses = 640;          // order 3 840: 80 tile columns of 48
constexpr int kBandMaxBorder = 64;            // most bordered planes the band layout tries
constexpr long long kBandBudgetBytes = 8ll << 30;   // device memory a band solve may take (8 GiB)
constexpr long long kDirectTileBytes = 48ll * 52 * 8;   // one 48 x 48 tile at leading dimension 52 (kAcTile doubles)

struct DirectTables {
  int nb = 0;    // tile rows of the padded order 48 nb
  int nbp = 0;   // tile rows of the poses (>= 6 N / 48); the bordered planes' rows start at tile row nbp
  std::vector<int> inc_pose, inc_plane, inc_lo, inc_hi;
  std::vector<int> inc_ptr;             // per plane l: its incidences [inc_ptr[l], inc_ptr[l + 1])
  std::vector<int> lp_ptr, lp_a, lp_b, fp_ptr, fp_f;
  std::vector<int> first, toff, poff;   // per tile row: first tile column, tile offset (+ total); per pose: first pair index
  std::vector<int> col_ptr, col_row;    // per tile column K: the tile rows i > K with first[i] <= K, ascending
  std::vector<int> border, binc;        // bordered planes (ascending); [lo, hi) of each one's incidences
  long long bytes = 0;                  // device memory of the solve's tiles, vectors and tables
  // nested-dissection layout (kind 2, order 1; empty otherwise): tile columns are numbered in the new order.  Tiles are stored
  // level by level, the columns of a level ascending, each column's tiles row-ascending (its diagonal tile first).
  int order = 0;                        // 0: insertion order (the envelope above), 1: nested dissection
  int nlev = 0;                         // levels of the elimination tree
  long long nupd = 0;                   // tile products of one factorization (update-list entries)
  std::vector<int> nd_perm, nd_pos;     // new column -> original tile, original tile -> new column
  std::vector<int> nd_parent, nd_level; // per column: elimination-tree parent (-1: a root), level (0: a leaf)
  std::vector<int> nd_cptr, nd_crow;    // per column j: the tile rows i >= j of L's pattern, ascending
  std::vector<int> nd_toff;             // per column: storage index of its diagonal tile (its tiles follow it)
  std::vector<int> nd_lptr, nd_lcol, nd_ltptr;   // per level: its columns (ascending), its tile range
  std::vector<int> nd_trow, nd_tcol;    // per stored tile: tile row, tile column
  std::vector<int> nd_uptr, nd_upd;     // per stored tile (i, j): pairs (tile of L_iK, tile of L_jK), K < j ascending
  std::vector<int> nd_rptr, nd_rtile;   // per tile row j: the tiles (j, K), K < j ascending
  std::vector<int> nd_dev;              // the tables above that the device reads, packed (NdTable)

  // the storage index of tile (i, j), i >= j, of the factor's order, or -1 outside the stored pattern
  int tile(int i, int j) const {
    if (order != 1) return j < first[i] ? -1 : toff[i] + j - first[i];
    const int* b = nd_crow.data() + nd_cptr[j];
    const int n = nd_cptr[j + 1] - nd_cptr[j], p = (int)(std::lower_bound(b, b + n, i) - b);
    return (p == n || b[p] != i) ? -1 : nd_toff[j] + p;
  }
  // padded row r of the bordered order -> its row in the factor's order (the identity in insertion order)
  int row(int r) const { return order == 1 ? 48 * nd_pos[r / 48] + r % 48 : r; }
  int ntile() const { return order == 1 ? nd_cptr[nb] : toff[nb]; }   // stored tiles
};

// ---- nested-dissection order of the pose tiles (kind 2, order 1) ----
// Connected components one after another (by their lowest tile); a component is bisected by the BFS level structure from a
// pseudo-peripheral tile: the separator is the tiles of the median level adjacent to the level after it, ordered after both
// halves.  Parts of at most kNdLeaf tiles, and parts whose level structure has fewer than three levels, keep insertion order.
constexpr int kNdLeaf = 4;
// the ND tables the device reads, packed into one array (DirectTables::nd_dev): entry 0 the number of levels, entries 1 .. 13
// the offsets of the tables
enum NdTable { ND_NLEV = 0, ND_POS, ND_PERM, ND_LPTR, ND_LCOL, ND_LTPTR, ND_TOFF, ND_CPTR, ND_TROW, ND_TCOL, ND_UPTR, ND_UPD,
               ND_RPTR, ND_RTILE, ND_HDR };

struct NdOrder {
  const std::vector<std::vector<int>>& adj;
  std::vector<int> in, comp, seen, lev, out;
  int stamp = 0, vstamp = 0;
  explicit NdOrder(const std::vector<std::vector<int>>& a)
      : adj(a), in(a.size(), 0), comp(a.size(), 0), seen(a.size(), 0), lev(a.size(), 0) {}

  // BFS level structure from r inside the part stamped s: tiles level by level (each level ascending), level pointers
  void bfs(int r, int s, std::vector<int>& q, std::vector<int>& lp) {
    vstamp++;
    q.assign(1, r); lp.assign(1, 0);
    seen[r] = vstamp; lev[r] = 0;
    size_t h = 0;
    while (h < q.size()) {
      const size_t e = q.size();
      lp.push_back((int)e);
      for (; h < e; h++)
        for (int u : adj[q[h]])
          if (in[u] == s && seen[u] != vstamp) { seen[u] = vstamp; lev[u] = lev[q[h]] + 1; q.push_back(u); }
      std::sort(q.begin() + e, q.end());
    }
  }
  void dissect(std::vector<int> S) {   // S ascending
    if ((int)S.size() <= kNdLeaf) { out.insert(out.end(), S.begin(), S.end()); return; }
    const int s = ++stamp;
    for (int t : S) in[t] = s;
    std::vector<int> q, lp;
    {   // components
      std::vector<std::vector<int>> comps;
      for (int t : S) {
        if (comp[t] == s) continue;
        bfs(t, s, q, lp);
        for (int u : q) comp[u] = s;
        std::sort(q.begin(), q.end());
        comps.push_back(q);
      }
      if (comps.size() > 1) { for (auto& cpt : comps) dissect(cpt); return; }
    }
    // pseudo-peripheral tile: from the lowest tile, move to the lowest tile of the last level while the depth grows
    int v = S[0];
    bfs(v, s, q, lp);
    for (;;) {
      const int h = (int)lp.size() - 1, u = q[lp[h - 1]];
      std::vector<int> q2, lp2;
      bfs(u, s, q2, lp2);
      if ((int)lp2.size() - 1 <= h) { bfs(v, s, q, lp); break; }
      v = u; q.swap(q2); lp.swap(lp2);
    }
    const int h = (int)lp.size() - 1;
    if (h <= 2) { out.insert(out.end(), S.begin(), S.end()); return; }
    int m = 0;   // the level holding the median tile, kept off both ends
    while (2 * lp[m + 1] < (int)S.size()) m++;
    m = std::max(1, std::min(h - 2, m));
    std::vector<int> A, B, sep;
    for (int k = 0; k < lp[m]; k++) A.push_back(q[k]);
    for (int k = lp[m]; k < lp[m + 1]; k++) {
      bool far = false;
      for (int u : adj[q[k]]) if (in[u] == s && seen[u] == vstamp && lev[u] == m + 1) { far = true; break; }
      (far ? sep : A).push_back(q[k]);
    }
    for (int k = lp[m + 1]; k < (int)q.size(); k++) B.push_back(q[k]);
    std::sort(A.begin(), A.end()); std::sort(B.begin(), B.end());
    dissect(A);
    dissect(B);
    out.insert(out.end(), sep.begin(), sep.end());
  }
};

// Symbolic Cholesky at tile granularity of the matrix whose lower pattern is alow (per column j: rows i > j, any order):
// column patterns (ascending, diagonal first), elimination-tree parents and levels.  Returns the number of levels.
inline int nd_symbolic(int nb, std::vector<std::vector<int>>& alow, std::vector<int>& cptr, std::vector<int>& crow,
                       std::vector<int>& parent, std::vector<int>& level) {
  std::vector<std::vector<int>> kids(nb);
  std::vector<int> mark(nb, -1), col;
  cptr.assign(nb + 1, 0); crow.clear(); parent.assign(nb, -1); level.assign(nb, 0);
  int nlev = 0;
  for (int j = 0; j < nb; j++) {
    col.assign(1, j); mark[j] = j;
    for (int i : alow[j]) if (mark[i] != j) { mark[i] = j; col.push_back(i); }
    for (int c : kids[j]) {
      for (int p = cptr[c] + 1; p < cptr[c + 1]; p++) {
        const int i = crow[p];
        if (i != j && mark[i] != j) { mark[i] = j; col.push_back(i); }
      }
      level[j] = std::max(level[j], level[c] + 1);
    }
    std::sort(col.begin(), col.end());
    crow.insert(crow.end(), col.begin(), col.end());
    cptr[j + 1] = (int)crow.size();
    if (col.size() > 1) { parent[j] = col[1]; kids[col[1]].push_back(j); }
    nlev = std::max(nlev, level[j] + 1);
  }
  return nlev;
}

// The nested-dissection layout that borders the planes with bslot >= 0 (nbord of them): the tile order (new -> original),
// L's pattern, and the device bytes it takes
inline long long nd_layout(const Compiled& c, const std::vector<int>& inc_ptr, const std::vector<int>& inc_pose,
                           const std::vector<int>& bslot, int nbord, DirectTables& d) {
  const int N = c.N, M = c.M;
  const int nbp = std::max(1, (6 * N + 47) / 48), nb = nbp + (3 * nbord + 47) / 48;
  d.nbp = nbp; d.nb = nb;
  // pose-tile graph: a pose-pose factor, or an eliminated plane seen from both tiles
  std::vector<std::vector<int>> adj(nbp), bt(nb);   // bt[t]: pose tiles coupled to bordered tile t
  long long lp = 0, fp = 0;
  for (int f = 0; f < c.Epf; f++) {
    if (c.pf_j[f] < 0) continue;
    fp++;
    const int u = c.pf_i[f] / 8, v = c.pf_j[f] / 8;
    if (u != v) { adj[u].push_back(v); adj[v].push_back(u); }
  }
  std::vector<int> tl;
  for (int l = 0; l < M; l++) {
    const int n = inc_ptr[l + 1] - inc_ptr[l];
    if (n == 0) continue;
    tl.clear();
    for (int i = inc_ptr[l]; i < inc_ptr[l + 1]; i++) if (tl.empty() || tl.back() != inc_pose[i] / 8) tl.push_back(inc_pose[i] / 8);
    if (bslot[l] >= 0) {
      std::vector<int>& b = bt[nbp + 3 * bslot[l] / 48];
      b.insert(b.end(), tl.begin(), tl.end());
      continue;
    }
    lp += (long long)n * (n + 1) / 2;
    for (int u : tl)
      for (int v : tl) if (u != v) adj[u].push_back(v);
  }
  for (auto& a : adj) { std::sort(a.begin(), a.end()); a.erase(std::unique(a.begin(), a.end()), a.end()); }
  NdOrder nd(adj);
  std::vector<int> all(nbp);
  for (int t = 0; t < nbp; t++) all[t] = t;
  nd.dissect(all);
  d.nd_perm = nd.out;
  for (int t = nbp; t < nb; t++) d.nd_perm.push_back(t);   // bordered tiles last: the root of the elimination tree
  d.nd_pos.assign(nb, 0);
  for (int j = 0; j < nb; j++) d.nd_pos[d.nd_perm[j]] = j;
  std::vector<std::vector<int>> alow(nb);
  auto couple = [&](int u, int v) {
    const int a = d.nd_pos[u], b = d.nd_pos[v];
    if (a > b) alow[b].push_back(a); else if (b > a) alow[a].push_back(b);
  };
  for (int u = 0; u < nbp; u++) for (int v : adj[u]) if (v > u) couple(u, v);
  for (int t = nbp; t < nb; t++) for (int u : bt[t]) couple(t, u);
  d.nlev = nd_symbolic(nb, alow, d.nd_cptr, d.nd_crow, d.nd_parent, d.nd_level);
  const long long T = d.nd_cptr[nb];
  d.nupd = 0;
  for (int j = 0; j < nb; j++) { const long long m = d.nd_cptr[j + 1] - d.nd_cptr[j] - 1; d.nupd += m * (m + 1) / 2; }
  const long long ninc = (long long)inc_pose.size();
  const long long ints = 5ll * nb + 2ll * d.nlev + 132 * T + 2 * d.nupd + 2 * lp + fp + 3 * ninc + 3ll * nbord + 7 + ND_HDR;
  return (T + nb) * kDirectTileBytes                                 // tiles, pivot inverses
         + 8 * (2ll * 48 * nb + 36 * ninc + 3ll * nbord) + 4 * ints;   // solve vectors, W / Y per incidence, border rhs, tables
}

// the device tables of the chosen nested-dissection layout: tile storage by level, update lists, row lists
inline void nd_tables(DirectTables& d) {
  const int nb = d.nb;
  d.nd_lptr.assign(d.nlev + 1, 0);
  for (int j = 0; j < nb; j++) d.nd_lptr[d.nd_level[j] + 1]++;
  for (int l = 0; l < d.nlev; l++) d.nd_lptr[l + 1] += d.nd_lptr[l];
  d.nd_lcol.assign(nb, 0);
  {
    std::vector<int> fill(d.nd_lptr.begin(), d.nd_lptr.end() - 1);
    for (int j = 0; j < nb; j++) d.nd_lcol[fill[d.nd_level[j]]++] = j;
  }
  const int T = d.nd_cptr[nb];
  d.nd_toff.assign(nb, 0); d.nd_ltptr.assign(d.nlev + 1, 0);
  d.nd_trow.assign(T, 0); d.nd_tcol.assign(T, 0);
  int t = 0;
  for (int l = 0; l < d.nlev; l++) {
    d.nd_ltptr[l] = t;
    for (int k = d.nd_lptr[l]; k < d.nd_lptr[l + 1]; k++) {
      const int j = d.nd_lcol[k];
      d.nd_toff[j] = t;
      for (int p = d.nd_cptr[j]; p < d.nd_cptr[j + 1]; p++, t++) { d.nd_trow[t] = d.nd_crow[p]; d.nd_tcol[t] = j; }
    }
  }
  d.nd_ltptr[d.nlev] = t;
  d.nd_uptr.assign(T + 1, 0);
  d.nd_rptr.assign(nb + 1, 0);
  for (int pass = 0; pass < 2; pass++) {
    std::vector<int> fill, rfill;
    if (pass == 1) {
      for (int q = 0; q < T; q++) d.nd_uptr[q + 1] += d.nd_uptr[q];
      for (int j = 0; j < nb; j++) d.nd_rptr[j + 1] += d.nd_rptr[j];
      d.nd_upd.assign(std::max(2, 2 * d.nd_uptr[T]), 0);
      d.nd_rtile.assign(std::max(1, d.nd_rptr[nb]), 0);
      fill.assign(d.nd_uptr.begin(), d.nd_uptr.end() - 1);
      rfill.assign(d.nd_rptr.begin(), d.nd_rptr.end() - 1);
    }
    for (int K = 0; K < nb; K++) {   // ascending K: every list comes out K-ascending
      const int p0 = d.nd_cptr[K] + 1, p1 = d.nd_cptr[K + 1], t0 = d.nd_toff[K] + 1 - p0;
      for (int a = p0; a < p1; a++) {
        const int i = d.nd_crow[a];
        if (pass == 0) d.nd_rptr[i + 1]++; else d.nd_rtile[rfill[i]++] = t0 + a;
        for (int b = p0; b <= a; b++) {
          const int q = d.tile(i, d.nd_crow[b]);
          if (pass == 0) d.nd_uptr[q + 1]++;
          else { const int at = fill[q]++; d.nd_upd[2 * at] = t0 + a; d.nd_upd[2 * at + 1] = t0 + b; }
        }
      }
    }
  }
  const std::vector<int>* tab[ND_HDR] = {nullptr, &d.nd_pos, &d.nd_perm, &d.nd_lptr, &d.nd_lcol, &d.nd_ltptr, &d.nd_toff,
                                         &d.nd_cptr, &d.nd_trow, &d.nd_tcol, &d.nd_uptr, &d.nd_upd, &d.nd_rptr, &d.nd_rtile};
  d.nd_dev.assign(ND_HDR, 0);
  d.nd_dev[ND_NLEV] = d.nlev;
  for (int k = 1; k < ND_HDR; k++) {
    d.nd_dev[k] = (int)d.nd_dev.size();
    d.nd_dev.insert(d.nd_dev.end(), tab[k]->begin(), tab[k]->end());
  }
}

// first[] of a layout that borders the planes with bslot >= 0 (nbord of them), and the device bytes it takes
inline long long band_envelope(const Compiled& c, const std::vector<int>& inc_ptr, const std::vector<int>& inc_pose,
                               const std::vector<int>& bslot, int nbord, std::vector<int>& first, int& nbp, int& nb) {
  const int N = c.N, M = c.M;
  nbp = std::max(1, (6 * N + 47) / 48);
  nb = nbp + (3 * nbord + 47) / 48;
  std::vector<int> mp(N);   // smallest pose each pose couples to
  for (int a = 0; a < N; a++) mp[a] = a;
  for (int f = 0; f < c.Epf; f++) {
    if (c.pf_j[f] < 0) continue;
    const int hi = std::max(c.pf_i[f], c.pf_j[f]), lo = std::min(c.pf_i[f], c.pf_j[f]);
    mp[hi] = std::min(mp[hi], lo);
  }
  first.assign(nb, 0);
  for (int i = 0; i < nb; i++) first[i] = i;
  long long lp = 0;
  for (int l = 0; l < M; l++) {
    const int n = inc_ptr[l + 1] - inc_ptr[l];
    if (n == 0) continue;
    const int pmin = inc_pose[inc_ptr[l]];   // incidences are pose-ascending inside a plane
    if (bslot[l] >= 0) {
      const int t = nbp + 3 * bslot[l] / 48;
      first[t] = std::min(first[t], pmin / 8);
    } else {
      lp += (long long)n * (n + 1) / 2;
      for (int i = inc_ptr[l]; i < inc_ptr[l + 1]; i++) mp[inc_pose[i]] = std::min(mp[inc_pose[i]], pmin);
    }
  }
  for (int a = 0; a < N; a++) first[a / 8] = std::min(first[a / 8], mp[a] / 8);   // 8 poses of 6 rows per tile
  long long tiles = 0, npair = 0, fp = 0;
  for (int i = 0; i < nb; i++) tiles += i - first[i] + 1;
  for (int a = 0; a < N; a++) npair += a - 8 * first[a / 8] + 1;
  for (int f = 0; f < c.Epf; f++) fp += c.pf_j[f] >= 0;
  const long long ninc = (long long)inc_pose.size();
  const long long ints = 2 * (npair + 1) + 2 * lp + fp + 3 * ninc + nb + (nb + 1) + N + (nb + 1) + (tiles - nb) + 3 * nbord;
  return (tiles + 3ll * nb) * kDirectTileBytes   // tiles, two pivot-column snapshots, pivot inverses
         + 8 * (2ll * 48 * nb + 36 * ninc + 3ll * nbord) + 4 * ints;   // solve vectors, W / Y per incidence, border rhs, tables
}

// Bordering: rank the planes by `key` (descending; ties: lower index) and border the k first, k = 0 .. min(M, 64), whichever
// k takes the fewest device bytes (ties: the smaller k); bytes(bslot, k) is the device bytes of a layout.  Out: the bordered
// planes (ascending) and each plane's slot among them (-1: eliminated).
template <typename Bytes>
inline void choose_border(const std::vector<int>& key, Bytes bytes, std::vector<int>& border, std::vector<int>& bslot) {
  const int M = (int)key.size();
  std::vector<int> order(M);
  for (int l = 0; l < M; l++) order[l] = l;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return key[x] > key[y]; });
  auto pick = [&](int k) {
    border.assign(order.begin(), order.begin() + k);
    std::sort(border.begin(), border.end());
    bslot.assign(M, -1);
    for (int q = 0; q < k; q++) bslot[border[q]] = q;
  };
  long long best = -1;
  int best_k = 0;
  for (int k = 0; k <= std::min(M, kBandMaxBorder); k++) {
    pick(k);
    const long long b = bytes(bslot, k);
    if (best < 0 || b < best) { best = b; best_k = k; }
  }
  pick(best_k);
}

// The per-pose-pair assembly lists; pair(a, b) is the index of the pose pair (a, b), a >= b in insertion order.  lp: the
// incidence pairs (i, j), i >= j, of every eliminated plane (incidences are pose-ascending inside a plane: i >= j gives
// a >= b); fp: the pose-pose factors, f * 2 + side (side 1: a is the factor's second pose).
template <typename Pair>
inline void pair_lists(const Compiled& c, const std::vector<int>& bslot, size_t np, Pair pair, DirectTables& d) {
  d.lp_ptr.assign(np + 1, 0);
  d.fp_ptr.assign(np + 1, 0);
  for (int pass = 0; pass < 2; pass++) {
    std::vector<int> lfill, ffill;
    if (pass == 1) {
      for (size_t q = 0; q < np; q++) { d.lp_ptr[q + 1] += d.lp_ptr[q]; d.fp_ptr[q + 1] += d.fp_ptr[q]; }
      d.lp_a.assign(std::max(1, d.lp_ptr[np]), 0);
      d.lp_b.assign(std::max(1, d.lp_ptr[np]), 0);
      d.fp_f.assign(std::max(1, d.fp_ptr[np]), 0);
      lfill.assign(d.lp_ptr.begin(), d.lp_ptr.end() - 1);
      ffill.assign(d.fp_ptr.begin(), d.fp_ptr.end() - 1);
    }
    for (int l = 0; l < c.M; l++) {
      if (bslot[l] >= 0) continue;
      for (int i = d.inc_ptr[l]; i < d.inc_ptr[l + 1]; i++)
        for (int j = d.inc_ptr[l]; j <= i; j++) {
          const size_t q = pair(d.inc_pose[i], d.inc_pose[j]);
          if (pass == 0) d.lp_ptr[q + 1]++;
          else { const int at = lfill[q]++; d.lp_a[at] = i; d.lp_b[at] = j; }
        }
    }
    for (int f = 0; f < c.Epf; f++) {
      if (c.pf_j[f] < 0) continue;
      for (int side = 0; side < 2; side++) {
        const int a = side ? c.pf_j[f] : c.pf_i[f], b = side ? c.pf_i[f] : c.pf_j[f];
        if (a < b) continue;
        const size_t q = pair(a, b);
        if (pass == 0) d.fp_ptr[q + 1]++;
        else d.fp_f[ffill[q]++] = f * 2 + side;
      }
    }
  }
}

// kind 2, order 1: the nested-dissection layout.  Bordering ranks the planes by the number of distinct pose tiles that observe
// them: a revisited plane has a wide span but a small clique, so the span rule of the insertion order is the wrong measure here.
inline bool build_nd(const Compiled& c, DirectTables& d, std::string& err) {
  const int N = c.N, M = c.M;
  std::vector<int> ntile(M, 0), bslot;
  for (int l = 0; l < M; l++) {
    int last = -1;
    for (int i = d.inc_ptr[l]; i < d.inc_ptr[l + 1]; i++)
      if (d.inc_pose[i] / 8 != last) { last = d.inc_pose[i] / 8; ntile[l]++; }
  }
  choose_border(ntile, [&](const std::vector<int>& bs, int k) { DirectTables t; return nd_layout(c, d.inc_ptr, d.inc_pose, bs, k, t); },
                d.border, bslot);
  const int nbord = (int)d.border.size();
  d.bytes = nd_layout(c, d.inc_ptr, d.inc_pose, bslot, nbord, d);
  if (d.bytes > kBandBudgetBytes) {
    err = "band linear solver (nested-dissection order): the graph needs " + std::to_string(d.bytes) + " bytes of device memory (" +
          std::to_string(N) + " poses, " + std::to_string(nbord) + " bordered planes, " + std::to_string(d.nd_cptr[d.nb]) +
          " tiles); the budget is " + std::to_string(kBandBudgetBytes) + " bytes (use the PCG solver, kind 0)";
    return false;
  }
  for (int l : d.border) { d.binc.push_back(d.inc_ptr[l]); d.binc.push_back(d.inc_ptr[l + 1]); }
  nd_tables(d);
  // pair (a, b) lies in the stored tile t that holds it, at 64 t + 8 (a % 8) + b % 8
  pair_lists(c, bslot, (size_t)64 * d.nd_cptr[d.nb], [&](int a, int b) {
    const int i = d.nd_pos[a / 8], j = d.nd_pos[b / 8];
    return (size_t)64 * d.tile(std::max(i, j), std::min(i, j)) + 8 * (a % 8) + b % 8;
  }, d);
  return true;
}

// kind 1: dense (at most kDirectMaxPoses poses); kind 2: band, within kBandBudgetBytes, in insertion order (order 0) or
// nested-dissection order (order 1)
inline bool build_direct(const Compiled& c, DirectTables& d, std::string& err, int kind = 1, int order = 0) {
  d = DirectTables();
  const int N = c.N, M = c.M;
  if (kind == 1 && N > kDirectMaxPoses) {
    err = "direct linear solver: the graph has " + std::to_string(N) + " live poses; the dense solve handles at most " +
          std::to_string(kDirectMaxPoses) + " (use the PCG solver, kind 0)";
    return false;
  }
  d.inc_ptr.assign(M + 1, 0);
  for (int l = 0; l < M; l++) {
    for (int s = c.pl_ptr[l]; s < c.pl_ptr[l + 1];) {
      int e = s + 1;
      while (e < c.pl_ptr[l + 1] && c.pl_pose[e] == c.pl_pose[s]) e++;
      d.inc_pose.push_back(c.pl_pose[s]); d.inc_plane.push_back(l); d.inc_lo.push_back(s); d.inc_hi.push_back(e);
      s = e;
    }
    d.inc_ptr[l + 1] = (int)d.inc_pose.size();
  }
  if (kind == 2 && order == 1) {
    d.order = 1;
    if (!build_nd(c, d, err)) { d = DirectTables(); return false; }
    return true;
  }
  std::vector<int> bslot(M, -1);
  if (kind == 1) {
    d.nbp = d.nb = std::max(1, (6 * N + 47) / 48);
    d.first.assign(d.nb, 0);
  } else {   // bordering ranks the planes by observer span (pose order)
    std::vector<int> span(M, 0);
    for (int l = 0; l < M; l++)
      if (d.inc_ptr[l + 1] > d.inc_ptr[l]) span[l] = d.inc_pose[d.inc_ptr[l + 1] - 1] - d.inc_pose[d.inc_ptr[l]];
    choose_border(span, [&](const std::vector<int>& bs, int k) {
      std::vector<int> fk;
      int nbp = 0, nb = 0;
      return band_envelope(c, d.inc_ptr, d.inc_pose, bs, k, fk, nbp, nb);
    }, d.border, bslot);
    const int nbord = (int)d.border.size();
    d.bytes = band_envelope(c, d.inc_ptr, d.inc_pose, bslot, nbord, d.first, d.nbp, d.nb);
    if (d.bytes > kBandBudgetBytes) {
      err = "band linear solver: the graph needs " + std::to_string(d.bytes) + " bytes of device memory (" +
            std::to_string(N) + " poses, " + std::to_string(nbord) + " bordered planes); the budget is " +
            std::to_string(kBandBudgetBytes) + " bytes (use the PCG solver, kind 0)";
      d = DirectTables();
      return false;
    }
    for (int l : d.border) { d.binc.push_back(d.inc_ptr[l]); d.binc.push_back(d.inc_ptr[l + 1]); }
  }
  const int nb = d.nb;
  d.toff.assign(nb + 1, 0);
  for (int i = 0; i < nb; i++) d.toff[i + 1] = d.toff[i] + i - d.first[i] + 1;
  d.col_ptr.assign(nb + 1, 0);
  for (int i = 0; i < nb; i++)
    for (int K = d.first[i]; K < i; K++) d.col_ptr[K + 1]++;
  for (int K = 0; K < nb; K++) d.col_ptr[K + 1] += d.col_ptr[K];
  d.col_row.assign(std::max(1, d.col_ptr[nb]), 0);
  {
    std::vector<int> fill(d.col_ptr.begin(), d.col_ptr.end() - 1);
    for (int i = 0; i < nb; i++)
      for (int K = d.first[i]; K < i; K++) d.col_row[fill[K]++] = i;
  }
  d.poff.assign(N + 1, 0);
  for (int a = 0; a < N; a++) d.poff[a + 1] = d.poff[a] + a - 8 * d.first[a / 8] + 1;
  pair_lists(c, bslot, (size_t)d.poff[N], [&](int a, int b) { return (size_t)d.poff[a] + b - 8 * d.first[a / 8]; }, d);
  return true;
}

// ------------------------------------------------------------------------------------------------
// Marginal covariances from the nested-dissection factor (DESIGN.md section 5.4), built by the first covariance call of a
// layout.  Sigma = S^-1 is stored in the tiles of L's pattern (same storage index as L); in the new order, with
// R_j = the tile rows i > j of column j:
//   off-diagonal  Sigma_ij = -(sum_{k in R_j} Sigma_ik L_kj) L_jj^-1,     i in R_j
//   diagonal      Sigma_jj = L_jj^-T (L_jj^-1 - sum_{k in R_j} L_kj^T Sigma_kj)
// Every Sigma_ik read is a stored tile: i and k both lie in R_j, a clique of the pattern, so (max, min) is stored, and its
// column min(i, k) is an ancestor of j (a higher level).  The diagonal tile's list is its column's own tiles, in storage
// order; the off-diagonal tiles' lists are below.
// ------------------------------------------------------------------------------------------------
// the covariance tables the device reads, packed into one array (CovTables::dev): entries 0 .. 3 the offsets of the tables
enum CovTable { COV_SPTR = 0, COV_SEL, COV_PPTR, COV_PAIR, COV_HDR };

struct CovTables {
  uint64_t topo = 0;                  // layout version the tables were built for (0: none)
  std::vector<int> sel_ptr, sel;      // per stored tile (i, j), i > j: (Sigma tile (i,k) or (k,i)) * 2 + transposed, L tile (k, j),
                                      // k in R_j ascending (empty for diagonal tiles)
  std::vector<int> pair_ptr, pair;    // per eliminated plane: its observer pairs (incidences qa >= qb), 4 ints each: qa, qb,
                                      // Sigma tile, in-tile offset * 2 + transposed (the block Sigma_{pose qa, pose qb})
  std::vector<int> dev;               // the tables above that the device reads, packed (CovTable)
  long long nsel = 0;                 // list entries of the off-diagonal tiles
  long long bytes = 0;                // device memory of the Sigma tiles and these tables
};

// The stored place of the block of Sigma whose rows start at row r0 and columns at c0 (both in the bordered order: 6 N pose
// rows, then 3 per bordered plane from row 48 nbp), when its rows and columns each lie inside one tile: element (p, s) is at
// tile * kAcTile + (flag ? off + s * ld + p : off + p * ld + s) with ld = 52.  False when the tile is not stored.
inline bool cov_block_at(const DirectTables& d, int r0, int c0, int& tile, int& off, int& flag) {
  const int ti = d.nd_pos[r0 / 48], tj = d.nd_pos[c0 / 48], er = r0 % 48, ec = c0 % 48;
  tile = d.tile(std::max(ti, tj), std::min(ti, tj));
  if (tile < 0) return false;
  flag = ti < tj ? 1 : 0;
  off = flag ? ec * 52 + er : er * 52 + ec;
  return true;
}

// The first row of a node's block in the bordered order, or -1 for an eliminated plane.  `pose`: compiled pose / plane index.
inline int cov_row(const DirectTables& d, bool pose, int idx) {
  if (pose) return 6 * idx;
  const auto it = std::lower_bound(d.border.begin(), d.border.end(), idx);
  if (it == d.border.end() || *it != idx) return -1;
  return 48 * d.nbp + 3 * (int)(it - d.border.begin());
}

constexpr int kCovSelBytes = 8;   // bytes per off-diagonal list entry

// Build the covariance tables of an ND layout; false (with a message) when the Sigma tiles, these tables and the layout's own
// memory together exceed the band budget.
inline bool build_cov(const Compiled& c, const DirectTables& d, CovTables& cv, std::string& err) {
  cv = CovTables();
  const int nb = d.nb, T = d.nd_cptr[nb], M = c.M;
  cv.nsel = 0;
  for (int j = 0; j < nb; j++) { const long long m = d.nd_cptr[j + 1] - d.nd_cptr[j] - 1; cv.nsel += m * m; }
  std::vector<char> bord(M, 0);
  for (int l : d.border) bord[l] = 1;
  long long npair = 0;
  for (int l = 0; l < M; l++)
    if (!bord[l]) { const long long n = d.inc_ptr[l + 1] - d.inc_ptr[l]; npair += n * (n + 1) / 2; }
  cv.bytes = (long long)T * kDirectTileBytes + kCovSelBytes * cv.nsel + 4ll * (T + 1) + 16 * npair + 4ll * (M + 1) + 4 * COV_HDR;
  if (d.bytes + cv.bytes > kBandBudgetBytes) {
    err = "marginal covariances: the graph needs " + std::to_string(d.bytes + cv.bytes) + " bytes of device memory (" +
          std::to_string(d.bytes) + " for the factorization, " + std::to_string(cv.bytes) + " for the Sigma tiles and the selected-" +
          "inversion lists, " + std::to_string(T) + " tiles); the budget is " + std::to_string(kBandBudgetBytes) + " bytes";
    cv = CovTables();
    return false;
  }
  cv.sel_ptr.assign(T + 1, 0);
  cv.sel.reserve(2 * cv.nsel);
  for (int t = 0; t < T; t++) {   // storage order
    const int i = d.nd_trow[t], j = d.nd_tcol[t];
    if (i != j) {
      for (int p = d.nd_cptr[j] + 1; p < d.nd_cptr[j + 1]; p++) {
        const int k = d.nd_crow[p];
        cv.sel.push_back(2 * d.tile(std::max(i, k), std::min(i, k)) + (i < k ? 1 : 0));
        cv.sel.push_back(d.nd_toff[j] + p - d.nd_cptr[j]);
      }
    }
    cv.sel_ptr[t + 1] = (int)(cv.sel.size() / 2);
  }
  cv.pair_ptr.assign(M + 1, 0);
  for (int l = 0; l < M; l++) {
    if (!bord[l])
      for (int qa = d.inc_ptr[l]; qa < d.inc_ptr[l + 1]; qa++)
        for (int qb = d.inc_ptr[l]; qb <= qa; qb++) {
          int tile = 0, off = 0, flag = 0;
          if (!cov_block_at(d, 6 * d.inc_pose[qa], 6 * d.inc_pose[qb], tile, off, flag)) {   // (eliminating l coupled them)
            err = "marginal covariances: internal error: an observer pair of an eliminated plane lies outside L's pattern";
            cv = CovTables();
            return false;
          }
          cv.pair.insert(cv.pair.end(), {qa, qb, tile, 2 * off + flag});
        }
    cv.pair_ptr[l + 1] = (int)(cv.pair.size() / 4);
  }
  const std::vector<int>* tab[COV_HDR] = {&cv.sel_ptr, &cv.sel, &cv.pair_ptr, &cv.pair};
  cv.dev.assign(COV_HDR, 0);
  for (int k = 0; k < COV_HDR; k++) {
    cv.dev[k] = (int)cv.dev.size();
    cv.dev.insert(cv.dev.end(), tab[k]->begin(), tab[k]->end());
  }
  return true;
}

}  // namespace pus
