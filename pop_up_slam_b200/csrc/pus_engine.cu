// pus_engine.cu -- persistent LM kernel entry, host-side engine (HBM layout, upload / solve /
// download) and the extern "C" entry points declared in include/popup_gpu.h.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC ...
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"
#include "pus_export.cuh"
#include "pus_graph.hpp"
#include "pus_stages.cuh"

namespace pus {
// the device code is instantiated twice: kplain (here) = the single-GPU kernel, spanning hooks compiled out; kspan
// (pus_span.cu) = one graph spanning ranks.  Both define the same types with the same layout; the host uses kplain's.
namespace kplain {
#define PUS_NO_SPAN 1
#include "pus_kernels.cuh"
#include "pus_driver.cuh"
#undef PUS_NO_SPAN
}  // namespace kplain
using namespace kplain;
// the second instantiation (pus::kspan, spanning hooks compiled in) lives in pus_span.cu
void* span_kernel_ptr();
size_t span_devgraph_bytes();
cudaError_t span_kernel_prepare();
// the third (pus::kdirect, pus_direct.cu): the kernel of handles in direct linear-solver mode
void* direct_kernel_ptr();
size_t direct_devgraph_bytes();
cudaError_t direct_kernel_prepare();

// ---------------------------------------------------------------------------------------------
// host engine
// ---------------------------------------------------------------------------------------------
thread_local std::string g_err;

#define CUDA_OK(call)                                                                      \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e__);                         \
      return -1;                                                                           \
    }                                                                                      \
  } while (0)

struct Solver {
  int device = 0;
  Graph g;
  pus_properties prop;
  int robust_kind = 0;
  double robust_b = 1.0;
  int jac_numeric = 0;
  int linear_solver = 0;       // 0: PCG, 1: exact dense Cholesky of the reduced pose system, 2: exact band Cholesky (pus_set_linear_solver)
  int ordering = 0;            // kind 2: 0 insertion order, 1 nested dissection (pus_set_direct_ordering)
  pus_solver_options opt;
  Compiled c;
  DirectTables dt;             // (direct mode only)
  uint64_t compiled_topo = 0;
  bool meas_dirty = true;
  int span_w = 1, span_r = 0;  // one graph spanning ranks: world / rank and the peers' arenas (CUDA IPC mappings)
  std::vector<void*> span_peers;
  uint64_t span_topo = 0;
  double* arena = nullptr;     // mirror arena of the last upload (DevGraph::gbar + the PCG vectors)
  size_t arena_bytes = 0;
  void* scratch = nullptr;     // grow-only device scratch of the refresh / projection entry points
  size_t scratch_bytes = 0;
  std::vector<int> fid2slot;   // pose-plane factor id -> pose-major edge slot (built on demand)
  uint64_t fid2slot_topo = 0;
  bool uploaded = false;
  int step = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaStream_t saved_stream = nullptr;   // this handle's own stream while it rides on a batch's stream (adopt_stream / release_stream)
  bool saved_own = false, borrowing = false;
  int borrow_depth = 0;
  bool values_dirty = false;             // host values changed since the last upload (pus_init_*): device copies are stale
  DevGraph* d_batch = nullptr;           // parameter blocks of a batched launch (grow-only)
  LmResult* d_batch_res = nullptr;       // results of a batched launch, contiguous: ONE device->host copy per batch
  int d_batch_cap = 0;
  // resident tables of pus_refresh_bind / pus_refresh_run (frames' ground segments, invK, factor <-> plane-row map)
  struct RefreshTables {
    bool bound = false;
    int n_frames = 0, n_seg = 0, n_rows = 0, n_map = 0;
    int cap_frames = 0, cap_seg = 0, cap_map = 0;  // room of the carved sections (a plane map appends into them)
    const void* owner = nullptr;                  // the plane map that appends to these tables; nullptr after pus_refresh_bind
    std::vector<int> frame_node, map_fid, mrow;   // host copies: pose node id per frame, factor id and plane row per map entry
    uint64_t slot_topo = 0;                       // layout version the device slot / pose-index tables were built for
    void* mem = nullptr; size_t bytes = 0;        // one allocation carved into the pointers below
    int *d_fpose = nullptr, *d_ptr = nullptr, *d_rf = nullptr, *d_mrow = nullptr, *d_mslot = nullptr;
    float *d_segs = nullptr, *d_K = nullptr, *d_T = nullptr, *d_ps = nullptr;
    double* d_out = nullptr;
  } rt;
  bool meas_device_newer = false;        // pus_refresh_run(h, NULL) left newer pose-plane measurements on the device than in the host mirrors
  // per-layout tables of the error / Jacobian export (pus_export.cuh), built by the first export after a layout rebuild
  struct ExportTables {
    uint64_t topo = 0;                    // compiled_topo they were built for (0: none)
    long long rows = 0, cols = 0, nnz = 0;
    std::vector<ExportRec> rec;           // per record of the layout
    std::vector<int> fid2rec;             // factor id -> record, -1 dead
    std::vector<int> live_row;            // first row of the k-th live factor (factor order), then the total row count
    void* mem = nullptr; size_t bytes = 0;   // device: rec, row_ptr [rows + 1], col_idx [nnz]
    ExportRec* d_rec = nullptr;
    int *d_row_ptr = nullptr, *d_col_idx = nullptr;
    bool structure = false;               // d_row_ptr / d_col_idx filled for this layout
    cudaEvent_t ev_copy = nullptr;        // recorded after an export's device-to-host copies
  } xt;
  // marginal covariances (pus_marginal_covariances / pus_covariance_blocks; kind 2 in ND order only): the tables of the layout,
  // built by its first covariance call, and Sigma on the device, valid until the next launch, upload or change of the
  // linearisation (any of them sets valid = false)
  struct CovState {
    CovTables t;
    bool valid = false;
    void* mem = nullptr; size_t bytes = 0;   // device: Sigma tiles, then the packed tables
  } cov;
  std::map<std::string, std::pair<double*, size_t>> named;  // debug access to double buffers
  DevGraph hd;
  DevGraph* d_graph = nullptr;
  LmResult* d_res = nullptr;
  LmTrace* d_trace = nullptr;
  unsigned* d_bar = nullptr;
  LmResult res;
  int path[5] = {0, 0, 0, 0, 0};   // the last debug launch's path report (PathBit flags, team size, levels, SP, owned blocks)
  LmTrace trace;
  pus_stats stats;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int num_sms = 0;

  Solver() {
    std::memset(&prop, 0, sizeof(prop));
    prop.method = 0; prop.epsilon2 = 1e-2; prop.epsilon_abs = 1e-3; prop.epsilon_rel = 1e-5; prop.max_iterations = 500;
    prop.lm_lambda0 = 1e-6; prop.lm_lambda_factor = 10.; prop.mod_update = 1; prop.mod_batch = 100; prop.mod_solve = 1;
    std::memset(&opt, 0, sizeof(opt));
    opt.pcg_rel_tol = 1e-8; opt.pcg_max_iter = 2000;   // 4 decades under the 1e-4 parity bar (DESIGN.md)
    std::memset(&stats, 0, sizeof(stats));
    std::memset(&res, 0, sizeof(res));
    std::memset(&hd, 0, sizeof(hd));
    trace_n = 0;
  }
  int trace_n;

  // Device buffers are recycled across topology changes: the n-th allocation of a rebuild re-uses the n-th buffer of
  // the previous one when it is large enough (grown by 1.5x otherwise), so the frame-by-frame use of the reference
  // (one structural edit per key-frame, Mapping.cpp:464-554) does not pay ~70 cudaFree + cudaMalloc per frame.
  struct Slot { void* p; size_t cap; };
  std::vector<Slot> pool;
  size_t pool_next = 0;
  void free_device() {
    for (Slot& sl : pool) cudaFree(sl.p);
    pool.clear();
    recycle_device();
  }
  void recycle_device() {
    pool_next = 0;
    named.clear();
    uploaded = false;
    compiled_topo = 0;
  }
  template <typename T>
  int dalloc(T** out, size_t n, const char* name = nullptr) {
    const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
    if (pool_next == pool.size()) {
      void* p = nullptr;
      CUDA_OK(cudaMalloc(&p, bytes));
      pool.push_back(Slot{p, bytes});
    } else if (pool[pool_next].cap < bytes) {
      cudaFree(pool[pool_next].p);
      pool[pool_next].p = nullptr; pool[pool_next].cap = 0;
      const size_t cap = bytes + bytes / 2;
      void* p = nullptr;
      CUDA_OK(cudaMalloc(&p, cap));
      pool[pool_next] = Slot{p, cap};
    }
    void* p = pool[pool_next++].p;
    *out = reinterpret_cast<T*>(p);
    if (name) named[name] = std::make_pair(reinterpret_cast<double*>(p), n);
    return 0;
  }
  template <typename T>
  int dupload(const T** out, const std::vector<T>& v, long long* bytes) {
    T* p = nullptr;
    if (dalloc(&p, v.size()) < 0) return -1;
    if (!v.empty()) CUDA_OK(cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream));
    *bytes += (long long)(v.size() * sizeof(T));
    *out = p;
    return 0;
  }
};

static int ensure_device(Solver* s) {
  int ndev = 0;
  cudaError_t de = cudaGetDeviceCount(&ndev);
  if (de != cudaSuccess || ndev <= 0) {
    g_err = std::string("no CUDA device available (") + cudaGetErrorString(de) + "); libpopup_gpu has no CPU fallback";
    return -1;
  }
  if (s->device >= ndev) { g_err = "bad device ordinal"; return -1; }
  CUDA_OK(cudaSetDevice(s->device));
  if (!s->stream && !s->own_stream) {
    CUDA_OK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    s->own_stream = true;
  }
  if (!s->ev0) { CUDA_OK(cudaEventCreate(&s->ev0)); CUDA_OK(cudaEventCreate(&s->ev1)); }
  if (!s->num_sms) {
    cudaDeviceProp p;
    CUDA_OK(cudaGetDeviceProperties(&p, s->device));
    s->num_sms = p.multiProcessorCount;
    CUDA_OK(cudaFuncSetAttribute(kplain::lm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    CUDA_OK(span_kernel_prepare());
    CUDA_OK(direct_kernel_prepare());
    if (span_devgraph_bytes() != sizeof(DevGraph) || direct_devgraph_bytes() != sizeof(DevGraph)) {
      g_err = "device-code instantiations disagree on the DevGraph layout";
      return -1;
    }
  }
  return 0;
}

// pose-plane measurements refreshed on the device (pus_refresh_run without a host buffer) -> host factor store + compiled copy
static int sync_measurements_to_host(Solver* s) {
  if (!s->meas_device_newer) return 0;
  s->meas_device_newer = false;
  if (!s->uploaded || s->compiled_topo == 0) return 0;
  Compiled& c = s->c;
  if (!c.nslot) return 0;
  CUDA_OK(cudaSetDevice(s->device));
  CUDA_OK(cudaMemcpyAsync(c.pp_meas.data(), s->hd.pp_meas, c.pp_meas.size() * 8, cudaMemcpyDeviceToHost, s->stream));
  CUDA_OK(cudaStreamSynchronize(s->stream));
  for (int e = 0; e < c.nslot; e++)
    if (c.pp_fid[e] >= 0) std::memcpy(s->g.factors[c.pp_fid[e]].meas, &c.pp_meas[(size_t)e * 4], 4 * sizeof(double));
  return 0;
}

// (re)build the HBM image of the graph.  Topology arrays are re-uploaded only after a structural edit;
// vertex values always; measurements when pus_set_measurement touched them.
static int upload(Solver* s) {
  s->cov.valid = false;
  if (ensure_device(s) < 0) return -1;
  cudaEvent_t e0 = s->ev0, e1 = s->ev1;
  long long bytes = 0;
  CUDA_OK(cudaEventRecord(e0, s->stream));
  {   // preconditioner levels: by graph size, or forced through pus_solver_options.reserved[2] (bit 3: three, bit 4: two)
    const int want = (s->opt.reserved[2] & 8) ? 3 : ((s->opt.reserved[2] & 16) ? 2 : 0);
    if (want != s->g.force_levels) { s->g.force_levels = want; s->g.topo_version++; }
  }
  const bool rebuild = (s->compiled_topo != s->g.topo_version) || !s->uploaded;
  if ((rebuild || s->meas_dirty) && s->meas_device_newer && sync_measurements_to_host(s) < 0) return -1;   // (the layout is rebuilt from the host store)
  if (rebuild) {
    s->recycle_device();
    std::string err;
    if (!compile_graph(s->g, s->c, err)) { g_err = err; return -1; }
    if (s->linear_solver != 0 && !build_direct(s->c, s->dt, err, s->linear_solver, s->ordering)) { g_err = err; return -1; }
    const Compiled& c = s->c;
    if (kSmRc + 6 * c.nc * 8 > kSmemBytes) { g_err = "graph too large for the coarse-space shared-memory buffer"; return -1; }
    DevGraph& d = s->hd;
    std::memset(&d, 0, sizeof(d));
    d.N = c.N; d.M = c.M; d.Epl = c.Epl; d.Epf = c.Epf; d.Elp = c.Elp; d.ntile = c.ntile; d.ntile_pl = c.ntile_pl; d.nslot = c.nslot;
    d.nblk = c.nblk; d.nc = c.nc;
    d.SP = c.SP; d.inv_SP = 1.0 / (double)c.SP; d.ldmc = 6 * c.nc_pad; d.n_upart = c.n_upart; d.n_ypart = c.n_ypart; d.nce = c.nce; d.ngrp = c.ngrp;
#define UP(field) if (s->dupload(&d.field, c.field, &bytes) < 0) return -1
    UP(pp_pose); UP(pp_plane); UP(pp_ptr); UP(pp_end); UP(pm2pl); UP(pm_part); UP(ypart_ptr); UP(tile_ptr); UP(blk_part_ptr);
    UP(grp_of_slot); UP(pp_meas); UP(pp_sinf); UP(pp_rays); UP(pp_kind);
    d.n_f2 = c.n_f2;
    UP(pl2pm); UP(pl_ptr); UP(pl_plane); UP(pl_pose); UP(pl_part); UP(upart_ptr); UP(heavy); UP(huge);
    d.n_heavy = c.n_heavy; d.n_huge = c.n_huge;
    UP(pf_i); UP(pf_j); UP(pinc_ptr); UP(pinc); UP(pnbr); UP(pf_meas); UP(pf_sinf);
    UP(lp_plane); UP(linc_ptr); UP(linc); UP(lp_meas); UP(lp_sinf);
    UP(blk_grp_ptr); UP(grp_plane); UP(grp_mem_ptr); UP(grp_mem); UP(blk_simple); UP(grp_info); UP(grp_info2); UP(at_plane); UP(at_lo); UP(at_hi); UP(at_ptr); UP(as_plane);
    d.n_atask = c.n_atask; d.n_asplit = c.n_asplit;
    d.res_nt = c.res_nt; d.res_ng = c.res_ng; d.res_np = c.res_np;
    UP(blk_ovf); d.n_ovf_blk = c.n_ovf_blk;
    UP(ce_ptr); UP(ce_node); UP(ce_plane); UP(ce_lo); UP(ce_hi); UP(n2ce_ptr); UP(n2ce);
    UP(hv_plane); UP(lp_ptr); UP(lp_cea); UP(lp_ceb); UP(fp_ptr); UP(fp_f);
    d.n_hv = c.n_hv;
    UP(ce2_node); UP(ce2_plane); UP(ce2_lo); UP(ce2_hi); UP(g2_ptr); UP(g2_ce);
    d.levels = c.levels; d.nc2 = c.nc2; d.nce2 = c.nce2; d.ng2 = c.ng2;
#undef UP
    const size_t N = c.N, M = c.M, E = c.nslot, T = c.ntile, TL = c.ntile_pl;
#define AL(field, n, name) if (s->dalloc(&d.field, (size_t)(n), name) < 0) return -1
    AL(pose_lin, N * 7, "pose_lin"); AL(pose_trial, N * 7, "pose_trial"); AL(pose_init, N * 7, "pose_init");
    AL(plane_lin, M * 4, "plane_lin"); AL(plane_trial, M * 4, "plane_trial"); AL(plane_init, M * 4, "plane_init");
    AL(W, T * kWStride, "Wtiles"); AL(Wt, TL * kWStride, "Wttiles"); AL(JP, E * 21, "JP"); AL(JL, E * 12, "JL");
    AL(PF, (size_t)c.Epf * 120, "PF"); AL(LP, (size_t)c.Elp * 12, "LP");
    AL(Hpp, N * 36, "Hpp"); AL(gp, N * 6, "gp"); AL(Hll, M * 9, "Hll"); AL(gl, M * 3, "gl"); AL(Hinv, M * 9, "Hinv");
    AL(ypart, 8, "ypart"); AL(upartb, (size_t)std::max(1, c.ngrp) * 3, "upartb"); AL(hpart, (size_t)std::max(1, c.n_atask) * 9, "hpart");
    AL(ovf, c.n_ovf, "ovf");
    AL(Binv, (size_t)c.nblk * kPackedBlock, "Binv"); AL(Wc, (size_t)c.nce * 18, "Wc"); AL(Yc, (size_t)c.nce * 18, "Yc");
    AL(Ac, ac_elems(6 * c.nc_pad), nullptr); AL(Atri, ac_tri_doubles(6 * c.nc_pad), "Atri"); AL(Apan, ac_panel_doubles(6 * c.nc_pad), "Apan");
    AL(Wc2, (size_t)c.nce2 * 18, "Wc2"); AL(Yc2, (size_t)c.nce2 * 18, "Yc2"); AL(D2inv, (size_t)c.ng2 * kBlockDim * kBlockDim, "D2inv");
    {
      // The vectors the PCG phases exchange live in ONE allocation (the "mirror arena"): when one graph spans several
      // ranks every rank lays it out identically, so a peer's copy of any element is at a fixed byte offset.
      struct Item { double** p; size_t n; const char* name; };
      const Item items[] = {
          {&d.vl, M * 3, "vl"}, {&d.dl, M * 3, "dl"}, {&d.upart, (size_t)c.n_upart * 3, "upart"},
          {&d.x, N * 6, "x"}, {&d.r, N * 6, "r"}, {&d.z, N * 6, "z"}, {&d.q, N * 6, "q"},
          {&d.b, N * 6 + (s->linear_solver == 2 ? 3 * s->dt.border.size() : 0), "b"},   // (band solve: then 3 per bordered plane)
          {&d.pv[0], N * 6, "pv0"}, {&d.pv[1], N * 6, "pv1"}, {&d.xprev, N * 6, "xprev"}, {&d.zc, (size_t)6 * c.nc, "zc"},
          {&d.zc2, (size_t)6 * c.nc2, "zc2"}, {&d.rc3, (size_t)6 * c.nc, "rc3"},
          {&d.rcpart[0], (size_t)c.nblk * 12, "rcpart0"}, {&d.rcpart[1], (size_t)c.nblk * 12, "rcpart1"},
          {&d.qcpart, (size_t)c.nblk * 12, "qcpart"}, {&d.red, (size_t)4 * 4 * 2048, "red"}};
      size_t total = 32;   // first 256 bytes: the cross-rank barrier counter and its persisted target
      for (const Item& it : items) total += (std::max<size_t>(it.n, 1) + 31) / 32 * 32;
      double* arena = nullptr;
      if (s->dalloc(&arena, total) < 0) return -1;
      CUDA_OK(cudaMemsetAsync(arena, 0, 256, s->stream));
      s->arena = arena; s->arena_bytes = total * sizeof(double);
      d.gbar = reinterpret_cast<unsigned*>(arena);
      size_t off = 32;
      for (const Item& it : items) {
        *it.p = arena + off;
        s->named[it.name] = std::make_pair(arena + off, it.n);
        off += (std::max<size_t>(it.n, 1) + 31) / 32 * 32;
      }
      d.span_w = 1; d.span_r = 0;
    }
    if (s->linear_solver != 0) {   // the direct solve's tables and its tile store (dense: about 65 MB at the 640-pose cap)
      static_assert(kDirectTileBytes == kAcTile * 8, "band byte count: tile size");
      const DirectTables& dt = s->dt;
      const size_t nb = dt.nb, ninc = dt.inc_pose.size();
      d.dnb = dt.nb; d.dninc = (int)ninc; d.dnbp = dt.nbp; d.dnbord = (int)dt.border.size();
#define UPD(field, vec) if (s->dupload(&d.field, vec, &bytes) < 0) return -1
      UPD(dinc_plane, dt.inc_plane); UPD(dinc_lo, dt.inc_lo); UPD(dinc_hi, dt.inc_hi);
      UPD(dlp_ptr, dt.lp_ptr); UPD(dlp_a, dt.lp_a); UPD(dlp_b, dt.lp_b); UPD(dfp_ptr, dt.fp_ptr); UPD(dfp_f, dt.fp_f);
      UPD(dfirst, dt.first); UPD(dtoff, dt.toff); UPD(dpoff, dt.poff); UPD(dcol_ptr, dt.col_ptr); UPD(dcol_row, dt.col_row);
      UPD(dbord, dt.border); UPD(dbinc, dt.binc);
      if (dt.order == 1) UPD(dnd, dt.nd_dev);
#undef UPD
      AL(Wd, ninc * 18, "Wd"); AL(Yd, ninc * 18, "Yd");
      AL(Sd, (size_t)dt.ntile() * kAcTile, nullptr); AL(Dsnap, dt.order == 1 ? 1 : 2 * nb * kAcTile, nullptr); AL(Dinv, nb * kAcTile, nullptr);
      AL(dvec, 2 * 48 * nb, nullptr);
      if (s->dalloc(&d.dflag, 1) < 0) return -1;
    }
#undef AL
    CUDA_OK(cudaMemsetAsync(d.W, 0, T * kWStride * sizeof(double), s->stream));
    CUDA_OK(cudaMemsetAsync(d.Wt, 0, TL * kWStride * sizeof(double), s->stream));
    if (s->dalloc(&s->d_graph, 1) < 0 || s->dalloc(&s->d_res, 1) < 0 || s->dalloc(&s->d_trace, 1) < 0 ||
        s->dalloc(&s->d_bar, 32 * 1024) < 0)
      return -1;
    d.res = s->d_res; d.trace = s->d_trace;
    s->compiled_topo = s->g.topo_version;
    s->meas_dirty = false;
  } else {
    // values / measurements only
    Compiled& c = s->c;
    for (int p = 0; p < c.N; p++) std::memcpy(&c.pose_val[(size_t)p * 7], s->g.nodes[c.pose_node[p]].v, 7 * sizeof(double));
    for (int l = 0; l < c.M; l++) std::memcpy(&c.plane_val[(size_t)l * 4], s->g.nodes[c.plane_node[l]].v, 4 * sizeof(double));
    if (s->meas_dirty) {
      for (int e = 0; e < c.nslot; e++) if (c.pp_fid[e] >= 0) std::memcpy(&c.pp_meas[(size_t)e * 4], s->g.factors[c.pp_fid[e]].meas, 4 * sizeof(double));
      for (int f = 0; f < c.Epf; f++) std::memcpy(&c.pf_meas[(size_t)f * 6], s->g.factors[c.pf_fid[f]].meas, 6 * sizeof(double));
      for (int f = 0; f < c.Elp; f++) std::memcpy(&c.lp_meas[(size_t)f * 4], s->g.factors[c.lp_fid[f]].meas, 4 * sizeof(double));
      if (c.nslot) CUDA_OK(cudaMemcpyAsync(const_cast<double*>(s->hd.pp_meas), c.pp_meas.data(), c.pp_meas.size() * 8, cudaMemcpyHostToDevice, s->stream));
      if (c.Epf) CUDA_OK(cudaMemcpyAsync(const_cast<double*>(s->hd.pf_meas), c.pf_meas.data(), c.pf_meas.size() * 8, cudaMemcpyHostToDevice, s->stream));
      if (c.Elp) CUDA_OK(cudaMemcpyAsync(const_cast<double*>(s->hd.lp_meas), c.lp_meas.data(), c.lp_meas.size() * 8, cudaMemcpyHostToDevice, s->stream));
      bytes += (long long)(c.pp_meas.size() + c.pf_meas.size() + c.lp_meas.size()) * 8;
      s->meas_dirty = false;
    }
  }
  const Compiled& c = s->c;
  if (c.N) {
    CUDA_OK(cudaMemcpyAsync(s->hd.pose_init, c.pose_val.data(), c.pose_val.size() * 8, cudaMemcpyHostToDevice, s->stream));
    CUDA_OK(cudaMemcpyAsync(s->hd.pose_lin, s->hd.pose_init, c.pose_val.size() * 8, cudaMemcpyDeviceToDevice, s->stream));
  }
  if (c.M) {
    CUDA_OK(cudaMemcpyAsync(s->hd.plane_init, c.plane_val.data(), c.plane_val.size() * 8, cudaMemcpyHostToDevice, s->stream));
    CUDA_OK(cudaMemcpyAsync(s->hd.plane_lin, s->hd.plane_init, c.plane_val.size() * 8, cudaMemcpyDeviceToDevice, s->stream));
  }
  bytes += (long long)(c.pose_val.size() + c.plane_val.size()) * 8;
  CUDA_OK(cudaEventRecord(e1, s->stream));
  CUDA_OK(cudaEventSynchronize(e1));
  float ms = 0;
  CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  s->stats.h2d_ms = ms;
  s->stats.h2d_bytes = bytes;
  s->uploaded = true;
  s->values_dirty = false;
  return 0;
}

static void fill_params(Solver* s, LmParams& p, int mode, int restore_init, int debug_stage, double debug_lambda) {
  p.method = s->prop.method; p.eps2 = s->prop.epsilon2; p.eps_abs = s->prop.epsilon_abs; p.eps_rel = s->prop.epsilon_rel;
  p.max_iter = s->prop.max_iterations; p.lambda0 = s->prop.lm_lambda0; p.lambda_factor = s->prop.lm_lambda_factor;
  p.robust_kind = s->robust_kind; p.robust_b = s->robust_b; p.jac_numeric = s->jac_numeric;
  p.pcg_tol = s->opt.pcg_rel_tol; p.pcg_max_iter = s->opt.pcg_max_iter;
  p.prec_refresh = s->opt.reserved[0] == 1 ? 0 : 1;
  p.blocks_always = s->opt.reserved[0] == 2 ? 1 : 0;
  // rebuild when its > pct% of the post-build count + add.  The dense coarse inverse goes stale mostly through lambda (four
  // rejected steps in a row move it from 1e-6 to 1e-2): 130 % for two-level graphs such as config 3; the three-level set-up of
  // large graphs is dearer per build and wants 200 % (tools/refresh_sweep.py re-measures both)
  p.refresh_pct = s->opt.reserved[3] > 0 ? s->opt.reserved[3] : (s->c.levels == 3 ? 200 : 130);
  p.refresh_add = 8;
  p.fine_timers = (s->opt.reserved[2] & 64) ? 2 : ((s->opt.reserved[2] & 1) ? 1 : 0);   // bit 6: sub-phases of linearize instead     // reserved[2] bit 0: sub-phase timers inside the PCG phases
  p.timer_rank = (s->opt.reserved[2] >> 8) & 0xff;   // bits 8-15: the CTA that keeps the phase timers
  p.tma_mode = (s->opt.reserved[2] & 2) ? 1 : ((s->opt.reserved[2] & 4) ? 2 : 0);  // bit 1: always stage tiles by TMA, bit 2: never
  p.warm_start = s->opt.reserved[1] == 1 ? 0 : 1;      // reserved[1] = 1: never warm-start PCG after a rejected step  // reserved[0] = 1: rebuild the preconditioner every solve
  p.mode = mode; p.debug_stage = debug_stage; p.debug_lambda = debug_lambda; p.restore_init = restore_init;
}

// block-resident PCG loop: two levels with one hat node per pose block, every CTA's owned blocks in one round, and the per-CTA
// layout (W tiles + packed preconditioner block + records per owned block) within the shared memory of an SM.  Graphs with a
// pose block over the shared-memory limits of the general loop's pose phase (kMaxGrp / kMaxPart) run in the general loop.
static bool resident_fits(const Compiled& cc, int team) {
  const int nown = (cc.nblk + team - 1) / team;
  return cc.levels == 2 && cc.SP == kBlockPoses && cc.n_ovf_blk == 0 && nown >= 1 && nown <= kSlots && cc.res_ng <= 511 && cc.res_np <= 8191 &&
         res_layout(cc.res_nt, cc.res_ng, cc.res_np, 6 * cc.nc, nown).total <= (size_t)kSmemBytes;
}

static int auto_team(const Solver* s, int limit) {
  if (s->opt.team_ctas > 0) return std::min(std::max(1, s->opt.team_ctas), limit);
  int need = std::max((s->c.ntile + kWarps - 1) / kWarps, (s->c.nblk + kSlots - 1) / kSlots);
  need = std::max(need, (6 * s->c.nc + kWarps - 1) / kWarps);  // one warp per row of the coarse inverse
  need = std::max(need, (6 * s->c.nc_pad + 15) / 16);           // about 16 rows of A_c per CTA: a few tiles each in its inversion
  // a CTA per 16-pose block when the device has room: the phases of the PCG loop are latency-bound, so fewer owned blocks per
  // CTA shorten every phase
  if (s->c.nblk <= limit) return std::min(std::max(std::max(need, s->c.nblk), 1), limit);
  if (need * 2 > limit) need = limit;   // a graph that wants most of the device gets all of it (one CTA on every SM)
  return std::min(std::max(need, 1), limit);
}

// launch the persistent kernel over `n` solvers (all on the device / stream of the first)
static int launch(Solver** ss, int n, int mode, int restore_init, int debug_stage, double debug_lambda) {
  Solver* s0 = ss[0];
  if (mode != MODE_COV)
    for (int i = 0; i < n; i++) ss[i]->cov.valid = false;   // (a solve or a debug stage overwrites the factor)
  if (ensure_device(s0) < 0) return -1;
  for (int i = 0; i < n; i++) {
    if (!ss[i]->uploaded) { g_err = "graph not uploaded"; return -1; }
    if (ss[i]->device != s0->device) { g_err = "all graphs of a batch must live on one device"; return -1; }
  }
  const bool direct = s0->linear_solver != 0;   // dense and band handles share the direct solve's kernel
  for (int i = 0; i < n; i++)
    if ((ss[i]->linear_solver != 0) != direct) { g_err = "one launch cannot mix direct and PCG handles"; return -1; }
  void* const kern = direct ? direct_kernel_ptr() : (void*)kplain::lm_kernel;
  int per_sm = 0;
  CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, kSmemBytes));
  if (per_sm < 1) { g_err = "lm_kernel does not fit on an SM"; return -1; }
  const int max_ctas = s0->num_sms * 1;
  int team = 1, grid = 1;
  if (n == 1) {
    team = auto_team(s0, max_ctas);
    grid = team;
  } else {
    int share = std::max(1, max_ctas / n);
    int need = 1;
    for (int i = 0; i < n; i++) need = std::max(need, auto_team(ss[i], max_ctas));
    team = std::min(share, need);
    // Several waves of larger teams can beat one wave of small ones: the block-resident PCG loop only fits when a CTA owns few
    // pose blocks, and the general loop is 2-3 times slower per solve.  Cost model fitted on the solve times of TUM-scale graphs
    // (19 blocks; the general loop's cost grows with the number of rounds over kSlots blocks), used as a ratio only:
    // cost(t) = waves(t) * (resident ? 3.0 + 0.2 b : 4.3 + 4.2 ceil(b / kSlots)), b = blocks per CTA.  So 32 graphs run as two
    // waves of sixteen 9-CTA teams rather than one wave of 4-CTA teams, and 64 graphs keep 2-CTA teams.
    bool forced = false;
    for (int i = 0; i < n; i++) forced = forced || ss[i]->opt.team_ctas > 0 || ss[i]->hd.span_w > 1;
    if (!forced) {
      double best = 1e300;
      int best_t = team;
      for (int t = 1; t <= std::min(need, max_ctas); t++) {
        const int teams_t = std::min(n, max_ctas / t), waves = (n + teams_t - 1) / teams_t;
        double worst = 0;
        for (int i = 0; i < n; i++) {
          const Compiled& cc = ss[i]->c;
          const int b = (cc.nblk + t - 1) / t;
          const bool res = resident_fits(cc, t) && !(ss[i]->opt.reserved[2] & 32);
          worst = std::max(worst, res ? 3.0 + 0.2 * b : 4.3 + 4.2 * ((b + kSlots - 1) / kSlots));
        }
        const double cost = waves * worst;
        if (cost <= best) { best = cost; best_t = t; }   // (ties: the larger team)
      }
      team = best_t;
    }
    int teams = std::min(n, max_ctas / team);
    grid = teams * team;
  }
  // Small teams run as ONE thread-block cluster (cluster barrier / DSMEM mbarriers and reductions instead of the global-memory
  // barrier).  Cluster sizes 2, 4, 8, 16 (16 = the non-portable size; PUS_CLUSTER caps it, 0 = off).  A team whose natural size
  // is one of those becomes a cluster as it is; a single small graph that would get a CTA per pose block is cut down to the
  // largest such size when every CTA then owns at most two blocks (config 2, 19 blocks: one 16-CTA cluster rather than 19 CTAs
  // with the global barrier).  Batches whose teams would not all be resident as clusters keep the global barrier (8 graphs:
  // 18-CTA teams rather than fewer, smaller resident clusters).  Which cluster sizes fit is asked of the device
  // (cudaOccupancyMaxActiveClusters), so the choice follows the SM count per GPC of the part.
  bool spanning = false;
  for (int i = 0; i < n; i++) spanning = spanning || (ss[i]->hd.span_w > 1);
  int use_cluster = 0;
  {
    static const int max_cluster = [] { const char* e = getenv("PUS_CLUSTER"); int v = e ? atoi(e) : 16; return v < 0 ? 0 : (v > 16 ? 16 : v); }();
    bool off = false;
    for (int i = 0; i < n; i++) off = off || (ss[i]->opt.reserved[2] & (1 << 16));   // reserved[2] bit 16: global-memory barrier only
    if (!spanning && !off && max_cluster > 1 && team > 1) {
      int cl = 2;
      while (cl * 2 <= std::min(team, max_cluster)) cl *= 2;
      int t = 0;
      if (cl == team) t = cl;
      else if (n == 1 && s0->opt.team_ctas <= 0 && s0->c.levels == 2 && s0->c.nblk <= 2 * cl) t = cl;
      if (t > 1) {
        if (t > 8) cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        const int teams = (n == 1) ? 1 : std::min(n, max_ctas / t);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(teams * t); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmemBytes; cfg.stream = s0->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = t; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        // per kernel and cluster size (one device type per process)
        static int active_cache[2][17] = {{-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
                                          {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1}};
        int active = active_cache[direct][t];
        if (active < 0) {
          active = 0;
          if (cudaOccupancyMaxActiveClusters(&active, kern, &cfg) != cudaSuccess) { active = 0; cudaGetLastError(); }
          active_cache[direct][t] = active;
        }
        if (active >= teams) {
          team = t; grid = teams * t; use_cluster = 1;
        } else {
          cudaGetLastError();
        }
      }
    }
  }
  // per-graph parameter blocks
  std::vector<DevGraph> hg(n);
  for (int i = 0; i < n; i++) {
    fill_params(ss[i], ss[i]->hd.prm, mode, restore_init, debug_stage, debug_lambda);
    {
      // block-resident PCG loop: two levels with one hat node per pose block, every CTA's owned blocks in one round, and the
      // per-CTA layout (W tiles + packed preconditioner block + records per owned block) within the shared memory of an SM
      const bool fits = resident_fits(ss[i]->c, team);
      ss[i]->hd.prm.resident = (fits && !(ss[i]->opt.reserved[2] & 32) && ss[i]->hd.span_w <= 1) ? 1 : 0;   // reserved[2] bit 5: off
    }
    hg[i] = ss[i]->hd;
  }
  DevGraph* d_graphs = s0->d_graph;
  if (n > 1) {
    if (s0->d_batch_cap < n) {
      if (s0->d_batch) cudaFree(s0->d_batch);
      if (s0->d_batch_res) cudaFree(s0->d_batch_res);
      s0->d_batch = nullptr; s0->d_batch_res = nullptr; s0->d_batch_cap = 0;
      CUDA_OK(cudaMalloc(&s0->d_batch, sizeof(DevGraph) * (size_t)n));
      CUDA_OK(cudaMalloc(&s0->d_batch_res, sizeof(LmResult) * (size_t)n));
      s0->d_batch_cap = n;
    }
    d_graphs = s0->d_batch;
    for (int i = 0; i < n; i++) hg[i].res = s0->d_batch_res + i;   // (the handles' own result slots are not used by this launch)
  }
  CUDA_OK(cudaMemcpyAsync(d_graphs, hg.data(), sizeof(DevGraph) * n, cudaMemcpyHostToDevice, s0->stream));
  CUDA_OK(cudaMemsetAsync(s0->d_bar, 0, 32 * 1024 * sizeof(unsigned), s0->stream));
  CUDA_OK(cudaEventRecord(s0->ev0, s0->stream));
  const DevGraph* a0 = d_graphs;
  int a1 = n, a2 = team;
  unsigned* a3 = s0->d_bar;
  int a4 = use_cluster;
  void* args[] = {(void*)&a0, (void*)&a1, (void*)&a2, (void*)&a3, (void*)&a4};
  void* kfn = spanning ? span_kernel_ptr() : kern;
  cudaError_t le;
  if (use_cluster) {
    // a team only synchronises inside its cluster, whose CTAs the hardware co-schedules: no cooperative launch needed
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmemBytes; cfg.stream = s0->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = team; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    le = cudaLaunchKernelExC(&cfg, kfn, args);
    if (le != cudaSuccess) {   // (never seen; the same grid also runs with the global-memory barrier)
      cudaGetLastError();
      use_cluster = 0; a4 = 0;
      le = cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(kThreads), args, kSmemBytes, s0->stream);
    }
  } else {
    le = cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(kThreads), args, kSmemBytes, s0->stream);
  }
  if (le != cudaSuccess) { g_err = std::string(use_cluster ? "cudaLaunchKernelExC (cluster): " : "cudaLaunchCooperativeKernel: ") + cudaGetErrorString(le); return -1; }
  CUDA_OK(cudaEventRecord(s0->ev1, s0->stream));
  cudaError_t se = cudaEventSynchronize(s0->ev1);
  if (se != cudaSuccess) { g_err = std::string("lm_kernel: ") + cudaGetErrorString(se); return -1; }
  float ms = 0;
  CUDA_OK(cudaEventElapsedTime(&ms, s0->ev0, s0->ev1));
  std::vector<LmResult> hres;
  if (n > 1) {
    hres.resize(n);
    CUDA_OK(cudaMemcpyAsync(hres.data(), s0->d_batch_res, sizeof(LmResult) * (size_t)n, cudaMemcpyDeviceToHost, s0->stream));
    CUDA_OK(cudaStreamSynchronize(s0->stream));
  }
  for (int i = 0; i < n; i++) {
    Solver* s = ss[i];
    if (n > 1) {
      s->res = hres[i];
    } else {
      CUDA_OK(cudaMemcpyAsync(&s->res, s->d_res, sizeof(LmResult), cudaMemcpyDeviceToHost, s0->stream));
      CUDA_OK(cudaStreamSynchronize(s0->stream));
    }
    if (mode == MODE_DEBUG) {   // the path report rides in fields a debug launch leaves unused: moved aside, the statistics keep 0
      LmResult& r = s->res;
      const int rep[5] = {r.status, r.iterations, r.accepted, r.chi2_evals, r.trace_n};
      std::memcpy(s->path, rep, sizeof(rep));
      r.status = r.iterations = r.accepted = r.chi2_evals = r.trace_n = 0;
    }
    pus_stats& st = s->stats;
    st.lm_iterations = s->res.iterations; st.accepted = s->res.accepted; st.relinearizations = s->res.relin;
    st.chi2_evals = s->res.chi2_evals; st.pcg_iterations = direct ? 0 : s->res.pcg_iters; st.chi2_initial = s->res.chi2_initial;
    st.chi2_final = s->res.chi2_final; st.kernel_ms = ms; st.n_poses = s->c.N; st.n_planes = s->c.M; st.n_pose_plane = s->c.Epl;
    int npr = 0;
    for (int f = 0; f < s->c.Epf; f++) npr += s->c.pf_j[f] < 0;
    st.n_pose_prior = npr; st.n_odometry = s->c.Epf - npr; st.n_plane_prior = s->c.Elp;
    st.gpu_launches = 1; st.grid_ctas = grid; st.block_threads = kThreads;
    for (int k = 0; k < 24; k++) st.phase_ms[k] = s->res.phase_ns[k] * 1e-6;
    st.gpu_launches = 1;
  }
  return 0;
}

// The resident solve and the download act on the layout of the last upload: a structural edit, a change of linear-solver kind or
// of direct ordering since then (each bumps topo_version) would launch on, or download through, tables of another graph.
// Host-only, before any device work.
static int check_uploaded(const Solver* s) {
  if (!s->uploaded) { g_err = "graph not uploaded"; return -1; }
  if (s->compiled_topo != s->g.topo_version) { g_err = "graph changed since its upload: call pus_upload"; return -1; }
  return 0;
}

static int download(Solver** ss, int n) {
  Solver* s0 = ss[0];
  CUDA_OK(cudaSetDevice(s0->device));
  CUDA_OK(cudaEventRecord(s0->ev0, s0->stream));
  long long bytes = 0;
  for (int i = 0; i < n; i++) {
    Solver* s = ss[i];
    Compiled& c = s->c;
    if (c.N) CUDA_OK(cudaMemcpyAsync(c.pose_val.data(), s->hd.pose_lin, c.pose_val.size() * 8, cudaMemcpyDeviceToHost, s0->stream));
    if (c.M) CUDA_OK(cudaMemcpyAsync(c.plane_val.data(), s->hd.plane_lin, c.plane_val.size() * 8, cudaMemcpyDeviceToHost, s0->stream));
    CUDA_OK(cudaMemcpyAsync(&s->trace, s->d_trace, sizeof(LmTrace), cudaMemcpyDeviceToHost, s0->stream));
    bytes += (long long)(c.pose_val.size() + c.plane_val.size()) * 8;
  }
  CUDA_OK(cudaEventRecord(s0->ev1, s0->stream));
  CUDA_OK(cudaEventSynchronize(s0->ev1));
  float ms = 0;
  CUDA_OK(cudaEventElapsedTime(&ms, s0->ev0, s0->ev1));
  for (int i = 0; i < n; i++) {
    Solver* s = ss[i];
    Compiled& c = s->c;
    for (int p = 0; p < c.N; p++) std::memcpy(s->g.nodes[c.pose_node[p]].v, &c.pose_val[(size_t)p * 7], 7 * sizeof(double));
    for (int l = 0; l < c.M; l++) std::memcpy(s->g.nodes[c.plane_node[l]].v, &c.plane_val[(size_t)l * 4], 4 * sizeof(double));
    s->trace_n = s->res.trace_n;
    s->stats.d2h_ms = ms;
    s->stats.d2h_bytes = bytes / n;
  }
  return 0;
}

// a batch rides on the first handle's stream: the others drop their own stream (if any) and borrow it
// (for the duration of the batched call only: release_stream() gives every handle its own stream back, so a later
// pus_destroy of the first handle cannot leave the others with a dangling cudaStream_t)
static void adopt_stream(Solver* s, cudaStream_t st) {
  s->borrow_depth++;
  if (s->borrowing) { s->stream = st; return; }
  s->saved_stream = s->stream; s->saved_own = s->own_stream; s->borrowing = true;
  s->own_stream = false;
  s->stream = st;
}
static void release_stream(Solver* s) {
  if (!s->borrowing || --s->borrow_depth > 0) return;
  s->stream = s->saved_stream; s->own_stream = s->saved_own; s->borrowing = false;
  s->saved_stream = nullptr; s->saved_own = false;
}
// The handle array of a *_many call: no null entry, and no handle twice (two teams would solve one graph's device buffers at
// once).  Host-only, before any device work.
static int check_batch(const pus_handle* hs, int n, const char* fn) {
  if (!hs) { g_err = std::string(fn) + ": null handle array"; return -1; }
  std::vector<std::pair<pus_handle, int>> v(n);
  for (int i = 0; i < n; i++) {
    if (!hs[i]) { g_err = std::string(fn) + ": handle " + std::to_string(i) + " is null"; return -1; }
    v[i] = std::make_pair(hs[i], i);
  }
  std::sort(v.begin(), v.end());
  for (int i = 1; i < n; i++)
    if (v[i].first == v[i - 1].first) {
      g_err = std::string(fn) + ": handles " + std::to_string(v[i - 1].second) + " and " + std::to_string(v[i].second) + " are the same handle";
      return -1;
    }
  return 0;
}
struct BatchStreams {   // RAII: handles 1..n-1 ride on handle 0's stream until the call returns
  pus_handle* hs; int n;
  BatchStreams(pus_handle* h, int k, cudaStream_t st) : hs(h), n(k) { for (int i = 1; i < n; i++) adopt_stream(reinterpret_cast<Solver*>(hs[i]), st); }
  ~BatchStreams() { for (int i = 1; i < n; i++) release_stream(reinterpret_cast<Solver*>(hs[i])); }
};

}  // namespace pus

// ---------------------------------------------------------------------------------------------
// C-ABI
// ---------------------------------------------------------------------------------------------
using namespace pus;
#define SV(h) (reinterpret_cast<Solver*>(h))
#define NEED(h) if (!(h)) { g_err = "null handle"; return -1; }

// launchers of pus_popup.cu (compiled without FMA contraction: float32 pop-up arithmetic as the reference's)
namespace pus {
cudaError_t launch_refresh(cudaStream_t st, int n_frames, const int* d_frame_pose, const double* d_pose7, const int* d_seg_ptr,
                           const int* d_row_frame, int n_rows, const float* d_segs, const float* d_invK, float* d_Ts,
                           float* d_planes_sensor, int n_map, const int* d_map_row, const int* d_map_slot, double* d_pp_meas,
                           double* d_out);
cudaError_t launch_project(cudaStream_t st, int n, const int* d_plane_idx, const double* d_plane4, const float* d_in, float* d_out);
}  // namespace pus

// scratch for the refresh / projection entry points: carved from one grow-only device buffer owned by the solver
struct Scratch {
  Solver* s;
  cudaStream_t st;
  size_t off = 0;
  static size_t al(size_t b) { return (b + 255) / 256 * 256; }
  bool reserve(size_t bytes) {
    if (bytes <= s->scratch_bytes) return true;
    if (s->scratch) { cudaStreamSynchronize(st); cudaFree(s->scratch); s->scratch = nullptr; s->scratch_bytes = 0; }
    if (cudaMalloc(&s->scratch, bytes) != cudaSuccess) return false;
    s->scratch_bytes = bytes;
    return true;
  }
  template <typename T>
  T* put(const T* host, size_t n) {   // carve (and fill when host != nullptr)
    T* p = reinterpret_cast<T*>(static_cast<char*>(s->scratch) + off);
    off += al(std::max<size_t>(n, 1) * sizeof(T));
    if (off > s->scratch_bytes) return nullptr;
    if (host && n && cudaMemcpyAsync(p, host, n * sizeof(T), cudaMemcpyHostToDevice, st) != cudaSuccess) return nullptr;
    return p;
  }
};

extern "C" {

const char* pus_last_error(void) { return g_err.c_str(); }

// The handle itself (graph container, ids, values) is host state; the device is bound lazily by the
// first upload / optimise call, which fails loudly when no CUDA device is usable (no CPU fallback).
int pus_create(int device, pus_handle* out) {
  if (device < 0) { g_err = "bad device ordinal"; return -1; }
  Solver* s = new Solver();
  s->device = device;
  *out = s;
  return 0;
}
int pus_destroy(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  cudaSetDevice(s->device);
  for (void* pp : s->span_peers) if (pp) cudaIpcCloseMemHandle(pp);
  s->free_device();
  if (s->d_batch) cudaFree(s->d_batch);
  if (s->d_batch_res) cudaFree(s->d_batch_res);
  if (s->rt.mem) cudaFree(s->rt.mem);
  if (s->xt.mem) cudaFree(s->xt.mem);
  if (s->xt.ev_copy) cudaEventDestroy(s->xt.ev_copy);
  if (s->cov.mem) cudaFree(s->cov.mem);
  if (s->scratch) cudaFree(s->scratch);
  if (s->ev0) cudaEventDestroy(s->ev0);
  if (s->ev1) cudaEventDestroy(s->ev1);
  if (s->own_stream && s->stream) cudaStreamDestroy(s->stream);
  delete s;
  return 0;
}
int pus_set_stream(pus_handle h, void* st) {
  NEED(h);
  Solver* s = SV(h);
  if (s->own_stream && s->stream) cudaStreamDestroy(s->stream);
  s->own_stream = false;
  s->stream = reinterpret_cast<cudaStream_t>(st);  // nullptr: a library-owned stream is created on first use
  return 0;
}

int pus_add_pose(pus_handle h, const double* v) { NEED(h); return SV(h)->g.add_node(NODE_POSE, v); }
int pus_add_plane(pus_handle h, const double* v) { NEED(h); return SV(h)->g.add_node(NODE_PLANE, v); }
int pus_add_poses(pus_handle h, int n, const double* v, int* out) {
  NEED(h);
  int first = -1;
  for (int i = 0; i < n; i++) { int id = SV(h)->g.add_node(NODE_POSE, v ? v + 7 * i : nullptr); if (!i) first = id; if (out) out[i] = id; }
  return first;
}
int pus_add_planes(pus_handle h, int n, const double* v, int* out) {
  NEED(h);
  int first = -1;
  for (int i = 0; i < n; i++) { int id = SV(h)->g.add_node(NODE_PLANE, v ? v + 4 * i : nullptr); if (!i) first = id; if (out) out[i] = id; }
  return first;
}
int pus_init_pose(pus_handle h, int id, const double* v) {
  NEED(h);
  if (!SV(h)->g.ok_node(id, NODE_POSE)) { g_err = "bad pose id"; return -1; }
  SV(h)->g.init_node(id, v); SV(h)->values_dirty = true; return 0;
}
int pus_init_plane(pus_handle h, int id, const double* v) {
  NEED(h);
  if (!SV(h)->g.ok_node(id, NODE_PLANE)) { g_err = "bad plane id"; return -1; }
  SV(h)->g.init_node(id, v); SV(h)->values_dirty = true; return 0;
}
int pus_init_poses(pus_handle h, int n, const int* ids, const double* v) {
  for (int i = 0; i < n; i++) if (pus_init_pose(h, ids[i], v + 7 * i) < 0) return -1;
  return 0;
}
int pus_init_planes(pus_handle h, int n, const int* ids, const double* v) {
  for (int i = 0; i < n; i++) if (pus_init_plane(h, ids[i], v + 4 * i) < 0) return -1;
  return 0;
}
int pus_get_pose(pus_handle h, int id, double* out) {
  NEED(h);
  if (!SV(h)->g.ok_node(id, NODE_POSE)) { g_err = "bad pose id"; return -1; }
  std::memcpy(out, SV(h)->g.nodes[id].v, 7 * sizeof(double)); return 0;
}
int pus_get_plane(pus_handle h, int id, double* out) {
  NEED(h);
  if (!SV(h)->g.ok_node(id, NODE_PLANE)) { g_err = "bad plane id"; return -1; }
  std::memcpy(out, SV(h)->g.nodes[id].v, 4 * sizeof(double)); return 0;
}
int pus_get_poses(pus_handle h, int n, const int* ids, double* out) {
  for (int i = 0; i < n; i++) if (pus_get_pose(h, ids[i], out + 7 * i) < 0) return -1;
  return 0;
}
int pus_get_planes(pus_handle h, int n, const int* ids, double* out) {
  for (int i = 0; i < n; i++) if (pus_get_plane(h, ids[i], out + 4 * i) < 0) return -1;
  return 0;
}

static int chk(Solver* s, int r) { if (r < 0) g_err = s->g.err; return r; }
int pus_add_pose_prior(pus_handle h, int p, const double* m, const double* si) { NEED(h); return chk(SV(h), SV(h)->g.add_pose_prior(p, m, si)); }
int pus_add_odometry(pus_handle h, int a, int b, const double* m, const double* si) { NEED(h); return chk(SV(h), SV(h)->g.add_odometry(a, b, m, si)); }
int pus_add_pose_plane(pus_handle h, int p, int l, const double* m, const double* si) { NEED(h); return chk(SV(h), SV(h)->g.add_pose_plane(p, l, m, si)); }
int pus_add_pose_plane2(pus_handle h, int p, int l, const double* m, const double* rays, const double* si) { NEED(h); return chk(SV(h), SV(h)->g.add_pose_plane2(p, l, m, rays, si)); }
int pus_add_plane_prior(pus_handle h, int l, const double* m, const double* si) { NEED(h); return chk(SV(h), SV(h)->g.add_plane_prior(l, m, si)); }
int pus_add_odometry_bulk(pus_handle h, int n, const int* a, const int* b, const double* m, const double* si, int* out) {
  NEED(h);
  int first = -1;
  for (int i = 0; i < n; i++) {
    int f = chk(SV(h), SV(h)->g.add_odometry(a[i], b[i], m + 6 * i, si + 21 * i));
    if (f < 0) return f;
    if (!i) first = f;
    if (out) out[i] = f;
  }
  return first;
}
int pus_add_pose_plane_bulk(pus_handle h, int n, const int* a, const int* b, const double* m, const double* si, int* out) {
  NEED(h);
  int first = -1;
  for (int i = 0; i < n; i++) {
    int f = chk(SV(h), SV(h)->g.add_pose_plane(a[i], b[i], m + 4 * i, si + 6 * i));
    if (f < 0) return f;
    if (!i) first = f;
    if (out) out[i] = f;
  }
  return first;
}
int pus_set_measurement(pus_handle h, int fid, const double* m) {
  NEED(h);
  Solver* s = SV(h);
  if (!s->g.ok_factor(fid)) { g_err = "bad factor id"; return -1; }
  if (sync_measurements_to_host(s) < 0) return -1;
  HFactor& f = s->g.factors[fid];
  if (f.dim == 3) { std::memcpy(f.meas, m, 4 * sizeof(double)); normalize4(f.meas); }
  else std::memcpy(f.meas, m, 6 * sizeof(double));
  s->meas_dirty = true;
  return 0;
}
int pus_get_measurement(pus_handle h, int fid, double* m) {
  NEED(h);
  if (!SV(h)->g.ok_factor(fid)) { g_err = "bad factor id"; return -1; }
  if (sync_measurements_to_host(SV(h)) < 0) return -1;
  const HFactor& f = SV(h)->g.factors[fid];
  std::memcpy(m, f.meas, (f.dim == 3 ? 4 : 6) * sizeof(double)); return 0;
}
int pus_remove_factor(pus_handle h, int fid) {
  NEED(h);
  if (!SV(h)->g.ok_factor(fid)) { g_err = "bad factor id"; return -1; }
  SV(h)->g.remove_factor(fid); return 0;
}
int pus_remove_node(pus_handle h, int id) {
  NEED(h);
  if (id < 0 || id >= (int)SV(h)->g.nodes.size() || !SV(h)->g.nodes[id].alive) { g_err = "bad node id"; return -1; }
  SV(h)->g.remove_node(id); return 0;
}
int pus_num_nodes(pus_handle h) { NEED(h); return SV(h)->g.num_nodes(); }
int pus_num_factors(pus_handle h) { NEED(h); return SV(h)->g.num_factors(); }
int pus_factor_nodes(pus_handle h, int fid, int* out2) {
  NEED(h);
  if (!SV(h)->g.ok_factor(fid)) { g_err = "bad factor id"; return -1; }
  const HFactor& f = SV(h)->g.factors[fid];
  for (int k = 0; k < f.n_nodes; k++) out2[k] = f.nodes[k];
  return f.n_nodes;
}
int pus_node_factors(pus_handle h, int id, int* out, int cap) {
  NEED(h);
  const Graph& g = SV(h)->g;
  if (id < 0 || id >= (int)g.nodes.size() || !g.nodes[id].alive) { g_err = "bad node id"; return -1; }
  int c = 0;
  for (size_t i = 0; i < g.factors.size(); i++) {
    const HFactor& f = g.factors[i];
    if (!f.alive) continue;
    for (int k = 0; k < f.n_nodes; k++) if (f.nodes[k] == id) { if (c < cap) out[c] = (int)i; c++; break; }
  }
  return c;
}
int pus_node_start(pus_handle h, int id) { if (!h) return -1; return SV(h)->g.node_start(id); }
int pus_factor_row(pus_handle h, int fid) { if (!h) return -1; return SV(h)->g.factor_row(fid); }

int pus_get_properties(pus_handle h, pus_properties* out) { NEED(h); *out = SV(h)->prop; return 0; }
int pus_set_properties(pus_handle h, const pus_properties* in) { NEED(h); SV(h)->prop = *in; return 0; }
int pus_set_robust(pus_handle h, int kind, double b) {
  NEED(h);
  if (kind < 0 || kind > 2 || !(b > 0)) { g_err = "bad robust cost"; return -1; }
  SV(h)->robust_kind = kind; SV(h)->robust_b = b; SV(h)->cov.valid = false; return 0;
}
int pus_set_jacobian_mode(pus_handle h, int numeric) { NEED(h); SV(h)->jac_numeric = numeric ? 1 : 0; SV(h)->cov.valid = false; return 0; }
int pus_set_linear_solver(pus_handle h, int kind) {
  NEED(h);
  Solver* s = SV(h);
  if (kind < 0 || kind > 2) { g_err = "bad linear solver kind (0 = PCG, 1 = dense direct, 2 = band direct)"; return -1; }
  if (kind != s->linear_solver) { s->linear_solver = kind; s->g.topo_version++; }   // the next upload lays the graph out again
  return 0;
}
int pus_get_linear_solver(pus_handle h) { NEED(h); return SV(h)->linear_solver; }
int pus_set_direct_ordering(pus_handle h, int order) {
  NEED(h);
  Solver* s = SV(h);
  if (order < 0 || order > 1) { g_err = "bad direct ordering (0 = insertion order, 1 = nested dissection)"; return -1; }
  if (order != s->ordering) {   // (only kind 2 lays the graph out by it; the next upload of a kind-2 handle lays it out again)
    s->ordering = order;
    s->g.topo_version++;
  }
  return 0;
}
int pus_get_direct_ordering(pus_handle h) { NEED(h); return SV(h)->ordering; }
static int refuse_direct_span(Solver* s, const char* fn) {
  if (s->linear_solver == 0) return 0;
  g_err = std::string(fn) + ": the direct linear solvers do not span ranks (set the PCG solver, kind 0)";
  return -1;
}
int pus_get_solver_options(pus_handle h, pus_solver_options* out) { NEED(h); *out = SV(h)->opt; return 0; }
int pus_set_solver_options(pus_handle h, const pus_solver_options* in) { NEED(h); SV(h)->opt = *in; return 0; }

int pus_upload(pus_handle h) { NEED(h); return upload(SV(h)); }
int pus_upload_many(pus_handle* hs, int n) {
  if (n <= 0) return 0;
  if (check_batch(hs, n, "pus_upload_many") < 0) return -1;
  if (ensure_device(SV(hs[0])) < 0) return -1;
  BatchStreams bs(hs, n, SV(hs[0])->stream);
  for (int i = 0; i < n; i++) if (upload(SV(hs[i])) < 0) return -1;
  return 0;
}
static int solve_many(pus_handle* hs, int n, int* iters, int mode, int restore) {
  if (n <= 0) return 0;
  std::vector<Solver*> ss(n);
  for (int i = 0; i < n; i++) ss[i] = SV(hs[i]);
  for (int i = 0; i < n; i++) if (check_uploaded(ss[i]) < 0) return -1;
  if (ensure_device(ss[0]) < 0) return -1;
  BatchStreams bs(hs, n, ss[0]->stream);
  // direct-mode (dense and band) and PCG handles run in their own kernels: a mixed batch is two launches, one per kernel
  std::vector<Solver*> part[2];
  for (int i = 0; i < n; i++) part[ss[i]->linear_solver != 0].push_back(ss[i]);
  for (int k = 0; k < 2; k++)
    if (!part[k].empty() && launch(part[k].data(), (int)part[k].size(), mode, restore, 0, 0.0) < 0) return -1;
  if (iters) for (int i = 0; i < n; i++) iters[i] = ss[i]->res.iterations;
  return 0;
}
int pus_solve_resident(pus_handle h, int* iters) { NEED(h); return solve_many(&h, 1, iters, MODE_BATCH, 1); }
int pus_solve_resident_many(pus_handle* hs, int n, int* iters) {
  if (n <= 0) return 0;
  if (check_batch(hs, n, "pus_solve_resident_many") < 0) return -1;
  return solve_many(hs, n, iters, MODE_BATCH, 1);
}
int pus_download(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  if (check_uploaded(s) < 0) return -1;
  return download(&s, 1);
}
int pus_download_many(pus_handle* hs, int n) {
  if (n <= 0) return 0;
  if (check_batch(hs, n, "pus_download_many") < 0) return -1;
  std::vector<Solver*> ss(n);
  for (int i = 0; i < n; i++) ss[i] = SV(hs[i]);
  for (int i = 0; i < n; i++) if (check_uploaded(ss[i]) < 0) return -1;
  if (ensure_device(ss[0]) < 0) return -1;
  BatchStreams bs(hs, n, ss[0]->stream);
  return download(ss.data(), n);
}

int pus_batch_optimize(pus_handle h, int* iters) {
  NEED(h);
  Solver* s = SV(h);
  if (upload(s) < 0) return -1;
  if (solve_many(&h, 1, iters, MODE_BATCH, 0) < 0) return -1;
  return download(&s, 1);
}
int pus_batch_optimize_many(pus_handle* hs, int n, int* iters) {
  if (n <= 0) return 0;
  if (check_batch(hs, n, "pus_batch_optimize_many") < 0) return -1;
  Solver* s0 = SV(hs[0]);
  if (ensure_device(s0) < 0) return -1;
  BatchStreams bs(hs, n, s0->stream);
  if (pus_upload_many(hs, n) < 0) return -1;
  if (solve_many(hs, n, iters, MODE_BATCH, 0) < 0) return -1;
  return pus_download_many(hs, n);
}
// ---- one graph spanning several ranks ----
int pus_span_export(pus_handle h, void* out64) {
  NEED(h);
  Solver* s = SV(h);
  if (refuse_direct_span(s, "pus_span_export") < 0) return -1;
  if (upload(s) < 0) return -1;
  cudaIpcMemHandle_t mh;
  CUDA_OK(cudaIpcGetMemHandle(&mh, s->arena));
  static_assert(sizeof(mh) == 64, "CUDA IPC handle size");
  std::memcpy(out64, &mh, 64);
  return 0;
}
int pus_span_disconnect(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  for (void* p : s->span_peers) if (p) cudaIpcCloseMemHandle(p);
  s->span_peers.clear();
  s->span_w = 1; s->span_r = 0;
  return 0;
}
int pus_span_connect(pus_handle h, int rank, int world, const void* handles) {
  NEED(h);
  Solver* s = SV(h);
  if (world < 1 || world > 8 || rank < 0 || rank >= world) { g_err = "pus_span_connect: world must be 1..8"; return -1; }
  if (refuse_direct_span(s, "pus_span_connect") < 0) return -1;
  if (!s->uploaded || !s->arena) { g_err = "pus_span_connect: call pus_span_export first"; return -1; }
  pus_span_disconnect(h);
  CUDA_OK(cudaSetDevice(s->device));
  s->span_peers.assign(world, nullptr);
  for (int w = 0; w < world; w++) {
    if (w == rank) continue;
    cudaIpcMemHandle_t mh;
    std::memcpy(&mh, static_cast<const char*>(handles) + 64 * (size_t)w, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, mh, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { g_err = std::string("cudaIpcOpenMemHandle (peer ") + std::to_string(w) + "): " + cudaGetErrorString(e); pus_span_disconnect(h); return -1; }
    s->span_peers[w] = p;
  }
  s->span_w = world; s->span_r = rank;
  s->span_topo = s->compiled_topo;
  return 0;
}
static void span_fill(Solver* s, int rank, int world, const std::vector<char*>& arenas) {
  s->hd.span_w = world; s->hd.span_r = rank;
  for (int w = 0; w < 8; w++) s->hd.peer_delta[w] = (w < world) ? (long long)(arenas[w] - arenas[rank]) : 0;
}
int pus_span_optimize(pus_handle h, int* iters) {
  NEED(h);
  Solver* s = SV(h);
  if (refuse_direct_span(s, "pus_span_optimize") < 0) return -1;
  if (s->span_w <= 1) { g_err = "pus_span_optimize: not connected"; return -1; }
  if (upload(s) < 0) return -1;   // values only: a rebuild would move the arena the peers have mapped
  if (s->span_topo != s->compiled_topo) { g_err = "pus_span_optimize: the graph changed since pus_span_connect; export / connect again"; return -1; }
  std::vector<char*> arenas(s->span_w);
  for (int w = 0; w < s->span_w; w++) arenas[w] = (w == s->span_r) ? reinterpret_cast<char*>(s->arena) : static_cast<char*>(s->span_peers[w]);
  span_fill(s, s->span_r, s->span_w, arenas);
  int rc = solve_many(&h, 1, iters, MODE_BATCH, 0);
  s->hd.span_w = 1; s->hd.span_r = 0;
  if (rc < 0) return -1;
  return download(&s, 1);
}
int pus_span_emulate_optimize(pus_handle* hs, int world, int* iters) {
  if (world < 1 || world > 8) { g_err = "pus_span_emulate_optimize: world must be 1..8"; return -1; }
  if (check_batch(hs, world, "pus_span_emulate_optimize") < 0) return -1;
  for (int i = 0; i < world; i++) if (refuse_direct_span(SV(hs[i]), "pus_span_emulate_optimize") < 0) return -1;
  Solver* s0 = SV(hs[0]);
  if (ensure_device(s0) < 0) return -1;
  BatchStreams bs(hs, world, s0->stream);
  if (pus_upload_many(hs, world) < 0) return -1;
  std::vector<char*> arenas(world);
  for (int i = 0; i < world; i++) arenas[i] = reinterpret_cast<char*>(SV(hs[i])->arena);
  for (int i = 0; i < world; i++) span_fill(SV(hs[i]), i, world, arenas);
  std::vector<int> its(world, 0);
  int rc = solve_many(hs, world, its.data(), MODE_BATCH, 0);
  for (int i = 0; i < world; i++) { SV(hs[i])->hd.span_w = 1; SV(hs[i])->hd.span_r = 0; }
  if (rc < 0) return -1;
  if (iters) *iters = its[0];
  return pus_download_many(hs, world);
}

// Slam::update (Slam.cpp:157-196). PPS runs with mod_batch = 1 => every call is the batch step
// (relinearise + one Gauss-Newton step). Other settings would need iSAM's Givens incremental path.
int pus_update(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  int rc = 0;
  if (s->step % std::max(1, s->prop.mod_update) == 0) {
    if (s->step % std::max(1, s->prop.mod_batch) == 0) {
      if (upload(s) < 0) return -1;
      if (solve_many(&h, 1, nullptr, MODE_UPDATE, 0) < 0) return -1;
      rc = download(&s, 1);
    } else {
      g_err = "pus_update: incremental (Givens) steps are not implemented; set mod_batch = 1 as pop_planar_slam does";
      rc = -1;
    }
  }
  s->step++;
  return rc;
}
int pus_chi2(pus_handle h, double* out) {
  NEED(h);
  Solver* s = SV(h);
  if (upload(s) < 0) return -1;
  if (solve_many(&h, 1, nullptr, MODE_CHI2, 0) < 0) return -1;
  *out = s->res.chi2_final;
  return 0;
}

int pus_get_stats(pus_handle h, pus_stats* out) { NEED(h); *out = SV(h)->stats; return 0; }
int pus_get_trace(pus_handle h, int cap, double* lambda, double* e_new, double* e_before, double* dn, int* acc, int* pcg) {
  NEED(h);
  Solver* s = SV(h);
  int n = s->trace_n;
  for (int i = 0; i < n && i < cap; i++) {
    if (lambda) lambda[i] = s->trace.lambda[i];
    if (e_new) e_new[i] = s->trace.chi2_new[i];
    if (e_before) e_before[i] = s->trace.chi2_before[i];
    if (dn) dn[i] = s->trace.delta_norm[i];
    if (acc) acc[i] = s->trace.accepted[i];
    if (pcg) pcg[i] = s->trace.pcg[i];
  }
  return n;
}

// ---- debug hooks ----
// ---- device-resident measurement refresh / polygon re-projection (SURVEY 8f.1) ----
int pus_refresh_plane_measurements(pus_handle h, int n_frames, const int* frame_pose, const int* seg_ptr, const float* segs,
                                   const float* invK, int n_map, const int* map_fid, const int* map_frame, const int* map_row,
                                   double* new_meas) {
  NEED(h);
  Solver* s = SV(h);
  if (n_frames <= 0) return 0;
  std::vector<int> row_frame;
  if (const char* why = row_frames(n_frames, seg_ptr, row_frame)) { g_err = why; return -1; }
  // (re-upload when the topology OR the host values changed: update_plane_measurement uses pose_vertex->value())
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty) {
    if (upload(s) < 0) return -1;
  } else if (ensure_device(s) < 0) {
    return -1;
  }
  const Compiled& c = s->c;
  const int n_seg = seg_ptr[n_frames], n_rows = n_seg + n_frames;
  std::vector<int> fpose(n_frames), mrow(n_map), mslot(n_map);
  for (int f = 0; f < n_frames; f++) {
    if (!s->g.ok_node(frame_pose[f], NODE_POSE)) { g_err = "frame " + std::to_string(f) + ": not a pose node"; return -1; }
    fpose[f] = c.node_idx[frame_pose[f]];
  }
  if ((int)s->fid2slot.size() != (int)s->g.factors.size() || s->fid2slot_topo != s->compiled_topo) {
    s->fid2slot.assign(s->g.factors.size(), -1);
    for (int e = 0; e < c.nslot; e++) if (c.pp_fid[e] >= 0) s->fid2slot[c.pp_fid[e]] = e;
    s->fid2slot_topo = s->compiled_topo;
  }
  for (int m = 0; m < n_map; m++) {
    const int f = map_frame[m], fid = map_fid[m];
    if (f < 0 || f >= n_frames) { g_err = "map_frame out of range"; return -1; }
    const int ns = seg_ptr[f + 1] - seg_ptr[f];
    if (ns <= 0 || map_row[m] < 0 || map_row[m] > ns) { g_err = "map_row out of range (frames without segments produce no planes)"; return -1; }
    if (!s->g.ok_factor(fid) || s->g.factors[fid].kind != F_POSE_PLANE || s->fid2slot[fid] < 0) { g_err = "map_fid is not a pose-plane factor"; return -1; }
    mrow[m] = seg_ptr[f] + f + map_row[m];
    mslot[m] = s->fid2slot[fid];
  }
  CUDA_OK(cudaSetDevice(s->device));
  cudaStream_t st = s->stream;
  Scratch sc{s, st};
  if (!sc.reserve(Scratch::al(4 * (size_t)n_frames) + Scratch::al(4 * (size_t)(n_frames + 1)) + Scratch::al(4 * (size_t)n_rows) +
                  Scratch::al(16 * (size_t)std::max(n_seg, 1)) + Scratch::al(36) + 2 * Scratch::al(4 * (size_t)std::max(n_map, 1)) +
                  Scratch::al(64 * (size_t)n_frames) + Scratch::al(16 * (size_t)n_rows) + Scratch::al(32 * (size_t)std::max(n_map, 1)))) {
    g_err = "scratch allocation failed";
    return -1;
  }
  int* d_fpose = sc.put(fpose.data(), n_frames);
  int* d_ptr = sc.put(seg_ptr, n_frames + 1);
  int* d_rf = sc.put(row_frame.data(), n_rows);
  float* d_segs = sc.put(segs, (size_t)n_seg * 4);
  float* d_K = sc.put(invK, 9);
  int* d_mrow = sc.put(mrow.data(), n_map);
  int* d_mslot = sc.put(mslot.data(), n_map);
  float* d_T = sc.put<float>(nullptr, (size_t)n_frames * 16);
  float* d_ps = sc.put<float>(nullptr, (size_t)n_rows * 4);
  double* d_out = sc.put<double>(nullptr, (size_t)n_map * 4);
  if (!d_fpose || !d_ptr || !d_rf || !d_segs || !d_K || !d_mrow || !d_mslot || !d_T || !d_ps || !d_out) { g_err = "scratch allocation failed"; return -1; }
  s->cov.valid = false;   // (new measurements on the device)
  CUDA_OK(cudaMemsetAsync(d_ps, 0, (size_t)n_rows * 4 * sizeof(float), st));
  CUDA_OK(launch_refresh(st, n_frames, d_fpose, s->hd.pose_lin, d_ptr, d_rf, n_rows, d_segs, d_K, d_T, d_ps, n_map, d_mrow, d_mslot,
                         const_cast<double*>(s->hd.pp_meas), d_out));
  std::vector<double> out((size_t)n_map * 4);
  if (n_map) CUDA_OK(cudaMemcpyAsync(out.data(), d_out, out.size() * 8, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  for (int m = 0; m < n_map; m++) {   // host mirrors: the factor store and the compiled copy
    std::memcpy(s->g.factors[map_fid[m]].meas, &out[(size_t)m * 4], 4 * sizeof(double));
    std::memcpy(&s->c.pp_meas[(size_t)mslot[m] * 4], &out[(size_t)m * 4], 4 * sizeof(double));
  }
  if (new_meas && n_map) std::memcpy(new_meas, out.data(), out.size() * 8);
  return 0;
}

// ---- resident form: the frames' segment lists, invK and the factor map stay on the device between calls ----
static int refresh_slots(Solver* s) {   // (re)build the layout-dependent tables: pose index per frame, edge slot per map entry
  Solver::RefreshTables& t = s->rt;
  const Compiled& c = s->c;
  std::vector<int> fpose(t.n_frames), mslot(t.n_map);
  for (int f = 0; f < t.n_frames; f++) {
    if (!s->g.ok_node(t.frame_node[f], NODE_POSE)) { g_err = "pus_refresh_run: frame " + std::to_string(f) + " is no longer a pose node; bind again"; return -1; }
    fpose[f] = c.node_idx[t.frame_node[f]];
  }
  if ((int)s->fid2slot.size() != (int)s->g.factors.size() || s->fid2slot_topo != s->compiled_topo) {
    s->fid2slot.assign(s->g.factors.size(), -1);
    for (int e = 0; e < c.nslot; e++) if (c.pp_fid[e] >= 0) s->fid2slot[c.pp_fid[e]] = e;
    s->fid2slot_topo = s->compiled_topo;
  }
  for (int m = 0; m < t.n_map; m++) {
    const int fid = t.map_fid[m];
    if (t.owner && !s->g.ok_factor(fid)) { mslot[m] = -1; continue; }   // a plane map's landmark removed by its caller: skipped
    if (!s->g.ok_factor(fid) || s->g.factors[fid].kind != F_POSE_PLANE || s->fid2slot[fid] < 0) {
      g_err = "pus_refresh_run: map entry " + std::to_string(m) + " is no longer a pose-plane factor; bind again";
      return -1;
    }
    mslot[m] = s->fid2slot[fid];
  }
  CUDA_OK(cudaMemcpyAsync(t.d_fpose, fpose.data(), sizeof(int) * t.n_frames, cudaMemcpyHostToDevice, s->stream));
  if (t.n_map) CUDA_OK(cudaMemcpyAsync(t.d_mslot, mslot.data(), sizeof(int) * t.n_map, cudaMemcpyHostToDevice, s->stream));
  CUDA_OK(cudaStreamSynchronize(s->stream));   // (the staging vectors go out of scope)
  t.slot_topo = s->compiled_topo;
  return 0;
}

// the resident tables' sections, carved from one allocation for room of cap_frames frames, cap_seg segments and cap_map
// map entries (one row per segment plus a ground row per frame)
static size_t refresh_bytes(int cap_frames, int cap_seg, int cap_map) {
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t rows = (size_t)cap_seg + cap_frames, m = (size_t)std::max(cap_map, 1);
  return al(4 * (size_t)cap_frames) + al(4 * (size_t)(cap_frames + 1)) + al(4 * rows) + 2 * al(4 * m) + al(16 * (size_t)std::max(cap_seg, 1)) +
         al(36) + al(64 * (size_t)cap_frames) + al(16 * rows) + al(32 * m);
}
static void refresh_carve(Solver::RefreshTables& t, void* mem, int cap_frames, int cap_seg, int cap_map) {
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  char* base = static_cast<char*>(mem);
  size_t off = 0;
  auto carve = [&](size_t b) { void* p = base + off; off += al(b); return p; };
  const size_t rows = (size_t)cap_seg + cap_frames, m = (size_t)std::max(cap_map, 1);
  t.d_fpose = (int*)carve(4 * (size_t)cap_frames); t.d_ptr = (int*)carve(4 * (size_t)(cap_frames + 1)); t.d_rf = (int*)carve(4 * rows);
  t.d_mrow = (int*)carve(4 * m); t.d_mslot = (int*)carve(4 * m);
  t.d_segs = (float*)carve(16 * (size_t)std::max(cap_seg, 1)); t.d_K = (float*)carve(36); t.d_T = (float*)carve(64 * (size_t)cap_frames);
  t.d_ps = (float*)carve(16 * rows); t.d_out = (double*)carve(32 * m);
  t.cap_frames = cap_frames; t.cap_seg = cap_seg; t.cap_map = cap_map;
}

int pus_refresh_bind(pus_handle h, int n_frames, const int* frame_pose, const int* seg_ptr, const float* segs, const float* invK,
                     int n_map, const int* map_fid, const int* map_frame, const int* map_row) {
  NEED(h);
  Solver* s = SV(h);
  Solver::RefreshTables& t = s->rt;
  t.bound = false;
  if (n_frames <= 0 || n_map < 0) { g_err = "pus_refresh_bind: nothing to bind"; return -1; }
  std::vector<int> row_frame;
  if (const char* why = row_frames(n_frames, seg_ptr, row_frame)) { g_err = why; return -1; }
  if (ensure_device(s) < 0) return -1;
  const int n_seg = seg_ptr[n_frames], n_rows = n_seg + n_frames;
  t.frame_node.assign(frame_pose, frame_pose + n_frames);
  t.map_fid.assign(map_fid, map_fid + n_map);
  t.mrow.resize(n_map);
  for (int f = 0; f < n_frames; f++)
    if (!s->g.ok_node(frame_pose[f], NODE_POSE)) { g_err = "frame " + std::to_string(f) + ": not a pose node"; return -1; }
  for (int m = 0; m < n_map; m++) {
    const int f = map_frame[m];
    if (f < 0 || f >= n_frames) { g_err = "map_frame out of range"; return -1; }
    const int ns = seg_ptr[f + 1] - seg_ptr[f];
    if (ns <= 0 || map_row[m] < 0 || map_row[m] > ns) { g_err = "map_row out of range (frames without segments produce no planes)"; return -1; }
    if (!s->g.ok_factor(map_fid[m]) || s->g.factors[map_fid[m]].kind != F_POSE_PLANE) { g_err = "map_fid is not a pose-plane factor"; return -1; }
    t.mrow[m] = seg_ptr[f] + f + map_row[m];
  }
  const size_t need = refresh_bytes(n_frames, n_seg, n_map);
  CUDA_OK(cudaSetDevice(s->device));
  if (need > t.bytes) {
    if (t.mem) { cudaStreamSynchronize(s->stream); cudaFree(t.mem); t.mem = nullptr; t.bytes = 0; }
    CUDA_OK(cudaMalloc(&t.mem, need + need / 2));
    t.bytes = need + need / 2;
  }
  t.owner = nullptr;
  refresh_carve(t, t.mem, n_frames, n_seg, n_map);
  cudaStream_t st = s->stream;
  CUDA_OK(cudaMemcpyAsync(t.d_ptr, seg_ptr, 4 * (size_t)(n_frames + 1), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t.d_rf, row_frame.data(), 4 * (size_t)n_rows, cudaMemcpyHostToDevice, st));
  if (n_seg) CUDA_OK(cudaMemcpyAsync(t.d_segs, segs, 16 * (size_t)n_seg, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t.d_K, invK, 36, cudaMemcpyHostToDevice, st));
  if (n_map) CUDA_OK(cudaMemcpyAsync(t.d_mrow, t.mrow.data(), 4 * (size_t)n_map, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(t.d_ps, 0, 16 * (size_t)n_rows, st));
  CUDA_OK(cudaStreamSynchronize(st));
  t.n_frames = n_frames; t.n_seg = n_seg; t.n_rows = n_rows; t.n_map = n_map;
  t.slot_topo = 0;
  t.bound = true;
  return 0;
}

int pus_refresh_run(pus_handle h, double* new_meas) {
  NEED(h);
  Solver* s = SV(h);
  Solver::RefreshTables& t = s->rt;
  if (!t.bound) { g_err = "pus_refresh_run: call pus_refresh_bind first"; return -1; }
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty || s->meas_dirty) {
    if (upload(s) < 0) return -1;
  } else if (ensure_device(s) < 0) {
    return -1;
  }
  if (t.slot_topo != s->compiled_topo && refresh_slots(s) < 0) return -1;
  CUDA_OK(cudaSetDevice(s->device));
  cudaStream_t st = s->stream;
  s->cov.valid = false;   // (new measurements on the device)
  CUDA_OK(cudaEventRecord(s->ev0, st));
  CUDA_OK(launch_refresh(st, t.n_frames, t.d_fpose, s->hd.pose_lin, t.d_ptr, t.d_rf, t.n_rows, t.d_segs, t.d_K, t.d_T, t.d_ps, t.n_map, t.d_mrow,
                         t.d_mslot, const_cast<double*>(s->hd.pp_meas), t.d_out));
  CUDA_OK(cudaEventRecord(s->ev1, st));
  if (new_meas && t.n_map) {
    CUDA_OK(cudaMemcpyAsync(new_meas, t.d_out, (size_t)t.n_map * 32, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    for (int m = 0; m < t.n_map; m++) {   // host mirrors: the factor store and the compiled copy
      std::memcpy(s->g.factors[t.map_fid[m]].meas, new_meas + (size_t)m * 4, 4 * sizeof(double));
      std::memcpy(&s->c.pp_meas[(size_t)s->fid2slot[t.map_fid[m]] * 4], new_meas + (size_t)m * 4, 4 * sizeof(double));
    }
  } else {
    CUDA_OK(cudaEventSynchronize(s->ev1));
    if (t.n_map) s->meas_device_newer = true;   // host mirrors are refreshed lazily (pus_get_measurement, next layout rebuild)
  }
  float ms = 0;
  CUDA_OK(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
  s->stats.kernel_ms = ms; s->stats.gpu_launches = 3;
  return 0;
}

int pus_project_to_planes(pus_handle h, int n_points, const int* plane_of_point, const float* pts_in, float* pts_out) {
  NEED(h);
  Solver* s = SV(h);
  if (n_points <= 0) return 0;
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty) {
    if (upload(s) < 0) return -1;
  } else if (ensure_device(s) < 0) {
    return -1;
  }
  std::vector<int> idx(n_points);
  for (int i = 0; i < n_points; i++) {
    if (!s->g.ok_node(plane_of_point[i], NODE_PLANE)) { g_err = "point " + std::to_string(i) + ": not a plane node"; return -1; }
    idx[i] = s->c.node_idx[plane_of_point[i]];
  }
  CUDA_OK(cudaSetDevice(s->device));
  cudaStream_t st = s->stream;
  Scratch sc{s, st};
  if (!sc.reserve(Scratch::al(4 * (size_t)n_points) + 2 * Scratch::al(12 * (size_t)n_points))) { g_err = "scratch allocation failed"; return -1; }
  int* d_idx = sc.put(idx.data(), n_points);
  float* d_in = sc.put(pts_in, (size_t)n_points * 3);
  float* d_out = sc.put<float>(nullptr, (size_t)n_points * 3);
  if (!d_idx || !d_in || !d_out) { g_err = "scratch allocation failed"; return -1; }
  CUDA_OK(launch_project(st, n_points, d_idx, s->hd.plane_lin, d_in, d_out));
  CUDA_OK(cudaMemcpyAsync(pts_out, d_out, (size_t)n_points * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

// ---- weighted errors / stacked Jacobian at the current estimate (pus_export.cu) ----
}  // extern "C"

// ---- what a plane map (pus_map.cu) needs from its handle ----
namespace pus {
// the device estimates current: upload when the topology, the host values or the measurements changed
int engine_sync(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  if (s->g.nodes.empty()) { if (ensure_device(s) < 0) return -1; CUDA_OK(cudaSetDevice(s->device)); return 0; }
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty || s->meas_dirty) return upload(s);
  if (ensure_device(s) < 0) return -1;
  CUDA_OK(cudaSetDevice(s->device));
  return 0;
}
int engine_device(pus_handle h) { return SV(h)->device; }
cudaStream_t engine_stream(pus_handle h) { return SV(h)->stream; }
// the resident estimates of the last upload / solve, indexed by engine_node_index
const double* engine_pose_lin(pus_handle h) { return SV(h)->hd.pose_lin; }
const double* engine_plane_lin(pus_handle h) { return SV(h)->hd.plane_lin; }
// a live node's index into those arrays, or -1 (removed, or not of that kind: 0 pose, 1 plane); valid after engine_sync
int engine_node_index(pus_handle h, int id, int kind) {
  const Solver* s = SV(h);
  if (!s->g.ok_node(id, kind ? NODE_PLANE : NODE_POSE)) return -1;
  return s->c.node_idx[id];
}
bool engine_node_alive(pus_handle h, int id, int kind) { return SV(h)->g.ok_node(id, kind ? NODE_PLANE : NODE_POSE); }
int engine_iterations(pus_handle h) { return SV(h)->stats.lm_iterations; }
// Append one frame to the resident refresh tables owned by `owner`: its pose node, its n_segs segments (device pointer,
// copied on the device) and n_map (factor, plane row) entries.  The first append of an owner starts the tables afresh;
// the sections grow by half their size and only the new rows are written.  Refused when the caller rebound the tables.
int engine_refresh_append(pus_handle h, const void* owner, int pose_node, int n_segs, const float* d_segs, const float* invK,
                          int n_map, const int* fids, const int* rows) {
  NEED(h);
  Solver* s = SV(h);
  Solver::RefreshTables& t = s->rt;
  const bool fresh = t.owner != owner;
  const int nf = fresh ? 0 : t.n_frames, ns = fresh ? 0 : t.n_seg, nm = fresh ? 0 : t.n_map;
  const int need_f = nf + 1, need_s = ns + n_segs, need_m = nm + n_map;
  cudaStream_t st = s->stream;
  CUDA_OK(cudaSetDevice(s->device));
  if (fresh || need_f > t.cap_frames || need_s > t.cap_seg || need_m > t.cap_map) {
    const int cf = std::max(need_f, fresh ? 16 : t.cap_frames + t.cap_frames / 2);
    const int cs = std::max(need_s, fresh ? 256 : t.cap_seg + t.cap_seg / 2);
    const int cm = std::max(need_m, fresh ? 128 : t.cap_map + t.cap_map / 2);
    const size_t bytes = refresh_bytes(cf, cs, cm);
    void* mem = nullptr;
    CUDA_OK(cudaMalloc(&mem, bytes));
    Solver::RefreshTables old = t;
    refresh_carve(t, mem, cf, cs, cm);
    if (!fresh) {
      CUDA_OK(cudaMemcpyAsync(t.d_ptr, old.d_ptr, 4 * (size_t)(nf + 1), cudaMemcpyDeviceToDevice, st));
      CUDA_OK(cudaMemcpyAsync(t.d_rf, old.d_rf, 4 * (size_t)(ns + nf), cudaMemcpyDeviceToDevice, st));
      if (nm) CUDA_OK(cudaMemcpyAsync(t.d_mrow, old.d_mrow, 4 * (size_t)nm, cudaMemcpyDeviceToDevice, st));
      if (ns) CUDA_OK(cudaMemcpyAsync(t.d_segs, old.d_segs, 16 * (size_t)ns, cudaMemcpyDeviceToDevice, st));
      CUDA_OK(cudaMemcpyAsync(t.d_ps, old.d_ps, 16 * (size_t)(ns + nf), cudaMemcpyDeviceToDevice, st));
    }
    if (old.mem) { CUDA_OK(cudaStreamSynchronize(st)); cudaFree(old.mem); }
    t.mem = mem; t.bytes = bytes;
    CUDA_OK(cudaMemcpyAsync(t.d_K, invK, 36, cudaMemcpyHostToDevice, st));   // (every new allocation)
  }
  if (fresh) {
    const int zero = 0;
    CUDA_OK(cudaMemcpyAsync(t.d_ptr, &zero, 4, cudaMemcpyHostToDevice, st));
    t.frame_node.clear(); t.map_fid.clear(); t.mrow.clear();
    t.owner = owner;
  }
  const int end = need_s;
  std::vector<int> rf(n_segs + 1, nf), mrow(n_map);
  for (int m = 0; m < n_map; m++) mrow[m] = ns + nf + rows[m];
  CUDA_OK(cudaMemcpyAsync(t.d_ptr + nf + 1, &end, 4, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemcpyAsync(t.d_rf + ns + nf, rf.data(), 4 * (size_t)(n_segs + 1), cudaMemcpyHostToDevice, st));
  if (n_segs) CUDA_OK(cudaMemcpyAsync(t.d_segs + 4 * (size_t)ns, d_segs, 16 * (size_t)n_segs, cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemsetAsync(t.d_ps + 4 * (size_t)(ns + nf), 0, 16 * (size_t)(n_segs + 1), st));
  if (n_map) CUDA_OK(cudaMemcpyAsync(t.d_mrow + nm, mrow.data(), 4 * (size_t)n_map, cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaStreamSynchronize(st));   // (the staging vectors go out of scope)
  t.frame_node.push_back(pose_node);
  t.map_fid.insert(t.map_fid.end(), fids, fids + n_map);
  t.mrow.insert(t.mrow.end(), mrow.begin(), mrow.end());
  t.n_frames = need_f; t.n_seg = need_s; t.n_rows = need_s + need_f; t.n_map = need_m;
  t.slot_topo = 0;
  t.bound = true;
  return 0;
}
// whether `owner` still owns the handle's refresh tables (false once the caller rebound them)
bool engine_refresh_owned(pus_handle h, const void* owner) { return SV(h)->rt.owner == owner; }
// a destroyed map gives its tables up: they are unbound, and the next map's first append starts afresh
void engine_refresh_release(pus_handle h, const void* owner) {
  Solver::RefreshTables& t = SV(h)->rt;
  if (!owner || t.owner != owner) return;
  t.owner = nullptr;
  t.bound = false;
  t.n_frames = t.n_seg = t.n_rows = t.n_map = 0;
  t.frame_node.clear(); t.map_fid.clear(); t.mrow.clear();
}
}  // namespace pus

extern "C" {

// Every export starts as pus_project_to_planes does: re-upload when the topology, the host values or the measurements changed,
// otherwise only bind the device (the estimate on the device is then the one a resident solve left there).  The per-record
// table is rebuilt after a layout rebuild: one pass over the nodes (column of every live node) and one over the factors (first
// row and first value of every live factor), not Graph::node_start / factor_row per factor.
static int export_prepare(Solver* s, const char* fn) {
  if (s->g.num_factors() == 0) { g_err = std::string(fn) + ": the graph has no live factors"; return -1; }
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty || s->meas_dirty) {
    if (upload(s) < 0) return -1;
  } else if (ensure_device(s) < 0) {
    return -1;
  }
  Solver::ExportTables& x = s->xt;
  if (!x.ev_copy) CUDA_OK(cudaEventCreate(&x.ev_copy));
  if (x.topo == s->compiled_topo) return 0;
  const Graph& g = s->g;
  const Compiled& c = s->c;
  std::vector<int> col(g.nodes.size(), -1);
  long long cols = 0, rows = 0, nnz = 0;
  for (size_t i = 0; i < g.nodes.size(); i++)
    if (g.nodes[i].alive) { col[i] = (int)cols; cols += g.nodes[i].kind == NODE_POSE ? 6 : 3; }
  std::vector<int> frow(g.factors.size(), -1), fval(g.factors.size(), -1);
  x.live_row.clear();
  for (size_t f = 0; f < g.factors.size(); f++) {
    const HFactor& F = g.factors[f];
    if (!F.alive) continue;
    int ncols = 0;
    for (int k = 0; k < F.n_nodes; k++) ncols += g.nodes[F.nodes[k]].kind == NODE_POSE ? 6 : 3;
    frow[f] = (int)rows; fval[f] = (int)nnz;
    x.live_row.push_back((int)rows);
    rows += F.dim;
    nnz += (long long)F.dim * ncols;
    if (nnz > 0x7fffffffll || cols > 0x7fffffffll) {
      g_err = std::string(fn) + ": the Jacobian has more than 2^31 - 1 nonzeros or columns; its int32 indices cannot address it";
      x.topo = 0;
      return -1;
    }
  }
  x.live_row.push_back((int)rows);
  x.rows = rows; x.cols = cols; x.nnz = nnz;
  const int nrec = c.nslot + c.Epf + c.Elp;
  x.rec.assign(nrec, ExportRec{-1, -1, -1, -1});
  x.fid2rec.assign(g.factors.size(), -1);
  auto fill = [&](int q, int fid) {
    if (fid < 0) return;
    const HFactor& F = g.factors[fid];
    x.rec[q] = ExportRec{frow[fid], fval[fid], col[F.nodes[0]], F.n_nodes == 2 ? col[F.nodes[1]] : -1};
    x.fid2rec[fid] = q;
  };
  for (int e = 0; e < c.nslot; e++) fill(e, c.pp_fid[e]);
  for (int f = 0; f < c.Epf; f++) fill(c.nslot + f, c.pf_fid[f]);
  for (int f = 0; f < c.Elp; f++) fill(c.nslot + c.Epf + f, c.lp_fid[f]);
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t need = al(sizeof(ExportRec) * (size_t)std::max(nrec, 1)) + al(4 * (size_t)(rows + 1)) + al(4 * (size_t)std::max(nnz, 1ll));
  CUDA_OK(cudaSetDevice(s->device));
  if (need > x.bytes) {
    if (x.mem) { cudaStreamSynchronize(s->stream); cudaFree(x.mem); x.mem = nullptr; x.bytes = 0; }
    CUDA_OK(cudaMalloc(&x.mem, need));
    x.bytes = need;
  }
  char* base = static_cast<char*>(x.mem);
  x.d_rec = reinterpret_cast<ExportRec*>(base);
  x.d_row_ptr = reinterpret_cast<int*>(base + al(sizeof(ExportRec) * (size_t)std::max(nrec, 1)));
  x.d_col_idx = reinterpret_cast<int*>(reinterpret_cast<char*>(x.d_row_ptr) + al(4 * (size_t)(rows + 1)));
  if (nrec) CUDA_OK(cudaMemcpyAsync(x.d_rec, x.rec.data(), sizeof(ExportRec) * nrec, cudaMemcpyHostToDevice, s->stream));
  CUDA_OK(cudaStreamSynchronize(s->stream));   // (x.rec may be rebuilt before a later copy would have run)
  x.structure = false;
  x.topo = s->compiled_topo;
  return 0;
}

// evaluate records recs[0..n) (nullptr: every record) into d_err (and the Jacobian values / rhs when d_vals != nullptr);
// the kernel time goes to stats.kernel_ms
static int export_run(Solver* s, const int* d_recs, const int* d_orow, int n, double* d_err, double* d_vals, double* d_rhs) {
  const Compiled& c = s->c;
  const DevGraph& d = s->hd;
  ExportArgs a;
  a.pose_lin = d.pose_lin; a.plane_lin = d.plane_lin;
  a.pp_pose = d.pp_pose; a.pp_plane = d.pp_plane; a.pp_meas = d.pp_meas; a.pp_sinf = d.pp_sinf; a.pp_rays = d.pp_rays;
  a.pp_kind = d.pp_kind; a.n_f2 = c.n_f2;
  a.pf_i = d.pf_i; a.pf_j = d.pf_j; a.pf_meas = d.pf_meas; a.pf_sinf = d.pf_sinf;
  a.lp_plane = d.lp_plane; a.lp_meas = d.lp_meas; a.lp_sinf = d.lp_sinf;
  a.nslot = c.nslot; a.Epf = c.Epf; a.Elp = c.Elp;
  a.robust_kind = s->robust_kind; a.robust_b = s->robust_b; a.numeric = s->jac_numeric;
  a.rec = s->xt.d_rec; a.recs = d_recs; a.orow = d_orow; a.n = n;
  a.err = d_err; a.vals = d_vals; a.rhs = d_rhs;
  CUDA_OK(cudaEventRecord(s->ev0, s->stream));
  CUDA_OK(launch_export(s->stream, a));
  CUDA_OK(cudaEventRecord(s->ev1, s->stream));
  return 0;
}
// wait for the export; kernel time = ev0 -> ev1 around the evaluation, copy time = ev1 -> ev_copy (recorded here, after the
// device-to-host copies the caller enqueued)
static int export_finish(Solver* s, int launches, long long d2h_bytes) {
  CUDA_OK(cudaEventRecord(s->xt.ev_copy, s->stream));
  CUDA_OK(cudaEventSynchronize(s->xt.ev_copy));
  float ms = 0, ms2 = 0;
  CUDA_OK(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
  CUDA_OK(cudaEventElapsedTime(&ms2, s->ev1, s->xt.ev_copy));
  s->stats.kernel_ms = ms; s->stats.d2h_ms = ms2; s->stats.d2h_bytes = d2h_bytes; s->stats.gpu_launches = launches;
  return 0;
}

// the errors of every live factor into device scratch; returns the scratch pointer (nullptr on failure)
static double* export_all_errors(Solver* s, Scratch& sc, size_t extra) {
  const Solver::ExportTables& x = s->xt;
  if (!sc.reserve(Scratch::al(8 * (size_t)x.rows) + extra)) { g_err = "scratch allocation failed"; return nullptr; }
  double* d_err = sc.put<double>(nullptr, (size_t)x.rows);
  if (!d_err) { g_err = "scratch allocation failed"; return nullptr; }
  if (export_run(s, nullptr, nullptr, (int)x.rec.size(), d_err, nullptr, nullptr) < 0) return nullptr;
  return d_err;
}

// sum of squares of rows [lo, rows) of the weighted errors (fixed order); chi2 of the whole graph for lo = 0
static int export_sumsq(Solver* s, long long lo, double* out) {
  Scratch sc{s, s->stream};
  const size_t extra = Scratch::al(8 * kExportRedBlocks) + Scratch::al(8);
  double* d_err = export_all_errors(s, sc, extra);
  if (!d_err) return -1;
  double* part = sc.put<double>(nullptr, kExportRedBlocks);
  double* d_out = sc.put<double>(nullptr, 1);
  if (!part || !d_out) { g_err = "scratch allocation failed"; return -1; }
  CUDA_OK(launch_sumsq(s->stream, d_err, lo, s->xt.rows, part, d_out));
  CUDA_OK(cudaMemcpyAsync(out, d_out, 8, cudaMemcpyDeviceToHost, s->stream));
  return export_finish(s, 3, 8);
}

long long pus_weighted_errors(pus_handle h, double* out, long long capacity) {
  NEED(h);
  Solver* s = SV(h);
  if (export_prepare(s, "pus_weighted_errors") < 0) return -1;
  const long long rows = s->xt.rows;
  if (!out) return rows;   // size query
  if (capacity < rows) { g_err = "pus_weighted_errors: capacity " + std::to_string(capacity) + " < " + std::to_string(rows) + " rows"; return -1; }
  Scratch sc{s, s->stream};
  double* d_err = export_all_errors(s, sc, 0);
  if (!d_err) return -1;
  CUDA_OK(cudaMemcpyAsync(out, d_err, 8 * (size_t)rows, cudaMemcpyDeviceToHost, s->stream));
  if (export_finish(s, 1, 8 * rows) < 0) return -1;
  return rows;
}

int pus_factor_errors(pus_handle h, int n, const int* fids, double* out) {
  NEED(h);
  Solver* s = SV(h);
  if (n < 0 || (n > 0 && (!fids || !out))) { g_err = "pus_factor_errors: bad arguments"; return -1; }
  for (int i = 0; i < n; i++)
    if (!s->g.ok_factor(fids[i])) { g_err = "pus_factor_errors: bad factor id " + std::to_string(fids[i]); return -1; }
  if (export_prepare(s, "pus_factor_errors") < 0) return -1;
  if (n == 0) return 0;
  std::vector<int> recs(n), orow(n);
  int total = 0;
  for (int i = 0; i < n; i++) {
    recs[i] = s->xt.fid2rec[fids[i]];
    orow[i] = total;
    total += s->g.factors[fids[i]].dim;
  }
  Scratch sc{s, s->stream};
  if (!sc.reserve(2 * Scratch::al(4 * (size_t)n) + Scratch::al(8 * (size_t)total))) { g_err = "scratch allocation failed"; return -1; }
  int* d_recs = sc.put(recs.data(), n);
  int* d_orow = sc.put(orow.data(), n);
  double* d_err = sc.put<double>(nullptr, total);
  if (!d_recs || !d_orow || !d_err) { g_err = "scratch allocation failed"; return -1; }
  if (export_run(s, d_recs, d_orow, n, d_err, nullptr, nullptr) < 0) return -1;
  CUDA_OK(cudaMemcpyAsync(out, d_err, 8 * (size_t)total, cudaMemcpyDeviceToHost, s->stream));
  if (export_finish(s, 1, 8ll * total) < 0) return -1;   // (also keeps recs / orow alive until their copies ran)
  return total;
}

int pus_jacobian_dims(pus_handle h, long long* rows, long long* cols) {
  NEED(h);
  const Solver* s = SV(h);
  if (s->xt.topo != 0 && s->xt.topo == s->compiled_topo && s->compiled_topo == s->g.topo_version) {   // the export's tables are current
    if (rows) *rows = s->xt.rows;
    if (cols) *cols = s->xt.cols;
    return 0;
  }
  const Graph& g = s->g;   // (no export since the last structural edit: one pass over the host graph)
  long long r = 0, c = 0;
  for (const HFactor& f : g.factors) if (f.alive) r += f.dim;
  for (const HNode& n : g.nodes) if (n.alive) c += n.kind == NODE_POSE ? 6 : 3;
  if (rows) *rows = r;
  if (cols) *cols = c;
  return 0;
}

long long pus_jacobian(pus_handle h, int* row_ptr, int* col_idx, double* values, double* rhs, long long cap_nnz) {
  NEED(h);
  Solver* s = SV(h);
  if (export_prepare(s, "pus_jacobian") < 0) return -1;
  Solver::ExportTables& x = s->xt;
  if (cap_nnz == 0) return x.nnz;   // size query
  if (cap_nnz < x.nnz) { g_err = "pus_jacobian: cap_nnz " + std::to_string(cap_nnz) + " < " + std::to_string(x.nnz) + " nonzeros"; return -1; }
  cudaStream_t st = s->stream;
  const int nrec = (int)x.rec.size();
  if ((row_ptr || col_idx) && !x.structure) {   // once per layout
    CUDA_OK(launch_export_structure(st, x.d_rec, nrec, s->c.nslot, s->c.Epf, s->hd.pf_j, (int)x.rows, (int)x.nnz, x.d_row_ptr, x.d_col_idx));
    x.structure = true;
  }
  Scratch sc{s, st};
  double* d_vals = nullptr;
  double* d_rhs = nullptr;
  CUDA_OK(cudaEventRecord(s->ev0, st));
  CUDA_OK(cudaEventRecord(s->ev1, st));
  if (values || rhs) {
    if (!sc.reserve(2 * Scratch::al(8 * (size_t)x.rows) + Scratch::al(8 * (size_t)x.nnz))) { g_err = "scratch allocation failed"; return -1; }
    double* d_err = sc.put<double>(nullptr, (size_t)x.rows);
    d_rhs = sc.put<double>(nullptr, (size_t)x.rows);
    d_vals = sc.put<double>(nullptr, (size_t)x.nnz);
    if (!d_err || !d_rhs || !d_vals) { g_err = "scratch allocation failed"; return -1; }
    if (export_run(s, nullptr, nullptr, nrec, d_err, d_vals, d_rhs) < 0) return -1;
  }
  long long bytes = 0;
  if (row_ptr) { CUDA_OK(cudaMemcpyAsync(row_ptr, x.d_row_ptr, 4 * (size_t)(x.rows + 1), cudaMemcpyDeviceToHost, st)); bytes += 4 * (x.rows + 1); }
  if (col_idx) { CUDA_OK(cudaMemcpyAsync(col_idx, x.d_col_idx, 4 * (size_t)x.nnz, cudaMemcpyDeviceToHost, st)); bytes += 4 * x.nnz; }
  if (values) { CUDA_OK(cudaMemcpyAsync(values, d_vals, 8 * (size_t)x.nnz, cudaMemcpyDeviceToHost, st)); bytes += 8 * x.nnz; }
  if (rhs) { CUDA_OK(cudaMemcpyAsync(rhs, d_rhs, 8 * (size_t)x.rows, cudaMemcpyDeviceToHost, st)); bytes += 8 * x.rows; }
  if (export_finish(s, (values || rhs) ? 1 : 0, bytes) < 0) return -1;
  return x.nnz;
}

int pus_normalized_chi2(pus_handle h, double* out) {
  NEED(h);
  Solver* s = SV(h);
  if (!out) { g_err = "pus_normalized_chi2: null output"; return -1; }
  if (export_prepare(s, "pus_normalized_chi2") < 0) return -1;
  double chi2 = 0;
  if (export_sumsq(s, 0, &chi2) < 0) return -1;
  *out = chi2 / (double)(s->xt.rows - s->xt.cols);   // as Slam.cpp:287-289 (no guard for rows <= columns there either)
  return 0;
}

int pus_local_chi2(pus_handle h, int last_n, double* out) {
  NEED(h);
  Solver* s = SV(h);
  if (!out) { g_err = "pus_local_chi2: null output"; return -1; }
  if (export_prepare(s, "pus_local_chi2") < 0) return -1;
  const std::vector<int>& lr = s->xt.live_row;   // nlive + 1 entries
  const int nlive = (int)lr.size() - 1;
  const long long lo = last_n <= 0 ? lr[nlive] : lr[std::max(0, nlive - last_n)];
  return export_sumsq(s, lo, out);
}

// ---- graph text I/O (host only) ----
int pus_save_graph(pus_handle h, const char* path, int precision) {
  NEED(h);
  Solver* s = SV(h);
  if (sync_measurements_to_host(s) < 0) return -1;
  FILE* fp = std::fopen(path, "wb");
  if (!fp) { g_err = std::string("pus_save_graph: cannot open ") + path; return -1; }
  const int prec = precision > 0 ? precision : 6;
  auto num = [&](double v) { char b[64]; std::snprintf(b, sizeof b, "%.*g", prec, v); return std::string(b); };
  auto pose_str = [&](const double* p7) {   // Pose3d::write, Pose3d.h:169-172
    double yaw, pitch, roll;
    quat_to_euler(p7 + 3, yaw, pitch, roll);
    return "(" + num(p7[0]) + ", " + num(p7[1]) + ", " + num(p7[2]) + "; " + num(yaw) + ", " + num(pitch) + ", " + num(roll) + ")";
  };
  auto xyzypr_str = [&](const double* m) {
    return "(" + num(m[0]) + ", " + num(m[1]) + ", " + num(m[2]) + "; " + num(m[3]) + ", " + num(m[4]) + ", " + num(m[5]) + ")";
  };
  auto plane_str = [&](const double* v) { return "(" + num(v[0]) + ", " + num(v[1]) + ", " + num(v[2]) + "; " + num(v[3]) + ")"; };
  static const char* kFactorName[4] = {"Pose3d_Factor", "Pose3d_Pose3d_Factor", "Pose3d_Plane3d_Factor", "Pose3d_Factor"};
  for (size_t f = 0; f < s->g.factors.size(); f++) {   // Graph::write: factors first (Graph.h:121-125)
    const HFactor& F = s->g.factors[f];
    if (!F.alive) continue;
    std::string line = kFactorName[F.kind];
    for (int i = 0; i < F.n_nodes; i++) line += " " + std::to_string(F.nodes[i]);
    line += " " + (F.dim == 3 ? plane_str(F.meas) : xyzypr_str(F.meas)) + " {";
    const int ne = F.dim * (F.dim + 1) / 2;
    for (int i = 0; i < ne; i++) line += (i ? "," : "") + num(F.sinf[i]);
    line += "}\n";
    std::fputs(line.c_str(), fp);
  }
  for (size_t n = 0; n < s->g.nodes.size(); n++) {     // then nodes (Graph.h:126-130)
    const HNode& N = s->g.nodes[n];
    if (!N.alive) continue;
    std::string line = std::string(N.kind == NODE_POSE ? "Pose3d_Node " : "Plane3d_Node ") + std::to_string(n) + " " +
                       (N.kind == NODE_POSE ? pose_str(N.v) : plane_str(N.v)) + "\n";
    std::fputs(line.c_str(), fp);
  }
  std::fclose(fp);
  return 0;
}

int pus_load_isam_dataset(pus_handle h, const char* path, int* n_poses, int* n_factors) {
  NEED(h);
  Solver* s = SV(h);
  FILE* fp = std::fopen(path, "rb");
  if (!fp) { g_err = std::string("pus_load_isam_dataset: cannot open ") + path; return -1; }
  std::map<unsigned, int> mapper;   // dataset pose index -> node id (Loader's _pose_mapper)
  int added_p = 0, added_f = 0, lineno = 0, rc = 0;
  char buf[4096];
  auto node_of = [&](unsigned idx, bool create) {
    auto it = mapper.find(idx);
    if (it != mapper.end()) return it->second;
    if (!create) return -1;
    const int id = s->g.add_node(NODE_POSE, nullptr);
    mapper[idx] = id;
    added_p++;
    return id;
  };
  while (rc == 0 && std::fgets(buf, sizeof buf, fp)) {
    lineno++;
    char key[64];
    int off = 0;
    if (std::sscanf(buf, "%63s%n", key, &off) != 1) continue;
    const std::string kw(key);
    const char* args = buf + off;
    if (kw == "EDGE3") {   // Loader.cpp:316-365
      unsigned i0, i1;
      double x, y, z, roll, pitch, yaw, I[21];
      int res = std::sscanf(args, "%u %u %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg %lg",
                            &i0, &i1, &x, &y, &z, &roll, &pitch, &yaw, I, I + 1, I + 2, I + 3, I + 4, I + 5, I + 6, I + 7, I + 8, I + 9, I + 10,
                            I + 11, I + 12, I + 13, I + 14, I + 15, I + 16, I + 17, I + 18, I + 19, I + 20);
      if (res != 29 && res != 8) { g_err = "EDGE3: parse error at line " + std::to_string(lineno); rc = -1; break; }
      double meas[6] = {x, y, z, yaw, pitch, roll};   // Pose3d(x, y, z, yaw, pitch, roll): the file stores roll pitch yaw
      double si[21];
      if (res == 8) {
        int q = 0;
        for (int r = 0; r < 6; r++) for (int cc = r; cc < 6; cc++) si[q++] = (r == cc) ? 1.0 : 0.0;
      } else {
        // rows 0-2 as given; rotational block reversed: [i66 i56 i46; 0 i55 i45; 0 0 i44] (Loader.cpp:343-345)
        const double i44 = I[15], i45 = I[16], i46 = I[17], i55 = I[18], i56 = I[19], i66 = I[20];
        const double full[21] = {I[0], I[1], I[2], I[3], I[4], I[5], I[6], I[7], I[8], I[9], I[10], I[11], I[12], I[13], I[14],
                                 i66, i56, i46, i55, i45, i44};
        std::memcpy(si, full, sizeof full);
      }
      unsigned from, to;
      if (i0 < i1) { to = i1; from = i0; }
      else {   // reverse the constraint: delta = Pose3d(delta.oTw())  (Loader.cpp:349-356)
        double p7[7], Ti[16], inv7[7], yw, pt, rl;
        pose_from_xyzypr(meas, p7);
        pose_to_Tinv(p7, Ti);
        T_to_pose(Ti, inv7);
        quat_to_euler(inv7 + 3, yw, pt, rl);
        meas[0] = inv7[0]; meas[1] = inv7[1]; meas[2] = inv7[2]; meas[3] = yw; meas[4] = pt; meas[5] = rl;
        to = i0; from = i1;
      }
      if (mapper.empty()) {   // Loader::add_prior: first pose = dataset index 0, prior at the origin, sqrtinf 100 I
        const int id0 = node_of(0, true);
        double zero[6] = {0, 0, 0, 0, 0, 0}, s100[21];
        int q = 0;
        for (int r = 0; r < 6; r++) for (int cc = r; cc < 6; cc++) s100[q++] = (r == cc) ? 100.0 : 0.0;
        if (s->g.add_pose_prior(id0, zero, s100) < 0) { g_err = s->g.err; rc = -1; break; }
        added_f++;
      }
      const int a = node_of(from, false), b = node_of(to, true);
      if (a < 0) { g_err = "EDGE3: pose " + std::to_string(from) + " not seen before line " + std::to_string(lineno); rc = -1; break; }
      if (s->g.add_odometry(a, b, meas, si) < 0) { g_err = s->g.err; rc = -1; break; }
      added_f++;
    } else if (kw == "POSE3D_INIT") {   // Loader.cpp:366-383
      unsigned idx;
      double x, y, z, roll, pitch, yaw;
      if (std::sscanf(args, "%u %lg %lg %lg %lg %lg %lg", &idx, &x, &y, &z, &roll, &pitch, &yaw) != 7) {
        g_err = "POSE3D_INIT: parse error at line " + std::to_string(lineno); rc = -1; break;
      }
      if (mapper.find(idx) == mapper.end()) {
        const double v[6] = {x, y, z, yaw, pitch, roll};
        double p7[7];
        pose_from_xyzypr(v, p7);
        const int id = s->g.add_node(NODE_POSE, p7);
        mapper[idx] = id;
        added_p++;
      }
    } else if (kw == "EDGE3_INIT" || kw == "POSE3D_TRUE" || kw == "EDGE3_TRUE" || kw == "SOLVE") {
      continue;   // as upstream (Loader.cpp:385-394)
    } else if (kw[0] == '#') {
      continue;
    } else {
      g_err = "keyword '" + kw + "' (line " + std::to_string(lineno) + ") is not part of the 3-D pose-graph grammar this back end loads";
      rc = -1;
    }
  }
  std::fclose(fp);
  if (n_poses) *n_poses = added_p;
  if (n_factors) *n_factors = added_f;
  return rc;
}

// order of the direct solve's system without padding (6 N, then 3 per bordered plane), and row r's row in the padded layout
static int direct_order(const Solver* s) { return 6 * s->c.N + 3 * (int)s->dt.border.size(); }
static int direct_row(const Solver* s, int r) { return r < 6 * s->c.N ? r : 48 * s->dt.nbp + r - 6 * s->c.N; }

// ---- marginal covariances (DESIGN.md section 5.4) ----
// Refuse every handle but kind 2 in ND order; re-upload as the exports do; build the layout's tables on the first call and
// check them against the budget before anything is allocated or launched.
static int cov_prepare(Solver* s, const char* fn) {
  if (s->linear_solver != 2 || s->ordering != 1) {
    g_err = std::string(fn) + ": covariances are recovered from the nested-dissection factor only; call pus_set_linear_solver(h, 2) "
            "and pus_set_direct_ordering(h, 1) (this handle: linear solver kind " + std::to_string(s->linear_solver) +
            ", ordering " + std::to_string(s->ordering) + ")";
    return -1;
  }
  if (s->g.num_factors() == 0) { g_err = std::string(fn) + ": the graph has no live factors"; return -1; }
  if (!s->uploaded || s->compiled_topo != s->g.topo_version || s->values_dirty || s->meas_dirty) {
    if (upload(s) < 0) return -1;
  } else if (ensure_device(s) < 0) {
    return -1;
  }
  Solver::CovState& cv = s->cov;
  if (cv.t.topo == s->compiled_topo) return 0;
  cv.valid = false;
  std::string err;
  if (!build_cov(s->c, s->dt, cv.t, err)) { g_err = std::string(fn) + ": " + err; return -1; }
  const size_t sig = (size_t)s->dt.ntile() * kAcTile * 8, need = sig + cv.t.dev.size() * 4;
  CUDA_OK(cudaSetDevice(s->device));
  if (need > cv.bytes) {
    if (cv.mem) { cudaStreamSynchronize(s->stream); cudaFree(cv.mem); cv.mem = nullptr; cv.bytes = 0; }
    if (cudaMalloc(&cv.mem, need) != cudaSuccess) {
      cudaGetLastError();
      g_err = std::string(fn) + ": cannot allocate " + std::to_string(need) + " bytes for the Sigma tiles";
      cv.t = CovTables();
      return -1;
    }
    cv.bytes = need;
  }
  CUDA_OK(cudaMemcpyAsync(static_cast<char*>(cv.mem) + sig, cv.t.dev.data(), cv.t.dev.size() * 4, cudaMemcpyHostToDevice, s->stream));
  CUDA_OK(cudaStreamSynchronize(s->stream));
  cv.t.topo = s->compiled_topo;
  return 0;
}

// One covariance launch: Sigma first when it is not valid, then the records `rec` (header, gather records, columns, column
// records; see Phase::cov_gather / cov_columns) into nout doubles.  The handle's results, statistics and estimate are kept.
static int cov_run(Solver* s, const char* fn, const std::vector<int>& rec, size_t nout, double* out) {
  Solver::CovState& cv = s->cov;
  Scratch sc{s, s->stream};
  if (!sc.reserve(Scratch::al(4 * rec.size()) + Scratch::al(8 * std::max<size_t>(nout, 1)))) { g_err = "scratch allocation failed"; return -1; }
  int* d_rec = sc.put(rec.data(), rec.size());
  double* d_out = sc.put<double>(nullptr, nout);
  if (!d_rec || !d_out) { g_err = "scratch allocation failed"; return -1; }
  const bool compute = !cv.valid;
  s->hd.Sig = static_cast<double*>(cv.mem);
  s->hd.dcov = reinterpret_cast<const int*>(static_cast<char*>(cv.mem) + (size_t)s->dt.ntile() * kAcTile * 8);
  s->hd.crec = d_rec; s->hd.covout = d_out;
  const LmResult res = s->res;
  const pus_stats st = s->stats;
  const int rc = launch(&s, 1, MODE_COV, 0, compute ? 1 : 0, 0.0);
  const float ms = s->stats.kernel_ms;
  s->res = res; s->stats = st; s->stats.kernel_ms = ms;
  s->hd.crec = nullptr; s->hd.covout = nullptr;
  if (rc < 0) { cv.valid = false; return -1; }
  if (compute) {
    unsigned flag = 0;
    CUDA_OK(cudaMemcpy(&flag, s->hd.dflag, sizeof(flag), cudaMemcpyDeviceToHost));
    if (flag) {
      g_err = std::string(fn) + ": the undamped reduced system has a non-positive pivot, so J^T J is not positive definite at the "
              "estimate (for example a graph without a pose prior, whose gauge is free); nothing is stored";
      return -1;
    }
    cv.valid = true;
  }
  if (nout) CUDA_OK(cudaMemcpy(out, d_out, nout * 8, cudaMemcpyDeviceToHost));
  return 0;
}

// a live node: its compiled index, its dimension, its first row in the bordered order (-1: an eliminated plane)
struct CovNode { bool pose; int idx, dim, row; };
static bool cov_node(const Solver* s, int id, CovNode& n, const char* fn) {
  const Graph& g = s->g;
  if (id < 0 || id >= (int)g.nodes.size() || !g.nodes[id].alive) { g_err = std::string(fn) + ": bad node id " + std::to_string(id); return false; }
  n.pose = g.nodes[id].kind == NODE_POSE;
  n.idx = s->c.node_idx[id];
  n.dim = n.pose ? 6 : 3;
  n.row = cov_row(s->dt, n.pose, n.idx);
  return true;
}

// records of the block (a, b), dim(a) x dim(b) row-major at out[o]: from Sigma's tiles when both nodes are kept and their tile
// is stored, else one column solve per column of b (columns shared by every block with the same right-hand node)
struct CovRecs {
  std::vector<int> gather, cols, crec;
  std::map<int, int> col_of;   // right-hand node id -> its first column
};
static void cov_block(const Solver* s, const CovNode& a, const CovNode& b, int bid, int o, CovRecs& R) {
  const DirectTables& dt = s->dt;
  const std::vector<int>& ip = dt.inc_ptr;
  int tile = 0, off = 0, flag = 0;
  if (a.row >= 0 && b.row >= 0 && cov_block_at(dt, a.row, b.row, tile, off, flag)) {
    for (int p = 0; p < a.dim; p++)
      for (int q = 0; q < b.dim; q++)
        R.gather.insert(R.gather.end(), {0, o + p * b.dim + q, -1, tile, flag ? off + q * kAcLd + p : off + p * kAcLd + q, 0, 0, 0});
    return;
  }
  auto it = R.col_of.find(bid);
  if (it == R.col_of.end()) {
    it = R.col_of.emplace(bid, (int)(R.cols.size() / 6)).first;
    for (int q = 0; q < b.dim; q++) {
      if (b.row >= 0) {
        const int r = b.row + q;   // its entry of the right-hand side: 6 N pose rows, then 3 per bordered plane
        R.cols.insert(R.cols.end(), {0, r < 6 * s->c.N ? r : 6 * s->c.N + r - 48 * dt.nbp, 0, 0, 0, 0});
      } else {
        R.cols.insert(R.cols.end(), {1, ip[b.idx], ip[b.idx + 1], q, 0, 0});
      }
    }
  }
  // (column records are grouped by column in cov_finish)
  for (int q = 0; q < b.dim; q++)
    for (int p = 0; p < a.dim; p++) {
      const int col = it->second + q, oo = o + p * b.dim + q;
      if (a.row >= 0) R.crec.insert(R.crec.end(), {col, 0, oo, a.row + p, 0, 0, 0});
      else R.crec.insert(R.crec.end(), {col, 1, oo, ip[a.idx], ip[a.idx + 1], p, (!b.pose && b.row < 0 && b.idx == a.idx) ? a.idx * 9 + p * 3 + q : -1});
    }
}
// the packed record array of cov_run: header, gather records, columns (with their record ranges), column records by column
static std::vector<int> cov_finish(CovRecs& R) {
  const int ncol = (int)(R.cols.size() / 6), ng = (int)(R.gather.size() / 8);
  std::vector<std::vector<int>> by(ncol);
  for (size_t k = 0; k < R.crec.size(); k += 7) by[R.crec[k]].insert(by[R.crec[k]].end(), R.crec.begin() + k + 1, R.crec.begin() + k + 7);
  std::vector<int> out = {ng, ncol, 8, 0, 0, 0, 0, 0};
  out.insert(out.end(), R.gather.begin(), R.gather.end());
  out[3] = (int)out.size();
  const size_t cbase = out.size();
  out.insert(out.end(), R.cols.begin(), R.cols.end());
  out[4] = (int)out.size();
  int e = 0;
  for (int k = 0; k < ncol; k++) {
    out[cbase + 6 * k + 4] = e;
    out.insert(out.end(), by[k].begin(), by[k].end());
    e += (int)(by[k].size() / 6);
    out[cbase + 6 * k + 5] = e;
  }
  return out;
}

int pus_marginal_covariances(pus_handle h, int n, const int* ids, double* out) {
  NEED(h);
  Solver* s = SV(h);
  const char* fn = "pus_marginal_covariances";
  if (n < 0) { g_err = std::string(fn) + ": n < 0"; return -1; }
  if (cov_prepare(s, fn) < 0) return -1;
  CovRecs R;
  int o = 0;
  for (int k = 0; k < n; k++) {
    CovNode a;
    if (!cov_node(s, ids[k], a, fn)) return -1;
    if (a.row >= 0) {
      cov_block(s, a, a, ids[k], o, R);
    } else {   // an eliminated plane: entries r <= c, mirrored
      for (int r = 0; r < 3; r++)
        for (int cc = r; cc < 3; cc++) R.gather.insert(R.gather.end(), {1, o + 3 * r + cc, r == cc ? -1 : o + 3 * cc + r, a.idx, r, cc, 0, 0});
    }
    o += a.dim * a.dim;
  }
  if (cov_run(s, fn, cov_finish(R), (size_t)o, out) < 0) return -1;
  return o;
}

long long pus_covariance_blocks(pus_handle h, int n_pairs, const int* id_pairs, double* out) {
  NEED(h);
  Solver* s = SV(h);
  const char* fn = "pus_covariance_blocks";
  if (n_pairs < 0) { g_err = std::string(fn) + ": n_pairs < 0"; return -1; }
  if (cov_prepare(s, fn) < 0) return -1;
  CovRecs R;
  long long o = 0;
  for (int k = 0; k < n_pairs; k++) {
    CovNode a, b;
    if (!cov_node(s, id_pairs[2 * k], a, fn) || !cov_node(s, id_pairs[2 * k + 1], b, fn)) return -1;
    if (o + a.dim * b.dim > 0x7fffffffll) { g_err = std::string(fn) + ": more than 2^31 - 1 output values in one call"; return -1; }
    cov_block(s, a, b, id_pairs[2 * k + 1], (int)o, R);
    o += a.dim * b.dim;
  }
  if (cov_run(s, fn, cov_finish(R), (size_t)o, out) < 0) return -1;
  return o;
}

long long pus_debug_fetch(pus_handle h, const char* name, double* out, long long cap) {
  NEED(h);
  Solver* s = SV(h);
  const Compiled& c = s->c;
  std::string nm(name);
  cudaSetDevice(s->device);
  auto ints = [&](const std::vector<int>& v) -> long long {
    if ((long long)v.size() <= cap) for (size_t i = 0; i < v.size(); i++) out[i] = v[i];
    return (long long)v.size();
  };
  if (nm == "pp_fid") return ints(c.pp_fid);
  if (nm == "pp_pose") return ints(c.pp_pose);
  if (nm == "pp_plane") return ints(c.pp_plane);
  if (nm == "pf_fid") return ints(c.pf_fid);
  if (nm == "pose_node") return ints(c.pose_node);
  if (nm == "plane_node") return ints(c.plane_node);
  if (nm == "pl2pm") return ints(c.pl2pm);
  if (nm == "pm_part") return ints(c.pm_part);
  if (nm == "pl_part") return ints(c.pl_part);
  if (nm == "ypart_ptr") return ints(c.ypart_ptr);
  if (nm == "upart_ptr") return ints(c.upart_ptr);
  if (nm == "ce_node") return ints(c.ce_node);
  if (nm == "ce_plane") return ints(c.ce_plane);
  if (nm == "ce_lo") return ints(c.ce_lo);
  if (nm == "ce_hi") return ints(c.ce_hi);
  if (nm == "grp_plane") return ints(c.grp_plane);
  if (nm == "grp_mem") return ints(c.grp_mem);
  if (nm == "grp_mem_ptr") return ints(c.grp_mem_ptr);
  if (nm == "blk_grp_ptr") return ints(c.blk_grp_ptr);
  if (nm == "blk_part_ptr") return ints(c.blk_part_ptr);
  if (nm == "blk_ovf") return ints(c.blk_ovf);   // (empty: no pose block over the pose phase's shared-memory limits)
  // direct mode: the host tables of the assembly of S
  if (nm == "dinc_pose") return ints(s->dt.inc_pose);
  if (nm == "dinc_plane") return ints(s->dt.inc_plane);
  if (nm == "dinc_lo") return ints(s->dt.inc_lo);
  if (nm == "dinc_hi") return ints(s->dt.inc_hi);
  if (nm == "dlp_ptr") return ints(s->dt.lp_ptr);
  if (nm == "dlp_a") return ints(s->dt.lp_a);
  if (nm == "dlp_b") return ints(s->dt.lp_b);
  if (nm == "dfp_ptr") return ints(s->dt.fp_ptr);
  if (nm == "dfp_f") return ints(s->dt.fp_f);
  // band mode: the bordered planes, the first tile column of every tile row, and the device bytes of the solve
  if (nm == "bborder") return ints(s->dt.border);
  if (nm == "bfirst") return ints(s->dt.first);
  if (nm == "bbytes") { if (cap >= 1) out[0] = (double)s->dt.bytes; return 1; }
  // nested-dissection layout: the tile order (new column -> original tile), the elimination tree, L's pattern, the levels,
  // the tile storage (per column its diagonal tile's index; per tile its row and column) and the update lists
  if (nm == "ndtile") return ints(s->dt.nd_perm);
  if (nm == "ndparent") return ints(s->dt.nd_parent);
  if (nm == "ndcptr") return ints(s->dt.nd_cptr);
  if (nm == "ndcrow") return ints(s->dt.nd_crow);
  if (nm == "ndlevel") return ints(s->dt.nd_level);
  if (nm == "ndtoff") return ints(s->dt.nd_toff);
  if (nm == "ndtrow") return ints(s->dt.nd_trow);
  if (nm == "ndtcol") return ints(s->dt.nd_tcol);
  if (nm == "nduptr") return ints(s->dt.nd_uptr);
  if (nm == "ndupd") return ints(s->dt.nd_upd);
  // marginal covariances of the ND layout (built here from the current tables): the selected-inversion list of every stored
  // tile, the plane incidence ranges, the eliminated planes' observer-pair lists and the device bytes
  if (nm.compare(0, 3, "cov") == 0) {
    if (s->dt.order != 1) { g_err = nm + ": not a nested-dissection layout"; return -1; }
    CovTables t;
    std::string err;
    if (!build_cov(c, s->dt, t, err)) { g_err = err; return -1; }
    if (nm == "covsptr") return ints(t.sel_ptr);
    if (nm == "covsel") return ints(t.sel);
    if (nm == "covincptr") return ints(s->dt.inc_ptr);
    if (nm == "covpptr") return ints(t.pair_ptr);
    if (nm == "covpair") return ints(t.pair);
    if (nm == "covbytes") { if (cap >= 1) out[0] = (double)t.bytes; return 1; }
  }
  if (nm == "pf_i") return ints(c.pf_i);
  if (nm == "pf_j") return ints(c.pf_j);
  if (nm == "pl_pose") return ints(c.pl_pose);
  if (nm == "pl_ptr") return ints(c.pl_ptr);
  if (nm == "dims") {
    double d[12] = {(double)c.N, (double)c.M, (double)c.Epl, (double)c.Epf, (double)c.Elp, (double)c.ntile, (double)c.nblk, (double)c.nc, (double)c.nce, (double)c.ngrp, (double)c.nslot, (double)c.ntile_pl};
    if (cap >= 12) std::memcpy(out, d, sizeof(d));
    if (cap >= 14) { out[12] = c.SP; out[13] = c.nc_pad; }
    if (cap >= 18) { out[14] = c.levels; out[15] = c.nc2; out[16] = c.ng2; out[17] = c.nce2; }
    return cap >= 18 ? 18 : (cap >= 14 ? 14 : 12);
  }
  if (nm == "path") {   // what the kernel reported of the last debug launch: PathBit flags, team size, levels, SP, most owned blocks
    for (int k = 0; k < 5 && k < cap; k++) out[k] = (double)s->path[k];
    return 5;
  }
  if (!s->uploaded) { g_err = "nothing uploaded"; return -1; }
  if (nm == "W" || nm == "Wt") {  // de-tiled: [slots][18] in pose-major slot order (W) or plane-major order (Wt)
    const bool pm = (nm == "W");
    size_t nt = pm ? c.ntile : c.ntile_pl, n = nt * kWStride;
    std::vector<double> tmp(n);
    if (cudaMemcpy(tmp.data(), pm ? s->hd.W : s->hd.Wt, n * 8, cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
    long long cnt = (long long)nt * 32 * 18;
    if (cnt <= cap)
      for (size_t e = 0; e < nt * 32; e++)
        for (int k = 0; k < 18; k++) out[e * 18 + k] = tmp[(e >> 5) * kWStride + k * 32 + (e & 31)];
    return cnt;
  }
  if (nm == "Sdir" || nm == "Ldir") {   // direct mode: S after the assembly (debug stage 4) or L after the factorization, n x n
    if (s->linear_solver == 0) { g_err = "not in direct linear-solver mode"; return -1; }
    const DirectTables& dt = s->dt;
    const int n = direct_order(s);   // (band: 6 N pose rows, then 3 per bordered plane, padding stripped)
    const size_t total = (size_t)dt.ntile() * kAcTile;
    std::vector<double> tmp(total);
    if (cudaMemcpy(tmp.data(), s->hd.Sd, total * 8, cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
    const long long cnt = (long long)n * n;
    if (cnt <= cap) {   // Sdir in the bordered order; Ldir, the factor of P S P^T, in the factor's order
      std::vector<int> nr(n), rows(n);
      for (int r = 0; r < n; r++) { nr[r] = dt.row(direct_row(s, r)); rows[r] = r; }
      if (nm == "Ldir") std::sort(rows.begin(), rows.end(), [&](int x, int y) { return nr[x] < nr[y]; });
      for (int a = 0; a < n; a++)
        for (int b = 0; b < n; b++) {
          const int I = std::max(nr[rows[a]], nr[rows[b]]), J = std::min(nr[rows[a]], nr[rows[b]]);
          const int t = (b > a) ? -1 : dt.tile(I / 48, J / 48);
          out[(size_t)a * n + b] = t < 0 ? 0.0 : tmp[(size_t)t * kAcTile + (I % 48) * kAcLd + J % 48];
        }
    }
    return cnt;
  }
  if (nm == "dflag") {   // direct mode: 1 when the last factorization met a non-positive pivot, else 0
    if (s->linear_solver == 0) { g_err = "not in direct linear-solver mode"; return -1; }
    unsigned f = 0;
    if (cudaMemcpy(&f, s->hd.dflag, sizeof(f), cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
    if (cap >= 1) out[0] = f ? 1.0 : 0.0;
    return 1;
  }
  if (nm == "delta") {   // [x (6 N) | dl (3 M)] of the last linear solve
    const long long cnt = 6ll * c.N + 3ll * c.M;
    if (cnt <= cap) {
      if (c.N && cudaMemcpy(out, s->hd.x, (size_t)c.N * 48, cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
      if (c.M && cudaMemcpy(out + 6 * c.N, s->hd.dl, (size_t)c.M * 24, cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
    }
    return cnt;
  }
  if (nm == "Acinv") {  // de-tiled: row-major ldm x ldm, the stored fp32 values widened
    const int ldm = 6 * c.nc_pad;
    const size_t n = ac_elems(ldm);
    std::vector<float> tmp(n);
    if (cudaMemcpy(tmp.data(), s->hd.Ac, n * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
    long long cnt = (long long)ldm * ldm;
    if (cnt <= cap)
      for (int r = 0; r < ldm; r++)
        for (int q = 0; q < ldm; q++) out[(size_t)r * ldm + q] = tmp[ac_index(ldm, r, q)];
    return cnt;
  }
  auto it = s->named.find(nm);
  if (it == s->named.end()) { g_err = "unknown buffer " + nm; return -1; }
  long long cnt = (long long)it->second.second;
  if (cnt <= cap && cnt > 0)
    if (cudaMemcpy(out, it->second.first, (size_t)cnt * 8, cudaMemcpyDeviceToHost) != cudaSuccess) { g_err = "memcpy"; return -1; }
  return cnt;
}
long long pus_debug_store(pus_handle h, const char* name, const double* in, long long count) {
  NEED(h);
  Solver* s = SV(h);
  s->cov.valid = false;
  cudaSetDevice(s->device);
  if (std::string(name) == "Sdir") {   // direct mode: a dense row-major S (n x n) for debug stage 5, laid out as direct_assemble does
    if (s->linear_solver == 0) { g_err = "Sdir: not in direct linear-solver mode"; return -1; }
    if (!s->uploaded) { g_err = "Sdir: call pus_upload first"; return -1; }
    const DirectTables& dt = s->dt;
    const int nb = dt.nb, n = direct_order(s);
    if (count != (long long)n * n) {
      g_err = s->linear_solver == 1 ? "Sdir: expected (6 N)^2 = " + std::to_string((long long)n * n) + " elements"
                                    : "Sdir: expected (6 N + 3 B)^2 = " + std::to_string((long long)n * n) + " elements";
      return -1;
    }
    std::vector<int> orig(48 * nb, -1);   // row in the factor's order -> row of the stored matrix (-1: padding)
    for (int r = 0; r < n; r++) orig[dt.row(direct_row(s, r))] = r;
    for (int r = 0; r < n; r++)
      for (int q = 0; q < r; q++) {
        const int pr = dt.row(direct_row(s, r)), pq = dt.row(direct_row(s, q));
        if (in[(size_t)r * n + q] != 0.0 && dt.tile(std::max(pr, pq) / 48, std::min(pr, pq) / 48) < 0) {
          g_err = "Sdir: entry (" + std::to_string(r) + ", " + std::to_string(q) + ") lies outside " +
                  (dt.order == 1 ? "the nested-dissection pattern" : "the band layout's envelope");
          return -1;
        }
      }
    std::vector<double> tiles((size_t)dt.ntile() * kAcTile, 0.0);   // the lower half, identity padding
    for (int ti = 0; ti < nb; ti++)
      for (int tj = 0; tj <= ti; tj++) {
        const int t = dt.tile(ti, tj);
        if (t < 0) continue;
        for (int er = 0; er < 48; er++)
          for (int ec = 0; ec < 48; ec++) {
            const int i = 48 * ti + er, j = 48 * tj + ec, oi = orig[i], oj = orig[j];
            tiles[(size_t)t * kAcTile + er * kAcLd + ec] =
                j > i ? 0.0 : ((oi < 0 || oj < 0) ? (i == j ? 1.0 : 0.0) : in[(size_t)std::max(oi, oj) * n + std::min(oi, oj)]);
          }
      }
    if (cudaMemcpy(s->hd.Sd, tiles.data(), tiles.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess) { g_err = "memcpy"; return -1; }
    if (dt.order == 1) return count;
    for (int ti = 0; ti < nb; ti++) {   // a row's first tile is also the pivot-column snapshot of the step that first reads it
      const int f = dt.first[ti];
      if (cudaMemcpy(s->hd.Dsnap + ((size_t)(f & 1) * nb + ti) * kAcTile, tiles.data() + (size_t)dt.toff[ti] * kAcTile, kAcTile * 8,
                     cudaMemcpyHostToDevice) != cudaSuccess) { g_err = "memcpy"; return -1; }
    }
    return count;
  }
  auto it = s->named.find(name);
  if (it == s->named.end()) { g_err = std::string("unknown buffer ") + name; return -1; }
  if (count > (long long)it->second.second) { g_err = "too many elements"; return -1; }
  if (cudaMemcpy(it->second.first, in, (size_t)count * 8, cudaMemcpyHostToDevice) != cudaSuccess) { g_err = "memcpy"; return -1; }
  return count;
}
int pus_debug_run_stage(pus_handle h, int stage, double lambda) {
  NEED(h);
  Solver* s = SV(h);
  if (!s->uploaded) { g_err = "call pus_upload first"; return -1; }
  if (stage == 5 && s->linear_solver == 0) { g_err = "debug stage 5 factors a stored Sdir: direct linear-solver mode only"; return -1; }
  return launch(&s, 1, MODE_DEBUG, 0, stage, lambda);
}

// host-only hook for the CPU test-suite: compile the graph and report array sizes without touching a GPU
int pus_debug_compile(pus_handle h) {
  NEED(h);
  Solver* s = SV(h);
  std::string err;
  if (!compile_graph(s->g, s->c, err)) { g_err = err; return -1; }
  if (s->linear_solver != 0 && !build_direct(s->c, s->dt, err, s->linear_solver, s->ordering)) { g_err = err; return -1; }
  return 0;
}

}  // extern "C"
