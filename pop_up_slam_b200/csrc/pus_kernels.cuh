// pus_kernels.cuh -- the device-resident Levenberg-Marquardt / Gauss-Newton loop for pose-plane
// factor graphs, written for sm_90a (H100): one persistent kernel, one CTA per SM, the CTAs of a
// "team" cooperate on one graph through a global-memory barrier (teams of one CTA for batches of
// small graphs).  Per LM trial step:
//   linearise   every residual + closed-form 3x6 / 3x3 (6x6) Jacobian blocks in one sweep, W = Jp^T Jl
//               written in both pose-major and plane-major warp tiles ([tile][18][32] doubles)
//   assemble    Hpp, gp (per pose), Hll, gl (per plane) by fixed-order gathers (no float atomics)
//   Schur       Hll^-1 (3x3); dense 96x96 diagonal blocks of S = Hpp - W Hll^-1 W^T built by pose-pair ownership and
//               inverted in shared memory (blocked Gauss-Jordan, rank-8 updates on the FP64 tensor cores);
//               Galerkin coarse operator on piecewise-linear trajectory modes, assembled output-stationary and
//               inverted in place by a symmetric block sweep of its lower triangle (48x48 tiles split over the team,
//               pivot-column snapshots staged by bulk async copies, DMMA tile updates, look-ahead pivot inversion)
//   PCG         implicit-Schur operator: plane-major sweep (W^T p), plane solve, pose-major sweep (W v),
//               two-level additive preconditioner, deterministic segmented reductions; on large graphs the W / Wt
//               tiles and the dense preconditioner blocks stream through shared memory by cp.async.bulk + mbarrier
//   update      exmap of every vertex, trial chi2, accept / reject, lambda rule -- all on device
// Control flow follows Optimizer::levenberg_marquardt / gauss_newton / relinearize of the reference
// (pop_planar_slam/Thirdparty/isam/isamlib/Optimizer.cpp:371-467, 286-366, 114-185).
//
// This file is included TWICE by pus_engine.cu, inside namespace pus::kplain (PUS_NO_SPAN defined: the single-GPU
// kernel, stores and barriers compiled without the spanning hooks) and inside pus::kspan (one graph spanning
// ranks, DESIGN.md section 8).  It therefore has no include guard, no #include and no namespace of its own.

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kSlots = 5;  // pose blocks handled concurrently by one CTA (5 x 96 = 480 threads)
constexpr int kTraceCap = 1024;
constexpr int kMaxStage = 64;  // staged group members in the dense-block build

enum KernelMode { MODE_BATCH = 0, MODE_UPDATE = 1, MODE_DEBUG = 2, MODE_CHI2 = 3, MODE_COV = 4 };

// MODE_DEBUG only: the branches the linear solve took, OR-ed into LmResult::status by the code that took them
// (pus_debug_fetch "path"; LmResult::iterations / accepted / chi2_evals / trace_n then hold the team size, the preconditioner
// levels, the hat spacing SP and the largest number of pose blocks one CTA owns)
enum PathBit {
  kPathResident = 1,       // block-resident loop (pcg_resident)
  kPathTma = 2,            // W / Wt tiles staged by TMA
  kPathTmaRing = 4,        // dense blocks applied from the three-stage bulk-copy ring
  kPathApplySmem = 8,      // dense blocks applied from the shared-memory cache (plain loop)
  kPathApplyL2 = 16,       // dense blocks applied straight from L2 (plain loop)
  kPathL3Local = 32,       // three levels, level 3 applied by every CTA itself
  kPathCluster = 64,       // the team is one thread-block cluster
  kPathResListed = 128,    // resident loop: heavy planes summed once per CTA
  kPathResUnlisted = 256,  // resident loop: heavy planes past kResHeavy, summed by a warp of their block
  kPathResTail = 512,      // resident loop: pose-pose factors past the first two neighbours (loop closures)
  kPathResWide = 1024,     // resident loop: a pose block with more than 96 plane groups
  kPathCoarseTail = 2048,  // two levels: coarse residual over more than 8 blocks per hat interval
};

struct LmParams {
  int method;  // 0 GN, 1 LM
  double eps2, eps_abs, eps_rel;
  int max_iter;
  double lambda0, lambda_factor;
  int robust_kind;
  double robust_b;
  double pcg_tol;
  int pcg_max_iter;
  int mode;
  int debug_stage;
  double debug_lambda;
  int restore_init;
  int prec_refresh;  // 1: lazy preconditioner refresh (default), 0: rebuild for every solve
  int warm_start;    // 1: PCG starts from the previous step after a rejected LM step
  int fine_timers;   // 1: sub-phase timers (perturbs the run slightly)
  int refresh_pct, refresh_add;  // lazy preconditioner refresh threshold
  int tma_mode;      // 0: TMA-staged W/Wt tiles when a warp owns several tiles (large graphs), 1: always, 2: never
  int blocks_always; // 1: the dense 16-pose blocks (level 1) are rebuilt for every linear solve, only the coarse level(s) lazily
  int jac_numeric;   // 1: reference-Jacobian mode (central differences, numericalDiff.cpp:41-87) instead of the closed forms
  int timer_rank;    // CTA of the team whose thread 0 keeps the phase timers (diagnostics; default 0)
  int resident;      // 1: the PCG loop runs block-resident (pcg_resident: operator, preconditioner blocks and vectors of the owned
                     //    pose blocks stay in shared memory / registers; set by the host when the layout fits the team)
};

struct LmResult {
  int iterations, accepted, relin, chi2_evals;
  long long pcg_iters;
  double chi2_initial, chi2_final;
  int trace_n, status;
  unsigned long long phase_ns[24];
};

struct LmTrace {
  double lambda[kTraceCap], chi2_new[kTraceCap], chi2_before[kTraceCap], delta_norm[kTraceCap];
  int accepted[kTraceCap], pcg[kTraceCap];
};

struct DevGraph {
  int N, M, Epl, Epf, Elp, ntile, ntile_pl, nslot, nblk, nc, SP, n_upart, n_ypart, nce, ngrp;
  double inv_SP;
  int ldmc;  // leading dimension of A_c (6 * nc rounded up to whole 48-wide pivot blocks)
  // vertex values
  double *pose_lin, *pose_trial, *pose_init, *plane_lin, *plane_trial, *plane_init;
  // pose-plane edges (pose-major) and plane-major view
  const int *pp_pose, *pp_plane, *pp_ptr, *pp_end, *pm2pl, *pm_part, *ypart_ptr, *tile_ptr, *blk_part_ptr, *grp_of_slot;
  const double *pp_meas, *pp_sinf, *pp_rays;
  const int* pp_kind;
  int n_f2;   // number of Pose3d_Plane3d_Factor2 edges (0: pp_rays / pp_kind are dummies)
  const int *pl2pm, *pl_ptr, *pl_plane, *pl_pose, *pl_part, *upart_ptr, *heavy, *huge;
  int n_heavy, n_huge;
  // pose factors / plane priors
  const int *pf_i, *pf_j, *pinc_ptr, *pinc, *pnbr;
  const double *pf_meas, *pf_sinf;
  const int *lp_plane, *linc_ptr, *linc;
  const double *lp_meas, *lp_sinf;
  // dense-block groups, coarse pairs
  const int *blk_grp_ptr, *grp_plane, *grp_mem_ptr, *grp_mem, *blk_simple, *grp_info;
  const int* grp_info2;         // block-resident PCG: {plane, first per-block partial, number of partials, own slot} per group
  int res_nt, res_ng, res_np;   // largest tile / group / (tile, pose)-run count of any pose block
  int n_ovf_blk;                // pose blocks over kMaxGrp / kMaxPart (0: blk_ovf is a dummy)
  const int* blk_ovf;           // per block: offset of its pose-phase vectors in `ovf`, -1 = shared memory
  double* ovf;                  // overflow scratch of the fused pose phase (group vectors, then run sums, per block)
  double* upartb;               // [ngrp][3] per-(block, plane) partial sums of W^T p
  const int *at_plane, *at_lo, *at_hi, *at_ptr, *as_plane;   // Hll / gl assembly tasks (chunks of a plane's edges), split planes
  int n_atask, n_asplit;
  double* hpart;                // [n_atask][9] partial sums of the split planes
  const int *ce_ptr, *ce_node, *ce_plane, *ce_lo, *ce_hi, *n2ce_ptr, *n2ce;
  const int *hv_plane, *lp_ptr, *lp_cea, *lp_ceb, *fp_ptr, *fp_f;
  int n_hv;
  // three-level preconditioner (large graphs): hat nodes every 16 poses, block-Jacobi in groups of kGroupNodes nodes
  int levels, nc2, nce2, ng2;
  const int *ce2_node, *ce2_plane, *ce2_lo, *ce2_hi, *g2_ptr, *g2_ce;
  double *Wc2, *Yc2, *D2inv, *zc2, *rc3;
  // work buffers
  double *W, *Wt, *JP, *JL, *PF, *LP;
  double *Hpp, *gp, *Hll, *gl, *Hinv, *vl, *dl;
  double *upart, *ypart;
  double *Binv, *Wc, *Yc;
  float *Ac;                    // A_c^-1 for the applies (ac_index), rounded to fp32: the preconditioner, not the operator
  double *Atri, *Apan;          // the triangle and panel buffers of its inversion (fp64)
  double *x, *r, *z, *q, *b, *pv[2], *xprev, *zc;
  double *rcpart[2], *qcpart;
  double *red;
  // one graph spanning several ranks (DESIGN.md section 8): rank / world, byte offsets from this rank's mirrored arena
  // to every peer's (0 for itself), and the cross-rank barrier counter that lives inside the arena
  int span_w, span_r;
  long long peer_delta[8];
  unsigned* gbar;
  LmParams prm;
  LmResult* res;
  LmTrace* trace;
  // exact direct solves (pus::kdirect only; zero / null for PCG handles): the reduced system of order 48 dnb as the envelope
  // of its lower triangle in 48x48 tiles (pus_graph.hpp, DirectTables), tile (I, J) at dtile(I, J) = dtoff[I] + J - dfirst[I];
  // the dense solve has dfirst = 0, no bordered plane and dnbp = dnb
  int dnb, dninc, dnbp, dnbord;                           // tile rows; incidences; pose tile rows; bordered planes
  const int *dinc_plane, *dinc_lo, *dinc_hi;              // (pose, plane) incidences, plane-major: plane-major slot range
  const int *dlp_ptr, *dlp_a, *dlp_b, *dfp_ptr, *dfp_f;  // per envelope pose pair a >= b: incidence pairs (plane-ascending), factor sides
  const int *dfirst, *dtoff, *dpoff;                     // per tile row: first tile column, tile offset; per pose: first pair index
  const int *dcol_ptr, *dcol_row;                        // per tile column K: the tile rows i > K of the envelope in it
  const int *dbord, *dbinc;                              // bordered planes (ascending); [lo, hi) of each one's incidences
  double *Wd, *Yd;       // [dninc][18]: W_al (summed over the pair's edges) and W_al Hll_d^-1
  double *Sd;            // S, factored in place into L
  double *Dsnap;         // [2 step parities][dnb] pivot-column snapshots
  double *Dinv;          // [dnb] L_KK^-1
  double *dvec;          // [2][48 dnb] triangular-solve vectors
  unsigned* dflag;       // set when a pivot is not positive
  // nested-dissection layout (null otherwise): its tables packed into one array (pus_graph.hpp, NdTable; nd(k) below); the
  // pose-pair lists are indexed 64 t + 8 (a % 8) + b % 8 by the stored tile t of the pair; the envelope tables above are unused
  const int* dnd;
  // marginal covariances (pus::kdirect, ND layout; null otherwise, DESIGN.md section 5.4): Sigma in the tiles of L's pattern,
  // the packed selected-inversion and plane-pair tables (pus_graph.hpp, CovTable; cov(k) below), and one call's records
  // (header: gather records, columns, their offsets) and output
  double* Sig;
  const int* dcov;
  const int* crec;
  double* covout;
};

// The graph descriptor of the solve in progress and the dynamic shared memory, named at namespace scope so that every
// access compiles to LDS / STS with an immediate address (through a reference or a pointer kept in a struct they became
// generic loads behind a local-memory load of the pointer -- on the critical path of every PCG phase).
__shared__ DevGraph g_sG;
extern __shared__ __align__(128) unsigned char g_smem[];
#define G g_sG

// ---------------------------------------------------------------------------------------------
struct Ctx {
  int rank, tsize;       // CTA rank within its team, CTAs per team
  unsigned* bar;         // team barrier counter (zeroed by the host before launch)
  unsigned bar_target;   // thread 0 only
  int red_slot;
  int smem_cache_ok;     // the dense-block cache in shared memory holds this solve's blocks
  int l3_local;          // three-level mode, small level 3: every CTA applies A_3^-1 itself (no exchange of its result)
  int use_tma;           // this graph streams its W / Wt tiles through the per-warp TMA staging buffers
  unsigned tma_par;      // phase parity of this warp's two staging mbarriers (bit s = stage s)
  unsigned gj_par;       // phase parity of the coarse inversion's four mbarriers (bit s = mbarrier s)
  // spanning mode: the team seen by the split PCG phases covers the CTAs of all ranks (rank = span_r * ltsize + lrank);
  // the replicated phases (linearise, Schur set-up, update) use the local view.  `mirror` = stores to the shared PCG
  // vectors are repeated into every peer's arena.
  int span_w, span_r, lrank, ltsize, mirror;
  long long peer_delta[8];
  unsigned* gbar;
  unsigned gbar_target;  // thread 0 only
  unsigned char* smem;   // dynamic shared memory
  unsigned long long* rflag;   // flag-stamped reduction slots of this team ([2 sets][tsize][2 words], zeroed by the host per launch)
  unsigned red_seq;      // sequence number of the last flag-stamped reduction (same on every thread of the team)
  int light;             // 1: team_barrier() / team_reduce<1>() use the fence-free barrier and the flag-stamped reduction
  int cluster;           // 1: the team is one thread-block cluster (small graphs): cluster barrier / DSMEM mbarrier, reductions through DSMEM
  unsigned cl_par;       // phase parity of the cluster mbarrier (same on every thread)
};

__device__ __forceinline__ double ldc(const double* p) { return __ldcg(p); }
__device__ __forceinline__ int ldc(const int* p) { return __ldcg(p); }

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Team barrier for the PCG loops, without the L1 invalidation that a gpu-scope fence or an acquire load implies (CCTL.IVALL
// throws away every cached local-memory line of the SM -- the spilled loop state -- three times per PCG iteration).  Release
// side: one release-reduction (orders the CTA's prior writes, through the CTA barrier, before the arrival).  Wait side:
// relaxed polling; every value another CTA wrote is read with ld.global.cg (L2) inside those loops, so nothing stale in L1 can
// be observed.  The full team_barrier() (fence + invalidate) brackets the loops.
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Teams of up to 16 CTAs are launched as one thread-block cluster.  Outside the PCG loops the team barrier is the hardware
// cluster barrier (every thread arrives; release / acquire at cluster scope = the fences + L1 invalidation of the
// global-counter barrier).  Inside the loops (`light`) it is an mbarrier in every CTA's shared memory that counts one remote
// arrival per CTA of the cluster: a lane per peer sends `mbarrier.arrive.release.cluster` through DSMEM (one warp-wide fence
// orders the CTA's global writes, through the CTA barrier, before the arrivals), thread 0 polls its own mbarrier with a
// relaxed wait -- no L1 invalidation (the spilled loop state stays cached), and everything another CTA wrote is read with
// ld.global.cg as in the global-counter version.  One-value reductions ride on the same arrival: the partial is stored into
// slot [rank] of every peer's buffer before the arrive.
constexpr int kSmClBar = 1056;   // the cluster mbarrier (u64), between the pipeline mbarriers and the work area
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned mapa_u32(unsigned a, unsigned cta) {
  unsigned ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(cta));
  return ra;
}
__device__ __forceinline__ void st_dsmem_f64(const void* local_smem, unsigned cta, double v) {
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(mapa_u32((unsigned)__cvta_generic_to_shared(local_smem), cta)), "d"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive_peer_release(unsigned local_bar, unsigned cta) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(mapa_u32(local_bar, cta)) : "memory");
}
__device__ __forceinline__ void mbar_wait_relaxed(unsigned bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.relaxed.cluster.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok)
                 : "r"(bar), "r"(parity)
                 : "memory");
  } while (!ok);
}
__device__ __forceinline__ void cluster_barrier_light(Ctx& c) {
  __syncthreads();
  if (threadIdx.x < 32) {
    const unsigned b = (unsigned)__cvta_generic_to_shared(g_smem + kSmClBar);
    if ((int)threadIdx.x < c.tsize) mbar_arrive_peer_release(b, threadIdx.x);
    if (threadIdx.x == 0) mbar_wait_relaxed(b, c.cl_par);
  }
  c.cl_par ^= 1u;
  __syncthreads();
}
__device__ __forceinline__ void team_barrier_light(Ctx& c) {
  if (c.cluster) { cluster_barrier_light(c); return; }
  __syncthreads();
  if (c.tsize > 1) {
    if (threadIdx.x == 0) {
      c.bar_target += (unsigned)c.tsize;
      asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(c.bar), "r"(1u) : "memory");
      while ((int)(ld_relaxed_u32(c.bar) - c.bar_target) < 0) { }
    }
    __syncthreads();
  }
}

// All CTAs of the team must call this the same number of times.  In the global view of a spanning solve the barrier
// covers the CTAs of every rank: each CTA adds one to its own rank's counter and to every peer's (system-scope
// atomics through peer-mapped memory), and waits for its own counter.
__device__ __forceinline__ void team_barrier(Ctx& c) {
  if (c.light) { team_barrier_light(c); return; }   // inside the single-GPU PCG loops (set / cleared by schur_solve)
  if (c.cluster) { cluster_sync_all(); return; }
  __syncthreads();
#ifndef PUS_NO_SPAN
  if (c.mirror) {
    if (threadIdx.x == 0) {
      c.gbar_target += (unsigned)c.tsize;
      __threadfence_system();
      for (int w = 0; w < c.span_w; w++)
        atomicAdd_system(reinterpret_cast<unsigned*>(reinterpret_cast<char*>(c.gbar) + c.peer_delta[w]), 1u);
      const unsigned long long t0 = gtime();
      // (wrap-safe: the counters persist across launches and may pass 2^32 after many spanning solves)
      while ((int)(ld_acquire_sys_u32(c.gbar) - c.gbar_target) < 0) {
        if (gtime() - t0 > 20000000000ull) __trap();   // a peer never arrived (20 s): fail instead of hanging the GPU
      }
      __threadfence_system();
    }
    __syncthreads();
    return;
  }
#endif
  if (c.tsize > 1) {
    if (threadIdx.x == 0) {
      c.bar_target += (unsigned)c.tsize;
      __threadfence();
      atomicAdd(c.bar, 1u);
      while ((int)(ld_acquire_u32(c.bar) - c.bar_target) < 0) { }
      __threadfence();
    }
    __syncthreads();
  }
}


// store to a PCG vector that every rank keeps a full copy of (no-op distinction outside the spanning global view)
template <typename T>
__device__ __forceinline__ void put(const Ctx& c, T* p, T v) {
  *p = v;
#ifdef PUS_NO_SPAN
  return;
#endif
  if (c.mirror)
    for (int w = 0; w < c.span_w; w++)
      if (w != c.span_r) *reinterpret_cast<T*>(reinterpret_cast<char*>(p) + c.peer_delta[w]) = v;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// ---- TMA (bulk async copy) + mbarrier helpers: one elected lane issues, the whole warp waits ----
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy writes (st.global by the lineariser) -> async-proxy reads (cp.async.bulk)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  const unsigned b = smem_u32(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(b)
               : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_copy_1d(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 1/x to full double precision without the IEEE division sequence: hardware seed + two Newton steps
__device__ __forceinline__ double fast_rcp(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);   // seed: ~20 bits; two Newton steps reach double precision
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  return fma(r, e, r);
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  const unsigned b = smem_u32(bar);
  unsigned ok;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok)
                 : "r"(b), "r"(parity)
                 : "memory");
  } while (!ok);
}

// FP64 tensor-core MMA, D(8x8) += A(8x4, row) * B(4x8, col): lane holds a = A[lane/4][lane%4], b = B[lane%4][lane/4],
// c[0..1] = C[lane/4][2*(lane%4) + {0,1}]
__device__ __forceinline__ void dmma884(double* cacc, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(cacc[0]), "+d"(cacc[1])
               : "d"(a), "d"(b));
}

// A_c^-1 as the PCG applies read it: full rows of fp32, stored as 48-row x 128-column tiles with a padded row stride (528
// bytes: every row of a tile starts 16-byte aligned)
constexpr int kGjChunk = 128, kGjLdR = kGjChunk + 4;
constexpr int kGjTile = 48 * kGjLdR;   // elements per tile
__host__ __device__ inline int ac_chunks(int ldm) { return (ldm + kGjChunk - 1) / kGjChunk; }
__host__ __device__ inline size_t ac_index(int ldm, int row, int col) {
  return ((size_t)(row / 48) * ac_chunks(ldm) + (col / kGjChunk)) * kGjTile + (size_t)(row % 48) * kGjLdR + (col % kGjChunk);
}
__host__ __device__ inline size_t ac_elems(int ldm) { return (size_t)(ldm / 48) * ac_chunks(ldm) * kGjTile; }
// A_c while it is assembled and inverted: the lower triangle only, as 48x48 tiles (I, J), I >= J, each stored with a
// padded row stride (conflict-free DMMA fragment loads; one bulk copy moves a tile).  Tiles are numbered band by band
// (bands of two tile rows), column by column inside a band: (0,0) (1,0) (1,1) | (2,0) (3,0) (2,1) (3,1) (2,2) (3,2) (3,3) | ...
// so that a contiguous range of tile numbers is a compact patch (few tile rows, few tile columns).
constexpr int kAcLd = 52, kAcTile = 48 * kAcLd;
__host__ __device__ inline int ac_ntri(int ldm) { const int nb = ldm / 48; return nb * (nb + 1) / 2; }
__host__ __device__ inline int tri_index(int nb, int i, int j) {
  const int b = i >> 1;
  const int p = (2 * b + 1 < nb) ? (j <= 2 * b ? 2 * j + (i - 2 * b) : 4 * b + 2) : j;
  return b * (2 * b + 1) + p;
}
__host__ __device__ inline void tri_tile(int nb, int t, int& i, int& j) {
  int b = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.25);
  while (b > 0 && b * (2 * b + 1) > t) b--;
  while ((b + 1) * (2 * b + 3) <= t) b++;
  const int p = t - b * (2 * b + 1);
  if (2 * b + 1 < nb) {
    if (p < 4 * b + 2) { j = p >> 1; i = 2 * b + (p & 1); }
    else { i = j = 2 * b + 1; }
  } else {
    i = 2 * b; j = p;
  }
}
// device buffers of the inversion: the triangle, the pivot-column snapshots [2 step parities][nb tiles] and the pivot
// inverses [2 step parities] (one allocation: snapshots, then inverses)
__host__ __device__ inline size_t ac_tri_doubles(int ldm) { return (size_t)ac_ntri(ldm) * kAcTile; }
__host__ __device__ inline size_t ac_panel_doubles(int ldm) { return (size_t)(2 * (ldm / 48) + 2) * kAcTile; }
// A diagonal tile counts as this many tile updates when the triangle is split over the team: its owner updates it first
// in the step before it becomes the pivot, inverts it and publishes the inverse while the other CTAs update their tiles
constexpr int kPivotWeight = 10;

// shared-memory carve-up (bytes)
constexpr int kSmRed = 0;                            // [kWarps][4] + [4] doubles
constexpr int kSmRedBytes = (kWarps * 4 + 8) * 8;
constexpr int kSmWork = 1024 + 64;                   // start of the phase-specific area
// dense-block build: S0, S1 (96x96), Wg, Yg (kMaxStage x 18), P (36), Hinv (9)
constexpr int kLdS = kBlockDim + 4;                  // padded row stride of the 96x96 block (conflict-free MMA fragments)
constexpr int kFastTiles = 16, kFastGrp = 96;         // limits of the fast dense-block build (tiles / planes per block)
constexpr int kSmS0 = kSmWork;
constexpr int kSmS1 = kSmS0 + kBlockDim * kLdS * 8;
constexpr int kSmWg = kSmS1 + kBlockDim * kLdS * 8;  // slow path: staged group; fast path: (group, pose) -> slot table
constexpr int kSmYg = kSmWg + kMaxStage * 18 * 8;
constexpr int kSmP = kSmYg + kMaxStage * 18 * 8;     // [96][12] coefficient columns of the inner inversion step
constexpr int kSmHi = kSmP + kBlockDim * 12 * 8;
constexpr int kSmBuildEnd = kSmHi + 16 * 8;
// PCG phases: sA, sB [kSlots*96], szc [kSlots][12][8], rc [6*nc]
constexpr int kSmA = kSmWork;
constexpr int kSmB = kSmA + kSlots * kBlockDim * 8;
constexpr int kSmZc = kSmB + kSlots * kBlockDim * 8;
constexpr int kSmRc = kSmZc + kSlots * 12 * 8 * 8;
// fused pose phase (aliases the coarse-residual area): plane-group vectors and (tile, pose) partial sums
constexpr int kSmVg = kSmRc;
constexpr int kSmYp = kSmVg + kSlots * kMaxGrp * 3 * 8;
constexpr int kSmPoseEnd = kSmYp + kSlots * kMaxPart * 6 * 8;
static_assert(kSmPoseEnd <= kSmBuildEnd, "shared-memory carve-up");
static_assert(kFastTiles * 18 * 32 * 8 <= kBlockDim * kLdS * 8, "fast-build staging must fit the second block buffer");
static_assert(kFastGrp * (16 * 2 + 9 * 8) <= 2 * kMaxStage * 18 * 8, "slot table + Hll^-1 must fit the group staging area");
// PCG: packed-symmetric copies of the owned dense blocks (upper triangle, 4656 doubles each)
constexpr int kPackedBlock = kBlockDim * (kBlockDim + 1) / 2;
constexpr int kSmCache = 72 * 1024;                   // after the PCG work area (rc may use up to 72 KB - kSmRc)
constexpr int kCacheBlocks = 4;
constexpr int kSmCacheEnd = kSmCache + kCacheBlocks * kPackedBlock * 8;
constexpr int kSmemBytes = 225 * 1024;   // (almost) everything an SM offers next to the static DevGraph copy (>= kSmBuildEnd, kSmCacheEnd, kSmTmaEnd; kSmRc + 6*nc*8 and the
                                         // block-resident layout are checked on the host)
static_assert(kSmBuildEnd <= kSmemBytes && kSmCacheEnd <= kSmemBytes, "dynamic shared memory");
static_assert(kSmPoseEnd <= kSmCache, "pose-phase buffers overlap the block cache");
// TMA staging (large graphs; replaces the block cache): per warp two 4608-byte W / Wt tiles, filled by
// cp.async.bulk and signalled through one mbarrier per stage
constexpr int kSmBar = 768;                           // [kWarps][2] mbarriers (u64)
constexpr int kSmGjBar = 1024;                        // mbarriers of the coarse inversion (4) / the block ring (3)
constexpr int kSmTma = kSmCache;
constexpr int kTileBytes = 18 * 32 * 8;
constexpr int kSmTmaEnd = kSmTma + kWarps * 2 * kTileBytes;
static_assert(kSmBar + kWarps * 2 * 8 <= kSmGjBar && kSmGjBar + 32 <= kSmWork, "mbarriers overlap the work area");
static_assert(kSmTmaEnd <= 227 * 1024, "TMA staging buffers");
// coarse inversion: eight 48x48 tiles (P, two T rows, three snapshot tiles, two staging tiles), the coefficient columns of the pivot
// inversion and the owned tile range -- the same for every team size
static_assert(kSmWork + (8 * kAcTile + 48 * 12 + 2) * 8 <= kSmemBytes, "coarse inversion buffers");
static_assert(kSmWork % 16 == 0 && kSmRc % 16 == 0, "coarse residuals are read with 128-bit shared loads");
static_assert(kSmemBytes <= 227 * 1024, "dynamic shared memory");


// ---- block-resident PCG (pcg_resident): shared-memory layout of one CTA.  Every owned pose block ("slot") keeps, for the
// whole linear solve, its W tiles, its packed preconditioner block, the packed static edge / group records and the
// per-iteration scratch; the strides are the graph-wide maxima so that every CTA computes the same offsets.
__host__ __device__ inline int r16(int x) { return (x + 15) & ~15; }
constexpr int kResHeavy = 8;   // distinct heavy planes (seen from > 8 pose blocks) a CTA sums once for all its blocks
struct ResLay {
  int hdr, sP, sR, src, slot0, stride;       // header (tile / group counts per slot), direction, residual / q, coarse residual
  int o_ei, o_gi, o_gm, o_mem, o_W, o_B;     // per slot: scratch at 0 (edge products | group vectors + run sums), then these
  int total;
};
__host__ __device__ inline ResLay res_layout(int nt, int ng, int np, int ldm, int nown) {
  ResLay L;
  L.hdr = kSmWork;
  L.sP = L.hdr + 64 + kResHeavy * 16 + kResHeavy * 16 * 3 * 8;   // + list of CTA-wide heavy planes and their per-warp partial sums
  L.sR = L.sP + nown * kBlockDim * 8;
  L.src = L.sR + nown * kBlockDim * 8;
  L.slot0 = L.src + r16(ldm * 8);
  const int ua = nt * 32 * 24, ub = r16(ng * 24) + np * 48;
  const int uc = 6 * kBlockDim * 8;   // phase C: row sums and up to five warps' column partials of z = Binv r
  L.o_ei = r16(ua > ub ? (ua > uc ? ua : uc) : (ub > uc ? ub : uc));
  L.o_gi = L.o_ei + nt * 128;
  L.o_gm = L.o_gi + ng * 16;
  L.o_mem = L.o_gm + r16(ng * 8);
  L.o_W = L.o_mem + r16(nt * 64);
  L.o_B = L.o_W + nt * 18 * 32 * 8;
  L.stride = L.o_B + kBlockDim * (kBlockDim + 1) / 2 * 8;
  L.total = L.slot0 + nown * L.stride;
  return L;
}

// deterministic team-wide sum of K (<= 4) values; result broadcast to every thread.
// warp partials -> CTA partial (warp 0) -> global slot -> team barrier -> every CTA's warp 0 sums the
// per-CTA partials with strided lanes + a shuffle tree (fixed order, so all CTAs get identical bits).
__device__ __forceinline__ double team_reduce_flag(Ctx& c, double v);
template <int K>
__device__ __forceinline__ void team_reduce(Ctx& c, double* red, double* v) {
  if (K == 1 && c.light) { v[0] = team_reduce_flag(c, v[0]); return; }
  double* s = reinterpret_cast<double*>(g_smem + kSmRed);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = warp_sum(v[k]);
  __syncthreads();  // protect s from a previous use
  if (lane == 0)
    for (int k = 0; k < K; k++) s[warp * 4 + k] = v[k];
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      double acc = (lane < kWarps) ? s[lane * 4 + k] : 0.0;
      acc = warp_sum(acc);
      if (lane == 0) {
        if (c.tsize > 1) put(c, &red[((size_t)c.red_slot * c.tsize + c.rank) * 4 + k], acc);
        else s[kWarps * 4 + k] = acc;
      }
    }
  }
  if (c.tsize > 1) {
    team_barrier(c);
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        double acc = 0;
        for (int r = lane; r < c.tsize; r += 32) acc += ldc(red + ((size_t)c.red_slot * c.tsize + r) * 4 + k);
        acc = warp_sum(acc);
        if (lane == 0) s[kWarps * 4 + k] = acc;
      }
    }
    c.red_slot = (c.red_slot + 1) & 3;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = s[kWarps * 4 + k];
}


// Team-wide sum of one value without an atomic counter: every CTA stamps its partial with the reduction's sequence number
// (two 8-byte words {value half, seq}, each store single-copy atomic) and warp 0 of every CTA polls all the slots until they
// carry that number, then adds them in a fixed order (identical bits on every CTA).  One store + one polled load instead of
// store, atomic, polled counter, load.  Double-buffered: a CTA can start reduction n+2 only after every CTA has read n.
// Memory ordering as in team_barrier_light: CTA barrier, release store of the second word, relaxed polling, L2 reads.
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ double team_reduce_flag(Ctx& c, double v) {
  double* s = reinterpret_cast<double*>(g_smem + kSmRed);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect s from a previous use; all global writes of the phase are done
  if (lane == 0) s[warp * 4] = v;
  __syncthreads();
  c.red_seq++;
  if (c.cluster) {
    // every CTA leaves its partial in slot [rank] of every CTA's buffer (two buffers, by the parity of the sequence number: a
    // CTA can be one reduction ahead of the slowest reader) and then arrives on that CTA's mbarrier; fixed-order sum
    const int b = 2 + (int)(c.red_seq & 1u);
    if (warp == 0) {
      double acc = (lane < kWarps) ? s[lane * 4] : 0.0;
      acc = warp_sum(acc);
      const unsigned mb = (unsigned)__cvta_generic_to_shared(g_smem + kSmClBar);
      if (lane < c.tsize) {
        st_dsmem_f64(s + c.rank * 4 + b, (unsigned)lane, acc);
        mbar_arrive_peer_release(mb, (unsigned)lane);
      }
      if (lane == 0) mbar_wait_relaxed(mb, c.cl_par);
    }
    c.cl_par ^= 1u;
    __syncthreads();
    double tot = 0;
    for (int r = 0; r < c.tsize; r++) tot += s[r * 4 + b];
    return tot;
  }
  const int nw = (c.tsize + 31) >> 5;
  if (c.tsize > 1 && nw <= kWarps) {
    // one slot per thread: warp w polls slots 32 w .. 32 w + 31 (a single round trip to L2 for the whole team instead of
    // tsize / 32 dependent ones by warp 0), butterfly sum per warp, then every thread adds the nw warp sums in warp order
    const unsigned seq = c.red_seq;
    unsigned long long* slots = c.rflag + (size_t)(seq & 1u) * c.tsize * 2;
    if (warp == 0) {
      double acc = (lane < kWarps) ? s[lane * 4] : 0.0;
      acc = warp_sum(acc);
      if (lane == 0) {
        const unsigned long long b = (unsigned long long)__double_as_longlong(acc);
        st_relaxed_u64(slots + (size_t)c.rank * 2, (b & 0xffffffffull) | ((unsigned long long)seq << 32));
        st_release_u64(slots + (size_t)c.rank * 2 + 1, (b >> 32) | ((unsigned long long)seq << 32));   // (orders every prior write)
      }
    }
    if (warp < nw) {
      const int r = warp * 32 + lane;
      double val = 0;
      if (r < c.tsize) {
        unsigned long long w0, w1;
        do {
          w0 = ld_relaxed_u64(slots + (size_t)r * 2);
          w1 = ld_relaxed_u64(slots + (size_t)r * 2 + 1);
        } while ((unsigned)(w0 >> 32) != seq || (unsigned)(w1 >> 32) != seq);
        val = __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
      }
      val = warp_sum(val);
      if (lane == 0) s[warp * 4 + 1] = val;
    }
    __syncthreads();
    double tot = 0;
    for (int w = 0; w < nw; w++) tot += s[w * 4 + 1];
    return tot;
  }
  if (warp == 0) {
    double acc = (lane < kWarps) ? s[lane * 4] : 0.0;
    acc = warp_sum(acc);
    if (c.tsize > 1) {
      const unsigned seq = c.red_seq;
      unsigned long long* slots = c.rflag + (size_t)(seq & 1u) * c.tsize * 2;
      if (lane == 0) {
        const unsigned long long b = (unsigned long long)__double_as_longlong(acc);
        st_relaxed_u64(slots + (size_t)c.rank * 2, (b & 0xffffffffull) | ((unsigned long long)seq << 32));
        st_release_u64(slots + (size_t)c.rank * 2 + 1, (b >> 32) | ((unsigned long long)seq << 32));   // (orders every prior write)
      }
      double tot = 0;
      for (int r = lane; r < c.tsize; r += 32) {
        unsigned long long w0, w1;
        do {
          w0 = ld_relaxed_u64(slots + (size_t)r * 2);
          w1 = ld_relaxed_u64(slots + (size_t)r * 2 + 1);
        } while ((unsigned)(w0 >> 32) != seq || (unsigned)(w1 >> 32) != seq);
        tot += __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
      }
      acc = warp_sum(tot);
    }
    if (lane == 0) s[kWarps * 4] = acc;
  }
  __syncthreads();
  return s[kWarps * 4];
}

// segmented (by sorted key) suffix sums inside a warp: afterwards the first lane of every run of equal
// keys holds the run's total, accumulated in a fixed order.  Returns true on that lane when the key is valid (>= 0).
template <int K>
__device__ __forceinline__ bool seg_suffix_sum(int key, double* v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int ok = __shfl_down_sync(0xffffffffu, key, d);
    bool take = (lane + d < 32) && (ok == key);
#pragma unroll
    for (int k = 0; k < K; k++) {
      double o = __shfl_down_sync(0xffffffffu, v[k], d);
      if (take) v[k] += o;
    }
  }
  const int pk = __shfl_up_sync(0xffffffffu, key, 1);
  return key >= 0 && (lane == 0 || pk != key);
}

// ---- arithmetic shared by the general PCG loop (schur_solve) and the block-resident one (pcg_resident) ----
// Each helper fixes one summation order and expression shape for all its callers.  Loads stay with the
// callers wherever they are issued early for latency; the loader argument (LdS: shared memory or registers, LdL2:
// ld.global.cg) only selects the load instruction of the operands the helper reads itself.
struct LdS {
  __device__ __forceinline__ double operator()(const double* p) const { return *p; }
};
struct LdL2 {
  __device__ __forceinline__ double operator()(const double* p) const { return __ldcg(p); }
};

// h[0..2] . u[0..2]: one row of a 3x3 product (Hll^-1 u)
template <class Ld = LdS>
__device__ __forceinline__ double dot3(const double* h, const double* u) {
  const Ld ld;
  return ld(h) * u[0] + ld(h + 1) * u[1] + ld(h + 2) * u[2];
}
// v = H u, H a row-major 3x3 already in registers
__device__ __forceinline__ void mat3_vec(const double* H, const double* u, double* v) {
#pragma unroll
  for (int b = 0; b < 3; b++) v[b] = dot3(H + b * 3, u);
}

// sum of the 3-vector partials part[a0 .. a1) by one warp: 8 strided partials per lane in flight, then a fixed-order tree;
// every lane gets the sums
__device__ __forceinline__ void warp_sum_partials(const double* part, int a0, int a1, int lane, double* uu) {
  uu[0] = 0; uu[1] = 0; uu[2] = 0;
  for (int tb = a0 + lane; tb < a1; tb += 256) {
    double pr[8][3];
#pragma unroll
    for (int t = 0; t < 8; t++)
#pragma unroll
      for (int b = 0; b < 3; b++) pr[t][b] = (tb + 32 * t < a1) ? ldc(part + (size_t)(tb + 32 * t) * 3 + b) : 0.0;
#pragma unroll
    for (int t = 0; t < 8; t++)
#pragma unroll
      for (int b = 0; b < 3; b++) uu[b] += pr[t][b];
  }
#pragma unroll
  for (int b = 0; b < 3; b++) uu[b] = warp_sum(uu[b]);
}

// v = Hll^-1 of plane l times the sum of its n <= 8 partials part[t0 .. t0 + n), by one thread (all 33 loads in one batch)
__device__ __forceinline__ void plane_vec_small(const double* part, int t0, int n, int l, double* v) {
  double pr[8][3], Hi[9];
#pragma unroll
  for (int t = 0; t < 8; t++)
#pragma unroll
    for (int b = 0; b < 3; b++) pr[t][b] = (t < n) ? ldc(part + (size_t)(t0 + t) * 3 + b) : 0.0;
#pragma unroll
  for (int t = 0; t < 9; t++) Hi[t] = ldc(G.Hinv + (size_t)l * 9 + t);
  double uu[3] = {0, 0, 0};
#pragma unroll
  for (int t = 0; t < 8; t++)
#pragma unroll
    for (int b = 0; b < 3; b++) uu[b] += pr[t][b];
  mat3_vec(Hi, uu, v);
}

// W_e^T x (6 -> 3) of one lane's edge in an [18][32] warp tile (w = tile + lane), accumulated into u
template <class Ld>
__device__ __forceinline__ void tile_wt_x(const double* w, const double* x, double* u) {
  const Ld ld;
#pragma unroll
  for (int a = 0; a < 6; a++) {
    const double xa = x[a];
#pragma unroll
    for (int b = 0; b < 3; b++) u[b] += ld(w + (a * 3 + b) * 32) * xa;
  }
}
// y = W_e v (3 -> 6) of one lane's edge in an [18][32] warp tile
template <class Ld>
__device__ __forceinline__ void tile_w_v(const double* w, double v0, double v1, double v2, double* y) {
  const Ld ld;
#pragma unroll
  for (int a = 0; a < 6; a++) y[a] = ld(w + (a * 3) * 32) * v0 + ld(w + (a * 3 + 1) * 32) * v1 + ld(w + (a * 3 + 2) * 32) * v2;
}

// coefficients of row `row` of the pose-pose blocks towards the first two neighbours of a pose (the odometry chain), from its
// pnbr record {f0 * 2 + side0, neighbour0, f1 * 2 + side1, neighbour1} (f < 0: none) into a[n * 6 + col]; returns the number of
// such neighbours
__device__ __forceinline__ int nbr_coeffs(int4 nb, int row, double* a) {
  const int nf = (nb.x >= 0) + (nb.z >= 0);
  const double* Ab[2] = {G.PF + (size_t)(max(nb.x, 0) >> 1) * 120 + 72, G.PF + (size_t)(max(nb.z, 0) >> 1) * 120 + 72};
  const int sd[2] = {nb.x & 1, nb.z & 1};
#pragma unroll
  for (int n2 = 0; n2 < 2; n2++)
#pragma unroll
    for (int cc = 0; cc < 6; cc++) a[n2 * 6 + cc] = (n2 < nf) ? (sd[n2] ? ldc(Ab[n2] + cc * 6 + row) : ldc(Ab[n2] + row * 6 + cc)) : 0.0;
  return nf;
}
// v + row `row` of the further pose-pose blocks (loop closures, incidences pinc[k0 .. k1)) times pvec
__device__ __forceinline__ double pose_pose_tail(int k0, int k1, int row, const double* pvec, double v) {
  for (int kk = k0; kk < k1; kk++) {
    const int inc = G.pinc[kk], f = inc >> 1, side = inc & 1;
    const int j = G.pf_j[f];
    if (j < 0) continue;
    const int oth = side ? G.pf_i[f] : j;
    const double* A12 = G.PF + (size_t)f * 120 + 72;
    for (int cc = 0; cc < 6; cc++) {
      const double a = side ? ldc(A12 + cc * 6 + row) : ldc(A12 + row * 6 + cc);
      v += a * ldc(pvec + (size_t)oth * 6 + cc);
    }
  }
  return v;
}

// row i of a packed upper triangle of a symmetric kBlockDim block: packed_row(B, i)[j] = (i, j) for j >= i
template <typename T>
__device__ __forceinline__ T* packed_row(T* B, int i) { return B + i * kBlockDim - (i * (i - 1)) / 2 - i; }
// row u of the packed symmetric block B times rv, one thread per row: rows j < u give (j, u), rows j >= u give (u, j)
template <class Ld>
__device__ __forceinline__ double packed_row_dot(const double* B, int u, const double* rv) {
  const Ld ld;
  double acc = 0;
  for (int j = 0; j < u; j++) acc += ld(packed_row(B, j) + u) * rv[j];
  const double* bu = packed_row(B, u);
  for (int j = u; j < kBlockDim; j++) acc += ld(bu + j) * rv[j];
  return acc;
}

// row of A_c^-1 (arow = its first element in the fp32 tiled layout) times the coarse residual src[0 .. ldm) (16-byte aligned),
// one warp per row: a lane owns the four columns 4 lane + 128 t of tile chunk t (one 128-bit load; the residual as two
// 128-bit shared loads), products and sums in fp64.  kFly chunks are loaded per round.  The block-resident loop takes 16 (up
// to 2 048 columns; A_c is at most 1 920 wide), so a row is one round of loads.  The general loop (schur_solve) holds many
// more live values, and loads in flight there cost spills in the whole loop: its two-level apply takes 8, its level-3 apply
// (a few hundred rows) 4.  Returns the row sum on every lane.
template <int kFly>
__device__ __forceinline__ double coarse_row_dot(const float* arow, const double* src, int ldm, int lane) {
  double acc = 0;
  for (int j0 = 4 * lane; j0 < ldm; j0 += kFly * kGjChunk) {
    float4 av[kFly];
#pragma unroll
    for (int t = 0; t < kFly; t++) {
      const int jj = j0 + kGjChunk * t;
      av[t] = (jj < ldm) ? __ldcg(reinterpret_cast<const float4*>(arow + (size_t)(jj / kGjChunk) * kGjTile + (jj % kGjChunk)))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int t = 0; t < kFly; t++) {
      const int jj = j0 + kGjChunk * t;
      if (jj < ldm) {   // (ldm = 6 nc is even: the lane's first pair is inside, its second may not be)
        const double2 s0 = *reinterpret_cast<const double2*>(src + jj);
        acc += (double)av[t].x * s0.x + (double)av[t].y * s0.y;
        if (jj + 2 < ldm) {
          const double2 s1 = *reinterpret_cast<const double2*>(src + jj + 2);
          acc += (double)av[t].z * s1.x + (double)av[t].w * s1.y;
        }
      }
    }
  }
  return warp_sum(acc);
}

// coarse residual src[i] = rc_old + rc_old' - alpha (qcpart + qcpart') when every coarse interval is one pose block (graphs up
// to 5120 poses): block `node` feeds the node through its slot 0, block `node-1` through slot 1.  Four outputs per thread, so
// that all 16 loads are in flight together.  (first: no q yet, rc_old only.)
__device__ __forceinline__ void coarse_residual(const double* rc_old, double alpha, bool first, double* src) {
  const int ldm = 6 * G.nc;
  for (int i0 = threadIdx.x; i0 < ldm; i0 += 4 * kThreads) {
    double va[4][2], vq[4][2];
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const int i = i0 + m * kThreads, node = i / 6, row = i - node * 6;
#pragma unroll
      for (int side = 0; side < 2; side++) {
        const int k = node - side;
        const bool ok = (i < ldm) && (k >= 0) && (k < G.nblk);
        va[m][side] = ok ? ldc(rc_old + (size_t)k * 12 + side * 6 + row) : 0.0;
        vq[m][side] = (ok && !first) ? ldc(G.qcpart + (size_t)k * 12 + side * 6 + row) : 0.0;
      }
    }
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const int i = i0 + m * kThreads;
      if (i < ldm) src[i] = (0.0 + (va[m][0] - alpha * vq[m][0])) + (va[m][1] - alpha * vq[m][1]);
    }
  }
}

// inverse of a 6x6 (symmetric positive definite in exact arithmetic) matrix by Gauss-Jordan, row-major
__device__ __forceinline__ void inv6(const double* A, double* Ai) {
  double a[36];
  for (int i = 0; i < 36; i++) a[i] = A[i];
  for (int k = 0; k < 6; k++) {
    double piv = 1.0 / a[k * 6 + k];
    for (int j = 0; j < 6; j++) a[k * 6 + j] = (j == k) ? piv : a[k * 6 + j] * piv;
    for (int i = 0; i < 6; i++) {
      if (i == k) continue;
      double f = a[i * 6 + k];
      for (int j = 0; j < 6; j++) a[i * 6 + j] = (j == k) ? -f * piv : a[i * 6 + j] - f * a[k * 6 + j];
    }
  }
  for (int i = 0; i < 36; i++) Ai[i] = a[i];
}

// one entry of a pivot step of the blocked Gauss-Jordan inversion (6x6 blocks, pivot block k, P = A_kk^-1):
//   (k,k): P ; (k,j): P A_kj ; (i,k): -A_ik P ; else A_ij - A_ik P A_kj
// (row, col) are scalar indices of the ldm x ldm matrix; `ld` loads a scalar of the source matrix.
template <typename Load>
__device__ __forceinline__ double gj_entry(Load ld, int ldm, int row, int col, int k, const double* P) {
  const int i = row / 6, r = row - i * 6, j = col / 6, cc = col - j * 6;
  if (i == k) {
    if (j == k) return P[r * 6 + cc];
    double s = 0;
#pragma unroll
    for (int t = 0; t < 6; t++) s += P[r * 6 + t] * ld((k * 6 + t) * ldm + col);
    return s;
  }
  double a[6];
#pragma unroll
  for (int t = 0; t < 6; t++) a[t] = ld(row * ldm + k * 6 + t);
  if (j == k) {
    double s = 0;
#pragma unroll
    for (int t = 0; t < 6; t++) s += a[t] * P[t * 6 + cc];
    return -s;
  }
  double b[6];
#pragma unroll
  for (int t = 0; t < 6; t++) b[t] = ld((k * 6 + t) * ldm + col);
  double s = ld(row * ldm + col);
#pragma unroll
  for (int t = 0; t < 6; t++) {
    double tr = 0;
#pragma unroll
    for (int u = 0; u < 6; u++) tr += a[u] * P[u * 6 + t];
    s -= tr * b[t];
  }
  return s;
}

// ---------------------------------------------------------------------------------------------
// phases
// ---------------------------------------------------------------------------------------------
// phase timer of the lead thread (CTA 0 of the team, thread 0): %globaltimer deltas accumulated in shared
// memory (a global read-modify-write per lap would itself cost ~1 us on the critical path) and flushed once.
constexpr int kL3Local = 192;   // three-level mode: level 3 of at most this many rows is applied by every CTA itself
constexpr int kSmTimer = 576;  // 24 x u64 inside the first KB of dynamic shared memory
struct Timer {
  bool on;
  unsigned long long t0;
  unsigned long long* acc;
  __device__ Timer(bool o) : on(o), t0(0), acc(reinterpret_cast<unsigned long long*>(g_smem + kSmTimer)) {
    if (on) { for (int i = 0; i < 24; i++) acc[i] = 0; t0 = gtime(); }
  }
  __device__ void sync() { if (on) t0 = gtime(); }
  __device__ void lap(int slot) {
    if (on) {
      unsigned long long t = gtime();
      acc[slot] += t - t0;
      t0 = t;
    }
  }
  __device__ void flush(LmResult* res) { if (on) for (int i = 0; i < 24; i++) res->phase_ns[i] = acc[i]; }
};

// In-place style inversion of an n x n (n = 8 NB) SPD matrix held in shared memory with row stride LD, by
// Gauss-Jordan with 8x8 inner blocks, ping-ponging between Mc and Mn (returns the buffer holding the inverse):
// per inner step J every warp inverts the 8x8 diagonal block in registers (lane = column, shuffles, no block
// sync), the threads form the coefficient columns TQ = -M[:,J] Q (+Q in the rows of J; these are also the pivot
// columns of the result), and the rank-8 update of the remaining tiles runs on the FP64 tensor cores.
// All threads of the CTA must call it; Mc must be complete (synchronised) on entry.
template <int NB, int LD>
__device__ __forceinline__ double* gj_invert_smem(double* Mc, double* Mn, double* TQ) {
  constexpr int n = 8 * NB, LDQ = 12;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fc = lane & 3, cidx = lane & 7;
  for (int J = 0; J < NB; J++) {
    double d[8];
#pragma unroll
    for (int a = 0; a < 8; a++) d[a] = Mc[(8 * J + a) * LD + 8 * J + cidx];
#pragma unroll
    for (int pp = 0; pp < 8; pp++) {
      const double piv = fast_rcp(__shfl_sync(0xffffffffu, d[pp], pp));
      double f[8];
#pragma unroll
      for (int a = 0; a < 8; a++) f[a] = __shfl_sync(0xffffffffu, d[a], pp);
      const double rs = (cidx == pp) ? piv : d[pp] * piv;
#pragma unroll
      for (int a = 0; a < 8; a++)
        if (a != pp) d[a] = (cidx == pp) ? -f[a] * piv : fma(-f[a], rs, d[a]);
      d[pp] = rs;
    }
    // d[s] = Q[s][cidx];  entry (i, cidx) of TQ for i = tid/8, tid/8 + 64, ...
    for (int i = tid >> 3; i < n; i += kThreads / 8) {
      double v;
      if (i >= 8 * J && i < 8 * J + 8) {
        const int rr = i - 8 * J;
        v = d[0];
#pragma unroll
        for (int a = 1; a < 8; a++) v = (rr == a) ? d[a] : v;
      } else {
        v = 0;
#pragma unroll
        for (int sx = 0; sx < 8; sx++) v = fma(-Mc[i * LD + 8 * J + sx], d[sx], v);
      }
      TQ[i * LDQ + cidx] = v;
      Mn[i * LD + 8 * J + cidx] = v;
    }
    __syncthreads();
    for (int u = warp; u < NB * (NB - 1); u += kWarps) {
      const int mi = u / (NB - 1), nj = u - mi * (NB - 1), ni = nj + (nj >= J ? 1 : 0);
      double cacc[2] = {0.0, 0.0};
      if (mi != J) {
        const double2 c2 = *reinterpret_cast<const double2*>(Mc + (8 * mi + fr) * LD + 8 * ni + 2 * fc);
        cacc[0] = c2.x; cacc[1] = c2.y;
      }
#pragma unroll
      for (int ks = 0; ks < 2; ks++)
        dmma884(cacc, TQ[(8 * mi + fr) * LDQ + 4 * ks + fc], Mc[(8 * J + 4 * ks + fc) * LD + 8 * ni + fr]);
      *reinterpret_cast<double2*>(Mn + (8 * mi + fr) * LD + 8 * ni + 2 * fc) = make_double2(cacc[0], cacc[1]);
    }
    __syncthreads();
    double* t = Mc; Mc = Mn; Mn = t;
  }
  return Mc;
}

// acc += A B for 48x48 tiles in shared memory (row stride kAcLd) on the FP64 tensor cores; B is read as Bm^T (BT) or Bm.
// Warp w owns the 8x8 output tiles q = w, w + 16, w + 32 (< 36): acc[s] = rows 8 (q / 6) + lane / 4, columns
// 8 (q % 6) + 2 (lane % 4) + {0, 1}.  Three accumulator chains per output tile (the MMA latency is long, the chain short).
template <bool BT>
__device__ __forceinline__ void mma48(double (&acc)[3][2], const double* A, const double* Bm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, fr = lane >> 2, fc = lane & 3;
#pragma unroll
  for (int s = 0; s < 3; s++) {
    const int q = warp + 16 * s;
    if (q < 36) {
      const int m = q / 6, n = q - 6 * m;
      const double* a = A + (8 * m + fr) * kAcLd + fc;
      const double* b = BT ? Bm + (8 * n + fr) * kAcLd + fc : Bm + fc * kAcLd + 8 * n + fr;
      double x[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
      for (int k = 0; k < 12; k++) dmma884(k % 3 == 0 ? acc[s] : x[k % 3 - 1], a[4 * k], BT ? b[4 * k] : b[4 * k * kAcLd]);
      acc[s][0] += x[0][0] + x[1][0];
      acc[s][1] += x[0][1] + x[1][1];
    }
  }
}
// accumulator s of mma48 holds row r, columns cc and cc + 1 of the tile; false when the warp has no s-th output tile
__device__ __forceinline__ bool mma48_frag(int s, int& r, int& cc) {
  const int lane = threadIdx.x & 31, q = (threadIdx.x >> 5) + 16 * s;
  r = 8 * (q / 6) + (lane >> 2);
  cc = 8 * (q % 6) + 2 * (lane & 3);
  return q < 36;
}
// dst (row stride kAcLd) <- sg acc, each accumulator at its place in the tile
__device__ __forceinline__ void mma48_store(double* dst, const double (&acc)[3][2], double sg = 1.0) {
  int r, cc;
#pragma unroll
  for (int s = 0; s < 3; s++)
    if (mma48_frag(s, r, cc)) *reinterpret_cast<double2*>(dst + r * kAcLd + cc) = make_double2(sg * acc[s][0], sg * acc[s][1]);
}
// acc <- the tile src (row stride kAcLd, read through L2), each accumulator from its place in the tile
__device__ __forceinline__ void mma48_load(double (&acc)[3][2], const double* src) {
  int r, cc;
#pragma unroll
  for (int s = 0; s < 3; s++)
    if (mma48_frag(s, r, cc)) {
      const double2 v = __ldcg(reinterpret_cast<const double2*>(src + r * kAcLd + cc));
      acc[s][0] = v.x; acc[s][1] = v.y;
    }
}

// Pose3d_Plane3d_Factor2 edges are rare (disabled in the shipped demo): keep their extra arithmetic out of the
// register allocation of the common path
// reference-Jacobian mode (pus_math.cuh: pose_plane_numeric / pose_factor_numeric): rarely used, kept out of line
__device__ __noinline__ void pose_plane_numeric_dev(const double* pose, const double* plane, const double* meas, const double* sinf,
                                                    int robust_kind, double robust_b, double* r, double* Jp, double* Jl, const double* rays) {
  pose_plane_numeric(pose, plane, meas, sinf, robust_kind, robust_b, r, Jp, Jl, rays);
}
__device__ __noinline__ void pose_factor_numeric_dev(const double* p1, const double* p2, const double* meas, const double* sinf,
                                                     int robust_kind, double robust_b, double* r, double* J1, double* J2) {
  pose_factor_numeric(p1, p2, meas, sinf, robust_kind, robust_b, r, J1, J2);
}
__device__ __noinline__ void pose_plane2_linearize(const double* pose, const double* plane, const double* rays, const double* sinf,
                                                   int robust_kind, double robust_b, double* r, double* Jp, double* Jl) {
  const double unit[4] = {1, 0, 0, 0};
  pose_plane_linearize(pose, plane, unit, sinf, robust_kind, robust_b, r, Jp, Jl, rays);
}

struct Phase {
  Ctx& c;
  Timer* ft = nullptr;  // optional fine-grained phase timer (lead thread)
  __device__ Phase(Ctx& cc) : c(cc) {}
  __device__ __forceinline__ void lap(int slot) { if (ft) ft->lap(slot); }
  // slots 6 / 22 / 23 are shared: sub-stages of the resident PCG loop (fine_timers == 1) or of linearize (fine_timers == 2)
  __device__ __forceinline__ void lap1(int slot) { if (ft && (G.prm.fine_timers & 1)) ft->lap(slot); }
  __device__ __forceinline__ void lap2(int slot) { if (ft && G.prm.fine_timers == 2) ft->lap(slot); }

  __device__ __forceinline__ int tid_team() const { return c.rank * kThreads + threadIdx.x; }
  __device__ __forceinline__ int nthr_team() const { return c.tsize * kThreads; }
  __device__ __forceinline__ int warp_team() const { return c.rank * kWarps + (threadIdx.x >> 5); }
  __device__ __forceinline__ int nwarp_team() const { return c.tsize * kWarps; }

  // -------- restore the uploaded initial estimate (repeatable resident solves) --------
  __device__ void restore_init() {
    for (int i = tid_team(); i < G.N * 7; i += nthr_team()) G.pose_lin[i] = G.pose_init[i];
    for (int i = tid_team(); i < G.M * 4; i += nthr_team()) G.plane_lin[i] = G.plane_init[i];
  }

  // -------- linearise: pose-plane edges --------
  __device__ void lin_pose_plane() {
    const int lane = threadIdx.x & 31;
    for (int tile = warp_team(); tile < G.ntile; tile += nwarp_team()) {
      int e = tile * 32 + lane;
      int p = G.pp_pose[e];
      if (p >= 0) {
        int l = G.pp_plane[e];
        double pose[7], pl[4], m[4], si[6];
        for (int i = 0; i < 7; i++) pose[i] = ldc(G.pose_lin + (size_t)p * 7 + i);
        for (int i = 0; i < 4; i++) pl[i] = ldc(G.plane_lin + (size_t)l * 4 + i);
        for (int i = 0; i < 4; i++) m[i] = G.pp_meas[(size_t)e * 4 + i];
        for (int i = 0; i < 6; i++) si[i] = G.pp_sinf[(size_t)e * 6 + i];
        double r[3], Jp[18], Jl[9];
        if (G.prm.jac_numeric)             // reference-Jacobian mode
          pose_plane_numeric_dev(pose, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, Jp, Jl,
                                 (G.n_f2 > 0 && G.pp_kind[e]) ? G.pp_rays + (size_t)e * 6 : nullptr);
        else if (G.n_f2 > 0 && G.pp_kind[e])   // Factor2: measurement re-popped from the edge's rays (kept out of line)
          pose_plane2_linearize(pose, pl, G.pp_rays + (size_t)e * 6, si, G.prm.robust_kind, G.prm.robust_b, r, Jp, Jl);
        else
          pose_plane_linearize(pose, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, Jp, Jl);
        double* w = G.W + (size_t)tile * kWStride + lane;
        int s = G.pm2pl[e];
        double* wt = G.Wt + (size_t)(s >> 5) * kWStride + (s & 31);
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
          for (int b = 0; b < 3; b++) {
            double v = Jp[a] * Jl[b] + Jp[6 + a] * Jl[3 + b] + Jp[12 + a] * Jl[6 + b];
            w[(a * 3 + b) * 32] = v;
            wt[(a * 3 + b) * 32] = v;
          }
        double* jp = G.JP + (size_t)e * 21;
        for (int i = 0; i < 18; i++) jp[i] = Jp[i];
        jp[18] = r[0]; jp[19] = r[1]; jp[20] = r[2];
        double* jl = G.JL + (size_t)e * 12;
        for (int i = 0; i < 9; i++) jl[i] = Jl[i];
        jl[9] = r[0]; jl[10] = r[1]; jl[11] = r[2];
      }
    }
    fence_proxy_async();  // W / Wt are read back through the async proxy (bulk copies) on large graphs
  }

  // -------- linearise: pose priors / odometry, plane priors --------
  __device__ void lin_other() {
    // Pose factors in chunks of 32, one chunk per CTA at a time: warp 0 evaluates residual and Jacobians (a lane per factor) and
    // leaves them in shared memory; the whole CTA then forms the 120 products per factor (J1^T J1, J2^T J2, J1^T J2, J1^T r,
    // J2^T r) -- a thread per output, coalesced stores -- instead of 650 dependent multiply-adds over local-memory arrays in the
    // one thread that owns the factor (graphs have few pose factors: that thread was the whole phase).
    {
      constexpr int LDJ = 79;   // J1[36] J2[36] r[6], odd stride
      double* sJ = reinterpret_cast<double*>(g_smem + kSmWork);
      const int tid = threadIdx.x, lane = tid & 31;
      const int nchunk = (G.Epf + 31) / 32;
      for (int ch = c.rank; ch < nchunk; ch += c.tsize) {
        const int f0 = ch * 32, nf = min(32, G.Epf - f0);
        __syncthreads();
        if (tid < 32 && lane < nf) {
          const int f = f0 + lane;
          const int i = G.pf_i[f], j = G.pf_j[f];
          double p1[7], p2[7], m[6], si[21];
          for (int t = 0; t < 7; t++) p1[t] = ldc(G.pose_lin + (size_t)i * 7 + t);
          if (j >= 0) for (int t = 0; t < 7; t++) p2[t] = ldc(G.pose_lin + (size_t)j * 7 + t);
          for (int t = 0; t < 6; t++) m[t] = G.pf_meas[(size_t)f * 6 + t];
          for (int t = 0; t < 21; t++) si[t] = G.pf_sinf[(size_t)f * 21 + t];
          double r[6], J1[36], J2[36];
          for (int t = 0; t < 36; t++) J2[t] = 0;
          if (G.prm.jac_numeric) pose_factor_numeric_dev(p1, j >= 0 ? p2 : nullptr, m, si, G.prm.robust_kind, G.prm.robust_b, r, J1, J2);
          else pose_factor_linearize(p1, j >= 0 ? p2 : nullptr, m, si, G.prm.robust_kind, G.prm.robust_b, r, J1, J2);
          double* o = sJ + lane * LDJ;
          for (int t = 0; t < 36; t++) { o[t] = J1[t]; o[36 + t] = J2[t]; }
          for (int t = 0; t < 6; t++) o[72 + t] = r[t];
        }
        __syncthreads();
        for (int q = tid; q < nf * 120; q += kThreads) {
          const int fl = q / 120, en = q - fl * 120;
          const double* J = sJ + fl * LDJ;
          double acc = 0;
          if (en < 108) {
            const int blk = en / 36, ab = en - blk * 36, a = ab / 6, b = ab - a * 6;
            const double* A = J + (blk == 1 ? 36 : 0);
            const double* B = J + (blk == 0 ? 0 : 36);
#pragma unroll
            for (int k = 0; k < 6; k++) acc += A[k * 6 + a] * B[k * 6 + b];
          } else {
            const int a = (en - 108) % 6;
            const double* A = J + (en >= 114 ? 36 : 0);
#pragma unroll
            for (int k = 0; k < 6; k++) acc += A[k * 6 + a] * J[72 + k];
          }
          G.PF[(size_t)(f0 + fl) * 120 + en] = acc;
        }
      }
      __syncthreads();
    }
    for (int f = tid_team(); f < G.Elp; f += nthr_team()) {
      int l = G.lp_plane[f];
      double pl[4], m[4], si[6];
      for (int t = 0; t < 4; t++) pl[t] = ldc(G.plane_lin + (size_t)l * 4 + t);
      for (int t = 0; t < 4; t++) m[t] = G.lp_meas[(size_t)f * 4 + t];
      for (int t = 0; t < 6; t++) si[t] = G.lp_sinf[(size_t)f * 6 + t];
      double r[3], Jl[9];
      if (G.prm.jac_numeric) pose_plane_numeric_dev(nullptr, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, Jl, nullptr);
      else pose_plane_linearize(nullptr, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, Jl);
      double* o = G.LP + (size_t)f * 12;
      for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) o[a * 3 + b] = Jl[a] * Jl[b] + Jl[3 + a] * Jl[3 + b] + Jl[6 + a] * Jl[6 + b];
        o[9 + a] = Jl[a] * r[0] + Jl[3 + a] * r[1] + Jl[6 + a] * r[2];
      }
    }
  }

  // -------- assemble Hpp / gp (thread per (pose, entry)) and Hll / gl (warp per plane) --------
  __device__ void assemble() {
    const long long total = (long long)G.N * 42;
    for (long long idx = tid_team(); idx < total; idx += nthr_team()) {
      int p = (int)(idx / 42), en = (int)(idx % 42);
      int e0 = G.pp_ptr[p], e1 = G.pp_end[p];
      int i0 = G.pinc_ptr[p], i1 = G.pinc_ptr[p + 1];
      double acc = 0;
      if (en < 36) {
        int a = en / 6, b = en % 6;
        for (int e = e0; e < e1; e++) {
          const double* jp = G.JP + (size_t)e * 21;
          acc += ldc(jp + a) * ldc(jp + b) + ldc(jp + 6 + a) * ldc(jp + 6 + b) + ldc(jp + 12 + a) * ldc(jp + 12 + b);
        }
        for (int k = i0; k < i1; k++) {
          int inc = G.pinc[k];
          acc += ldc(G.PF + (size_t)(inc >> 1) * 120 + (inc & 1) * 36 + en);
        }
        G.Hpp[(size_t)p * 36 + en] = acc;
      } else {
        int a = en - 36;
        for (int e = e0; e < e1; e++) {
          const double* jp = G.JP + (size_t)e * 21;
          acc += ldc(jp + a) * ldc(jp + 18) + ldc(jp + 6 + a) * ldc(jp + 19) + ldc(jp + 12 + a) * ldc(jp + 20);
        }
        for (int k = i0; k < i1; k++) {
          int inc = G.pinc[k];
          acc += ldc(G.PF + (size_t)(inc >> 1) * 120 + 108 + (inc & 1) * 6 + a);
        }
        G.gp[(size_t)p * 6 + a] = acc;
      }
    }
    const int lane = threadIdx.x & 31;
    // Hll / gl: a warp per task = chunk of at most kAsmChunk edges of one plane; a plane with a single task is finished here, the
    // others (the ground plane is seen from every pose) leave partial sums for assemble_split()
    for (int t = warp_team(); t < G.n_atask; t += nwarp_team()) {
      const int l = G.at_plane[t];
      double h[9];
      for (int k = 0; k < 9; k++) h[k] = 0;  // 0..5: Hll upper (00,01,02,11,12,22); 6..8: gl
      for (int s = G.at_lo[t] + lane; s < G.at_hi[t]; s += 32) {
        const double* jl = G.JL + (size_t)G.pl2pm[s] * 12;
        double J[12];
        for (int k = 0; k < 12; k++) J[k] = ldc(jl + k);
        h[0] += J[0] * J[0] + J[3] * J[3] + J[6] * J[6];
        h[1] += J[0] * J[1] + J[3] * J[4] + J[6] * J[7];
        h[2] += J[0] * J[2] + J[3] * J[5] + J[6] * J[8];
        h[3] += J[1] * J[1] + J[4] * J[4] + J[7] * J[7];
        h[4] += J[1] * J[2] + J[4] * J[5] + J[7] * J[8];
        h[5] += J[2] * J[2] + J[5] * J[5] + J[8] * J[8];
        h[6] += J[0] * J[9] + J[3] * J[10] + J[6] * J[11];
        h[7] += J[1] * J[9] + J[4] * J[10] + J[7] * J[11];
        h[8] += J[2] * J[9] + J[5] * J[10] + J[8] * J[11];
      }
      for (int k = 0; k < 9; k++) h[k] = warp_sum(h[k]);
      if (G.at_ptr[l + 1] - G.at_ptr[l] > 1) {
        if (lane == 0) for (int k = 0; k < 9; k++) G.hpart[(size_t)t * 9 + k] = h[k];
      } else if (lane == 0) {
        finish_plane(l, h);
      }
    }
  }
  __device__ __forceinline__ void finish_plane(int l, const double* h) {
    double H[9] = {h[0], h[1], h[2], h[1], h[3], h[4], h[2], h[4], h[5]};
    double gg[3] = {h[6], h[7], h[8]};
    for (int k = G.linc_ptr[l]; k < G.linc_ptr[l + 1]; k++) {
      const double* o = G.LP + (size_t)G.linc[k] * 12;
      for (int t = 0; t < 9; t++) H[t] += ldc(o + t);
      for (int t = 0; t < 3; t++) gg[t] += ldc(o + 9 + t);
    }
    for (int t = 0; t < 9; t++) G.Hll[(size_t)l * 9 + t] = H[t];
    for (int t = 0; t < 3; t++) G.gl[(size_t)l * 3 + t] = gg[t];
  }
  // second stage for the planes whose edges were gathered by several warps: a warp per plane adds the tasks' partial sums
  // (lane-strided, then the shuffle tree: fixed order) -- behind a team barrier after assemble()
  __device__ void assemble_split() {
    const int lane = threadIdx.x & 31;
    for (int q = warp_team(); q < G.n_asplit; q += nwarp_team()) {
      const int l = G.as_plane[q];
      double h[9];
      for (int k = 0; k < 9; k++) h[k] = 0;
      for (int t = G.at_ptr[l] + lane; t < G.at_ptr[l + 1]; t += 32)
        for (int k = 0; k < 9; k++) h[k] += ldc(G.hpart + (size_t)t * 9 + k);
      for (int k = 0; k < 9; k++) h[k] = warp_sum(h[k]);
      if (lane == 0) finish_plane(l, h);
    }
  }

  // -------- chi2 at the linearisation point (trial = false) or the trial values --------
  __device__ double chi2(bool trial) {
    const double* PV = trial ? G.pose_trial : G.pose_lin;
    const double* LV = trial ? G.plane_trial : G.plane_lin;
    double acc = 0;
    for (int e = tid_team(); e < G.nslot; e += nthr_team()) {
      int p = G.pp_pose[e], l = G.pp_plane[e];
      if (p < 0) continue;
      double pose[7], pl[4], m[4], si[6], r[3];
      for (int i = 0; i < 7; i++) pose[i] = ldc(PV + (size_t)p * 7 + i);
      for (int i = 0; i < 4; i++) pl[i] = ldc(LV + (size_t)l * 4 + i);
      for (int i = 0; i < 4; i++) m[i] = G.pp_meas[(size_t)e * 4 + i];
      for (int i = 0; i < 6; i++) si[i] = G.pp_sinf[(size_t)e * 6 + i];
      if (G.n_f2 > 0 && G.pp_kind[e])
        pose_plane2_linearize(pose, pl, G.pp_rays + (size_t)e * 6, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, nullptr);
      else
        pose_plane_linearize(pose, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, nullptr);
      acc += r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    }
    for (int f = tid_team(); f < G.Epf; f += nthr_team()) {
      int i = G.pf_i[f], j = G.pf_j[f];
      double p1[7], p2[7], m[6], si[21], r[6];
      for (int t = 0; t < 7; t++) p1[t] = ldc(PV + (size_t)i * 7 + t);
      if (j >= 0) for (int t = 0; t < 7; t++) p2[t] = ldc(PV + (size_t)j * 7 + t);
      for (int t = 0; t < 6; t++) m[t] = G.pf_meas[(size_t)f * 6 + t];
      for (int t = 0; t < 21; t++) si[t] = G.pf_sinf[(size_t)f * 21 + t];
      pose_factor_linearize(p1, j >= 0 ? p2 : nullptr, m, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, nullptr);
      for (int t = 0; t < 6; t++) acc += r[t] * r[t];
    }
    for (int f = tid_team(); f < G.Elp; f += nthr_team()) {
      int l = G.lp_plane[f];
      double pl[4], m[4], si[6], r[3];
      for (int t = 0; t < 4; t++) pl[t] = ldc(LV + (size_t)l * 4 + t);
      for (int t = 0; t < 4; t++) m[t] = G.lp_meas[(size_t)f * 4 + t];
      for (int t = 0; t < 6; t++) si[t] = G.lp_sinf[(size_t)f * 6 + t];
      pose_plane_linearize(nullptr, pl, m, si, G.prm.robust_kind, G.prm.robust_b, r, nullptr, nullptr);
      acc += r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    }
    double v[1] = {acc};
    team_reduce<1>(c, G.red, v);
    return v[0];
  }

  // -------- Schur setup, part 1: damped Hll^-1 and vl = Hll^-1 gl --------
  __device__ void plane_inverse(double lambda) {
    for (int l = tid_team(); l < G.M; l += nthr_team()) {
      double H[9], Hi[9];
      for (int t = 0; t < 9; t++) H[t] = ldc(G.Hll + (size_t)l * 9 + t);
      H[0] *= (1 + lambda); H[4] *= (1 + lambda); H[8] *= (1 + lambda);  // Cholesky.cpp:91-97
      sym3_inverse(H, Hi);
      for (int t = 0; t < 9; t++) G.Hinv[(size_t)l * 9 + t] = Hi[t];
      double g0 = ldc(G.gl + (size_t)l * 3), g1 = ldc(G.gl + (size_t)l * 3 + 1), g2 = ldc(G.gl + (size_t)l * 3 + 2);
      for (int t = 0; t < 3; t++) G.vl[(size_t)l * 3 + t] = Hi[t * 3] * g0 + Hi[t * 3 + 1] * g1 + Hi[t * 3 + 2] * g2;
    }
  }

  // -------- Schur setup, part 2: dense diagonal blocks of S, inverted in shared memory --------
  __device__ void build_blocks(double lambda) {
    constexpr int LD = kLdS;
    double* S0 = reinterpret_cast<double*>(g_smem + kSmS0);
    double* S1 = reinterpret_cast<double*>(g_smem + kSmS1);
    double* Wg = reinterpret_cast<double*>(g_smem + kSmWg);
    double* Yg = reinterpret_cast<double*>(g_smem + kSmYg);
    double* TQ = reinterpret_cast<double*>(g_smem + kSmP);
    double* His = reinterpret_cast<double*>(g_smem + kSmHi);
    const int tid = threadIdx.x;
    for (int k = c.rank; k < G.nblk; k += c.tsize) {
      const int p0 = k * kBlockPoses;
      const int np = min(kBlockPoses, G.N - p0);
      __syncthreads();
      for (int i = tid; i < kBlockDim * LD; i += kThreads) S0[i] = 0.0;
      __syncthreads();
      // diagonal 6x6 blocks (damped) and identity padding
      for (int i = tid; i < kBlockPoses * 36; i += kThreads) {
        int pi = i / 36, en = i % 36, a = en / 6, b = en % 6;
        double v;
        if (pi < np) {
          v = ldc(G.Hpp + (size_t)(p0 + pi) * 36 + en);
          if (a == b) v *= (1 + lambda);
        } else {
          v = (a == b) ? 1.0 : 0.0;
        }
        S0[(pi * 6 + a) * LD + pi * 6 + b] = v;
      }
      __syncthreads();
      // pose-pose factors with both ends inside the block (handled from side 0)
      for (int pi = 0; pi < np; pi++) {
        int i0 = G.pinc_ptr[p0 + pi], i1 = G.pinc_ptr[p0 + pi + 1];
        for (int kk = i0; kk < i1; kk++) {
          int inc = G.pinc[kk];
          if (inc & 1) continue;
          int f = inc >> 1, j = G.pf_j[f];
          if (j < p0 || j >= p0 + np || j == p0 + pi) continue;
          int pj = j - p0;
          if (tid < 36) {
            int a = tid / 6, b = tid % 6;
            double v = ldc(G.PF + (size_t)f * 120 + 72 + tid);
            S0[(pi * 6 + a) * LD + pj * 6 + b] += v;
            S0[(pj * 6 + b) * LD + pi * 6 + a] += v;
          }
          __syncthreads();
        }
      }
      const int g0 = G.blk_grp_ptr[k], ng = G.blk_grp_ptr[k + 1] - g0;
      if (G.blk_simple[k]) {
        // fast path (no pose of the block observes a plane twice, <= kFastTiles tiles, <= kFastGrp planes): stage
        // the block's W tiles in the second block buffer, the planes' Hll^-1 and a (group, pose) -> slot table;
        // then every pose pair (pi, pj) is owned by two threads that walk the groups and accumulate their 6x6
        // entries in registers -- no atomics, no per-group synchronisation, fixed summation order.
        double* Wst = S1;
        unsigned short* memb = reinterpret_cast<unsigned short*>(Wg);
        double* Hst = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(Wg) + kFastGrp * 16 * 2);
        const int t0 = G.tile_ptr[k], nt = G.tile_ptr[k + 1] - t0;
        for (int i = tid; i < nt * kWStride; i += kThreads) Wst[i] = ldc(G.W + (size_t)t0 * kWStride + i);
        for (int i = tid; i < ng * 8; i += kThreads) reinterpret_cast<unsigned*>(memb)[i] = 0xffffffffu;
        for (int i = tid; i < ng * 9; i += kThreads) Hst[i] = ldc(G.Hinv + (size_t)G.grp_plane[g0 + i / 9] * 9 + i % 9);
        __syncthreads();
        for (int sl = tid; sl < nt * 32; sl += kThreads) {
          const int e = t0 * 32 + sl, p = G.pp_pose[e];
          if (p >= 0) memb[G.grp_of_slot[e] * 16 + (p - p0)] = (unsigned short)sl;
        }
        __syncthreads();
        {
          const int pair = tid >> 1, half = tid & 1, pi = pair >> 4, pj = pair & 15;
          double acc[3][6];
#pragma unroll
          for (int a = 0; a < 3; a++)
#pragma unroll
            for (int b = 0; b < 6; b++) acc[a][b] = 0.0;
          for (int g = 0; g < ng; g++) {
            const int si = memb[g * 16 + pi], sj = memb[g * 16 + pj];
            if (si == 0xffff || sj == 0xffff) continue;
            const double* wi = Wst + (si >> 5) * kWStride + (si & 31) + (half * 9) * 32;
            const double* wj = Wst + (sj >> 5) * kWStride + (sj & 31);
            const double* Hi = Hst + g * 9;
            double yv[3][3];   // rows 3*half .. 3*half+2 of  W_i Hll^-1
#pragma unroll
            for (int a = 0; a < 3; a++) {
              const double w0 = wi[(a * 3) * 32], w1 = wi[(a * 3 + 1) * 32], w2 = wi[(a * 3 + 2) * 32];
#pragma unroll
              for (int t = 0; t < 3; t++) yv[a][t] = w0 * Hi[t] + w1 * Hi[3 + t] + w2 * Hi[6 + t];
            }
#pragma unroll
            for (int b = 0; b < 6; b++) {
              const double w0 = wj[(b * 3) * 32], w1 = wj[(b * 3 + 1) * 32], w2 = wj[(b * 3 + 2) * 32];
#pragma unroll
              for (int a = 0; a < 3; a++) acc[a][b] += yv[a][0] * w0 + yv[a][1] * w1 + yv[a][2] * w2;
            }
          }
#pragma unroll
          for (int a = 0; a < 3; a++)
#pragma unroll
            for (int b = 0; b < 6; b++) S0[(pi * 6 + half * 3 + a) * LD + pj * 6 + b] -= acc[a][b];
        }
      } else {
        // general path: minus W Hll^-1 W^T restricted to the block, one plane group at a time
        for (int g = g0; g < g0 + ng; g++) {
          const int m0 = G.grp_mem_ptr[g], m = G.grp_mem_ptr[g + 1] - m0;
          const int l = G.grp_plane[g];
          __syncthreads();
          if (tid < 9) His[tid] = ldc(G.Hinv + (size_t)l * 9 + tid);
          const bool staged = (m <= kMaxStage);
          if (staged) {
            for (int i = tid; i < m * 18; i += kThreads) {
              int mi = i / 18, kk = i % 18;
              int e = G.grp_mem[m0 + mi];
              Wg[i] = ldc(G.W + (size_t)(e >> 5) * kWStride + kk * 32 + (e & 31));
            }
          }
          __syncthreads();
          if (staged) {
            for (int i = tid; i < m * 18; i += kThreads) {
              int mi = i / 18, kk = i % 18, a = kk / 3, b = kk % 3;
              Yg[i] = Wg[mi * 18 + a * 3] * His[0 * 3 + b] + Wg[mi * 18 + a * 3 + 1] * His[1 * 3 + b] + Wg[mi * 18 + a * 3 + 2] * His[2 * 3 + b];
            }
          }
          __syncthreads();
          // Members of a group are in pose-major slot order, so the observations one pose makes of this plane are
          // contiguous.  Every (pose, pose) entry is owned by the thread of the FIRST member pair that maps to it, which
          // sums the contributions of all duplicate pairs in a fixed order: no atomics, bit-reproducible.
          const int total = m * m * 36;
          for (int idx = tid; idx < total; idx += kThreads) {
            int mi = idx / (36 * m), rem = idx % (36 * m);
            int mj = rem / 36, en = rem % 36, a = en / 6, b = en % 6;
            const int ppi = G.pp_pose[G.grp_mem[m0 + mi]], ppj = G.pp_pose[G.grp_mem[m0 + mj]];
            if ((mi > 0 && G.pp_pose[G.grp_mem[m0 + mi - 1]] == ppi) || (mj > 0 && G.pp_pose[G.grp_mem[m0 + mj - 1]] == ppj)) continue;
            const int pi = ppi - p0, pj = ppj - p0;
            double acc = 0;
            for (int ui = mi; ui < m && G.pp_pose[G.grp_mem[m0 + ui]] == ppi; ui++)
              for (int uj = mj; uj < m && G.pp_pose[G.grp_mem[m0 + uj]] == ppj; uj++) {
                double v;
                if (staged) {
                  v = Yg[ui * 18 + a * 3] * Wg[uj * 18 + b * 3] + Yg[ui * 18 + a * 3 + 1] * Wg[uj * 18 + b * 3 + 1] +
                      Yg[ui * 18 + a * 3 + 2] * Wg[uj * 18 + b * 3 + 2];
                } else {
                  const int ei = G.grp_mem[m0 + ui], ej = G.grp_mem[m0 + uj];
                  double wi[3], wj[3];
                  for (int t = 0; t < 3; t++) {
                    wi[t] = ldc(G.W + (size_t)(ei >> 5) * kWStride + (a * 3 + t) * 32 + (ei & 31));
                    wj[t] = ldc(G.W + (size_t)(ej >> 5) * kWStride + (b * 3 + t) * 32 + (ej & 31));
                  }
                  v = 0;
                  for (int t = 0; t < 3; t++) {
                    double y = wi[0] * His[0 * 3 + t] + wi[1] * His[1 * 3 + t] + wi[2] * His[2 * 3 + t];
                    v += y * wj[t];
                  }
                }
                acc += v;
              }
            S0[(pi * 6 + a) * LD + pj * 6 + b] -= acc;
          }
        }
      }
      __syncthreads();
      // inversion in shared memory (S0 <-> S1), then the dense copy for the PCG
      const double* inv = gj_invert_smem<kBlockDim / 8, LD>(S0, S1, TQ);
      // packed upper triangle (row i holds the entries j >= i): half the bytes the PCG streams, and exactly symmetric.
      // One warp per row.  (The flat form -- idx / 96, idx % 96, store if j >= i -- is miscompiled for sm_90a by the CUDA
      // 12.9 ptxas: in the peeled first iterations the j >= i test reads a register that still holds a value of the
      // inversion above, so stores of rows 0-10 were dropped at random.)
      double* out = G.Binv + (size_t)k * kPackedBlock;
      for (int i = tid >> 5; i < kBlockDim; i += kWarps) {
        double* orow = packed_row(out, i);
        for (int j = i + (tid & 31); j < kBlockDim; j += 32) orow[j] = inv[i * LD + j];
      }
    }
    fence_proxy_async();  // Binv is streamed by bulk copies in precondition() on large graphs
    __syncthreads();
  }

  __device__ __forceinline__ double hat(int p, int node) const {
    int d = p - node * G.SP;
    if (d < 0) d = -d;
    return d >= G.SP ? 0.0 : 1.0 - (double)d * G.inv_SP;
  }
  // level-2 hat (a node every kL2Spacing = 16 poses)
  __device__ __forceinline__ double hat2(int p, int node) const {
    int d = p - node * kL2Spacing;
    if (d < 0) d = -d;
    return d >= kL2Spacing ? 0.0 : 1.0 - (double)d * (1.0 / kL2Spacing);
  }
  // hat of the level the residual restrictions (rcpart / qcpart, 12 values per pose block) live on
  __device__ __forceinline__ double hat_r(int p, int node) const { return G.levels == 3 ? hat2(p, node) : hat(p, node); }
  __device__ __forceinline__ int sp_r() const { return G.levels == 3 ? kL2Spacing : G.SP; }
  // coarse part of z at pose p, row: interpolation of the published node vectors (two levels: zc; three: zc2 [+ zc])
  __device__ __forceinline__ double coarse_z(int p, int row) const {
    if (G.levels != 3) {
      const int c0 = p / G.SP;
      return hat(p, c0) * ldc(G.zc + (size_t)c0 * 6 + row) + hat(p, c0 + 1) * ldc(G.zc + (size_t)min(c0 + 1, G.nc - 1) * 6 + row);
    }
    const int a = p / kL2Spacing;
    const int d = p - a * kL2Spacing;
    double v = node2_z(a, row);
    if (d) { const double t = (double)d * (1.0 / kL2Spacing); v = (1.0 - t) * v + t * node2_z(min(a + 1, G.nc2 - 1), row); }
    return v;
  }
  __device__ __forceinline__ double node2_z(int a, int row) const {
    double v = ldc(G.zc2 + (size_t)a * 6 + row);
    if (!c.l3_local) {   // level 3 is distributed: its part is interpolated by the consumer
      const int p = a * kL2Spacing, c0 = p / G.SP;
      v += hat(p, c0) * ldc(G.zc + (size_t)c0 * 6 + row) + hat(p, c0 + 1) * ldc(G.zc + (size_t)min(c0 + 1, G.nc - 1) * 6 + row);
    }
    return v;
  }

  // -------- Schur setup, part 3: coarse pairs Wc = P^T W (warp per (plane, node) pair) --------
  __device__ void coarse_wc() {
    coarse_wc_level(G.nce, G.ce_node, G.ce_plane, G.ce_lo, G.ce_hi, G.SP, G.inv_SP, G.Wc, G.Yc);
    if (G.levels == 3) coarse_wc_level(G.nce2, G.ce2_node, G.ce2_plane, G.ce2_lo, G.ce2_hi, kL2Spacing, 1.0 / kL2Spacing, G.Wc2, G.Yc2);
  }
  __device__ void coarse_wc_level(int nce, const int* ce_node, const int* ce_plane, const int* ce_lo, const int* ce_hi, int SP, double inv_SP,
                                  double* Wc, double* Yc) {
    const int lane = threadIdx.x & 31;
    for (int ce = warp_team(); ce < nce; ce += nwarp_team()) {
      int node = ce_node[ce];
      double acc[18];
      for (int k = 0; k < 18; k++) acc[k] = 0;
      for (int s = ce_lo[ce] + lane; s < ce_hi[ce]; s += 32) {
        int d = G.pl_pose[s] - node * SP;
        if (d < 0) d = -d;
        double w = d >= SP ? 0.0 : 1.0 - (double)d * inv_SP;
        const double* wt = G.Wt + (size_t)(s >> 5) * kWStride + (s & 31);
        for (int k = 0; k < 18; k++) acc[k] += w * ldc(wt + k * 32);
      }
      for (int k = 0; k < 18; k++) acc[k] = warp_sum(acc[k]);
      if (lane < 18) {
        double v = acc[0];
#pragma unroll
        for (int k = 1; k < 18; k++) if (lane == k) v = acc[k];
        Wc[(size_t)ce * 18 + lane] = v;
        // Yc = Wc * Hll_d^-1 (6x3), entry (r, b) = lane
        const int r = lane / 3, b = lane - r * 3;
        const double* Hi = G.Hinv + (size_t)ce_plane[ce] * 9;
        double y = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          double w = acc[0];
#pragma unroll
          for (int q = 1; q < 18; q++) if (r * 3 + k == q) w = acc[q];
          y += w * ldc(Hi + k * 3 + b);
        }
        Yc[(size_t)ce * 18 + lane] = y;
      }
    }
  }

  // -------- Schur setup (three levels): the 96 x 96 diagonal blocks of P2^T S P2 (groups of kGroupNodes level-2 nodes),
  // assembled and inverted in shared memory by the owning CTA.  Pose part and pose-pose factors: entry-stationary (every
  // thread owns entries and walks the poses in the node's support); planes: one plane at a time, its (<= 16) nodes inside
  // the group as a dense rank-3 update from the staged Yc2 / Wc2 rows.  Fixed summation order, no atomics.
  __device__ void build_groups(double lambda) {
    constexpr int LD = kLdS;
    double* S0 = reinterpret_cast<double*>(g_smem + kSmS0);
    double* S1 = reinterpret_cast<double*>(g_smem + kSmS1);
    double* Yst = reinterpret_cast<double*>(g_smem + kSmWg);   // [<=16][18]
    double* Wst = reinterpret_cast<double*>(g_smem + kSmYg);   // [<=16][18]
    double* TQ = reinterpret_cast<double*>(g_smem + kSmP);
    int* nloc = reinterpret_cast<int*>(g_smem + kSmHi);        // node of the staged rows, relative to the group
    const int tid = threadIdx.x;
    for (int g = c.rank; g < G.ng2; g += c.tsize) {
      const int a0 = g * kGroupNodes;
      const int na = min(kGroupNodes, G.nc2 - a0);
      __syncthreads();
      for (int idx = tid; idx < kBlockDim * kBlockDim; idx += kThreads) {
        const int i = idx / kBlockDim, j = idx - i * kBlockDim;
        const int ai = i / 6, r = i - ai * 6, bj = j / 6, cc = j - bj * 6;
        double v = 0.0;
        if (ai >= na || bj >= na) {
          v = (i == j) ? 1.0 : 0.0;
        } else {
          const int a = a0 + ai, b = a0 + bj;
          const int plo = max(0, (a - 1) * kL2Spacing + 1), phi = min(G.N, (a + 1) * kL2Spacing);
          for (int p = plo; p < phi; p++) {
            const double ha = hat2(p, a), hb = hat2(p, b);
            if (hb != 0.0) {
              double h = ldc(G.Hpp + (size_t)p * 36 + r * 6 + cc);
              if (r == cc) h *= (1 + lambda);
              v += ha * hb * h;
            }
            for (int k = G.pinc_ptr[p]; k < G.pinc_ptr[p + 1]; k++) {   // pose-pose blocks of Hpp coupling p to other poses
              const int inc = G.pinc[k], f = inc >> 1, side = inc & 1;
              const int jn = G.pf_j[f];
              if (jn < 0) continue;
              const int o = side ? G.pf_i[f] : jn;
              const double ho = hat2(o, b);
              if (ho == 0.0) continue;
              const double blk = side ? ldc(G.PF + (size_t)f * 120 + 72 + cc * 6 + r) : ldc(G.PF + (size_t)f * 120 + 72 + r * 6 + cc);
              v += ha * ho * blk;
            }
          }
        }
        S0[i * LD + j] = v;
      }
      __syncthreads();
      const int q1 = G.g2_ptr[g + 1];
      int q = G.g2_ptr[g];
      while (q < q1) {   // (uniform across the CTA)
        const int l = G.ce2_plane[G.g2_ce[q]];
        int qe = q + 1;
        while (qe < q1 && G.ce2_plane[G.g2_ce[qe]] == l) qe++;
        const int m = qe - q;
        for (int i = tid; i < m * 18; i += kThreads) {
          const int ce = G.g2_ce[q + i / 18];
          Yst[i] = ldc(G.Yc2 + (size_t)ce * 18 + i % 18);
          Wst[i] = ldc(G.Wc2 + (size_t)ce * 18 + i % 18);
        }
        if (tid < m) nloc[tid] = G.ce2_node[G.g2_ce[q + tid]] - a0;
        __syncthreads();
        for (int idx = tid; idx < m * m * 36; idx += kThreads) {
          const int mi = idx / (36 * m), rem = idx - mi * 36 * m, mj = rem / 36, en = rem - mj * 36, r = en / 6, cc = en - r * 6;
          const double* y = Yst + mi * 18 + r * 3;
          const double* w = Wst + mj * 18 + cc * 3;
          S0[(nloc[mi] * 6 + r) * LD + nloc[mj] * 6 + cc] -= y[0] * w[0] + y[1] * w[1] + y[2] * w[2];
        }
        __syncthreads();
        q = qe;
      }
      const double* inv = gj_invert_smem<kBlockDim / 8, LD>(S0, S1, TQ);
      double* out = G.D2inv + (size_t)g * kBlockDim * kBlockDim;
      for (int i = tid; i < kBlockDim * kBlockDim; i += kThreads) out[i] = inv[(i / kBlockDim) * LD + i % kBlockDim];
    }
    __syncthreads();
  }

  // -------- Schur setup, part 4: A_c = P^T S P, lower triangle of 48x48 tiles --------
  // Output-stationary: every thread owns entries (i, j) of the triangle of A_c = P^T S P and writes each exactly once
  // (coalesced along j inside a tile row):  pose part (supports of the two nodes overlap: |a-b| <= 1), pose-pose factors
  // coupling the supports (host-built per-pair list), light planes (host-built per-pair list of (Yc, Wc) products),
  // heavy planes (Yc / Wc rows of the plane staged per node in shared memory: dense rank-3 update, one pass each).
  // Tile column 0 also goes to the step-0 pivot-column snapshot of coarse_invert().
  __device__ void coarse_assemble(double lambda) {
    const int ldm = G.ldmc, nc = G.nc, n6 = 6 * nc, nb = ldm / 48;
    double* Yh = reinterpret_cast<double*>(g_smem + kSmWork);   // [nc][18]
    double* Wh = Yh + (size_t)nc * 18;                          // [nc][18]
    const int npass = max(1, G.n_hv);
    const long long total = (long long)ac_ntri(ldm) * 48 * 48;
    for (int pass = 0; pass < npass; pass++) {
      if (G.n_hv > 0) {
        __syncthreads();
        for (int i = threadIdx.x; i < nc * 36; i += kThreads) Yh[i] = 0.0;
        __syncthreads();
        const int l = G.hv_plane[pass];
        for (int i = threadIdx.x; i < (G.ce_ptr[l + 1] - G.ce_ptr[l]) * 18; i += kThreads) {
          const int ce = G.ce_ptr[l] + i / 18, kk = i % 18, node = G.ce_node[ce];
          Yh[node * 18 + kk] = ldc(G.Yc + (size_t)ce * 18 + kk);
          Wh[node * 18 + kk] = ldc(G.Wc + (size_t)ce * 18 + kk);
        }
        __syncthreads();
      }
      int tprev = -1, ti = 0, tj = 0;
      for (long long idx = tid_team(); idx < total; idx += nthr_team()) {
        const int t = (int)(idx / 2304), e = (int)(idx - (long long)t * 2304), er = e / 48, ec = e - er * 48;
        if (t != tprev) { tri_tile(nb, t, ti, tj); tprev = t; }
        const int i = 48 * ti + er, j = 48 * tj + ec;
        double* out = G.Atri + (size_t)t * kAcTile + er * kAcLd + ec;
        double* snap = (tj == 0) ? G.Apan + (size_t)ti * kAcTile + er * kAcLd + ec : nullptr;
        if (i >= n6 || j >= n6) {   // padding: identity
          if (pass == 0) {
            const double v = (i == j) ? 1.0 : 0.0;
            *out = v;
            if (snap) *snap = v;
          }
          continue;
        }
        const int a = i / 6, r = i - a * 6, b = j / 6, cc = j - b * 6;
        double v;
        if (pass == 0) {
          v = 0.0;
          if (a - b <= 1 && b - a <= 1) {   // P^T Hpp_d P on the overlap of the two supports
            const int plo = max(0, (max(a, b) - 1) * G.SP + 1), phi = min(G.N, (min(a, b) + 1) * G.SP);
            for (int p = plo; p < phi; p++) {
              double h = ldc(G.Hpp + (size_t)p * 36 + r * 6 + cc);
              if (r == cc) h *= (1 + lambda);
              v += hat(p, a) * hat(p, b) * h;
            }
          }
          const size_t pair = (size_t)a * nc + b;
          for (int k = G.fp_ptr[pair]; k < G.fp_ptr[pair + 1]; k++) {   // pose-pose blocks of Hpp
            const int fs = G.fp_f[k], f = fs >> 1, side = fs & 1;
            const int p = side ? G.pf_j[f] : G.pf_i[f], o = side ? G.pf_i[f] : G.pf_j[f];
            const double blk = side ? ldc(G.PF + (size_t)f * 120 + 72 + cc * 6 + r) : ldc(G.PF + (size_t)f * 120 + 72 + r * 6 + cc);
            v += hat(p, a) * hat(o, b) * blk;
          }
          for (int k = G.lp_ptr[pair]; k < G.lp_ptr[pair + 1]; k++) {   // minus Wc[a,l] Hll^-1 Wc[b,l]^T, light planes
            const double* y = G.Yc + (size_t)G.lp_cea[k] * 18 + r * 3;
            const double* w = G.Wc + (size_t)G.lp_ceb[k] * 18 + cc * 3;
            v -= ldc(y) * ldc(w) + ldc(y + 1) * ldc(w + 1) + ldc(y + 2) * ldc(w + 2);
          }
        } else {
          v = *out;   // written by this same thread in the previous pass
        }
        if (G.n_hv > 0) {
          const double* y = Yh + a * 18 + r * 3;
          const double* w = Wh + b * 18 + cc * 3;
          v -= y[0] * w[0] + y[1] * w[1] + y[2] * w[2];
        }
        *out = v;
        if (snap) *snap = v;
      }
    }
    fence_proxy_async();  // the snapshot is read by bulk copies in coarse_invert()
  }

  // -------- Schur setup, part 5: A_c^-1 by an in-place symmetric block sweep of the triangle ---------
  // Step K (pivot block K, P = A_KK^-1):  A_KK <- -P,  A_iK <- A_iK P,  A_ij <- A_ij - A_iK P A_Kj  (i, j != K).  The
  // matrix stays symmetric, so only the tiles (i, j), i >= j, are kept; after the last step they hold -A_c^-1.  SPD: no
  // pivoting.  Every CTA owns a contiguous range of tile numbers (a compact patch, see tri_index) for the whole inversion.
  // Step K overwrites pivot column K, so it reads only a snapshot of that column (C_i = A_iK, taken by the owners of
  // those tiles at the end of step K-1; double-buffered by step parity), P and the CTA's own tiles:  T_i = -C_i P once per
  // tile row of a band, then, column by column, the snapshot tile C_j streams in by bulk copy (two more in flight)
  // and every owned tile of the column gets  (i,j): A_ij + T_i C_j^T,  (K,j): P C_j^T,  (i,K): -T_i,  (K,K): -P
  // on the FP64 tensor cores.  Look-ahead: the owner of diagonal tile K+1 updates that tile first, inverts it and
  // publishes P_{K+1} before it updates the rest, so no CTA inverts a pivot redundantly (kPivotWeight gives it fewer
  // tiles).  One team barrier per step.  The last step writes -(its result), mirrored and rounded to fp32, into the full
  // layout of G.Ac.
  __device__ void coarse_invert() {
    const int ldm = G.ldmc, nb = ldm / 48, nt = ac_ntri(ldm);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, fr = lane >> 2, fc = lane & 3;
    double* Ps = reinterpret_cast<double*>(g_smem + kSmWork);   // P_K
    double* Tr = Ps + kAcTile;                                  // [2] T_i of the two tile rows of the current band
    double* Cb = Tr + 2 * kAcTile;                              // [3] snapshot tiles C_j (ring)
    double* Sb = Cb + 3 * kAcTile;                              // [2] C_i while T_i is formed; pivot inversion
    double* TQ = Sb + 2 * kAcTile;                              // [48][12] coefficient columns of gj_invert_smem
    int* rng = reinterpret_cast<int*>(TQ + 48 * 12);            // owned tile numbers [rng[0], rng[1])
    unsigned long long* mb = reinterpret_cast<unsigned long long*>(g_smem + kSmGjBar);   // [0..2]: Cb; [3]: Ps, Sb
    double* piv = G.Apan + (size_t)2 * nb * kAcTile;            // [2] P_K by step parity

    // owner(t): the CTA whose share of the total weight holds the middle of tile t (a diagonal tile weighs 1 + kPivotWeight)
    if (tid < 2) rng[tid] = nt;
    __syncthreads();
    {
      const long long T = c.tsize, W2 = 2ll * (nt + (long long)kPivotWeight * nb);
      auto owner = [&](int t) {
        int i, j;
        tri_tile(nb, t, i, j);
        const int b = i >> 1;
        const long long before = t + (long long)kPivotWeight * (2 * b + ((i == 2 * b + 1 && j >= 2 * b) ? 1 : 0));
        return (int)min(T - 1, (2 * before + 1 + (i == j ? kPivotWeight : 0)) * T / W2);
      };
      for (int t = tid; t < nt; t += kThreads) {
        const int o = owner(t), op = t > 0 ? owner(t - 1) : -1;
        if (o >= c.rank && op < c.rank) rng[0] = t;
        if (o > c.rank && op <= c.rank) rng[1] = t;
      }
    }
    __syncthreads();
    const int t0 = rng[0], t1 = rng[1];

    // bulk copies of up to three tiles on one mbarrier phase (the CTA's last accesses of dst are behind a barrier)
    auto fetch = [&](int bar, int n, double* d0, const double* s0, double* d1 = nullptr, const double* s1 = nullptr,
                     double* d2 = nullptr, const double* s2 = nullptr) {
      if (tid == 0) {
        fence_proxy_async();
        mbar_expect_tx(mb + bar, (unsigned)(n * kAcTile * 8));
        tma_copy_1d(d0, s0, (unsigned)(kAcTile * 8), mb + bar);
        if (n > 1) tma_copy_1d(d1, s1, (unsigned)(kAcTile * 8), mb + bar);
        if (n > 2) tma_copy_1d(d2, s2, (unsigned)(kAcTile * 8), mb + bar);
      }
    };
    auto wait = [&](int bar) {
      mbar_wait(mb + bar, (c.gj_par >> bar) & 1u);
      c.gj_par ^= 1u << bar;
    };
    auto frag = [&](int s, int& r, int& cc) {   // position of accumulator s of mma48 in the 48x48 tile
      const int q = warp + 16 * s;
      r = 8 * (q / 6) + fr;
      cc = 8 * (q % 6) + 2 * fc;
      return q < 36;
    };
    auto form_T = [&](double* dst, const double* Ci) {   // dst = -Ci P
      double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
      mma48<false>(acc, Ci, Ps);
      int r, cc;
#pragma unroll
      for (int s = 0; s < 3; s++)
        if (frag(s, r, cc)) *reinterpret_cast<double2*>(dst + r * kAcLd + cc) = make_double2(-acc[s][0], -acc[s][1]);
    };
    auto group_end = [&](int t) {   // one past the column group that starts at owned tile t (the tiles of one column in one band)
      int i, j, i2, j2;
      tri_tile(nb, t, i, j);
      if (t + 1 < t1) {
        tri_tile(nb, t + 1, i2, j2);
        if (j2 == j && (i2 >> 1) == (i >> 1)) return t + 2;
      }
      return t + 1;
    };
    auto load_base = [&](int t, double (&acc)[3][2]) {
      const double* tile = G.Atri + (size_t)t * kAcTile;
      int r, cc;
#pragma unroll
      for (int s = 0; s < 3; s++)
        if (frag(s, r, cc)) {
          const double2 v = __ldcg(reinterpret_cast<const double2*>(tile + r * kAcLd + cc));
          acc[s][0] = v.x;
          acc[s][1] = v.y;
        }
    };

    for (int K = 0; K < nb; K++) {
      const bool last = (K == nb - 1);
      const double* snap = G.Apan + (size_t)(K & 1) * nb * kAcTile;    // C_i = snap + i kAcTile
      double* snapn = G.Apan + (size_t)((K + 1) & 1) * nb * kAcTile;   // the snapshot for step K + 1
      auto tile_col = [&](int t) { int i, j; tri_tile(nb, t, i, j); return j; };
      auto issue_col = [&](int t, int slot) {   // the snapshot tile of the column group starting at t, unless it is column K
        if (t < t1 && tile_col(t) != K) fetch(slot, 1, Cb + slot * kAcTile, snap + (size_t)tile_col(t) * kAcTile);
      };
      issue_col(t0, 0);
      if (t0 < t1) issue_col(group_end(t0), 1);
      const int d = K + 1;
      const bool ahead = !last && tri_index(nb, d, d) >= t0 && tri_index(nb, d, d) < t1;   // this CTA inverts the next pivot
      // P_K (for K = 0 nobody has published it: every CTA inverts A_00, snapshot tile 0), and C_{K+1} for the look-ahead
      if (K == 0) fetch(3, ahead ? 2 : 1, Sb + kAcTile, snap, Sb, snap + (size_t)d * kAcTile);
      else fetch(3, ahead ? 2 : 1, Ps, piv + (size_t)(K & 1) * kAcTile, Sb, snap + (size_t)d * kAcTile);
      wait(3);
      if (K == 0) {
        const double* inv = gj_invert_smem<6, kAcLd>(Sb + kAcTile, Ps, TQ);
        if (inv != Ps)
          for (int e = tid; e < 48 * 48; e += kThreads) Ps[(e / 48) * kAcLd + e % 48] = inv[(e / 48) * kAcLd + e % 48];
      }
      __syncthreads();
      lap1(7);
      // look-ahead: diagonal tile K+1 first, then P_{K+1} = its inverse for the next step
      if (ahead) {
        form_T(Tr, Sb);
        __syncthreads();
        double acc[3][2];
        load_base(tri_index(nb, d, d), acc);
        mma48<true>(acc, Tr, Sb);
        double* Md = Tr + kAcTile;
        int r, cc;
#pragma unroll
        for (int s = 0; s < 3; s++)
          if (frag(s, r, cc)) *reinterpret_cast<double2*>(Md + r * kAcLd + cc) = make_double2(acc[s][0], acc[s][1]);
        __syncthreads();
        const double* inv = gj_invert_smem<6, kAcLd>(Md, Sb + kAcTile, TQ);
        double* out = piv + (size_t)(d & 1) * kAcTile;
        for (int e = tid; e < 48 * 48; e += kThreads) out[(e / 48) * kAcLd + e % 48] = inv[(e / 48) * kAcLd + e % 48];
        __syncthreads();
      }
      lap1(6);
      // the owned tiles, column group by column group (a group: the tiles of one column inside one band, at most two)
      int band = -1, g = 0;
      for (int t = t0; t < t1;) {
        int i0, j;
        tri_tile(nb, t, i0, j);
        const int b = i0 >> 1, te = group_end(t);
        if (b != band) {   // T_i of the band's rows that the owned tiles need
          band = b;
          bool need[2] = {false, false};
          for (int u = t; u < min(t1, (b + 1) * (2 * b + 3)); u++) {
            int iu, ju;
            tri_tile(nb, u, iu, ju);
            if (iu != K) need[iu - 2 * b] = true;
          }
          if (need[0] || need[1]) {
            const int r0 = need[0] ? 0 : 1;
            fetch(3, need[0] && need[1] ? 2 : 1, Sb + r0 * kAcTile, snap + (size_t)(2 * b + r0) * kAcTile, Sb + kAcTile,
                  snap + (size_t)(2 * b + 1) * kAcTile);
            wait(3);
            for (int r = 0; r < 2; r++)
              if (need[r]) form_T(Tr + r * kAcTile, Sb + r * kAcTile);
            __syncthreads();
          }
          lap1(7);
        }
        if (te < t1) issue_col(group_end(te), (g + 2) % 3);
        // the tiles' own values are read while the snapshot tile is still in flight
        double acc[2][3][2];
#pragma unroll
        for (int k = 0; k < 2; k++) {
          int i, jj;
          if (t + k < te) tri_tile(nb, t + k, i, jj);
#pragma unroll
          for (int s = 0; s < 3; s++) acc[k][s][0] = acc[k][s][1] = 0.0;
          if (t + k < te && i != K && j != K) load_base(t + k, acc[k]);
        }
        if (j != K) wait(g % 3);
        const double* Cj = Cb + (g % 3) * kAcTile;
#pragma unroll
        for (int k = 0; k < 2; k++) {
          const int u = t + k;
          if (u >= te) continue;
          int i, jj;
          tri_tile(nb, u, i, jj);
          if (!last && i == d && j == d) continue;   // done by the look-ahead
          const double* Ti = Tr + (i - 2 * b) * kAcTile;
          int r, cc;
          if (j == K) {   // (K,K): -P;  (i,K): -T_i
            const double* src = (i == K) ? Ps : Ti;
#pragma unroll
            for (int s = 0; s < 3; s++)
              if (frag(s, r, cc)) { acc[k][s][0] = -src[r * kAcLd + cc]; acc[k][s][1] = -src[r * kAcLd + cc + 1]; }
          } else if (i == K) {
            mma48<true>(acc[k], Ps, Cj);
          } else {
            mma48<true>(acc[k], Ti, Cj);
          }
#pragma unroll
          for (int s = 0; s < 3; s++) {
            if (!frag(s, r, cc)) continue;
            if (last) {   // -(result) into the apply layout in fp32, mirrored (both copies get one rounding: exactly symmetric);
                          // a diagonal tile contributes its lower half only
              const int R = 48 * i + r, C = 48 * j + cc;
              const float v0 = (float)-acc[k][s][0], v1 = (float)-acc[k][s][1];
              if (i != j) {
                *reinterpret_cast<float2*>(G.Ac + ac_index(ldm, R, C)) = make_float2(v0, v1);
                G.Ac[ac_index(ldm, C, R)] = v0;
                G.Ac[ac_index(ldm, C + 1, R)] = v1;
              } else {
                if (r >= cc) { G.Ac[ac_index(ldm, R, C)] = v0; G.Ac[ac_index(ldm, C, R)] = v0; }
                if (r >= cc + 1) { G.Ac[ac_index(ldm, R, C + 1)] = v1; G.Ac[ac_index(ldm, C + 1, R)] = v1; }
              }
            } else {
              *reinterpret_cast<double2*>(G.Atri + (size_t)u * kAcTile + r * kAcLd + cc) = make_double2(acc[k][s][0], acc[k][s][1]);
              if (i == d) {   // C_j = A_{j,K+1} = A_{K+1,j}^T
                snapn[(size_t)j * kAcTile + cc * kAcLd + r] = acc[k][s][0];
                snapn[(size_t)j * kAcTile + (cc + 1) * kAcLd + r] = acc[k][s][1];
              } else if (j == d) {
                *reinterpret_cast<double2*>(snapn + (size_t)i * kAcTile + r * kAcLd + cc) = make_double2(acc[k][s][0], acc[k][s][1]);
              }
            }
          }
        }
        __syncthreads();   // Cb[g % 3] is free for group g + 3
        g++;
        t = te;
      }
      lap1(21);
      fence_proxy_async();   // the snapshot and P_{K+1} are read by bulk copies in the next step
      team_barrier(c);
      lap1(22);
    }
  }

  // -------- plane-major sweep: upart = segmented sums of Wt^T * (va + beta*vb)[pose] --------
  // (zc != nullptr: the gathered vector also gets its coarse part P*zc added on the fly, see precondition())
  __device__ void sweep_planes(const double* va, const double* vb, double beta, const double* zc = nullptr) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int step = nwarp_team();
    if (c.use_tma) {
      // Large graphs: a warp owns several tiles.  Software pipeline, three tiles deep: the Wt tile after this one
      // (4608 contiguous bytes) is in flight as one bulk async copy into the other staging buffer, the per-edge
      // gathers of the next tile are issued before this tile is multiplied, and the edge indices are read two tiles
      // ahead -- no dependent-load latency is exposed in steady state.
      double* buf = reinterpret_cast<double*>(g_smem + kSmTma) + warp * 2 * kWStride;
      unsigned long long* bar = reinterpret_cast<unsigned long long*>(g_smem + kSmBar) + warp * 2;
      int tile = warp_team(), st = 0;
      __syncwarp();
      if (lane == 0 && tile < G.ntile_pl) {
        fence_proxy_async();
        tma_load_1d(buf, G.Wt + (size_t)tile * kWStride, kTileBytes, bar);
      }
      // (on large graphs the callers pass one fully formed vector: vb == nullptr, zc == nullptr)
      int keyC = -1, pC = 0, keyN = -1, pN = 0;
      if (tile < G.ntile_pl) { keyC = G.pl_plane[tile * 32 + lane]; pC = G.pl_pose[tile * 32 + lane]; }
      if (tile + step < G.ntile_pl) { keyN = G.pl_plane[(tile + step) * 32 + lane]; pN = G.pl_pose[(tile + step) * 32 + lane]; }
      double x[6] = {0, 0, 0, 0, 0, 0};
      if (keyC >= 0)
        for (int a = 0; a < 6; a++) x[a] = ldc(va + (size_t)pC * 6 + a);
      for (; tile < G.ntile_pl; tile += step, st ^= 1) {
        if (lane == 0 && tile + step < G.ntile_pl)
          tma_load_1d(buf + (st ^ 1) * kWStride, G.Wt + (size_t)(tile + step) * kWStride, kTileBytes, bar + (st ^ 1));
        int keyNN = -1, pNN = 0;
        if (tile + 2 * step < G.ntile_pl) { keyNN = G.pl_plane[(tile + 2 * step) * 32 + lane]; pNN = G.pl_pose[(tile + 2 * step) * 32 + lane]; }
        double xn[6] = {0, 0, 0, 0, 0, 0};   // gathers of the next tile, consumed in the next iteration
        if (keyN >= 0) {
#pragma unroll
          for (int a = 0; a < 6; a++) xn[a] = ldc(va + (size_t)pN * 6 + a);
        }
        double u[3] = {0, 0, 0};
        mbar_wait(bar + st, (c.tma_par >> st) & 1u);
        c.tma_par ^= (1u << st);
        if (keyC >= 0) tile_wt_x<LdS>(buf + st * kWStride + lane, x, u);
        if (seg_suffix_sum<3>(keyC, u)) {
          double* o = G.upart + (size_t)G.pl_part[tile * 32 + lane] * 3;
          put(c, o, u[0]); put(c, o + 1, u[1]); put(c, o + 2, u[2]);
        }
#pragma unroll
        for (int a = 0; a < 6; a++) x[a] = xn[a];
        keyC = keyN; pC = pN; keyN = keyNN; pN = pNN;
        __syncwarp();  // every lane is done with this stage before lane 0 refills it
      }
      return;
    }
    for (int tile = warp_team(); tile < G.ntile_pl; tile += step) {
      int s = tile * 32 + lane;
      int key = G.pl_plane[s];
      double u[3] = {0, 0, 0};
      if (key >= 0) {
        int p = G.pl_pose[s];
        double x[6];
        for (int a = 0; a < 6; a++) x[a] = ldc(va + (size_t)p * 6 + a);
        if (vb) for (int a = 0; a < 6; a++) x[a] += beta * ldc(vb + (size_t)p * 6 + a);
        if (zc) {
          if (G.levels != 3) {
            const int c0 = p / G.SP;
            const double h0 = hat(p, c0), h1 = hat(p, c0 + 1);
            const double* z0 = zc + (size_t)c0 * 6;
            const double* z1 = zc + (size_t)min(c0 + 1, G.nc - 1) * 6;
            for (int a = 0; a < 6; a++) x[a] += h0 * ldc(z0 + a) + h1 * ldc(z1 + a);
          } else {
            for (int a = 0; a < 6; a++) x[a] += coarse_z(p, a);
          }
        }
        tile_wt_x<LdL2>(G.Wt + (size_t)tile * kWStride + lane, x, u);
      }
      if (seg_suffix_sum<3>(key, u)) {
        double* o = G.upart + (size_t)G.pl_part[s] * 3;
        put(c, o, u[0]); put(c, o + 1, u[1]); put(c, o + 2, u[2]);
      }
    }
  }

  // -------- plane solve: mode 0: vl = Hinv * sum(upart) ; mode 1: dl = Hinv * (-gl - sum(upart)), returns |dl|^2
  __device__ double solve_planes(int mode) {
    const int lane = threadIdx.x & 31;
    double nrm = 0;
    for (int l = warp_team(); l < G.M; l += nwarp_team()) {
      double u[3] = {0, 0, 0};
      for (int k = G.upart_ptr[l] + lane; k < G.upart_ptr[l + 1]; k += 32)
        for (int b = 0; b < 3; b++) u[b] += ldc(G.upart + (size_t)k * 3 + b);
      for (int b = 0; b < 3; b++) u[b] = warp_sum(u[b]);
      if (lane == 0) {
        double Hi[9];
        for (int t = 0; t < 9; t++) Hi[t] = ldc(G.Hinv + (size_t)l * 9 + t);
        if (mode == 1) for (int b = 0; b < 3; b++) u[b] = -ldc(G.gl + (size_t)l * 3 + b) - u[b];
        double* o = (mode == 0 ? G.vl : G.dl) + (size_t)l * 3;
        for (int t = 0; t < 3; t++) {
          double v = dot3(Hi + t * 3, u);
          put(c, o + t, v);
          nrm += v * v;
        }
      }
    }
    return nrm;
  }

  // -------- large graphs: vl = Hll_d^-1 * sum(upart) for the heavy planes only (> 8 partial sums), once per PCG
  // iteration instead of once per pose block inside pose_phase()
  __device__ void solve_heavy() {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // planes with > 512 partial sums (a ground plane seen from every pose): one CTA each, fixed-order tree
    for (int hh = c.rank; hh < G.n_huge; hh += c.tsize) {
      const int l = G.huge[hh];
      const int t0 = G.upart_ptr[l], n = G.upart_ptr[l + 1] - t0;
      double* s = reinterpret_cast<double*>(g_smem + kSmRed);
      double uu[3] = {0, 0, 0};
      for (int tb = t0 + (int)threadIdx.x; tb < t0 + n; tb += 4 * kThreads) {
        double pr[4][3];
#pragma unroll
        for (int t = 0; t < 4; t++)
#pragma unroll
          for (int b = 0; b < 3; b++) pr[t][b] = (tb + kThreads * t < t0 + n) ? ldc(G.upart + (size_t)(tb + kThreads * t) * 3 + b) : 0.0;
#pragma unroll
        for (int t = 0; t < 4; t++)
#pragma unroll
          for (int b = 0; b < 3; b++) uu[b] += pr[t][b];
      }
      for (int b = 0; b < 3; b++) uu[b] = warp_sum(uu[b]);
      __syncthreads();
      if (lane == 0) for (int b = 0; b < 3; b++) s[warp * 4 + b] = uu[b];
      __syncthreads();
      if (threadIdx.x < 3) {
        double tot[3] = {0, 0, 0};
        for (int w = 0; w < kWarps; w++)
          for (int b = 0; b < 3; b++) tot[b] += s[w * 4 + b];
        const int o = threadIdx.x;
        put(c, &G.vl[(size_t)l * 3 + o], dot3<LdL2>(G.Hinv + (size_t)l * 9 + o * 3, tot));
      }
      __syncthreads();
    }
    for (int h = warp_team(); h < G.n_heavy; h += nwarp_team()) {
      const int l = G.heavy[h];
      if (l < 0) continue;
      double uu[3];
      warp_sum_partials(G.upart, G.upart_ptr[l], G.upart_ptr[l + 1], lane, uu);
      if (lane < 3) put(c, &G.vl[(size_t)l * 3 + lane], dot3<LdL2>(G.Hinv + (size_t)l * 9 + lane * 3, uu));
    }
  }

  // number of rounds every CTA of the team runs over its owned pose blocks
  __device__ __forceinline__ int rounds() const { return (G.nblk + c.tsize * kSlots - 1) / (c.tsize * kSlots); }

  // coarse restriction of the per-slot vector in `sv` (smem [kSlots][96]); writes 12 values per block
  __device__ __forceinline__ void restrict_block(const double* sv, int slot, int u, int k, int np, double* out) {
    if (u < 12 && k < G.nblk) {
      int node = u / 6, row = u % 6;
      int p0 = k * kBlockPoses, c0 = p0 / sp_r();
      double acc = 0;
      for (int pi = 0; pi < np; pi++) acc += hat_r(p0 + pi, c0 + node) * sv[slot * kBlockDim + pi * 6 + row];
      put(c, &out[(size_t)k * 12 + u], acc);
    }
  }

  // -------- PCG: owner part of the direction update p_new = z + beta p_old --------
  __device__ void update_direction(int cur, double beta) {
    const int tid = threadIdx.x, slot = tid / kBlockDim, u = tid % kBlockDim;
    const int nrounds = rounds();
    for (int rd = 0; rd < nrounds; rd++) {
      int k = c.rank + c.tsize * (slot + kSlots * rd);
      int p = k * kBlockPoses + u / 6;
      if (slot < kSlots && k < G.nblk && p < G.N) {
        const int row = u % 6;
        size_t o = (size_t)p * 6 + row;
        put(c, &G.pv[cur ^ 1][o], ldc(G.z + o) + beta * ldc(G.pv[cur] + o) + coarse_z(p, row));
      }
    }
  }

  // -------- fused pose phase, per owned 16-pose block and entirely inside the owning CTA:
  //   1. v_g  = Hll^-1 * (sum of the plane-major partials of plane g)     [apply]   or   Hll^-1 gl   [rhs]
  //   2. y    = segmented sums over the block's pose-major tiles of W_e * v_{g(e)}        (shared memory)
  //   3. apply: q = (Hpp + lambda diag) p + (pose-pose blocks) p_other - y ; qc = P^T q ; returns partial p.q
  //      rhs  : b = -gp + y ; x = 0, r = b, p = z = q = 0 ; rcpart[0] = P^T b
  // A block with more than kMaxGrp plane groups or kMaxPart (tile, pose) runs keeps v_g and the run sums in its own range of
  // the global overflow scratch (offset blk_ovf[k], written and read only by the owning CTA, through L2) instead of shared
  // memory; the sums and their order are the same.
  __device__ double pose_phase(bool rhs, const double* pvec, double lambda, double* qout, double* qc) {
    double* sA = reinterpret_cast<double*>(g_smem + kSmA);
    double* vg = reinterpret_cast<double*>(g_smem + kSmVg);
    double* yp = reinterpret_cast<double*>(g_smem + kSmYp);
    const int tid = threadIdx.x, slot = tid / kBlockDim, u = tid % kBlockDim;
    const int lane = tid & 31, wis = u >> 5;  // warp within the slot (3 warps per slot)
    double* tbuf = reinterpret_cast<double*>(g_smem + kSmTma) + (tid >> 5) * 2 * kWStride;  // TMA staging (large graphs)
    unsigned long long* tbar = reinterpret_cast<unsigned long long*>(g_smem + kSmBar) + (tid >> 5) * 2;
    double dot = 0;
    const int nrounds = rounds();
    // plane-group record of this thread for the coming round (static data, read one round ahead)
    int g0N = 0, ngN = 0, ovN = -1;
    int4 giN = make_int4(0, 0, 0, 0);
    auto next_groups = [&](int rd) {
      const int k = c.rank + c.tsize * (slot + kSlots * rd);
      g0N = 0; ngN = 0; ovN = -1;
      if (rd < nrounds && slot < kSlots && k < G.nblk) {
        g0N = G.blk_grp_ptr[k];
        ngN = G.blk_grp_ptr[k + 1] - g0N;
        if (u < ngN) giN = *reinterpret_cast<const int4*>(G.grp_info + (size_t)(g0N + u) * 4);
        if (G.n_ovf_blk) ovN = G.blk_ovf[k];
      }
    };
    next_groups(0);
    for (int rd = 0; rd < nrounds; rd++) {
      const int k = c.rank + c.tsize * (slot + kSlots * rd);
      const bool live = (slot < kSlots) && (k < G.nblk);
      const int p = k * kBlockPoses + u / 6, row = u % 6;
      const int np = live ? min(kBlockPoses, G.N - k * kBlockPoses) : 0;
      const bool on = live && (p < G.N);
      const int g0 = g0N, ng = ngN;
      const int4 gi0 = giN;
      // over-limit block: v_g at ovf[ov + 3 g], the run sums at ovf[ov + 3 ng + 6 (part - part0)]  (uniform per slot)
      const int ov = ovN;
      __syncthreads();
      next_groups(rd + 1);
      if (slot < kSlots) sA[slot * kBlockDim + u] = 0.0;
      // first W tile of this warp (large graphs: bulk copy) and its edge indices: in flight while the plane-group
      // vectors are formed
      int keyN = -1, gosN = 0, partN = 0;
      if (live) {
        const int t0 = G.tile_ptr[k], nt = G.tile_ptr[k + 1] - t0;
        if (wis < nt) {
          if (c.use_tma && lane == 0) {
            fence_proxy_async();
            tma_load_1d(tbuf, G.W + (size_t)(t0 + wis) * kWStride, kTileBytes, tbar);
          }
          const int e = (t0 + wis) * 32 + lane;
          keyN = G.pp_pose[e]; gosN = G.grp_of_slot[e]; partN = G.pm_part[e];
        }
      }
      if (live) {
        // plane-group vectors: one thread per group when the plane has <= 8 partial sums (all loads in one
        // batch), one warp per group for heavy planes (the ground plane is seen from every pose)
        for (int g = u; g < ng; g += kBlockDim) {
          const int4 gi = (g == u) ? gi0 : *reinterpret_cast<const int4*>(G.grp_info + (size_t)(g0 + g) * 4);
          const int l = gi.x;
          double vv[3];
          bool set = true;
          if (rhs) {
            for (int b = 0; b < 3; b++) vv[b] = ldc(G.vl + (size_t)l * 3 + b);
          } else {
            if (gi.z <= 8) {
              plane_vec_small(G.upart, gi.y, gi.z, l, vv);
            } else if (c.use_tma) {   // large graph: solve_heavy() already reduced this plane
              for (int b = 0; b < 3; b++) vv[b] = ldc(G.vl + (size_t)l * 3 + b);
            } else {
              set = false;            // heavy plane: summed by a warp below
            }
          }
          if (set) {
            if (ov < 0) {
              for (int b = 0; b < 3; b++) vg[(slot * kMaxGrp + g) * 3 + b] = vv[b];
            } else {
              for (int b = 0; b < 3; b++) __stcg(G.ovf + ov + g * 3 + b, vv[b]);
            }
          }
        }
        if (!rhs && !c.use_tma) {
          for (int g = wis; g < ng; g += 3) {   // heavy planes: a warp sums the partials
            const int l = G.grp_plane[g0 + g];
            const int t0 = G.upart_ptr[l], n = G.upart_ptr[l + 1] - t0;
            if (n <= 8) continue;
            double uu[3];
            warp_sum_partials(G.upart, t0, t0 + n, lane, uu);
            if (lane < 3) {
              const double v = dot3<LdL2>(G.Hinv + (size_t)l * 9 + lane * 3, uu);
              if (ov < 0) vg[(slot * kMaxGrp + g) * 3 + lane] = v;
              else __stcg(G.ovf + ov + g * 3 + lane, v);
            }
          }
        }
      }
      __syncthreads();
      if (!rhs) lap(21);
      if (live) {
        const int t0 = G.tile_ptr[k], nt = G.tile_ptr[k + 1] - t0, part0 = G.blk_part_ptr[k];
        int st = 0;
        // (edge indices are read one tile ahead: static arrays whose latency would otherwise be exposed per tile)
        for (int t = wis; t < nt; t += 3, st ^= 1) {
          if (c.use_tma && lane == 0 && t + 3 < nt)
            tma_load_1d(tbuf + (st ^ 1) * kWStride, G.W + (size_t)(t0 + t + 3) * kWStride, kTileBytes, tbar + (st ^ 1));
          const int key = keyN, gos = gosN, part = partN;
          if (t + 3 < nt) {
            const int e = (t0 + t + 3) * 32 + lane;
            keyN = G.pp_pose[e]; gosN = G.grp_of_slot[e]; partN = G.pm_part[e];
          }
          double y[6] = {0, 0, 0, 0, 0, 0};
          double v0 = 0, v1 = 0, v2 = 0;
          if (key >= 0) {
            if (ov < 0) {
              const double* v = vg + (slot * kMaxGrp + gos) * 3;
              v0 = v[0]; v1 = v[1]; v2 = v[2];
            } else {
              const double* v = G.ovf + ov + gos * 3;
              v0 = __ldcg(v); v1 = __ldcg(v + 1); v2 = __ldcg(v + 2);
            }
          }
          if (c.use_tma) {
            mbar_wait(tbar + st, (c.tma_par >> st) & 1u);
            c.tma_par ^= (1u << st);
            if (key >= 0) tile_w_v<LdS>(tbuf + st * kWStride + lane, v0, v1, v2, y);
          } else if (key >= 0) {
            tile_w_v<LdL2>(G.W + (size_t)(t0 + t) * kWStride + lane, v0, v1, v2, y);
          }
          if (seg_suffix_sum<6>(key, y)) {
            if (ov < 0) {
              double* o = yp + (slot * kMaxPart + (part - part0)) * 6;
              for (int a = 0; a < 6; a++) o[a] = y[a];
            } else {
              double* o = G.ovf + ov + ng * 3 + (part - part0) * 6;
              for (int a = 0; a < 6; a++) __stcg(o + a, y[a]);
            }
          }
          __syncwarp();  // stage consumed by every lane before it is refilled
        }
      }
      __syncthreads();
      if (!rhs) lap(22);
      if (on) {
        const int part0 = G.blk_part_ptr[k];
        double ysum = 0;
        if (ov < 0) {
          for (int t = G.ypart_ptr[p]; t < G.ypart_ptr[p + 1]; t++) ysum += yp[(slot * kMaxPart + (t - part0)) * 6 + row];
        } else {
          const double* ys = G.ovf + ov + ng * 3 + row;
          for (int t = G.ypart_ptr[p]; t < G.ypart_ptr[p + 1]; t++) ysum += __ldcg(ys + (t - part0) * 6);
        }
        const size_t o = (size_t)p * 6 + row;
        if (rhs) {
          double v = -ldc(G.gp + o) + ysum;
          put(c, &G.b[o], v); put(c, &G.r[o], v); put(c, &G.x[o], 0.0); put(c, &G.pv[0][o], 0.0); put(c, &G.pv[1][o], 0.0);
          put(c, &G.z[o], 0.0); put(c, &G.q[o], 0.0);
          sA[slot * kBlockDim + u] = v;
        } else {
          const double* H = G.Hpp + (size_t)p * 36 + row * 6;
          double pr = 0, v = 0;
#pragma unroll
          for (int cc = 0; cc < 6; cc++) {
            double pc = ldc(pvec + (size_t)p * 6 + cc);
            double h = ldc(H + cc);
            if (cc == row) { pr = pc; h *= (1 + lambda); }
            v += h * pc;
          }
          {
            // pose-pose blocks: the first two neighbours (the odometry chain) come resolved from the host-built
            // record and are loaded together, the rest loop over the incidence list
            const int4 nb = *reinterpret_cast<const int4*>(G.pnbr + (size_t)p * 8);
            const int2 nr = *reinterpret_cast<const int2*>(G.pnbr + (size_t)p * 8 + 4);
            const double* xo[2] = {pvec + (size_t)max(nb.y, 0) * 6, pvec + (size_t)max(nb.w, 0) * 6};
            double av[12], xv[2][6];
            const int nf = nbr_coeffs(nb, row, av);
#pragma unroll
            for (int n2 = 0; n2 < 2; n2++)
#pragma unroll
              for (int cc = 0; cc < 6; cc++) xv[n2][cc] = (n2 < nf) ? ldc(xo[n2] + cc) : 0.0;
#pragma unroll
            for (int n2 = 0; n2 < 2; n2++)
#pragma unroll
              for (int cc = 0; cc < 6; cc++) v += av[n2 * 6 + cc] * xv[n2][cc];
            v = pose_pose_tail(nr.x, nr.y, row, pvec, v);
          }
          v -= ysum;
          qout[o] = v;   // (q is only read back by the owner of the block: not mirrored)
          sA[slot * kBlockDim + u] = v;
          dot += pr * v;
        }
      }
      __syncthreads();
      if (live && (rhs || qc)) restrict_block(sA, slot, u, k, np, rhs ? G.rcpart[0] : qc);
      if (!rhs) lap(23);
    }
    return dot;
  }

  // -------- PCG: copy the owned dense blocks (upper triangles) into shared memory for the whole solve ----
  __device__ void cache_blocks() {
    double* cache = reinterpret_cast<double*>(g_smem + kSmCache);
    __syncthreads();
    for (int ci = 0; ci < kCacheBlocks; ci++) {
      // cached block ci of this CTA = owned block of (slot = ci % kSlots, round = ci / kSlots)
      int k = c.rank + c.tsize * ((ci % kSlots) + kSlots * (ci / kSlots));
      if (k >= G.nblk) continue;
      const double* B = G.Binv + (size_t)k * kPackedBlock;
      for (int idx = threadIdx.x; idx < kPackedBlock; idx += kThreads) cache[(size_t)ci * kPackedBlock + idx] = ldc(B + idx);
    }
    __syncthreads();
  }

  // -------- three-level preconditioner, coarse part: level-3 residual from the level-2 partials; level-3 rows (distributed
  // over the team, or applied by every CTA when the level is small); level-2 nodes: one warp per node = its 6 rows of the
  // group's 96 x 96 inverse.  Publishes zc2 (and zc when level 3 is distributed); returns the partial of r.z it owns.
  __device__ double coarse_three_level(double alpha, const double* rc_old, bool first) {
    double* src = reinterpret_cast<double*>(g_smem + kSmRc);   // level-3 residual [6 nc]
    double* z3s = reinterpret_cast<double*>(g_smem + kSmZc);   // level-3 solution when it is applied locally (<= kL3Local rows)
    const int tid = threadIdx.x, lane = tid & 31;
    const int ldm = 6 * G.nc, m = G.SP / kL2Spacing;
    // level-2 residual of node a: per-block partials of the previous iteration, updated linearly (r_new = r - alpha q)
    auto rc2 = [&](int a, int row) -> double {
      double v = 0.0;
      if (a < G.nblk) {
        v += ldc(rc_old + (size_t)a * 12 + row);
        if (!first) v -= alpha * ldc(G.qcpart + (size_t)a * 12 + row);
      }
      if (a >= 1) {
        v += ldc(rc_old + (size_t)(a - 1) * 12 + 6 + row);
        if (!first) v -= alpha * ldc(G.qcpart + (size_t)(a - 1) * 12 + 6 + row);
      }
      return v;
    };
    __syncthreads();
    // level-3 residual, one warp per level-3 node: lanes = the level-2 nodes in its support (all their partial loads in flight
    // together), fixed-order shuffle tree per row.  Small level 3: every CTA assembles all of it (no exchange).  Large graphs:
    // the nodes are distributed over the team (assembling all of it in every CTA costs 24 loads per level-2 node per CTA --
    // 75 k loads on 50 k poses), published, and read back behind one extra team barrier.
    {
      const int w0 = c.l3_local ? (tid >> 5) : warp_team(), wstep = c.l3_local ? kWarps : nwarp_team();
      for (int A = w0; A < G.nc; A += wstep) {
        const int alo = max(0, (A - 1) * m + 1), ahi = min(G.nc2, (A + 1) * m);
        double acc[6] = {0, 0, 0, 0, 0, 0};
        for (int a = alo + lane; a < ahi; a += 32) {
          int d = a - A * m;
          if (d < 0) d = -d;
          const double h = 1.0 - (double)d / (double)m;
          double v[6];
#pragma unroll
          for (int row = 0; row < 6; row++) v[row] = rc2(a, row);
#pragma unroll
          for (int row = 0; row < 6; row++) acc[row] += h * v[row];
        }
#pragma unroll
        for (int row = 0; row < 6; row++) acc[row] = warp_sum(acc[row]);
        if (lane < 6) {
          double v = acc[0];
#pragma unroll
          for (int row = 1; row < 6; row++) if (lane == row) v = acc[row];
          if (c.l3_local) src[A * 6 + lane] = v;
          else put(c, &G.rc3[A * 6 + lane], v);
        }
      }
    }
    if (!c.l3_local) {
      team_barrier(c);
      for (int i = tid; i < ldm; i += kThreads) src[i] = ldc(G.rc3 + i);
    }
    __syncthreads();
    lap(13);
    const float* Ai = G.Ac;
    double dot = 0.0;
    if (c.l3_local) {
      for (int i = tid >> 5; i < ldm; i += kWarps) {
        const double acc = coarse_row_dot<4>(Ai + ac_index(G.ldmc, i, 0), src, ldm, lane);
        if (lane == 0) {
          z3s[i] = acc;
          if (c.rank == 0) dot += src[i] * acc;
        }
      }
      __syncthreads();
    } else {
      const int nw = nwarp_team();
      for (int i = warp_team(); i < ldm; i += nw) {
        const double acc = coarse_row_dot<4>(Ai + ac_index(G.ldmc, i, 0), src, ldm, lane);
        if (lane == 0) { put(c, &G.zc[i], acc); dot += src[i] * acc; }
      }
    }
    const int nw2 = nwarp_team();
    for (int a = warp_team(); a < G.nc2; a += nw2) {
      const int g = a / kGroupNodes, a0 = g * kGroupNodes;
      double rg[3];
#pragma unroll
      for (int t = 0; t < 3; t++) {
        const int e = lane + 32 * t, an = a0 + e / 6, row = e % 6;
        rg[t] = (an < G.nc2) ? rc2(an, row) : 0.0;
      }
      const double* D = G.D2inv + (size_t)g * kBlockDim * kBlockDim + (size_t)((a - a0) * 6) * kBlockDim;
      for (int rr = 0; rr < 6; rr++) {
        double acc = ldc(D + rr * kBlockDim + lane) * rg[0] + ldc(D + rr * kBlockDim + lane + 32) * rg[1] + ldc(D + rr * kBlockDim + lane + 64) * rg[2];
        acc = warp_sum(acc);
        const int e = (a - a0) * 6 + rr;
        const double sel = (e < 32) ? rg[0] : (e < 64 ? rg[1] : rg[2]);
        const double rme = __shfl_sync(0xffffffffu, sel, e & 31);
        if (lane == 0) {
          double zv = acc;
          dot += rme * acc;
          if (c.l3_local) {
            const int p = a * kL2Spacing, c0 = p / G.SP;
            zv += hat(p, c0) * z3s[c0 * 6 + rr] + hat(p, c0 + 1) * z3s[min(c0 + 1, G.nc - 1) * 6 + rr];
          }
          put(c, &G.zc2[(size_t)a * 6 + rr], zv);
        }
      }
    }
    return dot;
  }

  // -------- PCG: x += alpha p ; r -= alpha q ; z = M^-1 r (dense block + coarse) ; returns partial r.z ----
  // rc_old / rc_new: ping-pong buffers of per-block coarse restrictions of r
  __device__ double precondition(double alpha, const double* pvec, const double* rc_old, double* rc_new,
                                 bool first) {
    double* sA = reinterpret_cast<double*>(g_smem + kSmA);   // r_new per slot
    double* src = reinterpret_cast<double*>(g_smem + kSmRc); // coarse residual, 6*nc
    const int tid = threadIdx.x, slot = tid / kBlockDim, u = tid % kBlockDim;
    const int ldm = 6 * G.nc;
    const int bpn = G.SP / kBlockPoses;  // blocks per coarse interval
    double dot = 0;
    if (G.levels == 3) {
      dot = coarse_three_level(alpha, rc_old, first);
    } else {
      // full coarse residual rc = sum_k rc_old[k] - alpha * sum_k qcpart[k]  (linear in r)
      __syncthreads();
      if (bpn == 1) coarse_residual(rc_old, alpha, first, src);
      else
      for (int i = tid; i < ldm; i += kThreads) {
        int node = i / 6, row = i % 6;
        // blocks with c0 == node feed `node` through their slot 0, blocks with c0 == node-1 through slot 1;
        // issue all loads before the (fixed-order) sums
        double va[2][8], vq[2][8];
  #pragma unroll
        for (int side = 0; side < 2; side++) {
          int cint = node - side;
          int k0 = cint * bpn;
  #pragma unroll
          for (int t = 0; t < 8; t++) {
            int k = k0 + t;
            bool ok = (cint >= 0) && (t < bpn) && (k < G.nblk);
            va[side][t] = ok ? ldc(rc_old + (size_t)k * 12 + side * 6 + row) : 0.0;
            vq[side][t] = (ok && !first) ? ldc(G.qcpart + (size_t)k * 12 + side * 6 + row) : 0.0;
          }
        }
        double acc = 0;
  #pragma unroll
        for (int side = 0; side < 2; side++)
  #pragma unroll
          for (int t = 0; t < 8; t++) acc += va[side][t] - alpha * vq[side][t];
        if (bpn > 8) {  // (spacing > 128 poses: rare large graphs) remaining blocks, plain loop
          if (G.prm.mode == MODE_DEBUG && i == 0) atomicOr(&G.res->status, (int)kPathCoarseTail);
          for (int side = 0; side < 2; side++) {
            int cint = node - side;
            if (cint < 0) continue;
            int k0 = cint * bpn + 8, k1 = min(G.nblk, cint * bpn + bpn);
            for (int k = k0; k < k1; k++) {
              double v = ldc(rc_old + (size_t)k * 12 + side * 6 + row);
              if (!first) v -= alpha * ldc(G.qcpart + (size_t)k * 12 + side * 6 + row);
              acc += v;
            }
          }
        }
        src[i] = acc;
      }
      __syncthreads();
      lap(13);
      const float* Ai = G.Ac;
      // coarse part, distributed over the team: one warp per row of A_c^-1.  z is never formed with its coarse
      // part; r.z = r.z_local + rc.zc (rc = P^T r), and the consumers of z add P*zc on the fly.
      {
        const int lane = tid & 31;
        const int nw = nwarp_team();
        for (int i = warp_team(); i < ldm; i += nw) {
          const double acc = coarse_row_dot<8>(Ai + ac_index(G.ldmc, i, 0), src, ldm, lane);
          if (lane == 0) { put(c, &G.zc[i], acc); dot += src[i] * acc; }
        }
      }
    }
    lap(14);
    const int nrd = rounds();
    const int sr_off = kSmRc + ((ldm * 8 + 127) / 128) * 128;   // staged residuals of all rounds, after the coarse residual
    if (c.use_tma && sr_off + nrd * kSlots * kBlockDim * 8 <= kSmTma) {
      // Large graphs: (A) update x, r of every owned pose and keep the new residuals of all rounds in shared memory
      // (loads of three rounds in flight together), then (B) stream the owned dense blocks Binv[k] through the
      // two 72 KB staging buffers with one bulk async copy each (the next block in flight while this one is applied).
      double* sR = reinterpret_cast<double*>(g_smem + sr_off);
      if (G.prm.mode == MODE_DEBUG && tid == 0) atomicOr(&G.res->status, (int)kPathTmaRing);
      __syncthreads();
      for (int rd0 = 0; rd0 < nrd; rd0 += 3) {
        double vr[3], vp[3], vq[3], vx[3];
#pragma unroll
        for (int t = 0; t < 3; t++) {
          const int rd = rd0 + t, k = c.rank + c.tsize * (slot + kSlots * rd), p = k * kBlockPoses + u / 6;
          const bool on = (rd < nrd) && (slot < kSlots) && (k < G.nblk) && (p < G.N);
          const size_t o = (size_t)p * 6 + u % 6;
          vr[t] = on ? ldc(G.r + o) : 0.0;
          vp[t] = (on && !first) ? ldc(pvec + o) : 0.0;
          vq[t] = (on && !first) ? ldc(G.q + o) : 0.0;
          vx[t] = (on && !first) ? ldc(G.x + o) : 0.0;
        }
#pragma unroll
        for (int t = 0; t < 3; t++) {
          const int rd = rd0 + t, k = c.rank + c.tsize * (slot + kSlots * rd), p = k * kBlockPoses + u / 6;
          if (rd >= nrd || slot >= kSlots) continue;
          const bool on = (k < G.nblk) && (p < G.N);
          double rn = vr[t];
          if (on && !first) {
            const size_t o = (size_t)p * 6 + u % 6;
            rn -= alpha * vq[t];
            G.x[o] = vx[t] + alpha * vp[t];   // x, r: owner-only during the iteration (x is published once at the end)
            G.r[o] = rn;
          }
          sR[(rd * kSlots + slot) * kBlockDim + u] = on ? rn : 0.0;
        }
      }
      __syncthreads();
      unsigned long long* gbar = reinterpret_cast<unsigned long long*>(g_smem + kSmGjBar);
      double* bbuf = reinterpret_cast<double*>(g_smem + kSmTma);
      constexpr unsigned kBlockBytes = kPackedBlock * 8;   // packed upper triangle: 37 248 bytes, one bulk copy
      static_assert(kBlockBytes % 16 == 0 && 2 * kBlockBytes <= kSmTmaEnd - kSmTma, "two packed blocks must fit the staging area");
      const int nown = (G.nblk - c.rank + c.tsize - 1) / c.tsize;   // owned blocks: k = rank + tsize * ib
      // three-stage ring of 37 KB packed blocks: two bulk copies in flight while one block is applied
      static_assert(3 * kBlockBytes <= kSmTmaEnd - kSmTma, "three packed blocks must fit the staging area");
      if (tid == 0)
        for (int pre = 0; pre < 2 && pre < nown; pre++)
          tma_load_1d(bbuf + pre * kPackedBlock, G.Binv + (size_t)(c.rank + c.tsize * pre) * kPackedBlock, kBlockBytes, gbar + pre);
      for (int ib = 0; ib < nown; ib++) {
        const int k = c.rank + c.tsize * ib;
        const int stg = ib % 3;
        if (tid == 0 && ib + 2 < nown)
          tma_load_1d(bbuf + ((ib + 2) % 3) * kPackedBlock, G.Binv + (size_t)(k + 2 * c.tsize) * kPackedBlock, kBlockBytes, gbar + (ib + 2) % 3);
        const double* rv = sR + (size_t)ib * kBlockDim;   // (ib = slot + kSlots * rd: the staging order of part A)
        const int np = min(kBlockPoses, G.N - k * kBlockPoses);
        mbar_wait(gbar + stg, (c.gj_par >> stg) & 1u);
        c.gj_par ^= (1u << stg);
        if (tid < 4 * kBlockDim) {
          // four threads per row of the symmetric block (interleaved columns, fixed-order combination by two shuffles):
          // column part j < u reads element (j, u), row part j >= u reads element (u, j) of the packed upper triangle
          const int u = tid >> 2, qq = tid & 3;
          const double* cb = bbuf + stg * kPackedBlock;
          double zl = 0;
          for (int j = qq; j < u; j += 4) zl += packed_row(cb, j)[u] * rv[j];
          const double* cu = packed_row(cb, u);
          for (int j = u + ((qq - u) & 3); j < kBlockDim; j += 4) zl += cu[j] * rv[j];
          zl += __shfl_xor_sync(0xffffffffu, zl, 1);
          zl += __shfl_xor_sync(0xffffffffu, zl, 2);
          const int p = k * kBlockPoses + u / 6;
          if (qq == 0 && p < G.N) {
            G.z[(size_t)p * 6 + u % 6] = zl;   // large graphs: only the owner reads z (update_direction)
            dot += rv[u] * zl;
          }
        } else if (tid >= 4 * kBlockDim && tid < 4 * kBlockDim + 12) {
          restrict_block(rv, 0, tid - 4 * kBlockDim, k, np, rc_new);
        }
        __syncthreads();   // the buffer may be refilled
      }
      lap(15);
      return dot;
    }
    for (int rd = 0; rd < nrd; rd++) {
      int k = c.rank + c.tsize * (slot + kSlots * rd);
      int p = k * kBlockPoses + u / 6, row = u % 6;
      bool live = (slot < kSlots) && (k < G.nblk);
      int np = live ? min(kBlockPoses, G.N - k * kBlockPoses) : 0;
      bool on = live && (p < G.N);
      __syncthreads();
      double rn = 0;
      if (slot < kSlots) sA[slot * kBlockDim + u] = 0.0;
      if (on) {
        size_t o = (size_t)p * 6 + row;
        rn = ldc(G.r + o);
        if (!first) {
          double pp = ldc(pvec + o), qq = ldc(G.q + o), xx = ldc(G.x + o);
          rn -= alpha * qq;
          G.x[o] = xx + alpha * pp;
          G.r[o] = rn;
        }
        sA[slot * kBlockDim + u] = rn;
      }
      __syncthreads();
      if (live) restrict_block(sA, slot, u, k, np, rc_new);
      if (on) {
        // dense block: z_local = Binv[k] r_block (symmetric: read column u)
        const int ci = slot + kSlots * rd;
        const double* rv = sA + slot * kBlockDim;
        const bool cached = ci < kCacheBlocks && c.smem_cache_ok;
        const double zl = cached
                              ? packed_row_dot<LdS>(reinterpret_cast<const double*>(g_smem + kSmCache) + (size_t)ci * kPackedBlock, u, rv)
                              : packed_row_dot<LdL2>(G.Binv + (size_t)k * kPackedBlock, u, rv);   // straight from L2
        put(c, &G.z[(size_t)p * 6 + row], zl);
        dot += rn * zl;
        if (G.prm.mode == MODE_DEBUG && u == 0) atomicOr(&G.res->status, (int)(cached ? kPathApplySmem : kPathApplyL2));
      }
    }
    lap(15);
    return dot;
  }


  // -------- block-resident PCG loop (graphs whose owned blocks fit one CTA's shared memory; single-GPU, two levels) --------
  // Same recurrence, operator and preconditioner as the loop in schur_solve(), reorganised so that an iteration touches L2
  // only for what CTAs really exchange:
  //   A  p = z + P zc + beta p (registers / smem) ; W^T p of the OWN pose-major tiles from the smem copy of W ; fixed-order sums
  //      per (block, plane) group -> upartb ; p published for pose-pose neighbours in other blocks            -> team barrier
  //   B  v_g = Hll^-1 * (sum of the plane's per-block partials) ; y = W v from smem ; q = (Hpp + lambda D) p + pose-pose - y ;
  //      P^T q -> qcpart ; p.q                                                                                 -> team reduction
  //   C  coarse residual (linear update) ; A_c^-1 rows -> zc ; x, r updated in registers ; z = Binv r from smem ; r.z -> reduction
  // r, x, z, p, q of a row live in the registers of its thread for the whole solve.  Entry state (from the common prologue):
  // G.r, G.x, G.z (local part), G.zc, rcpart[rcb] ; exit: G.x.  Returns the iteration count.
  // Both loops call the same helpers for the arithmetic they share: tile_wt_x and seg_suffix_sum
  // (A, as in sweep_planes), plane_vec_small, warp_sum_partials, mat3_vec / dot3, tile_w_v, nbr_coeffs and pose_pose_tail (B, as in
  // solve_heavy and pose_phase), coarse_residual and coarse_row_dot (C, as in precondition).  The dense-block apply is its own: it
  // reads the folded copy below instead of the packed triangle, with two accumulators.
  __device__ int pcg_resident(double lambda, int rcb, const double rz0, double rz, const double tol2, Timer& tmr) {
    const int ldm = 6 * G.nc;
    const int nown_max = (G.nblk + c.tsize - 1) / c.tsize;
    const ResLay L = res_layout(G.res_nt, G.res_ng, G.res_np, ldm, nown_max);
    const int tid = threadIdx.x, slot = tid / kBlockDim, u = tid % kBlockDim, lane = tid & 31, warp = tid >> 5, wis = u >> 5;
    const int nown = (G.nblk - c.rank + c.tsize - 1) / c.tsize;   // owned blocks k = rank + tsize * slot
    int* hdr = reinterpret_cast<int*>(g_smem + L.hdr);            // [0..7] tiles per slot, [8..15] groups per slot
    double* sP = reinterpret_cast<double*>(g_smem + L.sP);
    double* sR = reinterpret_cast<double*>(g_smem + L.sR);
    double* src = reinterpret_cast<double*>(g_smem + L.src);
    __syncthreads();
    // ---- static per-solve caches ----
    for (int s = 0; s < nown; s++) {
      const int kb = c.rank + c.tsize * s;
      unsigned char* sb = g_smem + L.slot0 + s * L.stride;
      const int t0 = G.tile_ptr[kb], nt = G.tile_ptr[kb + 1] - t0, e0 = t0 * 32;
      const int g0 = G.blk_grp_ptr[kb], ng = G.blk_grp_ptr[kb + 1] - g0, part0 = G.blk_part_ptr[kb];
      if (tid == 0) { hdr[s] = nt; hdr[8 + s] = ng; }
      int* ei = reinterpret_cast<int*>(sb + L.o_ei);
      for (int e = tid; e < nt * 32; e += kThreads) {
        const int pp = G.pp_pose[e0 + e];
        ei[e] = pp < 0 ? 31 : ((pp - kb * kBlockPoses) | (G.grp_of_slot[e0 + e] << 5) | ((G.pm_part[e0 + e] - part0) << 14));
      }
      int4* gi = reinterpret_cast<int4*>(sb + L.o_gi);
      int2* gm = reinterpret_cast<int2*>(sb + L.o_gm);
      unsigned short* mem = reinterpret_cast<unsigned short*>(sb + L.o_mem);
      const int mb = G.grp_mem_ptr[g0];
      for (int g = tid; g < ng; g += kThreads) {
        gi[g] = *reinterpret_cast<const int4*>(G.grp_info2 + (size_t)(g0 + g) * 4);
        const int m0 = G.grp_mem_ptr[g0 + g], m1 = G.grp_mem_ptr[g0 + g + 1];
        gm[g] = make_int2(m0 - mb, m1 - m0);
      }
      const int nm = G.grp_mem_ptr[g0 + ng] - mb;
      for (int m = tid; m < nm; m += kThreads) mem[m] = (unsigned short)(G.grp_mem[mb + m] - e0);
      double* Wc = reinterpret_cast<double*>(sb + L.o_W);
      const double* Wg = G.W + (size_t)t0 * kWStride;
      for (int i = tid; i < nt * kWStride; i += kThreads) Wc[i] = ldc(Wg + i);
      // the packed upper triangle of the symmetric block, folded into a 48 x 97 rectangle: row a < 48 keeps its entries (a, b) at
      // [a][b]; row a >= 48 (96 - a entries) fills the unused left part of row 95 - a ([d] for d = b - a < 95 - a, the last one at
      // [96]).  Same 4656 doubles, but every row is reached with a constant odd stride: the mat-vec below is a plain thread-per-row
      // loop without bank conflicts, shuffles or index arithmetic.
      double* Bc = reinterpret_cast<double*>(sb + L.o_B);
      const double* Bg = G.Binv + (size_t)kb * kPackedBlock;
      for (int i = tid; i < kBlockDim * kBlockDim; i += kThreads) {
        const int ra = i / kBlockDim, cb2 = i - ra * kBlockDim;
        if (cb2 < ra) continue;
        const double v = ldc(packed_row(Bg, ra) + cb2);
        const int fi = kBlockDim - 1 - ra, d = cb2 - ra;
        Bc[ra < kBlockDim / 2 ? ra * 97 + cb2 : fi * 97 + (d < fi ? d : 96)] = v;
      }
    }
    // ---- per-thread state: row `row` of pose p in owned block k ----
    const bool live = slot < nown;
    const int k = c.rank + c.tsize * (live ? slot : 0);
    const int p = k * kBlockPoses + u / 6, row = u % 6;
    const bool on = live && p < G.N;
    const int np = live ? min(kBlockPoses, G.N - k * kBlockPoses) : 0;
    const size_t o = (size_t)p * 6 + row;
    unsigned char* sb = g_smem + L.slot0 + (live ? slot : 0) * L.stride;
    double* sE = reinterpret_cast<double*>(sb);                    // phase A: per-edge W_e^T p  [tiles * 32][3]
    double* vg = reinterpret_cast<double*>(sb);                    // phase B: plane-group vectors [ng][3] ...
    double* yp = reinterpret_cast<double*>(sb + r16(G.res_ng * 24));   // ... and (tile, pose)-run sums [np][6]
    const int4* gi = reinterpret_cast<const int4*>(sb + L.o_gi);
    const int2* gm = reinterpret_cast<const int2*>(sb + L.o_gm);
    const unsigned short* mem = reinterpret_cast<const unsigned short*>(sb + L.o_mem);
    const double* Bc = reinterpret_cast<const double*>(sb + L.o_B);
    double r_u = 0, x_u = 0, z_u = 0, p_u = 0, q_u = 0;
    int yp0 = 0, ypn = 0;
    int4 nb = make_int4(-1, -1, -1, -1);
    int2 nr = make_int2(0, 0);
    if (on) {
      r_u = ldc(G.r + o); x_u = ldc(G.x + o); z_u = ldc(G.z + o);
      yp0 = G.ypart_ptr[p] - G.blk_part_ptr[k];
      ypn = G.ypart_ptr[p + 1] - G.ypart_ptr[p];
      nb = *reinterpret_cast<const int4*>(G.pnbr + (size_t)p * 8);
      nr = *reinterpret_cast<const int2*>(G.pnbr + (size_t)p * 8 + 4);
    }
    // row `row` of pose p of the pose part of the operator, static for this solve: (Hpp + lambda D) row and the rows of the
    // pose-pose blocks towards the first two neighbours (the odometry chain).  Kept per thread for the whole loop (registers or,
    // spilled, lane-interleaved local memory = coalesced) instead of 18 scattered 8-byte loads per iteration.
    double trow[18];
#pragma unroll
    for (int t = 0; t < 18; t++) trow[t] = 0.0;
    const int nf = (nb.x >= 0) + (nb.z >= 0);
    const int oth0 = max(nb.y, 0), oth1 = max(nb.w, 0);
    if (on) {
      const double* H = G.Hpp + (size_t)p * 36 + row * 6;
#pragma unroll
      for (int cc = 0; cc < 6; cc++) trow[cc] = ldc(H + cc) * (cc == row ? (1 + lambda) : 1.0);
      nbr_coeffs(nb, row, trow + 6);
    }
    __syncthreads();
    // planes seen from more than 8 pose blocks (the ground plane from all): summed once per CTA by all its warps instead of
    // once per owned block -- a list of the distinct ones among this CTA's groups; a listed group carries -(index + 1) as its
    // partial count.  (More than kResHeavy distinct ones: the rest keep the per-block warp loop.)
    int* hvl = reinterpret_cast<int*>(g_smem + L.hdr + 64);   // [kResHeavy][4] = {plane, first partial, count, -}
    if (tid == 0) {
      int nh = 0, unlisted = 0;
      for (int s = 0; s < nown; s++) {
        int4* gs = reinterpret_cast<int4*>(g_smem + L.slot0 + s * L.stride + L.o_gi);
        for (int g = 0; g < hdr[8 + s]; g++) {
          const int4 q = gs[g];
          if (q.z <= 8) continue;
          int h = 0;
          while (h < nh && hvl[h * 4] != q.x) h++;
          if (h == nh) {
            if (nh == kResHeavy) { unlisted = 1; continue; }
            hvl[h * 4] = q.x; hvl[h * 4 + 1] = q.y; hvl[h * 4 + 2] = q.z;
            nh++;
          }
          gs[g].z = -(h + 1);
        }
      }
      hdr[7] = nh;
      if (G.prm.mode == MODE_DEBUG) atomicOr(&G.res->status, (nh ? (int)kPathResListed : 0) | (unlisted ? (int)kPathResUnlisted : 0));
    }
    if (G.prm.mode == MODE_DEBUG) {
      if (on && nr.y > nr.x) atomicOr(&G.res->status, (int)kPathResTail);
      if (live && u == 0 && hdr[8 + slot] > kBlockDim) atomicOr(&G.res->status, (int)kPathResWide);
    }
    __syncthreads();
    const int ng = live ? hdr[8 + slot] : 0;
    const int nh = hdr[7];
    int wpe = kWarps;   // warps per listed plane (power of two)
    while (wpe > 1 && wpe * nh > kWarps) wpe >>= 1;
    double* hvp = reinterpret_cast<double*>(g_smem + L.hdr + 64 + kResHeavy * 16);   // [kResHeavy][kWarps][3] partial sums
    const float* Ai = G.Ac;
    double* pvec = G.pv[0];
    int it = 0;
    double beta = 0.0;
    while (it < G.prm.pcg_max_iter) {
      tmr.sync();
      // ================= A =================
      if (on) {
        const int d = p - k * kBlockPoses;
        const double h1 = (double)d * (1.0 / kBlockPoses);
        const double cz = (1.0 - h1) * ldc(G.zc + (size_t)k * 6 + row) + h1 * ldc(G.zc + (size_t)min(k + 1, G.nc - 1) * 6 + row);
        p_u = (z_u + cz) + beta * p_u;
        pvec[o] = p_u;
      }
      if (live) sP[slot * kBlockDim + u] = on ? p_u : 0.0;
      __syncthreads();
      {
        int cnt = 0;
        for (int s = 0; s < nown; s++) {
          const int nts = hdr[s];
          for (int t = 0; t < nts; t++, cnt++) {
            if ((cnt & (kWarps - 1)) != warp) continue;
            unsigned char* sbs = g_smem + L.slot0 + s * L.stride;
            const int info = reinterpret_cast<const int*>(sbs + L.o_ei)[t * 32 + lane];
            const int pe = info & 31;
            double uu[3] = {0, 0, 0};
            if (pe != 31)
              tile_wt_x<LdS>(reinterpret_cast<const double*>(sbs + L.o_W) + t * kWStride + lane, sP + s * kBlockDim + pe * 6, uu);
            double* se = reinterpret_cast<double*>(sbs) + (size_t)(t * 32 + lane) * 3;
            se[0] = uu[0]; se[1] = uu[1]; se[2] = uu[2];
          }
        }
      }
      __syncthreads();
      if (live) {
        for (int g = u; g < ng; g += kBlockDim) {
          const int2 m = gm[g];
          double s0 = 0, s1 = 0, s2 = 0;
          for (int i = 0; i < m.y; i += 4) {   // (four members per round: their loads are independent; fixed summation order)
            double e4[4][3];
#pragma unroll
            for (int q = 0; q < 4; q++) {
              const double* se = sE + (size_t)mem[m.x + min(i + q, m.y - 1)] * 3;
              const bool ok = i + q < m.y;
              e4[q][0] = ok ? se[0] : 0.0; e4[q][1] = ok ? se[1] : 0.0; e4[q][2] = ok ? se[2] : 0.0;
            }
#pragma unroll
            for (int q = 0; q < 4; q++) { s0 += e4[q][0]; s1 += e4[q][1]; s2 += e4[q][2]; }
          }
          double* uo = G.upartb + (size_t)gi[g].w * 3;
          uo[0] = s0; uo[1] = s1; uo[2] = s2;
        }
      }
      team_barrier_light(c);
      tmr.lap(16);
      // ================= B =================
      if (live) {
        for (int g = u; g < ng; g += kBlockDim) {
          const int4 gq = gi[g];
          if (gq.z >= 0 && gq.z <= 8) plane_vec_small(G.upartb, gq.y, gq.z, gq.x, vg + g * 3);
        }
        for (int g = wis; g < ng; g += 3) {   // unlisted planes seen from more than 8 pose blocks: a warp of the block sums the partials
          const int4 gq = gi[g];
          const int l = gq.x, t0 = gq.y, n = gq.z;
          if (n <= 8) continue;
          double uu[3];
          warp_sum_partials(G.upartb, t0, t0 + n, lane, uu);
          if (lane < 3) vg[g * 3 + lane] = dot3<LdL2>(G.Hinv + (size_t)l * 9 + lane * 3, uu);
        }
      }
      // listed heavy planes: `wpe` warps each, every warp one contiguous chunk of the plane's per-block partials
      double hHi[9];
      int hidx = -1, hg = -1;
      if (live)
        for (int g = u; g < ng; g += kBlockDim)
          if (gi[g].z < 0) {   // (at most one listed group per thread: ng <= 96 here, else the tail loop below)
            hg = g; hidx = -gi[g].z - 1;
#pragma unroll
            for (int t = 0; t < 9; t++) hHi[t] = ldc(G.Hinv + (size_t)gi[g].x * 9 + t);
            break;
          }
      if (warp < nh * wpe) {
        const int h = warp / wpe, j = warp - h * wpe;
        const int t0 = hvl[h * 4 + 1], n = hvl[h * 4 + 2];
        const int per = (n + wpe - 1) / wpe, a0 = t0 + j * per, a1 = min(t0 + n, a0 + per);
        double uu[3];
        warp_sum_partials(G.upartb, a0, a1, lane, uu);
        if (lane < 3) hvp[(h * kWarps + j) * 3 + lane] = (lane == 0) ? uu[0] : (lane == 1 ? uu[1] : uu[2]);
      }
      if (nh) {
        __syncthreads();
        if (hidx >= 0) {
          double uu[3] = {0, 0, 0};
          for (int j = 0; j < wpe; j++)
            for (int b = 0; b < 3; b++) uu[b] += hvp[(hidx * kWarps + j) * 3 + b];
          mat3_vec(hHi, uu, vg + hg * 3);
          for (int g = hg + kBlockDim; g < ng; g += kBlockDim)   // (blocks with more than 96 groups: further listed groups of this thread)
            if (gi[g].z < 0) {
              const int hi2 = -gi[g].z - 1, l2 = gi[g].x;
              double u2[3] = {0, 0, 0};
              for (int j = 0; j < wpe; j++)
                for (int b = 0; b < 3; b++) u2[b] += hvp[(hi2 * kWarps + j) * 3 + b];
              for (int b = 0; b < 3; b++) vg[g * 3 + b] = dot3<LdL2>(G.Hinv + (size_t)l2 * 9 + b * 3, u2);
            }
        }
      }
      __syncthreads();
      lap(21);
      {
        int cnt = 0;
        for (int s = 0; s < nown; s++) {
          const int nts = hdr[s];
          for (int t = 0; t < nts; t++, cnt++) {
            if ((cnt & (kWarps - 1)) != warp) continue;
            unsigned char* sbs = g_smem + L.slot0 + s * L.stride;
            const int info = reinterpret_cast<const int*>(sbs + L.o_ei)[t * 32 + lane];
            const int pe = info & 31, key = (pe == 31) ? -1 : pe;
            double y[6] = {0, 0, 0, 0, 0, 0};
            if (key >= 0) {
              const double* vv = reinterpret_cast<const double*>(sbs) + ((info >> 5) & 511) * 3;
              tile_w_v<LdS>(reinterpret_cast<const double*>(sbs + L.o_W) + t * kWStride + lane, vv[0], vv[1], vv[2], y);
            }
            if (seg_suffix_sum<6>(key, y)) {
              double* yo = reinterpret_cast<double*>(sbs + r16(G.res_ng * 24)) + (size_t)(info >> 14) * 6;
#pragma unroll
              for (int a = 0; a < 6; a++) yo[a] = y[a];
            }
          }
        }
      }
      __syncthreads();
      lap(17);
      double dot = 0;
      if (on) {
        double ysum = 0;
        for (int t = 0; t < ypn; t++) ysum += yp[(size_t)(yp0 + t) * 6 + row];
        double vv = 0;
        {
          double va = 0, vb = 0;   // (three independent chains)
          const double* po = sP + slot * kBlockDim + (u / 6) * 6;
#pragma unroll
          for (int cc = 0; cc < 6; cc++) vv += trow[cc] * po[cc];
          if (nf > 0) {
            const bool here = (oth0 / kBlockPoses) == k;
#pragma unroll
            for (int cc = 0; cc < 6; cc++)
              va += trow[6 + cc] * (here ? sP[slot * kBlockDim + (oth0 - k * kBlockPoses) * 6 + cc] : ldc(pvec + (size_t)oth0 * 6 + cc));
          }
          if (nf > 1) {
            const bool here = (oth1 / kBlockPoses) == k;
#pragma unroll
            for (int cc = 0; cc < 6; cc++)
              vb += trow[12 + cc] * (here ? sP[slot * kBlockDim + (oth1 - k * kBlockPoses) * 6 + cc] : ldc(pvec + (size_t)oth1 * 6 + cc));
          }
          vv += va + vb;
          vv = pose_pose_tail(nr.x, nr.y, row, pvec, vv);   // further pose-pose factors of this pose (loop closures)
        }
        q_u = vv - ysum;
        dot = p_u * q_u;
      }
      if (live) sR[slot * kBlockDim + u] = on ? q_u : 0.0;
      __syncthreads();
      if (live) restrict_block(sR, slot, u, k, np, G.qcpart);
      lap(18);
      const double pq = team_reduce_flag(c, dot);
      tmr.lap(19);
      if (!(pq > 0.0)) break;
      const double alpha = rz / pq;
      // ================= C =================
      const double* rc_old = G.rcpart[rcb];
      double* rc_new = G.rcpart[rcb ^ 1];
      coarse_residual(rc_old, alpha, false, src);
      if (on) { x_u += alpha * p_u; r_u -= alpha * q_u; }
      if (live) sR[slot * kBlockDim + u] = on ? r_u : 0.0;
      __syncthreads();
      lap(13);
      if (live) restrict_block(sR, slot, u, k, np, rc_new);
      dot = 0;
      {
        // rows of A_c^-1, one per warp: when the CTAs that own one pose block fewer than the others have enough warps for all
        // the rows, only they take rows (warp-major interleave), so the CTAs with the extra block are not the last to arrive
        const int n3 = G.nblk % c.tsize, ne = c.tsize - n3;
        const bool bal = n3 > 0 && ne * kWarps >= ldm;
        const int nw = bal ? ne * kWarps : nwarp_team();
        const int w0 = bal ? (c.rank >= n3 ? warp * ne + (c.rank - n3) : ldm) : warp_team();
        for (int i = w0; i < ldm; i += nw) {
          const double acc = coarse_row_dot<16>(Ai + ac_index(G.ldmc, i, 0), src, ldm, lane);
          if (lane == 0) { G.zc[i] = acc; dot += src[i] * acc; }
        }
      }
      lap(14);
      {
        // z = Binv r of every owned block from the folded copy: four warps per block (rows 0-31, 32-47, 48-79, 80-95, so that
        // a warp is on one side of the fold), a lane per row, two accumulators; consecutive lanes read consecutive or
        // odd-strided words in every segment of the row.
        double* sZ = sE;   // [96] per slot (scratch, free in phase C)
        for (int task = warp; task < 4 * nown; task += kWarps) {
          const int s = task >> 2, part = task & 3;
          const int uu = (part == 0 ? 0 : part == 1 ? 32 : part == 2 ? 48 : 80) + lane;
          const bool act = (part & 1) ? lane < 16 : true;
          unsigned char* sbs = g_smem + L.slot0 + s * L.stride;
          const double* F = reinterpret_cast<const double*>(sbs + L.o_B);
          const double* rv = sR + s * kBlockDim;
          double a0 = 0, a1 = 0;
          if (act) {
            if (part < 2) {            // uu < 48: (j, uu) at [j][uu] for j < uu, (uu, j) at [uu][j] for j >= uu
              const double* col = F + uu;
              int j = 0;
              for (; j + 1 < uu; j += 2) { a0 += col[j * 97] * rv[j]; a1 += col[(j + 1) * 97] * rv[j + 1]; }
              if (j < uu) a0 += col[j * 97] * rv[j];
              const double* rowp = F + uu * 97;
              j = uu;
              for (; j + 1 < kBlockDim; j += 2) { a0 += rowp[j] * rv[j]; a1 += rowp[j + 1] * rv[j + 1]; }
              if (j < kBlockDim) a0 += rowp[j] * rv[j];
            } else {                   // uu >= 48
              const double* col = F + uu;
#pragma unroll 4
              for (int j = 0; j < 48; j += 2) { a0 += col[j * 97] * rv[j]; a1 += col[(j + 1) * 97] * rv[j + 1]; }
              // 48 <= j < uu: (j, uu) lives in row 95 - j at [uu - j] (or [96] when uu == 95)
              const int last = (uu == kBlockDim - 1) ? 1 : 0;
              for (int j = 48; j < uu; j++) a0 += F[(kBlockDim - 1 - j) * 97 + (last ? 96 : uu - j)] * rv[j];
              // j >= uu: (uu, j) lives in row fi = 95 - uu at [j - uu], the last one (j = 95) at [96]
              const double* rowp = F + (kBlockDim - 1 - uu) * 97 - uu;
              for (int j = uu; j < kBlockDim - 1; j++) a1 += rowp[j] * rv[j];
              a1 += F[(kBlockDim - 1 - uu) * 97 + 96] * rv[kBlockDim - 1];
            }
            reinterpret_cast<double*>(sbs)[uu] = a0 + a1;
          }
        }
        lap1(22);
        __syncthreads();
        lap1(23);
        if (on) { z_u = sZ[u]; dot += r_u * z_u; }
      }
      lap(15);
      const double rz_new = team_reduce_flag(c, dot);
      tmr.lap(20);
      rcb ^= 1;
      it++;
      if (!(rz_new > tol2 * rz0)) break;
      beta = rz_new / rz;
      rz = rz_new;
    }
    if (on) {
      G.x[o] = x_u;
      if (G.prm.mode == MODE_DEBUG) { G.r[o] = r_u; G.z[o] = z_u; G.q[o] = q_u; }   // the exit state, as the general loop leaves it
    }
    team_barrier(c);
    return it;
  }

  // -------- spanning solves: the owners publish the final x to every rank (during the iteration x is owner-only) ----
  __device__ void publish_x() {
    if (!c.mirror) return;
    const int tid = threadIdx.x, slot = tid / kBlockDim, u = tid % kBlockDim;
    for (int rd = 0; rd < rounds(); rd++) {
      const int k = c.rank + c.tsize * (slot + kSlots * rd), p = k * kBlockPoses + u / 6;
      if (slot < kSlots && k < G.nblk && p < G.N) {
        const size_t o = (size_t)p * 6 + u % 6;
        put(c, &G.x[o], ldc(G.x + o));
      }
    }
  }

  // -------- |x|^2 over owned poses --------
  __device__ double norm_x() {
    double acc = 0;
    for (int i = tid_team(); i < G.N * 6; i += nthr_team()) { double v = ldc(G.x + i); acc += v * v; put(c, &G.xprev[i], v); }
    return acc;
  }

  // -------- trial = lin (+) delta --------
  __device__ void apply_delta() {
    for (int p = tid_team(); p < G.N; p += nthr_team()) {
      double v[7], d[6], o[7];
      for (int i = 0; i < 7; i++) v[i] = ldc(G.pose_lin + (size_t)p * 7 + i);
      for (int i = 0; i < 6; i++) d[i] = ldc(G.x + (size_t)p * 6 + i);
      pose_exmap(v, d, o);
      for (int i = 0; i < 7; i++) G.pose_trial[(size_t)p * 7 + i] = o[i];
    }
    for (int l = tid_team(); l < G.M; l += nthr_team()) {
      double v[4], d[3], o[4];
      for (int i = 0; i < 4; i++) v[i] = ldc(G.plane_lin + (size_t)l * 4 + i);
      for (int i = 0; i < 3; i++) d[i] = ldc(G.dl + (size_t)l * 3 + i);
      plane_exmap(v, d, o);
      for (int i = 0; i < 4; i++) G.plane_trial[(size_t)l * 4 + i] = o[i];
    }
  }
  __device__ void accept_trial() {
    for (int i = tid_team(); i < G.N * 7; i += nthr_team()) G.pose_lin[i] = ldc(G.pose_trial + i);
    for (int i = tid_team(); i < G.M * 4; i += nthr_team()) G.plane_lin[i] = ldc(G.plane_trial + i);
  }

#ifdef PUS_DIRECT
  // ================= exact direct solve (DESIGN.md section 5): dense Cholesky of the reduced pose system =================
  // Every sum below has one order that does not depend on the team: each output entry is written by one thread, and the
  // tile products of the factorization read the same operands whichever CTA computes them.  No atomics.
  __device__ __forceinline__ static int dtile(int i, int j) { return ldc(G.dtoff + i) + j - ldc(G.dfirst + i); }
  __device__ __forceinline__ static int dpair(int a, int b) { return ldc(G.dpoff + a) + b - 8 * ldc(G.dfirst + a / 8); }
  template <typename T>
  __device__ __forceinline__ static T* tile_at(T* base, int t) { return base + (size_t)t * kAcTile; }
  __device__ __forceinline__ static const int* nd(int k) { return G.dnd + ldc(G.dnd + k); }   // table k of the ND layout

  // W_al = sum of the (pose a, plane l) edges' W blocks in slot order, Y_al = W_al Hll_d^-1
  __device__ void direct_wy() {
    for (int q = tid_team(); q < G.dninc; q += nthr_team()) {
      const int l = G.dinc_plane[q];
      double w[18];
      for (int k = 0; k < 18; k++) w[k] = 0.0;
      for (int s = G.dinc_lo[q]; s < G.dinc_hi[q]; s++)
        for (int k = 0; k < 18; k++) w[k] += ldc(G.Wt + (size_t)(s >> 5) * kWStride + k * 32 + (s & 31));
      double Hi[9];
      for (int t = 0; t < 9; t++) Hi[t] = ldc(G.Hinv + (size_t)l * 9 + t);
      for (int r = 0; r < 6; r++)
        for (int m = 0; m < 3; m++) {
          G.Wd[(size_t)q * 18 + r * 3 + m] = w[r * 3 + m];
          G.Yd[(size_t)q * 18 + r * 3 + m] = w[r * 3] * Hi[m] + w[r * 3 + 1] * Hi[3 + m] + w[r * 3 + 2] * Hi[6 + m];
        }
    }
  }

  // S = Hpp_d + (pose-pose blocks) - sum_l Y_al W_bl^T over the eliminated planes, entry by entry (output-stationary): the
  // diagonal block, then the pose-pose factor blocks in factor order, then the plane products in plane order.  Band layout:
  // a bordered plane's rows hold W_al^T against its observers and its damped Hll block on the diagonal (0 against the other
  // bordered planes).  Upper halves of diagonal tiles are 0, the padding is identity.  The first tile of each row also goes
  // to the pivot-column snapshot of the step that first reads it (step first[i], parity first[i] & 1).
  // Entry (i, j), i >= j, of S in the bordered order; pair(a, b) is the index of the pose pair's lists.
  template <typename Pair>
  __device__ __forceinline__ static double direct_entry(int i, int j, double lambda, Pair pair) {
    const int n6 = 6 * G.N, np6 = 48 * G.dnbp;
    double v = 0.0;
    if (i >= np6) {   // a bordered plane's row
      const int k = i - np6, kb = k / 3, m = k - kb * 3;
      if (k >= 3 * G.dnbord) {
        v = (i == j) ? 1.0 : 0.0;
      } else if (j >= np6) {
        if ((j - np6) / 3 == kb) {
          const int cc = j - np6 - kb * 3;
          v = ldc(G.Hll + (size_t)ldc(G.dbord + kb) * 9 + m * 3 + cc);
          if (m == cc) v *= (1 + lambda);   // Cholesky.cpp:91-97
        }
      } else if (j < n6) {   // W_al of the incidence (pose b, plane): incidences are pose-ascending inside a plane
        const int b = j / 6, r = j - b * 6;
        int lo = ldc(G.dbinc + 2 * kb), hi = ldc(G.dbinc + 2 * kb + 1);
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (ldc(G.pl_pose + ldc(G.dinc_lo + mid)) < b) lo = mid + 1; else hi = mid;
        }
        if (lo < ldc(G.dbinc + 2 * kb + 1) && ldc(G.pl_pose + ldc(G.dinc_lo + lo)) == b) v = ldc(G.Wd + (size_t)lo * 18 + r * 3 + m);
      }
    } else if (i >= n6) {
      v = (i == j) ? 1.0 : 0.0;
    } else {
      const int a = i / 6, r = i - a * 6, b = j / 6, cc = j - b * 6;
      if (a == b) {
        v = ldc(G.Hpp + (size_t)a * 36 + r * 6 + cc);
        if (r == cc) v *= (1 + lambda);   // Cholesky.cpp:91-97
      }
      const size_t q = pair(a, b);
      for (int k = G.dfp_ptr[q]; k < G.dfp_ptr[q + 1]; k++) {
        const int fs = G.dfp_f[k], f = fs >> 1;
        v += (fs & 1) ? ldc(G.PF + (size_t)f * 120 + 72 + cc * 6 + r) : ldc(G.PF + (size_t)f * 120 + 72 + r * 6 + cc);
      }
      for (int k = G.dlp_ptr[q]; k < G.dlp_ptr[q + 1]; k++) {
        const double* y = G.Yd + (size_t)G.dlp_a[k] * 18 + r * 3;
        const double* w = G.Wd + (size_t)G.dlp_b[k] * 18 + cc * 3;
        v -= ldc(y) * ldc(w) + ldc(y + 1) * ldc(w + 1) + ldc(y + 2) * ldc(w + 2);
      }
    }
    return v;
  }

  __device__ void direct_assemble(double lambda) {
    if (G.dnd) { nd_assemble(lambda); return; }
    const int nb = G.dnb;
    const long long total = (long long)ldc(G.dtoff + nb) * 2304;
    int tprev = -1, ti = 0, tj = 0, f0 = 0;
    for (long long idx = tid_team(); idx < total; idx += nthr_team()) {
      const int t = (int)(idx / 2304), e = (int)(idx - (long long)t * 2304), er = e / 48, ec = e - er * 48;
      if (t != tprev) {   // tile row: the last one whose offset is <= t
        int lo = 0, hi = nb - 1;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (ldc(G.dtoff + mid) <= t) lo = mid; else hi = mid - 1;
        }
        ti = lo;
        f0 = ldc(G.dfirst + ti);
        tj = f0 + t - ldc(G.dtoff + ti);
        tprev = t;
      }
      const int i = 48 * ti + er, j = 48 * tj + ec;
      const double v = j > i ? 0.0 : direct_entry(i, j, lambda, dpair);
      tile_at(G.Sd, t)[er * kAcLd + ec] = v;
      if (tj == f0) tile_at(G.Dsnap + (size_t)(tj & 1) * nb * kAcTile, ti)[er * kAcLd + ec] = v;
    }
  }

  // band layout: b = [-gp + sum over the eliminated planes of Y_al g_l ; -g_l of the bordered planes].  The list of the pair
  // (a, a) holds exactly one record (q, q) per eliminated incidence q of pose a, plane-ascending; in the ND layout that pair
  // lies in the diagonal tile of a's tile.  (The dense solve forms b in pose_phase, with every plane eliminated.)
  __device__ void direct_rhs() {
    const int n6 = 6 * G.N;
    for (int i = tid_team(); i < n6; i += nthr_team()) {
      const int a = i / 6, r = i - a * 6;
      const size_t q = G.dnd ? (size_t)64 * ldc(nd(ND_TOFF) + ldc(nd(ND_POS) + a / 8)) + 9 * (a & 7) : (size_t)dpair(a, a);
      double v = -ldc(G.gp + i);
      for (int k = G.dlp_ptr[q]; k < G.dlp_ptr[q + 1]; k++) {
        const int inc = G.dlp_a[k];
        const double* y = G.Yd + (size_t)inc * 18 + r * 3;
        const double* g = G.gl + (size_t)G.dinc_plane[inc] * 3;
        v += ldc(y) * ldc(g) + ldc(y + 1) * ldc(g + 1) + ldc(y + 2) * ldc(g + 2);
      }
      G.b[i] = v;
    }
    for (int k = tid_team(); k < 3 * G.dnbord; k += nthr_team()) G.b[n6 + k] = -ldc(G.gl + (size_t)ldc(G.dbord + k / 3) * 3 + k % 3);
  }

  // one CTA: A (48x48, lower half read) <- L = chol(A) with a zero upper half, Li <- L^-1.
  // Returns false when a pivot is not positive (the outputs are then meaningless).
  __device__ bool chol48(double* A, double* Li) {
    const int tid = threadIdx.x;
    bool ok = true;
    for (int k = 0; k < 48; k++) {
      __syncthreads();
      const double d = A[k * kAcLd + k];
      ok = ok && (d > 0.0);
      const double s = (d > 0.0) ? sqrt(d) : 1.0;
      __syncthreads();
      if (tid >= k && tid < 48) A[tid * kAcLd + k] = (tid == k) ? s : A[tid * kAcLd + k] / s;
      __syncthreads();
      for (int e = tid; e < 48 * 48; e += kThreads) {
        const int i = e / 48, j = e - i * 48;
        if (j > k && i >= j) A[i * kAcLd + j] -= A[i * kAcLd + k] * A[j * kAcLd + k];
      }
    }
    __syncthreads();
    for (int e = tid; e < 48 * 48; e += kThreads) {
      const int i = e / 48, j = e - i * 48;
      if (j > i) A[i * kAcLd + j] = 0.0;
    }
    if (tid < 48) {   // column tid of L^-1 by forward substitution
      const int cl = tid;
      for (int i = 0; i < 48; i++) {
        double v = 0.0;
        if (i >= cl) {
          v = (i == cl) ? 1.0 : 0.0;
          for (int m = cl; m < i; m++) v -= A[i * kAcLd + m] * Li[m * kAcLd + cl];
          v /= A[i * kAcLd + i];
        }
        Li[i * kAcLd + cl] = v;
      }
    }
    __syncthreads();
    return ok;
  }

  // entry i of b in the padded bordered order (6 N pose entries, then 3 per bordered plane from row 48 nbp; 0 in the padding)
  __device__ __forceinline__ static double padded_b(int i) {
    const int n6 = 6 * G.N, np6 = 48 * G.dnbp;
    return (i < n6) ? ldc(G.b + i) : ((i >= np6 && i < np6 + 3 * G.dnbord) ? ldc(G.b + n6 + i - np6) : 0.0);
  }

  __device__ void load_tile(double* dst, const double* src) {
    for (int e = threadIdx.x; e < 48 * 48; e += kThreads) dst[(e / 48) * kAcLd + e % 48] = ldc(src + (e / 48) * kAcLd + e % 48);
  }
  __device__ void store_tile(double* dst, const double* src) {
    for (int e = threadIdx.x; e < 48 * 48; e += kThreads) dst[(e / 48) * kAcLd + e % 48] = src[(e / 48) * kAcLd + e % 48];
  }

  // S = L L^T in place, right-looking by tile columns, one team barrier per step.  Tile t belongs to CTA t % tsize.  Step K
  // visits the envelope only: the tile rows i with first[i] <= K and the trailing tiles (i, j) with first[j] <= K as well
  // (L_jK = 0 otherwise).  It reads pivot column K only from its snapshot (published by the owners of those tiles at the end
  // of step K-1, or by the assembly for the rows that start at column K; double-buffered by step parity), so the owners may
  // overwrite it with L in the same step:
  //   panel     L_iK = C_i L_KK^-T
  //   trailing  A_ij <- A_ij - L_iK L_jK^T,  K < j <= i
  // on the FP64 tensor cores.  A CTA forms -L_iK once per tile row in which it owns a trailing tile and L_jK for every such
  // tile; each product reads only L_KK^-1 and snapshot tiles, so every CTA that forms it gets the same bits.  (A trailing
  // update through A_KK^-1 or L_KK^-1 alone, with one product per tile, loses backward stability when A_KK is ill-conditioned:
  // DESIGN.md section 5.1.)  Look-ahead: the owner of tile (K+1, K+1) updates it first (unless row K+1 starts at column
  // K+1), factors it and publishes L_{K+1}^-1; step 0's pivot is factored by every CTA from the snapshot.
  __device__ void direct_factor() {
    if (G.dnd) { nd_factor(); return; }
    const int nb = G.dnb, tid = threadIdx.x;
    double* Li = reinterpret_cast<double*>(g_smem + kSmWork);
    double* Ci = Li + kAcTile;
    double* Ti = Ci + kAcTile;
    double* Cj = Ti + kAcTile;
    double* Md = Cj + kAcTile;
    const int T = c.tsize;
    auto form_T = [&]() {   // Ti = -L_iK = -(Ci Li^T)
      double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
      mma48<true>(acc, Ci, Li);
      mma48_store(Ti, acc, -1.0);
    };
    auto update = [&](int i, int j, double (&acc)[3][2]) {   // Cj (loaded) <- L_jK = Cj Li^T, then acc = A_ij + Ti L_jK^T
      {
        double l[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        mma48<true>(l, Cj, Li);
        __syncthreads();
        mma48_store(Cj, l);
        __syncthreads();
      }
      mma48_load(acc, tile_at(G.Sd, dtile(i, j)));
      mma48<true>(acc, Ti, Cj);
    };
    auto factor_pivot = [&](int d, bool publish) {   // Md holds A_dd: L_dd into the store, L_dd^-1 out
      const bool ok = chol48(Md, Li);
      if (!ok && tid == 0) *G.dflag = 1u;
      if (publish) {
        store_tile(tile_at(G.Sd, dtile(d, d)), Md);
        store_tile(tile_at(G.Dinv, d), Li);
      }
    };

    for (int K = 0; K < nb; K++) {
      const double* snap = G.Dsnap + (size_t)(K & 1) * nb * kAcTile;
      double* snapn = G.Dsnap + (size_t)((K + 1) & 1) * nb * kAcTile;
      if (K == 0) {
        load_tile(Md, snap);
        factor_pivot(0, c.rank == 0);
      } else {
        load_tile(Li, tile_at(G.Dinv, K));
      }
      __syncthreads();
      const int d = K + 1;
      int trow = -1, trowT = -1;   // tile rows whose C_i / T_i are in shared memory (T_i only once an owned trailing tile needs it)
      if (d < nb && dtile(d, d) % T == c.rank) {   // look-ahead
        const bool coupled = ldc(G.dfirst + d) <= K;
        if (coupled) {
          load_tile(Ci, tile_at(snap, d));
          __syncthreads();
          form_T();
          store_tile(Cj, Ci);
          __syncthreads();
          double acc[3][2];
          update(d, d, acc);
          mma48_store(Md, acc);
        } else {   // row d starts at column d: its pivot is the assembled tile
          load_tile(Md, tile_at(G.Sd, dtile(d, d)));
        }
        // (Li of step K is needed below for the panel and T_i: keep a copy of it, then restore)
        __syncthreads();
        double* Lsave = Cj;
        store_tile(Lsave, Li);
        __syncthreads();
        factor_pivot(d, true);
        __syncthreads();
        store_tile(Li, Lsave);
        __syncthreads();
        if (coupled) trow = trowT = d;
      }
      for (int p = ldc(G.dcol_ptr + K); p < ldc(G.dcol_ptr + K + 1); p++) {   // the rows i > K of column K
        const int i = ldc(G.dcol_row + p);
        const int t0 = dtile(i, K);
        int j = K + ((c.rank - t0 % T) % T + T) % T;
        for (; j <= i; j += T) {
          if (i == d && j == d) continue;                // done by the look-ahead
          if (j > K && ldc(G.dfirst + j) > K) {           // L_jK = 0: no update; step K+1 still reads the tile's snapshot
            if (j == d) load_tile(tile_at(snapn, i), tile_at(G.Sd, dtile(i, d)));
            continue;
          }
          if (trow != i) {
            __syncthreads();
            load_tile(Ci, tile_at(snap, i));
            __syncthreads();
            trow = i;
          }
          if (j != K && trowT != i) {   // (read after the barrier that precedes the C_j load below)
            form_T();
            trowT = i;
          }
          double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
          if (j == K) {   // panel: L_iK = C_i L_KK^-T
            mma48<true>(acc, Ci, Li);
            mma48_store(tile_at(G.Sd, t0), acc);
            continue;
          }
          __syncthreads();
          load_tile(Cj, tile_at(snap, j));
          __syncthreads();
          update(i, j, acc);
          mma48_store(tile_at(G.Sd, dtile(i, j)), acc);
          if (j == d) mma48_store(tile_at(snapn, i), acc);
        }
      }
      __syncthreads();
      team_barrier(c);
    }
  }

  // L y = b, then L^T x = y, blocked by tile row with the stored L_KK^-1; one team barrier per tile row.  Every CTA forms
  // y_K (x_K) itself from the finished part of the vector, then the team subtracts its contribution from the rows still open
  // (each entry by one thread, in step order), within the envelope: forward, the rows of tile column K; backward, the tile
  // columns first[K] .. K-1 of row K.  dvec[0] = the running right-hand side / x, dvec[1] = y.  b holds 6 N pose entries,
  // then 3 per bordered plane.
  __device__ void direct_trsv() {
    if (G.dnd) { nd_trsv(); return; }
    const int nb = G.dnb, n = 48 * nb, tid = threadIdx.x;
    double* rv = G.dvec;
    double* yv = G.dvec + n;
    double* sv = reinterpret_cast<double*>(g_smem + kSmWork);   // [48] the vector piece of this step, [48] its product
    for (int i = tid_team(); i < n; i += nthr_team()) rv[i] = padded_b(i);
    team_barrier(c);
    for (int K = 0; K < nb; K++) {   // forward: y_K = L_KK^-1 r_K;  r_J -= L_JK y_K  (J > K)
      const double* Li = tile_at(G.Dinv, K);
      if (tid < 48) sv[tid] = ldc(rv + 48 * K + tid);
      __syncthreads();
      if (tid < 48) {
        double v = 0.0;
        for (int m = 0; m <= tid; m++) v += ldc(Li + tid * kAcLd + m) * sv[m];
        sv[48 + tid] = v;
        if (c.rank == 0) yv[48 * K + tid] = v;
      }
      __syncthreads();
      const int p0 = ldc(G.dcol_ptr + K), nr = 48 * (ldc(G.dcol_ptr + K + 1) - p0);
      for (int e = tid_team(); e < nr; e += nthr_team()) {
        const int tr = ldc(G.dcol_row + p0 + e / 48), row = 48 * tr + e % 48;
        const double* Lr = tile_at(G.Sd, dtile(tr, K)) + (row % 48) * kAcLd;
        double v = ldc(rv + row);
        for (int m = 0; m < 48; m++) v -= ldc(Lr + m) * sv[48 + m];
        rv[row] = v;
      }
      __syncthreads();
      team_barrier(c);
    }
    for (int K = nb - 1; K >= 0; K--) {   // backward: x_K = L_KK^-T y_K;  y_J -= L_KJ^T x_K  (J < K)
      const double* Li = tile_at(G.Dinv, K);
      if (tid < 48) sv[tid] = ldc(yv + 48 * K + tid);
      __syncthreads();
      if (tid < 48) {
        double v = 0.0;
        for (int m = tid; m < 48; m++) v += ldc(Li + m * kAcLd + tid) * sv[m];
        sv[48 + tid] = v;
        if (c.rank == 0) rv[48 * K + tid] = v;
      }
      __syncthreads();
      for (int row = 48 * ldc(G.dfirst + K) + tid_team(); row < 48 * K; row += nthr_team()) {
        const double* Lc = tile_at(G.Sd, dtile(K, row / 48)) + (row % 48);
        double v = ldc(yv + row);
        for (int m = 0; m < 48; m++) v -= ldc(Lc + m * kAcLd) * sv[48 + m];
        yv[row] = v;
      }
      __syncthreads();
      team_barrier(c);
    }
  }

  // ---- nested-dissection layout (DESIGN.md section 5.3): the stored tiles of L's pattern in the permuted order ----
  // S tile by tile, each entry by one thread: tile (ti, tj) of the new order holds the original tiles (perm ti, perm tj); an
  // entry above the original diagonal is read from its mirror (the pair lists hold the original orientation a >= b).
  __device__ __noinline__ void nd_assemble(double lambda) {
    const long long total = (long long)ldc(nd(ND_LTPTR) + ldc(G.dnd)) * 2304;
    for (long long idx = tid_team(); idx < total; idx += nthr_team()) {
      const int t = (int)(idx / 2304), e = (int)(idx - (long long)t * 2304), er = e / 48, ec = e - er * 48;
      const int ti = ldc(nd(ND_TROW) + t), tj = ldc(nd(ND_TCOL) + t);
      double v = 0.0;
      if (ti != tj || ec <= er) {
        int i = 48 * ldc(nd(ND_PERM) + ti) + er, j = 48 * ldc(nd(ND_PERM) + tj) + ec;
        if (j > i) { const int x = i; i = j; j = x; }
        v = direct_entry(i, j, lambda, [t](int a, int b) { return (size_t)64 * t + 8 * (a & 7) + (b & 7); });
      }
      tile_at(G.Sd, t)[er * kAcLd + ec] = v;
    }
  }

  // S = L L^T in place, left-looking, level by level of the elimination tree (a column's children lie on lower levels, so
  // every L_iK it reads is final).  Stored tile t belongs to CTA (t - first tile of its level) % tsize.  Per level:
  //   (a) C_ij = A_ij - sum_K L_iK L_jK^T over the tile's update list, in list order, on the FP64 tensor cores; the owner of a
  //       diagonal tile factors it (chol48) and publishes L_jj^-1;          team barrier
  //   (b) panels L_ij = C_ij L_jj^-T;                                        team barrier
  // Each product reads two final L tiles, so every CTA that forms a tile gets the same bits.
  __device__ __noinline__ void nd_factor() {
    const int tid = threadIdx.x, T = c.tsize;
    double* Li = reinterpret_cast<double*>(g_smem + kSmWork);
    double* Xa = Li + kAcTile;
    double* Xb = Xa + kAcTile;
    for (int l = 0; l < ldc(G.dnd); l++) {
      const int t0 = ldc(nd(ND_LTPTR) + l), t1 = ldc(nd(ND_LTPTR) + l + 1);
      for (int t = t0 + c.rank; t < t1; t += T) {
        double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        double* tile = tile_at(G.Sd, t);
        mma48_load(acc, tile);
        for (int u = ldc(nd(ND_UPTR) + t); u < ldc(nd(ND_UPTR) + t + 1); u++) {
          const double* A = tile_at(G.Sd, ldc(nd(ND_UPD) + 2 * u));
          const double* B = tile_at(G.Sd, ldc(nd(ND_UPD) + 2 * u + 1));
          __syncthreads();
          for (int e = tid; e < 48 * 48; e += kThreads) {
            const int o = (e / 48) * kAcLd + e % 48;
            Xa[o] = -ldc(A + o);
            Xb[o] = ldc(B + o);
          }
          __syncthreads();
          mma48<true>(acc, Xa, Xb);
        }
        const int j = ldc(nd(ND_TCOL) + t);
        if (ldc(nd(ND_TROW) + t) == j) {   // diagonal: factor it, publish L_jj and L_jj^-1
          __syncthreads();
          mma48_store(Xa, acc);
          const bool ok = chol48(Xa, Li);
          if (!ok && tid == 0) *G.dflag = 1u;
          store_tile(tile, Xa);
          store_tile(tile_at(G.Dinv, j), Li);
        } else {
          mma48_store(tile, acc);
        }
      }
      __syncthreads();
      team_barrier(c);
      for (int t = t0 + c.rank; t < t1; t += T) {   // panels
        const int j = ldc(nd(ND_TCOL) + t);
        if (ldc(nd(ND_TROW) + t) == j) continue;
        double* tile = tile_at(G.Sd, t);
        __syncthreads();
        load_tile(Xa, tile);
        load_tile(Li, tile_at(G.Dinv, j));
        __syncthreads();
        double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        mma48<true>(acc, Xa, Li);
        mma48_store(tile, acc);
      }
      __syncthreads();
      team_barrier(c);
    }
  }

  // L y = b by ascending level, L^T x = y by descending level, one team barrier per level.  Groups of 48 threads own one
  // column each (group g of CTA rank takes the level's columns rank * groups + g, then every tsize * groups-th); each entry
  // is a gather in list order by one thread, then the product with L_jj^-1.  b is gathered into the new order first and x
  // scattered back, so dvec[0] ends as in the envelope layout.
  __device__ __noinline__ void nd_trsv() {
    constexpr int kGroups = kThreads / 48;
    const int nb = G.dnb, n = 48 * nb, tid = threadIdx.x, g = tid / 48, r = tid - 48 * g;
    double* rv = G.dvec;
    double* yv = G.dvec + n;   // the vector in the new order: b, then y, then x, in place
    double* sv = reinterpret_cast<double*>(g_smem + kSmWork) + 48 * g;
    for (int i = tid_team(); i < n; i += nthr_team()) yv[48 * ldc(nd(ND_POS) + i / 48) + i % 48] = padded_b(i);
    team_barrier(c);
    for (int l = 0; l < ldc(G.dnd); l++) {   // forward: y_j = L_jj^-1 (b_j - sum_K L_jK y_K)
      const int k1 = ldc(nd(ND_LPTR) + l + 1);
      for (int base = ldc(nd(ND_LPTR) + l) + c.rank * kGroups; base < k1; base += c.tsize * kGroups) {
        const bool act = g < kGroups && base + g < k1;
        const int j = act ? ldc(nd(ND_LCOL) + base + g) : 0;
        if (act) {
          double v = ldc(yv + 48 * j + r);
          for (int p = ldc(nd(ND_RPTR) + j); p < ldc(nd(ND_RPTR) + j + 1); p++) {
            const int t = ldc(nd(ND_RTILE) + p), K = ldc(nd(ND_TCOL) + t);
            const double* Lr = tile_at(G.Sd, t) + r * kAcLd;
            for (int m = 0; m < 48; m++) v -= ldc(Lr + m) * ldc(yv + 48 * K + m);
          }
          sv[r] = v;
        }
        __syncthreads();
        if (act) {
          const double* Li = tile_at(G.Dinv, j);
          double v = 0.0;
          for (int m = 0; m <= r; m++) v += ldc(Li + r * kAcLd + m) * sv[m];
          yv[48 * j + r] = v;
        }
        __syncthreads();
      }
      team_barrier(c);
    }
    for (int l = ldc(G.dnd) - 1; l >= 0; l--) {   // backward: x_j = L_jj^-T (y_j - sum_i L_ij^T x_i)
      const int k1 = ldc(nd(ND_LPTR) + l + 1);
      for (int base = ldc(nd(ND_LPTR) + l) + c.rank * kGroups; base < k1; base += c.tsize * kGroups) {
        const bool act = g < kGroups && base + g < k1;
        const int j = act ? ldc(nd(ND_LCOL) + base + g) : 0;
        if (act) {
          double v = ldc(yv + 48 * j + r);
          const int d = ldc(nd(ND_TOFF) + j), cnt = ldc(nd(ND_CPTR) + j + 1) - ldc(nd(ND_CPTR) + j);
          for (int t = d + 1; t < d + cnt; t++) {
            const int i = ldc(nd(ND_TROW) + t);
            const double* Lc = tile_at(G.Sd, t) + r;
            for (int m = 0; m < 48; m++) v -= ldc(Lc + m * kAcLd) * ldc(yv + 48 * i + m);
          }
          sv[r] = v;
        }
        __syncthreads();
        if (act) {
          const double* Li = tile_at(G.Dinv, j);
          double v = 0.0;
          for (int m = r; m < 48; m++) v += ldc(Li + m * kAcLd + r) * sv[m];
          yv[48 * j + r] = v;
        }
        __syncthreads();
      }
      team_barrier(c);
    }
    for (int i = tid_team(); i < n; i += nthr_team()) rv[i] = ldc(yv + 48 * ldc(nd(ND_POS) + i / 48) + i % 48);
    team_barrier(c);
  }

  // ---- marginal covariances from the ND factor (DESIGN.md section 5.4) ----
  __device__ __forceinline__ static const int* cov(int k) { return G.dcov + ldc(G.dcov + k); }   // table k of CovTable

  // Selected inversion: Sigma = S^-1 on L's tile pattern (in the new order), by descending level, with the tile ownership of
  // nd_factor.  Per level:
  //   (a) off-diagonal tiles  Sigma_ij = -(sum_k Sigma_ik L_kj) L_jj^-1 over the tile's list (k ascending); Sigma_ik is stored
  //       at (i, k) or, transposed, at (k, i);                                team barrier
  //   (b) diagonal tiles      Sigma_jj = L_jj^-T (L_jj^-1 - sum_k L_kj^T Sigma_kj) over the column's own tiles, stored as
  //       (X + X^T) / 2;                                                       team barrier
  // L_jj^-1 is applied once per output tile, after the sum, instead of forming L_kj L_jj^-1 per list entry: one product per
  // tile instead of one per entry, and no staging buffer.  Every product reads final tiles in a fixed order, so every CTA
  // that forms a tile gets the same bits.  L stays as it is (the column solves read it).
  __device__ __noinline__ void nd_selinv() {
    const int tid = threadIdx.x, T = c.tsize;
    double* Xa = reinterpret_cast<double*>(g_smem + kSmWork);
    double* Xb = Xa + kAcTile;
    auto load = [&](double* dst, const double* src, bool tr) {   // dst = src or src^T
      for (int e = tid; e < 48 * 48; e += kThreads) {
        const int r = e / 48, cc = e - r * 48;
        dst[r * kAcLd + cc] = ldc(src + (tr ? cc * kAcLd + r : r * kAcLd + cc));
      }
    };
    for (int l = ldc(G.dnd) - 1; l >= 0; l--) {
      const int t0 = ldc(nd(ND_LTPTR) + l), t1 = ldc(nd(ND_LTPTR) + l + 1);
      for (int t = t0 + c.rank; t < t1; t += T) {   // (a)
        const int j = ldc(nd(ND_TCOL) + t);
        if (ldc(nd(ND_TROW) + t) == j) continue;
        double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        for (int u = ldc(cov(COV_SPTR) + t); u < ldc(cov(COV_SPTR) + t + 1); u++) {
          const int sg = ldc(cov(COV_SEL) + 2 * u), lt = ldc(cov(COV_SEL) + 2 * u + 1);
          __syncthreads();
          load(Xa, tile_at(G.Sig, sg >> 1), sg & 1);
          load(Xb, tile_at(G.Sd, lt), false);
          __syncthreads();
          mma48<false>(acc, Xa, Xb);
        }
        __syncthreads();
        mma48_store(Xa, acc, -1.0);
        load(Xb, tile_at(G.Dinv, j), false);
        __syncthreads();
        double out[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        mma48<false>(out, Xa, Xb);
        mma48_store(tile_at(G.Sig, t), out);
      }
      __syncthreads();
      team_barrier(c);
      for (int t = t0 + c.rank; t < t1; t += T) {   // (b)
        const int j = ldc(nd(ND_TCOL) + t);
        if (ldc(nd(ND_TROW) + t) != j) continue;
        const int cnt = ldc(nd(ND_CPTR) + j + 1) - ldc(nd(ND_CPTR) + j);
        double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        for (int k = t + 1; k < t + cnt; k++) {
          __syncthreads();
          load(Xa, tile_at(G.Sd, k), true);
          load(Xb, tile_at(G.Sig, k), false);
          __syncthreads();
          mma48<false>(acc, Xa, Xb);
        }
        __syncthreads();
        load(Xb, tile_at(G.Dinv, j), false);
        load(Xa, tile_at(G.Dinv, j), true);
        __syncthreads();
        {
          int r, cc;
#pragma unroll
          for (int s = 0; s < 3; s++)
            if (mma48_frag(s, r, cc)) { Xb[r * kAcLd + cc] -= acc[s][0]; Xb[r * kAcLd + cc + 1] -= acc[s][1]; }
        }
        __syncthreads();
        double out[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
        mma48<false>(out, Xa, Xb);
        __syncthreads();
        mma48_store(Xa, out);
        __syncthreads();
        double* dst = tile_at(G.Sig, t);
        for (int e = tid; e < 48 * 48; e += kThreads) {
          const int r = e / 48, cc = e - r * 48;
          dst[r * kAcLd + cc] = 0.5 * (Xa[r * kAcLd + cc] + Xa[cc * kAcLd + r]);
        }
      }
      __syncthreads();
      team_barrier(c);
    }
  }

  // The gather records of one covariance call, one output entry per thread (crec header: [0] count, [2] offset; 8 ints each):
  //   kind 0  out[o1] = Sigma element (tile, in-tile offset)                        (a pose or bordered plane inside the pattern)
  //   kind 1  entry (r, c) of an eliminated plane l:  (Hll^-1)_rc + sum over its observer pairs (a >= b) of
  //           (Y_a^T Sigma_ab Y_b)_rc, plus (Y_a^T Sigma_ab Y_b)_cr when a != b;  to out[o1] and out[o2] (o2 = -1: none)
  __device__ __noinline__ void cov_gather() {
    const int n = ldc(G.crec);
    const int* rec = G.crec + ldc(G.crec + 2);
    for (int k = tid_team(); k < n; k += nthr_team()) {
      const int* e = rec + 8 * k;
      const int o1 = ldc(e + 1), o2 = ldc(e + 2);
      double v;
      if (ldc(e) == 0) {
        v = ldc(tile_at(G.Sig, ldc(e + 3)) + ldc(e + 4));
      } else {
        const int l = ldc(e + 3), r = ldc(e + 4), cc = ldc(e + 5);
        v = ldc(G.Hinv + (size_t)l * 9 + r * 3 + cc);
        for (int u = ldc(cov(COV_PPTR) + l); u < ldc(cov(COV_PPTR) + l + 1); u++) {
          const int* q = cov(COV_PAIR) + 4 * u;
          const int qa = ldc(q), qb = ldc(q + 1), code = ldc(q + 3);
          const double* S = tile_at(G.Sig, ldc(q + 2)) + (code >> 1);
          const double* ya = G.Yd + (size_t)qa * 18;
          const double* yb = G.Yd + (size_t)qb * 18;
          for (int p = 0; p < 6; p++)
            for (int s = 0; s < 6; s++) {
              const double sig = ldc(S + ((code & 1) ? s * kAcLd + p : p * kAcLd + s));
              v += ldc(ya + p * 3 + r) * sig * ldc(yb + s * 3 + cc);
              if (qa != qb) v += ldc(ya + p * 3 + cc) * sig * ldc(yb + s * 3 + r);
            }
        }
      }
      G.covout[o1] = v;
      if (o2 >= 0) G.covout[o2] = v;
    }
  }

  // Blocks outside the pattern, one column of the right-hand node at a time (crec header: [1] columns, [3] their offset,
  // 6 ints each: kind, a, b, c, first and end record; [4] the records' offset, 6 ints each).  A column is x = S^-1 rhs by
  // nd_trsv with rhs = e_a (kind 0: a pose or bordered plane, a its row of b) or -Y_{.l} column c (kind 1: an eliminated
  // plane l, its incidences [a, b)); x is then the column of Sigma over the kept unknowns.  Records:
  //   kind 0  out[o] = x[a]                                                          (a kept row)
  //   kind 1  out[o] = -sum_{q in [a, b)} (Y_q^T x_pose(q))_c + (e >= 0 ? Hll^-1 entry e : 0)   (row c of an eliminated plane)
  __device__ __noinline__ void cov_columns() {
    const int ncol = ldc(G.crec + 1), nk = 6 * G.N + 3 * G.dnbord;
    const int* col = G.crec + ldc(G.crec + 3);
    const int* rec = G.crec + ldc(G.crec + 4);
    for (int k = 0; k < ncol; k++) {
      const int* cl = col + 6 * k;
      const int kind = ldc(cl), a = ldc(cl + 1), b = ldc(cl + 2), cc = ldc(cl + 3);
      for (int i = tid_team(); i < nk; i += nthr_team()) G.b[i] = 0.0;
      team_barrier(c);
      if (kind == 0) {
        if (tid_team() == 0) G.b[a] = 1.0;
      } else {
        for (int q = a + tid_team(); q < b; q += nthr_team()) {
          const int p = ldc(G.pl_pose + ldc(G.dinc_lo + q));
          for (int r = 0; r < 6; r++) G.b[6 * p + r] = -ldc(G.Yd + (size_t)q * 18 + r * 3 + cc);
        }
      }
      team_barrier(c);
      nd_trsv();
      for (int e = ldc(cl + 4) + tid_team(); e < ldc(cl + 5); e += nthr_team()) {
        const int* x = rec + 6 * e;
        double v;
        if (ldc(x) == 0) {
          v = ldc(G.dvec + ldc(x + 2));
        } else {
          const int m = ldc(x + 4), h = ldc(x + 5);
          double s = 0.0;
          for (int q = ldc(x + 2); q < ldc(x + 3); q++) {
            const int p = ldc(G.pl_pose + ldc(G.dinc_lo + q));
            for (int r = 0; r < 6; r++) s += ldc(G.Yd + (size_t)q * 18 + r * 3 + m) * ldc(G.dvec + 6 * p + r);
          }
          v = (h >= 0 ? ldc(G.Hinv + h) : 0.0) - s;
        }
        G.covout[ldc(x + 1)] = v;
      }
      team_barrier(c);
    }
  }
#endif
};
