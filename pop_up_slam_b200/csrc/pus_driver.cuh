// pus_driver.cuh -- device-side Levenberg-Marquardt / Gauss-Newton driver and the persistent kernel entry.
// Included twice by pus_engine.cu right after pus_kernels.cuh (same namespaces, see there).
// ---------------------------------------------------------------------------------------------
// device: LM / GN driver
// ---------------------------------------------------------------------------------------------
__device__ void linearize(Phase& ph, Ctx& c) {
  if (ph.ft) ph.ft->sync();
  ph.lin_pose_plane();
  ph.lap2(6);
  ph.lin_other();
  team_barrier(c);
  ph.lap2(22);
  ph.assemble();
  if (G.n_asplit > 0) { team_barrier(c); ph.assemble_split(); }
  team_barrier(c);
  ph.lap2(23);
}

// Schur complement set-up for a damping value.  Hll^-1 (part of the operator) is always rebuilt; the two-level
// preconditioner (dense diagonal blocks + coarse Galerkin inverse) only when `rebuild` -- a stale
// preconditioner changes the PCG iteration count, never the solution.
__device__ __forceinline__ bool G_levels3(const Phase&) { return G.levels == 3; }
__device__ void schur_setup(Phase& ph, Ctx& c, double lambda, Timer& ft, bool rebuild) {
  ft.sync();
  ph.plane_inverse(lambda);
  team_barrier(c);
  ft.lap(8);
  if (!rebuild && !G.prm.blocks_always) return;
  ph.build_blocks(lambda);
  ft.lap(9);
  if (!rebuild) { team_barrier(c); return; }   // level 1 refreshed for this linearisation, coarse level kept
  ph.coarse_wc();
  team_barrier(c);
  ft.lap(10);
  ph.coarse_assemble(lambda);
  if (G_levels3(ph)) ph.build_groups(lambda);   // level 2: needs Wc2 / Yc2 (behind the barrier above) only
  team_barrier(c);
  ft.lap(11);
  ph.coarse_invert();
  ft.lap(12);
}

// Solve (Hpp_d - W Hll_d^-1 W^T) x = -gp + W Hll_d^-1 gl by preconditioned CG, then back-substitute the
// planes.  Returns |delta|; *its = PCG iterations.
// `warm`: start from the previous solution (kept in G.xprev) -- used after a rejected LM step, where only lambda changed.
__device__ __forceinline__ void span_view(Ctx& c, bool global) {
  if (c.span_w <= 1) return;
  if (global) { c.rank = c.span_r * c.ltsize + c.lrank; c.tsize = c.span_w * c.ltsize; c.mirror = 1; }
  else { c.rank = c.lrank; c.tsize = c.ltsize; c.mirror = 0; }
}

__device__ double schur_solve(Phase& ph, Ctx& c, double lambda, int* its, Timer& ft, bool warm) {
  // spanning solve: the PCG phases are split over the CTAs of all ranks (every rank keeps full copies of the vectors)
  span_view(c, true);
  const bool resident = G.prm.resident && !c.use_tma && !c.mirror;   // block-resident loop (pcg_resident): loads its own caches
  if (G.prm.mode == MODE_DEBUG && threadIdx.x == 0) {   // path report (PathBit); the apply branches add theirs as they run
    LmResult* res = G.res;
    atomicOr(&res->status, (resident ? (int)kPathResident : 0) | (c.use_tma ? (int)kPathTma : 0) |
                               (c.l3_local ? (int)kPathL3Local : 0) | (c.cluster ? (int)kPathCluster : 0));
    atomicMax(&res->trace_n, (G.nblk - c.rank + c.tsize - 1) / c.tsize);   // owned pose blocks k = rank + tsize * i
    if (c.rank == 0) { res->iterations = c.tsize; res->accepted = G.levels; res->chi2_evals = G.SP; }
  }
  if (!c.use_tma && !resident) {   // (large graphs use that shared memory for the TMA staging buffers instead)
    ph.cache_blocks();
    c.smem_cache_ok = 1;
  }
  ph.pose_phase(true, nullptr, lambda, nullptr, nullptr);  // rhs, with vl = Hll^-1 gl from plane_inverse
  team_barrier(c);
  double v[2];
  int rcb = 0, cur = 0, it = 0;
  v[0] = ph.precondition(0.0, nullptr, G.rcpart[0], G.rcpart[1], true);
  team_reduce<1>(c, G.red, v);
  rcb = 1;
  const double rz0 = v[0];
  double rz = rz0, beta = 0.0;
  const double tol2 = G.prm.pcg_tol * G.prm.pcg_tol;
  bool done = false;
  if (warm && rz0 > 0.0) {
    // one pseudo-iteration with direction p = x_prev and step 1:  x = x_prev, r = b - S x_prev, z = M^-1 r
    ph.sweep_planes(G.xprev, nullptr, 0.0);
    team_barrier(c);
    if (c.use_tma) { ph.solve_heavy(); team_barrier(c); }
    ph.pose_phase(false, G.xprev, lambda, G.q, G.qcpart);
    team_barrier(c);
    v[0] = ph.precondition(1.0, G.xprev, G.rcpart[rcb], G.rcpart[rcb ^ 1], false);
    team_reduce<1>(c, G.red, v);
    rcb ^= 1;
    rz = v[0];
    if (!(rz > tol2 * rz0)) done = true;
  }
  if (rz0 > 0.0 && !done && resident) {
    it = ph.pcg_resident(lambda, rcb, rz0, rz, tol2, ft);
  } else if (rz0 > 0.0 && !done) {
    c.light = c.mirror ? 0 : 1;   // every value the loop exchanges between CTAs is read through L2 (ld.global.cg / bulk copies)
    while (it < G.prm.pcg_max_iter) {
      ft.sync();
      ph.update_direction(cur, beta);
      if (c.use_tma) {   // large graphs: publish the new direction first, the sweep then gathers 6 values per edge
        team_barrier(c);
        ph.sweep_planes(G.pv[cur ^ 1], nullptr, 0.0);
      } else {
        ph.sweep_planes(G.z, G.pv[cur], beta, G.zc);
      }
      team_barrier(c);
      if (c.use_tma) { ph.solve_heavy(); team_barrier(c); }
      ft.lap(16);
      v[0] = ph.pose_phase(false, G.pv[cur ^ 1], lambda, G.q, G.qcpart);
      team_reduce<1>(c, G.red, v);
      ft.lap(19);
      const double pq = v[0];
      if (!(pq > 0.0)) break;  // breakdown (not SPD / exhausted precision)
      const double alpha = rz / pq;
      v[0] = ph.precondition(alpha, G.pv[cur ^ 1], G.rcpart[rcb], G.rcpart[rcb ^ 1], false);
      team_reduce<1>(c, G.red, v);
      ft.lap(20);
      rcb ^= 1;
      it++;
      const double rz_new = v[0];
      if (!(rz_new > tol2 * rz0)) break;
      beta = rz_new / rz;
      rz = rz_new;
      cur ^= 1;
    }
    c.light = 0;
  }
  *its = it;
  // planes: dl = Hll_d^-1 (-gl - W^T x)
  if (c.mirror) { ph.publish_x(); team_barrier(c); }
  ph.sweep_planes(G.x, nullptr, 0.0);
  team_barrier(c);
  v[0] = ph.solve_planes(1) + ph.norm_x();  // (also keeps a copy of x for the next warm start)
  team_reduce<1>(c, G.red, v);
  span_view(c, false);
  return sqrt(v[0]);
}

#ifdef PUS_DIRECT
// Exact direct solve (pus::kdirect): replaces schur_setup / schur_solve.  Sub-timers: 8 plane inverses, 10 per-incidence
// W / Y blocks, 11 assembly of S, 12 factorization, 13 right-hand side, 14 triangular solves.
__device__ void direct_setup(Phase& ph, Ctx& c, double lambda, Timer& ft) {
  ft.sync();
  if (c.rank == 0 && threadIdx.x == 0) *G.dflag = 0u;
  ph.plane_inverse(lambda);
  team_barrier(c);
  ft.lap(8);
  ph.direct_wy();
  team_barrier(c);
  ft.lap(10);
  ph.direct_assemble(lambda);
  team_barrier(c);
  ft.lap(11);
  if (G.prm.mode == MODE_DEBUG && G.prm.debug_stage == 4) return;   // stop after the assembly ("Sdir")
  ph.direct_factor();
  ft.lap(12);
}

// x = S^-1 b, then the planes as schur_solve does (the bordered planes too: the same delta in exact arithmetic).  *its = 0, or -1 after a non-positive pivot: then delta = 0.
__device__ double direct_solve(Phase& ph, Ctx& c, double lambda, int* its, Timer& ft) {
  if (G.prm.mode == MODE_DEBUG && G.prm.debug_stage == 4) { *its = 0; return 0.0; }
  ft.sync();
  const bool failed = __ldcg(G.dflag) != 0u;
  double v[1];
  if (failed) {
    for (int i = ph.tid_team(); i < G.N * 6; i += ph.nthr_team()) G.x[i] = 0.0;
    for (int i = ph.tid_team(); i < G.M * 3; i += ph.nthr_team()) G.dl[i] = 0.0;
    team_barrier(c);
    *its = -1;
    return 0.0;
  }
  if (G.dnbord) ph.direct_rhs();                                // band layout with bordered planes
  else ph.pose_phase(true, nullptr, lambda, nullptr, nullptr);   // b = -gp + W Hll_d^-1 gl
  team_barrier(c);
  ft.lap(13);
  ph.direct_trsv();
  for (int i = ph.tid_team(); i < G.N * 6; i += ph.nthr_team()) G.x[i] = ldc(G.dvec + i);
  team_barrier(c);
  ft.lap(14);
  ph.sweep_planes(G.x, nullptr, 0.0);
  team_barrier(c);
  v[0] = ph.solve_planes(1) + ph.norm_x();
  team_reduce<1>(c, G.red, v);
  *its = 0;
  return sqrt(v[0]);
}
#define schur_setup(ph, c, lambda, ft, rebuild) direct_setup(ph, c, lambda, ft)
#define schur_solve(ph, c, lambda, its, ft, warm) ((void)(warm), direct_solve(ph, c, lambda, its, ft))
// a failed factorization (|delta| = 0) is a rejected LM step, not convergence
#define PUS_SOLVE_FAILED(its) || ((its) < 0 && iter < kTraceCap)
#else
#define PUS_SOLVE_FAILED(its)
#endif

__device__ void run_graph_impl(Ctx& c) {
  Phase ph(c);
  const LmParams& P = G.prm;
  const bool lead = (c.rank == 0 && threadIdx.x == 0);
  LmResult* res = G.res;
  const bool tlead = (c.rank == (P.timer_rank < c.tsize ? P.timer_rank : 0) && threadIdx.x == 0);
  Timer tm(tlead);
  Timer& ft = tm;
  ph.ft = (P.fine_timers ? &tm : nullptr);
  if (lead) {
    res->iterations = 0; res->accepted = 0; res->relin = 0; res->chi2_evals = 0; res->pcg_iters = 0;
    res->trace_n = 0; res->status = 0; res->chi2_initial = 0; res->chi2_final = 0;
    for (int i = 0; i < 24; i++) res->phase_ns[i] = 0;
  }
  c.span_w = G.span_w > 1 ? G.span_w : 1;
  c.span_r = G.span_r;
  c.lrank = c.rank; c.ltsize = c.tsize; c.mirror = 0;
  for (int w = 0; w < 8; w++) c.peer_delta[w] = G.peer_delta[w];
  c.gbar = G.gbar;
  c.use_tma = (P.tma_mode == 1) || (P.tma_mode == 0 && G.ntile_pl > 2 * c.tsize * kWarps);
  c.smem_cache_ok = 0;
  c.l3_local = (G.levels == 3 && 6 * G.nc <= kL3Local) ? 1 : 0;
  if (P.restore_init) { ph.restore_init(); team_barrier(c); }
  if (P.mode == MODE_CHI2) {
    double e = ph.chi2(false);
    if (lead) { res->chi2_final = e; res->chi2_initial = e; res->chi2_evals = 1; }
    return;
  }
#ifdef PUS_DIRECT
  if (P.mode == MODE_COV) {   // marginal covariances (ND layout; DESIGN.md section 5.4).  debug_stage 1: Sigma first
    if (P.debug_stage == 1) {   // linearise at the estimate, factor undamped, invert on the pattern
      linearize(ph, c);
      direct_setup(ph, c, 0.0, ft);
      if (__ldcg(G.dflag) != 0u) return;   // a non-positive pivot: the host reports it and keeps nothing
      ph.nd_selinv();
    }
    ph.cov_gather();
    ph.cov_columns();
    team_barrier(c);
    return;
  }
#endif
  if (P.mode == MODE_DEBUG) {
    if (P.debug_stage == 9) {   // micro-benchmark: 1000 team barriers, 1000 team reductions (phase_ms[0], [1])
      tm.sync();
      for (int i = 0; i < 1000; i++) team_barrier(c);
      tm.lap(0);
      double v[1] = {1.0};
      for (int i = 0; i < 1000; i++) { v[0] = 1.0; team_reduce<1>(c, G.red, v); }
      tm.lap(1);
      if (tlead) tm.flush(res);
      return;
    }
    if (P.debug_stage == 3) {  // q = S * pv[0] with the current linearisation / Schur set-up
      ph.sweep_planes(G.pv[0], nullptr, 0.0);
      team_barrier(c);
      if (c.use_tma) { ph.solve_heavy(); team_barrier(c); }
      ph.pose_phase(false, G.pv[0], P.debug_lambda, G.q, nullptr);
      team_barrier(c);
      return;
    }
#ifdef PUS_DIRECT
    if (P.debug_stage == 5) {  // factor the S stored with pus_debug_store("Sdir"), then x = S^-1 b for the stored b
      if (lead) *G.dflag = 0u;
      team_barrier(c);
      ph.direct_factor();
      if (__ldcg(G.dflag) == 0u) {
        ph.direct_trsv();
        for (int i = ph.tid_team(); i < G.N * 6; i += ph.nthr_team()) G.x[i] = ldc(G.dvec + i);
        for (int k = ph.tid_team(); k < 3 * G.dnbord; k += ph.nthr_team())   // a bordered plane's part of x goes to its dl
          G.dl[(size_t)ldc(G.dbord + k / 3) * 3 + k % 3] = ldc(G.dvec + 48 * G.dnbp + k);
        team_barrier(c);
      }
      return;
    }
#endif
    linearize(ph, c);
    if (lead) res->relin = 1;
    if (P.debug_stage >= 1) {
      schur_setup(ph, c, P.debug_lambda, ft, true);
      if (P.debug_stage >= 2) {
        int its = 0;
        double dn = schur_solve(ph, c, P.debug_lambda, &its, ft, false);
        if (lead) { res->pcg_iters = its; res->chi2_final = dn; }
      }
    }
    if (tlead) tm.flush(res);
    return;
  }

  // ---- Optimizer::levenberg_marquardt / gauss_newton / relinearize ----
  tm.lap(7);
  linearize(ph, c);
  tm.lap(0);
  int relin = 1, nchi = 0, accepted = 0, iter = 0, its = 0;
  long long pcg_total = 0;
  double lambda = (P.method == 1 && P.mode == MODE_BATCH) ? P.lambda0 : 0.0;
  double err = 0.0;
  if (P.mode == MODE_BATCH) { err = ph.chi2(false); nchi++; }
  tm.lap(4);
  const double err0 = err;
  schur_setup(ph, c, lambda, ft, true);
  int prec_builds = 1;
  tm.lap(1);
  double dnorm = schur_solve(ph, c, lambda, &its, ft, false);
  pcg_total += its;
  int its_ref = its;  // PCG iterations right after the last preconditioner build
  tm.lap(2);
  if (P.mode == MODE_UPDATE) {
    // Optimizer::relinearize (GN branch): estimate = linpoint (+) h_gn
    ph.apply_delta();
    team_barrier(c);
    ph.accept_trial();
    team_barrier(c);
    tm.lap(3);
  } else if (P.method == 1) {
    int last_pcg = its;
    while ((P.max_iter <= 0 || iter < P.max_iter) && (dnorm > P.eps2 PUS_SOLVE_FAILED(its)) && err > P.eps_abs) {
      iter++;
      ph.apply_delta();
      team_barrier(c);
      tm.lap(3);
      double err_new = ph.chi2(true);
      nchi++;
      tm.lap(4);
      double diff = err - err_new;
      bool stop = false;
      if (lead && iter <= kTraceCap) {
        LmTrace* t = G.trace;
        t->lambda[iter - 1] = lambda; t->chi2_new[iter - 1] = err_new; t->chi2_before[iter - 1] = err;
        t->delta_norm[iter - 1] = dnorm; t->accepted[iter - 1] = diff > 0.0 ? 1 : 0; t->pcg[iter - 1] = last_pcg;
      }
      const bool rejected = !(diff > 0.0);
      if (diff > 0.0) {
        accepted++;
        ph.accept_trial();
        team_barrier(c);
        if (diff < P.eps_rel * err) {
          err = err_new;  // the linearisation point keeps the step (Optimizer.cpp:431-435, 466)
          stop = true;
        } else {
          lambda /= P.lambda_factor;
          err = err_new;
          tm.lap(3);
          linearize(ph, c);
          relin++;
          tm.lap(0);
        }
      } else {
        lambda *= P.lambda_factor;
      }
      if (stop) break;
      {
        // refresh the preconditioner only when the last solve needed clearly more iterations than the one right
        // after the previous build (deterministic rule, identical on every CTA)
        const bool rebuild = (P.prec_refresh == 0) || (last_pcg > its_ref * P.refresh_pct / 100 + P.refresh_add);
        schur_setup(ph, c, lambda, ft, rebuild);
        tm.lap(1);
        dnorm = schur_solve(ph, c, lambda, &its, ft, rejected && P.warm_start);
        if (rebuild) { its_ref = its; prec_builds++; }
      }
      last_pcg = its;
      pcg_total += its;
      tm.lap(2);
    }
  } else {
    double diff = P.eps_rel * err + 1;
    int last_pcg = its;
    while ((P.max_iter <= 0 || iter < P.max_iter) && dnorm > P.eps2 && err > P.eps_abs && fabs(diff) > P.eps_rel * err) {
      iter++;
      ph.apply_delta();
      team_barrier(c);
      ph.accept_trial();
      team_barrier(c);
      tm.lap(3);
      linearize(ph, c);
      relin++;
      tm.lap(0);
      double err_new = ph.chi2(false);
      nchi++;
      tm.lap(4);
      diff = err - err_new;
      if (lead && iter <= kTraceCap) {
        LmTrace* t = G.trace;
        t->lambda[iter - 1] = 0.0; t->chi2_new[iter - 1] = err_new; t->chi2_before[iter - 1] = err;
        t->delta_norm[iter - 1] = dnorm; t->accepted[iter - 1] = 1; t->pcg[iter - 1] = last_pcg;
      }
      accepted++;
      err = err_new;
      {
        const bool rebuild = (P.prec_refresh == 0) || (last_pcg > its_ref * P.refresh_pct / 100 + P.refresh_add);
        schur_setup(ph, c, 0.0, ft, rebuild);
        tm.lap(1);
        dnorm = schur_solve(ph, c, 0.0, &its, ft, false);
        if (rebuild) { its_ref = its; prec_builds++; }
      }
      last_pcg = its;
      pcg_total += its;
      tm.lap(2);
    }
  }
  if (lead) {
    res->iterations = iter; res->accepted = accepted; res->relin = relin; res->chi2_evals = nchi;
    res->pcg_iters = pcg_total; res->chi2_initial = err0; res->chi2_final = err;
    res->trace_n = iter < kTraceCap ? iter : kTraceCap;
    res->status = prec_builds;
  }
  if (tlead) {
    tm.acc[5] = (unsigned long long)prec_builds * 1000000ull;
    tm.flush(res);
  }
}

// spanning solves keep the cross-rank barrier count across launches (every rank executes the same number of global
// barriers per solve, so the counters are never reset while peers may already be running)
__device__ void run_graph(Ctx& c) {
  if (G.span_w > 1 && threadIdx.x == 0) c.gbar_target = __ldcg(G.gbar + 1);
  run_graph_impl(c);
  if (G.span_w > 1) {
    __syncthreads();
    if (threadIdx.x == 0) G.gbar[1] = c.gbar_target;
  }
}

__global__ void __launch_bounds__(kThreads, 1) lm_kernel(const DevGraph* graphs, int n_graphs, int team_ctas, unsigned* bars, int cluster) {
  unsigned char* const smem = g_smem;
  const int n_teams = gridDim.x / team_ctas;
  const int team = blockIdx.x / team_ctas;
  if (team >= n_teams) return;
  Ctx c;
  c.rank = blockIdx.x % team_ctas;
  c.tsize = team_ctas;
  c.bar = bars + team * 32;
  c.bar_target = 0;
  c.red_slot = 0;
  c.smem_cache_ok = 0;
  c.smem = g_smem;
  c.use_tma = 0;
  c.tma_par = 0;
  c.gj_par = 0;
  c.span_w = 1; c.span_r = 0; c.mirror = 0; c.gbar = nullptr; c.gbar_target = 0;
  c.rflag = reinterpret_cast<unsigned long long*>(bars + 8192) + (size_t)team * team_ctas * 4;
  c.red_seq = 0;
  c.light = 0;
  c.cluster = (cluster && team_ctas > 1) ? 1 : 0;   // launched with cluster dimension = team_ctas
  c.cl_par = 0;
  if (threadIdx.x == 0) {
    if (c.cluster) mbar_init(reinterpret_cast<unsigned long long*>(smem + kSmClBar), (unsigned)team_ctas);
    unsigned long long* gbar = reinterpret_cast<unsigned long long*>(smem + kSmGjBar);
    mbar_init(gbar, 1);
    mbar_init(gbar + 1, 1);
    mbar_init(gbar + 2, 1);
    mbar_init(gbar + 3, 1);
  }
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(smem + kSmBar) + (threadIdx.x >> 5) * 2;
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (c.cluster) cluster_sync_all();   // every CTA of the cluster runs before the first store into a peer's shared memory
  for (int g = team; g < n_graphs; g += n_teams) {
    __syncthreads();
    const int* src = reinterpret_cast<const int*>(graphs + g);
    int* dst = reinterpret_cast<int*>(&g_sG);
    for (int i = threadIdx.x; i < (int)(sizeof(DevGraph) / sizeof(int)); i += kThreads) dst[i] = src[i];
    __syncthreads();
    run_graph(c);
  }
  if (c.cluster) cluster_sync_all();   // no CTA exits while a peer may still address its shared memory
}

#undef PUS_SOLVE_FAILED
#ifdef PUS_DIRECT
#undef schur_setup
#undef schur_solve
#endif
#undef G
