// TEST INFRASTRUCTURE ONLY.  The oracle's entry points (oracle/oracle_capi.cpp, included unmodified) plus the stacked exports
// with the shapes of the product's pus_weighted_errors / pus_factor_errors / pus_jacobian / pus_normalized_chi2 /
// pus_local_chi2, over the oracle's own restatement of Slam::weighted_errors (Slam.cpp:254-264), Slam::jacobian_partial
// (Slam.cpp:395-432: Slam::jacobian(J) in oracle_slam.hpp), normalized_chi2 and local_chi2 (Slam.cpp:270-289).  Compiled by
// the tests into a temporary library (tests/export_native.py); nothing in the product links it.
#include <algorithm>

#include "../oracle/oracle_capi.cpp"

namespace {
long long live_rows(Slam* s) { return s->dim_measure(); }
long long live_cols(Slam* s) {
  long long c = 0;
  for (const auto& n : s->nodes) if (n.alive) c += node_dim(n.kind);
  return c;
}
}  // namespace

extern "C" {

int orc_jacobian_dims(void* h, long long* rows, long long* cols) {
  if (rows) *rows = live_rows(S(h));
  if (cols) *cols = live_cols(S(h));
  return 0;
}

// Slam::weighted_errors(ESTIMATE): Factor::error of every live factor in factor order
long long orc_weighted_errors(void* h, double* out, long long cap) {
  Slam* s = S(h);
  const long long rows = live_rows(s);
  if (!out) return rows;
  if (cap < rows) { g_err = "capacity"; return -1; }
  long long r = 0;
  for (const auto& f : s->factors) {
    if (!f.alive) continue;
    s->error(f, ESTIMATE, out + r);
    r += f.dim;
  }
  return rows;
}

int orc_factor_errors(void* h, int n, const int* fids, double* out) {
  Slam* s = S(h);
  int r = 0;
  for (int i = 0; i < n; i++) {
    if (fids[i] < 0 || fids[i] >= (int)s->factors.size() || !s->factors[fids[i]].alive) { g_err = "bad factor id"; return -1; }
    s->error(s->factors[fids[i]], ESTIMATE, out + r);
    r += s->factors[fids[i]].dim;
  }
  return r;
}

// Slam::jacobian() at the estimate (copied to the linearisation point first, as orc_normal_equations does): CSR with the
// columns of every row ascending, zeros stored; rhs = -residual (Jacobian.h:97-98).  cap_nnz = 0: size query.
long long orc_jacobian(void* h, int* row_ptr, int* col_idx, double* values, double* rhs, long long cap_nnz) {
  Slam* s = S(h);
  s->estimate_to_linpoint();
  std::vector<LinFactor> J;
  s->jacobian(J);   // (update_starts inside: node columns of Slam::update_starts)
  s->estimate_to_linpoint();
  long long nnz = 0;
  for (const LinFactor& lf : J) nnz += (long long)lf.dim * (lf.ndim[0] + (lf.n_nodes == 2 ? lf.ndim[1] : 0));
  if (cap_nnz == 0) return nnz;
  if (cap_nnz < nnz) { g_err = "cap_nnz"; return -1; }
  long long v = 0, row = 0;
  if (row_ptr) row_ptr[0] = 0;
  for (const LinFactor& lf : J) {
    const int ncols = lf.ndim[0] + (lf.n_nodes == 2 ? lf.ndim[1] : 0);
    int order[2] = {0, 1};
    if (lf.n_nodes == 2 && s->nodes[lf.nodes[1]].start < s->nodes[lf.nodes[0]].start) std::swap(order[0], order[1]);
    for (int i = 0; i < lf.dim; i++, row++) {
      for (int q = 0; q < lf.n_nodes; q++) {
        const int k = order[q], off = (k == 1) ? lf.ndim[0] : 0, c0 = s->nodes[lf.nodes[k]].start;
        for (int j = 0; j < lf.ndim[k]; j++, v++) {
          if (col_idx) col_idx[v] = c0 + j;
          if (values) values[v] = lf.H[i * ncols + off + j];
        }
      }
      if (row_ptr) row_ptr[row + 1] = (int)v;
      if (rhs) rhs[row] = lf.rhs[i];
    }
  }
  return nnz;
}

// Slam::normalized_chi2  Slam.cpp:287-289
int orc_normalized_chi2(void* h, double* out) {
  Slam* s = S(h);
  *out = s->chi2(ESTIMATE) / (double)(live_rows(s) - live_cols(s));
  return 0;
}

// Slam::local_chi2  Slam.cpp:270-285: the last_n most recent live factors
int orc_local_chi2(void* h, int last_n, double* out) {
  Slam* s = S(h);
  double acc = 0, r[6];
  int n = 0;
  for (int i = (int)s->factors.size() - 1; i >= 0 && n < last_n; i--) {
    const auto& f = s->factors[i];
    if (!f.alive) continue;
    s->error(f, ESTIMATE, r);
    for (int k = 0; k < f.dim; k++) acc += r[k] * r[k];
    n++;
  }
  *out = acc;
  return 0;
}

}  // extern "C"
