// TEST INFRASTRUCTURE ONLY.  The reference driver (oracle/ref_driver.cpp, included unmodified) plus ref_* exports over the
// UNMODIFIED reference's own methods:
//   Slam::weighted_errors(ESTIMATE)  Slam.cpp:254-264      Factor::error(ESTIMATE)  Factor.h:67-77
//   Slam::jacobian()                 Slam.cpp:379-432      (jacobian_partial, or jacobian_numerical_columnwise when
//                                                           Properties::force_numerical_jacobian is set), SparseSystem -> CSR
//   Slam::normalized_chi2            Slam.cpp:287-289      Slam::local_chi2  Slam.cpp:270-285
// Linked by the tests (tests/export_native.py) against the reference objects `make -C oracle ref` left in oracle/_ref/obj.
#include "../oracle/ref_driver.cpp"

extern "C" {

int ref_jacobian_dims(void* h, long long* rows, long long* cols) {
  Slam& s = H(h)->slam;
  long long r = 0, c = 0;
  for (Factor* f : s.get_factors()) r += f->dim();
  for (Node* n : s.get_nodes()) c += n->dim();
  if (rows) *rows = r;
  if (cols) *cols = c;
  return 0;
}

long long ref_weighted_errors(void* h, double* out, long long cap) {
  const Eigen::VectorXd e = H(h)->slam.weighted_errors(ESTIMATE);
  if (!out) return (long long)e.size();
  if (cap < (long long)e.size()) { g_err = "capacity"; return -1; }
  for (int i = 0; i < (int)e.size(); i++) out[i] = e(i);
  return (long long)e.size();
}

int ref_factor_errors(void* h, int n, const int* fids, double* out) {
  int r = 0;
  for (int i = 0; i < n; i++) {
    const int d = ref_factor_error(h, fids[i], out + r);
    if (d < 0) return -1;
    r += d;
  }
  return r;
}

// Slam::jacobian() with force_numerical_jacobian = columnwise.  Like ref_factor_jacobian, every node's estimate is copied to
// its linearisation point first: Slam::jacobian() differentiates at LINPOINT, which after a solve equals the estimate, while
// in a freshly built graph the two can differ; the export evaluates at the estimate.  cap_nnz = 0: size query.
long long ref_jacobian(void* h, int columnwise, int* row_ptr, int* col_idx, double* values, double* rhs, long long cap_nnz) {
  Slam& s = H(h)->slam;
  Properties p = s.properties();
  const bool saved = p.force_numerical_jacobian;
  p.force_numerical_jacobian = columnwise != 0;
  s.set_properties(p);
  for (Node* n : s.get_nodes()) n->estimate_to_linpoint();
  SparseSystem J = s.jacobian();
  p.force_numerical_jacobian = saved;
  s.set_properties(p);
  long long nnz = 0;
  for (int r = 0; r < J.num_rows(); r++) nnz += J.get_row(r).nnz();
  if (cap_nnz == 0) return nnz;
  if (cap_nnz < nnz) { g_err = "cap_nnz"; return -1; }
  long long v = 0;
  if (row_ptr) row_ptr[0] = 0;
  for (int r = 0; r < J.num_rows(); r++) {
    for (SparseVectorIter it(J.get_row(r)); it.valid(); it.next(), v++) {
      double val;
      const int c = it.get(val);
      if (col_idx) col_idx[v] = c;
      if (values) values[v] = val;
    }
    if (row_ptr) row_ptr[r + 1] = (int)v;
    if (rhs) rhs[r] = J.rhs()(r);
  }
  return nnz;
}

int ref_normalized_chi2(void* h, double* out) { *out = H(h)->slam.normalized_chi2(); return 0; }
int ref_local_chi2(void* h, int last_n, double* out) { *out = H(h)->slam.local_chi2(last_n); return 0; }

}  // extern "C"
