// TEST INFRASTRUCTURE ONLY.  The reference driver (oracle/ref_driver.cpp, included unmodified) plus one entry over the
// UNMODIFIED reference's own covariance recovery:
//   ref_covariance_blocks   Slam::covariances().access(node_pair_list)   Covariances.cpp:107-150 (covariance.cpp's
//                           cov_marginal / recover over Slam::_R, the factor the last update() / batch step left)
// Blocks dim(first) x dim(second), row-major, packed in pair order, as pus_covariance_blocks writes them.  Linked by
// tests/cov_ref_api.py against the reference objects `make -C oracle ref` left in oracle/_ref/obj.
#include "../oracle/ref_driver.cpp"

extern "C" {

long long ref_covariance_blocks(void* h, int n_pairs, const int* id_pairs, double* out) {
  Handle* s = H(h);
  Covariances::node_pair_list_t pairs;
  for (int k = 0; k < n_pairs; k++) {
    const int a = id_pairs[2 * k], b = id_pairs[2 * k + 1];
    if (a < 0 || b < 0 || a >= (int)s->nodes.size() || b >= (int)s->nodes.size() || !s->nalive[a] || !s->nalive[b]) {
      g_err = "bad node id";
      return -1;
    }
    pairs.push_back(std::make_pair(s->nodes[a], s->nodes[b]));
  }
  const std::list<Eigen::MatrixXd> blocks = s->slam.covariances().access(pairs);
  if ((int)blocks.size() != n_pairs) { g_err = "Covariances::access returned no blocks (no factor yet: call update first)"; return -1; }
  long long o = 0;
  for (const Eigen::MatrixXd& m : blocks)
    for (int i = 0; i < m.rows(); i++)
      for (int j = 0; j < m.cols(); j++) out[o++] = m(i, j);
  return o;
}

}  // extern "C"
