// A small corridor solved through include/isam_facade.hpp, then read back through the export methods iSAM users call after a
// solve: Slam::weighted_errors, normalized_chi2, local_chi2, Factor::error and Slam::jacobian.  Prints them;
// tests/test_gpu_export.py (test_facade_export_replay) runs it and checks them against each other.
#include <cmath>
#include <cstdio>
#include <exception>
#include <vector>

#include "../include/isam_facade.hpp"

using namespace isam;

static MatrixXd diag_matrix(const std::vector<double>& d) {
  MatrixXd m((int)d.size(), (int)d.size());
  for (size_t i = 0; i < d.size(); i++)
    for (size_t j = 0; j < d.size(); j++) m((int)i, (int)j) = (i == j) ? d[i] : 0.0;
  return m;
}

static int run() {
  Slam slam;
  Properties prop = slam.properties();
  prop.method = LEVENBERG_MARQUARDT;
  slam.set_properties(prop);
  Covariance poseCov(diag_matrix({1e-4, 1e-4, 1e-4, 1e-6, 1e-6, 1e-6}));
  Covariance planeCov(diag_matrix({1e-4, 1e-4, 1e-4}));
  const int n_poses = 12, n_walls = 4;
  std::vector<Pose3d_Node*> poses;
  std::vector<Plane3d_Node*> walls;
  std::vector<Factor*> factors;
  for (int i = 0; i < n_poses; i++) {
    Pose3d_Node* p = new Pose3d_Node();
    slam.add_node(p);
    if (i == 0) factors.push_back(new Pose3d_Factor(p, Pose3d(0, 0, 1, 0, 0, 0), poseCov));
    else factors.push_back(new Pose3d_Pose3d_Factor(poses.back(), p, Pose3d(0.5 + 0.001 * i, 0.002 * (i % 3), 0, 0.01, 0, 0), poseCov));
    slam.add_factor(factors.back());
    poses.push_back(p);
    for (int k = 0; k < n_walls; k++) {
      if ((int)walls.size() <= k) { walls.push_back(new Plane3d_Node()); slam.add_node(walls.back()); }
      // walls x = 2 + 1.5 k seen from pose i (at x ~ 0.5 i): sensor-frame plane n = (1, 0, 0), d = -(2 + 1.5 k - 0.5 i)
      const double d = -(2.0 + 1.5 * k - 0.5 * i) + 0.003 * ((i + k) % 4);
      factors.push_back(new Pose3d_Plane3d_Factor(p, walls[k], Plane3d(Vector4d(1, 0.01 * k, 0, d)), planeCov, false));
      slam.add_factor(factors.back());
    }
  }
  const int it = slam.batch_optimization();
  const double chi2 = slam.chi2();
  VectorXd e = slam.weighted_errors();
  double ss = 0;
  for (int i = 0; i < (int)e.size(); i++) ss += e[i] * e[i];
  printf("iterations %d\nchi2 %.17g\nsumsq %.17g\nrows %d\n", it, chi2, ss, (int)e.size());
  printf("normalized_chi2 %.17g\n", slam.normalized_chi2());
  for (int n : {0, 1, 5, 1000}) printf("local_chi2 %d %.17g\n", n, slam.local_chi2(n));
  VectorXd fe = factors[7]->error();
  printf("factor_error 7");
  for (int i = 0; i < (int)fe.size(); i++) printf(" %.17g", fe[i]);
  printf("\n");
  SparseJacobian J = slam.jacobian();
  double rhs_err = 0;
  for (long long r = 0; r < J.rows; r++) rhs_err = std::fmax(rhs_err, std::fabs(J.rhs[(size_t)r] + e[(int)r]));
  printf("jacobian %lld %lld %lld %.3g\n", J.rows, J.cols, (long long)J.values.size(), rhs_err);
  for (Factor* f : factors) delete f;
  for (Pose3d_Node* p : poses) delete p;
  for (Plane3d_Node* w : walls) delete w;
  return 0;
}

int main() {
  try { return run(); }
  catch (const std::exception& ex) { fprintf(stderr, "facade_export_replay: %s\n", ex.what()); return 1; }
}
