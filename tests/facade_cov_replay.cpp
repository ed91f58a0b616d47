// The frame-sequence replay of facade_replay.cpp (the same input format) on a band façade in nested-dissection order, then
// isam::Covariances through Slam::covariances(): marginal() of every node on its own, marginals() of several lists, a
// joint marginal(list) and access(pairs).  Prints the façade's own Jacobian (Slam::jacobian(), CSR) with them, so that
// tests/test_gpu_covariance.py checks every block and its place against an inverse of J^T J at the same estimate.
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <vector>

#include "../include/isam_facade.hpp"
#include <list>

using namespace isam;

static int run(int argc, char** argv);
// a diagonal covariance for either flavour of the facade's dense types (built-in, or Eigen with -DISAM_FACADE_USE_EIGEN: what
// Mapping.cpp itself does at :64-67 -- MatrixXd::Zero + diagonal entries)
static MatrixXd diag_matrix(const std::vector<double>& d) {
  MatrixXd m((int)d.size(), (int)d.size());
  for (size_t i = 0; i < d.size(); i++)
    for (size_t j = 0; j < d.size(); j++) m((int)i, (int)j) = (i == j) ? d[i] : 0.0;
  return m;
}

int main(int argc, char** argv) {
  try { return run(argc, argv); }
  catch (const std::exception& e) { fprintf(stderr, "facade_cov_replay: %s\n", e.what()); return 1; }
}
static int run(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: facade_cov_replay <frames.txt>\n"); return 2; }
  FILE* f = fopen(argv[1], "r");
  if (!f) { perror("open"); return 2; }
  int n_frames, n_planes, ground;
  if (fscanf(f, "%d %d %d", &n_frames, &n_planes, &ground) != 3) return 2;
  Slam slam;
  slam.set_linear_solver(Slam::LINEAR_SOLVER_BAND);
  slam.set_direct_ordering(Slam::ORDERING_NESTED_DISSECTION);
  Properties prop = slam.properties();   // Mapping.cpp:31-43
  prop.method = LEVENBERG_MARQUARDT;
  prop.mod_batch = 1;
  prop.quiet = true;
  prop.epsilon2 *= 0.1;
  prop.epsilon_abs *= 0.1;
  prop.epsilon_rel *= 0.1;
  slam.set_properties(prop);
  std::vector<Pose3d_Node*> poses;
  std::vector<Plane3d_Node*> planes(n_planes, nullptr);
  double pose_sig[6], ground_sig;
  for (int i = 0; i < 6; i++) if (fscanf(f, "%lf", &pose_sig[i]) != 1) return 2;
  if (fscanf(f, "%lf", &ground_sig) != 1) return 2;
  std::vector<double> pv(6);
  for (int i = 0; i < 6; i++) pv[i] = pose_sig[i] * pose_sig[i];
  Covariance poseCov(diag_matrix(pv));
  Covariance groundCov(diag_matrix({ground_sig * ground_sig, ground_sig * ground_sig, ground_sig * ground_sig}));
  for (int fr = 0; fr < n_frames; fr++) {
    double o[6];
    for (int i = 0; i < 6; i++) if (fscanf(f, "%lf", &o[i]) != 1) return 2;
    Pose3d temp_pose(o[0], o[1], o[2], o[3], o[4], o[5]);
    Pose3d estimate_pose;
    if (!poses.empty()) estimate_pose = poses.back()->value().oplus(temp_pose);   // Mapping.cpp:414-416
    Pose3d_Node* poseNode = new Pose3d_Node();
    slam.add_node(poseNode);
    if (poses.empty()) {
      slam.add_factor(new Pose3d_Factor(poseNode, temp_pose, poseCov));            // Mapping.cpp:470-473
    } else {
      poseNode->init(estimate_pose);                                               // Mapping.cpp:475
      slam.add_factor(new Pose3d_Pose3d_Factor(poses.back(), poseNode, temp_pose, poseCov));
    }
    poses.push_back(poseNode);
    if (fr == 0) estimate_pose = poseNode->value();
    int nobs;
    if (fscanf(f, "%d", &nobs) != 1) return 2;
    for (int k = 0; k < nobs; k++) {
      int pl; double m[4], sig;
      if (fscanf(f, "%d %lf %lf %lf %lf %lf", &pl, &m[0], &m[1], &m[2], &m[3], &sig) != 6) return 2;
      Plane3d measure(Vector4d(m[0], m[1], m[2], m[3]));
      if (!planes[pl]) {
        planes[pl] = new Plane3d_Node();
        slam.add_node(planes[pl]);
        planes[pl]->init(measure.transform_from(estimate_pose.oTw()));             // Mapping.cpp:497-499
        if (pl == ground) slam.add_factor(new Plane3d_Factor(planes[pl], Plane3d(Vector4d(0, 0, -1, 0)), groundCov));
      }
      Covariance cov(diag_matrix({sig * sig, sig * sig, sig * sig}));
      slam.add_factor(new Pose3d_Plane3d_Factor(poseNode, planes[pl], measure, cov, false));
    }
    if (fr % 5 == 0) slam.batch_optimization(); else slam.update();                 // Mapping.cpp:550-554
  }
  SparseJacobian J = slam.jacobian();
  printf("J %lld %lld %d\n", J.rows, J.cols, (int)J.values.size());
  for (int x : J.row_ptr) printf("%d ", x);
  printf("\n");
  for (int x : J.col_idx) printf("%d ", x);
  printf("\n");
  for (double x : J.values) printf("%.17g ", x);
  printf("\n");
  std::vector<Node*> nodes(slam.get_nodes().begin(), slam.get_nodes().end());
  for (Node* n : nodes) printf("node %d %d\n", n->unique_id(), n->dim());
  auto dump = [](const char* tag, const MatrixXd& m, int r, int c) {
    printf("%s %d %d", tag, r, c);
    for (int i = 0; i < r; i++)
      for (int j = 0; j < c; j++) printf(" %.17g", mget(m, i, j));
    printf("\n");
  };
  const Covariances& cov = slam.covariances();
  for (Node* n : nodes) dump("marginal", cov.marginal(std::list<Node*>{n}), n->dim(), n->dim());
  Covariances::node_lists_t lists;
  lists.push_back({nodes[0], nodes[nodes.size() - 1], nodes[1]});
  lists.push_back({nodes[nodes.size() / 2], nodes[2]});
  for (const MatrixXd& m : cov.marginals(lists)) dump("joint", m, mrows(m), mrows(m));
  Covariances::node_pair_list_t pairs;
  pairs.push_back(std::make_pair(nodes[0], nodes[nodes.size() - 1]));
  pairs.push_back(std::make_pair(nodes[nodes.size() - 1], nodes[1]));
  pairs.push_back(std::make_pair(nodes[3], nodes[3]));
  const std::list<MatrixXd> acc = cov.access(pairs);
  auto it = acc.begin();
  for (const auto& p : pairs) { dump("access", *it, p.first->dim(), p.second->dim()); ++it; }
  return 0;
}
