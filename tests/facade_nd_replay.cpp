// The frame-sequence replay of facade_replay.cpp with the solver handle in band direct linear-solver mode, nested-dissection
// order: every isam::Slam the replay constructs called Slam::set_linear_solver(LINEAR_SOLVER_BAND) and
// Slam::set_direct_ordering(ORDERING_NESTED_DISSECTION) first.  Built and run by tests/test_gpu_nd_solve.py, which compares
// its output with the closed-form oracle.
#include "../include/isam_facade.hpp"

namespace isam {
struct NdSlam : Slam {
  NdSlam() {
    set_linear_solver(LINEAR_SOLVER_BAND);
    set_direct_ordering(ORDERING_NESTED_DISSECTION);
  }
};
}  // namespace isam

#define Slam NdSlam
#include "facade_replay.cpp"
