// The frame-sequence replay of facade_replay.cpp with the solver handle in direct linear-solver mode: every isam::Slam the
// replay constructs is one that called Slam::set_linear_solver(LINEAR_SOLVER_DIRECT) first.  Built and run by
// tests/test_gpu_direct_solve.py, which compares its output with the closed-form oracle.
#include "../include/isam_facade.hpp"

namespace isam {
struct DirectSlam : Slam {
  DirectSlam() { set_linear_solver(LINEAR_SOLVER_DIRECT); }
};
}  // namespace isam

#define Slam DirectSlam
#include "facade_replay.cpp"
