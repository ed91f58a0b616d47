// The frame-sequence replay of facade_replay.cpp with the solver handle in band direct linear-solver mode: every isam::Slam
// the replay constructs is one that called Slam::set_linear_solver(LINEAR_SOLVER_BAND) first.  Built and run by
// tests/test_gpu_band_solve.py, which compares its output with the closed-form oracle.
#include "../include/isam_facade.hpp"

namespace isam {
struct BandSlam : Slam {
  BandSlam() { set_linear_solver(LINEAR_SOLVER_BAND); }
};
}  // namespace isam

#define Slam BandSlam
#include "facade_replay.cpp"
