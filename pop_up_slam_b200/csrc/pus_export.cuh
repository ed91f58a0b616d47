// pus_export.cuh -- the interface between pus_engine.cu and the export kernels of pus_export.cu (weighted errors and the
// stacked sparse Jacobian of the whole graph at the current estimate: pus_weighted_errors, pus_factor_errors, pus_jacobian,
// pus_normalized_chi2, pus_local_chi2).
//
// Records.  The kernels run one thread per factor record of the uploaded layout, in the order
//   [0, nslot)                    pose-plane slots (pad slots have pp_pose = -1 and no factor)
//   [nslot, nslot + Epf)          pose factors (prior / odometry)
//   [nslot + Epf, ... + Elp)      plane priors
// and take every output offset from a per-record table built on the host once per layout:
//   row  first row of the factor in the stacked system (iSAM's factor order), -1 for a pad slot
//   val  index of the factor's first stored value; its dim rows hold ncols values each, ncols = sum of its nodes' dims
//   ca   column of the factor's first node (pose of a pose-plane edge / odometry pose 1 / prior's node)
//   cb   column of its second node (plane of a pose-plane edge / odometry pose 2), -1 for unary factors
// Within a row the columns ascend (the two nodes' blocks are swapped when cb < ca), and zeros stay stored, as
// Slam::jacobian_partial does (Slam.cpp:425).
#pragma once
#include <cuda_runtime.h>

namespace pus {

struct ExportRec {
  int row, val, ca, cb;
};

struct ExportArgs {
  // layout and estimate (device pointers of the uploaded graph)
  const double* pose_lin;
  const double* plane_lin;
  const int* pp_pose;
  const int* pp_plane;
  const double* pp_meas;
  const double* pp_sinf;
  const double* pp_rays;
  const int* pp_kind;
  int n_f2;
  const int* pf_i;
  const int* pf_j;
  const double* pf_meas;
  const double* pf_sinf;
  const int* lp_plane;
  const double* lp_meas;
  const double* lp_sinf;
  int nslot, Epf, Elp;
  int robust_kind;
  double robust_b;
  int numeric;                 // 1: the blocks by central differences (pus_set_jacobian_mode(h, 1)), 0: closed forms
  const ExportRec* rec;        // per-record table
  // what to evaluate: records recs[0..n) (recs == nullptr: records 0..n), errors written from row orow[i] (orow == nullptr:
  // from rec[].row)
  const int* recs;
  const int* orow;
  int n;
  double* err;                 // weighted, robustified errors at the estimate
  double* vals;                // Jacobian values (nullptr: errors only)
  double* rhs;                 // -(the residual the blocks were formed with); with vals only
};

cudaError_t launch_export(cudaStream_t st, const ExportArgs& a);
// CSR structure of the layout: row_ptr [rows + 1], col_idx [nnz]
cudaError_t launch_export_structure(cudaStream_t st, const ExportRec* rec, int nrec, int nslot, int Epf, const int* pf_j, int rows, int nnz, int* row_ptr, int* col_idx);
// sum of squares of x[lo, hi) in a fixed order: per-block partial sums over fixed chunks, then one block over the partials
// (part: at least kExportRedBlocks doubles of scratch); out: one double on the device
constexpr int kExportRedBlocks = 256;
cudaError_t launch_sumsq(cudaStream_t st, const double* x, long long lo, long long hi, double* part, double* out);

}  // namespace pus
