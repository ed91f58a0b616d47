// pus_export.cu -- the weighted errors and the stacked sparse Jacobian of the whole graph at the current estimate, on the
// device: one thread per factor record (pus_export.cuh), evaluated with the residual / Jacobian functions of pus_math.cuh
// that the solver's lineariser uses.  Reproduces
//   Slam::weighted_errors(ESTIMATE)   ISAM/isamlib/Slam.cpp:254-264   (Factor::error, ISAM/include/isam/Factor.h:67-77)
//   Slam::jacobian()                  ISAM/isamlib/Slam.cpp:379-432   (rows in factor order, columns in node order,
//                                                                       rhs = Jacobian::rhs() = -residual, Jacobian.h:97-98)
//   Slam::local_chi2 / normalized_chi2  ISAM/isamlib/Slam.cpp:270-289 (through launch_sumsq: a fixed-order reduction)
#include <cuda_runtime.h>

#include "pus_export.cuh"
#include "pus_math.cuh"

namespace pus {

// the central-difference blocks are long: kept out of line so that the closed-form path keeps its registers
__device__ __noinline__ void export_pose_plane_numeric(const double* pose, const double* plane, const double* meas, const double* sinf,
                                                       int robust_kind, double robust_b, double* r, double* Jp, double* Jl,
                                                       const double* rays) {
  pose_plane_numeric(pose, plane, meas, sinf, robust_kind, robust_b, r, Jp, Jl, rays);
}
__device__ __noinline__ void export_pose_factor_numeric(const double* p1, const double* p2, const double* meas, const double* sinf,
                                                        int robust_kind, double robust_b, double* r, double* J1, double* J2) {
  pose_factor_numeric(p1, p2, meas, sinf, robust_kind, robust_b, r, J1, J2);
}

// the dim rows of one factor: block A (wa columns from ca) and block B (wb columns from cb), in ascending column order
__device__ __forceinline__ void put_blocks(double* vals, int val, int dim, int wa, int wb, bool a_first, const double* JA,
                                           const double* JB) {
  const int ncols = wa + wb, offa = a_first ? 0 : wb, offb = a_first ? wa : 0;
  for (int r = 0; r < dim; r++) {
    double* row = vals + (size_t)val + (size_t)r * ncols;
    for (int k = 0; k < wa; k++) row[offa + k] = JA[r * wa + k];
    for (int k = 0; k < wb; k++) row[offb + k] = JB[r * wb + k];
  }
}

__global__ void export_kernel(const ExportArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int q = a.recs ? a.recs[i] : i;
  const ExportRec R = a.rec[q];
  if (R.row < 0) return;   // pad slot
  const int orow = a.orow ? a.orow[i] : R.row;
  const bool jac = a.vals != nullptr;
  double r[6], rj[6], JA[36], JB[36];
  int dim, wa, wb;
  if (q < a.nslot) {   // pose-plane edge (Pose3d_Plane3d_Factor, or Factor2 when the slot carries rays)
    const int p = a.pp_pose[q], l = a.pp_plane[q];
    double pose[7], pl[4], m[4], si[6];
    for (int t = 0; t < 7; t++) pose[t] = a.pose_lin[(size_t)p * 7 + t];
    for (int t = 0; t < 4; t++) pl[t] = a.plane_lin[(size_t)l * 4 + t];
    for (int t = 0; t < 4; t++) m[t] = a.pp_meas[(size_t)q * 4 + t];
    for (int t = 0; t < 6; t++) si[t] = a.pp_sinf[(size_t)q * 6 + t];
    const double* rays = (a.n_f2 > 0 && a.pp_kind[q]) ? a.pp_rays + (size_t)q * 6 : nullptr;
    dim = 3; wa = 6; wb = 3;
    if (!jac) {
      pose_plane_linearize(pose, pl, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr, rays);
    } else if (a.numeric) {
      pose_plane_linearize(pose, pl, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr, rays);
      export_pose_plane_numeric(pose, pl, m, si, a.robust_kind, a.robust_b, rj, JA, JB, rays);
    } else {
      pose_plane_linearize(pose, pl, m, si, a.robust_kind, a.robust_b, r, JA, JB, rays);
      for (int t = 0; t < 3; t++) rj[t] = r[t];
    }
  } else if (q < a.nslot + a.Epf) {   // pose prior / odometry
    const int f = q - a.nslot, pi = a.pf_i[f], pj = a.pf_j[f];
    double p1[7], p2[7], m[6], si[21];
    for (int t = 0; t < 7; t++) p1[t] = a.pose_lin[(size_t)pi * 7 + t];
    if (pj >= 0) for (int t = 0; t < 7; t++) p2[t] = a.pose_lin[(size_t)pj * 7 + t];
    for (int t = 0; t < 6; t++) m[t] = a.pf_meas[(size_t)f * 6 + t];
    for (int t = 0; t < 21; t++) si[t] = a.pf_sinf[(size_t)f * 21 + t];
    const double* p2p = pj >= 0 ? p2 : nullptr;
    dim = 6; wa = 6; wb = pj >= 0 ? 6 : 0;
    if (!jac) {
      pose_factor_linearize(p1, p2p, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr);
    } else if (a.numeric) {
      pose_factor_linearize(p1, p2p, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr);
      export_pose_factor_numeric(p1, p2p, m, si, a.robust_kind, a.robust_b, rj, JA, JB);
    } else {
      pose_factor_linearize(p1, p2p, m, si, a.robust_kind, a.robust_b, r, JA, JB);
      for (int t = 0; t < 6; t++) rj[t] = r[t];
    }
  } else {   // plane prior
    const int f = q - a.nslot - a.Epf, l = a.lp_plane[f];
    double pl[4], m[4], si[6];
    for (int t = 0; t < 4; t++) pl[t] = a.plane_lin[(size_t)l * 4 + t];
    for (int t = 0; t < 4; t++) m[t] = a.lp_meas[(size_t)f * 4 + t];
    for (int t = 0; t < 6; t++) si[t] = a.lp_sinf[(size_t)f * 6 + t];
    dim = 3; wa = 3; wb = 0;
    if (!jac) {
      pose_plane_linearize(nullptr, pl, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr);
    } else if (a.numeric) {
      pose_plane_linearize(nullptr, pl, m, si, a.robust_kind, a.robust_b, r, nullptr, nullptr);
      export_pose_plane_numeric(nullptr, pl, m, si, a.robust_kind, a.robust_b, rj, nullptr, JA, nullptr);
    } else {
      pose_plane_linearize(nullptr, pl, m, si, a.robust_kind, a.robust_b, r, nullptr, JA);
      for (int t = 0; t < 3; t++) rj[t] = r[t];
    }
  }
  for (int t = 0; t < dim; t++) a.err[(size_t)orow + t] = r[t];
  if (!jac) return;
  put_blocks(a.vals, R.val, dim, wa, wb, R.cb < 0 || R.ca < R.cb, JA, JB);
  for (int t = 0; t < dim; t++) a.rhs[(size_t)R.row + t] = -rj[t];
}

__global__ void export_structure_kernel(const ExportRec* __restrict__ rec, int nrec, int nslot, int Epf, const int* __restrict__ pf_j, int rows, int nnz, int* row_ptr, int* col_idx) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0) row_ptr[rows] = nnz;
  if (q >= nrec) return;
  const ExportRec R = rec[q];
  if (R.row < 0) return;
  int dim, wa, wb;
  if (q < nslot) { dim = 3; wa = 6; wb = 3; }
  else if (q < nslot + Epf) { dim = 6; wa = 6; wb = pf_j[q - nslot] >= 0 ? 6 : 0; }
  else { dim = 3; wa = 3; wb = 0; }
  const bool a_first = R.cb < 0 || R.ca < R.cb;
  const int ncols = wa + wb, offa = a_first ? 0 : wb, offb = a_first ? wa : 0;
  for (int r = 0; r < dim; r++) {
    const int base = R.val + r * ncols;
    row_ptr[R.row + r] = base;
    for (int k = 0; k < wa; k++) col_idx[base + offa + k] = R.ca + k;
    for (int k = 0; k < wb; k++) col_idx[base + offb + k] = R.cb + k;
  }
}

// fixed-order sum of squares: block b sums the chunk [lo + b chunk, lo + (b + 1) chunk) thread-strided, then a shared-memory
// tree; the second launch adds the block sums the same way.  The order depends only on (lo, hi): repeated calls are bit-identical.
constexpr int kRedThreads = 256;
__device__ __forceinline__ double block_tree(double v, double* sm) {
  sm[threadIdx.x] = v;
  __syncthreads();
  for (int s = kRedThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  return sm[0];
}
__global__ void sumsq_part_kernel(const double* __restrict__ x, long long lo, long long hi, double* part) {
  __shared__ double sm[kRedThreads];
  const long long len = hi - lo, chunk = (len + gridDim.x - 1) / gridDim.x;
  const long long b0 = lo + (long long)blockIdx.x * chunk, b1 = min(hi, b0 + chunk);
  double acc = 0;
  for (long long k = b0 + threadIdx.x; k < b1; k += kRedThreads) acc += x[k] * x[k];
  const double s = block_tree(acc, sm);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void sumsq_final_kernel(const double* __restrict__ part, int n, double* out) {
  __shared__ double sm[kRedThreads];
  double acc = 0;
  for (int k = threadIdx.x; k < n; k += kRedThreads) acc += part[k];
  const double s = block_tree(acc, sm);
  if (threadIdx.x == 0) *out = s;
}

cudaError_t launch_export(cudaStream_t st, const ExportArgs& a) {
  if (a.n > 0) export_kernel<<<(a.n + 127) / 128, 128, 0, st>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_export_structure(cudaStream_t st, const ExportRec* rec, int nrec, int nslot, int Epf, const int* pf_j, int rows, int nnz, int* row_ptr, int* col_idx) {
  export_structure_kernel<<<(nrec + 255) / 256 + (nrec == 0), 256, 0, st>>>(rec, nrec, nslot, Epf, pf_j, rows, nnz, row_ptr, col_idx);
  return cudaGetLastError();
}
cudaError_t launch_sumsq(cudaStream_t st, const double* x, long long lo, long long hi, double* part, double* out) {
  if (hi < lo) hi = lo;
  sumsq_part_kernel<<<kExportRedBlocks, kRedThreads, 0, st>>>(x, lo, hi, part);
  sumsq_final_kernel<<<1, kRedThreads, 0, st>>>(part, kExportRedBlocks, out);
  return cudaGetLastError();
}

}  // namespace pus
