// popup_noise.hpp -- isam::Covariance / Information -> upper-triangular sqrt-information (ISAM/include/isam/Noise.h:36-62),
// shared by the isam facade (isam_facade.hpp) and the plane map (pus_map.cu), so that a graph the map builds and one a
// facade replay builds carry the same bits.
#pragma once
#include <cmath>
#include <stdexcept>
#include <vector>

namespace pus_noise {
// in-place Cholesky A = U^T U of a small SPD matrix; returns U (upper), row-major n x n
inline std::vector<double> chol_upper(std::vector<double> A, int n) {
  std::vector<double> U((size_t)n * n, 0.0);
  for (int i = 0; i < n; i++)
    for (int j = i; j < n; j++) {
      double s = A[(size_t)i * n + j];
      for (int k = 0; k < i; k++) s -= U[(size_t)k * n + i] * U[(size_t)k * n + j];
      if (i == j) { if (!(s > 0)) throw std::runtime_error("Noise: matrix not positive definite"); U[(size_t)i * n + i] = std::sqrt(s); }
      else U[(size_t)i * n + j] = s / U[(size_t)i * n + i];
    }
  return U;
}
inline std::vector<double> inverse_spd(const std::vector<double>& A, int n) {
  std::vector<double> M = A, I((size_t)n * n, 0.0);
  for (int i = 0; i < n; i++) I[(size_t)i * n + i] = 1;
  for (int k = 0; k < n; k++) {
    double p = M[(size_t)k * n + k];
    for (int j = 0; j < n; j++) { M[(size_t)k * n + j] /= p; I[(size_t)k * n + j] /= p; }
    for (int i = 0; i < n; i++) if (i != k) {
      double f = M[(size_t)i * n + k];
      for (int j = 0; j < n; j++) { M[(size_t)i * n + j] -= f * M[(size_t)k * n + j]; I[(size_t)i * n + j] -= f * I[(size_t)k * n + j]; }
    }
  }
  return I;
}
// the upper triangle of U (n x n, row-major), row by row: the C-ABI's sqrt-information layout
inline std::vector<double> pack_upper(const std::vector<double>& U, int n) {
  std::vector<double> p;
  for (int r = 0; r < n; r++)
    for (int c = r; c < n; c++) p.push_back(U[(size_t)r * n + c]);
  return p;
}
// Covariance(sigmas.cwiseProduct(sigmas).asDiagonal()) (Mapping.cpp:66-67, 510-512), packed upper triangle row by row
inline std::vector<double> covariance_diag_packed(const double* sigmas, int n) {
  std::vector<double> cov((size_t)n * n, 0.0);
  for (int i = 0; i < n; i++) cov[(size_t)i * n + i] = sigmas[i] * sigmas[i];
  return pack_upper(chol_upper(inverse_spd(cov, n), n), n);
}
}  // namespace pus_noise
