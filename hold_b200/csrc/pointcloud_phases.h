// Point-cloud evaluation arithmetic (utils/eval_modules.py: pytorch3d's chamfer_distance / knn_points and open3d's
// point-to-point ICP), as __host__ __device__ steps that the kernels of pointcloud.cuh run and tests/test_cpu_pointcloud.py
// runs on the host against oracle/pointcloud_oracle.py.  pytorch3d v0.7.4 and open3d are not in the tree: their rules are
// restated here, unpinned, and in the oracle; the two files change together (DESIGN.md row 4d).
//
//  - distance: knnc::exact_dist, ((dx*dx + dy*dy) + dz*dz) without FMA contraction, in float (knn_points) or double (ICP);
//  - top-K: knnc::TopK / knnc::insert, the K best in lexicographic (distance, index) order;
//  - Umeyama (Eigen::umeyama, as open3d's TransformationEstimationPointToPoint calls it): means, then the demeaned
//    cross-covariance Sigma = (1/m) sum (d - mu_d)(s - mu_s)^T and the source variance; Sigma = U diag(sv) V^T by one-sided
//    Jacobi in double (fixed sweep count, singular values descending); S = diag(1, 1, -1) when det U det V < 0, else I;
//    R = U S V^T, c = tr(diag(sv) S) / var_s with scaling, else 1; t = mu_d - c R mu_s.  No correspondence: the identity;
//  - ICP bookkeeping (open3d's RegistrationICP): fitness = n_corr / n_source, inlier_rmse = sqrt(sum d^2 / n_corr) (0 without
//    correspondences); stop once |d fitness| < relative_fitness and |d rmse| < relative_rmse.
#pragma once
#include <math.h>

#include "knn_phases.h"

namespace hold {
namespace pc {

using knnc::exact_dist;
using knnc::insert;
using knnc::TopK;

// All K slots empty: a candidate enters when (d, j) < (bound, bound_idx).  knn_points: (+inf, INT_MAX); the ICP search:
// (max_corr^2, -1), so only d^2 < max_corr^2 (strict, as nanoflann's radius result set) can enter.
template <int K, typename T>
HOLD_HD void top_init(TopK<K, T>& r, T bound, int bound_idx) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int k = 0; k < K; ++k) r.d[k] = bound, r.i[k] = bound_idx;
}
// candidate j at (x, y, z) for the query (px, py, pz)
template <int K, typename T>
HOLD_HD void consider(TopK<K, T>& r, T px, T py, T pz, T x, T y, T z, int j) {
  const T d = exact_dist(x, y, z, px, py, pz);
  if (d < r.d[K - 1] || (d == r.d[K - 1] && j < r.i[K - 1])) insert(r, d, j);
}

// ---- 3x3 SVD and Umeyama, double

HOLD_HD double det3(const double* a) {   // row-major
  return a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
}

constexpr int kJacobiSweeps = 10;   // one-sided Jacobi converges quadratically; a 3x3 needs 4-6 sweeps, later ones are no-ops

// A = U diag(sv) V^T (row-major 3x3), sv descending and >= 0, U and V orthogonal.  One-sided Jacobi on the columns of A,
// then U = the normalised columns; a column whose singular value is (numerically) zero is completed to an orthonormal U
// (u2 by Gram-Schmidt against an axis when a2 vanishes, u3 = +-(u1 x u2)), which any SVD of a rank-deficient A may do.
HOLD_HD void svd3(const double* A, double* U, double* sv, double* V) {
  double a[3][3], v[3][3];   // a[c] = column c of A, v[c] = column c of V
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) a[c][r] = A[r * 3 + c], v[c][r] = r == c ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep)
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double al = 0.0, be = 0.0, ga = 0.0;
      for (int r = 0; r < 3; ++r) al += a[p][r] * a[p][r], be += a[q][r] * a[q][r], ga += a[p][r] * a[q][r];
      if (!(fabs(ga) > 1e-17 * sqrt(al * be))) continue;   // orthogonal to working precision (or a zero column)
      const double ze = (be - al) / (2.0 * ga);
      const double t = (ze >= 0.0 ? 1.0 : -1.0) / (fabs(ze) + sqrt(1.0 + ze * ze));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
      for (int r = 0; r < 3; ++r) {
        const double x = a[p][r], y = a[q][r];
        a[p][r] = c * x - s * y, a[q][r] = s * x + c * y;
        const double vx = v[p][r], vy = v[q][r];
        v[p][r] = c * vx - s * vy, v[q][r] = s * vx + c * vy;
      }
    }
  double n[3];
  int o[3] = {0, 1, 2};
  for (int c = 0; c < 3; ++c) n[c] = sqrt(a[c][0] * a[c][0] + a[c][1] * a[c][1] + a[c][2] * a[c][2]);
  for (int x = 0; x < 2; ++x)   // descending, stable
    for (int y = 0; y < 2 - x; ++y)
      if (n[o[y]] < n[o[y + 1]]) { const int t = o[y]; o[y] = o[y + 1]; o[y + 1] = t; }
  double u[3][3];
  const double tiny = 1e-300;
  // u1
  if (n[o[0]] > tiny) for (int r = 0; r < 3; ++r) u[0][r] = a[o[0]][r] / n[o[0]];
  else u[0][0] = 1.0, u[0][1] = 0.0, u[0][2] = 0.0;
  // u2: the second column made orthogonal to u1; an axis when it vanishes
  double w[3], pr = 0.0;
  for (int r = 0; r < 3; ++r) w[r] = a[o[1]][r], pr += w[r] * u[0][r];
  for (int r = 0; r < 3; ++r) w[r] -= pr * u[0][r];
  double wn = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(wn > 1e-15 * n[o[0]] && wn > tiny)) {
    int k = 0;
    for (int r = 1; r < 3; ++r)
      if (fabs(u[0][r]) < fabs(u[0][k])) k = r;
    pr = u[0][k];
    for (int r = 0; r < 3; ++r) w[r] = (r == k ? 1.0 : 0.0) - pr * u[0][r];
    wn = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  }
  for (int r = 0; r < 3; ++r) u[1][r] = w[r] / wn;
  // u3 = +-(u1 x u2), the sign that makes a3 . u3 >= 0
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  const double s3 = a[o[2]][0] * u[2][0] + a[o[2]][1] * u[2][1] + a[o[2]][2] * u[2][2];
  if (s3 < 0.0) u[2][0] = -u[2][0], u[2][1] = -u[2][1], u[2][2] = -u[2][2];
  for (int c = 0; c < 3; ++c) {
    sv[c] = n[o[c]];
    for (int r = 0; r < 3; ++r) U[r * 3 + c] = u[c][r], V[r * 3 + c] = v[o[c]][r];
  }
}

// Moments of the m correspondences (source s, destination d): sum_s, sum_d (first pass) and, around the means, the
// cross-covariance sum  sum (d - mu_d)(s - mu_s)^T (row-major) and sum |s - mu_s|^2 (second pass).
struct Moments {
  double m;          // number of correspondences
  double mu_s[3], mu_d[3];
  double sig[9];     // (1/m) sum (d - mu_d)(s - mu_s)^T
  double var_s;      // (1/m) sum |s - mu_s|^2
};

// first pass: m, sum_s, sum_d -> the means (Eigen scales by 1/m)
HOLD_HD void moments_means(double m, const double* sum_s, const double* sum_d, Moments& mo) {
  mo.m = m;
  const double inv = m > 0.0 ? 1.0 / m : 0.0;
  for (int k = 0; k < 3; ++k) mo.mu_s[k] = sum_s[k] * inv, mo.mu_d[k] = sum_d[k] * inv;
}
// second pass, one correspondence: its 9 cross-covariance terms (row-major) and |s - mu_s|^2
HOLD_HD void moments_terms(const double* s, const double* d, const Moments& mo, double* out /*[10]*/) {
  const double ds[3] = {s[0] - mo.mu_s[0], s[1] - mo.mu_s[1], s[2] - mo.mu_s[2]};
  const double dd[3] = {d[0] - mo.mu_d[0], d[1] - mo.mu_d[1], d[2] - mo.mu_d[2]};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) out[r * 3 + c] = dd[r] * ds[c];
  out[9] = ds[0] * ds[0] + ds[1] * ds[1] + ds[2] * ds[2];
}
// second pass: the sums of moments_terms -> Sigma and var_s
HOLD_HD void moments_cov(const double* sums /*[10]*/, Moments& mo) {
  const double inv = mo.m > 0.0 ? 1.0 / mo.m : 0.0;
  for (int k = 0; k < 9; ++k) mo.sig[k] = sums[k] * inv;
  mo.var_s = sums[9] * inv;
}

// The update [c R | t] as a row-major 3x4 from the moments (Eigen::umeyama).  m = 0: the identity.
HOLD_HD void umeyama(const Moments& mo, bool with_scaling, double* Tout /*[12]*/) {
  for (int k = 0; k < 12; ++k) Tout[k] = (k % 5 == 0) ? 1.0 : 0.0;
  if (!(mo.m > 0.0)) return;
  double U[9], sv[3], V[9];
  svd3(mo.sig, U, sv, V);
  const double S3 = det3(U) * det3(V) < 0.0 ? -1.0 : 1.0;
  double R[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = U[r * 3 + 0] * V[c * 3 + 0] + U[r * 3 + 1] * V[c * 3 + 1] + S3 * U[r * 3 + 2] * V[c * 3 + 2];
  const double c = with_scaling ? (sv[0] + sv[1] + S3 * sv[2]) / mo.var_s : 1.0;
  for (int r = 0; r < 3; ++r) {
    const double rs = R[r * 3] * mo.mu_s[0] + R[r * 3 + 1] * mo.mu_s[1] + R[r * 3 + 2] * mo.mu_s[2];
    Tout[r * 4 + 3] = mo.mu_d[r] - c * rs;
    for (int k = 0; k < 3; ++k) Tout[r * 4 + k] = c * R[r * 3 + k];
  }
}

// x <- T x for a row-major 3x4 (or the top of a 4x4) transform
HOLD_HD void apply3x4(const double* T, double* x) {
  const double y0 = T[0] * x[0] + T[1] * x[1] + T[2] * x[2] + T[3];
  const double y1 = T[4] * x[0] + T[5] * x[1] + T[6] * x[2] + T[7];
  const double y2 = T[8] * x[0] + T[9] * x[1] + T[10] * x[2] + T[11];
  x[0] = y0, x[1] = y1, x[2] = y2;
}
// T (4x4, row-major) <- [upd; 0 0 0 1] * T
HOLD_HD void compose(const double* upd, double* T) {
  double o[12];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      o[r * 4 + c] = upd[r * 4] * T[c] + upd[r * 4 + 1] * T[4 + c] + upd[r * 4 + 2] * T[8 + c] + upd[r * 4 + 3] * T[12 + c];
  for (int k = 0; k < 12; ++k) T[k] = o[k];
}

// ---- ICP bookkeeping (open3d RegistrationICP / GetRegistrationResultAndCorrespondences)

HOLD_HD void fitness_rmse(double n_corr, double err2, double n_source, double* fitness, double* rmse) {
  if (n_corr > 0.0) *fitness = n_corr / n_source, *rmse = sqrt(err2 / n_corr);
  else *fitness = 0.0, *rmse = 0.0;
}
HOLD_HD bool converged(double fit0, double rmse0, double fit1, double rmse1, double rel_fitness, double rel_rmse) {
  return fabs(fit0 - fit1) < rel_fitness && fabs(rmse0 - rmse1) < rel_rmse;
}

}  // namespace pc
}  // namespace hold
