// Host run of the point-cloud evaluation steps (hold_b200/csrc/pointcloud_phases.h) as the kernels of pointcloud.cuh run
// them: the top-K scan in candidate order, the ICP correspondence search, the 3x3 SVD, Umeyama and the ICP bookkeeping.
#include <limits.h>
#include <math.h>

#include "../../hold_b200/csrc/pointcloud_phases.h"

using namespace hold::pc;

template <int K, typename T>
static void scan(int Q, int P, const T* q, const T* p, int Kout, T bound, int bound_idx, T* d, int* idx) {
  for (int a = 0; a < Q; ++a) {
    TopK<K, T> top;
    top_init(top, bound, bound_idx);
    for (int j = 0; j < P; ++j) consider(top, q[3 * a], q[3 * a + 1], q[3 * a + 2], p[3 * j], p[3 * j + 1], p[3 * j + 2], j);
    for (int k = 0; k < Kout; ++k) d[a * Kout + k] = top.d[k], idx[a * Kout + k] = top.i[k];
  }
}

// knn_points' scan: K best of p [P,3] for each q [Q,3]; slots past P keep (inf, INT_MAX)
extern "C" int topk_host(int Q, int P, const float* q, const float* p, int K, float* d, int* idx) {
  if (K == 1) scan<1, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else if (K <= 2) scan<2, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else if (K <= 4) scan<4, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else if (K <= 8) scan<8, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else if (K <= 16) scan<16, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else if (K <= 32) scan<32, float>(Q, P, q, p, K, INFINITY, INT_MAX, d, idx);
  else return -1;
  return 0;
}

// the ICP correspondence: nearest in double with d^2 < max_d2, else index -1
extern "C" void corr_host(int Q, int P, const double* q, const double* p, double max_d2, double* d, int* idx) {
  scan<1, double>(Q, P, q, p, 1, max_d2, -1, d, idx);
}

extern "C" void svd3_host(const double* A, double* U, double* sv, double* V) { svd3(A, U, sv, V); }

// two-pass moments of m correspondences, then the update as a row-major 3x4
extern "C" void umeyama_host(int m, const double* src, const double* dst, int with_scaling, double* T) {
  double ss[3] = {0, 0, 0}, sd[3] = {0, 0, 0};
  for (int i = 0; i < m; ++i)
    for (int k = 0; k < 3; ++k) ss[k] += src[3 * i + k], sd[k] += dst[3 * i + k];
  Moments mo;
  moments_means((double)m, ss, sd, mo);
  double sums[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, t[10];
  for (int i = 0; i < m; ++i) {
    moments_terms(src + 3 * i, dst + 3 * i, mo, t);
    for (int k = 0; k < 10; ++k) sums[k] += t[k];
  }
  moments_cov(sums, mo);
  umeyama(mo, with_scaling != 0, T);
}

extern "C" void compose_host(const double* upd, double* T) { compose(upd, T); }
extern "C" void apply_host(const double* T, double* x) { apply3x4(T, x); }
extern "C" void fitness_rmse_host(double n_corr, double err2, double n_source, double* out) { fitness_rmse(n_corr, err2, n_source, out, out + 1); }
extern "C" int converged_host(double f0, double r0, double f1, double r1, double rf, double rr) { return converged(f0, r0, f1, r1, rf, rr); }
