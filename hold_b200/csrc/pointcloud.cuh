// Kernels of the point-cloud evaluation (utils/eval_modules.py): exact K-nearest neighbours (hold_knn_points) and
// open3d's point-to-point ICP (hold_icp); arithmetic in pointcloud_phases.h.
//
// Both searches are brute force with nothing of size P1 x P2: one query point per thread, its K best kept in registers
// (knnc::TopK, templated on K and on the scalar type), the CTA staging kPcThreads candidates at a time in shared memory; a
// candidate is rejected against the current K-th (distance, index) before it touches the list.
//
// ICP runs N independent (source, target) pairs with no host synchronisation: every one of max_iteration iterations is
// enqueued (4 launches each), and a pair that has converged turns them into no-ops through its `done` flag, as the sampler
// rounds do (DESIGN.md §3.2), so the call can be captured in a CUDA graph.  Every sum over correspondences is a per-CTA
// shuffle tree, then the CTAs' partials added in CTA order by one thread: bitwise reproducible, and a pair's bits do not
// depend on the other pairs of the batch.
//
// The K-NN backward (hold_knn_points_bwd) adds in a fixed order with no atomic: a query's gradient sums its slots in k order,
// and a target's gradient sums the slots that chose it in ascending (query, k) order, found through inverse_map.cuh.
#pragma once
#include <limits.h>

#include "common.cuh"
#include "inverse_map.cuh"
#include "pointcloud_phases.h"

namespace hold {

constexpr int kPcThreads = 256;
constexpr int kIcpPart = 10;   // partial sums per CTA: the most any ICP reduction needs (the cross-covariance + var_s)

template <typename T>
struct alignas(4 * sizeof(T)) Pt4 {
  T x, y, z, w;
};

// lengths[n] clamped to [0, P] (NULL: P); a length outside sets kErrBadLength when `report`
__device__ __forceinline__ int pc_length(const int* lengths, int n, int P, int* err, bool report) {
  if (lengths == nullptr) return P;
  const int l = lengths[n];
  if (l >= 0 && l <= P) return l;
  if (report) atomicOr(err, kErrBadLength);
  return l < 0 ? 0 : P;
}

// This CTA's queries (one per thread, searching when `live`) against the candidates [0, L2) of p2 (one batch element's
// [P2,3] fp32, converted to T as staged).  Every thread of the CTA calls it: it synchronises the CTA.
template <int K, typename T>
__device__ __forceinline__ void cta_scan(pc::TopK<K, T>& top, bool live, T px, T py, T pz, const float* __restrict__ p2, int L2,
                                         Pt4<T>* s) {
  for (int j0 = 0; j0 < L2; j0 += kPcThreads) {
    const int j = j0 + threadIdx.x;
    __syncthreads();   // the previous tile is consumed
    if (j < L2) s[threadIdx.x] = Pt4<T>{(T)p2[(size_t)j * 3], (T)p2[(size_t)j * 3 + 1], (T)p2[(size_t)j * 3 + 2], T(0)};
    __syncthreads();
    const int n = min(kPcThreads, L2 - j0);
    if (live) {
#pragma unroll 4
      for (int c = 0; c < n; ++c) {
        const Pt4<T> q = s[c];
        pc::consider(top, px, py, pz, q.x, q.y, q.z, j0 + c);
      }
    }
  }
}

// knn_points: dists / idx [N,P1,Kout] (Kout <= K); padding slots (row >= lengths1[n] or k >= lengths2[n]) hold 0.
template <int K>
__global__ void __launch_bounds__(kPcThreads) k_knn(int N, int P1, const float* __restrict__ p1, const int* __restrict__ len1, int P2,
                                                    const float* __restrict__ p2, const int* __restrict__ len2, int Kout,
                                                    float* __restrict__ dists, int* __restrict__ idx, int* err) {
  __shared__ Pt4<float> s[kPcThreads];
  const bool report = blockIdx.x == 0 && threadIdx.x == 0;
  for (int n = blockIdx.y; n < N; n += gridDim.y) {   // CTA-uniform
    const int L1 = pc_length(len1, n, P1, err, report), L2 = pc_length(len2, n, P2, err, report);
    const int i = blockIdx.x * kPcThreads + threadIdx.x;
    const bool live = i < L1;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (live) {
      const float* q = p1 + ((size_t)n * P1 + i) * 3;
      px = q[0], py = q[1], pz = q[2];
    }
    pc::TopK<K, float> top;
    pc::top_init(top, INFINITY, INT_MAX);
    if ((int)blockIdx.x * kPcThreads < L1) cta_scan(top, live, px, py, pz, p2 + (size_t)n * P2 * 3, L2, s);
    if (i < P1) {
      const size_t o = ((size_t)n * P1 + i) * Kout;
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (k < Kout) {
          const bool v = live && k < L2;
          dists[o + k] = v ? top.d[k] : 0.f;
          idx[o + k] = v ? top.i[k] : 0;
        }
    }
  }
}

// ---- K-NN backward

struct KnnBwdArgs {
  int N, P1, P2, K;
  const float *p1, *p2;
  const int *len1, *len2;
  const int* idx;          // [N,P1,K] from k_knn
  const float* g_dists;    // [N,P1,K]
  const float* g_knn;      // [N,P1,K,3] or NULL
  float *g_p1, *g_p2;      // [N,P1,3], [N,P2,3], overwritten
  float* contrib;          // [N,P1,K,3]: each slot's d loss / d p2 through dists
  int* keys;               // [N,P1,K]: n P2 + idx for a slot that reaches p2, else N P2
  InvMap map;
  int* err;
};

// One thread per query row: g_p1 = sum over the valid slots in k order of 2 (p1 - p2[idx]) g_dists; the slots' keys and p2
// parts.  A slot reaches p2 through dists when it is valid (row < lengths1, k < lengths2), through knn when k < lengths2.
__global__ void __launch_bounds__(kPcThreads) k_knn_bwd_rows(KnnBwdArgs a) {
  const int64_t row = (int64_t)blockIdx.x * kPcThreads + threadIdx.x;
  if (row >= (int64_t)a.N * a.P1) return;
  const int n = (int)(row / a.P1), i = (int)(row % a.P1);
  const bool report = row == 0;
  const int L1 = pc_length(a.len1, n, a.P1, a.err, report), L2 = pc_length(a.len2, n, a.P2, a.err, report);
  const float* q = a.p1 + row * 3;
  float g1[3] = {0.f, 0.f, 0.f};
  for (int k = 0; k < a.K; ++k) {
    const int64_t slot = row * a.K + k;
    const int j = a.idx[slot];
    const bool in = k < L2 && j >= 0 && j < L2, vd = in && i < L1;
    float c[3] = {0.f, 0.f, 0.f};
    if (vd) {
      const float* t = a.p2 + ((size_t)n * a.P2 + j) * 3;
      const float gd = a.g_dists[slot];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const float d = __fmul_rn(2.f * (q[e] - t[e]), gd);
        g1[e] += d;
        c[e] = -d;
      }
    }
    a.keys[slot] = vd || (in && a.g_knn) ? n * a.P2 + j : a.N * a.P2;
#pragma unroll
    for (int e = 0; e < 3; ++e) a.contrib[slot * 3 + e] = c[e];
  }
#pragma unroll
  for (int e = 0; e < 3; ++e) a.g_p1[row * 3 + e] = g1[e];
}

// One thread per target: the slots that chose it, in ascending (query, k) order; the dists part and the knn part are summed
// apart and added last.
__global__ void __launch_bounds__(kPcThreads) k_knn_bwd_targets(KnnBwdArgs a) {
  const int t = blockIdx.x * kPcThreads + threadIdx.x;
  if (t >= a.N * a.P2) return;
  float sd[3] = {0.f, 0.f, 0.f}, sk[3] = {0.f, 0.f, 0.f};
  for (int e = a.map.first[t]; e < a.map.first[t + 1]; ++e) {
    const size_t slot = a.map.order[e];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      sd[c] += a.contrib[slot * 3 + c];
      if (a.g_knn) sk[c] += a.g_knn[slot * 3 + c];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) a.g_p2[(size_t)t * 3 + c] = a.g_knn ? sd[c] + sk[c] : sd[c];
}

// ---- ICP

struct IcpPair {
  double T[16];        // accumulated transformation (row-major 4x4)
  double upd[12];      // the current iteration's update [cR | t]
  pc::Moments mo;      // means from the last correspondence pass, then the cross-covariance
  double fitness, rmse;
  int Ls, Lt;          // clamped lengths
  int done, iters;
};

// sum of v over the CTA (shuffle tree per warp, then the warps in order) -> out[0 .. M)
template <int M>
__device__ __forceinline__ void cta_sum(double (&v)[M], double* __restrict__ out) {
  __shared__ double s[kPcThreads / 32][M];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < M; ++k) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], off);
    if (lane == 0) s[warp][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < M) {
    double t = 0.0;
    for (int w = 0; w < kPcThreads / 32; ++w) t += s[w][threadIdx.x];
    out[threadIdx.x] = t;
  }
}

struct IcpArgs {
  int N, Ps, Pt, nb;               // nb: CTAs per pair over the source points
  const float* src;                // [N,Ps,3]
  const int* src_len;
  const float* tgt;                // [N,Pt,3]
  const int* tgt_len;
  const double* init;              // [N,4,4] or NULL
  double max_d2;                   // correspondences need d^2 < max_d2 (< 0: none)
  double rel_fitness, rel_rmse;
  int with_scaling;
  IcpPair* st;                     // [N]
  double* xs;                      // [N,Ps,3] the transformed source
  int* corr;                       // [N,Ps] target index or -1
  double* part;                    // [N,nb,kIcpPart]
  int* err;
};

// pair state and the source transformed by init (or copied)
__global__ void __launch_bounds__(kPcThreads) k_icp_start(IcpArgs a) {
  const int n = blockIdx.y, i = blockIdx.x * kPcThreads + threadIdx.x;
  const bool report = blockIdx.x == 0 && threadIdx.x == 0;
  const int Ls = pc_length(a.src_len, n, a.Ps, a.err, report), Lt = pc_length(a.tgt_len, n, a.Pt, a.err, report);
  double T[16];
  for (int k = 0; k < 16; ++k) T[k] = a.init ? a.init[(size_t)n * 16 + k] : (k % 5 == 0 ? 1.0 : 0.0);
  if (report) {
    IcpPair& p = a.st[n];
    for (int k = 0; k < 16; ++k) p.T[k] = T[k];
    p.Ls = Ls, p.Lt = Lt, p.done = 0, p.iters = 0, p.fitness = 0.0, p.rmse = 0.0;
  }
  if (i < Ls) {
    const float* q = a.src + ((size_t)n * a.Ps + i) * 3;
    double x[3] = {(double)q[0], (double)q[1], (double)q[2]};
    if (a.init) pc::apply3x4(T, x);
    double* o = a.xs + ((size_t)n * a.Ps + i) * 3;
    o[0] = x[0], o[1] = x[1], o[2] = x[2];
  }
}

// (kApply: the source moved by the pair's update first) the nearest target point of each source point within max_d2;
// partials [count, sum d^2, sum source (3), sum target (3)]
template <bool kApply>
__global__ void __launch_bounds__(kPcThreads) k_icp_corr(IcpArgs a) {
  __shared__ Pt4<double> s[kPcThreads];
  const int n = blockIdx.y, i = blockIdx.x * kPcThreads + threadIdx.x;
  const IcpPair& p = a.st[n];
  if (p.done) return;   // CTA-uniform
  const int Ls = p.Ls, Lt = p.Lt;
  const bool live = i < Ls;
  double x[3] = {0.0, 0.0, 0.0};
  double* xp = a.xs + ((size_t)n * a.Ps + (live ? i : 0)) * 3;
  if (live) {
    x[0] = xp[0], x[1] = xp[1], x[2] = xp[2];
    if (kApply) {
      pc::apply3x4(p.upd, x);
      xp[0] = x[0], xp[1] = x[1], xp[2] = x[2];
    }
  }
  pc::TopK<1, double> top;
  pc::top_init(top, a.max_d2, -1);
  if ((int)blockIdx.x * kPcThreads < Ls) cta_scan(top, live, x[0], x[1], x[2], a.tgt + (size_t)n * a.Pt * 3, Lt, s);
  const bool hit = live && top.i[0] >= 0;
  if (live) a.corr[(size_t)n * a.Ps + i] = hit ? top.i[0] : -1;
  double v[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (hit) {
    const float* t = a.tgt + ((size_t)n * a.Pt + top.i[0]) * 3;
    v[0] = 1.0, v[1] = top.d[0];
    v[2] = x[0], v[3] = x[1], v[4] = x[2], v[5] = (double)t[0], v[6] = (double)t[1], v[7] = (double)t[2];
  }
  cta_sum(v, a.part + ((size_t)n * a.nb + blockIdx.x) * kIcpPart);
}

// one thread per pair: fitness / rmse of the correspondences just found, the convergence test (iteration `it` >= 0) and the
// means for the next update
__global__ void k_icp_eval(IcpArgs a, int it) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  IcpPair& p = a.st[n];
  if (p.done) return;
  double v[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < a.nb; ++b)
    for (int k = 0; k < 8; ++k) v[k] += a.part[((size_t)n * a.nb + b) * kIcpPart + k];
  double fit, rmse;
  pc::fitness_rmse(v[0], v[1], (double)p.Ls, &fit, &rmse);
  if (it >= 0) {
    p.iters = it + 1;
    if (pc::converged(p.fitness, p.rmse, fit, rmse, a.rel_fitness, a.rel_rmse)) p.done = 1;
  }
  p.fitness = fit, p.rmse = rmse;
  pc::moments_means(v[0], v + 2, v + 5, p.mo);
}

// the second Umeyama pass: partials of the demeaned cross-covariance and source variance
__global__ void __launch_bounds__(kPcThreads) k_icp_cov(IcpArgs a) {
  const int n = blockIdx.y, i = blockIdx.x * kPcThreads + threadIdx.x;
  const IcpPair& p = a.st[n];
  if (p.done) return;
  double v[kIcpPart];
#pragma unroll
  for (int k = 0; k < kIcpPart; ++k) v[k] = 0.0;
  const int j = i < p.Ls ? a.corr[(size_t)n * a.Ps + i] : -1;
  if (j >= 0) {
    const double* x = a.xs + ((size_t)n * a.Ps + i) * 3;
    const float* t = a.tgt + ((size_t)n * a.Pt + j) * 3;
    const double s3[3] = {x[0], x[1], x[2]}, d3[3] = {(double)t[0], (double)t[1], (double)t[2]};
    pc::moments_terms(s3, d3, p.mo, v);
  }
  cta_sum(v, a.part + ((size_t)n * a.nb + blockIdx.x) * kIcpPart);
}

// one thread per pair: Umeyama update, T <- update T
__global__ void k_icp_update(IcpArgs a) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  IcpPair& p = a.st[n];
  if (p.done) return;
  double v[kIcpPart];
  for (int k = 0; k < kIcpPart; ++k) v[k] = 0.0;
  for (int b = 0; b < a.nb; ++b)
    for (int k = 0; k < kIcpPart; ++k) v[k] += a.part[((size_t)n * a.nb + b) * kIcpPart + k];
  pc::moments_cov(v, p.mo);
  pc::umeyama(p.mo, a.with_scaling != 0, p.upd);
  pc::compose(p.upd, p.T);
}

__global__ void k_icp_out(IcpArgs a, double* __restrict__ transformation, double* __restrict__ fitness, double* __restrict__ rmse,
                          int* __restrict__ iterations) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  const IcpPair& p = a.st[n];
  for (int k = 0; k < 16; ++k) transformation[(size_t)n * 16 + k] = p.T[k];
  fitness[n] = p.fitness, rmse[n] = p.rmse, iterations[n] = p.iters;
}

}  // namespace hold
