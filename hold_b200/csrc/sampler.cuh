// ErrorBoundSampler.get_z_vals (engine/ray_sampler.py:128-352, VolSDF Algorithm 1) as device-driven rounds:
// one warp per ray, the ray's <=640 (z, sdf) pairs in shared memory, warp-shuffle scans for the cumsums,
// the batch-global convergence test `beta.max() > beta0` (:244) as an atomicMax + a 1-thread gate kernel —
// the host never synchronises.
#pragma once
#include "common.cuh"

namespace hold {

struct SamplerArgs {
  int R, rays_per_frame;
  int n_eval, n_samples, n_extra, beta_iters, max_iters;
  float eps, add_tiny, near, r_sphere, beta_min;
  const float* cam;
  const float* dirs;
  const float* beta_param;
  float* z;       // [R, kMaxZ] merged, sorted
  float* sdf;     // [R, kMaxZ]
  float* znew;    // [R, n_eval] samples of the current round (round 0: the uniform set)
  float* sdfnew;  // [R, n_eval]
  float* beta;    // [R]
  float* far;     // [R]
  SamplerState* st;
  int* err;
  // training-mode randomness (NULL in eval)
  const float* jitter;
  const float* u_rand;
  const int* extra_idx;  // [max_iters, n_extra]: row (rounds - 1) is used
  float* z_out;  // [R, n_samples + n_extra + 2]
  int* iters_out;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// exclusive scan of one value per lane.  (Not inclusive - v: the last sample's free energy is 1e10 * sigma, and
// subtracting it back would cancel the whole prefix.)
__device__ __forceinline__ float warp_excl_scan(float v, int lane) {
  float x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  float e = __shfl_up_sync(0xffffffffu, x, 1);
  return lane == 0 ? 0.f : e;
}

// The reference's cumsums run on torch tensors whose CPU kernel accumulates in double and rounds every output to float
// (at::acc_type<float, false>); a CUDA scan accumulates in float.  Either way each prefix is within an ulp of the exact sum.
// The kernels here keep the TERMS in float (as the reference does) and accumulate the prefixes in double: the inverse-CDF step
// thresholds cdf[i+1] - cdf[i] at 1e-5 (ray_sampler.py:304), and in empty space that difference is 1e-5 / (1 + 639e-5) =
// 0.994e-5 — one float ulp of a two-level float scan is enough to flip the branch (with float prefixes a share of the final samples
// moves by up to a bin width, tests/test_gpu_sampler_rounds.py).
__device__ __forceinline__ double warp_excl_scan_d(double v, int lane) {
  double x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    double y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  double e = __shfl_up_sync(0xffffffffu, x, 1);
  return lane == 0 ? 0.0 : e;
}

__device__ __forceinline__ float expf_cr(float x) { return (float)exp((double)x); }

// in-place bitonic sort (ascending) of n = power of two floats in shared memory by one warp, with payload
__device__ __forceinline__ void warp_bitonic(float* key, float* val, int n, int lane) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n; i += 32) {
        int ixj = i ^ j;
        if (ixj > i) {
          bool up = ((i & k) == 0);
          float a = key[i], b = key[ixj];
          if ((a > b) == up) {
            key[i] = b, key[ixj] = a;
            if (val != nullptr) { float t = val[i]; val[i] = val[ixj]; val[ixj] = t; }
          }
        }
      }
      __syncwarp();
    }
  }
}

// get_sphere_intersections (ray_sampler.py:6-25) far root + UniformSampler.get_z_vals (:54-80) + Lemma-2 beta (:149-155)
__global__ void __launch_bounds__(128) k_sampler_init(SamplerArgs a) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.st->iters = 0;
    a.st->done = 0;
    for (int i = 0; i < 8; ++i) a.st->beta_max_bits[i] = 0u;
  }
  if (warp >= a.R) return;
  const int r = warp;
  float cx = a.cam[3 * r], cy = a.cam[3 * r + 1], cz = a.cam[3 * r + 2];
  float dx = a.dirs[3 * r], dy = a.dirs[3 * r + 1], dz = a.dirs[3 * r + 2];
  float bdot = dx * cx + dy * cy + dz * cz;
  float cn = sqrtf(cx * cx + cy * cy + cz * cz);
  float under = bdot * bdot - (cn * cn - a.r_sphere * a.r_sphere);
  if (under <= 0.f) {
    if (lane == 0) atomicOr(a.err, kErrRayMiss);
    under = 0.f;
  }
  float far = fmaxf(sqrtf(under) - bdot, 0.f);
  if (lane == 0) a.far[r] = far;
  const int Ne = a.n_eval;
  float sumsq = 0.f;
  // z_k = near*(1-t_k) + far*t_k, t = linspace(0,1,Ne); optional stratified jitter
  for (int k = lane; k < Ne; k += 32)
    a.znew[(size_t)r * Ne + k] = stratified_z(a.near, far, Ne, k, a.jitter ? a.jitter + (size_t)r * Ne + k : nullptr);
  __syncwarp();
  for (int k = lane; k + 1 < Ne; k += 32) {
    float d = a.znew[(size_t)r * Ne + k + 1] - a.znew[(size_t)r * Ne + k];
    sumsq += d * d;
  }
  sumsq = warp_sum(sumsq);
  if (lane == 0) {
    float bound = (1.0f / (4.0f * logf(a.eps + 1.0f))) * sumsq;
    a.beta[r] = sqrtf(bound);
  }
}

// 1 thread: is round `it` still part of the while loop (ray_sampler.py:160)?  Runs before the round's kernels.
__global__ void k_round_gate(SamplerState* st, int it, const float* beta_param, float beta_min, int max_iters) {
  float beta0 = fabsf(beta_param[0]) + beta_min;
  bool active = true;
  for (int j = 0; j < it; ++j) {
    float bm = __uint_as_float(st->beta_max_bits[j]);
    bool upsample = (bm > beta0) && (j + 1 < max_iters);
    if (!upsample) active = false;
  }
  st->done = active ? 0 : 1;
}

struct RaySmem {
  float* z;
  float* s;
  float* dstar;
  float* delta;
  float* t0;
  float* t1;
};

// `cap` = elements per array for THIS launch (sampler_cap(): round `it` holds (it + 1) n_eval samples, not kMaxZ): six arrays of kMaxZ
// floats per ray allowed 3 blocks = 12 warps per SM (ncu: 18 % of the warp slots, `wait` / short-scoreboard stalls unhidden).
__device__ __forceinline__ RaySmem ray_smem(float* base, int warp_in_block, int cap) {
  RaySmem m;
  float* p = base + (size_t)warp_in_block * 6 * cap;
  m.z = p, m.s = p + cap, m.dstar = p + 2 * cap, m.delta = p + 3 * cap, m.t0 = p + 4 * cap, m.t1 = p + 5 * cap;
  return m;
}
// capacity the two round kernels need at round `it`: the merged buffer, the power-of-two padded new samples (bitonic sort) and the
// power-of-two padded final set
static inline int sampler_cap(int it, int n_eval, int n_final) {
  int np2 = 1, sp2 = 1;
  while (np2 < n_eval) np2 <<= 1;
  while (sp2 < n_final) sp2 <<= 1;
  int cap = (it + 1) * n_eval;
  if (cap < np2) cap = np2;
  if (cap < sp2) cap = sp2;
  return (cap + 31) & ~31;
}

// Theorem-1 bound d* per interval (ray_sampler.py:191-206)
__device__ __forceinline__ void compute_dstar(const RaySmem& m, int n, int lane) {
  for (int i = lane; i < n - 1; i += 32) {
    float a = m.z[i + 1] - m.z[i];
    float b = fabsf(m.s[i]), c = fabsf(m.s[i + 1]);
    bool first = a * a + b * b <= c * c;
    bool second = a * a + c * c <= b * b;
    float d = 0.f;
    if (first) d = b;
    if (second) d = c;
    float sp = (a + b + c) / 2.0f;
    float area = sp * (sp - a) * (sp - b) * (sp - c);
    if (!first && !second && (b + c - a > 0.f)) d = (2.0f * sqrtf(area)) / a;
    float s0 = m.s[i], s1 = m.s[i + 1];
    float sg0 = (s0 > 0.f) ? 1.f : ((s0 < 0.f) ? -1.f : 0.f), sg1 = (s1 > 0.f) ? 1.f : ((s1 < 0.f) ? -1.f : 0.f);
    m.dstar[i] = (sg0 * sg1 == 1.f) ? d : 0.f;
    m.delta[i] = a;
  }
  __syncwarp();
}

// get_error_bound (ray_sampler.py:354-366) for one ray held by one warp; lanes own contiguous segments.
__device__ __forceinline__ float error_bound(const RaySmem& m, int n, float beta, int lane) {
  const int nb = n - 1;
  const int seg = (nb + 31) / 32;
  const int lo = min(lane * seg, nb), hi = min(lo + seg, nb);
  double accI = 0.0, accE = 0.0;
  const float inv4b2 = 4.0f * beta * beta;
  for (int i = lo; i < hi; ++i) {
    const float d = m.delta[i];
    const float fe = d * laplace_density(m.s[i], beta);              // free energy of interval i (contributes to I_{i+1})
    const float es = expf(-m.dstar[i] / beta) * (d * d) / inv4b2;
    m.t0[i] = fe, m.t1[i] = es;                                      // float terms, double prefixes
    accI += (double)fe, accE += (double)es;
  }
  double runI = warp_excl_scan_d(accI, lane), runE = warp_excl_scan_d(accE, lane);
  float best = -INFINITY;
  for (int i = lo; i < hi; ++i) {
    const float Iex = (float)runI;   // exclusive: sum_{j<i} delta_j sigma_j
    runI += (double)m.t0[i];
    runE += (double)m.t1[i];
    const float Ein = (float)runE;
    const float bo = (fminf(expf(Ein), 1.0e6f) - 1.0f) * expf(-Iex);
    best = fmaxf(best, bo);
  }
  return warp_max(best);
}

// Round part A: merge the round's new (z, sdf) into the sorted buffers, d*, beta line search (:179-220),
// contribute to the batch-global max.
__global__ void __launch_bounds__(128) k_sampler_merge_beta(SamplerArgs a, int it, int cap) {
  if (a.st->done) return;
  extern __shared__ float smem[];
  const int wib = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int r = blockIdx.x * (blockDim.x / 32) + wib;
  if (r >= a.R) return;
  RaySmem m = ray_smem(smem, wib, cap);
  const int Ne = a.n_eval, n_old = it * Ne, n = n_old + Ne;
  // new samples -> t0/t1 (sorted by z; the inverse-CDF output is monotone up to rounding, sort keeps
  // torch.sort's multiset semantics); Ne is padded to a power of two with +inf
  int np2 = 1;
  while (np2 < Ne) np2 <<= 1;
  for (int k = lane; k < np2; k += 32) {
    m.t0[k] = (k < Ne) ? a.znew[(size_t)r * Ne + k] : INFINITY;
    m.t1[k] = (k < Ne) ? a.sdfnew[(size_t)r * Ne + k] : 0.f;
  }
  for (int k = lane; k < n_old; k += 32) {
    m.dstar[k] = a.z[(size_t)r * kMaxZ + k];  // old z (staging)
    m.delta[k] = a.sdf[(size_t)r * kMaxZ + k];
  }
  __syncwarp();
  warp_bitonic(m.t0, m.t1, np2, lane);
  // stable parallel merge: old entries first on ties
  for (int i = lane; i < n_old; i += 32) {
    float key = m.dstar[i];
    int lo = 0, hi = Ne;  // # new strictly less than key
    while (lo < hi) { int mid = (lo + hi) >> 1; if (m.t0[mid] < key) lo = mid + 1; else hi = mid; }
    m.z[i + lo] = key, m.s[i + lo] = m.delta[i];
  }
  for (int j = lane; j < Ne; j += 32) {
    float key = m.t0[j];
    int lo = 0, hi = n_old;  // # old less-or-equal key
    while (lo < hi) { int mid = (lo + hi) >> 1; if (m.dstar[mid] <= key) lo = mid + 1; else hi = mid; }
    m.z[j + lo] = key, m.s[j + lo] = m.t1[j];
  }
  __syncwarp();
  for (int k = lane; k < n; k += 32) {
    a.z[(size_t)r * kMaxZ + k] = m.z[k];
    a.sdf[(size_t)r * kMaxZ + k] = m.s[k];
  }
  compute_dstar(m, n, lane);
  const float beta0 = fabsf(a.beta_param[0]) + a.beta_min;
  float beta = a.beta[r];
  float e0 = error_bound(m, n, beta0, lane);
  if (e0 <= a.eps) beta = beta0;
  float bmin = beta0, bmax = beta;
  // A ray whose bound already holds at beta0 keeps beta0 through the line search (mid == beta0 every step), so
  // the 10 extra evaluations are skipped for it — the result is bit-identical (ray_sampler.py:211-219).
  const int n_bis = (e0 <= a.eps) ? 0 : a.beta_iters;
  for (int j = 0; j < n_bis; ++j) {
    float mid = (bmin + bmax) / 2.0f;
    float e = error_bound(m, n, mid, lane);
    if (e <= a.eps) bmax = mid;
    if (e > a.eps) bmin = mid;
  }
  if (lane == 0) {
    a.beta[r] = bmax;
    atomicMax(&a.st->beta_max_bits[it], __float_as_uint(fmaxf(bmax, 0.f)));
  }
}

// Round part B: opacity / error-bound PDF -> inverse-CDF samples (:223-307); either the next round's Ne new
// samples or the final set (N from the weight CDF + near + far + strided extras, sorted; :313-336).
__global__ void __launch_bounds__(128) k_sampler_resample(SamplerArgs a, int it, int cap) {
  if (a.st->done) return;
  extern __shared__ float smem[];
  const int wib = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int r = blockIdx.x * (blockDim.x / 32) + wib;
  const float beta0 = fabsf(a.beta_param[0]) + a.beta_min;
  const float bmaxg = __uint_as_float(a.st->beta_max_bits[it]);
  const bool upsample = (bmaxg > beta0) && (it + 1 < a.max_iters);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.st->iters = it + 1;
    if (a.iters_out != nullptr) a.iters_out[0] = it + 1;
  }
  if (r >= a.R) return;
  RaySmem m = ray_smem(smem, wib, cap);
  const int Ne = a.n_eval, n = (it + 1) * Ne;
  for (int k = lane; k < n; k += 32) {
    m.z[k] = a.z[(size_t)r * kMaxZ + k];
    m.s[k] = a.sdf[(size_t)r * kMaxZ + k];
  }
  __syncwarp();
  compute_dstar(m, n, lane);
  const float beta = a.beta[r];
  // lane-segment scans over the n samples: free energy (exclusive -> transmittance) and, when upsampling,
  // the error integral (inclusive) over the n-1 intervals.  Float terms, double prefixes (see warp_excl_scan_d).
  const int seg = (n + 31) / 32;
  const int lo = min(lane * seg, n), hi = min(lo + seg, n);
  double accF = 0.0, accE = 0.0;
  const float inv4b2 = 4.0f * beta * beta;
  for (int i = lo; i < hi; ++i) {
    const float d = (i < n - 1) ? m.delta[i] : 1.0e10f;
    const float fe = d * laplace_density(m.s[i], beta);
    accF += (double)fe;
    if (i < n - 1) {
      const float es = expf(-m.dstar[i] / beta) * (d * d) / inv4b2;
      accE += (double)es;
      m.t1[i] = es;
    }
    m.delta[i] = fe;   // reuse: free energy
  }
  double runF = warp_excl_scan_d(accF, lane), runE = warp_excl_scan_d(accE, lane);
  double psum = 0.0;
  for (int i = lo; i < hi; ++i) {
    if (i < n - 1) {
      const float T = expf(-(float)runF);      // exclusive prefix of the free energy
      runE += (double)m.t1[i];
      float pdf;
      // exp(E) - 1 and 1 - exp(-fe) cancel to a few ulps of 1 where E resp. fe are tiny (empty space), and those ulps ARE the pdf
      // there (floor 1e-6 / 1e-5): the inverse CDF integrates them over hundreds of bins.  expf_cr is the correctly rounded float
      // exponential (what a <= 1 ulp libm such as the reference's returns almost always); CUDA's expf (2 ulp) measurably moved
      // 1.8 % of the final samples beyond 1e-4 R_s of the exact answer against the reference's own 0.2 % (teacher-forced test).
      if (upsample) pdf = (fminf(expf_cr((float)runE), 1.0e6f) - 1.0f) * T + a.add_tiny;
      else pdf = (1.0f - expf_cr(-m.delta[i])) * T + 1e-5f;
      m.dstar[i] = pdf;
      psum += (double)pdf;
    }
    runF += (double)m.delta[i];
  }
  // pdf.sum(-1): float result of a double accumulation
  double tot_d = psum;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot_d += __shfl_xor_sync(0xffffffffu, tot_d, o);
  const float total = (float)tot_d;
  // cdf[0] = 0, cdf[i+1] = cumsum(pdf/total) -> stored in t0[0..n)
  double accC = 0.0;
  const int nb = n - 1;
  const int segb = (nb + 31) / 32;
  const int lob = min(lane * segb, nb), hib = min(lob + segb, nb);
  __syncwarp();
  for (int i = lob; i < hib; ++i) {
    const float pn = m.dstar[i] / total;
    m.t1[i] = pn;
    accC += (double)pn;
  }
  double runC = warp_excl_scan_d(accC, lane);
  __syncwarp();
  for (int i = lob; i < hib; ++i) {
    runC += (double)m.t1[i];
    m.t0[i + 1] = (float)runC;
  }
  if (lane == 0) m.t0[0] = 0.f;
  __syncwarp();
  const float* cdf = m.t0;
  const int N = upsample ? Ne : a.n_samples;
  const bool rand_u = (!upsample) && (a.u_rand != nullptr);
  // samples -> m.s (reused; sdf no longer needed), then emitted
  float* out = m.s;
  for (int k = lane; k < N; k += 32) {
    float u = rand_u ? a.u_rand[(size_t)r * N + k] : torch_linspace(0.f, 1.f, N, k);
    int l = 0, h = n;  // searchsorted(right=True): first idx with cdf[idx] > u
    while (l < h) { int mid = (l + h) >> 1; if (cdf[mid] <= u) l = mid + 1; else h = mid; }
    int below = max(l - 1, 0), above = min(l, n - 1);
    float c0 = cdf[below], c1 = cdf[above], b0 = m.z[below], b1 = m.z[above];
    float den = c1 - c0;
    if (den < 1e-5f) den = 1.0f;
    float t = (u - c0) / den;
    out[k] = b0 + t * (b1 - b0);
  }
  __syncwarp();
  if (upsample) {
    for (int k = lane; k < Ne; k += 32) a.znew[(size_t)r * Ne + k] = out[k];
    return;
  }
  // final set: [samples(N), near, far, z[extra idx] (Nx)] sorted
  const int Nx = a.n_extra, S = N + Nx + 2;
  if (lane == 0) { out[N] = a.near; out[N + 1] = a.far[r]; }
  for (int k = lane; k < Nx; k += 32) {
    int idx = (a.extra_idx != nullptr) ? min(max(a.extra_idx[it * Nx + k], 0), n - 1) : (int)torch_linspace(0.f, (float)(n - 1), Nx, k);
    out[N + 2 + k] = m.z[idx];
  }
  int sp2 = 1;
  while (sp2 < S) sp2 <<= 1;
  for (int k = S + lane; k < sp2; k += 32) out[k] = INFINITY;
  __syncwarp();
  warp_bitonic(out, nullptr, sp2, lane);
  for (int k = lane; k < S; k += 32) a.z_out[(size_t)r * S + k] = out[k];
}

}  // namespace hold
