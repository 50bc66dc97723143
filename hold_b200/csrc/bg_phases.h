// Sample depths along a ray and the NeRF++ background's 32-sample integral with its reverse mode, written as host-executable
// per-sample steps (tests/host/bg_host.cpp runs them with g++; sampler.cuh and background.cuh run them on the device).
//   depths: UniformSampler.get_z_vals (engine/ray_sampler.py:54-80), optionally stratified by a caller-drawn uniform (:70-78);
//           the background's inverse_sample (:82-85) flipped (background.py:63-68): sample k at depth 1/R_s ... 0
//   integral (bg_volume_rendering, background.py:137-165): fe_k = dist_k |sdf_k|, T_k = exp(-sum_{i<k} fe_i),
//           w_k = (1 - e^{-fe_k}) T_k, only = sum_k w_k rgb_k, bg_rgb = w_fg only, bg_semantics = w_fg [1, 0, 0, 0]
//   reverse: g = g_only + w_fg g_rgb, d rgb_k = w_k g, d w_k = <rgb_k, g>,
//           d fe_k = d w_k e^{-fe_k} T_k - sum_{i>k} d w_i w_i,  d sdf_k = d fe_k dist_k sign(sdf_k) (0 at sdf = 0, torch's abs),
//           d w_fg = <only, g_rgb> + g_semantics[0]
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define HOLD_HD __host__ __device__ __forceinline__
#else
#ifndef HOLD_HD
#define HOLD_HD inline
#endif
#endif

namespace hold {

constexpr int kBgN = 32;   // N_samples_inverse_sphere

// torch.linspace(start, end, steps)[i] in fp32 — symmetric evaluation like ATen's linspace kernel
// (RangeFactories: first half from start, second half from end).
HOLD_HD float torch_linspace(float start, float end, int steps, int i) {
  if (steps == 1) return start;
  float step = (end - start) / (float)(steps - 1);
  int half = steps / 2;
  // ATen's linspace kernels (CPU and CUDA) evaluate start + step * i as one fused multiply-add (checked against torch.linspace
  // bit for bit, tests/test_cpu_host.py); spelled out so that host and device builds agree
  return (i < half) ? fmaf(step, (float)i, start) : fmaf(-step, (float)(steps - i - 1), end);
}

// z_k = near (1 - t_k) + far t_k, t = linspace(0, 1, n).  u (NULL: eval mode) stratifies it: z_k = lower + (upper - lower) u with
// lower / upper the midpoints to the neighbours (z_0 / z_{n-1} at the ends).
HOLD_HD float stratified_z(float near, float far, int n, int k, const float* u) {
  const float t = torch_linspace(0.f, 1.f, n, k);
  const float zk = near * (1.0f - t) + far * t;
  if (u == nullptr) return zk;
  float lower = zk, upper = zk;
  if (k > 0) {
    const float tm = torch_linspace(0.f, 1.f, n, k - 1);
    lower = 0.5f * (zk + (near * (1.0f - tm) + far * tm));
  }
  if (k + 1 < n) {
    const float t1 = torch_linspace(0.f, 1.f, n, k + 1);
    upper = 0.5f * ((near * (1.0f - t1) + far * t1) + zk);
  }
  return lower + (upper - lower) * *u;
}

// depth of the background's sample k (flipped order, 1/R_s -> 0).  u: the uniform of the UN-flipped sample kBgN - 1 - k (the
// layout inverse_sample's jitter has), or NULL for the fixed shells.
HOLD_HD float bg_depth(int k, float r_sphere, const float* u = nullptr) {
  return stratified_z(0.f, 1.f, kBgN, kBgN - 1 - k, u) * (1.0f / r_sphere);
}

// interval after sample k (flipped order): z_k - z_{k+1}, the last one 1e10.  z: the un-flipped depths of the ray, or NULL for
// the fixed shells.
HOLD_HD float bg_interval(const float* z, float r_sphere, int k) {
  if (k + 1 >= kBgN) return 1.0e10f;
  if (z != nullptr) return z[kBgN - 1 - k] - z[kBgN - 2 - k];
  return bg_depth(k, r_sphere) - bg_depth(k + 1, r_sphere);
}

// the forward integral of one ray (sequential over the samples, as k_bg_composite runs it): only[3] = sum_k w_k rgb_k
HOLD_HD void bg_integrate_ray(const float* z /*[32] un-flipped or NULL*/, float r_sphere, const float* sdf /*[32]*/,
                              const float* rgb /*[32,3]*/, float only[3]) {
  float cum = 0.f;
  only[0] = only[1] = only[2] = 0.f;
  for (int k = 0; k < kBgN; ++k) {
    const float fe = bg_interval(z, r_sphere, k) * fabsf(sdf[k]);   // AbsDensity
    const float w = (1.0f - expf(-fe)) * expf(-cum);
    cum += fe;
    only[0] += w * rgb[3 * k], only[1] += w * rgb[3 * k + 1], only[2] += w * rgb[3 * k + 2];
  }
}

// ---- reverse mode, per sample.  The device runs one lane per sample and forms the two sums with warp scans; the host loops.
struct BgSampleBwd {
  float w, e, T, dw;   // weight, e^{-fe}, transmittance before the sample, d w
};

// fe_excl = sum_{i<k} fe_i.  g[3] = g_only + w_fg g_rgb.  Writes d rgb_k.
HOLD_HD BgSampleBwd bg_bwd_sample(float fe, float fe_excl, const float* rgb_k, const float g[3], float* d_rgb_k) {
  BgSampleBwd s;
  s.e = expf(-fe);
  s.T = expf(-fe_excl);
  s.w = (1.0f - s.e) * s.T;
  d_rgb_k[0] = s.w * g[0], d_rgb_k[1] = s.w * g[1], d_rgb_k[2] = s.w * g[2];
  s.dw = rgb_k[0] * g[0] + rgb_k[1] * g[1] + rgb_k[2] * g[2];
  return s;
}

// dww_after = sum_{i>k} d w_i w_i
HOLD_HD float bg_bwd_dsdf(const BgSampleBwd& s, float dww_after, float dist, float sdf) {
  const float dfe = s.dw * s.e * s.T - dww_after;
  const float sg = (sdf > 0.f) ? 1.f : ((sdf < 0.f) ? -1.f : 0.f);
  return dfe * dist * sg;
}

// g[3] = g_only + w_fg g_rgb (either upstream may be NULL = 0)
HOLD_HD void bg_bwd_seed(const float* g_rgb, const float* g_only, float w_fg, float g[3]) {
  for (int c = 0; c < 3; ++c) g[c] = (g_only ? g_only[c] : 0.f) + w_fg * (g_rgb ? g_rgb[c] : 0.f);
}

HOLD_HD float bg_bwd_dwfg(const float only[3], const float* g_rgb, const float* g_sem) {
  float d = g_sem ? g_sem[0] : 0.f;
  if (g_rgb) d += only[0] * g_rgb[0] + only[1] * g_rgb[1] + only[2] * g_rgb[2];
  return d;
}

}  // namespace hold
