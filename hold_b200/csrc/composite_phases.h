// merge_factors (hold/hold_utils.py:76-121) + density2weight (engine/volsdf_utils.py:220-251) + the five integrals of
// volumetric_render (hold/hold_utils.py:243-271) for one ray, forward and reverse, written as host-executable walks
// (tests/host/composite_host.cpp runs them with g++; composite.cuh runs one per thread).  The per-node z lists are already
// sorted, so the reference's torch.sort over the concatenation is a stable n-way merge (ties -> lower node first).
#pragma once
#include <math.h>
#include <stddef.h>

#include "../../include/hold_b200.h"

#if defined(__CUDACC__)
#define HOLD_HD __host__ __device__ __forceinline__
#else
#ifndef HOLD_HD
#define HOLD_HD inline
#endif
#endif

namespace hold {

struct CompositeArgs {
  int n, R, S;
  const float* color[HOLD_MAX_NODES];
  const float* normal[HOLD_MAX_NODES];
  const float* density[HOLD_MAX_NODES];
  const float* z[HOLD_MAX_NODES];
  int class_id[HOLD_MAX_NODES];
  hold_render_out out;
  int drop_head, drop_tail;  // (n-1, n) for the composite; (0, 0) for a single node
  int single_zmax_last;      // per-node render: z_max = z[:, -1] (hold_net.py:79-80)
};

HOLD_HD void composite_ray(const CompositeArgs& a, int r) {
  const int n = a.n, S = a.S, total = n * S;
  int head[HOLD_MAX_NODES];
  const float* zr[HOLD_MAX_NODES];
#pragma unroll
  for (int k = 0; k < HOLD_MAX_NODES; ++k) { head[k] = 0; zr[k] = (k < n) ? a.z[k] + (size_t)r * S : nullptr; }
  const int first = a.drop_head, last = total - a.drop_tail;  // keep merged positions [first, last)
  const int M = last - first;
  // z_max: merged position total - n (composite) or the node's last z
  float acc_rgb[3] = {0.f, 0.f, 0.f}, acc_n[3] = {0.f, 0.f, 0.f}, acc_sem[4] = {0.f, 0.f, 0.f, 0.f};
  float acc_mask = 0.f, acc_depth = 0.f, cum = 0.f;
  // pending sample (needs the next z to close its interval)
  bool have = false;
  float pz = 0.f, psig = 0.f, pc[3] = {0, 0, 0}, pn[3] = {0, 0, 0};
  int pcls = 0, kept = 0;
  float* wout = (a.out.fg_weights != nullptr) ? a.out.fg_weights + (size_t)r * M : nullptr;

  auto close_interval = [&](float znext) {
    float fe = (znext - pz) * psig;
    float alpha = 1.0f - expf(-fe);
    float T = expf(-cum);
    float w = alpha * T;
    cum += fe;
    acc_rgb[0] += pc[0] * w, acc_rgb[1] += pc[1] * w, acc_rgb[2] += pc[2] * w;
    acc_n[0] += pn[0] * w, acc_n[1] += pn[1] * w, acc_n[2] += pn[2] * w;
    acc_mask += w;
    acc_depth += pz * w;
    acc_sem[pcls] += w;
    if (wout != nullptr) wout[kept - 1] = w;
  };

  for (int t = 0; t < total; ++t) {
    int best = -1;
    float bz = 0.f;
#pragma unroll
    for (int k = 0; k < HOLD_MAX_NODES; ++k) {
      if (k < n && head[k] < S) {
        float zk = zr[k][head[k]];
        if (best < 0 || zk < bz) { best = k; bz = zk; }
      }
    }
    int j = head[best]++;
    if (t >= first && t < last) {
      if (have) close_interval(bz);
      size_t off = (size_t)r * S + j;
      pz = bz;
      psig = a.density[best][off];
      const float* c = a.color[best] + 3 * off;
      const float* nn = a.normal[best] + 3 * off;
      pc[0] = c[0], pc[1] = c[1], pc[2] = c[2];
      pn[0] = nn[0], pn[1] = nn[1], pn[2] = nn[2];
      pcls = a.class_id[best];
      have = true;
      ++kept;
    } else if (t >= last) {
      // first dropped tail element: merged[total - n] == z_max for the composite (drop_tail == n)
      if (have && t == total - n && !a.single_zmax_last) { close_interval(bz); have = false; }
    }
  }
  if (have) close_interval(pz);  // per-node render: z_max = own last z -> zero-length last interval
  if (a.out.fg_rgb) { a.out.fg_rgb[3 * r] = acc_rgb[0], a.out.fg_rgb[3 * r + 1] = acc_rgb[1], a.out.fg_rgb[3 * r + 2] = acc_rgb[2]; }
  if (a.out.normal) { a.out.normal[3 * r] = acc_n[0], a.out.normal[3 * r + 1] = acc_n[1], a.out.normal[3 * r + 2] = acc_n[2]; }
  if (a.out.mask_prob) a.out.mask_prob[r] = fminf(fmaxf(acc_mask, 0.f), 1.f);
  if (a.out.depth) a.out.depth[r] = acc_depth;
  if (a.out.fg_semantics) {
#pragma unroll
    for (int c = 0; c < 4; ++c) a.out.fg_semantics[4 * r + c] = acc_sem[c];
  }
  if (a.out.bg_weights) a.out.bg_weights[r] = expf(-cum);
}

// Reverse mode of composite_ray: gradients of the five integrals + bg_weights w.r.t. every node's colour, normal and density
// (z_vals come from the sampler, which runs without autograd in the reference: ray_sampler.py:169-178, mano_node.py:100-111).
//   w_i = (1 - e^{-fe_i}) T_i,  fe_i = sigma_i (z_{i+1} - z_i),  T_i = exp(-sum_{j<i} fe_j),  bg = exp(-sum_all fe)
//   dL/dfe_i = dw_i e^{-fe_i} T_i - sum_{j>i} dw_j w_j - d_bg bg,   dw_i = c_i.d_rgb + [0 <= mask <= 1] d_mask + n_i.d_nrm + z_i d_depth + d_sem[class_i]
// A forward merge for the total free energy and the clamp gate, then the SAME merge walked backwards (largest z first, ties ->
// higher node first = the exact reverse of the stable forward order) carrying the suffix sums.
struct CompositeBwdArgs {
  int n, R, S;
  const float* color[HOLD_MAX_NODES];
  const float* normal[HOLD_MAX_NODES];
  const float* density[HOLD_MAX_NODES];
  const float* z[HOLD_MAX_NODES];
  int class_id[HOLD_MAX_NODES];
  hold_render_out g;               // upstream gradients (any pointer may be NULL = zero); fg_weights is ignored
  float* d_color[HOLD_MAX_NODES];
  float* d_normal[HOLD_MAX_NODES];
  float* d_density[HOLD_MAX_NODES];
  int drop_head, drop_tail, single_zmax_last;
  int accumulate;                  // add to the d_* buffers instead of overwriting them
};

HOLD_HD void composite_bwd_ray(const CompositeBwdArgs& a, int r) {
  const int n = a.n, S = a.S, total = n * S;
  const int first = a.drop_head, last = total - a.drop_tail;
  const float* zr[HOLD_MAX_NODES];
  int head[HOLD_MAX_NODES];
#pragma unroll
  for (int k = 0; k < HOLD_MAX_NODES; ++k) { head[k] = 0; zr[k] = (k < n) ? a.z[k] + (size_t)r * S : nullptr; }
  // ---- forward merge: total free energy of the kept intervals, sum of weights (clamp gate).  acc_mask and cum repeat
  // composite_ray's float arithmetic, so the gate and bg are the forward's bits.  The transmittance of sample i is recovered
  // below as exp(-(total - suffix - fe_i)): in float that difference of two large sums of the same terms cancels to
  // ulp(total) * #samples, which at optical depths of hundreds is 1e-4 of T, so the total and the suffix are kept in double.
  float cum = 0.f, acc_mask = 0.f, pz = 0.f, psig = 0.f;
  double total_fe = 0.0;
  bool have = false;
  for (int t = 0; t < total; ++t) {
    int best = -1;
    float bz = 0.f;
#pragma unroll
    for (int k = 0; k < HOLD_MAX_NODES; ++k)
      if (k < n && head[k] < S) {
        const float zk = zr[k][head[k]];
        if (best < 0 || zk < bz) { best = k; bz = zk; }
      }
    const int j = head[best]++;
    if (t >= first && t < last) {
      if (have) { const float fe = (bz - pz) * psig; acc_mask += (1.0f - expf(-fe)) * expf(-cum); cum += fe; total_fe += fe; }
      pz = bz, psig = a.density[best][(size_t)r * S + j], have = true;
    } else if (t >= last) {
      if (have && t == total - n && !a.single_zmax_last) {
        const float fe = (bz - pz) * psig;
        acc_mask += (1.0f - expf(-fe)) * expf(-cum);
        cum += fe, total_fe += fe, have = false;
      }
    }
  }
  // (per-node render: the last interval has zero length and contributes nothing)
  const float bg = expf(-cum);
  const float g_rgb[3] = {a.g.fg_rgb ? a.g.fg_rgb[3 * r] : 0.f, a.g.fg_rgb ? a.g.fg_rgb[3 * r + 1] : 0.f, a.g.fg_rgb ? a.g.fg_rgb[3 * r + 2] : 0.f};
  const float g_nrm[3] = {a.g.normal ? a.g.normal[3 * r] : 0.f, a.g.normal ? a.g.normal[3 * r + 1] : 0.f, a.g.normal ? a.g.normal[3 * r + 2] : 0.f};
  const float g_mask = (a.g.mask_prob && acc_mask >= 0.f && acc_mask <= 1.f) ? a.g.mask_prob[r] : 0.f;
  const float g_depth = a.g.depth ? a.g.depth[r] : 0.f;
  float g_sem[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) g_sem[c] = a.g.fg_semantics ? a.g.fg_semantics[4 * r + c] : 0.f;
  const float g_bg = a.g.bg_weights ? a.g.bg_weights[r] : 0.f;
  // ---- backward merge from the tails
  int tail[HOLD_MAX_NODES];
#pragma unroll
  for (int k = 0; k < HOLD_MAX_NODES; ++k) tail[k] = S - 1;
  float znext = 0.f;          // z of merged position t + 1
  double suffix_fe = 0.0;     // sum_{j > i} fe_j over kept intervals
  float G = 0.f;              // sum_{j > i} dw_j w_j
  for (int t = total - 1; t >= 0; --t) {
    int best = -1;
    float bz = 0.f;
#pragma unroll
    for (int k = HOLD_MAX_NODES - 1; k >= 0; --k)
      if (k < n && tail[k] >= 0) {
        const float zk = zr[k][tail[k]];
        if (best < 0 || zk > bz) { best = k; bz = zk; }   // strict >: among equal z the HIGHER node comes later in the forward order
      }
    const int j = tail[best]--;
    const size_t off = (size_t)r * S + j;
    float dc[3] = {0.f, 0.f, 0.f}, dn[3] = {0.f, 0.f, 0.f}, dsig = 0.f;
    if (t >= first && t < last) {
      // interval end: the next merged z; the last kept sample of the composite ends at merged[total - n] = merged[last]; a
      // per-node render ends at its own last z (zero length)
      const float zend = (t == last - 1 && a.single_zmax_last) ? bz : znext;
      const float sig = a.density[best][off];
      const float delta = zend - bz;
      const float fe = delta * sig;
      const float T = expf(-(float)(total_fe - suffix_fe - (double)fe));
      const float e = expf(-fe);
      const float w = (1.0f - e) * T;
      const float* c = a.color[best] + 3 * off;
      const float* nn = a.normal[best] + 3 * off;
      const float dw = c[0] * g_rgb[0] + c[1] * g_rgb[1] + c[2] * g_rgb[2] + g_mask + nn[0] * g_nrm[0] + nn[1] * g_nrm[1] + nn[2] * g_nrm[2] +
                       bz * g_depth + g_sem[a.class_id[best]];
      const float dfe = dw * e * T - G - g_bg * bg;
      dsig = dfe * delta;
      dc[0] = w * g_rgb[0], dc[1] = w * g_rgb[1], dc[2] = w * g_rgb[2];
      dn[0] = w * g_nrm[0], dn[1] = w * g_nrm[1], dn[2] = w * g_nrm[2];
      G += dw * w;
      suffix_fe += fe;
    }
    if (a.accumulate) {
      a.d_color[best][3 * off] += dc[0], a.d_color[best][3 * off + 1] += dc[1], a.d_color[best][3 * off + 2] += dc[2];
      a.d_normal[best][3 * off] += dn[0], a.d_normal[best][3 * off + 1] += dn[1], a.d_normal[best][3 * off + 2] += dn[2];
      a.d_density[best][off] += dsig;
    } else {
      a.d_color[best][3 * off] = dc[0], a.d_color[best][3 * off + 1] = dc[1], a.d_color[best][3 * off + 2] = dc[2];
      a.d_normal[best][3 * off] = dn[0], a.d_normal[best][3 * off + 1] = dn[1], a.d_normal[best][3 * off + 2] = dn[2];
      a.d_density[best][off] = dsig;
    }
    znext = bz;
  }
}

}  // namespace hold
