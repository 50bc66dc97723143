// Host run of the background's depth and integration steps (hold_b200/csrc/bg_phases.h): the forward as k_bg_composite runs it,
// the reverse mode with the two warp scans of k_bg_composite_bwd done as loops.
#include "../../hold_b200/csrc/bg_phases.h"

using namespace hold;

// z [R,32] un-flipped depths of inverse_sample; jitter [R,32] or NULL
extern "C" void bg_depths_host(int R, float r_sphere, const float* jitter, float* z) {
  for (int r = 0; r < R; ++r)
    for (int k = 0; k < kBgN; ++k) {
      const int j = kBgN - 1 - k;
      z[r * kBgN + j] = bg_depth(k, r_sphere, jitter ? jitter + r * kBgN + j : nullptr);
    }
}

// the foreground's stratified_z over n samples of R rays: near, far [R], u [R,n] or NULL -> z [R,n]
extern "C" void stratified_z_host(int R, int n, float near, const float* far, const float* u, float* z) {
  for (int r = 0; r < R; ++r)
    for (int k = 0; k < n; ++k) z[r * n + k] = stratified_z(near, far[r], n, k, u ? u + r * n + k : nullptr);
}

extern "C" void bg_integrate_host(int R, const float* z, const float* sdf, const float* rgb, const float* wfg, float* bg_rgb,
                                  float* only, float* sem) {
  for (int r = 0; r < R; ++r) {
    bg_integrate_ray(z + r * kBgN, 0.f, sdf + r * kBgN, rgb + r * kBgN * 3, only + 3 * r);
    for (int c = 0; c < 3; ++c) bg_rgb[3 * r + c] = wfg[r] * only[3 * r + c];
    sem[4 * r] = wfg[r], sem[4 * r + 1] = sem[4 * r + 2] = sem[4 * r + 3] = 0.f;
  }
}

extern "C" void bg_integrate_bwd_host(int R, const float* z, const float* sdf, const float* rgb, const float* wfg, const float* g_rgb,
                                      const float* g_only, const float* g_sem, float* d_sdf, float* d_rgb, float* d_wfg) {
  for (int r = 0; r < R; ++r) {
    float g[3], fe[kBgN], dist[kBgN], after[kBgN];
    BgSampleBwd b[kBgN];
    bg_bwd_seed(g_rgb ? g_rgb + 3 * r : nullptr, g_only ? g_only + 3 * r : nullptr, wfg[r], g);
    float excl = 0.f, only[3] = {0.f, 0.f, 0.f};
    for (int k = 0; k < kBgN; ++k) {
      const int p = r * kBgN + k;
      dist[k] = bg_interval(z + r * kBgN, 0.f, k);
      fe[k] = dist[k] * fabsf(sdf[p]);
      b[k] = bg_bwd_sample(fe[k], excl, rgb + 3 * p, g, d_rgb + 3 * p);
      excl += fe[k];
      for (int c = 0; c < 3; ++c) only[c] += b[k].w * rgb[3 * p + c];
    }
    float suf = 0.f;
    for (int k = kBgN - 1; k >= 0; --k) {
      after[k] = suf;
      suf += b[k].dw * b[k].w;
    }
    for (int k = 0; k < kBgN; ++k) d_sdf[r * kBgN + k] = bg_bwd_dsdf(b[k], after[k], dist[k], sdf[r * kBgN + k]);
    d_wfg[r] = bg_bwd_dwfg(only, g_rgb ? g_rgb + 3 * r : nullptr, g_sem ? g_sem + 4 * r : nullptr);
  }
}
