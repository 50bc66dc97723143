// Host run of the soft-silhouette rasteriser's per-pixel steps (hold_b200/csrc/raster_phases.h), one exported function per
// step, element-wise over n inputs.
#include "../../hold_b200/csrc/raster_phases.h"

using namespace hold::raster;

// pixel centres: x [W], y [H]
extern "C" void pix_ndc_host(int H, int W, float* x, float* y) {
  const int s = H < W ? H : W;
  for (int j = 0; j < W; ++j) x[j] = pix_ndc(j, W, s);
  for (int i = 0; i < H; ++i) y[i] = pix_ndc(i, H, s);
}

// barycentrics of points p [n,2] in triangles v [n,9]: b [n,3] screen, bp [n,3] perspective-corrected, c [n,3] bp clipped
extern "C" void bary_host(int n, const float* p, const float* v, float* b, float* bp, float* c) {
  for (int k = 0; k < n; ++k) {
    barycentric(p[2 * k], p[2 * k + 1], v + 9 * k, b + 3 * k);
    for (int e = 0; e < 3; ++e) bp[3 * k + e] = b[3 * k + e];
    perspective_correct(v + 9 * k + 6, bp + 3 * k);
    clip_barycentric(bp + 3 * k, c + 3 * k);
  }
}

// segment distance and its reverse mode: p [n,2], a [n,2], b [n,2], g [n] -> d [n], ga [n,2], gb [n,2]
extern "C" void seg_host(int n, const float* p, const float* a, const float* b, const float* g, float* d, float* ga, float* gb) {
  for (int k = 0; k < n; ++k) {
    d[k] = seg_sqdist(p[2 * k], p[2 * k + 1], a[2 * k], a[2 * k + 1], b[2 * k], b[2 * k + 1]);
    ga[2 * k] = ga[2 * k + 1] = gb[2 * k] = gb[2 * k + 1] = 0.f;
    seg_sqdist_bwd(p[2 * k], p[2 * k + 1], a[2 * k], a[2 * k + 1], b[2 * k], b[2 * k + 1], g[k], ga + 2 * k, gb + 2 * k);
  }
}

// the whole per-pixel test of n (pixel, face) pairs: ok [n], pz [n], dist [n], inside [n]
extern "C" void pixel_face_host(int n, const float* p, const float* v, float blur, float sigma, int persp, int clip, int cull,
                                int* ok, float* pz, float* dist, int* inside) {
  const Opts o{blur, sigma, persp != 0, clip != 0, cull != 0};
  for (int k = 0; k < n; ++k) {
    float bb[4];
    Frag f{0.f, 0.f, false, 0};
    ok[k] = face_setup(v + 9 * k, o, bb) && pixel_face(v + 9 * k, bb, p[2 * k], p[2 * k + 1], o, f);
    pz[k] = f.pz, dist[k] = f.dist, inside[k] = f.inside;
  }
}

// the blend of one pixel's m kept faces (signed distances sd [m]): silhouette, and d sil / d sd [m]
extern "C" void blend_host(int m, const float* sd, float sigma, float* sil, float* dsd) {
  float Q = 1.f;
  for (int k = 0; k < m; ++k) Q *= blend_q(sd[k], sigma);
  *sil = 1.f - Q;
  for (int k = 0; k < m; ++k) dsd[k] = blend_dsd(Q, sd[k], sigma);
}
