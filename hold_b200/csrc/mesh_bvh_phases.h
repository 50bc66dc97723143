// Per-item arithmetic of the BVH signed-distance query (mesh_bvh.cuh), compiled for the host as well
// (tests/host/mesh_bvh_host.cpp).  The result is bit for bit what the brute force of mesh_sdf_phases.h gives:
//   * distance: the lexicographic minimum of (tri_sqdist, face) over the faces whose tri_sqdist is below 3e38 (acc_face's
//     ascending strict < skips NaN and never takes a value >= its 3e38 start).  A node is pruned only when a lower bound of the
//     computed tri_sqdist of every face inside its box exceeds the best so far (bvh_box_lower);
//   * sign: the fast winding number (Barill et al. 2018, first order, beta = 4) decides only when | |w| - 0.5 | >= 0.25; inside
//     that band, and for NaN, the caller sums tri_solid_angle over all faces in ascending order as k_mesh_sdf does.
// Tree: linear BVH of Karras 2012 over 30-bit Morton codes of the face centroids, ties broken by face index.  Internal nodes
// 0 .. F-2 (root 0), leaf of sorted position i = node F-1+i, so for F == 1 the root is the only leaf.
#pragma once
#include <stdint.h>
#include "mesh_sdf_phases.h"

namespace hold {
namespace meshbvh {

constexpr int kMaxFaces = 1 << 24;   // depth <= 30 code bits + 24 index bits, so the query's stack holds the deepest path
constexpr int kStack = 64;
constexpr float kBeta = 4.0f;        // far field when |c - p| > kBeta r.  The first-order error falls as 1 / kBeta^2: on the
                                     // test meshes at most 0.124 with 2, 0.025 with 4 (tests/test_cpu_mesh_bvh.py)
constexpr float kBand = 0.25f;       // the fast winding number decides when | |w| - 0.5 | >= kBand
constexpr float kRel = 1e-5f;        // pruning margin: relative to the distance ...
constexpr float kAbs = 1e-5f;        // ... and absolute, in units of the largest coordinate magnitude

// 64 bytes, four float4 on the device: box (lo, r) (hi, area), far-field centroid, area-weighted normal sum
struct alignas(16) Node {
  float lo[3], r;
  float hi[3], area;
  float c[3], pad0;
  float n[3], pad1;
};

HOLD_HD uint32_t expand_bits10(uint32_t v) {
  v &= 1023u;
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

HOLD_HD uint32_t quantise10(float x, float lo, float inv) {
  const float t = fminf(fmaxf((x - lo) * inv * 1024.0f, 0.0f), 1023.0f);   // fmaxf drops NaN
  return (uint32_t)t;
}

// Morton code of the centroid of (a, b, c), 10 bits per axis over the box [lo, lo + 1 / inv] (inv 0 on a flat axis)
HOLD_HD int morton_code(const float* a, const float* b, const float* c, const float* lo, const float* inv) {
  uint32_t code = 0;
  for (int k = 0; k < 3; ++k) {
    const float x = (a[k] + b[k] + c[k]) * (1.0f / 3.0f);
    code |= expand_bits10(quantise10(x, lo[k], inv[k])) << (2 - k);
  }
  return (int)code;
}

HOLD_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __clz((int)x);
#else
  return x ? __builtin_clz(x) : 32;
#endif
}

// Karras's delta: common prefix length of the keys (code, index) at sorted positions i and j; -1 outside [0, F)
HOLD_HD int prefix(const int* codes, int F, int i, int j) {
  if (j < 0 || j >= F) return -1;
  const uint32_t ci = (uint32_t)codes[i], cj = (uint32_t)codes[j];
  return ci != cj ? clz32(ci ^ cj) : 32 + clz32((uint32_t)i ^ (uint32_t)j);
}

// children (node ids) of internal node i in [0, F-2]
HOLD_HD void karras_children(const int* codes, int F, int i, int* left, int* right) {
  const int d = prefix(codes, F, i, i + 1) - prefix(codes, F, i, i - 1) >= 0 ? 1 : -1;
  const int dmin = prefix(codes, F, i, i - d);
  int lmax = 2;
  while (prefix(codes, F, i, i + lmax * d) > dmin) lmax *= 2;
  int l = 0;
  for (int t = lmax / 2; t >= 1; t /= 2)
    if (prefix(codes, F, i, i + (l + t) * d) > dmin) l += t;
  const int j = i + l * d;
  const int dnode = prefix(codes, F, i, j);
  int s = 0, t = l;
  do {
    t = (t + 1) >> 1;
    if (prefix(codes, F, i, i + (s + t) * d) > dnode) s += t;
  } while (t > 1);
  const int g = i + s * d + (d < 0 ? -1 : 0);
  *left = (i < j ? i : j) == g ? F - 1 + g : g;
  *right = (i > j ? i : j) == g + 1 ? F - 1 + g + 1 : g + 1;
}

HOLD_HD float corner_radius(const Node& o) {
  float s = 0.f;
  for (int k = 0; k < 3; ++k) {
    const float e = fmaxf(o.c[k] - o.lo[k], o.hi[k] - o.c[k]);
    s += e * e;
  }
  return sqrtf(s);
}

HOLD_HD void leaf_node(const float* a, const float* b, const float* c, Node& o) {
  const float ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  o.n[0] = 0.5f * (ab[1] * ac[2] - ab[2] * ac[1]);
  o.n[1] = 0.5f * (ab[2] * ac[0] - ab[0] * ac[2]);
  o.n[2] = 0.5f * (ab[0] * ac[1] - ab[1] * ac[0]);
  o.area = sqrtf(meshsdf::dot3(o.n, o.n));
  for (int k = 0; k < 3; ++k) {
    o.lo[k] = fminf(fminf(a[k], b[k]), c[k]);
    o.hi[k] = fmaxf(fmaxf(a[k], b[k]), c[k]);
    o.c[k] = (a[k] + b[k] + c[k]) * (1.0f / 3.0f);
  }
  o.r = corner_radius(o);
  o.pad0 = o.pad1 = 0.f;
}

// parent of (L, R), always in that order
HOLD_HD void merge_node(const Node& L, const Node& R, Node& o) {
  o.area = L.area + R.area;
  const bool w = o.area > 0.f;
  const float wl = w ? L.area / o.area : 0.5f, wr = w ? R.area / o.area : 0.5f;
  for (int k = 0; k < 3; ++k) {
    o.lo[k] = fminf(L.lo[k], R.lo[k]);
    o.hi[k] = fmaxf(L.hi[k], R.hi[k]);
    o.n[k] = L.n[k] + R.n[k];
    o.c[k] = wl * L.c[k] + wr * R.c[k];
  }
  o.r = corner_radius(o);
  o.pad0 = o.pad1 = 0.f;
}

// A lower bound of the computed tri_sqdist(p, ...) of any triangle inside [lo, hi]; scale >= every coordinate magnitude of p
// and of the triangle.  tri_sqdist's closest point is a vertex, a convex combination on an edge, or barycentric inside the
// face: its rounding moves it at most a few ulp of scale out of the box, and the squared sum loses a few ulp of the result.
// kAbs (about 170 ulp of scale) and kRel (about 170 ulp) cover both with a wide margin (tests/test_cpu_mesh_bvh.py).
HOLD_HD float box_lower(const float* lo, const float* hi, const float* p, float scale) {
  float s = 0.f;
  for (int k = 0; k < 3; ++k) {
    const float e = fmaxf(fmaxf(lo[k] - p[k], p[k] - hi[k]), 0.f);
    s += e * e;
  }
  const float t = sqrtf(s) * (1.0f - kRel) - kAbs * scale;
  return t > 0.f ? t * t * (1.0f - kRel) : 0.f;
}

// The traversals read the tree through T: T::node(n) -> Node, T::children(n, &l, &r), T::face(n) -> the face of leaf node n,
// T::tri(f, float[9]) -> its vertices.  stack: kStack ints.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <typename T>
HOLD_HD void nearest(const T& t, int F, const float* p, float scale, int* stack, float& best, int& best_f) {
  best = 3.0e38f, best_f = -1;
  int sp = 0;
  stack[sp++] = 0;
  while (sp > 0) {
    const int n = stack[--sp];
    const Node o = t.node(n);
    if (box_lower(o.lo, o.hi, p, scale) > best) continue;
    if (n >= F - 1) {
      const int f = t.face(n);
      float tri[9];
      t.tri(f, tri);
      const float d = meshsdf::tri_sqdist(p, tri, tri + 3, tri + 6);
      if (d < best || (d == best && best_f >= 0 && f < best_f)) best = d, best_f = f;
      continue;
    }
    int l, r;
    t.children(n, &l, &r);
    const Node ol = t.node(l), orr = t.node(r);
    const float bl = box_lower(ol.lo, ol.hi, p, scale), br = box_lower(orr.lo, orr.hi, p, scale);
    // nearer child on top
    if (bl <= br) {
      if (br <= best) stack[sp++] = r;
      if (bl <= best) stack[sp++] = l;
    } else {
      if (bl <= best) stack[sp++] = l;
      if (br <= best) stack[sp++] = r;
    }
  }
}

// fast winding number (not yet divided by 4 pi): far nodes by their dipole, near leaves by their exact solid angle
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <typename T>
HOLD_HD float fast_winding(const T& t, int F, const float* p, int* stack) {
  float w = 0.f;
  int sp = 0;
  stack[sp++] = 0;
  while (sp > 0) {
    const int n = stack[--sp];
    const Node o = t.node(n);
    const float d[3] = {o.c[0] - p[0], o.c[1] - p[1], o.c[2] - p[2]};
    const float d2 = meshsdf::dot3(d, d), rr = kBeta * o.r;
    if (d2 > rr * rr) {
      w += meshsdf::dot3(o.n, d) / (d2 * sqrtf(d2));
    } else if (n >= F - 1) {
      float tri[9];
      t.tri(t.face(n), tri);
      w += meshsdf::tri_solid_angle(p, tri, tri + 3, tri + 6);
    } else {
      int l, r;
      t.children(n, &l, &r);
      stack[sp++] = r;
      stack[sp++] = l;
    }
  }
  return w;
}

// true: the fast value w (divided by 4 pi) cannot decide the sign, sum exactly (NaN lands here)
HOLD_HD bool in_band(float w) { return !(fabsf(fabsf(w) - 0.5f) >= kBand); }

HOLD_HD bool is_finite3(const float* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

HOLD_HD float signed_dist(float best, bool inside) {
  const float d = sqrtf(best);
  return inside ? -d : d;
}

}  // namespace meshbvh
}  // namespace hold
