// Soft-silhouette mesh rasterisation (the pose refinement of optimize_ckpt.py, fitting/utils.py:101-118): the per-pixel
// arithmetic of pytorch3d v0.7.4's MeshRasterizer (rasterize_meshes, CheckPixelInsideFace) and SoftSilhouetteShader
// (sigmoid_alpha_blend), restated without its source.  This header and oracle/soft_raster_oracle.py are the only two places
// that encode the rules; the boundary is unpinned (DESIGN.md row 4c).  Compiles for the host (tests/host/raster_host.cpp).
//
// Per pixel and face (face records from face_setup):
//   1. skip when max z < 0, |area| <= 1e-8, culling and area < 0 (face_setup: all pixels), or the pixel lies outside the xy
//      bounding box expanded by sqrt(blur_radius);
//   2. screen barycentrics b (pytorch3d's BarycentricCoordsForward: area + 1e-8 in the denominator), perspective correction
//      (b_i z_j z_k / max(sum, 1e-8)), clipping (b >= 0, / max(sum, 1e-8));
//   3. pz = sum b_i z_i with the clipped b; skip when pz < 0;
//   4. dist = squared xy distance to the nearest edge segment (edges 01, 02, 12; the first of equals);
//   5. inside = all unclipped b > 0; signed_dist = inside ? -dist : dist; skip when outside and dist >= blur_radius.
// Selection: the K candidates of smallest key (pz, face).  Blend: p = sigmoid(-signed_dist / sigma), silhouette =
// 1 - prod_k (1 - p_k).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HOLD_HD __host__ __device__ __forceinline__
#else
#ifndef HOLD_HD
#define HOLD_HD inline
#endif
#endif

namespace hold {
namespace raster {

constexpr float kEps = 1e-8f;

struct Opts {
  float blur_radius;   // compared with the SQUARED distance
  float sigma;
  bool perspective_correct, clip_barycentric_coords, cull_backfaces;
};

// Centre of pixel (row i, col j) in pytorch3d NDC: +x left, +y up, the shorter side spans [-1, 1].
HOLD_HD float pix_ndc(int idx, int n, int s) { return (float)(n - 2 * idx - 1) / (float)s; }

// pytorch3d's EdgeFunctionForward(p, v0, v1)
HOLD_HD float edge_fn(float px, float py, float ax, float ay, float bx, float by) {
  return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

HOLD_HD float min3(float a, float b, float c) { return fminf(a, fminf(b, c)); }
HOLD_HD float max3(float a, float b, float c) { return fmaxf(a, fmaxf(b, c)); }

// Face-wide part of step 1.  v: x0 y0 x1 y1 x2 y2 z0 z1 z2.  Returns false when the face is skipped for every pixel, else
// writes the bounding box expanded by sqrt(blur_radius): xmin, xmax, ymin, ymax.
HOLD_HD bool face_setup(const float* v, const Opts& o, float* bbox) {
  const float zmax = max3(v[6], v[7], v[8]);
  const float area = edge_fn(v[0], v[1], v[2], v[3], v[4], v[5]);
  if (zmax < 0.f || (area <= kEps && area >= -kEps) || (o.cull_backfaces && area < 0.f)) return false;
  const float r = sqrtf(o.blur_radius);
  bbox[0] = min3(v[0], v[2], v[4]) - r, bbox[1] = max3(v[0], v[2], v[4]) + r;
  bbox[2] = min3(v[1], v[3], v[5]) - r, bbox[3] = max3(v[1], v[3], v[5]) + r;
  return true;
}

HOLD_HD bool outside_bbox(const float* bbox, float px, float py) {
  return px > bbox[1] || px < bbox[0] || py > bbox[3] || py < bbox[2];
}

// Screen barycentrics of (px, py) in triangle v (BarycentricCoordsForward).
HOLD_HD void barycentric(float px, float py, const float* v, float* b) {
  const float area = edge_fn(v[4], v[5], v[0], v[1], v[2], v[3]) + kEps;
  b[0] = edge_fn(px, py, v[2], v[3], v[4], v[5]) / area;
  b[1] = edge_fn(px, py, v[4], v[5], v[0], v[1]) / area;
  b[2] = edge_fn(px, py, v[0], v[1], v[2], v[3]) / area;
}

HOLD_HD void perspective_correct(const float* z, float* b) {
  const float t0 = b[0] * z[1] * z[2], t1 = z[0] * b[1] * z[2], t2 = z[0] * z[1] * b[2];
  const float d = fmaxf(t0 + t1 + t2, kEps);
  b[0] = t0 / d, b[1] = t1 / d, b[2] = t2 / d;
}

HOLD_HD void clip_barycentric(const float* b, float* c) {
  c[0] = fmaxf(b[0], 0.f), c[1] = fmaxf(b[1], 0.f), c[2] = fmaxf(b[2], 0.f);
  const float d = fmaxf(c[0] + c[1] + c[2], kEps);
  c[0] /= d, c[1] /= d, c[2] /= d;
}

// Squared distance from p to the segment a-b.  d = (p - a) - t (b - a) keeps the rounding relative to the (small) distance
// rather than to the coordinates: with sigma = 1e-4 the silhouette's slope is up to 2500 per unit of squared distance.
HOLD_HD float seg_sqdist(float px, float py, float ax, float ay, float bx, float by) {
  const float bax = bx - ax, bay = by - ay, pax = px - ax, pay = py - ay;
  const float l2 = bax * bax + bay * bay;
  if (l2 <= kEps) {
    const float dx = px - bx, dy = py - by;
    return dx * dx + dy * dy;
  }
  const float t = fminf(fmaxf((bax * pax + bay * pay) / l2, 0.f), 1.f);
  const float dx = pax - t * bax, dy = pay - t * bay;
  return dx * dx + dy * dy;
}

// Reverse mode of seg_sqdist: g = d loss / d dist -> ga, gb (xy), accumulated.  t is held fixed: inside (0, 1) the distance
// is stationary in t, at a clamp t is constant (pytorch3d's PointLineDistanceBackward does the same).
HOLD_HD void seg_sqdist_bwd(float px, float py, float ax, float ay, float bx, float by, float g, float* ga, float* gb) {
  const float bax = bx - ax, bay = by - ay, pax = px - ax, pay = py - ay;
  const float l2 = bax * bax + bay * bay;
  if (l2 <= kEps) {
    gb[0] += -2.f * g * (px - bx), gb[1] += -2.f * g * (py - by);
    return;
  }
  const float t = fminf(fmaxf((bax * pax + bay * pay) / l2, 0.f), 1.f);
  const float dx = pax - t * bax, dy = pay - t * bay;
  ga[0] += -2.f * g * (1.f - t) * dx, ga[1] += -2.f * g * (1.f - t) * dy;
  gb[0] += -2.f * g * t * dx, gb[1] += -2.f * g * t * dy;
}

// The three edges in pytorch3d's order: (v0, v1), (v0, v2), (v1, v2).
HOLD_HD int edge_a(int e) { return e == 2 ? 1 : 0; }
HOLD_HD int edge_b(int e) { return e == 0 ? 1 : 2; }

// Squared distance to the nearest edge; *edge = its index (the first of equals, as PointTriangleDistanceBackward picks).
HOLD_HD float tri_sqdist(float px, float py, const float* v, int* edge) {
  float best = 0.f;
  for (int e = 0; e < 3; ++e) {
    const int a = edge_a(e), b = edge_b(e);
    const float d = seg_sqdist(px, py, v[2 * a], v[2 * a + 1], v[2 * b], v[2 * b + 1]);
    if (e == 0 || d < best) best = d, *edge = e;
  }
  return best;
}

// Reverse mode of tri_sqdist through its nearest edge: g -> gv[6] (xy of the three vertices), accumulated.
// (Branches with constant indices keep v and gv in registers on the device.)
HOLD_HD void tri_sqdist_bwd(float px, float py, const float* v, int edge, float g, float* gv) {
  if (edge == 0) seg_sqdist_bwd(px, py, v[0], v[1], v[2], v[3], g, gv, gv + 2);
  else if (edge == 1) seg_sqdist_bwd(px, py, v[0], v[1], v[4], v[5], g, gv, gv + 4);
  else seg_sqdist_bwd(px, py, v[2], v[3], v[4], v[5], g, gv + 2, gv + 4);
}

struct Frag {
  float pz;     // interpolated depth: the selection key with the face index
  float dist;   // squared distance to the nearest edge
  bool inside;  // signed_dist = inside ? -dist : dist
  int edge;     // nearest edge (tri_sqdist)
};

// Steps 1 (pixel part) to 5 for a face that passed face_setup.  v: x0 y0 x1 y1 x2 y2 z0 z1 z2.  False = not a candidate.
HOLD_HD bool pixel_face(const float* v, const float* bbox, float px, float py, const Opts& o, Frag& f) {
  if (outside_bbox(bbox, px, py)) return false;
  float b[3], c[3];
  barycentric(px, py, v, b);
  if (o.perspective_correct) perspective_correct(v + 6, b);
  if (o.clip_barycentric_coords) clip_barycentric(b, c);
  else c[0] = b[0], c[1] = b[1], c[2] = b[2];
  f.pz = c[0] * v[6] + c[1] * v[7] + c[2] * v[8];
  if (f.pz < 0.f) return false;
  f.dist = tri_sqdist(px, py, v, &f.edge);
  f.inside = b[0] > 0.f && b[1] > 0.f && b[2] > 0.f;
  return f.inside || f.dist < o.blur_radius;
}

// Selection key: (pz, face) in one unsigned integer of 31 + fbits bits (pz >= 0, so its float bits order as integers; -0 is
// mapped to +0).  fbits = bits of the largest face index.
HOLD_HD uint64_t frag_key(float pz, int face, int fbits) {
  union { float f; uint32_t u; } c;
  c.f = pz + 0.f;
  return ((uint64_t)c.u << fbits) | (uint64_t)(uint32_t)face;
}

HOLD_HD float signed_dist(const Frag& f) { return f.inside ? -f.dist : f.dist; }

// 1 - p = sigmoid(signed_dist / sigma), computed directly so that it keeps its relative precision when p is near 1 (and is
// exactly 0 when it underflows).
HOLD_HD float blend_q(float sd, float sigma) { return 1.f / (1.f + expf(-sd / sigma)); }
HOLD_HD float blend_p(float sd, float sigma) { return 1.f / (1.f + expf(sd / sigma)); }

// silhouette = 1 - Q, Q = prod_k q_k over the kept faces (Q = 1, silhouette 0, when none is kept).
// Its gradient with respect to face k's signed distance:
//   d sil / d sd_k = (d sil / d p_k) (d p_k / d sd_k) = prod_{j != k} q_j * (-p_k q_k / sigma) = -p_k Q / sigma.
// The factor q_k of d p / d sd completes the exclusion product, so the gradient needs Q alone: no division by 1 - p_k, and
// it stays right when some q_j is 0 (then Q = 0, and the exact value is below the smallest float: |.| <= q_j / sigma).
HOLD_HD float blend_dsd(float Q, float sd, float sigma) { return -blend_p(sd, sigma) * Q / sigma; }

// d loss / d dist of a kept face, given d loss / d silhouette = g.
HOLD_HD float blend_ddist(float g, float Q, const Frag& f, float sigma) {
  const float gsd = g * blend_dsd(Q, signed_dist(f), sigma);
  return f.inside ? -gsd : gsd;
}

}  // namespace raster
}  // namespace hold
