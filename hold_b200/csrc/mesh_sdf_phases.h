// SURVEY §8f rank 3 — training-only loss targets: signed distance of canonical sample points to a closed triangle mesh,
// i.e. what compute_mano_cano_sdf / check_off_in_surface_points_cano_mesh (engine/volsdf_utils.py:172-217) obtain from
// kaolin v0.10.0 (absent from the reference's tree): `kaolin.metrics.trianglemesh.point_to_mesh_distance` = squared distance
// to the nearest face (brute force over faces) and `kaolin.ops.mesh.check_sign` = inside/outside of the watertight
// mesh.  Distance: closest point on a triangle by Voronoi regions (Ericson, Real-Time Collision Detection 5.1.5).
// Sign: generalized winding number, sum of the faces' signed solid angles (van Oosterom & Strackee 1983) / 4 pi — for a
// watertight mesh exactly the inside/outside predicate that kaolin's ray-parity test computes, without a ray direction
// to be unlucky with.  The per-point arithmetic below compiles for the host as well (tests/host/mesh_sdf_host.cpp).
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
namespace meshsdf {

HOLD_HD float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// squared distance from p to triangle (a, b, c)
HOLD_HD float tri_sqdist(const float* p, const float* a, const float* b, const float* c) {
  const float ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  const float ap[3] = {p[0] - a[0], p[1] - a[1], p[2] - a[2]};
  const float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
  float q[3];
  bool done = false;
  if (d1 <= 0.f && d2 <= 0.f) { q[0] = a[0], q[1] = a[1], q[2] = a[2]; done = true; }                       // vertex a
  float d3 = 0.f, d4 = 0.f, d5 = 0.f, d6 = 0.f;
  if (!done) {
    const float bp[3] = {p[0] - b[0], p[1] - b[1], p[2] - b[2]};
    d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.f && d4 <= d3) { q[0] = b[0], q[1] = b[1], q[2] = b[2]; done = true; }                        // vertex b
  }
  if (!done) {
    const float vc = d1 * d4 - d3 * d2;
    if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {                                                                // edge ab
      const float v = d1 / (d1 - d3);
      for (int k = 0; k < 3; ++k) q[k] = a[k] + v * ab[k];
      done = true;
    }
  }
  if (!done) {
    const float cp[3] = {p[0] - c[0], p[1] - c[1], p[2] - c[2]};
    d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.f && d5 <= d6) { q[0] = c[0], q[1] = c[1], q[2] = c[2]; done = true; }                        // vertex c
  }
  if (!done) {
    const float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {                                                                // edge ac
      const float w = d2 / (d2 - d6);
      for (int k = 0; k < 3; ++k) q[k] = a[k] + w * ac[k];
      done = true;
    }
  }
  if (!done) {
    const float va = d3 * d6 - d5 * d4;
    if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) {                                                  // edge bc
      const float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
      for (int k = 0; k < 3; ++k) q[k] = b[k] + w * (c[k] - b[k]);
      done = true;
    }
  }
  if (!done) {                                                                                                // face interior
    const float vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
    const float denom = 1.0f / (va + vb + vc);
    const float v = vb * denom, w = vc * denom;
    for (int k = 0; k < 3; ++k) q[k] = a[k] + ab[k] * v + ac[k] * w;
  }
  const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
  return dx * dx + dy * dy + dz * dz;
}

// signed solid angle of triangle (a, b, c) seen from p (positive for outward-facing = counter-clockwise seen from outside)
HOLD_HD float tri_solid_angle(const float* p, const float* a, const float* b, const float* c) {
  const float ra[3] = {a[0] - p[0], a[1] - p[1], a[2] - p[2]}, rb[3] = {b[0] - p[0], b[1] - p[1], b[2] - p[2]};
  const float rc[3] = {c[0] - p[0], c[1] - p[1], c[2] - p[2]};
  const float la = sqrtf(dot3(ra, ra)), lb = sqrtf(dot3(rb, rb)), lc = sqrtf(dot3(rc, rc));
  const float det = ra[0] * (rb[1] * rc[2] - rb[2] * rc[1]) - ra[1] * (rb[0] * rc[2] - rb[2] * rc[0]) + ra[2] * (rb[0] * rc[1] - rb[1] * rc[0]);
  const float den = la * lb * lc + dot3(ra, rb) * lc + dot3(rb, rc) * la + dot3(rc, ra) * lb;
  return 2.0f * atan2f(det, den);
}

struct PointAcc {
  float best;     // min squared distance so far
  int best_f;     // its face (lowest index among equals)
  float omega;    // sum of solid angles
};
HOLD_HD void acc_init(PointAcc& s) { s.best = 3.0e38f, s.best_f = -1, s.omega = 0.f; }
HOLD_HD void acc_face(PointAcc& s, const float* p, const float* tri /*9 floats*/, int f) {
  const float d = tri_sqdist(p, tri, tri + 3, tri + 6);
  if (d < s.best) { s.best = d; s.best_f = f; }
  s.omega += tri_solid_angle(p, tri, tri + 3, tri + 6);
}
// signed distance: negative inside (volsdf_utils.py:180-186: sign = 1 - 2 * inside)
HOLD_HD float acc_sdf(const PointAcc& s) {
  const float w = s.omega * (1.0f / 12.566370614359172f);
  const bool inside = fabsf(w) > 0.5f;
  const float d = sqrtf(s.best);
  return inside ? -d : d;
}

}  // namespace meshsdf
}  // namespace hold
