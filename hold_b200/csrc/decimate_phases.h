// Arithmetic of the quadric edge-collapse decimation (decimate.cuh, hold_decimate), compiled for the device and for the host
// (tests/host/decimate_host.cpp runs the same rounds sequentially over these functions).  Garland-Heckbert quadric error
// metrics, restated, not meshlab's code: meshlab collapses in sequential greedy order, these rounds collapse an independent set
// of cheap edges at a time, so the results are held to geometry rather than to meshlab's output (DESIGN.md §6).
//
// Everything is double without FMA contraction (HOLD_DADD / HOLD_DMUL, as knnc::exact_dist), so the device and a g++ build with
// -ffp-contract=off give the same bits.  A vertex's star is the list of its (face, corner) items 3 f + c in ascending order,
// order[first[v] .. first[v + 1]), as inverse_map.cuh builds it.  A dead face has -1 at its three corners.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "knn_phases.h"   // HOLD_HD, HOLD_DADD, HOLD_DMUL

namespace hold {
namespace decim {

constexpr int kMaxStar = 24;            // a vertex with a larger star never moves; no collapse makes a larger one
constexpr double kDetRel = 1e-10;       // |det A| <= kDetRel max|A_ij|^3: the optimal position is not solved for
constexpr uint64_t kNoKey = ~0ull;      // not a candidate; every valid key is smaller (its high word is a non-negative float)

HOLD_HD int next_corner(int c) { return c == 2 ? 0 : c + 1; }
HOLD_HD int prev_corner(int c) { return c == 0 ? 2 : c - 1; }

HOLD_HD double dot3(const double* a, const double* b) {
  return HOLD_DADD(HOLD_DADD(HOLD_DMUL(a[0], b[0]), HOLD_DMUL(a[1], b[1])), HOLD_DMUL(a[2], b[2]));
}

// (p1 - p0) x (p2 - p0): twice the area, along the face's normal
HOLD_HD void tri_normal(const double* p0, const double* p1, const double* p2, double* n) {
  const double e1[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
  const double e2[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
  n[0] = HOLD_DADD(HOLD_DMUL(e1[1], e2[2]), -HOLD_DMUL(e1[2], e2[1]));
  n[1] = HOLD_DADD(HOLD_DMUL(e1[2], e2[0]), -HOLD_DMUL(e1[0], e2[2]));
  n[2] = HOLD_DADD(HOLD_DMUL(e1[0], e2[1]), -HOLD_DMUL(e1[1], e2[0]));
}

// The area-weighted plane quadric A (n, d)(n, d)^T of a face, n the unit normal, d = -n . p0, A the area; stored as the upper
// triangle of the symmetric 4x4 in row order: xx xy xz xw yy yz yw zz zw ww.  A face of zero area has the zero quadric.
HOLD_HD void plane_quadric(const double* p0, const double* p1, const double* p2, double* q) {
  double n[3];
  tri_normal(p0, p1, p2, n);
  const double len2 = dot3(n, n);
  if (!(len2 > 0.0)) {
    for (int k = 0; k < 10; ++k) q[k] = 0.0;
    return;
  }
  const double len = sqrt(len2);
  const double a[4] = {n[0] / len, n[1] / len, n[2] / len, 0.0};
  const double pa[4] = {a[0], a[1], a[2], -dot3(a, p0)};
  const double w = HOLD_DMUL(0.5, len);
  int k = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = i; j < 4; ++j) q[k++] = HOLD_DMUL(w, HOLD_DMUL(pa[i], pa[j]));
}

// x^T Q x for x = (x, y, z, 1), the terms added in row order
HOLD_HD double quadric_cost(const double* q, const double* x) {
  double t = HOLD_DMUL(q[0], HOLD_DMUL(x[0], x[0]));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[1], HOLD_DMUL(x[0], x[1]))));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[2], HOLD_DMUL(x[0], x[2]))));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[3], x[0])));
  t = HOLD_DADD(t, HOLD_DMUL(q[4], HOLD_DMUL(x[1], x[1])));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[5], HOLD_DMUL(x[1], x[2]))));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[6], x[1])));
  t = HOLD_DADD(t, HOLD_DMUL(q[7], HOLD_DMUL(x[2], x[2])));
  t = HOLD_DADD(t, HOLD_DMUL(2.0, HOLD_DMUL(q[8], x[2])));
  return HOLD_DADD(t, q[9]);
}

HOLD_HD double det_term(double a, double b, double c, double d) { return HOLD_DADD(HOLD_DMUL(a, b), -HOLD_DMUL(c, d)); }

// The collapse of an edge (a, b) with quadrics qa, qb: Q = qa + qb, x = the position that minimises x^T Q x (the 3x3 system
// solved by cofactors); when |det| is below kDetRel max|A_ij|^3 or the solution is not finite, the cheapest of a, b and the
// midpoint, ties in that order.  Returns the cost, clamped at 0.
HOLD_HD double edge_solve(const double* qa, const double* qb, const double* a, const double* b, double* x) {
  double q[10];
  for (int k = 0; k < 10; ++k) q[k] = HOLD_DADD(qa[k], qb[k]);
  const double c00 = det_term(q[4], q[7], q[5], q[5]), c01 = det_term(q[5], q[2], q[1], q[7]), c02 = det_term(q[1], q[5], q[4], q[2]);
  const double c11 = det_term(q[0], q[7], q[2], q[2]), c12 = det_term(q[1], q[2], q[0], q[5]), c22 = det_term(q[0], q[4], q[1], q[1]);
  const double det = HOLD_DADD(HOLD_DADD(HOLD_DMUL(q[0], c00), HOLD_DMUL(q[1], c01)), HOLD_DMUL(q[2], c02));
  const double s = fmax(fmax(fmax(fabs(q[0]), fabs(q[1])), fmax(fabs(q[2]), fabs(q[4]))), fmax(fabs(q[5]), fabs(q[7])));
  if (s > 0.0 && fabs(det) > HOLD_DMUL(kDetRel, HOLD_DMUL(s, HOLD_DMUL(s, s)))) {
    const double r[3] = {-q[3], -q[6], -q[8]};
    const double c0[3] = {c00, c01, c02}, c1[3] = {c01, c11, c12}, c2[3] = {c02, c12, c22};
    const double y[3] = {dot3(c0, r) / det, dot3(c1, r) / det, dot3(c2, r) / det};
    if (isfinite(y[0]) && isfinite(y[1]) && isfinite(y[2])) {
      const double cost = quadric_cost(q, y);
      x[0] = y[0], x[1] = y[1], x[2] = y[2];
      return fmax(cost, 0.0);
    }
  }
  const double m[3] = {HOLD_DMUL(0.5, HOLD_DADD(a[0], b[0])), HOLD_DMUL(0.5, HOLD_DADD(a[1], b[1])), HOLD_DMUL(0.5, HOLD_DADD(a[2], b[2]))};
  double best = fmax(quadric_cost(q, a), 0.0);
  x[0] = a[0], x[1] = a[1], x[2] = a[2];
  const double cb = fmax(quadric_cost(q, b), 0.0);
  if (cb < best) best = cb, x[0] = b[0], x[1] = b[1], x[2] = b[2];
  const double cm = fmax(quadric_cost(q, m), 0.0);
  if (cm < best) best = cm, x[0] = m[0], x[1] = m[1], x[2] = m[2];
  return best;
}

// high word: the bits of float(cost), monotone for cost >= 0; low word: the half-edge id.  A total order of the edges that
// depends on the mesh alone.
HOLD_HD uint64_t edge_key(double cost, int h) {
  const float c = (float)cost;
  uint32_t bits;
  memcpy(&bits, &c, sizeof(bits));
  return ((uint64_t)bits << 32) | (uint32_t)h;
}

// 4 sqrt(3) A / (l0^2 + l1^2 + l2^2): 1 for an equilateral triangle, 0 for a degenerate one
HOLD_HD double tri_quality(const double* p0, const double* p1, const double* p2) {
  double n[3];
  tri_normal(p0, p1, p2, n);
  const double e0[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
  const double e1[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double e2[3] = {p0[0] - p2[0], p0[1] - p2[1], p0[2] - p2[2]};
  const double l2 = HOLD_DADD(HOLD_DADD(dot3(e0, e0), dot3(e1, e1)), dot3(e2, e2));
  if (!(l2 > 0.0)) return 0.0;
  return HOLD_DMUL(3.4641016151377544, sqrt(dot3(n, n))) / l2;   // 2 sqrt(3) |n|, |n| = 2 A
}

HOLD_HD void load3(const float* P, int v, double* p) { p[0] = P[3 * v], p[1] = P[3 * v + 1], p[2] = P[3 * v + 2]; }

// A vertex never moves when its star is empty or larger than kMaxStar, touches a degenerate face, lies on an edge without
// exactly one reverse half-edge (a boundary or non-manifold edge), or is not one closed fan (two fans pinched at the vertex).
HOLD_HD bool vertex_frozen(const int* F, const int* it, int n) {
  if (n == 0 || n > kMaxStar) return true;
  for (int s = 0; s < n; ++s) {
    const int f = it[s] / 3, c = it[s] % 3, v = F[it[s]];
    const int nx = F[3 * f + next_corner(c)], pv = F[3 * f + prev_corner(c)];
    if (nx == v || pv == v || nx == pv) return true;
    int out_nx = 0, in_nx = 0;
    for (int t = 0; t < n; ++t) {
      const int g = it[t] / 3, d = it[t] % 3;
      out_nx += F[3 * g + next_corner(d)] == nx;
      in_nx += F[3 * g + prev_corner(d)] == nx;
    }
    if (out_nx != 1 || in_nx != 1) return true;   // each edge v-w is v->w once and w->v once
  }
  // one fan: from face 0, the face that holds nx->v follows the one that holds v->nx
  int cur = 0, steps = 0;
  do {
    const int nx = F[3 * (it[cur] / 3) + next_corner(it[cur] % 3)];
    int t = 0;
    while (F[3 * (it[t] / 3) + prev_corner(it[t] % 3)] != nx) ++t;
    cur = t, ++steps;
  } while (cur != 0 && steps <= n);
  return steps != n;
}

// The half-edge h = 3 f + c, from u = F[h] to v: a candidate when u < v (one key per edge) and the collapse (u, v) -> x is
// valid.  Returns its key (kNoKey: none) and writes x, rounded to float as the vertex will hold it.  Valid when
//  - neither end is frozen;
//  - the link condition holds: u and v have exactly two common neighbours;
//  - no vertex is left with valence < 3 (the merged vertex, and the two common neighbours, whose stars lose a face);
//  - the merged star has at most kMaxStar faces;
//  - no surviving face of star(u) + star(v) flips (n_new . n_old <= 0 rejects, so does a face that becomes degenerate);
//  - the worst quality of the new faces is at least min(qthr, the worst quality of the old star).
HOLD_HD uint64_t edge_candidate(int h, const int* F, const float* P, const double* Q, const int* order, const int* first,
                                const int* frozen, double qthr, float* x_out) {
  const int f = h / 3, c = h % 3, u = F[h];
  if (u < 0) return kNoKey;
  const int v = F[3 * f + next_corner(c)];
  if (!(u < v) || frozen[u] || frozen[v]) return kNoKey;
  const int* sa = order + first[u];
  const int* sb = order + first[v];
  const int na = first[u + 1] - first[u], nb = first[v + 1] - first[v];
  if (na + nb - 4 > kMaxStar || na + nb - 4 < 3) return kNoKey;
  int common = 0;
  for (int i = 0; i < na; ++i) {
    const int w = F[3 * (sa[i] / 3) + next_corner(sa[i] % 3)];
    for (int j = 0; j < nb; ++j)
      if (F[3 * (sb[j] / 3) + next_corner(sb[j] % 3)] == w) {
        if (first[w + 1] - first[w] <= 3) return kNoKey;
        ++common;
      }
  }
  if (common != 2) return kNoKey;
  double pu[3], pv[3], xd[3];
  load3(P, u, pu), load3(P, v, pv);
  const double cost = edge_solve(Q + 10 * (size_t)u, Q + 10 * (size_t)v, pu, pv, xd);
  float xf[3] = {(float)xd[0], (float)xd[1], (float)xd[2]};
  const double x[3] = {xf[0], xf[1], xf[2]};
  double q_old = 1e300, q_new = 1e300;
  for (int side = 0; side < 2; ++side) {
    const int* s = side ? sb : sa;
    const int n = side ? nb : na, me = side ? v : u, other = side ? u : v;
    for (int i = 0; i < n; ++i) {
      const int g = s[i] / 3;
      double p[3][3], pn[3][3];
      bool dying = false;
      for (int k = 0; k < 3; ++k) {
        const int w = F[3 * g + k];
        load3(P, w, p[k]);
        dying |= w == other;
        for (int e = 0; e < 3; ++e) pn[k][e] = w == me ? x[e] : p[k][e];
      }
      q_old = fmin(q_old, tri_quality(p[0], p[1], p[2]));
      if (dying) continue;
      double n0[3], n1[3];
      tri_normal(p[0], p[1], p[2], n0);
      tri_normal(pn[0], pn[1], pn[2], n1);
      if (!(dot3(n0, n1) > 0.0)) return kNoKey;
      q_new = fmin(q_new, tri_quality(pn[0], pn[1], pn[2]));
    }
  }
  if (q_new < fmin(qthr, q_old)) return kNoKey;
  x_out[0] = xf[0], x_out[1] = xf[1], x_out[2] = xf[2];
  return edge_key(cost, h);
}

// Vertex v's quadric: the plane quadrics of its star's faces added in ascending face order
HOLD_HD void vertex_quadric(int v, const int* F, const float* P, const int* order, const int* first, double* q) {
  for (int k = 0; k < 10; ++k) q[k] = 0.0;
  for (int e = first[v]; e < first[v + 1]; ++e) {
    const int g = order[e] / 3;
    double p[3][3], fq[10];
    for (int k = 0; k < 3; ++k) load3(P, F[3 * g + k], p[k]);
    plane_quadric(p[0], p[1], p[2], fq);
    for (int k = 0; k < 10; ++k) q[k] = HOLD_DADD(q[k], fq[k]);
  }
}

// m(v): the smallest key <= cut of the edges at v (each edge's key sits on its half-edge from the smaller id)
HOLD_HD uint64_t vertex_min_key(int v, const int* F, const int* order, const int* first, const uint64_t* key, uint64_t cut) {
  uint64_t m = kNoKey;
  for (int e = first[v]; e < first[v + 1]; ++e) {
    const int i = order[e], f = i / 3, c = i % 3;
    const uint64_t k0 = key[i], k1 = key[3 * f + prev_corner(c)];
    if (k0 <= cut && k0 < m) m = k0;
    if (k1 <= cut && k1 < m) m = k1;
  }
  return m;
}

// the minimum of in[] over v's closed 1-ring
HOLD_HD uint64_t ring_min(int v, const int* F, const int* order, const int* first, const uint64_t* in) {
  uint64_t m = in[v];
  for (int e = first[v]; e < first[v + 1]; ++e) {
    const int i = order[e], f = i / 3, c = i % 3;
    const uint64_t a = in[F[3 * f + next_corner(c)]], b = in[F[3 * f + prev_corner(c)]];
    m = a < m ? a : m;
    m = b < m ? b : m;
  }
  return m;
}

// The collapse of half-edge h's edge (u, v) -> x: u takes x and Q_u + Q_v, the two faces on the edge die, the other faces of
// star(v) take u for v.  Touches star(u) + star(v) and Q_u, P_u only.
HOLD_HD void apply_collapse(int h, int* F, float* P, double* Q, const int* order, const int* first, const float* x) {
  const int f = h / 3, u = F[h], v = F[3 * f + next_corner(h % 3)];
  P[3 * u] = x[0], P[3 * u + 1] = x[1], P[3 * u + 2] = x[2];
  for (int k = 0; k < 10; ++k) Q[10 * (size_t)u + k] = HOLD_DADD(Q[10 * (size_t)u + k], Q[10 * (size_t)v + k]);
  for (int e = first[v]; e < first[v + 1]; ++e) {
    const int i = order[e], g = i / 3;
    if (F[3 * g] == u || F[3 * g + 1] == u || F[3 * g + 2] == u) F[3 * g] = F[3 * g + 1] = F[3 * g + 2] = -1;
    else F[i] = u;
  }
}

}  // namespace decim
}  // namespace hold
