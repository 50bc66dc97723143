// Arithmetic of the largest-component selection (mesh_cc.cuh, hold_largest_component), compiled for the host as well
// (tests/host/mesh_cc_host.cpp).  The selection is bit for bit what hold_b200.meshing.largest_component computes with scipy and
// numpy, the reference's trimesh.split(only_watertight=False) + argmax of the component areas (utils/meshing.py:58-70):
//   * graph: vertices joined by the face edges (0,1), (1,2), (2,0); a face belongs to the component of its first vertex;
//   * labels: a component is labelled by its smallest vertex id.  scipy numbers components in that same order, so comparing
//     labels compares scipy's numbers;
//   * area: per face in float32, as numpy's cross and norm round it: a = v1 - v0, b = v2 - v0, the cross components
//     fl(fl(a_i b_j) - fl(a_j b_i)), then 0.5 sqrt(fl(fl(x^2 + y^2) + z^2));
//   * sums: per component in double, in ascending face order (np.bincount);
//   * choice: np.argmax, the first NaN if any, else the first maximum: ties go to the smaller label.
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
namespace meshcc {

// float32 operations with no contraction into FMA on the device; the host build uses -ffp-contract=off
#if defined(__CUDA_ARCH__)
HOLD_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
HOLD_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
HOLD_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
HOLD_HD float fsqrt(float a) { return __fsqrt_rn(a); }
#else
HOLD_HD float fmul(float a, float b) { return a * b; }
HOLD_HD float fadd(float a, float b) { return a + b; }
HOLD_HD float fsub(float a, float b) { return a - b; }
HOLD_HD float fsqrt(float a) { return sqrtf(a); }
#endif

// 0.5 |(v1 - v0) x (v2 - v0)| of face f, as numpy computes it in float32
HOLD_HD float face_area(const float* P, const int* F, int f) {
  const float* v0 = P + 3 * (size_t)F[3 * (size_t)f];
  const float* v1 = P + 3 * (size_t)F[3 * (size_t)f + 1];
  const float* v2 = P + 3 * (size_t)F[3 * (size_t)f + 2];
  const float a[3] = {fsub(v1[0], v0[0]), fsub(v1[1], v0[1]), fsub(v1[2], v0[2])};
  const float b[3] = {fsub(v2[0], v0[0]), fsub(v2[1], v0[1]), fsub(v2[2], v0[2])};
  const float x = fsub(fmul(a[1], b[2]), fmul(a[2], b[1]));
  const float y = fsub(fmul(a[2], b[0]), fmul(a[0], b[2]));
  const float z = fsub(fmul(a[0], b[1]), fmul(a[1], b[0]));
  return fmul(0.5f, fsqrt(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z))));
}

// The root of x's tree, halving the path on the way (ECL-CC's find with pointer jumping).  Every parent is at most its child
// and lies in the child's component, so a stale read only shortens less, and every write keeps both properties.  `Ptr` is a plain
// pointer on the host and a volatile one on the device, where other threads hook and halve concurrently.
template <typename Ptr>
HOLD_HD int cc_find(Ptr parent, int x) {
  int cur = parent[x];
  if (cur != x) {
    int prev = x, next;
    while (cur > (next = parent[cur])) {
      parent[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// The root of x's tree without writing: the labels pass, once every join is done.  Halving there could overwrite a vertex's
// final label with an ancestor that is not the root.
template <typename Ptr>
HOLD_HD int cc_root(Ptr parent, int x) {
  int next;
  while ((next = parent[x]) != x) x = next;
  return x;
}

// Joins the components of a and b: the larger root is hung under the smaller one by compare-and-swap, cas(&parent[r], r, s)
// returning the old value; on a lost race the new parent of r is tried next.  Once every edge is joined, each component has
// one root, its smallest vertex (that vertex's parent can be neither smaller nor another vertex), whatever the order of the
// joins.
template <typename Ptr, typename Cas>
HOLD_HD void cc_unite(Ptr parent, int a, int b, Cas&& cas) {
  int ra = cc_find(parent, a), rb = cc_find(parent, b);
  while (ra != rb) {
    if (ra < rb) {
      const int old = cas(parent, rb, ra);
      if (old == rb) break;
      rb = old;
    } else {
      const int old = cas(parent, ra, rb);
      if (old == ra) break;
      ra = old;
    }
  }
}

// np.argmax's order: is component (s, l) chosen before (t, m)?  The first NaN wins, else the larger sum, ties to the smaller
// label.  A total order on distinct labels, so any reduction tree picks the same component.
HOLD_HD bool cc_before(double s, int l, double t, int m) {
  const bool ns = s != s, nt = t != t;
  if (ns || nt) return ns && (!nt || l < m);
  return s > t || (s == t && l < m);
}

// the double sum of the areas of one component's faces, items[0, n) in ascending face order, as np.bincount adds them
HOLD_HD double cc_sum(const float* area, const int* items, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += (double)area[items[i]];
  return s;
}

}  // namespace meshcc
}  // namespace hold
