// Sequential host restatement of hold_mesh_sdf_bvh (hold_b200/csrc/mesh_bvh.cuh) over the same mesh_bvh_phases.h: Morton codes,
// a stable sort by (code, face), Karras's links, a post-order refit from (left, right), and the query with its trust band.
#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

#include "../../hold_b200/csrc/mesh_bvh_phases.h"

using namespace hold;
using meshbvh::Node;

namespace {

struct Tree {
  int F = 0;
  std::vector<int> codes, order;      // codes in sorted order; faces in sorted order
  std::vector<int> left, right;       // [F-1]
  std::vector<Node> nodes;            // [2F-1]
  const float* verts = nullptr;
  const int* faces = nullptr;
  Node node(int n) const { return nodes[n]; }
  void children(int n, int* l, int* r) const { *l = left[n], *r = right[n]; }
  int face(int n) const { return order[n - (F - 1)]; }
  void tri(int f, float* t) const {
    for (int e = 0; e < 3; ++e)
      for (int k = 0; k < 3; ++k) t[3 * e + k] = verts[3 * faces[3 * f + e] + k];
  }
};

void refit(Tree& t, int n) {
  if (n >= t.F - 1) {
    float tri[9];
    t.tri(t.face(n), tri);
    meshbvh::leaf_node(tri, tri + 3, tri + 6, t.nodes[n]);
    return;
  }
  refit(t, t.left[n]);
  refit(t, t.right[n]);
  meshbvh::merge_node(t.nodes[t.left[n]], t.nodes[t.right[n]], t.nodes[n]);
}

void build(Tree& t, int V, int F, const float* verts, const int* faces) {
  t.F = F, t.verts = verts, t.faces = faces;
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f}, inv[3];
  for (int i = 0; i < V; ++i)
    for (int k = 0; k < 3; ++k) lo[k] = fminf(lo[k], verts[3 * i + k]), hi[k] = fmaxf(hi[k], verts[3 * i + k]);
  for (int k = 0; k < 3; ++k) {
    const float e = hi[k] - lo[k];
    inv[k] = e > 0.f ? 1.0f / e : 0.f;
  }
  std::vector<int> code(F);
  for (int f = 0; f < F; ++f) {
    float tri[9];
    t.tri(f, tri);
    code[f] = meshbvh::morton_code(tri, tri + 3, tri + 6, lo, inv);
  }
  t.order.resize(F);
  std::iota(t.order.begin(), t.order.end(), 0);
  std::stable_sort(t.order.begin(), t.order.end(), [&](int a, int b) { return code[a] < code[b]; });
  t.codes.resize(F);
  for (int i = 0; i < F; ++i) t.codes[i] = code[t.order[i]];
  t.left.assign(std::max(F - 1, 0), -1), t.right.assign(std::max(F - 1, 0), -1);
  for (int i = 0; i < F - 1; ++i) meshbvh::karras_children(t.codes.data(), F, i, &t.left[i], &t.right[i]);
  t.nodes.resize(2 * F - 1);
  refit(t, 0);
}

}  // namespace

extern "C" {

int bvh_morton_host(int F, const float* tris, const float* lo, const float* inv, int* codes) {
  for (int f = 0; f < F; ++f) codes[f] = meshbvh::morton_code(tris + 9 * f, tris + 9 * f + 3, tris + 9 * f + 6, lo, inv);
  return 0;
}

int bvh_karras_host(int F, const int* sorted_codes, int* left, int* right) {
  for (int i = 0; i < F - 1; ++i) meshbvh::karras_children(sorted_codes, F, i, left + i, right + i);
  return 0;
}

// lower[i] = box_lower(box of triangle i, p_i, scale_i), d[i] = tri_sqdist(p_i, triangle i)
int bvh_bound_host(int N, const float* tris, const float* pts, const float* scale, float* lower, float* d) {
  for (int i = 0; i < N; ++i) {
    const float *a = tris + 9 * i, *p = pts + 3 * i;
    Node o;
    meshbvh::leaf_node(a, a + 3, a + 6, o);
    lower[i] = meshbvh::box_lower(o.lo, o.hi, p, scale[i]);
    d[i] = meshsdf::tri_sqdist(p, a, a + 3, a + 6);
  }
  return 0;
}

// the tree of one mesh: order [F], left / right [F-1], nodes [2F-1][16]
int bvh_build_host(int V, int F, const float* verts, const int* faces, int* order, int* left, int* right, float* nodes) {
  Tree t;
  build(t, V, F, verts, faces);
  std::copy(t.order.begin(), t.order.end(), order);
  std::copy(t.left.begin(), t.left.end(), left);
  std::copy(t.right.begin(), t.right.end(), right);
  for (int n = 0; n < 2 * F - 1; ++n) std::copy((const float*)&t.nodes[n], (const float*)&t.nodes[n] + 16, nodes + 16 * n);
  return 0;
}

// sdf / face_idx as k_bvh_query + k_bvh_band compute them; band[p] = 1 if the exact sum decided; w_fast / w_exact (nullable) the
// winding numbers (NaN where the fast one was not computed)
int bvh_sdf_host(int P, int V, int F, const float* points, const float* verts, const int* faces, float* sdf, int* face_idx, int* band,
                 float* w_fast, float* w_exact) {
  Tree t;
  build(t, V, F, verts, faces);
  const Node root = t.nodes[0];
  int stack[meshbvh::kStack];
  for (int i = 0; i < P; ++i) {
    const float* p = points + 3 * i;
    float best = 3.0e38f, w = NAN;
    int best_f = -1;
    bool in_band = true;
    if (meshbvh::is_finite3(p)) {
      float scale = fmaxf(fmaxf(fabsf(p[0]), fabsf(p[1])), fabsf(p[2]));
      for (int k = 0; k < 3; ++k) scale = fmaxf(scale, fmaxf(fabsf(root.lo[k]), fabsf(root.hi[k])));
      meshbvh::nearest(t, F, p, scale, stack, best, best_f);
      if (meshbvh::is_finite3(root.lo) && meshbvh::is_finite3(root.hi) && std::isfinite(root.area)) {
        w = meshbvh::fast_winding(t, F, p, stack) * (1.0f / 12.566370614359172f);
        in_band = meshbvh::in_band(w);
      }
    }
    meshsdf::PointAcc acc;
    acc_init(acc);
    if (in_band || w_exact) {
      for (int f = 0; f < F; ++f) {
        float tri[9];
        t.tri(f, tri);
        acc.omega += meshsdf::tri_solid_angle(p, tri, tri + 3, tri + 6);
      }
    }
    acc.best = best, acc.best_f = best_f;
    sdf[i] = in_band ? meshsdf::acc_sdf(acc) : meshbvh::signed_dist(best, fabsf(w) > 0.5f);
    face_idx[i] = best_f;
    band[i] = in_band;
    if (w_fast) w_fast[i] = w;
    if (w_exact) w_exact[i] = acc.omega * (1.0f / 12.566370614359172f);
  }
  return 0;
}

}  // extern "C"
