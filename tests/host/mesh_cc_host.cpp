// Sequential host restatement of hold_largest_component (hold_b200/csrc/mesh_cc.cuh) over the same mesh_cc_phases.h: the joins
// in a caller-given face order (the device's order is whatever its threads make it), labels, areas, the per-component sums over
// a stable counting sort of the faces by label, the argmax and the compaction.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../hold_b200/csrc/mesh_cc_phases.h"

using namespace hold::meshcc;

namespace {

int cas(int* p, int r, int s) {
  const int old = p[r];
  if (old == r) p[r] = s;
  return old;
}

}  // namespace

// labels [V] after joining the faces' edges in the order face_order [F] (NULL: ascending)
extern "C" void cc_labels_host(int V, int F, const int* faces, const int* face_order, int* labels) {
  for (int v = 0; v < V; ++v) labels[v] = v;
  for (int i = 0; i < F; ++i) {
    const int f = face_order ? face_order[i] : i;
    cc_unite(labels, faces[3 * f], faces[3 * f + 1], cas);
    cc_unite(labels, faces[3 * f + 1], faces[3 * f + 2], cas);
  }
  std::vector<int> parent(labels, labels + V);
  for (int v = 0; v < V; ++v) labels[v] = cc_root(parent.data(), v);
}

extern "C" void cc_areas_host(const float* P, int F, const int* faces, float* area) {
  for (int f = 0; f < F; ++f) area[f] = face_area(P, faces, f);
}

// hold_largest_component's contract (F > 0, every index in [0, V)); also returns labels [V], area [F], sums [V] and the chosen label
extern "C" int cc_largest_host(int V, const float* P, int F, const int* faces, const int* face_order, float* verts_out,
                               int* faces_out, int* V_out, int* F_out, int* labels, float* area, double* sums) {
  cc_labels_host(V, F, faces, face_order, labels);
  cc_areas_host(P, F, faces, area);
  std::vector<int> first(V + 1, 0), order(F);
  for (int f = 0; f < F; ++f) ++first[labels[faces[3 * f]] + 1];
  for (int v = 0; v < V; ++v) first[v + 1] += first[v];
  std::vector<int> pos(first.begin(), first.end() - 1);
  for (int f = 0; f < F; ++f) order[pos[labels[faces[3 * f]]]++] = f;
  int best = -1;
  for (int v = 0; v < V; ++v) {
    sums[v] = cc_sum(area, order.data() + first[v], first[v + 1] - first[v]);
    if (best < 0 || cc_before(sums[v], v, sums[best], best)) best = v;
  }
  std::vector<int> vnew(V + 1, 0);
  int nf = 0;
  for (int f = 0; f < F; ++f)
    if (labels[faces[3 * f]] == best)
      for (int k = 0; k < 3; ++k) vnew[faces[3 * f + k]] = 1;
  int nv = 0;
  for (int v = 0; v <= V; ++v) { const int t = vnew[v]; vnew[v] = nv; nv += t; }
  for (int v = 0; v < V; ++v)
    if (vnew[v + 1] != vnew[v]) memcpy(verts_out + 3 * (size_t)vnew[v], P + 3 * (size_t)v, 3 * sizeof(float));
  for (int f = 0; f < F; ++f)
    if (labels[faces[3 * f]] == best) {
      for (int k = 0; k < 3; ++k) faces_out[3 * nf + k] = vnew[faces[3 * f + k]];
      ++nf;
    }
  *V_out = vnew[V], *F_out = nf;
  return best;
}

// np.argmax's order, for the tests of NaN and ties
extern "C" int cc_before_host(double s, int l, double t, int m) { return cc_before(s, l, t, m); }
