// Host restatement of hold_decimate (hold_b200/csrc/decimate.cuh): the same rounds run sequentially over the same arithmetic
// (hold_b200/csrc/decimate_phases.h).  The stars come from a stable counting sort, the two selects from nth_element over the
// valid keys (they are unique, so both are well defined).  `reverse` visits the vertices, the half-edges and the collapses of
// every step in descending order: the result must not change, which is what lets the parallel rounds on the device match.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../hold_b200/csrc/decimate_phases.h"

using namespace hold::decim;

namespace {

constexpr int kMaxRounds = 1000;   // kDecMaxRounds

// stable counting sort of the live items by vertex: order[first[v] .. first[v + 1]) ascending
void stars(int V, const std::vector<int>& F, std::vector<int>& order, std::vector<int>& first) {
  const int n3 = (int)F.size();
  first.assign(V + 2, 0);
  for (int i = 0; i < n3; ++i) ++first[(F[i] >= 0 ? F[i] : V) + 1];
  for (int v = 0; v <= V; ++v) first[v + 1] += first[v];
  std::vector<int> pos(first.begin(), first.end() - 1);
  order.assign(n3, 0);
  for (int i = 0; i < n3; ++i) order[pos[F[i] >= 0 ? F[i] : V]++] = i;
}

// the k-th smallest of the valid keys; kNoKey - 1 (every valid key) when k >= their count
uint64_t kth(const std::vector<uint64_t>& keys, long k, long* n_valid) {
  std::vector<uint64_t> v;
  for (uint64_t x : keys)
    if (x != kNoKey) v.push_back(x);
  *n_valid = (long)v.size();
  if (k < 0 || k >= (long)v.size()) return kNoKey - 1;
  std::nth_element(v.begin(), v.begin() + k, v.end());
  return v[k];
}

template <typename Fn>
void visit(int n, int reverse, Fn&& fn) {
  if (reverse)
    for (int i = n - 1; i >= 0; --i) fn(i);
  else
    for (int i = 0; i < n; ++i) fn(i);
}

}  // namespace

// hold_decimate's contract; returns the number of rounds run
extern "C" int decimate_host(int V, const float* verts, int F, const int* faces, int target, float quality_threshold, int reverse,
                             float* verts_out, int* faces_out, int* V_out, int* F_out) {
  const int n3 = 3 * F;
  bool bad = false;
  for (int i = 0; i < n3; ++i) bad |= faces[i] < 0 || faces[i] >= V;
  if (bad || target >= F) {
    memcpy(verts_out, verts, sizeof(float) * 3 * (size_t)V);
    memcpy(faces_out, faces, sizeof(int) * (size_t)n3);
    *V_out = V, *F_out = F;
    return 0;
  }
  const double qthr = (double)quality_threshold;
  std::vector<float> P(verts, verts + 3 * (size_t)V), X(3 * (size_t)n3, 0.f);
  std::vector<int> Fw(faces, faces + n3), order, first, frozen(V);
  std::vector<double> Q(10 * (size_t)V);
  std::vector<uint64_t> key(n3), sel(n3), mA(V), mB(V);
  int F_live = F, rounds = 0;
  while (rounds < kMaxRounds && F_live > target) {
    stars(V, Fw, order, first);
    if (rounds == 0)
      visit(V, reverse, [&](int v) { vertex_quadric(v, Fw.data(), P.data(), order.data(), first.data(), Q.data() + 10 * (size_t)v); });
    visit(V, reverse, [&](int v) { frozen[v] = vertex_frozen(Fw.data(), order.data() + first[v], first[v + 1] - first[v]); });
    visit(n3, reverse, [&](int h) {
      key[h] = edge_candidate(h, Fw.data(), P.data(), Q.data(), order.data(), first.data(), frozen.data(), qthr, X.data() + 3 * (size_t)h);
    });
    long n_valid;
    kth(key, -1, &n_valid);
    const uint64_t cut = kth(key, (n_valid - 1) / 2, &n_valid);   // the median valid key
    visit(V, reverse, [&](int v) { mA[v] = vertex_min_key(v, Fw.data(), order.data(), first.data(), key.data(), cut); });
    visit(V, reverse, [&](int v) { mB[v] = ring_min(v, Fw.data(), order.data(), first.data(), mA.data()); });
    visit(V, reverse, [&](int v) { mA[v] = ring_min(v, Fw.data(), order.data(), first.data(), mB.data()); });
    visit(n3, reverse, [&](int h) {
      const uint64_t k = key[h];
      bool s = k <= cut;
      if (s) s = mA[Fw[h]] == k && mA[Fw[3 * (h / 3) + next_corner(h % 3)]] == k;
      sel[h] = s ? k : kNoKey;
    });
    const long need = (F_live - target + 1) / 2;
    long n_sel;
    const uint64_t cut2 = kth(sel, need - 1, &n_sel);
    const long collapses = std::min(n_sel, need);
    visit(n3, reverse, [&](int h) {
      if (sel[h] <= cut2) apply_collapse(h, Fw.data(), P.data(), Q.data(), order.data(), first.data(), X.data() + 3 * (size_t)h);
    });
    F_live -= 2 * (int)collapses;
    ++rounds;
    if (collapses == 0) break;
  }
  std::vector<int> vnew(V + 1, 0), fnew(F + 1, 0);
  for (int f = 0; f < F; ++f)
    if (Fw[3 * f] >= 0) {
      fnew[f] = 1;
      for (int k = 0; k < 3; ++k) vnew[Fw[3 * f + k]] = 1;
    }
  int nv = 0, nf = 0;
  for (int v = 0; v <= V; ++v) { const int t = vnew[v]; vnew[v] = nv; nv += t; }
  for (int f = 0; f <= F; ++f) { const int t = fnew[f]; fnew[f] = nf; nf += t; }
  for (int v = 0; v < V; ++v)
    if (vnew[v + 1] != vnew[v])
      for (int k = 0; k < 3; ++k) verts_out[3 * vnew[v] + k] = P[3 * (size_t)v + k];
  for (int f = 0; f < F; ++f)
    if (fnew[f + 1] != fnew[f])
      for (int k = 0; k < 3; ++k) faces_out[3 * fnew[f] + k] = vnew[Fw[3 * f + k]];
  *V_out = vnew[V], *F_out = fnew[F];
  return rounds;
}

// the phases one at a time, for the tests against numpy
extern "C" void plane_quadric_host(const double* p, double* q) { plane_quadric(p, p + 3, p + 6, q); }
extern "C" double edge_solve_host(const double* qa, const double* qb, const double* a, const double* b, double* x) {
  return edge_solve(qa, qb, a, b, x);
}
extern "C" double quadric_cost_host(const double* q, const double* x) { return quadric_cost(q, x); }
extern "C" uint64_t edge_key_host(double cost, int h) { return edge_key(cost, h); }
extern "C" double tri_quality_host(const double* p) { return tri_quality(p, p + 3, p + 6); }
