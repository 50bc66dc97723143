// Exact K = 15 nearest MANO vertices (pytorch3d.ops.knn_points contract, call site model/mano/deformer.py:85) for points that
// walk along a ray, with two prunings that cannot change the result:
//  (1) seeding: the previous sample's 15 neighbours are re-ranked for the new point; their largest distance tau bounds the new
//      15th-nearest distance from above, so only vertices with d < tau (ties: lower index) can enter;
//  (2) clusters: the 778 vertices are held in 49 groups of 16 that are spatially compact (ordered once, on the canonical hand,
//      by dominant bone and Morton code: hold_node_set_rig); per frame each group has a centre c and a radius r of its POSED
//      members.  |p - v| >= |p - c| - r for every member, so a group with |p - c| > r + sqrt(tau) (plus a rounding margin)
//      holds no candidate and its 16 distance evaluations are skipped.  Near the hand ~90 % of the groups go, far from it ~70 %.
// Survivors are evaluated with the reference's float expression ((p - v)^2).sum() without FMA contraction and merged in
// lexicographic (distance, index) order — bit-identical to a full scan (tests/test_cpu_knn.py runs this header on the host
// against brute force, including duplicate vertices, samples on vertices and jumps that invalidate the seeds).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define HOLD_HD __host__ __device__ __forceinline__
#else
#ifndef HOLD_HD
#define HOLD_HD inline
#endif
#endif
#if defined(__CUDA_ARCH__)
#define HOLD_FADD(a, b) __fadd_rn((a), (b))
#define HOLD_FMUL(a, b) __fmul_rn((a), (b))
#define HOLD_DADD(a, b) __dadd_rn((a), (b))
#define HOLD_DMUL(a, b) __dmul_rn((a), (b))
#else
#define HOLD_FADD(a, b) ((a) + (b))   // host build uses -ffp-contract=off
#define HOLD_FMUL(a, b) ((a) * (b))
#define HOLD_DADD(a, b) ((a) + (b))
#define HOLD_DMUL(a, b) ((a) * (b))
#endif

namespace hold {
namespace knnc {

constexpr int kK = 15, kNV = 778, kCand = 48, kClSize = 16, kNCl = (kNV + kClSize - 1) / kClSize;   // 49 groups
// the K best (distance, index) pairs in lexicographic order; the MANO KNN uses TopK<15, float>, the point-cloud KNN
// (pointcloud_phases.h) K = 1 .. 32 in float and K = 1 in double
template <int K, typename T>
struct TopK {
  T d[K];
  int i[K];
};
using Top = TopK<kK, float>;
struct V4 { float x, y, z; int idx; };      // cluster-ordered vertex: position + ORIGINAL index (padding: idx < 0, far away)
struct Cl { float x, y, z, r; };            // centre, radius

// the reference's expression, no FMA contraction (KNN selection is sensitive to the last bit)
HOLD_HD float exact_dist(float vx, float vy, float vz, float px, float py, float pz) {
  const float dx = px - vx, dy = py - vy, dz = pz - vz;
  return HOLD_FADD(HOLD_FADD(HOLD_FMUL(dx, dx), HOLD_FMUL(dy, dy)), HOLD_FMUL(dz, dz));
}
// the same expression in double (the ICP correspondence search)
HOLD_HD double exact_dist(double vx, double vy, double vz, double px, double py, double pz) {
  const double dx = px - vx, dy = py - vy, dz = pz - vz;
  return HOLD_DADD(HOLD_DADD(HOLD_DMUL(dx, dx), HOLD_DMUL(dy, dy)), HOLD_DMUL(dz, dz));
}
template <int K, typename T>
HOLD_HD void insert(TopK<K, T>& r, T dist, int v) {   // replace the last entry, bubble up; order (distance, index)
  r.d[K - 1] = dist;
  r.i[K - 1] = v;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int k = K - 1; k > 0; --k) {
    const bool sw = (r.d[k] < r.d[k - 1]) || (r.d[k] == r.d[k - 1] && r.i[k] < r.i[k - 1]);
    if (sw) {
      const T td = r.d[k]; r.d[k] = r.d[k - 1]; r.d[k - 1] = td;
      const int ti = r.i[k]; r.i[k] = r.i[k - 1]; r.i[k - 1] = ti;
    }
  }
}
// group centre / radius from the cluster-ordered posed vertices (one call per group and frame)
HOLD_HD Cl make_cluster(const V4* members) {
  float sx = 0.f, sy = 0.f, sz = 0.f;
  int n = 0;
  for (int j = 0; j < kClSize; ++j)
    if (members[j].idx >= 0) { sx += members[j].x, sy += members[j].y, sz += members[j].z; ++n; }
  Cl c;
  const float inv = 1.0f / (float)(n > 0 ? n : 1);
  c.x = sx * inv, c.y = sy * inv, c.z = sz * inv;
  float r2 = 0.f;
  for (int j = 0; j < kClSize; ++j)
    if (members[j].idx >= 0) {
      const float dx = members[j].x - c.x, dy = members[j].y - c.y, dz = members[j].z - c.z;
      r2 = fmaxf(r2, dx * dx + dy * dy + dz * dz);
    }
  c.r = sqrtf(r2) * 1.000001f + 1e-20f;   // never below the true radius
  return c;
}
// full exact scan (first sample of a walk, or seeds invalidated by a large step)
HOLD_HD void full_scan(const V4* svc, float px, float py, float pz, Top& r) {
  for (int k = 0; k < kK; ++k) { r.d[k] = 3.0e38f; r.i[k] = 0x7fffffff; }
  for (int j = 0; j < kNCl * kClSize; ++j) {
    const V4 v = svc[j];
    if (v.idx < 0) continue;
    const float dist = exact_dist(v.x, v.y, v.z, px, py, pz);
    if (dist < r.d[kK - 1] || (dist == r.d[kK - 1] && v.idx < r.i[kK - 1])) insert(r, dist, v.idx);
  }
}
// r holds the previous sample's neighbours on entry, this sample's on exit.  sv: posed vertices in ORIGINAL order [778*3]
// (the seeds are original indices), svc / cl: cluster order and groups of this frame.  Returns the number of groups visited.
HOLD_HD int seeded_clustered(const float* sv, const V4* svc, const Cl* cl, float px, float py, float pz, Top& r, unsigned short* cand) {
  int seed[kK];
  for (int k = 0; k < kK; ++k) { seed[k] = r.i[k]; r.d[k] = 3.0e38f; r.i[k] = 0x7fffffff; }
  for (int s = 0; s < kK; ++s) insert(r, exact_dist(sv[3 * seed[s]], sv[3 * seed[s] + 1], sv[3 * seed[s] + 2], px, py, pz), seed[s]);
  const float tau = r.d[kK - 1];
  const int itau = r.i[kK - 1];
  const float st = sqrtf(tau);
  int cnt = 0, visited = 0;
  for (int k = 0; k < kNCl; ++k) {
    const Cl c = cl[k];
    const float dx = px - c.x, dy = py - c.y, dz = pz - c.z;
    const float dc2 = dx * dx + dy * dy + dz * dz;
    const float lim = c.r + st;
    if (dc2 > lim * lim * 1.00001f + 1e-30f) continue;   // every member is farther than tau (margin >> the roundings above)
    ++visited;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < kClSize; ++j) {
      const V4 v = svc[k * kClSize + j];
      const float dist = exact_dist(v.x, v.y, v.z, px, py, pz);   // padding members sit at 1e18: never below tau
      if (dist < tau || (dist == tau && v.idx < itau)) {
        if (cnt < kCand) cand[cnt] = (unsigned short)v.idx;
        ++cnt;
      }
    }
  }
  if (cnt > kCand) {   // seeds were poor (large step along the ray): exact full scan
    full_scan(svc, px, py, pz, r);
    return -1;
  }
  for (int c = 0; c < cnt; ++c) {
    const int v = cand[c];
    bool present = false;
    for (int k = 0; k < kK; ++k) present |= (r.i[k] == v);
    if (present) continue;
    const float dist = exact_dist(sv[3 * v], sv[3 * v + 1], sv[3 * v + 2], px, py, pz);
    if (dist < r.d[kK - 1] || (dist == r.d[kK - 1] && v < r.i[kK - 1])) insert(r, dist, v);
  }
  return visited;
}

// Host side of hold_node_set_rig: order of the vertices in which consecutive groups of 16 are spatially compact and stay so under
// articulation — by dominant bone (argmax of the skinning weights), then by Morton code of the canonical position.
inline void cluster_order(const float* cano /*[778,3]*/, const float* skin_w /*[778,16]*/, int n_joints, unsigned short* perm /*[kNCl*16]*/) {
  float lo[3] = {1e30f, 1e30f, 1e30f}, hi[3] = {-1e30f, -1e30f, -1e30f};
  for (int v = 0; v < kNV; ++v)
    for (int c = 0; c < 3; ++c) { lo[c] = fminf(lo[c], cano[3 * v + c]); hi[c] = fmaxf(hi[c], cano[3 * v + c]); }
  unsigned long long key[kNV];
  for (int v = 0; v < kNV; ++v) {
    int jb = 0;
    for (int j = 1; j < n_joints; ++j)
      if (skin_w[v * n_joints + j] > skin_w[v * n_joints + jb]) jb = j;
    unsigned long long m = 0;
    unsigned q[3];
    for (int c = 0; c < 3; ++c) {
      const float t = (cano[3 * v + c] - lo[c]) / fmaxf(hi[c] - lo[c], 1e-20f);
      q[c] = (unsigned)fminf(fmaxf(t * 1023.0f, 0.f), 1023.f);
    }
    for (int b = 9; b >= 0; --b)
      for (int c = 0; c < 3; ++c) m = (m << 1) | ((q[c] >> b) & 1u);
    key[v] = ((unsigned long long)jb << 40) | (m << 10) | (unsigned long long)v;
  }
  for (int a = 1; a < kNV; ++a) {   // insertion sort of 778 keys (set_rig runs once)
    const unsigned long long k = key[a];
    int b = a - 1;
    while (b >= 0 && key[b] > k) { key[b + 1] = key[b]; --b; }
    key[b + 1] = k;
  }
  for (int j = 0; j < kNCl * kClSize; ++j) perm[j] = (j < kNV) ? (unsigned short)(key[j] & 1023ull) : (unsigned short)0xFFFF;
}

}  // namespace knnc
}  // namespace hold
