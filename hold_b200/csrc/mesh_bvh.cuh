// Signed distance of points to a triangle mesh through a linear BVH built on the device on every call (hold_mesh_sdf_bvh):
// the same bits as k_mesh_sdf in O(log F) work per point.  Arithmetic in mesh_bvh_phases.h.
//   build, per tree (one, or B when the vertices are batched): vertex box -> Morton codes of the face centroids (and the face
//   index check) -> stable radix sort (inverse_map.cuh's passes) -> Karras's internal nodes -> bottom-up refit, where integer
//   visit counters pick the second child's thread to build the parent from (left, right).  No floating-point atomic.
//   query: one thread per point, an explicit stack; the points whose fast winding number falls into the band are listed
//   (integer counter, any order) and k_bvh_band sums their exact solid angles over all faces in ascending face order.
#pragma once
#include "common.cuh"
#include "inverse_map.cuh"
#include "mesh_bvh_phases.h"

namespace hold {

constexpr int kBvhThreads = 128;

struct BvhArgs {
  int B, P, V, F, vstride, tstride;   // vstride: floats between frames' vertices (0 = shared); tstride: 1 = a tree per frame
  const float* points;
  const float* verts;
  const int* faces;
  float* sdf;
  int* face_idx;
  int* codes;                         // [trees, F] Morton codes in face order
  const int* sorted_codes;            // [F] of the tree being linked
  int* order;                         // [trees, F] faces in sorted order
  float4* nodes;                      // [trees, 2F, 4]
  int2* child;                        // [trees, F]
  int* parent;                        // [trees, 2F]
  int* visits;                        // [trees, F]
  float* bounds;                      // [trees, 8]
  int* state;                         // [0] = bad face index seen, [1] = band count
  int* band;                          // [B P]
  int* err;
};

struct BvhView {   // one tree, for the traversals of mesh_bvh_phases.h
  const float4* nodes;
  const int2* child;
  const int* order;
  const float* verts;
  const int* faces;
  int F;
  __device__ meshbvh::Node node(int n) const {
    meshbvh::Node o;
    float4* q = reinterpret_cast<float4*>(&o);
    const float4* s = nodes + 4 * (size_t)n;
    q[0] = __ldg(s), q[1] = __ldg(s + 1), q[2] = __ldg(s + 2), q[3] = __ldg(s + 3);
    return o;
  }
  __device__ void children(int n, int* l, int* r) const {
    const int2 c = __ldg(child + n);
    *l = c.x, *r = c.y;
  }
  __device__ int face(int n) const { return __ldg(order + n - (F - 1)); }
  __device__ void tri(int f, float* t) const {
    for (int e = 0; e < 3; ++e) {
      const int v = __ldg(faces + 3 * (size_t)f + e);
      t[3 * e] = __ldg(verts + 3 * (size_t)v), t[3 * e + 1] = __ldg(verts + 3 * (size_t)v + 1), t[3 * e + 2] = __ldg(verts + 3 * (size_t)v + 2);
    }
  }
};

// per tree (blockIdx.x): the box of all V vertices (min / max, any order gives the same bits)
__global__ void __launch_bounds__(1024) k_bvh_bounds(BvhArgs a) {
  __shared__ float s[32][6];
  const float* v = a.verts + (size_t)blockIdx.x * a.vstride;
  float m[6] = {3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f};
  for (int i = threadIdx.x; i < a.V; i += blockDim.x)
    for (int k = 0; k < 3; ++k) {
      const float x = v[3 * (size_t)i + k];
      m[k] = fminf(m[k], x), m[3 + k] = fmaxf(m[3 + k], x);
    }
  for (int o = 16; o > 0; o >>= 1)
    for (int k = 0; k < 3; ++k) {
      m[k] = fminf(m[k], __shfl_xor_sync(0xffffffffu, m[k], o));
      m[3 + k] = fmaxf(m[3 + k], __shfl_xor_sync(0xffffffffu, m[3 + k], o));
    }
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 6; ++k) s[threadIdx.x >> 5][k] = m[k];
  __syncthreads();
  if (threadIdx.x < 6) {
    float r = s[0][threadIdx.x];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = threadIdx.x < 3 ? fminf(r, s[w][threadIdx.x]) : fmaxf(r, s[w][threadIdx.x]);
    a.bounds[8 * blockIdx.x + threadIdx.x] = r;
  }
}

__device__ __forceinline__ bool bvh_face_ok(const BvhArgs& a, int f) {
  const int* t = a.faces + 3 * (size_t)f;
  return t[0] >= 0 && t[0] < a.V && t[1] >= 0 && t[1] < a.V && t[2] >= 0 && t[2] < a.V;
}

__device__ __forceinline__ void bvh_load_tri(const BvhArgs& a, const float* v, int f, float* t) {
  for (int e = 0; e < 3; ++e) {
    const int i = min(max(a.faces[3 * (size_t)f + e], 0), a.V - 1);   // a bad index was flagged; stay inside the array
    t[3 * e] = v[3 * (size_t)i], t[3 * e + 1] = v[3 * (size_t)i + 1], t[3 * e + 2] = v[3 * (size_t)i + 2];
  }
}

// codes[tree, f]; blockIdx.y = tree.  Tree 0 checks the face indices.
__global__ void __launch_bounds__(256) k_bvh_codes(BvhArgs a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
  if (f >= a.F) return;
  if (t == 0 && !bvh_face_ok(a, f)) {
    a.state[0] = 1;
    atomicOr(a.err, kErrBadSdfFace);
  }
  const float* bd = a.bounds + 8 * t;
  float lo[3], inv[3];
  for (int k = 0; k < 3; ++k) {
    const float e = bd[3 + k] - bd[k];
    lo[k] = bd[k], inv[k] = e > 0.f ? 1.0f / e : 0.f;
  }
  float tri[9];
  bvh_load_tri(a, a.verts + (size_t)t * a.vstride, f, tri);
  a.codes[(size_t)t * a.F + f] = meshbvh::morton_code(tri, tri + 3, tri + 6, lo, inv);
}

// internal nodes of one tree: children and parents (a.sorted_codes, a.child, a.parent point at the tree)
__global__ void __launch_bounds__(256) k_bvh_link(BvhArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) a.parent[0] = -1;
  if (i >= a.F - 1) return;
  int l, r;
  meshbvh::karras_children(a.sorted_codes, a.F, i, &l, &r);
  a.child[i] = make_int2(l, r);
  a.parent[l] = i, a.parent[r] = i;
}

__device__ __forceinline__ void bvh_store(float4* dst, const meshbvh::Node& o) {
  const float4* q = reinterpret_cast<const float4*>(&o);
  dst[0] = q[0], dst[1] = q[1], dst[2] = q[2], dst[3] = q[3];
}
__device__ __forceinline__ meshbvh::Node bvh_load_cg(const float4* src) {   // written by another CTA of this launch
  meshbvh::Node o;
  float4* q = reinterpret_cast<float4*>(&o);
  q[0] = __ldcg(src), q[1] = __ldcg(src + 1), q[2] = __ldcg(src + 2), q[3] = __ldcg(src + 3);
  return o;
}

// leaves, then up the tree: the second child to arrive builds the parent; blockIdx.y = tree
__global__ void __launch_bounds__(256) k_bvh_refit(BvhArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
  if (i >= a.F) return;
  const size_t tn = (size_t)t * 2 * a.F;
  float4* nodes = a.nodes + 4 * tn;
  const int2* child = a.child + (size_t)t * a.F;
  const int* parent = a.parent + tn;
  int* visits = a.visits + (size_t)t * a.F;
  float tri[9];
  bvh_load_tri(a, a.verts + (size_t)t * a.vstride, a.order[(size_t)t * a.F + i], tri);
  meshbvh::Node o;
  meshbvh::leaf_node(tri, tri + 3, tri + 6, o);
  int n = a.F - 1 + i;
  bvh_store(nodes + 4 * (size_t)n, o);
  for (;;) {
    const int p = parent[n];
    if (p < 0) return;
    __threadfence();
    if (atomicAdd(visits + p, 1) == 0) return;
    __threadfence();
    const int2 c = child[p];
    const meshbvh::Node L = bvh_load_cg(nodes + 4 * (size_t)c.x), R = bvh_load_cg(nodes + 4 * (size_t)c.y);
    meshbvh::merge_node(L, R, o);
    bvh_store(nodes + 4 * (size_t)p, o);
    n = p;
  }
}

// one thread per (frame blockIdx.y, point)
__global__ void __launch_bounds__(kBvhThreads) k_bvh_query(BvhArgs a) {
  const int b = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.P) return;
  const size_t ip = (size_t)b * a.P + p;
  if (a.state[0]) {   // an index outside [0, V): no tree
    a.sdf[ip] = __int_as_float(0x7fc00000);
    if (a.face_idx) a.face_idx[ip] = -1;
    return;
  }
  const int t = a.tstride * b;
  BvhView v{a.nodes + 4 * (size_t)t * 2 * a.F, a.child + (size_t)t * a.F, a.order + (size_t)t * a.F,
            a.verts + (size_t)b * a.vstride, a.faces, a.F};
  const float pt[3] = {a.points[3 * ip], a.points[3 * ip + 1], a.points[3 * ip + 2]};
  const meshbvh::Node root = v.node(0);
  int stack[meshbvh::kStack];
  float best = 3.0e38f;
  int best_f = -1;
  bool band = true;
  if (meshbvh::is_finite3(pt)) {   // else no face's tri_sqdist is below 3e38
    float scale = fmaxf(fmaxf(fabsf(pt[0]), fabsf(pt[1])), fabsf(pt[2]));
    for (int k = 0; k < 3; ++k) scale = fmaxf(scale, fmaxf(fabsf(root.lo[k]), fabsf(root.hi[k])));
    meshbvh::nearest(v, a.F, pt, scale, stack, best, best_f);
    const bool mesh_finite = meshbvh::is_finite3(root.lo) && meshbvh::is_finite3(root.hi) && isfinite(root.area);
    if (mesh_finite) {
      const float w = meshbvh::fast_winding(v, a.F, pt, stack) * (1.0f / 12.566370614359172f);
      band = meshbvh::in_band(w);
      a.sdf[ip] = meshbvh::signed_dist(best, fabsf(w) > 0.5f);
    }
  }
  if (band) {
    a.sdf[ip] = meshbvh::signed_dist(best, false);
    a.band[atomicAdd(a.state + 1, 1)] = (int)ip;
  }
  if (a.face_idx) a.face_idx[ip] = best_f;
}

// the listed points: omega summed over all faces in ascending order from 0, as k_mesh_sdf does
__global__ void __launch_bounds__(kBvhThreads) k_bvh_band(BvhArgs a) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.state[1]) return;
  const int ip = a.band[j], b = ip / a.P;
  const float* v = a.verts + (size_t)b * a.vstride;
  const float pt[3] = {a.points[3 * (size_t)ip], a.points[3 * (size_t)ip + 1], a.points[3 * (size_t)ip + 2]};
  meshsdf::PointAcc acc;
  meshsdf::acc_init(acc);
  for (int f = 0; f < a.F; ++f) {
    float tri[9];
    for (int e = 0; e < 3; ++e) {
      const int i = __ldg(a.faces + 3 * (size_t)f + e);
      tri[3 * e] = __ldg(v + 3 * (size_t)i), tri[3 * e + 1] = __ldg(v + 3 * (size_t)i + 1), tri[3 * e + 2] = __ldg(v + 3 * (size_t)i + 2);
    }
    acc.omega += meshsdf::tri_solid_angle(pt, tri, tri + 3, tri + 6);
  }
  // k_bvh_query stored sqrtf(best); acc_sdf of a zero distance gives the sign alone: -0 inside, +0 outside
  const float s = a.sdf[ip];
  acc.best = 0.f;
  a.sdf[ip] = signbit(meshsdf::acc_sdf(acc)) ? -fabsf(s) : fabsf(s);
}

}  // namespace hold
