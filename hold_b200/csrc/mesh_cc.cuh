// The connected component of largest surface area (hold_largest_component): the step of the reference's generate_mesh that
// trimesh.split + argmax of the areas performs (utils/meshing.py:58-70), on the device and bit for bit what
// hold_b200.meshing.largest_component gives.  Arithmetic and rules in mesh_cc_phases.h.
//
//  1. union-find over the face edges: integer compare-and-swap hooks the larger root under the smaller, finds halve their
//     paths; then, in a kernel of its own that only reads the forest, every vertex's label is its root, its component's
//     smallest vertex id, whatever the thread timing;
//  2. face areas in float32, each face keyed by its first vertex's label;
//  3. per-component sums in double in ascending face order, through inverse_map (keys = the face labels), one thread per
//     label.  The dominant component makes its thread's sum serial: about F double adds;
//  4. the argmax in one CTA, by meshcc::cc_before (a total order, so the reduction order does not matter);
//  5. compaction: flags, k_im_scan, the kept vertices in ascending old id and the kept faces in input order, remapped.
// Launches only, then one host read of the two output sizes.  No floating-point atomic: the only atomics are the integer
// compare-and-swaps of the hooking and the error flags.  A face index outside [0, V) flags the call: every later kernel
// skips its work, the output is empty and the device error word is set.
#pragma once
#include "common.cuh"
#include "inverse_map.cuh"
#include "mesh_cc_phases.h"

namespace hold {

constexpr int kCcThreads = 256, kCcArgmaxThreads = 1024;

struct CcState {
  int bad;    // a face index outside [0, V)
  int best;   // the chosen component's label
};

// parent[v] = v; faces checked
__global__ void k_cc_init(int V, int n3, const int* __restrict__ faces, int* __restrict__ parent, CcState* st, int* err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V) parent[i] = i;
  if (i < n3) {
    const int v = faces[i];
    if (v < 0 || v >= V) {
      atomicOr(&st->bad, 1);
      atomicOr(err, kErrBadCcFace);
    }
  }
}

// edges (0,1) and (1,2) of each face; (2,0) joins nothing they have not joined
__global__ void __launch_bounds__(kCcThreads) k_cc_unite(int F, const int* __restrict__ faces, int* parent, const CcState* st) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || st->bad) return;
  volatile int* p = parent;
  auto cas = [](volatile int* q, int r, int s) { return atomicCAS(const_cast<int*>(q + r), r, s); };
  const int a = faces[3 * (size_t)f], b = faces[3 * (size_t)f + 1], c = faces[3 * (size_t)f + 2];
  meshcc::cc_unite(p, a, b, cas);
  meshcc::cc_unite(p, b, c, cas);
}

// after every join: each vertex's label is its root (a separate array: the roots are read while labels are written)
__global__ void k_cc_labels(int V, const int* __restrict__ parent, const CcState* st, int* __restrict__ label) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || st->bad) return;
  label[v] = meshcc::cc_root(parent, v);
}

// face areas and keys (the label of the first vertex; V, no key, when the call is flagged)
__global__ void k_cc_area(int F, int V, const float* __restrict__ P, const int* __restrict__ faces, const int* __restrict__ label,
                          const CcState* st, float* __restrict__ area, int* __restrict__ key) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  if (st->bad) {
    area[f] = 0.f, key[f] = V;
    return;
  }
  area[f] = meshcc::face_area(P, faces, f);
  key[f] = label[faces[3 * (size_t)f]];
}

__global__ void k_cc_sums(int V, const float* __restrict__ area, InvMap m, double* __restrict__ sums) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) sums[v] = meshcc::cc_sum(area, m.order + m.first[v], m.first[v + 1] - m.first[v]);
}

// one CTA: the label np.argmax chooses (-1 when the call is flagged)
__global__ void __launch_bounds__(kCcArgmaxThreads) k_cc_argmax(int V, const double* __restrict__ sums, CcState* st) {
  __shared__ double s_s[kCcArgmaxThreads];
  __shared__ int s_l[kCcArgmaxThreads];
  double bs = 0.0;
  int bl = -1;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const double s = sums[v];
    if (bl < 0 || meshcc::cc_before(s, v, bs, bl)) bs = s, bl = v;
  }
  s_s[threadIdx.x] = bs, s_l[threadIdx.x] = bl;
  __syncthreads();
  for (int w = blockDim.x / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      const double t = s_s[threadIdx.x + w];
      const int m = s_l[threadIdx.x + w];
      if (m >= 0 && (s_l[threadIdx.x] < 0 || meshcc::cc_before(t, m, s_s[threadIdx.x], s_l[threadIdx.x])))
        s_s[threadIdx.x] = t, s_l[threadIdx.x] = m;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) st->best = st->bad ? -1 : s_l[0];
}

// compaction flags: a kept face, a vertex a kept face uses
__global__ void k_cc_flags(int F, const int* __restrict__ faces, const int* __restrict__ label, const CcState* st,
                           int* __restrict__ vnew, int* __restrict__ fnew) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int best = st->best;
  const bool keep = best >= 0 && label[faces[3 * (size_t)f]] == best;
  fnew[f] = keep;
  if (keep)
    for (int k = 0; k < 3; ++k) vnew[faces[3 * (size_t)f + k]] = 1;   // every writer stores the same value
}

__global__ void k_cc_out_verts(int V, const int* __restrict__ vnew, const float* __restrict__ P, float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || vnew[v + 1] == vnew[v]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)vnew[v] + k] = P[3 * (size_t)v + k];
}

__global__ void k_cc_out_faces(int F, const int* __restrict__ fnew, const int* __restrict__ vnew, const int* __restrict__ faces,
                               int* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || fnew[f + 1] == fnew[f]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)fnew[f] + k] = vnew[faces[3 * (size_t)f + k]];
}

}  // namespace hold
