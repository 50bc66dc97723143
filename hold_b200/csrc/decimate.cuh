// Quadric edge-collapse mesh decimation (hold_decimate): the object mesh of the pose refinement brought down to a raster-sized
// mesh, as pymeshlab's meshing_decimation_quadric_edge_collapse does in the reference's load_data.  Arithmetic in
// decimate_phases.h.
//
// Deterministic parallel rounds.  Faces stay in place, a dead face holding -1 at its corners, until the final compaction.  Each
// round:
//  1. the vertex stars over the live (face, corner) items, through inverse_map (dead items are keyed to the sentinel V);
//  2. every edge's key (decim::edge_candidate: float(cost) bits above the half-edge id, kNoKey when the collapse is invalid);
//     the candidates are the keys at most the median valid key, found by a radix select over the unique 64-bit keys;
//  3. an independent set by three min-propagations over the stars: m(v) the smallest candidate key at v, M(v) the smallest m
//     over v's closed 1-ring, M2(v) the smallest M over the closed 1-ring; an edge is selected iff its key is M2 at both ends.
//     Selected edges are then at least 3 hops apart, so their stars and 1-rings are disjoint and the collapses apply in any
//     order, without atomics;
//  4. when the round would go below target_faces, only the ceil((F_live - target) / 2) smallest selected keys are kept (the same
//     radix select);
//  5. the collapses (decim::apply_collapse).
// Every value a round computes is a function of the mesh alone, never of the schedule: the output is bitwise reproducible and
// equal to the sequential restatement in tests/host/decimate_host.cpp.  Each round ends with one host read of the live face
// count, so hold_decimate synchronises its stream every round and cannot be captured in a CUDA graph.  No kernel has a
// floating-point atomic; the select histograms count with integer atomics, whose totals do not depend on their order.
#pragma once
#include "common.cuh"
#include "decimate_phases.h"
#include "inverse_map.cuh"

namespace hold {

constexpr int kDecThreads = 256;
constexpr int kDecMaxRounds = 1000;

struct DecSelect {
  unsigned long long cut;   // after the 8 passes: the selected key (or kNoKey - 1: every valid key passes)
  int k;                    // rank still sought within the current prefix
  int done;
};

struct DecState {
  DecSelect sel[2];         // 0: the median cut of the candidates, 1: the trim of the selected edges
  int F_live, target;
  int collapses;            // of the last round
  int bad;                  // a face index outside [0, V)
};

// faces copied to the working buffer; an index outside [0, V) flags the call (the mesh is then returned unchanged)
__global__ void k_dec_init(int n3, int V, const int* __restrict__ faces, int* __restrict__ F, DecState* st, int* err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  const int v = faces[i];
  F[i] = v;
  if (v < 0 || v >= V) {
    atomicOr(&st->bad, 1);
    atomicOr(err, kErrBadMeshIndex);
  }
}

__global__ void k_dec_state(DecState* st, int F, int target) {
  st->F_live = F, st->target = target, st->collapses = 0, st->bad = 0;
}

// the stars' keys: a live item's vertex, V for a dead one
__global__ void k_dec_star_keys(int n3, int V, const int* __restrict__ F, int* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) keys[i] = F[i] >= 0 ? F[i] : V;
}

__global__ void k_dec_quadrics(int V, const int* __restrict__ F, const float* __restrict__ P, InvMap m, double* __restrict__ Q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) decim::vertex_quadric(v, F, P, m.order, m.first, Q + 10 * (size_t)v);
}

__global__ void k_dec_frozen(int V, const int* __restrict__ F, InvMap m, int* __restrict__ frozen) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) frozen[v] = decim::vertex_frozen(F, m.order + m.first[v], m.first[v + 1] - m.first[v]);
}

__global__ void __launch_bounds__(kDecThreads) k_dec_edges(int n3, const int* __restrict__ F, const float* __restrict__ P,
                                                           const double* __restrict__ Q, InvMap m, const int* __restrict__ frozen,
                                                           double qthr, uint64_t* __restrict__ key, float* __restrict__ X) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < n3) key[h] = decim::edge_candidate(h, F, P, Q, m.order, m.first, frozen, qthr, X + 3 * (size_t)h);
}

// One pass of the radix select of sel[which]: the count of each 8-bit digit (bits 56 - 8 pass ..) among the keys that match
// the prefix found so far.  hist[256] is zero on entry.
__global__ void __launch_bounds__(kDecThreads) k_dec_sel_hist(int n, const uint64_t* __restrict__ keys, const DecState* st, int which,
                                                              int pass, int* __restrict__ hist) {
  __shared__ int s[256];
  const DecSelect& q = st->sel[which];
  if (pass > 0 && q.done) return;   // CTA-uniform
  s[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 56 - 8 * pass;
  const uint64_t mask = pass == 0 ? 0ull : ~0ull << (64 - 8 * pass), prefix = q.cut & mask;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t k = keys[i];
    if ((k & mask) == prefix) atomicAdd(&s[(k >> shift) & 255], 1);
  }
  __syncthreads();
  if (s[threadIdx.x]) atomicAdd(&hist[threadIdx.x], s[threadIdx.x]);
}

// One thread: pick the digit that holds rank k and clear hist.  Pass 0 counts the valid keys (their top byte is at most 0x7f,
// kNoKey's is 0xff) and sets the rank: which 0 = the median, (n - 1) / 2; which 1 = the trim, ceil((F_live - target) / 2)
// collapses, which also updates F_live and the round's collapse count.
__global__ void k_dec_sel_pick(DecState* st, int which, int pass, int* __restrict__ hist) {
  DecSelect& q = st->sel[which];
  if (pass == 0) {
    int n = 0;
    for (int d = 0; d < 255; ++d) n += hist[d];
    q.done = 0, q.cut = 0;
    if (which == 0) {
      q.k = (n - 1) / 2;
      if (n == 0) q.done = 1, q.cut = decim::kNoKey - 1;
    } else {
      const int need = (st->F_live - st->target + 1) / 2;
      st->collapses = n < need ? n : need;
      st->F_live -= 2 * st->collapses;
      q.k = need - 1;
      if (n <= need) q.done = 1, q.cut = decim::kNoKey - 1;
    }
  }
  if (!q.done) {
    int cum = 0, d = 0;
    while (d < 255 && q.k >= cum + hist[d]) cum += hist[d++];
    q.k -= cum;
    q.cut |= (unsigned long long)d << (56 - 8 * pass);
  }
  for (int d = 0; d < 256; ++d) hist[d] = 0;
}

__global__ void k_dec_vmin(int V, const int* __restrict__ F, InvMap m, const uint64_t* __restrict__ key, const DecState* st,
                           uint64_t* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) out[v] = decim::vertex_min_key(v, F, m.order, m.first, key, st->sel[0].cut);
}

__global__ void k_dec_ring(int V, const int* __restrict__ F, InvMap m, const uint64_t* __restrict__ in, uint64_t* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) out[v] = decim::ring_min(v, F, m.order, m.first, in);
}

// an edge is selected iff its key is a candidate and M2 at both ends
__global__ void k_dec_select(int n3, const int* __restrict__ F, const uint64_t* __restrict__ key, const DecState* st,
                             const uint64_t* __restrict__ M2, uint64_t* __restrict__ sel) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n3) return;
  const uint64_t k = key[h];
  bool s = k <= st->sel[0].cut;
  if (s) {
    const int u = F[h], v = F[3 * (h / 3) + decim::next_corner(h % 3)];
    s = M2[u] == k && M2[v] == k;
  }
  sel[h] = s ? k : decim::kNoKey;
}

__global__ void k_dec_apply(int n3, const uint64_t* __restrict__ sel, const DecState* st, int* F, float* P, double* Q, InvMap m,
                            const float* __restrict__ X) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < n3 && sel[h] <= st->sel[1].cut) decim::apply_collapse(h, F, P, Q, m.order, m.first, X + 3 * (size_t)h);
}

// compaction: flags (a vertex that a live face uses, a live face), then exclusive scans give the new ids
__global__ void k_dec_flags(int F, const int* __restrict__ Fw, int* __restrict__ vnew, int* __restrict__ fnew) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const bool live = Fw[3 * f] >= 0;
  fnew[f] = live;
  if (live)
    for (int k = 0; k < 3; ++k) vnew[Fw[3 * f + k]] = 1;   // every writer stores the same value
}

__global__ void k_dec_out_verts(int V, const int* __restrict__ vnew, const float* __restrict__ P, float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || vnew[v + 1] == vnew[v]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)vnew[v] + k] = P[3 * (size_t)v + k];
}

__global__ void k_dec_out_faces(int F, const int* __restrict__ fnew, const int* __restrict__ vnew, const int* __restrict__ Fw,
                                int* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || fnew[f + 1] == fnew[f]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)fnew[f] + k] = vnew[Fw[3 * f + k]];
}

}  // namespace hold
