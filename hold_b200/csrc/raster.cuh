// Kernels of the soft-silhouette rasteriser (pose refinement, fitting/utils.py:101-118); arithmetic in raster_phases.h.
//
// k_raster_setup writes one record per (frame, face).  k_raster<bwd> runs one CTA per (frame, 16x16 tile), one pixel per
// thread: the face records stream through the CTA in chunks of 256, the faces whose box overlaps the tile are compacted in
// order (ballot), and every thread tests its pixel against them.  Per pixel the forward keeps the candidate count and the
// product Q of (1 - p).  When some pixel of the tile has more than K candidates, the tile bisects that pixel's K-th key
// (pz, face) bit by bit, one pass over the faces per bit, and redoes the product over the keys <= it: the selection is exact
// and nothing of size K per pixel is stored.  The silhouette is bitwise reproducible: each pixel multiplies its factors in
// face order.
//
// The backward adds in an order fixed by the inputs alone, with no atomic, so g_verts is bitwise reproducible and a frame's
// bits do not depend on the rest of the batch:
//   1. k_raster<true> recomputes the selection the same way and stores each pixel's Q and key threshold ([B,H,W] each);
//   2. k_raster_bwd_faces runs one warp per (frame, face, piece of the face's pixel box): the warp re-tests the piece's pixels
//      (pixel_face, key <= threshold), each lane adds its pixels' vertex-xy gradients in row-major order, a shuffle tree adds
//      the lanes, and lane 0 stores the piece's 6 sums ([B,F,kRbPieces,6]);
//   3. k_raster_bwd_verts sums, per vertex, its (face, corner) partials in ascending face order, then piece order: the
//      inverse of faces comes from inverse_map.cuh.
#pragma once
#include "common.cuh"
#include "raster_phases.h"
#include "inverse_map.cuh"

namespace hold {

constexpr int kRasterTile = 16;
constexpr int kRasterThreads = kRasterTile * kRasterTile;

// Record of face f of frame b, 4 float4: [xmin xmax ymin ymax] (the box expanded by sqrt(blur_radius)), [x0 y0 x1 y1],
// [x2 y2 z0 z1], [z2, vertex ids as int bits].  A face no pixel can take (behind the camera, zero area, culled, or with an
// out-of-range vertex id) gets an empty box, which no tile or pixel passes.
__global__ void k_raster_setup(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, raster::Opts o,
                               float4* __restrict__ rec, int* __restrict__ err) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (f >= F) return;
  int id[3];
  bool ok = true;
  for (int k = 0; k < 3; ++k) {
    id[k] = faces[(size_t)f * 3 + k];
    ok = ok && id[k] >= 0 && id[k] < V;
  }
  float v[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float bb[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  if (!ok) {
    atomicOr(err, kErrBadFace);   // the host validates faces; never read through a bad index
    id[0] = id[1] = id[2] = 0;
  } else {
    const float* vb = verts + (size_t)b * V * 3;
    for (int k = 0; k < 3; ++k) {
      v[2 * k] = vb[(size_t)id[k] * 3], v[2 * k + 1] = vb[(size_t)id[k] * 3 + 1], v[6 + k] = vb[(size_t)id[k] * 3 + 2];
    }
    if (!raster::face_setup(v, o, bb)) bb[0] = INFINITY, bb[1] = -INFINITY, bb[2] = INFINITY, bb[3] = -INFINITY;
  }
  float4* r = rec + ((size_t)b * F + f) * 4;
  r[0] = make_float4(bb[0], bb[1], bb[2], bb[3]);
  r[1] = make_float4(v[0], v[1], v[2], v[3]);
  r[2] = make_float4(v[4], v[5], v[6], v[7]);
  r[3] = make_float4(v[8], __int_as_float(id[0]), __int_as_float(id[1]), __int_as_float(id[2]));
}

struct RasterArgs {
  int V, F, H, W, K, fbits;
  raster::Opts o;
  const float4* rec;   // [B, F, 4] from k_raster_setup
  float* sil;          // forward: [B, H, W]
  int64_t* p2f;        // forward, optional (all three or none): [B, H, W, K]
  float* zbuf;
  float* dists;
  float* q;            // backward: per pixel, Q and the selection's key threshold [B, H, W]
  uint64_t* thr;
};

template <bool kBwd>
__global__ void __launch_bounds__(kRasterThreads) k_raster(RasterArgs a) {
  constexpr int kWarps = kRasterThreads / 32;
  __shared__ int s_list[kRasterThreads];                  // this chunk's faces that overlap the tile, in face order
  __shared__ int s_wcnt[kWarps];
  const int b = blockIdx.y, ntx = ceil_div(a.W, kRasterTile);
  const int i0 = (blockIdx.x / ntx) * kRasterTile, j0 = (blockIdx.x % ntx) * kRasterTile;
  const int i = i0 + threadIdx.x / kRasterTile, j = j0 + threadIdx.x % kRasterTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool live = i < a.H && j < a.W;
  const int s = min(a.H, a.W);
  const float px = raster::pix_ndc(j, a.W, s), py = raster::pix_ndc(i, a.H, s);
  // the tile's pixel centres span [tx0, tx1] x [ty0, ty1] (x and y decrease with the column and the row)
  const float tx0 = raster::pix_ndc(min(j0 + kRasterTile - 1, a.W - 1), a.W, s), tx1 = raster::pix_ndc(j0, a.W, s);
  const float ty0 = raster::pix_ndc(min(i0 + kRasterTile - 1, a.H - 1), a.H, s), ty1 = raster::pix_ndc(i0, a.H, s);
  const float4* rec = a.rec + (size_t)b * a.F * 4;
  const size_t pix = ((size_t)b * a.H + min(i, a.H - 1)) * a.W + min(j, a.W - 1);

  // One pass over the tile's faces: visit(slot, face) per overlapping face (live pixels only), then after(n) by all threads
  // once the chunk of n faces has been visited.
  auto pass = [&](auto&& visit, auto&& after) {
    for (int f0 = 0; f0 < a.F; f0 += kRasterThreads) {
      const int f = f0 + threadIdx.x;
      bool hit = false;
      if (f < a.F) {
        const float4 bb = rec[(size_t)f * 4];
        hit = !(bb.x > tx1 || bb.y < tx0 || bb.z > ty1 || bb.w < ty0);
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      __syncthreads();   // the previous chunk is consumed
      if (lane == 0) s_wcnt[warp] = __popc(m);
      __syncthreads();
      int off = 0, n = 0;
      for (int w = 0; w < kWarps; ++w) {
        const int c = s_wcnt[w];
        off += w < warp ? c : 0;
        n += c;
      }
      if (hit) s_list[off + __popc(m & ((1u << lane) - 1u))] = f;
      __syncthreads();
      if (live)
        for (int k = 0; k < n; ++k) visit(k, s_list[k]);
      after(n);
    }
  };
  auto nothing = [](int) {};
  float v[9];
  // test this pixel against face f (loads its record into v)
  auto test = [&](int f, raster::Frag& fr) {
    const float4* r = rec + (size_t)f * 4;
    const float4 r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3];
    const float bb[4] = {r0.x, r0.y, r0.z, r0.w};
    v[0] = r1.x, v[1] = r1.y, v[2] = r1.z, v[3] = r1.w, v[4] = r2.x, v[5] = r2.y, v[6] = r2.z, v[7] = r2.w, v[8] = r3.x;
    return raster::pixel_face(v, bb, px, py, a.o, fr);
  };

  int cnt = 0;
  float Q = 1.f;
  pass([&](int, int f) {
    raster::Frag fr;
    if (test(f, fr)) ++cnt, Q *= raster::blend_q(raster::signed_dist(fr), a.o.sigma);
  }, nothing);

  uint64_t thr = ~0ull;   // keep the candidates whose key is <= thr
  if (__syncthreads_or(cnt > a.K)) {
    const bool over = cnt > a.K;
    // the K-th smallest key: the largest x with #(key < x) < K, built from the top bit down
    uint64_t ans = 0;
    for (int bit = 30 + a.fbits; bit >= 0; --bit) {
      const uint64_t cand = ans | (1ull << bit);
      int c = 0;
      pass([&](int, int f) {
        raster::Frag fr;
        if (over && test(f, fr) && raster::frag_key(fr.pz, f, a.fbits) < cand) ++c;
      }, nothing);
      if (c < a.K) ans = cand;
    }
    if (over) thr = ans, Q = 1.f;
    pass([&](int, int f) {
      raster::Frag fr;
      if (over && test(f, fr) && raster::frag_key(fr.pz, f, a.fbits) <= thr) Q *= raster::blend_q(raster::signed_dist(fr), a.o.sigma);
    }, nothing);
  }

  if constexpr (!kBwd) {
    if (live) a.sil[pix] = 1.f - Q;
    if (a.p2f != nullptr) {
      // pytorch3d's fragments, sorted by key: insertion into this pixel's own K slots
      const size_t base = pix * a.K;
      if (live)
        for (int k = 0; k < a.K; ++k) a.p2f[base + k] = -1, a.zbuf[base + k] = -1.f, a.dists[base + k] = -1.f;
      const int64_t fb = (int64_t)b * a.F;
      int n = 0;
      pass([&](int, int f) {
        raster::Frag fr;
        if (!test(f, fr)) return;
        const uint64_t key = raster::frag_key(fr.pz, f, a.fbits);
        if (key > thr) return;
        int pos = n++;
        for (; pos > 0; --pos) {
          const size_t q = base + pos - 1;
          if (raster::frag_key(a.zbuf[q], (int)(a.p2f[q] - fb), a.fbits) < key) break;
          a.p2f[q + 1] = a.p2f[q], a.zbuf[q + 1] = a.zbuf[q], a.dists[q + 1] = a.dists[q];
        }
        a.p2f[base + pos] = fb + f, a.zbuf[base + pos] = fr.pz, a.dists[base + pos] = raster::signed_dist(fr);
      }, nothing);
    }
  } else if (live) {
    a.q[pix] = Q, a.thr[pix] = thr;
  }
}

constexpr int kRbWarps = 8;            // pieces per CTA of k_raster_bwd_faces
constexpr int kRbPieces = 16;          // the most pieces a face's pixel box is split into
constexpr int kRbPiecePixels = 256;    // the fewest pixels a piece is given when the box allows it

// Pixels whose centre may lie inside a face's expanded box (record word 0), with a pixel of margin; pixel_face still decides.
// An empty box gives no pixel, a NaN box the whole image.
struct PixBox {
  int i0, j0, ni, nj;
};
__device__ __forceinline__ PixBox pix_box(float4 bb, int H, int W) {
  const float s = (float)min(H, W);
  // pix_ndc(j) = (W - 2j - 1) / s decreases with j: x <= xmax  <=>  j >= (W - 1 - xmax s) / 2
  const float j0 = fmaxf(floorf((W - 1 - bb.y * s) * 0.5f) - 1.f, 0.f), j1 = fminf(ceilf((W - 1 - bb.x * s) * 0.5f) + 1.f, W - 1.f);
  const float i0 = fmaxf(floorf((H - 1 - bb.w * s) * 0.5f) - 1.f, 0.f), i1 = fminf(ceilf((H - 1 - bb.z * s) * 0.5f) + 1.f, H - 1.f);
  if (!(j0 <= j1 && i0 <= i1)) return PixBox{0, 0, 0, 0};
  return PixBox{(int)i0, (int)j0, (int)(i1 - i0) + 1, (int)(j1 - j0) + 1};
}
// pieces of a box: one per kRbPiecePixels pixels, 1 .. kRbPieces (an empty box has one piece, with no pixel)
__device__ __forceinline__ int pix_pieces(const PixBox& p) {
  const int64_t n = ((int64_t)p.ni * p.nj + kRbPiecePixels - 1) / kRbPiecePixels;
  return n < 1 ? 1 : n > kRbPieces ? kRbPieces : (int)n;
}

struct RasterBwdArgs {
  int V, F, H, W, fbits;
  raster::Opts o;
  const float4* rec;     // [B, F, 4] from k_raster_setup
  const float* q;        // [B, H, W] from k_raster<true>
  const uint64_t* thr;
  const float* g_sil;    // [B, H, W]
  float* part;           // [B, F, kRbPieces, 6]: each face's vertex-xy gradients per piece (the first pix_pieces are written)
  InvMap vmap;           // faces inverted: item 3 f + c, key = vertex id
  float* g_verts;        // [B, V, 3], overwritten (x and y; z = 0)
};

// grid (F * kRbPieces / kRbWarps, B), kRbWarps warps: one warp per (frame, face, piece)
__global__ void __launch_bounds__(kRbWarps * 32) k_raster_bwd_faces(RasterBwdArgs a) {
  const int b = blockIdx.y, f = blockIdx.x / (kRbPieces / kRbWarps);
  const int piece = (blockIdx.x % (kRbPieces / kRbWarps)) * kRbWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const float4* r = a.rec + ((size_t)b * a.F + f) * 4;
  const float4 r0 = r[0];
  const PixBox pb = pix_box(r0, a.H, a.W);
  const int np = pix_pieces(pb);
  if (piece >= np) return;   // warp-uniform
  const float4 r1 = r[1], r2 = r[2], r3 = r[3];
  const float bb[4] = {r0.x, r0.y, r0.z, r0.w};
  const float v[9] = {r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w, r3.x};
  const int s = min(a.H, a.W);
  const int64_t n = (int64_t)pb.ni * pb.nj, p1 = n * (piece + 1) / np;
  const size_t frame = (size_t)b * a.H * a.W;
  float gv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t p = n * piece / np + lane; p < p1; p += 32) {
    const int i = pb.i0 + (int)(p / pb.nj), j = pb.j0 + (int)(p % pb.nj);
    const size_t pix = frame + (size_t)i * a.W + j;
    const float g = a.g_sil[pix], Q = a.q[pix];
    if (g == 0.f || Q == 0.f) continue;   // Q = 0: every kept face's gradient is 0 (raster_phases.h)
    const float px = raster::pix_ndc(j, a.W, s), py = raster::pix_ndc(i, a.H, s);
    raster::Frag fr;
    if (!raster::pixel_face(v, bb, px, py, a.o, fr) || raster::frag_key(fr.pz, f, a.fbits) > a.thr[pix]) continue;
    const float gd = raster::blend_ddist(g, Q, fr, a.o.sigma);
    if (gd != 0.f) raster::tri_sqdist_bwd(px, py, v, fr.edge, gd, gv);
  }
#pragma unroll
  for (int c = 0; c < 6; ++c)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) gv[c] += __shfl_down_sync(0xffffffffu, gv[c], off);
  if (lane == 0) {
    float* out = a.part + (((size_t)b * a.F + f) * kRbPieces + piece) * 6;
#pragma unroll
    for (int c = 0; c < 6; ++c) out[c] = gv[c];
  }
}

// grid (ceil(V / 128), B), 128 threads: one thread per (frame, vertex)
__global__ void __launch_bounds__(128) k_raster_bwd_verts(RasterBwdArgs a) {
  const int vid = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (vid >= a.V) return;
  float sx = 0.f, sy = 0.f;
  for (int e = a.vmap.first[vid]; e < a.vmap.first[vid + 1]; ++e) {
    const int item = a.vmap.order[e], f = item / 3, c = item % 3;
    const size_t fb = (size_t)b * a.F + f;
    const int np = pix_pieces(pix_box(a.rec[fb * 4], a.H, a.W));
    const float* p = a.part + fb * kRbPieces * 6 + 2 * c;
    for (int k = 0; k < np; ++k) sx += p[k * 6], sy += p[k * 6 + 1];
  }
  float* g = a.g_verts + ((size_t)b * a.V + vid) * 3;
  g[0] = sx, g[1] = sy, g[2] = 0.f;
}

// keys of the (face, corner) items for inverse_map: the vertex id, or V for an index outside [0, V)
__global__ void k_raster_vert_keys(int n, int V, const int* __restrict__ faces, int* __restrict__ keys) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int id = faces[e];
  keys[e] = id >= 0 && id < V ? id : V;
}

}  // namespace hold
