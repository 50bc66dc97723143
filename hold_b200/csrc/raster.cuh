// Kernels of the soft-silhouette rasteriser (pose refinement, fitting/utils.py:101-118); arithmetic in raster_phases.h.
//
// k_raster_setup writes one record per (frame, face).  k_raster<bwd> runs one CTA per (frame, 16x16 tile), one pixel per
// thread: the face records stream through the CTA in chunks of 256, the faces whose box overlaps the tile are compacted in
// order (ballot), and every thread tests its pixel against them.  Per pixel the forward keeps the candidate count and the
// product Q of (1 - p).  When some pixel of the tile has more than K candidates, the tile bisects that pixel's K-th key
// (pz, face) bit by bit, one pass over the faces per bit, and redoes the product over the keys <= it: the selection is exact
// and nothing of size K per pixel is stored.  The backward recomputes the selection the same way.
//
// The backward accumulates the vertex gradients with fp32 atomics (per chunk in shared memory, then into g_verts): the
// gradient is not bitwise reproducible from run to run.  The silhouette is: each pixel multiplies its factors in face order.
#pragma once
#include "common.cuh"
#include "raster_phases.h"

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
  const float* g_sil;  // backward: [B, H, W] -> g_verts [B, V, 3] (accumulated; x and y only)
  float* g_verts;
};

template <bool kBwd>
__global__ void __launch_bounds__(kRasterThreads) k_raster(RasterArgs a) {
  constexpr int kWarps = kRasterThreads / 32;
  __shared__ int s_list[kRasterThreads];                  // this chunk's faces that overlap the tile, in face order
  __shared__ int s_wcnt[kWarps];
  __shared__ float s_g[kBwd ? kRasterThreads * 6 : 1];   // backward: the chunk's vertex-xy gradients
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
  } else {
    const float g = live ? a.g_sil[pix] : 0.f;
    const bool act = live && g != 0.f && Q != 0.f;   // Q = 0: every kept face's gradient is 0 (raster_phases.h)
    if (__syncthreads_or(act)) {
      for (int k = threadIdx.x; k < kRasterThreads * 6; k += kRasterThreads) s_g[k] = 0.f;
      pass([&](int slot, int f) {
        raster::Frag fr;
        if (!act || !test(f, fr) || raster::frag_key(fr.pz, f, a.fbits) > thr) return;
        const float gd = raster::blend_ddist(g, Q, fr, a.o.sigma);
        if (gd == 0.f) return;
        float gv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        raster::tri_sqdist_bwd(px, py, v, fr.edge, gd, gv);
        for (int c = 0; c < 6; ++c)
          if (gv[c] != 0.f) atomicAdd(&s_g[slot * 6 + c], gv[c]);
      }, [&](int n) {
        __syncthreads();
        for (int k = threadIdx.x; k < n * 6; k += kRasterThreads) {
          const float x = s_g[k];
          if (x == 0.f) continue;
          s_g[k] = 0.f;
          const float4 r3 = rec[(size_t)s_list[k / 6] * 4 + 3];
          const int c = k % 6, vid = __float_as_int(c < 2 ? r3.y : c < 4 ? r3.z : r3.w);
          atomicAdd(&a.g_verts[((size_t)b * a.V + vid) * 3 + (c & 1)], x);
        }
      });
    }
  }
}

}  // namespace hold
