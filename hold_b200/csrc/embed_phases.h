// The Fourier embedding of the tensor-core chains (engine/embedders.py:48-51), as host/device functions: the kernels (mlp_tc.cuh) inline
// them; tests/test_cpu_embed.py runs the same code on the host against the oracle's embedder (value and derivative, 3- and 4-d
// points, BARF weights, every group offset the kernels use).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HOLD_EHD __host__ __device__ __forceinline__
#else
#define HOLD_EHD inline
#endif

namespace hold {

HOLD_EHD float emb_int_as_float(int v) {
#if defined(__CUDA_ARCH__)
  return __int_as_float(v);
#else
  union { int i; float f; } u; u.i = v; return u.f;
#endif
}
HOLD_EHD int emb_rint_to_int(float k) {
#if defined(__CUDA_ARCH__)
  return __float2int_rn(k);
#else
  return (int)k;   // k is already integral (rintf)
#endif
}
HOLD_EHD float emb_ldg(const float* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// sin and cos of x for |x| < ~1e4 (the embeddings' arguments are coordinate * 2^k, k <= 9, |coordinate| <= a few): two-constant
// Cody-Waite reduction by pi/2 with FMAs, Taylor kernels on [-pi/4, pi/4]; max abs error 7.1e-8 over the range used (libm's sinf:
// 3.3e-8; the pin against the oracle's torch.sin is the stage tests' 1e-4).  No slow path, no calls, so that several of these
// interleave in the tile prologue and the skip-layer epilogue (libm's sinf / cosf sit behind a non-inlined call and run serially).
HOLD_EHD void sincos_cw(float x, float& s, float& c) {
  const float k = rintf(x * 0.63661977236758134f);
  float r = fmaf(k, -1.57079637050628662109375f, x);
  r = fmaf(k, 4.371138828673793e-8f, r);
  const float r2 = r * r;
  float sp = fmaf(r2, 2.7557319e-6f, -1.9841270e-4f);
  sp = fmaf(sp, r2, 8.3333333e-3f);
  sp = fmaf(sp, r2, -1.6666667e-1f);
  sp = fmaf(sp * r2, r, r);
  float cp = fmaf(r2, -2.7557319e-7f, 2.4801587e-5f);
  cp = fmaf(cp, r2, -1.3888889e-3f);
  cp = fmaf(cp, r2, 4.1666667e-2f);
  cp = fmaf(cp, r2, -0.5f);
  cp = fmaf(cp, r2, 1.0f);
  const int q = emb_rint_to_int(k);
  const float ss = (q & 1) ? cp : sp, cc = (q & 1) ? sp : cp;
  s = (q & 2) ? -ss : ss;
  c = ((q + 1) & 2) ? -cc : cc;
}

// NE consecutive elements e0 .. e0+NE-1 of the Fourier embedding (engine/embedders.py:48-51: [x, sin(2^0 x), cos(2^0 x), sin(2^1 x),
// ...], D coordinates per point, n_embed elements) or, DERIV, of its derivative w.r.t. the element's own coordinate.  Branch-free:
// the NE sin/cos chains interleave (per-element branches would serialise them on the tile's critical path).
// ew: optional per-element weights (BarfEmbedder).  Returns the mask of elements that exist (0 <= e < n_embed); v[i] is finite
// garbage elsewhere.
template <int D, bool DERIV, int NE>
HOLD_EHD uint32_t embedn_inl(int e0, int n_embed, float x0, float x1, float x2, float x3, const float* __restrict__ ew,
                             float (&v)[NE]) {
  uint32_t okm = 0;
  float w[NE];
  if (ew != nullptr) {
#pragma unroll
    for (int i = 0; i < NE; ++i) w[i] = emb_ldg(ew + (e0 + i < 0 ? 0 : (e0 + i > n_embed - 1 ? n_embed - 1 : e0 + i)));
  } else {
#pragma unroll
    for (int i = 0; i < NE; ++i) w[i] = 1.f;
  }
#pragma unroll
  for (int i = 0; i < NE; ++i) {
    const int e = e0 + i;
    const bool ok = (unsigned)e < (unsigned)n_embed;
    const int ec = ok ? e : 0;
    const int g = (D == 4) ? (ec >> 2) : ((ec * 171) >> 9);   // ec / D (ec < 256)
    const int d = ec - D * g;
    const int qq = g - 1;                                     // -1: the identity block
    const float pc = (d == 0) ? x0 : ((d == 1) ? x1 : ((d == 2 || D == 3) ? x2 : x3));
    const float f = emb_int_as_float((127 + ((qq > 0 ? qq : 0) >> 1)) << 23);
    float sn, cs;
    sincos_cw(pc * f, sn, cs);
    float r = DERIV ? ((qq & 1) ? -f * sn : f * cs) : ((qq & 1) ? cs : sn);
    r = (qq < 0) ? (DERIV ? 1.f : pc) : r;
    v[i] = r * w[i];
    okm |= ok ? (1u << i) : 0u;
  }
  return okm;
}

}  // namespace hold
