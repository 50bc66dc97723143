// SURVEY §8f rank 1 — the NeRF++ inverted-sphere background (model/renderables/background.py:35-165): 32 fixed samples
// per ray outside the bounding sphere, an 8x256 "implicit" MLP on the 4-d (unit direction, inverse depth) point with a
// 32-d per-frame code, a 315->128->3 colour head with a PE-4 view direction, |sdf| as density, own transmittance, and
// the final composite rgb = fg_rgb + bg_weight * bg_rgb (hold/hold_net.py:125-134).  ~1 % of the foreground's FLOPs;
// exact fp32 on CUDA cores, same fused-chain structure as mlp_simt.cuh.
#pragma once
#include "common.cuh"
#include "mlp_simt.cuh"

namespace hold {

constexpr int kBgActLd = 324;   // >= 320 (colour head input 315 -> 320) + 4
constexpr int kBgEmbLd = 88;
enum { BG_SDF = 0, BG_RGB = 1 };

struct BgArgs {
  int P, pts_per_frame;          // points = rays * 32, frame-major
  int n_layers;
  SimtLayer L[HOLD_MAX_LAYERS];
  const float* w_last;           // BG_SDF: lin8 row 0 [256]; BG_RGB: lin1 [3][128]
  const float* b_last;
  const float* cam;              // [R,3]
  const float* dirs;             // [R,3]
  const float* frame_code;       // [B,32]
  float r_sphere;
  float* sdf;                    // [P]
  float* feat;                   // [P,256]  (BG_SDF: out, BG_RGB: in)
  float* rgb;                    // [P,3]
};

// [x, sin(2^k x), cos(2^k x)]_k layout of engine/embedders.py:48-51 for a D-wide input
template <int D, int NF>
__device__ __forceinline__ void embed_generic(const float* x, float* dst) {
  for (int c = 0; c < D; ++c) dst[c] = x[c];
  for (int k = 0; k < NF; ++k) {
    const float f = (float)(1 << k);
    for (int c = 0; c < D; ++c) {
      dst[D + (2 * k) * D + c] = sinf(x[c] * f);
      dst[D + (2 * k + 1) * D + c] = cosf(x[c] * f);
    }
  }
}

template <int STAGE>
__global__ void __launch_bounds__(256, 1) k_bg_mlp(BgArgs a) {
  extern __shared__ __align__(16) float smem[];
  float* actA = smem;
  float* actB = actA + kTileRows * kBgActLd;
  float* wbuf = actB + kTileRows * kBgActLd;       // [2][kKC][256]
  float* emb = wbuf + 2 * kKC * 256;               // [64][kBgEmbLd]
  const int tid = threadIdx.x, tx = tid % 32, ty = tid / 32;
  const int n_tiles = ceil_div(a.P, kTileRows);
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p0 = tile * kTileRows;
    __syncthreads();
    // ---------------------------------------------------------------- prologue
    if (tid < kTileRows) {
      const int row = tid, p = p0 + row;
      float* dst = actA + row * kBgActLd;
      const int kpad = a.L[0].Kpad;
      if (p < a.P) {
        const int ray = p / kBgN, k = p % kBgN, b = p / a.pts_per_frame;
        const float o[3] = {a.cam[3 * ray], a.cam[3 * ray + 1], a.cam[3 * ray + 2]};
        const float d[3] = {a.dirs[3 * ray], a.dirs[3 * ray + 1], a.dirs[3 * ray + 2]};
        if (STAGE == BG_SDF) {
          float p4[4];
          depth2pts_outside(o, d, bg_depth(k, a.r_sphere), a.r_sphere, p4);
          embed_generic<4, 10>(p4, emb + row * kBgEmbLd);
          for (int e = 0; e < kBgEmbed; ++e) dst[e] = emb[row * kBgEmbLd + e];
          for (int e = 0; e < kBgFrame; ++e) dst[kBgEmbed + e] = a.frame_code[b * kBgFrame + e];
          for (int e = kBgEmbed + kBgFrame; e < kpad; ++e) dst[e] = 0.f;
        } else {
          embed_generic<3, 4>(d, dst);
          for (int e = 0; e < kBgFrame; ++e) dst[kBgView + e] = a.frame_code[b * kBgFrame + e];
          for (int e = 0; e < kFeat; ++e) dst[kBgView + kBgFrame + e] = a.feat[(size_t)p * kFeat + e];
          for (int e = kBgView + kBgFrame + kFeat; e < kpad; ++e) dst[e] = 0.f;
        }
      } else {
        for (int e = 0; e < kpad; ++e) dst[e] = 0.f;
        if (STAGE == BG_SDF)
          for (int e = 0; e < kBgEmbed; ++e) emb[row * kBgEmbLd + e] = 0.f;
      }
    }
    __syncthreads();
    float* in = actA;
    float* out = actB;
    for (int l = 0; l < a.n_layers; ++l) {
      const SimtLayer L = a.L[l];
      float acc[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      const int nchunks = L.Kpad / kKC;
      for (int q = tid; q < kKC * 64; q += 256) cp_async16(wbuf + q * 4, L.Wt + q * 4);
      cp_async_commit();
      for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
          const float* src = L.Wt + (size_t)(c + 1) * kKC * 256;
          float* dstw = wbuf + ((c + 1) & 1) * kKC * 256;
          for (int q = tid; q < kKC * 64; q += 256) cp_async16(dstw + q * 4, src + q * 4);
          cp_async_commit();
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        __syncthreads();
        const float* w = wbuf + (c & 1) * kKC * 256;
        const float* arow = in + (ty * 8) * kBgActLd + c * kKC;
#pragma unroll
        for (int kq = 0; kq < kKC; kq += 4) {
          float4 av[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) av[i] = *reinterpret_cast<const float4*>(arow + i * kBgActLd + kq);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const float4 w0 = *reinterpret_cast<const float4*>(w + (kq + kk) * 256 + 4 * tx);
            const float4 w1 = *reinterpret_cast<const float4*>(w + (kq + kk) * 256 + 128 + 4 * tx);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float av_ = (kk == 0) ? av[i].x : (kk == 1) ? av[i].y : (kk == 2) ? av[i].z : av[i].w;
              acc[i][0] += av_ * w0.x; acc[i][1] += av_ * w0.y; acc[i][2] += av_ * w0.z; acc[i][3] += av_ * w0.w;
              acc[i][4] += av_ * w1.x; acc[i][5] += av_ * w1.y; acc[i][6] += av_ * w1.z; acc[i][7] += av_ * w1.w;
            }
          }
        }
        __syncthreads();
      }
      const bool feat_layer = (STAGE == BG_SDF) && (l == a.n_layers - 1);
      float bj[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) bj[j] = L.bias[(j < 4 ? 4 * tx + j : 128 + 4 * tx + j - 4)];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = ty * 8 + i, p = p0 + row;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = (j < 4) ? 4 * tx + j : 128 + 4 * tx + j - 4;
          float z = acc[i][j] + bj[j];
          if (STAGE == BG_RGB) z = fmaxf(z, 0.f);
          else if (!feat_layer) z = softplus100(z);
          if (STAGE == BG_SDF && col >= L.N) z = emb[row * kBgEmbLd + (col - L.N)];  // skip connection (l == 3)
          v[j] = z;
        }
        if (feat_layer) {
          if (p < a.P) {
            *reinterpret_cast<float4*>(a.feat + (size_t)p * kFeat + 4 * tx) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(a.feat + (size_t)p * kFeat + 128 + 4 * tx) = make_float4(v[4], v[5], v[6], v[7]);
          }
        } else {
          *reinterpret_cast<float4*>(out + row * kBgActLd + 4 * tx) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(out + row * kBgActLd + 128 + 4 * tx) = make_float4(v[4], v[5], v[6], v[7]);
        }
      }
      __syncthreads();
      if (!feat_layer) { float* t = in; in = out; out = t; }
      const int warp = tid / 32;
      if (STAGE == BG_SDF && l == 7) {
        for (int i = 0; i < 8; ++i) {
          const int row = warp * 8 + i, p = p0 + row;
          float s = 0.f;
          for (int k = tx; k < 256; k += 32) s += in[row * kBgActLd + k] * a.w_last[k];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (tx == 0 && p < a.P) a.sdf[p] = s + a.b_last[0];
        }
      }
      if (STAGE == BG_RGB && l == a.n_layers - 1) {
        for (int i = 0; i < 8; ++i) {
          const int row = warp * 8 + i, p = p0 + row;
          for (int c = 0; c < 3; ++c) {
            float s = 0.f;
            for (int k = tx; k < 128; k += 32) s += in[row * kBgActLd + k] * a.w_last[c * 128 + k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (tx == 0 && p < a.P) a.rgb[3 * (size_t)p + c] = 1.0f / (1.0f + expf(-(s + a.b_last[c])));
          }
        }
      }
    }
  }
}
constexpr size_t kBgSmemBytes = (size_t)(2 * kTileRows * kBgActLd + 2 * kKC * 256 + kTileRows * kBgEmbLd) * sizeof(float);

// inverse_sample (ray_sampler.py:82-85, stratified when `jitter` [R,32] is given) + the per-sample inputs of Background.forward
// (background.py:56-100), one thread per (ray, flipped sample k), row p = ray * 32 + k: bg_z_vals [R,32] un-flipped, as
// inverse_sample returns it; PE-10 of depth2pts_outside -> pe_pts rows (84 columns); PE-4 of the view direction -> pe_view (27).
__global__ void __launch_bounds__(128) k_bg_encode(int R, float r_sphere, const float* __restrict__ cam, const float* __restrict__ dirs,
                                                   const float* __restrict__ jitter, float* __restrict__ z_out, float* __restrict__ pe_pts,
                                                   int ld_pts, float* __restrict__ pe_view, int ld_view) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R * kBgN) return;
  const int ray = p / kBgN, k = p % kBgN;
  const size_t zi = (size_t)ray * kBgN + (kBgN - 1 - k);
  const float depth = bg_depth(k, r_sphere, jitter ? jitter + zi : nullptr);
  z_out[zi] = depth;
  const float o[3] = {cam[3 * ray], cam[3 * ray + 1], cam[3 * ray + 2]};
  const float d[3] = {dirs[3 * ray], dirs[3 * ray + 1], dirs[3 * ray + 2]};
  float p4[4];
  depth2pts_outside(o, d, depth, r_sphere, p4);
  embed_generic<4, 10>(p4, pe_pts + (size_t)p * ld_pts);
  embed_generic<3, 4>(d, pe_view + (size_t)p * ld_view);
}

// bg_volume_rendering (background.py:137-165) over the flipped depths + Background.forward's outputs (:35-54).  z: the un-flipped
// depths [R,32] of hold_bg_encode, or NULL for the fixed shells (then z_bg, if given, receives them).
__global__ void k_bg_composite(int R, float r_sphere, const float* __restrict__ z, const float* __restrict__ sdf /*[R,32]*/,
                               const float* __restrict__ rgb /*[R,32,3]*/, const float* __restrict__ fg_bg_weights /*[R]*/,
                               float* __restrict__ bg_rgb, float* __restrict__ bg_rgb_only, float* __restrict__ bg_sem,
                               float* __restrict__ z_bg) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float acc[3];
  bg_integrate_ray(z ? z + (size_t)r * kBgN : nullptr, r_sphere, sdf + (size_t)r * kBgN, rgb + (size_t)r * kBgN * 3, acc);
  if (z_bg != nullptr)
    for (int k = 0; k < kBgN; ++k) z_bg[(size_t)r * kBgN + (kBgN - 1 - k)] = bg_depth(k, r_sphere);
  const float wbg = fg_bg_weights[r];
  for (int c = 0; c < 3; ++c) {
    if (bg_rgb_only) bg_rgb_only[3 * r + c] = acc[c];
    if (bg_rgb) bg_rgb[3 * r + c] = wbg * acc[c];
  }
  if (bg_sem) { bg_sem[4 * r] = wbg; bg_sem[4 * r + 1] = 0.f; bg_sem[4 * r + 2] = 0.f; bg_sem[4 * r + 3] = 0.f; }
}

// reverse mode of k_bg_composite w.r.t. sdf, rgb and fg_bg_weights (bg_phases.h), one warp per ray, lane k = flipped sample k:
// the transmittance is an exclusive prefix sum over the lanes, sum_{i>k} d w_i w_i an exclusive suffix sum.
__global__ void __launch_bounds__(128) k_bg_composite_bwd(int R, const float* __restrict__ z, const float* __restrict__ sdf,
                                                          const float* __restrict__ rgb, const float* __restrict__ fg_bg_weights,
                                                          const float* __restrict__ g_rgb, const float* __restrict__ g_only,
                                                          const float* __restrict__ g_sem, float* __restrict__ d_sdf,
                                                          float* __restrict__ d_rgb, float* __restrict__ d_wfg) {
  static_assert(kBgN == 32, "one lane per sample");
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) / 32, k = threadIdx.x % 32;
  if (r >= R) return;
  const size_t p = (size_t)r * kBgN + k;
  const float dist = bg_interval(z + (size_t)r * kBgN, 0.f, k);
  const float s = sdf[p];
  const float fe = dist * fabsf(s);
  float incl = fe;   // inclusive prefix sum of fe over the lanes
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if (k >= o) incl += v;
  }
  // exclusive sums by a shift, not by subtracting the own term: the last interval is 1e10 and would swamp the others
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (k == 0) excl = 0.f;
  float g[3];
  bg_bwd_seed(g_rgb ? g_rgb + 3 * r : nullptr, g_only ? g_only + 3 * r : nullptr, fg_bg_weights[r], g);
  const float* c = rgb + p * 3;
  const BgSampleBwd b = bg_bwd_sample(fe, excl, c, g, d_rgb + p * 3);
  float suf = b.dw * b.w;     // inclusive suffix sum of d w_i w_i
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_down_sync(0xffffffffu, suf, o);
    if (k + o < 32) suf += v;
  }
  float after = __shfl_down_sync(0xffffffffu, suf, 1);
  if (k == 31) after = 0.f;
  d_sdf[p] = bg_bwd_dsdf(b, after, dist, s);
  float only[3] = {b.w * c[0], b.w * c[1], b.w * c[2]};
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    for (int ch = 0; ch < 3; ++ch) only[ch] += __shfl_xor_sync(0xffffffffu, only[ch], o);
  if (k == 0) d_wfg[r] = bg_bwd_dwfg(only, g_rgb ? g_rgb + 3 * r : nullptr, g_sem ? g_sem + 4 * r : nullptr);
}

}  // namespace hold
