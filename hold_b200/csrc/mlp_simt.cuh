// Fused fp32 (CUDA-core) MLP chains — the exact-arithmetic mode (HOLD_MLP_FP32) of the SDF net
// (ImplicitNet.forward, networks/shape_net.py:84-130) and the colour net (RenderingNet.forward,
// networks/texture_net.py:46-101).  One CTA keeps a 64-row activation tile in shared memory for the whole
// chain; weights stream through a cp.async double buffer; nothing but inputs/outputs touches HBM.
//
// The SDF gradient (engine/volsdf_utils.py:89-96, autograd in the reference) is computed in FORWARD mode:
// a point occupies 4 consecutive rows [value, d/dx, d/dy, d/dz]; tangent rows see the same GEMMs (no bias)
// and are multiplied by softplus'(z) of their value row.
#pragma once
#include "common.cuh"

namespace hold {

enum { MLP_SDF_ONLY = 0, MLP_SDF_JVP = 1, MLP_COLOR = 2, MLP_SDF_REV = 3, MLP_BG_SDF = 4, MLP_BG_RGB = 5, MLP_LINEAR = 6 };  // 4, 5, 6: tensor cores only

constexpr int kTileRows = 64;
constexpr int kActLd = 308;   // >= 304 (colour-net input 302 -> 304) + 4
constexpr int kKC = 16;       // k-chunk of the weight pipeline
constexpr int kEmbLd = 40;

struct SimtLayer {
  const float* Wt;   // [Kpad][256]
  const float* bias; // [256]
  int Kpad;
  int N;             // valid outputs (<= 256)
};

struct SimtArgs {
  int P;                       // points
  int n_layers;                // GEMM layers (SDF: 8 (+1 feature layer in JVP mode), colour: 4)
  SimtLayer L[HOLD_MAX_LAYERS];
  const float* w_last;         // SDF: [256]; colour: [3][256]
  const float* b_last;         // SDF: [1];   colour: [3]
  // SDF inputs/outputs
  const float* xc;             // [P,3]
  const float* embed_w;        // [39] or NULL
  float* sdf;                  // [P]
  float* grad;                 // [P,3]   (JVP)
  float* feat;                 // [P,256] (JVP)
  // colour inputs/outputs
  const float* normal;         // [P,3]
  const float* pose_embed;     // [B,8] or NULL (zeros)
  const float* time_code;      // [B,32] or NULL
  int pts_per_frame;
  int k0;                      // colour-net true input width (270 / 302)
  float* rgb;                  // [P,3]
  const SamplerState* st;      // non-NULL: skip when the sampler has converged
};

__device__ __forceinline__ float softplus100(float x) {
  // nn.Softplus(beta=100), threshold 20 (shape_net.py:82)
  float bx = x * 100.0f;
  return (bx > 20.0f) ? x : log1pf(expf(bx)) / 100.0f;
}
__device__ __forceinline__ float softplus100_grad(float x) {
  float bx = x * 100.0f;
  float z = expf(bx);
  return (bx > 20.0f) ? 1.0f : z / (z + 1.0f);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Fourier embedding (engine/embedders.py:48-51) of a point, or its derivative w.r.t. coordinate c-1.
__device__ __forceinline__ void embed_row(float* dst /*[>=48]*/, float x, float y, float z, int comp,
                                          const float* __restrict__ ew, int kpad) {
  float p[3] = {x, y, z};
  for (int e = 0; e < kEmbed; ++e) {
    int d = e % 3;
    float v;
    if (e < 3) {
      v = (comp == 0) ? p[d] : ((comp - 1 == d) ? 1.0f : 0.0f);
    } else {
      int q = (e - 3) / 3;        // 0: sin f0, 1: cos f0, 2: sin f1, ...
      float f = (float)(1 << (q >> 1));
      float arg = p[d] * f;
      if (comp == 0) v = (q & 1) ? cosf(arg) : sinf(arg);
      else v = (comp - 1 == d) ? ((q & 1) ? -f * sinf(arg) : f * cosf(arg)) : 0.0f;
    }
    if (ew != nullptr) v *= ew[e];
    dst[e] = v;
  }
  for (int e = kEmbed; e < kpad; ++e) dst[e] = 0.0f;
}

template <int MODE>
__global__ void __launch_bounds__(256, 1) k_mlp_simt(SimtArgs a) {
  if (a.st != nullptr && a.st->done) return;
  extern __shared__ __align__(16) float smem[];
  float* actA = smem;
  float* actB = actA + kTileRows * kActLd;
  float* wbuf = actB + kTileRows * kActLd;       // [2][kKC][256]
  float* emb = wbuf + 2 * kKC * 256;             // [64][kEmbLd]
  const int tid = threadIdx.x, tx = tid % 32, ty = tid / 32;
  constexpr int RPP = (MODE == MLP_SDF_JVP) ? 4 : 1;  // rows per point
  constexpr int PPT = kTileRows / RPP;                // points per tile
  const int n_tiles = ceil_div(a.P, PPT);

  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p0 = tile * PPT;
    __syncthreads();
    // ---------------------------------------------------------------- prologue: build the layer-0 input tile
    if (MODE != MLP_COLOR) {
      if (tid < kTileRows) {
        int row = tid, p = p0 + row / RPP, comp = row % RPP;
        float x = 0.f, y = 0.f, z = 0.f;
        if (p < a.P) { x = a.xc[3 * (size_t)p], y = a.xc[3 * (size_t)p + 1], z = a.xc[3 * (size_t)p + 2]; }
        embed_row(emb + row * kEmbLd, x, y, z, comp, a.embed_w, kEmbLd);
        for (int e = 0; e < 48; ++e) actA[row * kActLd + e] = (e < kEmbLd) ? emb[row * kEmbLd + e] : 0.f;
      }
    } else {
      // [x_c(3), n(3), pose_embed(8), feat(256) (+ time_code(32))], zero padded to Kpad
      const int kpad = a.L[0].Kpad;
      for (int idx = tid; idx < kTileRows * kpad; idx += 256) {
        int row = idx / kpad, e = idx % kpad;
        int p = p0 + row;
        float v = 0.f;
        if (p < a.P) {
          int b = p / a.pts_per_frame;
          if (e < 3) v = a.xc[3 * (size_t)p + e];
          else if (e < 6) v = a.normal[3 * (size_t)p + e - 3];
          else if (e < 14) v = (a.pose_embed != nullptr) ? a.pose_embed[b * 8 + e - 6] : 0.f;
          else if (e < 14 + kFeat) v = a.feat[(size_t)p * kFeat + e - 14];
          else if (e < a.k0) v = a.time_code[b * 32 + e - 14 - kFeat];
        }
        actA[row * kActLd + e] = v;
      }
    }
    __syncthreads();
    float* in = actA;
    float* out = actB;
    // ---------------------------------------------------------------- GEMM chain
    for (int l = 0; l < a.n_layers; ++l) {
      const SimtLayer L = a.L[l];
      float acc[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      const int nchunks = L.Kpad / kKC;
      // prefetch chunk 0
      {
        const float* src = L.Wt;
        for (int q = tid; q < kKC * 64; q += 256) cp_async16(wbuf + q * 4, src + q * 4);
        cp_async_commit();
      }
      for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
          const float* src = L.Wt + (size_t)(c + 1) * kKC * 256;
          float* dst = wbuf + ((c + 1) & 1) * kKC * 256;
          for (int q = tid; q < kKC * 64; q += 256) cp_async16(dst + q * 4, src + q * 4);
          cp_async_commit();
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        __syncthreads();
        const float* w = wbuf + (c & 1) * kKC * 256;
        const float* arow = in + (ty * 8) * kActLd + c * kKC;
#pragma unroll
        for (int kq = 0; kq < kKC; kq += 4) {
          float4 av[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) av[i] = *reinterpret_cast<const float4*>(arow + i * kActLd + kq);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            float4 w0 = *reinterpret_cast<const float4*>(w + (kq + kk) * 256 + 4 * tx);
            float4 w1 = *reinterpret_cast<const float4*>(w + (kq + kk) * 256 + 128 + 4 * tx);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              float av_ = (kk == 0) ? av[i].x : (kk == 1) ? av[i].y : (kk == 2) ? av[i].z : av[i].w;
              acc[i][0] += av_ * w0.x; acc[i][1] += av_ * w0.y; acc[i][2] += av_ * w0.z; acc[i][3] += av_ * w0.w;
              acc[i][4] += av_ * w1.x; acc[i][5] += av_ * w1.y; acc[i][6] += av_ * w1.z; acc[i][7] += av_ * w1.w;
            }
          }
        }
        __syncthreads();
      }
      // ------------------------------------------------------------ epilogue
      const bool feat_layer = (MODE == MLP_SDF_JVP) && (l == a.n_layers - 1);
      float bj[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) bj[j] = L.bias[(j < 4 ? 4 * tx + j : 128 + 4 * tx + j - 4)];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = ty * 8 + i;
        const bool is_value = (MODE != MLP_SDF_JVP) || (row % 4 == 0);
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = (j < 4) ? 4 * tx + j : 128 + 4 * tx + j - 4;
          float z = acc[i][j] + (is_value ? bj[j] : 0.f);
          if (MODE == MLP_COLOR) z = fmaxf(z, 0.f);
          else if (MODE == MLP_SDF_ONLY) z = softplus100(z);
          if (MODE != MLP_COLOR && col >= L.N) z = emb[row * kEmbLd + (col - L.N)];  // skip connection (l == 3)
          v[j] = z;
        }
        if (feat_layer) {
          int p = p0 + row / 4;
          if (is_value && p < a.P) {
            *reinterpret_cast<float4*>(a.feat + (size_t)p * kFeat + 4 * tx) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(a.feat + (size_t)p * kFeat + 128 + 4 * tx) = make_float4(v[4], v[5], v[6], v[7]);
          }
        } else {
          *reinterpret_cast<float4*>(out + row * kActLd + 4 * tx) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(out + row * kActLd + 128 + 4 * tx) = make_float4(v[4], v[5], v[6], v[7]);
        }
      }
      __syncthreads();
      if (MODE == MLP_SDF_JVP && !feat_layer) {
        // activation pass: value rows a = softplus(z); tangent rows *= softplus'(z)
        for (int idx = tid; idx < PPT * 256; idx += 256) {
          int pt = idx / 256, col = idx % 256;
          if (col >= L.N) continue;  // embedding columns of the skip layer are already final
          float* base = out + (pt * 4) * kActLd + col;
          float z = base[0];
          float s = softplus100_grad(z);
          base[0] = softplus100(z);
          base[kActLd] *= s, base[2 * kActLd] *= s, base[3 * kActLd] *= s;
        }
        __syncthreads();
      }
      if (!feat_layer) { float* t = in; in = out; out = t; }
      // ------------------------------------------------------------ heads that hang off this layer's output
      if (MODE != MLP_COLOR && l == 7) {
        // sdf = w_sdf . a7 + b  (row 0 of lin8); tangent rows give d sdf / d x_c
        const int warp = tid / 32;
        for (int i = 0; i < 8; ++i) {
          int row = warp * 8 + i;
          float s = 0.f;
          for (int k = tx; k < 256; k += 32) s += in[row * kActLd + k] * a.w_last[k];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (tx == 0) {
            int p = p0 + row / RPP, comp = row % RPP;
            if (p < a.P) {
              if (comp == 0) a.sdf[p] = s + a.b_last[0];
              else a.grad[3 * (size_t)p + comp - 1] = s;
            }
          }
        }
      }
      if (MODE == MLP_COLOR && l == a.n_layers - 1) {
        const int warp = tid / 32;
        for (int i = 0; i < 8; ++i) {
          int row = warp * 8 + i, p = p0 + row;
          for (int c = 0; c < 3; ++c) {
            float s = 0.f;
            for (int k = tx; k < 256; k += 32) s += in[row * kActLd + k] * a.w_last[c * 256 + k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (tx == 0 && p < a.P) a.rgb[3 * (size_t)p + c] = 1.0f / (1.0f + expf(-(s + a.b_last[c])));
          }
        }
      }
    }
  }
}

constexpr size_t kSimtSmemBytes = (size_t)(2 * kTileRows * kActLd + 2 * kKC * 256 + kTileRows * kEmbLd) * sizeof(float);

// ------------------------------------------------------------------------------------------------ packing
// Fold weight-norm (w = v * g/||v||, shape_net.py:80) and write Wt[k][n] = scale * w[row_off + n][col_off + k]
// for k < K, n < N; zero elsewhere in the [Kpad][256] block.  One block per output row n.
__global__ void k_pack_layer(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ bias,
                             int in_dim, int row_off, int col_off, int K, int N, int Kpad, float scale,
                             float* __restrict__ Wt, float* __restrict__ b_out) {
  int n = blockIdx.x;  // 0..255
  __shared__ float red[32];
  float f = 0.f;
  if (n < N) {
    const float* vr = v + (size_t)(row_off + n) * in_dim;
    if (g != nullptr) {
      float ss = 0.f;
      for (int k = threadIdx.x; k < in_dim; k += blockDim.x) ss += vr[k] * vr[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = ss;
      __syncthreads();
      float tot = 0.f;
      for (int w = 0; w < blockDim.x / 32; ++w) tot += red[w];
      f = g[row_off + n] / sqrtf(tot);
    } else {
      f = 1.0f;
    }
    for (int k = threadIdx.x; k < Kpad; k += blockDim.x)
      Wt[(size_t)k * 256 + n] = (k < K) ? scale * (vr[col_off + k] * f) : 0.f;
    if (threadIdx.x == 0 && b_out != nullptr) b_out[n] = bias[row_off + n];
  } else {
    for (int k = threadIdx.x; k < Kpad; k += blockDim.x) Wt[(size_t)k * 256 + n] = 0.f;
    if (threadIdx.x == 0 && b_out != nullptr) b_out[n] = 0.f;
  }
}

// rows of a layer as plain vectors (sdf head / rgb head): out[r][k] = folded w[row_off + r][k]
__global__ void k_pack_rows(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ bias,
                            int in_dim, int row_off, int rows, float* __restrict__ out, float* __restrict__ b_out) {
  int r = blockIdx.x;
  if (r >= rows) return;
  __shared__ float red[32];
  const float* vr = v + (size_t)(row_off + r) * in_dim;
  float f = 1.0f;
  if (g != nullptr) {
    float ss = 0.f;
    for (int k = threadIdx.x; k < in_dim; k += blockDim.x) ss += vr[k] * vr[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < blockDim.x / 32; ++w) tot += red[w];
    f = g[row_off + r] / sqrtf(tot);
  }
  for (int k = threadIdx.x; k < in_dim; k += blockDim.x) out[(size_t)r * in_dim + k] = vr[k] * f;
  if (threadIdx.x == 0) b_out[r] = bias[row_off + r];
}

// lin_pose(pose_cond) per frame (texture_net.py:82): pe[b][o] = W[o,:] . cond[b,:] + bias[o]
__global__ void k_pose_embed(int B, const float* __restrict__ cond, const float* __restrict__ W,
                             const float* __restrict__ bias, float* __restrict__ pe) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 8) return;
  int b = i / 8, o = i % 8;
  float s = 0.f;
  for (int k = 0; k < 45; ++k) s += cond[b * 45 + k] * W[o * 45 + k];
  pe[i] = s + bias[o];
}

}  // namespace hold
