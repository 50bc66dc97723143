// Tensor-core path of the background nets (hold_bg_set_weights(..., HOLD_MLP_TC); HOLD_MLP_FP32 = the exact-fp32 CUDA-core path of background.cuh):
// k_mlp_tc<MLP_BG_SDF> = inverted-sphere point + PE-10 + frame code -> 8 x 256 Softplus(100) layers (skip at 4) -> sdf head
// + 256-d feature; k_mlp_tc<MLP_BG_RGB> = [feature | view PE-4 | frame code] (315) -> 128 ReLU -> 3 sigmoid.  Same fp16
// hi/lo split arithmetic as the foreground nets (tests/test_gpu_background.py holds it to the fp32 path).
#pragma once
#include "background.cuh"
#include "mlp_tc.cuh"

namespace hold {

struct TcBg {
  uint8_t* sdf_img[9] = {nullptr};
  int sdf_nst[9] = {0};
  uint8_t* rgb_img = nullptr;
  float* rgb_w_last = nullptr;   // [3][256]: lin1 rows padded from 128 to 256 columns with zeros
  uint8_t* sdf_imgT[9] = {nullptr};   // training backward: W_l^T of the 9 layers (l = 8: the feature rows)
  uint8_t* rgb_imgT[2] = {nullptr};   // colour lin0^T: to the 256 feature inputs / to [view (27) | frame code (32)]
  float* bias_s = nullptr;            // [10][256]: lin0..7 times kTcScaleA, lin8 (feature rows) plain, colour lin0 times kTcScaleA
};

__global__ void k_pad_rows(const float* __restrict__ src, int rows, int n_src, int n_dst, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * n_dst) return;
  const int r = i / n_dst, c = i % n_dst;
  dst[i] = (c < n_src) ? src[r * n_src + c] : 0.f;
}

static void tc_bg_free(TcBg*& t) {
  if (!t) return;
  for (int l = 0; l < 9; ++l) { cudaFree(t->sdf_img[l]); cudaFree(t->sdf_imgT[l]); }
  cudaFree(t->rgb_imgT[0]), cudaFree(t->rgb_imgT[1]);
  cudaFree(t->rgb_img), cudaFree(t->rgb_w_last), cudaFree(t->bias_s);
  delete t;
  t = nullptr;
}

static int tc_bg_init() {
  cudaError_t e = cudaFuncSetAttribute(k_mlp_tc<MLP_BG_SDF>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_BG_SDF>::kSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_tc<MLP_BG_RGB>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_BG_RGB>::kSmemBytes);
  if (e != cudaSuccess) { set_error("tensor-core background kernel attribute: %s", cudaGetErrorString(e)); return HOLD_E_CUDA; }
  return HOLD_OK;
}

// weight images of the plain (no weight-norm) background nets; ctx->bg_sdf / bg_rgb (fp32 packing) provide biases and heads
static int tc_bg_pack(hold_ctx* ctx, TcBg*& tp, const hold_mlp_weights* sdf, const hold_mlp_weights* rgb, cudaStream_t s) {
  if (!tp) tp = new TcBg();
  TcBg& t = *tp;
  for (int l = 0; l < 9; ++l) {
    const int K = (l == 0) ? kBgEmbed + kBgFrame : kHidden, kpad = (l == 0) ? 128 : 256;
    const int N = (l == 3) ? kHidden - kBgEmbed : kHidden, row_off = (l == 8) ? 1 : 0;
    t.sdf_nst[l] = kpad / 32;
    if (!t.sdf_img[l]) HOLD_CUDA(cudaMalloc((void**)&t.sdf_img[l], (size_t)t.sdf_nst[l] * kTcStageBytes));
    const float scale = (l == 4) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    k_tc_pack<<<256, 128, 0, s>>>(sdf->weight_v[l], nullptr, sdf->in_dim[l], row_off, N, K, kpad, scale, 0, t.sdf_img[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  const int K0 = kBgView + kBgFrame + kFeat;   // 315 -> 320
  if (!t.rgb_img) HOLD_CUDA(cudaMalloc((void**)&t.rgb_img, (size_t)10 * kTcStageBytes));
  k_tc_pack<<<256, 128, 0, s>>>(rgb->weight_v[0], nullptr, K0, 0, 128, K0, 320, 1.0f, kBgView + kBgFrame, t.rgb_img);
  HOLD_LAUNCH_CHECK(ctx);
  for (int l = 0; l < 9; ++l) {   // transposed images for the training backward (hold_linear, node = -1)
    const int K_in = (l == 0) ? kBgEmbed + kBgFrame : kHidden, N_out = (l == 3) ? kHidden - kBgEmbed : kHidden;
    if (!t.sdf_imgT[l]) HOLD_CUDA(cudaMalloc((void**)&t.sdf_imgT[l], (size_t)8 * kTcStageBytes));
    const float scale = (l == 4) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    k_tc_pack_T<<<256, 256, 0, s>>>(sdf->weight_v[l], nullptr, sdf->in_dim[l], l == 8 ? 1 : 0, N_out, K_in, 0, 0, scale, t.sdf_imgT[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int i = 0; i < 2; ++i) {
    if (!t.rgb_imgT[i]) HOLD_CUDA(cudaMalloc((void**)&t.rgb_imgT[i], (size_t)8 * kTcStageBytes));
    k_tc_pack_T<<<256, 256, 0, s>>>(rgb->weight_v[0], nullptr, K0, 0, 128, K0, i == 0 ? 1 : 2, kBgView + kBgFrame, 1.0f, t.rgb_imgT[i]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (!t.bias_s) HOLD_CUDA(cudaMalloc((void**)&t.bias_s, 10 * 256 * sizeof(float)));
  for (int l = 0; l < 10; ++l) {
    k_scale_vec<<<1, 256, 0, s>>>(l < 9 ? ctx->bg_sdf.bias[l] : ctx->bg_rgb.bias[0], 256, l == 8 ? 1.0f : kTcScaleA, t.bias_s + 256 * l);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (!t.rgb_w_last) HOLD_CUDA(cudaMalloc((void**)&t.rgb_w_last, 3 * 256 * sizeof(float)));
  k_pad_rows<<<3, 256, 0, s>>>(ctx->bg_rgb.w_last, 3, 128, 256, t.rgb_w_last);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

// one frame chunk: P = rays * 32 points -> sdf [P], feat [P,256], then rgb [P,3]
static int tc_bg_launch(hold_ctx* ctx, const TcBg& t, int P, const float* cam, const float* dirs, const float* frame_code,
                        float r_sphere, float* sdf, float* feat, float* rgb, cudaStream_t s) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.P = P, a.n_layers = 9, a.pts_per_frame = P;
  for (int l = 0; l < 9; ++l) {
    a.L[l].wimg = t.sdf_img[l], a.L[l].bias = t.bias_s + 256 * l, a.L[l].nst = t.sdf_nst[l];
    a.L[l].N = (l == 3) ? kHidden - kBgEmbed : kHidden;
  }
  a.w_last = ctx->bg_sdf.w_last, a.b_last = ctx->bg_sdf.b_last;
  a.cam = cam, a.dirs = dirs, a.frame_code = frame_code, a.r_sphere = r_sphere;
  a.sdf = sdf, a.feat = feat, a.err = ctx->dev_err, a.unscale = kTcUnscale, a.passes = 3;
  const int tiles = ceil_div(P, kTcRows), grid = min(tiles, ctx->sm_count);
  k_mlp_tc<MLP_BG_SDF><<<grid, kTcThreadsTotal, TcCfg<MLP_BG_SDF>::kSmemBytes, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  TcArgs c;
  memset(&c, 0, sizeof(c));
  c.P = P, c.n_layers = 1, c.pts_per_frame = P;
  c.L[0].wimg = t.rgb_img, c.L[0].bias = t.bias_s + 256 * 9, c.L[0].nst = 10, c.L[0].N = 256;
  c.w_last = t.rgb_w_last, c.b_last = ctx->bg_rgb.b_last;
  c.dirs = dirs, c.frame_code = frame_code, c.feat = feat, c.rgb = rgb, c.err = ctx->dev_err, c.unscale = kTcUnscale, c.passes = 3;
  c.k0 = kBgView + kBgFrame + kFeat;
  k_mlp_tc<MLP_BG_RGB><<<grid, kTcThreadsTotal, TcCfg<MLP_BG_RGB>::kSmemBytes, s>>>(c);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

}  // namespace hold
