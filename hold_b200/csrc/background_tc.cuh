// Tensor-core path of the background nets (hold_bg_set_weights(..., HOLD_MLP_TC); HOLD_MLP_FP32 = the exact-fp32 CUDA-core path of background.cuh):
// k_mlp_tc<MLP_BG_SDF> = inverted-sphere point + PE-10 + frame code -> 8 x 256 Softplus(100) layers (skip at 4) -> sdf head
// + 256-d feature; k_mlp_tc<MLP_BG_RGB> = [feature | view PE-4 | frame code] (315) -> 128 ReLU -> 3 sigmoid.  Same fp16
// hi/lo split arithmetic as the foreground nets (tests/test_gpu_background.py holds it to the fp32 path).
#pragma once
#include "background.cuh"
#include "mlp_tc.cuh"

namespace hold {

__global__ void k_pad_rows(const float* __restrict__ src, int rows, int n_src, int n_dst, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * n_dst) return;
  const int r = i / n_dst, c = i % n_dst;
  dst[i] = (c < n_src) ? src[r * n_src + c] : 0.f;
}

static int tc_bg_init() {
  cudaError_t e = cudaFuncSetAttribute(k_mlp_tc<MLP_BG_SDF>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_BG_SDF>::kSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_tc<MLP_BG_RGB>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_BG_RGB>::kSmemBytes);
  if (e != cudaSuccess) { set_error("tensor-core background kernel attribute: %s", cudaGetErrorString(e)); return HOLD_E_CUDA; }
  return HOLD_OK;
}

// one frame chunk: P = rays * 32 points -> sdf [P], feat [P,256], then rgb [P,3]
static int tc_bg_launch(hold_ctx* ctx, int P, const float* cam, const float* dirs, const float* frame_code, float r_sphere,
                        float* sdf, float* feat, float* rgb, cudaStream_t s) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.P = P, a.n_layers = ctx->bg_sdf.n_layers, a.pts_per_frame = P;
  tc_layers(ctx->bg_sdf, true, a);
  a.cam = cam, a.dirs = dirs, a.frame_code = frame_code, a.r_sphere = r_sphere;
  a.sdf = sdf, a.feat = feat, a.err = ctx->dev_err, a.unscale = kTcUnscale, a.passes = 3;
  const int tiles = ceil_div(P, kTcRows), grid = min(tiles, ctx->sm_count);
  k_mlp_tc<MLP_BG_SDF><<<grid, kTcThreadsTotal, TcCfg<MLP_BG_SDF>::kSmemBytes, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  TcArgs c;
  memset(&c, 0, sizeof(c));
  c.P = P, c.n_layers = ctx->bg_rgb.n_layers, c.pts_per_frame = P;
  tc_layers(ctx->bg_rgb, false, c);
  c.dirs = dirs, c.frame_code = frame_code, c.feat = feat, c.rgb = rgb, c.err = ctx->dev_err, c.unscale = kTcUnscale, c.passes = 3;
  c.k0 = ctx->bg_rgb.K[0];
  k_mlp_tc<MLP_BG_RGB><<<grid, kTcThreadsTotal, TcCfg<MLP_BG_RGB>::kSmemBytes, s>>>(c);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

}  // namespace hold
