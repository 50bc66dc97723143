// hold_b200 — shared declarations for the sm_90a kernels behind include/hold_b200.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include <string>
#include <vector>

#include "../../include/hold_b200.h"
#include "bg_phases.h"

namespace hold {

constexpr int kVerts = 778;    // MANO vertices
constexpr int kJoints = 16;    // MANO bones (num_full_tfs, model/mano/specs.py)
constexpr int kKnn = 15;       // MANODeformer K (mano_node.py:28)
constexpr int kEmbed = 39;     // 3 + 3*2*6 (engine/embedders.py:21-41, multires 6)
constexpr int kFeat = 256;     // feature_vector_size
constexpr int kHidden = 256;
constexpr int kMaxZ = 640;     // n_samples_eval * max_total_iters upper bound supported by the sampler kernels

// device error word bits
constexpr int kErrRayMiss = 1;
constexpr int kErrNonFinite = 2;
constexpr int kErrBadFace = 4;   // a face's vertex index is outside [0, V) (the rasteriser skips the face)

struct SamplerState {  // device-resident, one per node; written only by single-thread epilogues
  int iters;           // rounds executed so far
  int done;            // 1 once the final sample set has been produced
  unsigned beta_max_bits[8];  // per round: max over rays of beta (float bits, positive => monotone)
};

// One MLP (node or background, skip net or colour net) packed for both arithmetic modes by pack_skip_net / pack_colour_net
// (api.cu).  Layers 0 .. n_layers-1 are the GEMM layers; the 1- or 3-row output head is kept apart as plain rows.
struct PackedNet {
  int n_layers = 0;
  int K[HOLD_MAX_LAYERS], Kpad[HOLD_MAX_LAYERS], N[HOLD_MAX_LAYERS];   // packed inputs, K padded to kKC, valid outputs
  float* Wt[HOLD_MAX_LAYERS] = {nullptr};       // fp32 CUDA-core layout [Kpad][256] (k-major rows, n contiguous)
  float* bias[HOLD_MAX_LAYERS] = {nullptr};     // [256], zero beyond N
  uint8_t* img[HOLD_MAX_LAYERS] = {nullptr};    // tensor-core forward images: nst[l] stages of 32 k (mlp_tc.cuh)
  int nst[HOLD_MAX_LAYERS] = {0};
  uint8_t* imgT[HOLD_MAX_LAYERS] = {nullptr};   // transposed images, 8 stages each: skip net W_l^T; colour net lin0^T to the
                                                // features, lin0^T to the other inputs, then W_1..^T
  float* bias_s = nullptr;                      // [n_layers][256]: the biases as the tensor-core epilogues add them
  float* w_last = nullptr;                      // head: skip net row 0 of lin8 [256]; colour net [3][hidden width]
  float* b_last = nullptr;
  float* w_last_tc = nullptr;                   // colour head padded to [3][256] when the hidden width is narrower (tensor cores)
};

// grow-only workspaces of a hold_ctx, one per purpose
enum WsSlot { WS_Z = 0, WS_SDF, WS_ZNEW, WS_SDFNEW, WS_BETA, WS_FAR, WS_XC, WS_SSDF, WS_GRAD, WS_FEAT, WS_PE, WS_ZTMP, WS_SIG,
              WS_BGSDF, WS_BGFEAT, WS_BGRGB, WS_AMAX, WS_WARPBWD, WS_RASTER, WS_COUNT };

struct NodeState {
  bool configured = false, has_weights = false, has_rig = false;
  hold_node_cfg cfg;
  PackedNet sdf, rgb;
  float* lin_pose_w = nullptr;  // [8,45]
  float* lin_pose_b = nullptr;  // [8]
  float* cano_verts = nullptr;  // [778,3]
  float* skin_w = nullptr;      // [778,16]
  unsigned short* knn_perm = nullptr;   // [49*16] vertex groups of the cluster-pruned KNN (knn_phases.h), 0xFFFF = padding
  SamplerState* sstate = nullptr;
};

struct Buffer {
  void* p = nullptr;
  size_t bytes = 0;
};

}  // namespace hold

struct hold_ctx {
  int device = 0;
  int sm_count = 132;
  hold::NodeState nodes[HOLD_MAX_NODES];
  int* dev_err = nullptr;
  int64_t launches = 0;
  hold::Buffer ws[hold::WS_COUNT];
  hold::PackedNet bg_sdf, bg_rgb;  // background nets (tensor-core images only when bg_mlp_mode is HOLD_MLP_TC)
  bool has_bg = false;
  int bg_mlp_mode = 0;             // HOLD_MLP_* of the background nets (hold_bg_set_weights)
  int sampler_passes = 3;          // measurement hook (hold_debug_set key 3): MMA passes of the sampler-round SDF launches
  int tc_acc_comp = -1;            // measurement hook (hold_debug_set key 2): accumulator scale 1 + c * 2^-24 in the SDF chains; < 0: kTcAccComp
};

namespace hold {

void set_error(const char* fmt, ...);
int ws_get(hold_ctx* ctx, int slot, size_t bytes, void** out);  // grow-only workspace (api.cu)
#define HOLD_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      hold::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return HOLD_E_CUDA;                                                                 \
    }                                                                                     \
  } while (0)
#define HOLD_REQUIRE(cond, ...)      \
  do {                               \
    if (!(cond)) {                   \
      hold::set_error(__VA_ARGS__);  \
      return HOLD_E_BADARG;          \
    }                                \
  } while (0)
#define HOLD_LAUNCH_CHECK(ctx)       \
  do {                               \
    (ctx)->launches++;               \
    HOLD_CUDA(cudaPeekAtLastError()); \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// LaplaceDensity.density_func (engine/density.py:21-26)
__device__ inline float laplace_density(float s, float beta) {
  float sg = (s > 0.f) ? 1.f : ((s < 0.f) ? -1.f : 0.f);
  return (1.0f / beta) * (0.5f + 0.5f * sg * expm1f(-fabsf(s) / beta));
}

// ---- NeRF++ background geometry (model/renderables/background.py), shared by background.cuh and the tensor-core variant;
// the sample depths (kBgN, bg_depth) are in bg_phases.h
constexpr int kBgEmbed = 84;    // 4 + 4*2*10
constexpr int kBgFrame = 32;    // dim_frame_encoding
constexpr int kBgView = 27;     // 3 + 3*2*4

// Background.depth2pts_outside (background.py:102-135)
__device__ __forceinline__ void depth2pts_outside(const float o[3], const float d[3], float depth, float R, float p4[4]) {
  const float odd = d[0] * o[0] + d[1] * o[1] + d[2] * o[2];
  const float under = odd * odd - ((o[0] * o[0] + o[1] * o[1] + o[2] * o[2]) - R * R);
  const float ds = sqrtf(under) - odd;
  float ps[3], pm[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { ps[c] = o[c] + ds * d[c]; pm[c] = o[c] - odd * d[c]; }
  const float pmn = sqrtf(pm[0] * pm[0] + pm[1] * pm[1] + pm[2] * pm[2]);
  float ax[3] = {o[1] * ps[2] - o[2] * ps[1], o[2] * ps[0] - o[0] * ps[2], o[0] * ps[1] - o[1] * ps[0]};
  const float an = sqrtf(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
#pragma unroll
  for (int c = 0; c < 3; ++c) ax[c] = ax[c] / an;
  const float phi = asinf(pmn / R), theta = asinf(pmn * depth);
  const float ang = phi - theta, ca = cosf(ang), sa = sinf(ang);
  const float cr[3] = {ax[1] * ps[2] - ax[2] * ps[1], ax[2] * ps[0] - ax[0] * ps[2], ax[0] * ps[1] - ax[1] * ps[0]};
  const float dp = ax[0] * ps[0] + ax[1] * ps[1] + ax[2] * ps[2];
  float pn[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) pn[c] = ps[c] * ca + cr[c] * sa + ax[c] * dp * (1.0f - ca);
  const float nn = sqrtf(pn[0] * pn[0] + pn[1] * pn[1] + pn[2] * pn[2]);
  p4[0] = pn[0] / nn, p4[1] = pn[1] / nn, p4[2] = pn[2] / nn, p4[3] = depth;
}

}  // namespace hold
