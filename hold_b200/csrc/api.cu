// C ABI of hold_b200 (include/hold_b200.h): context, weight packing, launch sequences.  Host-side logic
// only — every arithmetic step of the path lives in the kernels included below.
#include <stdarg.h>
#include <stdlib.h>
#include <new>
#include <algorithm>

#include "common.cuh"
#include "geom.cuh"
#include "sampler.cuh"
#include "mlp_simt.cuh"
#include "mlp_tc.cuh"
#include "composite.cuh"
#include "background.cuh"
#include "background_tc.cuh"
#include "pose_bwd.cuh"
#include "mesh_sdf.cuh"
#include "mesh_bvh.cuh"
#include "raster.cuh"
#include "pointcloud.cuh"
#include "mise.cuh"
#include "mc.cuh"
#include "warp_bwd.cuh"
#include "train.cuh"
#include "wgrad_tc.cuh"
#include "decimate.cuh"
#include "mesh_cc.cuh"

namespace hold {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int ws_get(hold_ctx* ctx, int slot, size_t bytes, void** out) {
  Buffer& b = ctx->ws[slot];
  if (b.bytes < bytes) {
    if (b.p) HOLD_CUDA(cudaFree(b.p));
    b.p = nullptr, b.bytes = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
      set_error("workspace allocation of %zu bytes failed: %s", want, cudaGetErrorString(e));
      return HOLD_E_NOMEM;
    }
    b.bytes = want;
  }
  *out = b.p;
  return HOLD_OK;
}
#define WS(slot, type, count, var)                                                     \
  type* var = nullptr;                                                                 \
  {                                                                                    \
    void* _p;                                                                          \
    int _rc = ws_get(ctx, slot, sizeof(type) * (size_t)(count), &_p);                  \
    if (_rc) return _rc;                                                               \
    var = (type*)_p;                                                                   \
  }

static int dev_alloc(float** p, size_t n) {
  if (*p) return HOLD_OK;
  HOLD_CUDA(cudaMalloc((void**)p, n * sizeof(float)));
  return HOLD_OK;
}

static int check_node(hold_ctx* ctx, int node, bool need_weights) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(node >= 0 && node < HOLD_MAX_NODES, "node %d out of range", node);
  if (!ctx->nodes[node].configured) { set_error("node %d not configured", node); return HOLD_E_STATE; }
  if (need_weights && !ctx->nodes[node].has_weights) { set_error("node %d has no weights", node); return HOLD_E_STATE; }
  HOLD_CUDA(cudaSetDevice(ctx->device));   // launches go to the context's device whatever the caller's current device is
  return HOLD_OK;
}

// ------------------------------------------------------------------------------------------------ the two MLP shapes
// Skip net (ImplicitNet, networks/shape_net.py:13-49, and the background's implicit net): 9 Softplus layers, lin0 -> 256 x3 ->
// lin3 (256 - d_skip) -> [a_3 | embedding] / sqrt 2 -> 256 x4 -> lin8 (257: row 0 the sdf head, rows 1..256 the feature vector).
struct SkipNetShape {
  const char* name;   // in error messages
  int in_dim0;        // lin0 inputs of the caller's weights
  int k_in;           // lin0 inputs packed (the hand's 45 pose columns multiply zeros, shape_net.py:104-106)
  int d_skip;         // embedding columns re-fed at the skip
  int tc_kpad0;       // lin0's K padded in the tensor-core image
  bool weight_norm;   // weight_g allowed
  int n_out(int l) const { return l == 3 ? kHidden - d_skip : kHidden; }   // packed outputs (lin8: the feature rows)
  float scale(int l) const { return l == 4 ? (float)(1.0 / sqrt(2.0)) : 1.0f; }   // skip_in: cat([x, input]) / sqrt(2)
  int row_off(int l) const { return l == 8 ? 1 : 0; }   // lin8 row 0 is the sdf head (packed apart), rows 1..256 the features
};
// Colour net (RenderingNet, networks/texture_net.py:13-44, and the background's rendering net): lin0 over k0 inputs, n_hidden
// ReLU layers of `width` outputs in all, a 3-row sigmoid head.  Its tensor-core lin0 takes the 256 features first in A.
struct ColourNetShape {
  const char* name;
  int k0;             // lin0 inputs
  int lead;           // lin0 inputs before the features: [x_c, n, pose embed] (| time code after them) / [view PE-4, frame code]
  int width;          // hidden width
  int n_hidden;       // GEMM layers before the head
  bool weight_norm;
};
static SkipNetShape node_sdf_shape(bool hand) { return {"SDF", hand ? kEmbed + 45 : kEmbed, kEmbed, kEmbed, 64, true}; }
static ColourNetShape node_rgb_shape(bool hand) { return {"colour", hand ? 270 : 302, 14, 256, 4, true}; }
constexpr SkipNetShape kBgSdfShape = {"bg", kBgEmbed + kBgFrame, kBgEmbed + kBgFrame, kBgEmbed, 128, false};
constexpr ColourNetShape kBgRgbShape = {"bg colour", kBgView + kBgFrame + kFeat, kBgView + kBgFrame, 128, 1, false};

static int check_layer_tensors(const hold_mlp_weights* w, int l, const char* name, bool weight_norm) {
  HOLD_REQUIRE(w->weight_v[l] && w->bias[l], "%s lin%d has NULL tensors", name, l);
  HOLD_REQUIRE(weight_norm || !w->weight_g[l], "%s lin%d has weight_g, but this net has no weight-norm", name, l);
  return HOLD_OK;
}

static int check_skip_net(const hold_mlp_weights* w, const SkipNetShape& s) {
  HOLD_REQUIRE(w->n_layers == 9, "%s net must have 9 layers, got %d", s.name, w->n_layers);
  HOLD_REQUIRE(w->in_dim[0] == s.in_dim0, "%s lin0 in_dim %d, expected %d", s.name, w->in_dim[0], s.in_dim0);
  for (int l = 0; l < 9; ++l) {
    const int eo = (l == 8) ? kFeat + 1 : s.n_out(l), ei = (l == 0) ? s.in_dim0 : kHidden;
    HOLD_REQUIRE(w->out_dim[l] == eo && w->in_dim[l] == ei, "%s lin%d is %dx%d, expected %dx%d", s.name, l, w->out_dim[l], w->in_dim[l], eo, ei);
    int rc = check_layer_tensors(w, l, s.name, s.weight_norm);
    if (rc) return rc;
  }
  return HOLD_OK;
}

static int check_colour_net(const hold_mlp_weights* w, const ColourNetShape& s) {
  HOLD_REQUIRE(w->n_layers == s.n_hidden + 1, "%s net must have %d layers, got %d", s.name, s.n_hidden + 1, w->n_layers);
  HOLD_REQUIRE(w->in_dim[0] == s.k0, "%s lin0 in_dim %d, expected %d", s.name, w->in_dim[0], s.k0);
  for (int l = 0; l <= s.n_hidden; ++l) {
    const int eo = (l == s.n_hidden) ? 3 : s.width, ei = (l == 0) ? s.k0 : s.width;
    HOLD_REQUIRE(w->out_dim[l] == eo && w->in_dim[l] == ei, "%s lin%d is %dx%d, expected %dx%d", s.name, l, w->out_dim[l], w->in_dim[l], eo, ei);
    int rc = check_layer_tensors(w, l, s.name, s.weight_norm);
    if (rc) return rc;
  }
  return HOLD_OK;
}

// ------------------------------------------------------------------------------------------------ packing
// Both packers fold weight-norm and write the fp32 layout and the head; with `tc` also the tensor-core forward and transposed
// images and the scaled biases.  Buffers are allocated on first use and rewritten in place on every later call.
static int pack_skip_net(hold_ctx* ctx, PackedNet& m, const hold_mlp_weights* w, const SkipNetShape& s, bool tc, cudaStream_t st) {
  int rc;
  m.n_layers = 9;
  for (int l = 0; l < 9; ++l) {
    const int K = (l == 0) ? s.k_in : kHidden, Kpad = round_up(K, kKC);
    m.K[l] = K, m.Kpad[l] = Kpad, m.N[l] = s.n_out(l);
    if ((rc = dev_alloc(&m.Wt[l], (size_t)Kpad * 256))) return rc;
    if ((rc = dev_alloc(&m.bias[l], 256))) return rc;
    k_pack_layer<<<256, 128, 0, st>>>(w->weight_v[l], w->weight_g[l], w->bias[l], w->in_dim[l], s.row_off(l), 0, K, m.N[l], Kpad, s.scale(l),
                                      m.Wt[l], m.bias[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if ((rc = dev_alloc(&m.w_last, 256))) return rc;
  if ((rc = dev_alloc(&m.b_last, 4))) return rc;
  k_pack_rows<<<1, 128, 0, st>>>(w->weight_v[8], w->weight_g[8], w->bias[8], 256, 0, 1, m.w_last, m.b_last);
  HOLD_LAUNCH_CHECK(ctx);
  if (!tc) return HOLD_OK;
  for (int l = 0; l < 9; ++l) {
    const int kpad = (l == 0) ? s.tc_kpad0 : 256;
    m.nst[l] = kpad / 32;
    if (!m.img[l]) HOLD_CUDA(cudaMalloc((void**)&m.img[l], (size_t)m.nst[l] * kTcStageBytes));
    k_tc_pack<<<256, 128, 0, st>>>(w->weight_v[l], w->weight_g[l], w->in_dim[l], s.row_off(l), m.N[l], m.K[l], kpad, s.scale(l), 0, m.img[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int l = 0; l < 9; ++l) {  // W_l^T: layers 7..0 for the reverse-mode gradient, all 9 for the training backward
    if (!m.imgT[l]) HOLD_CUDA(cudaMalloc((void**)&m.imgT[l], (size_t)8 * kTcStageBytes));
    k_tc_pack_T<<<256, 256, 0, st>>>(w->weight_v[l], w->weight_g[l], w->in_dim[l], s.row_off(l), m.N[l], m.K[l], 0, 0, s.scale(l), m.imgT[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (!m.bias_s) HOLD_CUDA(cudaMalloc((void**)&m.bias_s, 9 * 256 * sizeof(float)));
  for (int l = 0; l < 9; ++l) {  // lin8 (the feature rows) is added unscaled
    k_scale_vec<<<1, 256, 0, st>>>(m.bias[l], 256, l == 8 ? 1.0f : kTcScaleA, m.bias_s + 256 * l);
    HOLD_LAUNCH_CHECK(ctx);
  }
  return HOLD_OK;
}

static int pack_colour_net(hold_ctx* ctx, PackedNet& m, const hold_mlp_weights* w, const ColourNetShape& s, bool tc, cudaStream_t st) {
  int rc;
  const int H = s.n_hidden;
  m.n_layers = H;
  for (int l = 0; l < H; ++l) {
    const int K = (l == 0) ? s.k0 : s.width, Kpad = round_up(K, kKC);
    m.K[l] = K, m.Kpad[l] = Kpad, m.N[l] = s.width;
    if ((rc = dev_alloc(&m.Wt[l], (size_t)Kpad * 256))) return rc;
    if ((rc = dev_alloc(&m.bias[l], 256))) return rc;
    k_pack_layer<<<256, 128, 0, st>>>(w->weight_v[l], w->weight_g[l], w->bias[l], w->in_dim[l], 0, 0, K, s.width, Kpad, 1.0f, m.Wt[l], m.bias[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if ((rc = dev_alloc(&m.w_last, 3 * s.width))) return rc;
  if ((rc = dev_alloc(&m.b_last, 4))) return rc;
  k_pack_rows<<<3, 128, 0, st>>>(w->weight_v[H], w->weight_g[H], w->bias[H], s.width, 0, 3, m.w_last, m.b_last);
  HOLD_LAUNCH_CHECK(ctx);
  if (!tc) return HOLD_OK;
  for (int l = 0; l < H; ++l) {  // lin0: A = [feature (256) | the other inputs], K padded to 320
    const int kpad = (l == 0) ? 320 : 256;
    m.nst[l] = kpad / 32;
    if (!m.img[l]) HOLD_CUDA(cudaMalloc((void**)&m.img[l], (size_t)m.nst[l] * kTcStageBytes));
    k_tc_pack<<<256, 128, 0, st>>>(w->weight_v[l], w->weight_g[l], w->in_dim[l], 0, s.width, m.K[l], kpad, 1.0f, l == 0 ? s.lead : 0, m.img[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int i = 0; i <= H; ++i) {  // transposes for the training backward: lin0 in two parts (its K = 320 > 256), then lin1..
    const int l = (i < 2) ? 0 : i - 1;
    if (!m.imgT[i]) HOLD_CUDA(cudaMalloc((void**)&m.imgT[i], (size_t)8 * kTcStageBytes));
    k_tc_pack_T<<<256, 256, 0, st>>>(w->weight_v[l], w->weight_g[l], w->in_dim[l], 0, s.width, w->in_dim[l], i == 0 ? 1 : (i == 1 ? 2 : 0), s.lead,
                                     1.0f, m.imgT[i]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (!m.bias_s) HOLD_CUDA(cudaMalloc((void**)&m.bias_s, (size_t)H * 256 * sizeof(float)));
  for (int l = 0; l < H; ++l) {
    k_scale_vec<<<1, 256, 0, st>>>(m.bias[l], 256, kTcScaleA, m.bias_s + 256 * l);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (s.width < 256) {  // the tensor-core head reads 256 columns
    if (!m.w_last_tc) HOLD_CUDA(cudaMalloc((void**)&m.w_last_tc, 3 * 256 * sizeof(float)));
    k_pad_rows<<<3, 256, 0, st>>>(m.w_last, 3, s.width, 256, m.w_last_tc);
    HOLD_LAUNCH_CHECK(ctx);
  }
  return HOLD_OK;
}

static void free_net(PackedNet& m) {
  for (int l = 0; l < HOLD_MAX_LAYERS; ++l) cudaFree(m.Wt[l]), cudaFree(m.bias[l]), cudaFree(m.img[l]), cudaFree(m.imgT[l]);
  cudaFree(m.bias_s), cudaFree(m.w_last), cudaFree(m.b_last), cudaFree(m.w_last_tc);
}

// hold_linear's matrix ids (include/hold_b200.h), the same for a node's nets and the background's
struct LinearMat {
  const uint8_t* img = nullptr;
  const float* bias = nullptr;
  int nst = 8, kmax = 0, nmax = 0;
};
static LinearMat linear_mat(const PackedNet& sdf, const PackedNet& rgb, int mat) {
  if (mat >= 0 && mat < sdf.n_layers) return {sdf.img[mat], sdf.bias[mat], sdf.nst[mat], sdf.K[mat], sdf.N[mat]};
  if (mat >= 16 && mat < 16 + sdf.n_layers) { const int l = mat - 16; return {sdf.imgT[l], nullptr, 8, sdf.N[l], sdf.K[l]}; }
  if (mat >= 32 && mat < 32 + rgb.n_layers) { const int l = mat - 32; return {rgb.img[l], rgb.bias[l], rgb.nst[l], 32 * rgb.nst[l], rgb.N[l]}; }
  if (mat >= 48 && mat <= 48 + rgb.n_layers) {  // lin0^T to the features / to the other inputs (at most 64), then lin1..^T
    const int i = mat - 48;
    return {rgb.imgT[i], nullptr, 8, rgb.N[i < 2 ? 0 : i - 1], i == 0 ? kFeat : (i == 1 ? 64 : rgb.K[i - 1])};
  }
  return {};
}

// ------------------------------------------------------------------------------------------------ MLP launches
// SimtArgs / BgArgs: layers 0 .. n-1 of a packed net's fp32 chain and its head
template <class Args>
static void simt_layers(const PackedNet& m, int n, Args& a) {
  a.n_layers = n;
  for (int l = 0; l < n; ++l) a.L[l].Wt = m.Wt[l], a.L[l].bias = m.bias[l], a.L[l].Kpad = m.Kpad[l], a.L[l].N = m.N[l];
  a.w_last = m.w_last, a.b_last = m.b_last;
}

static int launch_sdf(hold_ctx* ctx, NodeState& ns, int P, const float* xc, const float* embed_w, float* sdf,
                      float* grad, float* feat, const SamplerState* st, cudaStream_t s) {
  if (P <= 0) return HOLD_OK;
  const bool jvp = (grad != nullptr) || (feat != nullptr);
  if (ns.cfg.mlp_mode == HOLD_MLP_TC) return tc_launch_sdf(ctx, ns.sdf, P, xc, embed_w, sdf, grad, feat, st, s);
  SimtArgs a;
  memset(&a, 0, sizeof(a));
  simt_layers(ns.sdf, jvp ? 9 : 8, a);
  a.P = P, a.xc = xc, a.embed_w = embed_w, a.sdf = sdf, a.grad = grad, a.feat = feat, a.st = st;
  if (jvp) {
    HOLD_REQUIRE(grad != nullptr && feat != nullptr, "sdf eval with gradient needs both grad and feat buffers");
    int tiles = ceil_div(P, kTileRows / 4);
    k_mlp_simt<MLP_SDF_JVP><<<min(tiles, ctx->sm_count), 256, kSimtSmemBytes, s>>>(a);
  } else {
    int tiles = ceil_div(P, kTileRows);
    k_mlp_simt<MLP_SDF_ONLY><<<min(tiles, ctx->sm_count), 256, kSimtSmemBytes, s>>>(a);
  }
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

static int launch_rgb(hold_ctx* ctx, NodeState& ns, int P, int pts_per_frame, const float* xc, const float* normal,
                      const float* pe, const float* feat, const float* time_code, float* rgb, cudaStream_t s) {
  if (P <= 0) return HOLD_OK;
  if (ns.cfg.mlp_mode == HOLD_MLP_TC) return tc_launch_rgb(ctx, ns.rgb, P, pts_per_frame, xc, normal, pe, feat, time_code, rgb, s);
  SimtArgs a;
  memset(&a, 0, sizeof(a));
  simt_layers(ns.rgb, ns.rgb.n_layers, a);
  a.P = P, a.xc = xc, a.normal = normal, a.pose_embed = pe, a.feat = const_cast<float*>(feat), a.time_code = time_code;
  a.pts_per_frame = pts_per_frame, a.k0 = ns.rgb.K[0], a.rgb = rgb;
  int tiles = ceil_div(P, kTileRows);
  k_mlp_simt<MLP_COLOR><<<min(tiles, ctx->sm_count), 256, kSimtSmemBytes, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

static int launch_inverse_warp(hold_ctx* ctx, NodeState& ns, int B, int pts_per_frame, bool from_z, int nsamp, int zstride,
                               const float* zbuf, const float* cam, const float* dirs, const float* xin,
                               const hold_node_pose* pose, float* xc, int* knn_idx, uint8_t* outlier,
                               const SamplerState* st, cudaStream_t s) {
  if (pts_per_frame <= 0 || B <= 0) return HOLD_OK;
  dim3 grid(ceil_div(pts_per_frame, 128), B);
  const bool hand = ns.cfg.kind == HOLD_KIND_HAND;
  if (hand) {
    HOLD_REQUIRE(pose->posed_verts != nullptr, "hand node needs posed_verts");
    if (!ns.has_rig) { set_error("hand node has no rig (hold_node_set_rig)"); return HOLD_E_STATE; }
  }
  if (hand && from_z && knn_idx == nullptr && outlier == nullptr) {
    // hot path: consecutive samples of a ray per thread, KNN seeded from the previous sample
    const int rays = pts_per_frame / nsamp;
    // walk length per thread: 32 samples when that still fills the GPU (>= 2 waves of 4 blocks per SM), else shorter walks
    int seg_len = kSeg;
    while (seg_len > 4 && (long long)B * rays * ceil_div(nsamp, seg_len) < (long long)ctx->sm_count * 4 * 128 * 2) seg_len >>= 1;
    const int segs = ceil_div(nsamp, seg_len);
    dim3 g2(ceil_div(rays * segs, 128), B);
    k_inverse_warp_hand_rays<<<g2, 128, 0, s>>>(rays, nsamp, seg_len, zstride, zbuf, cam, dirs, pose->tfs, pose->posed_verts, ns.skin_w, ns.knn_perm, xc, st);
    HOLD_LAUNCH_CHECK(ctx);
    return HOLD_OK;
  }
#define IW(H, Z) k_inverse_warp<H, Z><<<grid, 128, 0, s>>>(pts_per_frame, nsamp, zstride, zbuf, cam, dirs, xin, pose->tfs, \
                                                          pose->posed_verts, ns.skin_w, xc, knn_idx, outlier, st, ctx->dev_err)
  if (hand && from_z) IW(true, true);
  else if (hand) IW(true, false);
  else if (from_z) IW(false, true);
  else IW(false, false);
#undef IW
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

}  // namespace hold

using namespace hold;

// ================================================================================================ C ABI
extern "C" {

int hold_version(void) { return HOLD_B200_VERSION; }
const char* hold_last_error(void) { return g_err; }

int hold_ctx_create(hold_ctx** out, int device) {
  HOLD_REQUIRE(out != nullptr, "out is NULL");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    set_error("no CUDA device: %s (hold_b200 has no CPU fallback)", cudaGetErrorString(e));
    return HOLD_E_CUDA;
  }
  HOLD_REQUIRE(device >= 0 && device < count, "device %d out of range (%d devices)", device, count);
  HOLD_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  HOLD_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; hold_b200 is built for sm_90a only", device, prop.major, prop.minor);
    return HOLD_E_CUDA;
  }
  hold_ctx* ctx = new (std::nothrow) hold_ctx();
  if (!ctx) { set_error("out of host memory"); return HOLD_E_NOMEM; }
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  HOLD_CUDA(cudaMalloc((void**)&ctx->dev_err, sizeof(int)));
  HOLD_CUDA(cudaMemset(ctx->dev_err, 0, sizeof(int)));
  HOLD_CUDA(cudaFuncSetAttribute(k_mlp_simt<MLP_SDF_ONLY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSimtSmemBytes));
  HOLD_CUDA(cudaFuncSetAttribute(k_mlp_simt<MLP_SDF_JVP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSimtSmemBytes));
  HOLD_CUDA(cudaFuncSetAttribute(k_mlp_simt<MLP_COLOR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSimtSmemBytes));
  const int samp_smem = 4 * 6 * kMaxZ * (int)sizeof(float);
  HOLD_CUDA(cudaFuncSetAttribute(k_sampler_merge_beta, cudaFuncAttributeMaxDynamicSharedMemorySize, samp_smem));
  HOLD_CUDA(cudaFuncSetAttribute(k_sampler_resample, cudaFuncAttributeMaxDynamicSharedMemorySize, samp_smem));
  HOLD_CUDA(cudaFuncSetAttribute(k_bg_mlp<BG_SDF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBgSmemBytes));
  HOLD_CUDA(cudaFuncSetAttribute(k_bg_mlp<BG_RGB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBgSmemBytes));
  int rc = tc_init(ctx);
  if (rc == HOLD_OK) rc = wgrad_init();
  if (rc == HOLD_OK) rc = tc_bg_init();
  if (rc) { delete ctx; return rc; }
  *out = ctx;
  return HOLD_OK;
}

int hold_ctx_destroy(hold_ctx* ctx) {
  if (!ctx) return HOLD_OK;
  cudaSetDevice(ctx->device);
  for (Buffer& b : ctx->ws) cudaFree(b.p);
  for (NodeState& ns : ctx->nodes) {
    free_net(ns.sdf), free_net(ns.rgb);
    cudaFree(ns.lin_pose_w), cudaFree(ns.lin_pose_b), cudaFree(ns.cano_verts), cudaFree(ns.skin_w), cudaFree(ns.sstate), cudaFree(ns.knn_perm);
  }
  free_net(ctx->bg_sdf), free_net(ctx->bg_rgb);
  cudaFree(ctx->dev_err);
  delete ctx;
  return HOLD_OK;
}

int hold_ctx_check(hold_ctx* ctx, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  cudaStream_t s = (cudaStream_t)stream;
  int h = 0;
  HOLD_CUDA(cudaMemcpyAsync(&h, ctx->dev_err, sizeof(int), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaStreamSynchronize(s));
  if (h != 0) HOLD_CUDA(cudaMemsetAsync(ctx->dev_err, 0, sizeof(int), s));
  if (h & 0x100) { set_error("tensor-core pipeline wait timed out (tag %d): protocol error in k_mlp_tc", (h >> 12) & 0xF); return HOLD_E_STATE; }
  if (h & kErrRayMiss) { set_error("a ray misses the scene bounding sphere (engine/ray_sampler.py:15-18)"); return HOLD_E_RAY_MISSES_SPHERE; }
  if (h & kErrNonFinite) { set_error("non-finite value (singular transform)"); return HOLD_E_NONFINITE; }
  if (h & kErrBadFace) { set_error("a face's vertex index is outside [0, V): the rasteriser skipped the face"); return HOLD_E_BADARG; }
  if (h & kErrBadLength) { set_error("a point-cloud length is outside [0, P]: the kernel clamped it"); return HOLD_E_BADARG; }
  if (h & kErrBadMeshIndex) { set_error("a face's vertex index is outside [0, V): hold_decimate returned the mesh unchanged"); return HOLD_E_BADARG; }
  if (h & kErrBadSdfFace) { set_error("a face's vertex index is outside [0, V): hold_mesh_sdf_bvh wrote NaN and face -1"); return HOLD_E_BADARG; }
  if (h & kErrBadCcFace) { set_error("a face's vertex index is outside [0, V): hold_largest_component returned an empty mesh"); return HOLD_E_BADARG; }
  return HOLD_OK;
}

int64_t hold_ctx_launch_count(hold_ctx* ctx) { return ctx ? ctx->launches : -1; }

int hold_node_configure(hold_ctx* ctx, int node, const hold_node_cfg* cfg) {
  HOLD_REQUIRE(ctx != nullptr && cfg != nullptr, "NULL argument");
  HOLD_REQUIRE(node >= 0 && node < HOLD_MAX_NODES, "node %d out of range", node);
  HOLD_REQUIRE(cfg->kind == HOLD_KIND_HAND || cfg->kind == HOLD_KIND_OBJECT, "bad kind %d", cfg->kind);
  HOLD_REQUIRE(cfg->class_id >= 0 && cfg->class_id < 4, "class_id %d out of [0,4)", cfg->class_id);
  HOLD_REQUIRE(cfg->n_samples_eval >= 2 && cfg->max_total_iters >= 1 && cfg->max_total_iters <= 8 &&
                   cfg->n_samples_eval * cfg->max_total_iters <= kMaxZ,
               "sampler buffer: n_samples_eval * max_total_iters must be <= %d", kMaxZ);
  HOLD_REQUIRE(cfg->n_samples >= 1 && cfg->n_samples <= cfg->n_samples_eval * cfg->max_total_iters, "bad n_samples");
  HOLD_REQUIRE(cfg->n_samples + cfg->n_samples_extra + 2 <= 512, "final sample count too large");
  HOLD_REQUIRE(cfg->mlp_mode == HOLD_MLP_FP32 || cfg->mlp_mode == HOLD_MLP_TC, "bad mlp_mode");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  NodeState& ns = ctx->nodes[node];
  ns.cfg = *cfg;
  if (!ns.sstate) HOLD_CUDA(cudaMalloc((void**)&ns.sstate, sizeof(SamplerState)));
  HOLD_CUDA(cudaMemset(ns.sstate, 0, sizeof(SamplerState)));
  ns.configured = true;
  return HOLD_OK;
}

int hold_node_set_weights(hold_ctx* ctx, int node, const hold_mlp_weights* sdf, const hold_mlp_weights* rgb,
                          const float* lin_pose_w, const float* lin_pose_b, void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  HOLD_REQUIRE(sdf != nullptr && rgb != nullptr, "NULL weights");
  NodeState& ns = ctx->nodes[node];
  cudaStream_t s = (cudaStream_t)stream;
  const bool hand = ns.cfg.kind == HOLD_KIND_HAND;
  const SkipNetShape ss = node_sdf_shape(hand);
  const ColourNetShape cs = node_rgb_shape(hand);
  if ((rc = check_skip_net(sdf, ss)) || (rc = check_colour_net(rgb, cs))) return rc;
  HOLD_REQUIRE(!hand || (lin_pose_w && lin_pose_b), "hand node needs lin_pose weights");
  // both arithmetic modes are packed: hold_linear (the training backward) uses the tensor-core images in either mode
  if ((rc = pack_skip_net(ctx, ns.sdf, sdf, ss, true, s)) || (rc = pack_colour_net(ctx, ns.rgb, rgb, cs, true, s))) return rc;
  if (hand) {
    rc = dev_alloc(&ns.lin_pose_w, 8 * 45);
    if (rc) return rc;
    rc = dev_alloc(&ns.lin_pose_b, 8);
    if (rc) return rc;
    HOLD_CUDA(cudaMemcpyAsync(ns.lin_pose_w, lin_pose_w, 8 * 45 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    HOLD_CUDA(cudaMemcpyAsync(ns.lin_pose_b, lin_pose_b, 8 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  ns.has_weights = true;
  return HOLD_OK;
}

int hold_node_set_rig(hold_ctx* ctx, int node, const float* cano_verts, const float* skin_weights, void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  HOLD_REQUIRE(cano_verts && skin_weights, "NULL rig tensors");
  NodeState& ns = ctx->nodes[node];
  HOLD_REQUIRE(ns.cfg.kind == HOLD_KIND_HAND, "only hand nodes have a rig");
  cudaStream_t s = (cudaStream_t)stream;
  rc = dev_alloc(&ns.cano_verts, kVerts * 3);
  if (rc) return rc;
  rc = dev_alloc(&ns.skin_w, kVerts * kJoints);
  if (rc) return rc;
  HOLD_CUDA(cudaMemcpyAsync(ns.cano_verts, cano_verts, kVerts * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemcpyAsync(ns.skin_w, skin_weights, kVerts * kJoints * sizeof(float), cudaMemcpyDeviceToDevice, s));
  {  // vertex groups of the cluster-pruned KNN (knn_phases.h): ordered once on the canonical hand, on the host
    static_assert(knnc::kNV == kVerts && knnc::kK == kKnn, "knn_phases.h constants");
    float* hv = (float*)malloc(sizeof(float) * kVerts * (3 + kJoints));
    HOLD_REQUIRE(hv != nullptr, "out of host memory");
    cudaError_t e = cudaMemcpyAsync(hv, ns.cano_verts, kVerts * 3 * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hv + kVerts * 3, ns.skin_w, kVerts * kJoints * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    unsigned short perm[knnc::kNCl * knnc::kClSize];
    if (e == cudaSuccess) {
      knnc::cluster_order(hv, hv + kVerts * 3, kJoints, perm);
      if (!ns.knn_perm) e = cudaMalloc((void**)&ns.knn_perm, sizeof(perm));
      if (e == cudaSuccess) e = cudaMemcpyAsync(ns.knn_perm, perm, sizeof(perm), cudaMemcpyHostToDevice, s);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // `perm` is a stack buffer
    }
    free(hv);
    if (e != cudaSuccess) { set_error("hold_node_set_rig: %s", cudaGetErrorString(e)); return HOLD_E_CUDA; }
  }
  ns.has_rig = true;
  return HOLD_OK;
}

int hold_mano_lbs(hold_ctx* ctx, const hold_mano_model* m, int B, const float* betas, const float* full_pose,
                  const float* transl, const float* scene_scale, const float* tfs_c_inv, float* verts, float* jnts,
                  float* tfs, float* v_posed, void* stream) {
  HOLD_REQUIRE(ctx && m, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(B >= 0, "negative batch");
  if (B == 0) return HOLD_OK;
  HOLD_REQUIRE(betas && full_pose && transl && scene_scale && verts && jnts && tfs && v_posed, "NULL tensor");
  HOLD_REQUIRE(m->parents_host && m->tip_ids_host, "NULL host arrays in mano model");
  ManoDev d;
  d.v_template = m->v_template, d.shapedirs = m->shapedirs, d.posedirs = m->posedirs, d.J_regressor = m->J_regressor;
  d.lbs_weights = m->lbs_weights, d.hands_mean = m->hands_mean;
  for (int i = 0; i < kJoints; ++i) {
    d.parents[i] = (i == 0) ? 0 : m->parents_host[i];
    HOLD_REQUIRE(i == 0 || (d.parents[i] >= 0 && d.parents[i] < i), "parents must be topologically ordered");
  }
  for (int i = 0; i < 5; ++i) {
    d.tips[i] = m->tip_ids_host[i];
    HOLD_REQUIRE(d.tips[i] >= 0 && d.tips[i] < kVerts, "tip id out of range");
  }
  constexpr int smem = (2 * kVerts * 3 + kJoints * 3 + kJoints * 9 + 136 + 2 * kJoints * 16 + 16) * (int)sizeof(float);
  static_assert(smem <= 48 * 1024, "k_mano_lbs fits the default dynamic shared memory limit (no per-device attribute needed)");
  k_mano_lbs<<<B, 256, smem, (cudaStream_t)stream>>>(d, betas, full_pose, transl, scene_scale, tfs_c_inv, verts, jnts, tfs, v_posed);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_mano_lbs_bwd(hold_ctx* ctx, const hold_mano_model* m, int B, const float* betas, const float* full_pose,
                      const float* transl, const float* scene_scale, const float* tfs_c_inv, const float* g_verts,
                      const float* g_jnts, const float* g_tfs, float* g_betas, float* g_pose, float* g_transl, float* g_scale,
                      void* stream) {
  HOLD_REQUIRE(ctx && m, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(B >= 0, "negative batch");
  if (B == 0) return HOLD_OK;
  HOLD_REQUIRE(betas && full_pose && transl && scene_scale && g_betas && g_pose && g_transl && g_scale, "NULL tensor");
  HOLD_REQUIRE(m->parents_host && m->tip_ids_host, "NULL host arrays in mano model");
  posebwd::ManoPtrs d;
  d.v_template = m->v_template, d.shapedirs = m->shapedirs, d.posedirs = m->posedirs, d.J_regressor = m->J_regressor;
  d.lbs_weights = m->lbs_weights, d.hands_mean = m->hands_mean;
  for (int i = 0; i < kJoints; ++i) {
    d.parents[i] = (i == 0) ? 0 : m->parents_host[i];
    HOLD_REQUIRE(i == 0 || (d.parents[i] >= 0 && d.parents[i] < i), "parents must be topologically ordered");
  }
  for (int i = 0; i < 5; ++i) {
    d.tips[i] = m->tip_ids_host[i];
    HOLD_REQUIRE(d.tips[i] >= 0 && d.tips[i] < kVerts, "tip id out of range");
  }
  const int nt = 256, smem = posebwd::mano_scratch_floats(nt) * (int)sizeof(float);
  HOLD_REQUIRE(smem <= 48 * 1024, "k_mano_lbs_bwd scratch exceeds the default dynamic shared memory limit");
  k_mano_lbs_bwd<<<B, nt, smem, (cudaStream_t)stream>>>(d, betas, full_pose, transl, scene_scale, tfs_c_inv, g_verts, g_jnts, g_tfs,
                                                        g_betas, g_pose, g_transl, g_scale);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_object_tf_bwd(hold_ctx* ctx, int B, const float* rot, const float* trans, const float* scene_scale, float obj_scale,
                       const float* denorm_mat, const float* pts_cano, int Nv, const float* g_verts, const float* g_tfs,
                       float* g_rot, float* g_trans, float* g_scene_scale, float* g_obj_scale, void* stream) {
  HOLD_REQUIRE(ctx && rot && trans && scene_scale && denorm_mat && g_rot && g_trans && g_scene_scale && g_obj_scale, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  if (B <= 0) return HOLD_OK;
  HOLD_REQUIRE(g_verts == nullptr || (pts_cano != nullptr && Nv > 0), "g_verts given without canonical points");
  const int nt = 256, smem = posebwd::obj_scratch_floats(nt) * (int)sizeof(float);
  k_object_tf_bwd<<<B, nt, smem, (cudaStream_t)stream>>>(Nv, rot, trans, scene_scale, obj_scale, denorm_mat, pts_cano, g_verts, g_tfs,
                                                         g_rot, g_trans, g_scene_scale, g_obj_scale);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_object_tf(hold_ctx* ctx, int B, const float* rot, const float* trans, const float* scene_scale, float obj_scale,
                   const float* denorm_mat, const float* pts_cano, int Nv, float* tfs, float* verts, void* stream) {
  HOLD_REQUIRE(ctx && rot && trans && scene_scale && denorm_mat && tfs, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  if (B <= 0) return HOLD_OK;
  HOLD_REQUIRE(verts == nullptr || (pts_cano != nullptr && Nv > 0), "verts requested without canonical points");
  dim3 grid(verts ? max(1, min(ceil_div(Nv, 128), 64)) : 1, B);
  k_object_tf<<<grid, 128, 0, (cudaStream_t)stream>>>(B, Nv, rot, trans, scene_scale, obj_scale, denorm_mat, pts_cano, tfs, verts);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_camera_rays(hold_ctx* ctx, int B, int P, const float* uv, const float* pose, const float* intrinsics,
                     float* ray_dirs, float* cam_loc, void* stream) {
  HOLD_REQUIRE(ctx && uv && pose && intrinsics && ray_dirs && cam_loc, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  if (B * P <= 0) return HOLD_OK;
  k_camera_rays<<<ceil_div(B * P, 256), 256, 0, (cudaStream_t)stream>>>(B, P, uv, pose, intrinsics, ray_dirs, cam_loc);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_sample(hold_ctx* ctx, int node, int R, int B, const float* cam_loc, const float* ray_dirs,
                const hold_node_pose* pose, const hold_sampler_rand* rnd, float* z_vals, int32_t* iters, void* stream) {
  int rc = check_node(ctx, node, true);
  if (rc) return rc;
  HOLD_REQUIRE(R >= 0 && B >= 1, "bad R/B");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(R % B == 0, "R (%d) must be B (%d) frames x rays, frame-major", R, B);
  HOLD_REQUIRE(cam_loc && ray_dirs && pose && z_vals, "NULL argument");
  HOLD_REQUIRE(pose->tfs && pose->beta_param, "pose needs tfs and beta_param");
  NodeState& ns = ctx->nodes[node];
  const hold_node_cfg& c = ns.cfg;
  cudaStream_t s = (cudaStream_t)stream;
  const int Ne = c.n_samples_eval;
  WS(WS_Z, float, (size_t)R * kMaxZ, zb);
  WS(WS_SDF, float, (size_t)R * kMaxZ, sb);
  WS(WS_ZNEW, float, (size_t)R * Ne, znew);
  WS(WS_SDFNEW, float, (size_t)R * Ne, sdfnew);
  WS(WS_BETA, float, R, betab);
  WS(WS_FAR, float, R, farb);
  WS(WS_XC, float, (size_t)R * Ne * 3, xc);
  SamplerArgs a;
  memset(&a, 0, sizeof(a));
  a.R = R, a.rays_per_frame = R / B;
  a.n_eval = Ne, a.n_samples = c.n_samples, a.n_extra = c.n_samples_extra, a.beta_iters = c.beta_iters, a.max_iters = c.max_total_iters;
  a.eps = c.eps, a.add_tiny = c.add_tiny, a.near = c.near, a.r_sphere = c.bounding_sphere, a.beta_min = c.beta_min;
  a.cam = cam_loc, a.dirs = ray_dirs, a.beta_param = pose->beta_param;
  a.z = zb, a.sdf = sb, a.znew = znew, a.sdfnew = sdfnew, a.beta = betab, a.far = farb, a.st = ns.sstate, a.err = ctx->dev_err;
  if (rnd) { a.jitter = rnd->jitter, a.u_rand = rnd->u, a.extra_idx = rnd->extra_idx; }
  a.z_out = z_vals, a.iters_out = iters;
  const int wpb = 4;
  k_sampler_init<<<ceil_div(R, wpb), wpb * 32, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  for (int it = 0; it < c.max_total_iters; ++it) {
    if (it > 0) {
      k_round_gate<<<1, 1, 0, s>>>(ns.sstate, it, pose->beta_param, c.beta_min, c.max_total_iters);
      HOLD_LAUNCH_CHECK(ctx);
    }
    rc = launch_inverse_warp(ctx, ns, B, (R / B) * Ne, true, Ne, Ne, znew, cam_loc, ray_dirs, nullptr, pose, xc, nullptr,
                             nullptr, ns.sstate, s);
    if (rc) return rc;
    rc = launch_sdf(ctx, ns, R * Ne, xc, pose->embed_w, sdfnew, nullptr, nullptr, ns.sstate, s);
    if (rc) return rc;
    const int cap = sampler_cap(it, Ne, c.n_samples + c.n_samples_extra + 2);
    const int samp_smem = wpb * 6 * cap * (int)sizeof(float);
    k_sampler_merge_beta<<<ceil_div(R, wpb), wpb * 32, samp_smem, s>>>(a, it, cap);
    HOLD_LAUNCH_CHECK(ctx);
    k_sampler_resample<<<ceil_div(R, wpb), wpb * 32, samp_smem, s>>>(a, it, cap);
    HOLD_LAUNCH_CHECK(ctx);
  }
  return HOLD_OK;
}

/* One iteration of the while loop of ErrorBoundSampler.get_z_vals (engine/ray_sampler.py:160-311) on caller-supplied state:
 * the sorted (z, sdf) of the previous rounds, this round's new samples and their sdf, beta per ray.  Runs exactly the kernels
 * hold_sample runs for round `it` (merge + d* + beta line search, then PDF -> inverse CDF), so that a round can be compared
 * with the reference in isolation (teacher forcing): upstream last-bit differences do not propagate into it. */
int hold_sampler_round(hold_ctx* ctx, int node, int R, int it, const float* z_old, const float* sdf_old, const float* z_new,
                       const float* sdf_new, const float* beta_in, const float* far, const float* beta_param,
                       float* z_merged, float* sdf_merged, float* beta_out, float* samples_out, int32_t* upsample_out,
                       void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  NodeState& ns = ctx->nodes[node];
  const hold_node_cfg& c = ns.cfg;
  HOLD_REQUIRE(R >= 0 && it >= 0 && it < c.max_total_iters, "bad R / round index");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(z_new && sdf_new && beta_in && far && beta_param && beta_out && samples_out, "NULL argument");
  HOLD_REQUIRE(it == 0 || (z_old && sdf_old), "round %d needs the previous rounds' (z, sdf)", it);
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int Ne = c.n_samples_eval, n_old = it * Ne, n = n_old + Ne;
  WS(WS_Z, float, (size_t)R * kMaxZ, zb);
  WS(WS_SDF, float, (size_t)R * kMaxZ, sb);
  WS(WS_ZNEW, float, (size_t)R * Ne, znew);
  WS(WS_SDFNEW, float, (size_t)R * Ne, sdfnew);
  WS(WS_BETA, float, R, betab);
  WS(WS_FAR, float, R, farb);
  WS(WS_ZTMP, float, (size_t)R * 512, zfin);
  if (n_old > 0) {
    HOLD_CUDA(cudaMemcpy2DAsync(zb, kMaxZ * sizeof(float), z_old, n_old * sizeof(float), n_old * sizeof(float), R, cudaMemcpyDeviceToDevice, s));
    HOLD_CUDA(cudaMemcpy2DAsync(sb, kMaxZ * sizeof(float), sdf_old, n_old * sizeof(float), n_old * sizeof(float), R, cudaMemcpyDeviceToDevice, s));
  }
  HOLD_CUDA(cudaMemcpyAsync(znew, z_new, (size_t)R * Ne * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemcpyAsync(sdfnew, sdf_new, (size_t)R * Ne * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemcpyAsync(betab, beta_in, (size_t)R * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemcpyAsync(farb, far, (size_t)R * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemsetAsync(ns.sstate, 0, sizeof(SamplerState), s));
  SamplerArgs a;
  memset(&a, 0, sizeof(a));
  a.R = R, a.rays_per_frame = R;
  a.n_eval = Ne, a.n_samples = c.n_samples, a.n_extra = c.n_samples_extra, a.beta_iters = c.beta_iters, a.max_iters = c.max_total_iters;
  a.eps = c.eps, a.add_tiny = c.add_tiny, a.near = c.near, a.r_sphere = c.bounding_sphere, a.beta_min = c.beta_min;
  a.beta_param = beta_param;
  a.z = zb, a.sdf = sb, a.znew = znew, a.sdfnew = sdfnew, a.beta = betab, a.far = farb, a.st = ns.sstate, a.err = ctx->dev_err;
  a.z_out = zfin, a.iters_out = nullptr;
  const int wpb = 4;
  const int cap = sampler_cap(it, Ne, c.n_samples + c.n_samples_extra + 2);
  const int samp_smem = wpb * 6 * cap * (int)sizeof(float);
  k_sampler_merge_beta<<<ceil_div(R, wpb), wpb * 32, samp_smem, s>>>(a, it, cap);
  HOLD_LAUNCH_CHECK(ctx);
  if (z_merged) HOLD_CUDA(cudaMemcpy2DAsync(z_merged, n * sizeof(float), zb, kMaxZ * sizeof(float), n * sizeof(float), R, cudaMemcpyDeviceToDevice, s));
  if (sdf_merged) HOLD_CUDA(cudaMemcpy2DAsync(sdf_merged, n * sizeof(float), sb, kMaxZ * sizeof(float), n * sizeof(float), R, cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemcpyAsync(beta_out, betab, (size_t)R * sizeof(float), cudaMemcpyDeviceToDevice, s));
  k_sampler_resample<<<ceil_div(R, wpb), wpb * 32, samp_smem, s>>>(a, it, cap);
  HOLD_LAUNCH_CHECK(ctx);
  // upsample decision of this round (ray_sampler.py:244-246), read back for the caller: it sizes samples_out
  unsigned int bits = 0;
  float b0 = 0.f;
  HOLD_CUDA(cudaMemcpyAsync(&bits, &ns.sstate->beta_max_bits[it], sizeof(bits), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaMemcpyAsync(&b0, beta_param, sizeof(float), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaStreamSynchronize(s));
  float bm;
  memcpy(&bm, &bits, sizeof(bm));
  const bool upsample = (bm > fabsf(b0) + c.beta_min) && (it + 1 < c.max_total_iters);
  if (upsample_out) *upsample_out = upsample ? 1 : 0;
  if (upsample) {
    HOLD_CUDA(cudaMemcpyAsync(samples_out, znew, (size_t)R * Ne * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else {
    const int S = c.n_samples + c.n_samples_extra + 2;
    HOLD_CUDA(cudaMemcpyAsync(samples_out, zfin, (size_t)R * S * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  return HOLD_OK;
}

int hold_shade(hold_ctx* ctx, int node, int R, int B, int S, const float* cam_loc, const float* ray_dirs,
               const hold_node_pose* pose, const hold_factors* out, void* stream) {
  int rc = check_node(ctx, node, true);
  if (rc) return rc;
  HOLD_REQUIRE(R >= 0 && B >= 1 && S >= 1, "bad R/B/S");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(R % B == 0, "R (%d) must be B (%d) frames x rays, frame-major", R, B);
  HOLD_REQUIRE(cam_loc && ray_dirs && pose && out, "NULL argument");
  HOLD_REQUIRE(out->z_vals && out->color && out->normal && out->density, "factors need z_vals, color, normal, density");
  HOLD_REQUIRE(pose->tfs && pose->beta_param, "pose needs tfs and beta_param");
  NodeState& ns = ctx->nodes[node];
  const bool hand = ns.cfg.kind == HOLD_KIND_HAND;
  if (!hand) HOLD_REQUIRE(pose->time_code != nullptr, "object node needs time_code");
  cudaStream_t s = (cudaStream_t)stream;
  const int rpf = R / B;
  const int max_pts = 1 << 20;
  const int rays_per_chunk = max(1, min(rpf, max_pts / S));
  const size_t cp = (size_t)rays_per_chunk * S;
  // canonical points of the WHOLE call in one launch (full grid, one vertex-group setup per block instead of one per 1 Mi-point
  // chunk, whose launches fill only part of a wave); the MLP stages below are chunked for their 1 GB feature buffer
  float* xc_all = out->canonical_pts;
  if (xc_all == nullptr) {
    WS(WS_XC, float, (size_t)R * S * 3, xc_ws);
    xc_all = xc_ws;
  }
  WS(WS_SSDF, float, cp, sdf_ws);
  WS(WS_GRAD, float, cp * 3, grad_ws);
  WS(WS_FEAT, float, cp * kFeat, feat_ws);
  float* pe = nullptr;
  if (hand && pose->pose_cond != nullptr) {
    WS(WS_PE, float, (size_t)B * 8, pe_ws);
    pe = pe_ws;
    k_pose_embed<<<ceil_div(B * 8, 64), 64, 0, s>>>(B, pose->pose_cond, ns.lin_pose_w, ns.lin_pose_b, pe);
    HOLD_LAUNCH_CHECK(ctx);
  } else if (hand) {
    // RenderingNet with a 45-dim pose of zeros still applies lin_pose: embed = bias (texture_net.py:80-82)
    HOLD_REQUIRE(false, "hand node needs pose_cond (pass zeros for the first 20 training epochs)");
  }
  rc = launch_inverse_warp(ctx, ns, B, rpf * S, true, S, S, out->z_vals, cam_loc, ray_dirs, nullptr, pose, xc_all, nullptr, nullptr, nullptr, s);
  if (rc) return rc;
  for (int b = 0; b < B; ++b) {
    hold_node_pose pb = *pose;
    pb.tfs = pose->tfs + (size_t)b * (hand ? kJoints * 16 : 16);
    if (hand) pb.posed_verts = pose->posed_verts + (size_t)b * kVerts * 3;
    for (int r0 = 0; r0 < rpf; r0 += rays_per_chunk) {
      const int rc_n = min(rays_per_chunk, rpf - r0);
      const size_t ray0 = (size_t)b * rpf + r0;
      const int P = rc_n * S;
      float* xc = xc_all + ray0 * S * 3;
      float* sdf = out->sdf ? out->sdf + ray0 * S : sdf_ws;
      rc = launch_sdf(ctx, ns, P, xc, pose->embed_w, sdf, grad_ws, feat_ws, nullptr, s);
      if (rc) return rc;
      dim3 grid(ceil_div(P, 128), 1);
      if (hand)
        k_normals_density<true><<<grid, 128, 0, s>>>(P, xc, grad_ws, sdf, pb.tfs, ns.cano_verts, ns.skin_w, pose->beta_param,
                                                    ns.cfg.beta_min, out->normal + ray0 * S * 3, out->density + ray0 * S);
      else
        k_normals_density<false><<<grid, 128, 0, s>>>(P, xc, grad_ws, sdf, pb.tfs, nullptr, nullptr, pose->beta_param,
                                                     ns.cfg.beta_min, out->normal + ray0 * S * 3, out->density + ray0 * S);
      HOLD_LAUNCH_CHECK(ctx);
      rc = launch_rgb(ctx, ns, P, P, xc, out->normal + ray0 * S * 3, pe ? pe + b * 8 : nullptr, feat_ws,
                      hand ? nullptr : pose->time_code + b * 32, out->color + ray0 * S * 3, s);
      if (rc) return rc;
    }
  }
  return HOLD_OK;
}

int hold_composite(hold_ctx* ctx, int n, int R, int S, const hold_factors* factors, const int32_t* class_ids_host,
                   const hold_render_out* comp, const hold_render_out* per_node, void* stream) {
  HOLD_REQUIRE(ctx && factors && class_ids_host, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(n >= 1 && n <= HOLD_MAX_NODES, "n = %d out of [1,%d]", n, HOLD_MAX_NODES);
  HOLD_REQUIRE(R >= 0 && S >= 2, "bad R/S");
  if (R == 0) return HOLD_OK;
  cudaStream_t s = (cudaStream_t)stream;
  CompositeArgs a;
  memset(&a, 0, sizeof(a));
  a.R = R, a.S = S;
  for (int k = 0; k < n; ++k) {
    HOLD_REQUIRE(factors[k].color && factors[k].normal && factors[k].density && factors[k].z_vals, "factors[%d] incomplete", k);
    HOLD_REQUIRE(class_ids_host[k] >= 0 && class_ids_host[k] < 4, "class id out of range");
  }
  if (comp != nullptr) {
    a.n = n;
    for (int k = 0; k < n; ++k) {
      a.color[k] = factors[k].color, a.normal[k] = factors[k].normal, a.density[k] = factors[k].density, a.z[k] = factors[k].z_vals;
      a.class_id[k] = class_ids_host[k];
    }
    a.out = *comp, a.drop_head = n - 1, a.drop_tail = n, a.single_zmax_last = 0;
    k_composite<<<ceil_div(R, 128), 128, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (per_node != nullptr) {
    for (int k = 0; k < n; ++k) {
      CompositeArgs b;
      memset(&b, 0, sizeof(b));
      b.R = R, b.S = S, b.n = 1;
      b.color[0] = factors[k].color, b.normal[0] = factors[k].normal, b.density[0] = factors[k].density, b.z[0] = factors[k].z_vals;
      b.class_id[0] = class_ids_host[k];
      b.out = per_node[k], b.drop_head = 0, b.drop_tail = 0, b.single_zmax_last = 1;
      k_composite<<<ceil_div(R, 128), 128, 0, s>>>(b);
      HOLD_LAUNCH_CHECK(ctx);
    }
  }
  return HOLD_OK;
}

int hold_composite_bwd(hold_ctx* ctx, int n, int R, int S, const hold_factors* factors, const int32_t* class_ids_host,
                       const hold_render_out* g_comp, const hold_render_out* g_per_node, const hold_factors* d_factors, void* stream) {
  HOLD_REQUIRE(ctx && factors && class_ids_host && d_factors, "NULL argument");
  HOLD_REQUIRE(n >= 1 && n <= HOLD_MAX_NODES, "n = %d out of [1,%d]", n, HOLD_MAX_NODES);
  HOLD_REQUIRE(R >= 0 && S >= 2, "bad R/S");
  HOLD_REQUIRE(g_comp != nullptr || g_per_node != nullptr, "no upstream gradient given");
  if (R == 0) return HOLD_OK;
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  for (int k = 0; k < n; ++k) {
    HOLD_REQUIRE(factors[k].color && factors[k].normal && factors[k].density && factors[k].z_vals, "factors[%d] incomplete", k);
    HOLD_REQUIRE(d_factors[k].color && d_factors[k].normal && d_factors[k].density, "d_factors[%d] needs color, normal, density", k);
    HOLD_REQUIRE(class_ids_host[k] >= 0 && class_ids_host[k] < 4, "class id out of range");
  }
  bool written = false;
  if (g_comp != nullptr) {
    CompositeBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.n = n, a.R = R, a.S = S;
    for (int k = 0; k < n; ++k) {
      a.color[k] = factors[k].color, a.normal[k] = factors[k].normal, a.density[k] = factors[k].density, a.z[k] = factors[k].z_vals;
      a.class_id[k] = class_ids_host[k];
      a.d_color[k] = d_factors[k].color, a.d_normal[k] = d_factors[k].normal, a.d_density[k] = d_factors[k].density;
    }
    a.g = *g_comp, a.drop_head = n - 1, a.drop_tail = n, a.single_zmax_last = 0, a.accumulate = 0;
    k_composite_bwd<<<ceil_div(R, 128), 128, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
    written = true;
  }
  if (g_per_node != nullptr) {
    for (int k = 0; k < n; ++k) {
      CompositeBwdArgs b;
      memset(&b, 0, sizeof(b));
      b.n = 1, b.R = R, b.S = S;
      b.color[0] = factors[k].color, b.normal[0] = factors[k].normal, b.density[0] = factors[k].density, b.z[0] = factors[k].z_vals;
      b.class_id[0] = class_ids_host[k];
      b.d_color[0] = d_factors[k].color, b.d_normal[0] = d_factors[k].normal, b.d_density[0] = d_factors[k].density;
      b.g = g_per_node[k], b.drop_head = 0, b.drop_tail = 0, b.single_zmax_last = 1, b.accumulate = written ? 1 : 0;
      k_composite_bwd<<<ceil_div(R, 128), 128, 0, s>>>(b);
      HOLD_LAUNCH_CHECK(ctx);
    }
  }
  return HOLD_OK;
}

int hold_render_fg(hold_ctx* ctx, int n, const int32_t* node_ids_host, int R, int B, const float* cam_loc,
                   const float* ray_dirs, const hold_node_pose* poses, const hold_factors* factors,
                   const hold_render_out* comp, const hold_render_out* per_node, int32_t* iters, void* stream) {
  HOLD_REQUIRE(ctx && node_ids_host && poses && factors, "NULL argument");
  HOLD_REQUIRE(n >= 1 && n <= HOLD_MAX_NODES, "n = %d out of [1,%d]", n, HOLD_MAX_NODES);
  int32_t cls[HOLD_MAX_NODES];
  int S = -1;
  for (int k = 0; k < n; ++k) {
    int node = node_ids_host[k];
    int rc = check_node(ctx, node, true);
    if (rc) return rc;
    const hold_node_cfg& c = ctx->nodes[node].cfg;
    int Sk = c.n_samples + c.n_samples_extra + 2;
    HOLD_REQUIRE(S < 0 || S == Sk, "all nodes must produce the same number of samples per ray");
    S = Sk;
    cls[k] = c.class_id;
  }
  for (int k = 0; k < n; ++k) {
    int rc = hold_sample(ctx, node_ids_host[k], R, B, cam_loc, ray_dirs, &poses[k], nullptr, factors[k].z_vals,
                         iters ? iters + k : nullptr, stream);
    if (rc) return rc;
    rc = hold_shade(ctx, node_ids_host[k], R, B, S, cam_loc, ray_dirs, &poses[k], &factors[k], stream);
    if (rc) return rc;
  }
  return hold_composite(ctx, n, R, S, factors, cls, comp, per_node, stream);
}

int hold_mesh_sdf(hold_ctx* ctx, int B, int P, const float* points, int V, const float* verts, int verts_batched, int F,
                  const int32_t* faces, float* sdf, int32_t* face_idx, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(B >= 0 && P >= 0 && V > 0 && F > 0, "bad sizes");
  if (B == 0 || P == 0) return HOLD_OK;
  HOLD_REQUIRE(points && verts && faces && sdf, "NULL argument");
  dim3 grid(ceil_div(P, 128), B);
  k_mesh_sdf<<<grid, 128, 0, (cudaStream_t)stream>>>(P, V, F, verts_batched ? V * 3 : 0, points, verts, faces, sdf, face_idx);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_mesh_sdf_bvh(hold_ctx* ctx, int B, int P, const float* points, int V, const float* verts, int verts_batched, int F,
                      const int32_t* faces, float* sdf, int32_t* face_idx, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(B >= 0 && P >= 0 && V > 0 && F > 0, "bad sizes");
  HOLD_REQUIRE(F <= meshbvh::kMaxFaces, "F = %d faces is over 2^24", F);
  HOLD_REQUIRE(B <= 65535 && (int64_t)B * P < (1ll << 31), "bad sizes B %d P %d", B, P);
  if (B == 0 || P == 0) return HOLD_OK;
  HOLD_REQUIRE(points && verts && faces && sdf, "NULL argument");
  cudaStream_t s = (cudaStream_t)stream;
  const int trees = verts_batched ? B : 1;
  // one workspace, sized from the arguments
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_st = take(2 * sizeof(int)), o_bd = take((size_t)trees * 8 * sizeof(float));
  const size_t o_codes = take((size_t)trees * F * sizeof(int)), o_order = take((size_t)trees * F * sizeof(int));
  const size_t o_nodes = take((size_t)trees * 2 * F * 4 * sizeof(float4)), o_child = take((size_t)trees * F * sizeof(int2));
  const size_t o_par = take((size_t)trees * 2 * F * sizeof(int)), o_vis = take((size_t)trees * F * sizeof(int));
  const size_t o_sort = take(3 * (size_t)F * sizeof(int)), o_hist = take(radix_sort_hist_ints(F) * sizeof(int));
  const size_t o_band = take((size_t)B * P * sizeof(int));
  WS(WS_MESH_BVH, uint8_t, off, ws);
  BvhArgs a{};
  a.B = B, a.P = P, a.V = V, a.F = F, a.vstride = verts_batched ? V * 3 : 0, a.tstride = verts_batched ? 1 : 0;
  a.points = points, a.verts = verts, a.faces = faces, a.sdf = sdf, a.face_idx = face_idx;
  a.state = (int*)(ws + o_st), a.bounds = (float*)(ws + o_bd), a.codes = (int*)(ws + o_codes), a.order = (int*)(ws + o_order);
  a.nodes = (float4*)(ws + o_nodes), a.child = (int2*)(ws + o_child), a.parent = (int*)(ws + o_par), a.visits = (int*)(ws + o_vis);
  a.band = (int*)(ws + o_band), a.err = ctx->dev_err;
  HOLD_CUDA(cudaMemsetAsync(a.state, 0, 2 * sizeof(int), s));
  HOLD_CUDA(cudaMemsetAsync(a.visits, 0, (size_t)trees * F * sizeof(int), s));
  k_bvh_bounds<<<trees, 1024, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_bvh_codes<<<dim3(ceil_div(F, 256), trees), 256, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  int* sb = (int*)(ws + o_sort);
  for (int t = 0; t < trees; ++t) {
    // 30 code bits: four passes, so the sorted faces land in vb[1], the tree's own order
    int* const kb[2] = {sb, sb + F};
    int* const vb[2] = {sb + 2 * (size_t)F, a.order + (size_t)t * F};
    const int *kout, *vout;
    int rc = radix_sort(ctx, a.codes + (size_t)t * F, F, 30, kb, vb, (int*)(ws + o_hist), &kout, &vout, s);
    if (rc) return rc;
    BvhArgs lt = a;
    lt.sorted_codes = kout, lt.child = a.child + (size_t)t * F, lt.parent = a.parent + (size_t)t * 2 * F;
    k_bvh_link<<<ceil_div(max(F - 1, 1), 256), 256, 0, s>>>(lt);
    HOLD_LAUNCH_CHECK(ctx);
  }
  k_bvh_refit<<<dim3(ceil_div(F, 256), trees), 256, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_bvh_query<<<dim3(ceil_div(P, kBvhThreads), B), kBvhThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_bvh_band<<<ceil_div(B * P, kBvhThreads), kBvhThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_off_in_surface(hold_ctx* ctx, int R, int S, const float* sdf, float threshold, uint8_t* off_surface,
                        uint8_t* in_surface, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(R >= 0 && S >= 1, "bad sizes");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(sdf != nullptr, "NULL argument");
  k_off_in_surface<<<ceil_div(R, 128), 128, 0, (cudaStream_t)stream>>>(R, S, sdf, threshold, off_surface, in_surface);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

// Shared by the rasteriser's forward and backward: validates the arguments and writes the face records (k_raster_setup).
static int raster_setup(hold_ctx* ctx, int B, int V, const float* verts_ndc, int F, const int32_t* faces, int H, int W,
                        const hold_raster_cfg* cfg, RasterArgs* a, void* stream) {
  HOLD_REQUIRE(ctx && verts_ndc && faces && cfg, "NULL argument");
  HOLD_REQUIRE(B >= 0 && B <= 65535 && V > 0 && F > 0 && H > 0 && W > 0 && (int64_t)ceil_div(H, kRasterTile) * ceil_div(W, kRasterTile) < (1ll << 31),
               "bad sizes B %d V %d F %d H %d W %d", B, V, F, H, W);
  HOLD_REQUIRE(cfg->faces_per_pixel >= 1 && cfg->faces_per_pixel <= HOLD_RASTER_MAX_K, "faces_per_pixel %d outside [1, %d]",
               cfg->faces_per_pixel, (int)HOLD_RASTER_MAX_K);
  HOLD_REQUIRE(cfg->sigma > 0.f && isfinite(cfg->sigma) && cfg->blur_radius >= 0.f && isfinite(cfg->blur_radius),
               "sigma %g must be > 0 and blur_radius %g >= 0", cfg->sigma, cfg->blur_radius);
  HOLD_CUDA(cudaSetDevice(ctx->device));
  *a = RasterArgs{};
  a->V = V, a->F = F, a->H = H, a->W = W, a->K = cfg->faces_per_pixel;
  while ((1ll << a->fbits) < F) ++a->fbits;
  a->o = raster::Opts{cfg->blur_radius, cfg->sigma, cfg->perspective_correct != 0, cfg->clip_barycentric_coords != 0,
                      cfg->cull_backfaces != 0};
  if (B == 0) return HOLD_OK;
  WS(WS_RASTER, float4, (size_t)B * F * 4, rec);
  k_raster_setup<<<dim3(ceil_div(F, 128), B), 128, 0, (cudaStream_t)stream>>>(V, F, verts_ndc, faces, a->o, rec, ctx->dev_err);
  HOLD_LAUNCH_CHECK(ctx);
  a->rec = rec;
  return HOLD_OK;
}

int hold_raster_silhouette(hold_ctx* ctx, int B, int V, const float* verts_ndc, int F, const int32_t* faces, int H, int W,
                           const hold_raster_cfg* cfg, float* sil, int64_t* pix_to_face, float* zbuf, float* dists, void* stream) {
  HOLD_REQUIRE(sil != nullptr, "NULL argument");
  const int nfrag = (pix_to_face != nullptr) + (zbuf != nullptr) + (dists != nullptr);
  HOLD_REQUIRE(nfrag == 0 || nfrag == 3, "pix_to_face, zbuf and dists are given together or not at all");
  RasterArgs a;
  int rc = raster_setup(ctx, B, V, verts_ndc, F, faces, H, W, cfg, &a, stream);
  if (rc || B == 0) return rc;
  a.sil = sil, a.p2f = pix_to_face, a.zbuf = zbuf, a.dists = dists;
  k_raster<false><<<dim3(ceil_div(H, kRasterTile) * ceil_div(W, kRasterTile), B), kRasterThreads, 0, (cudaStream_t)stream>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_raster_silhouette_bwd(hold_ctx* ctx, int B, int V, const float* verts_ndc, int F, const int32_t* faces, int H, int W,
                               const hold_raster_cfg* cfg, const float* g_sil, float* g_verts, void* stream) {
  HOLD_REQUIRE(g_sil != nullptr && g_verts != nullptr, "NULL argument");
  RasterArgs a;
  int rc = raster_setup(ctx, B, V, verts_ndc, F, faces, H, W, cfg, &a, stream);
  if (rc || B == 0) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  // one workspace, sized from the arguments: Q and thresholds per pixel, the faces' partials, the vertex map
  const size_t npix = (size_t)B * H * W, o_q = npix * sizeof(uint64_t), o_part = (o_q + npix * sizeof(float) + 255) & ~(size_t)255;
  const size_t o_keys = (o_part + (size_t)B * F * kRbPieces * 6 * sizeof(float) + 255) & ~(size_t)255;
  const size_t o_map = o_keys + (((size_t)F * 3 * sizeof(int) + 255) & ~(size_t)255);
  WS(WS_RASTER_BWD, uint8_t, o_map + inverse_map_ints(F * 3, V) * sizeof(int), ws);
  a.thr = (uint64_t*)ws, a.q = (float*)(ws + o_q);
  k_raster<true><<<dim3(ceil_div(H, kRasterTile) * ceil_div(W, kRasterTile), B), kRasterThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  RasterBwdArgs g;
  g.V = V, g.F = F, g.H = H, g.W = W, g.fbits = a.fbits, g.o = a.o;
  g.rec = a.rec, g.q = a.q, g.thr = a.thr, g.g_sil = g_sil, g.part = (float*)(ws + o_part), g.g_verts = g_verts;
  int* keys = (int*)(ws + o_keys);
  k_raster_vert_keys<<<ceil_div(F * 3, 256), 256, 0, s>>>(F * 3, V, faces, keys);
  HOLD_LAUNCH_CHECK(ctx);
  if ((rc = inverse_map(ctx, keys, F * 3, V, (int*)(ws + o_map), &g.vmap, s))) return rc;
  k_raster_bwd_faces<<<dim3(F * (kRbPieces / kRbWarps), B), kRbWarps * 32, 0, s>>>(g);
  HOLD_LAUNCH_CHECK(ctx);
  k_raster_bwd_verts<<<dim3(ceil_div(V, 128), B), 128, 0, s>>>(g);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_knn_points(hold_ctx* ctx, int N, int P1, const float* p1, const int32_t* lengths1, int P2, const float* p2,
                    const int32_t* lengths2, int K, float* dists, int32_t* idx, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(N >= 0 && P1 >= 0 && P2 >= 0, "bad sizes N %d P1 %d P2 %d", N, P1, P2);
  HOLD_REQUIRE(K >= 1 && K <= HOLD_KNN_MAX_K, "K %d outside [1, %d]", K, (int)HOLD_KNN_MAX_K);
  if (N == 0 || P1 == 0) return HOLD_OK;
  HOLD_REQUIRE(p1 && dists && idx && (P2 == 0 || p2), "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  const dim3 grid(ceil_div(P1, kPcThreads), min(N, 65535));
  cudaStream_t s = (cudaStream_t)stream;
#define HOLD_KNN_CASE(KT)                                                                                                    \
  k_knn<KT><<<grid, kPcThreads, 0, s>>>(N, P1, p1, lengths1, P2, p2, lengths2, K, dists, idx, ctx->dev_err)
  if (K == 1) HOLD_KNN_CASE(1);
  else if (K <= 2) HOLD_KNN_CASE(2);
  else if (K <= 4) HOLD_KNN_CASE(4);
  else if (K <= 8) HOLD_KNN_CASE(8);
  else if (K <= 16) HOLD_KNN_CASE(16);
  else HOLD_KNN_CASE(32);
#undef HOLD_KNN_CASE
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_knn_points_bwd(hold_ctx* ctx, int N, int P1, const float* p1, const int32_t* lengths1, int P2, const float* p2,
                        const int32_t* lengths2, int K, const int32_t* idx, const float* g_dists, const float* g_knn, float* g_p1,
                        float* g_p2, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(N >= 0 && P1 >= 0 && P2 >= 0, "bad sizes N %d P1 %d P2 %d", N, P1, P2);
  HOLD_REQUIRE(K >= 1 && K <= HOLD_KNN_MAX_K, "K %d outside [1, %d]", K, (int)HOLD_KNN_MAX_K);
  HOLD_REQUIRE((int64_t)N * P1 * K < (1ll << 31) && (int64_t)N * P2 < (1ll << 31), "N P1 K = %lld or N P2 = %lld slots is over 2^31",
               (long long)N * P1 * K, (long long)N * P2);
  if (N == 0) return HOLD_OK;
  HOLD_REQUIRE((P1 == 0 || (p1 && idx && g_dists && g_p1)) && (P2 == 0 || (p2 && g_p2)), "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  const int S = N * P1 * K, T = N * P2;
  KnnBwdArgs a{};
  a.N = N, a.P1 = P1, a.P2 = P2, a.K = K, a.p1 = p1, a.p2 = p2, a.len1 = lengths1, a.len2 = lengths2, a.idx = idx;
  a.g_dists = g_dists, a.g_knn = g_knn, a.g_p1 = g_p1, a.g_p2 = g_p2, a.err = ctx->dev_err;
  // one workspace, sized from the arguments: the slots' p2 parts, their keys, the inverse map
  const size_t o_keys = ((size_t)S * 3 * sizeof(float) + 255) & ~(size_t)255;
  const size_t o_map = o_keys + (((size_t)S * sizeof(int) + 255) & ~(size_t)255);
  WS(WS_KNN_BWD, uint8_t, o_map + inverse_map_ints(S, T) * sizeof(int), ws);
  a.contrib = (float*)ws, a.keys = (int*)(ws + o_keys);
  cudaStream_t s = (cudaStream_t)stream;
  if (S > 0) {
    k_knn_bwd_rows<<<ceil_div(N * P1, kPcThreads), kPcThreads, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (T == 0) return HOLD_OK;
  int rc = inverse_map(ctx, a.keys, S, T, (int*)(ws + o_map), &a.map, s);
  if (rc) return rc;
  k_knn_bwd_targets<<<ceil_div(T, kPcThreads), kPcThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_icp(hold_ctx* ctx, int N, int Ps, const float* source, const int32_t* src_lengths, int Pt, const float* target,
             const int32_t* tgt_lengths, const double* init, const hold_icp_cfg* cfg, double* transformation, double* fitness,
             double* inlier_rmse, int32_t* iterations, void* stream) {
  HOLD_REQUIRE(ctx != nullptr && cfg != nullptr, "NULL argument");
  HOLD_REQUIRE(N >= 0 && N <= 65535 && Ps >= 0 && Pt >= 0, "bad sizes N %d Ps %d Pt %d", N, Ps, Pt);
  HOLD_REQUIRE(cfg->max_iteration >= 0, "max_iteration %d < 0", cfg->max_iteration);
  HOLD_REQUIRE(!isnan(cfg->max_correspondence_distance) && !isnan(cfg->relative_fitness) && !isnan(cfg->relative_rmse),
               "NaN in hold_icp_cfg");
  if (N == 0) return HOLD_OK;
  HOLD_REQUIRE(transformation && fitness && inlier_rmse && iterations && (Ps == 0 || source) && (Pt == 0 || target),
               "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  IcpArgs a{};
  a.N = N, a.Ps = Ps, a.Pt = Pt, a.nb = max(1, ceil_div(Ps, kPcThreads));
  a.src = source, a.src_len = src_lengths, a.tgt = target, a.tgt_len = tgt_lengths, a.init = init;
  const double md = cfg->max_correspondence_distance;
  a.max_d2 = md > 0.0 ? md * md : -1.0;   // open3d: no correspondence unless max_correspondence_distance > 0
  a.rel_fitness = cfg->relative_fitness, a.rel_rmse = cfg->relative_rmse, a.with_scaling = cfg->with_scaling;
  a.err = ctx->dev_err;
  // one workspace: pair states, transformed source, per-CTA partials, correspondences
  const size_t b_st = (sizeof(IcpPair) * (size_t)N + 255) & ~(size_t)255;
  const size_t b_xs = (size_t)N * Ps * 3 * sizeof(double), b_part = (size_t)N * a.nb * kIcpPart * sizeof(double);
  const size_t o_xs = b_st, o_part = o_xs + ((b_xs + 255) & ~(size_t)255), o_corr = o_part + ((b_part + 255) & ~(size_t)255);
  WS(WS_ICP, uint8_t, o_corr + (size_t)N * Ps * sizeof(int) + 256, ws);
  a.st = (IcpPair*)ws, a.xs = (double*)(ws + o_xs), a.part = (double*)(ws + o_part), a.corr = (int*)(ws + o_corr);
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(a.nb, N);
  const int pair_blocks = ceil_div(N, 128);
  k_icp_start<<<grid, kPcThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_icp_corr<false><<<grid, kPcThreads, 0, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_icp_eval<<<pair_blocks, 128, 0, s>>>(a, -1);
  HOLD_LAUNCH_CHECK(ctx);
  for (int it = 0; it < cfg->max_iteration; ++it) {
    k_icp_cov<<<grid, kPcThreads, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
    k_icp_update<<<pair_blocks, 128, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
    k_icp_corr<true><<<grid, kPcThreads, 0, s>>>(a);
    HOLD_LAUNCH_CHECK(ctx);
    k_icp_eval<<<pair_blocks, 128, 0, s>>>(a, it);
    HOLD_LAUNCH_CHECK(ctx);
  }
  k_icp_out<<<pair_blocks, 128, 0, s>>>(a, transformation, fitness, inlier_rmse, iterations);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_decimate(hold_ctx* ctx, int V, const float* verts, int F, const int32_t* faces, int target_faces, float quality_threshold,
                  float* verts_out, int32_t* faces_out, int* V_out_host, int* F_out_host, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(V >= 0 && F >= 0 && target_faces >= 0, "bad sizes V %d F %d target_faces %d", V, F, target_faces);
  HOLD_REQUIRE((int64_t)F * 3 < (1ll << 31), "3 F = %lld half-edges is not below 2^31", (long long)F * 3);
  HOLD_REQUIRE(!isnan(quality_threshold), "quality_threshold is NaN");
  HOLD_REQUIRE(V_out_host && F_out_host && (V == 0 || (verts && verts_out)) && (F == 0 || (faces && faces_out)), "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int n3 = 3 * F;
  // one workspace, sized from the arguments
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_st = take(sizeof(DecState)), o_hist = take(256 * sizeof(int)), o_P = take((size_t)V * 3 * sizeof(float));
  const size_t o_Q = take((size_t)V * 10 * sizeof(double)), o_F = take((size_t)n3 * sizeof(int)), o_fz = take((size_t)V * sizeof(int));
  const size_t o_key = take((size_t)n3 * sizeof(uint64_t)), o_sel = take((size_t)n3 * sizeof(uint64_t));
  const size_t o_mA = take((size_t)V * sizeof(uint64_t)), o_mB = take((size_t)V * sizeof(uint64_t));
  const size_t o_X = take((size_t)n3 * 3 * sizeof(float)), o_sk = take((size_t)n3 * sizeof(int));
  const size_t o_vn = take((size_t)(V + 1) * sizeof(int)), o_fn = take((size_t)(F + 1) * sizeof(int));
  const size_t o_im = take(inverse_map_ints(n3, V) * sizeof(int));
  WS(WS_DECIMATE, uint8_t, off, ws);
  DecState* st = (DecState*)(ws + o_st);
  int* hist = (int*)(ws + o_hist);
  float* P = (float*)(ws + o_P);
  double* Q = (double*)(ws + o_Q);
  int *Fw = (int*)(ws + o_F), *frozen = (int*)(ws + o_fz), *skeys = (int*)(ws + o_sk), *vnew = (int*)(ws + o_vn), *fnew = (int*)(ws + o_fn);
  uint64_t *key = (uint64_t*)(ws + o_key), *sel = (uint64_t*)(ws + o_sel), *mA = (uint64_t*)(ws + o_mA), *mB = (uint64_t*)(ws + o_mB);
  float* X = (float*)(ws + o_X);
  const int gF3 = ceil_div(max(n3, 1), kDecThreads), gV = ceil_div(max(V, 1), kDecThreads);
  const int gSel = min(gF3, 4 * ctx->sm_count);
  DecState h{};
  auto read_state = [&]() -> int {
    HOLD_CUDA(cudaMemcpyAsync(&h, st, sizeof(DecState), cudaMemcpyDeviceToHost, s));
    HOLD_CUDA(cudaStreamSynchronize(s));
    return HOLD_OK;
  };
  k_dec_state<<<1, 1, 0, s>>>(st, F, target_faces);
  HOLD_LAUNCH_CHECK(ctx);
  if (F > 0) {
    k_dec_init<<<gF3, kDecThreads, 0, s>>>(n3, V, faces, Fw, st, ctx->dev_err);
    HOLD_LAUNCH_CHECK(ctx);
  }
  int rc = read_state();
  if (rc) return rc;
  if (h.bad || target_faces >= F) {
    if (V) HOLD_CUDA(cudaMemcpyAsync(verts_out, verts, (size_t)V * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (F) HOLD_CUDA(cudaMemcpyAsync(faces_out, faces, (size_t)n3 * sizeof(int), cudaMemcpyDeviceToDevice, s));
    *V_out_host = V, *F_out_host = F;
    return HOLD_OK;
  }
  HOLD_CUDA(cudaMemcpyAsync(P, verts, (size_t)V * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  HOLD_CUDA(cudaMemsetAsync(hist, 0, 256 * sizeof(int), s));
  auto select = [&](const uint64_t* keys, int which) -> int {
    for (int pass = 0; pass < 8; ++pass) {
      k_dec_sel_hist<<<gSel, kDecThreads, 0, s>>>(n3, keys, st, which, pass, hist);
      HOLD_LAUNCH_CHECK(ctx);
      k_dec_sel_pick<<<1, 1, 0, s>>>(st, which, pass, hist);
      HOLD_LAUNCH_CHECK(ctx);
    }
    return HOLD_OK;
  };
  InvMap m;
  for (int round = 0; round < kDecMaxRounds && h.F_live > target_faces; ++round) {
    k_dec_star_keys<<<gF3, kDecThreads, 0, s>>>(n3, V, Fw, skeys);
    HOLD_LAUNCH_CHECK(ctx);
    if ((rc = inverse_map(ctx, skeys, n3, V, (int*)(ws + o_im), &m, s))) return rc;
    if (round == 0) {
      k_dec_quadrics<<<gV, kDecThreads, 0, s>>>(V, Fw, P, m, Q);
      HOLD_LAUNCH_CHECK(ctx);
    }
    k_dec_frozen<<<gV, kDecThreads, 0, s>>>(V, Fw, m, frozen);
    HOLD_LAUNCH_CHECK(ctx);
    k_dec_edges<<<gF3, kDecThreads, 0, s>>>(n3, Fw, P, Q, m, frozen, (double)quality_threshold, key, X);
    HOLD_LAUNCH_CHECK(ctx);
    if ((rc = select(key, 0))) return rc;
    k_dec_vmin<<<gV, kDecThreads, 0, s>>>(V, Fw, m, key, st, mA);
    HOLD_LAUNCH_CHECK(ctx);
    k_dec_ring<<<gV, kDecThreads, 0, s>>>(V, Fw, m, mA, mB);
    HOLD_LAUNCH_CHECK(ctx);
    k_dec_ring<<<gV, kDecThreads, 0, s>>>(V, Fw, m, mB, mA);
    HOLD_LAUNCH_CHECK(ctx);
    k_dec_select<<<gF3, kDecThreads, 0, s>>>(n3, Fw, key, st, mA, sel);
    HOLD_LAUNCH_CHECK(ctx);
    if ((rc = select(sel, 1))) return rc;
    k_dec_apply<<<gF3, kDecThreads, 0, s>>>(n3, sel, st, Fw, P, Q, m, X);
    HOLD_LAUNCH_CHECK(ctx);
    if ((rc = read_state())) return rc;
    if (h.collapses == 0) break;
  }
  // compaction: surviving vertices and faces in ascending input order
  HOLD_CUDA(cudaMemsetAsync(vnew, 0, (size_t)(V + 1) * sizeof(int), s));
  HOLD_CUDA(cudaMemsetAsync(fnew + F, 0, sizeof(int), s));
  k_dec_flags<<<gF3, kDecThreads, 0, s>>>(F, Fw, vnew, fnew);
  HOLD_LAUNCH_CHECK(ctx);
  k_im_scan<<<1, 1024, 0, s>>>(vnew, V + 1);
  HOLD_LAUNCH_CHECK(ctx);
  k_im_scan<<<1, 1024, 0, s>>>(fnew, F + 1);
  HOLD_LAUNCH_CHECK(ctx);
  k_dec_out_verts<<<gV, kDecThreads, 0, s>>>(V, vnew, P, verts_out);
  HOLD_LAUNCH_CHECK(ctx);
  k_dec_out_faces<<<gF3, kDecThreads, 0, s>>>(F, fnew, vnew, Fw, faces_out);
  HOLD_LAUNCH_CHECK(ctx);
  HOLD_CUDA(cudaMemcpyAsync(V_out_host, vnew + V, sizeof(int), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaMemcpyAsync(F_out_host, fnew + F, sizeof(int), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaStreamSynchronize(s));
  return HOLD_OK;
}

int hold_largest_component(hold_ctx* ctx, int V, const float* verts, int F, const int32_t* faces, float* verts_out,
                           int32_t* faces_out, int* V_out_host, int* F_out_host, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(V >= 0 && F >= 0, "bad sizes V %d F %d", V, F);
  HOLD_REQUIRE((int64_t)F * 3 < (1ll << 31), "3 F = %lld corners is not below 2^31", (long long)F * 3);
  HOLD_REQUIRE(V_out_host && F_out_host && (V == 0 || (verts && verts_out)) && (F == 0 || (faces && faces_out)), "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  *V_out_host = 0, *F_out_host = 0;
  if (F == 0) return HOLD_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int n3 = 3 * F;
  // one workspace, sized from the arguments
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_st = take(sizeof(CcState)), o_par = take((size_t)V * sizeof(int)), o_lab = take((size_t)V * sizeof(int));
  const size_t o_area = take((size_t)F * sizeof(float));
  const size_t o_key = take((size_t)F * sizeof(int)), o_sum = take((size_t)V * sizeof(double));
  const size_t o_vn = take((size_t)(V + 1) * sizeof(int)), o_fn = take((size_t)(F + 1) * sizeof(int));
  const size_t o_im = take(inverse_map_ints(F, V) * sizeof(int));
  WS(WS_MESH_CC, uint8_t, off, ws);
  CcState* st = (CcState*)(ws + o_st);
  int *parent = (int*)(ws + o_par), *label = (int*)(ws + o_lab), *key = (int*)(ws + o_key), *vnew = (int*)(ws + o_vn), *fnew = (int*)(ws + o_fn);
  float* area = (float*)(ws + o_area);
  double* sums = (double*)(ws + o_sum);
  const int gF = ceil_div(F, kCcThreads), gV = ceil_div(max(V, 1), kCcThreads);
  HOLD_CUDA(cudaMemsetAsync(st, 0, sizeof(CcState), s));
  k_cc_init<<<ceil_div(max(V, n3), kCcThreads), kCcThreads, 0, s>>>(V, n3, faces, parent, st, ctx->dev_err);
  HOLD_LAUNCH_CHECK(ctx);
  k_cc_unite<<<gF, kCcThreads, 0, s>>>(F, faces, parent, st);
  HOLD_LAUNCH_CHECK(ctx);
  if (V > 0) {
    k_cc_labels<<<gV, kCcThreads, 0, s>>>(V, parent, st, label);
    HOLD_LAUNCH_CHECK(ctx);
  }
  k_cc_area<<<gF, kCcThreads, 0, s>>>(F, V, verts, faces, label, st, area, key);
  HOLD_LAUNCH_CHECK(ctx);
  InvMap m;
  int rc = inverse_map(ctx, key, F, V, (int*)(ws + o_im), &m, s);
  if (rc) return rc;
  if (V > 0) {
    k_cc_sums<<<gV, kCcThreads, 0, s>>>(V, area, m, sums);
    HOLD_LAUNCH_CHECK(ctx);
    k_cc_argmax<<<1, kCcArgmaxThreads, 0, s>>>(V, sums, st);
    HOLD_LAUNCH_CHECK(ctx);
  } else {
    HOLD_CUDA(cudaMemsetAsync(&st->best, 0xff, sizeof(int), s));   // every face is out of range: -1, nothing kept
  }
  // compaction: kept vertices in ascending old id, kept faces in input order
  HOLD_CUDA(cudaMemsetAsync(vnew, 0, (size_t)(V + 1) * sizeof(int), s));
  HOLD_CUDA(cudaMemsetAsync(fnew + F, 0, sizeof(int), s));
  k_cc_flags<<<gF, kCcThreads, 0, s>>>(F, faces, label, st, vnew, fnew);
  HOLD_LAUNCH_CHECK(ctx);
  k_im_scan<<<1, 1024, 0, s>>>(vnew, V + 1);
  HOLD_LAUNCH_CHECK(ctx);
  k_im_scan<<<1, 1024, 0, s>>>(fnew, F + 1);
  HOLD_LAUNCH_CHECK(ctx);
  if (V > 0) {
    k_cc_out_verts<<<gV, kCcThreads, 0, s>>>(V, vnew, verts, verts_out);
    HOLD_LAUNCH_CHECK(ctx);
  }
  k_cc_out_faces<<<gF, kCcThreads, 0, s>>>(F, fnew, vnew, faces, faces_out);
  HOLD_LAUNCH_CHECK(ctx);
  // the one host read: the two output sizes
  int sizes[2];
  HOLD_CUDA(cudaMemcpyAsync(&sizes[0], vnew + V, sizeof(int), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaMemcpyAsync(&sizes[1], fnew + F, sizeof(int), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaStreamSynchronize(s));
  *V_out_host = sizes[0], *F_out_host = sizes[1];
  return HOLD_OK;
}

int hold_inverse_warp_bwd(hold_ctx* ctx, int node, int B, int P, const float* x, const hold_node_pose* pose, const int32_t* knn_idx,
                          const float* g_xc, float* g_tfs, float* g_x, void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  HOLD_REQUIRE(B >= 0 && P >= 0, "bad sizes");
  if (B == 0) return HOLD_OK;
  HOLD_REQUIRE(pose && pose->tfs && g_tfs && (P == 0 || (x && g_xc)), "NULL argument");
  NodeState& ns = ctx->nodes[node];
  const bool hand = ns.cfg.kind == HOLD_KIND_HAND;
  cudaStream_t s = (cudaStream_t)stream;
  const int nb = max(1, ceil_div(P, 128));
  void* part = nullptr;
  if ((rc = ws_get(ctx, WS_WARPBWD,(size_t)B * nb * warpbwd::kJ * warpbwd::kG * sizeof(float), &part))) return rc;
  dim3 grid(nb, B);
  if (hand) {
    if (!ns.has_rig) { set_error("hand node has no rig (hold_node_set_rig)"); return HOLD_E_STATE; }
    HOLD_REQUIRE(P == 0 || (knn_idx && pose->posed_verts), "hand backward needs the forward's knn_idx and the posed vertices");
    k_inverse_warp_bwd_hand<<<grid, 128, 0, s>>>(P, x, knn_idx, pose->posed_verts, ns.skin_w, pose->tfs, g_xc, g_x, (float*)part);
    HOLD_LAUNCH_CHECK(ctx);
    k_inverse_warp_bwd_hand_final<<<B, 256, 0, s>>>(nb, (const float*)part, g_tfs);
  } else {
    k_inverse_warp_bwd_obj<<<grid, 128, 0, s>>>(P, x, pose->tfs, g_xc, g_x, (float*)part);
    HOLD_LAUNCH_CHECK(ctx);
    k_inverse_warp_bwd_obj_final<<<B, 16, 0, s>>>(nb, (const float*)part, g_tfs);
  }
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_mise_destroy(hold_mise* h) {
  if (!h) return HOLD_OK;
  cudaFree(h->g.val), cudaFree(h->g.state), cudaFree(h->queue), cudaFree(h->counter);
  for (int L = 0; L < mise::kMaxDepth; ++L) { cudaFree(h->g.sub[L]); cudaFree(h->g.mark[L]); }
  delete h;
  return HOLD_OK;
}

int hold_mise_create(hold_ctx* ctx, int resolution_0, int depth, float threshold, hold_mise** out, void* stream) {
  HOLD_REQUIRE(ctx && out, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(resolution_0 >= 1 && depth >= 0 && depth <= mise::kMaxDepth, "bad MISE shape");
  HOLD_REQUIRE(((long long)resolution_0 << depth) <= 1024, "MISE resolution above 1024 is not supported");
  hold_mise* h = new (std::nothrow) hold_mise();
  HOLD_REQUIRE(h != nullptr, "out of host memory");
  h->ctx = ctx;
  mise::Grid& g = h->g;
  memset(&g, 0, sizeof(g));
  g.res0 = resolution_0, g.depth = depth, g.R = resolution_0 << depth, g.G = g.R + 1, g.threshold = threshold;
  h->np = (size_t)g.G * g.G * g.G;
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMalloc((void**)&g.val, h->np * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc((void**)&g.state, h->np);
  if (e == cudaSuccess) e = cudaMalloc((void**)&h->queue, h->np * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc((void**)&h->counter, sizeof(unsigned int));
  for (int L = 0; L < depth && e == cudaSuccess; ++L) {
    const size_t n = (size_t)(resolution_0 << L) * (resolution_0 << L) * (resolution_0 << L);
    e = cudaMalloc((void**)&g.sub[L], n);
    if (e == cudaSuccess) e = cudaMalloc((void**)&g.mark[L], n * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMemsetAsync(g.sub[L], 0, n, s);
  }
  if (e == cudaSuccess) e = cudaMemsetAsync(g.val, 0, h->np * sizeof(float), s);
  if (e == cudaSuccess) e = cudaMemsetAsync(g.state, 0, h->np, s);
  if (e != cudaSuccess) {
    set_error("hold_mise_create: %s", cudaGetErrorString(e));
    hold_mise_destroy(h);
    return HOLD_E_CUDA;
  }
  const int n0 = (resolution_0 + 1) * (resolution_0 + 1) * (resolution_0 + 1);
  k_mise_init<<<ceil_div(n0, 256), 256, 0, s>>>(g);
  HOLD_LAUNCH_CHECK(ctx);
  *out = h;
  return HOLD_OK;
}

int hold_mise_query(hold_mise* h, int32_t* coords, int capacity, int* n_points, void* stream) {
  HOLD_REQUIRE(h && n_points, "NULL argument");
  HOLD_CUDA(cudaSetDevice(h->ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  HOLD_CUDA(cudaMemsetAsync(h->counter, 0, sizeof(unsigned int), s));
  k_mise_collect<<<h->ctx->sm_count * 8, 256, 0, s>>>(h->g, h->queue, h->counter, (unsigned int)h->np);
  HOLD_LAUNCH_CHECK(h->ctx);
  unsigned int n = 0;
  HOLD_CUDA(cudaMemcpyAsync(&n, h->counter, sizeof(n), cudaMemcpyDeviceToHost, s));
  HOLD_CUDA(cudaStreamSynchronize(s));   // the caller sizes its SDF query by n: one host sync per MISE round, as in the reference loop
  h->n_last = (int)n;
  *n_points = (int)n;
  if (n == 0 || coords == nullptr) return HOLD_OK;
  HOLD_REQUIRE(capacity >= (int)n, "coords buffer holds %d points, %u needed", capacity, n);
  k_mise_coords<<<ceil_div((int)n, 256), 256, 0, s>>>(h->g, h->queue, (int)n, coords);
  HOLD_LAUNCH_CHECK(h->ctx);
  return HOLD_OK;
}

int hold_mise_update(hold_mise* h, const float* values, int n_values, void* stream) {
  HOLD_REQUIRE(h && (values || n_values == 0), "NULL argument");
  HOLD_CUDA(cudaSetDevice(h->ctx->device));
  HOLD_REQUIRE(n_values == h->n_last, "update with %d values after a query of %d points", n_values, h->n_last);
  cudaStream_t s = (cudaStream_t)stream;
  if (n_values > 0) {
    k_mise_scatter<<<ceil_div(n_values, 256), 256, 0, s>>>(h->g, h->queue, n_values, values);
    HOLD_LAUNCH_CHECK(h->ctx);
  }
  h->n_last = 0;
  const mise::Grid& g = h->g;
  for (int L = 0; L < g.depth; ++L) {
    const size_t n = (size_t)(g.res0 << L) * (g.res0 << L) * (g.res0 << L);
    HOLD_CUDA(cudaMemsetAsync(g.mark[L], 0, n * sizeof(unsigned int), s));
  }
  if (g.depth == 0) return HOLD_OK;
  k_mise_mark<<<h->ctx->sm_count * 8, 256, 0, s>>>(g);
  HOLD_LAUNCH_CHECK(h->ctx);
  for (int L = 0; L < g.depth; ++L) {
    k_mise_subdivide<<<h->ctx->sm_count * 4, 256, 0, s>>>(g, L);
    HOLD_LAUNCH_CHECK(h->ctx);
  }
  return HOLD_OK;
}

int hold_mise_to_dense(hold_mise* h, float* out, void* stream) {
  HOLD_REQUIRE(h && out, "NULL argument");
  HOLD_CUDA(cudaSetDevice(h->ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  k_mise_dense_init<<<h->ctx->sm_count * 8, 256, 0, s>>>(h->g, out);
  HOLD_LAUNCH_CHECK(h->ctx);
  for (int axis = 0; axis < 3; ++axis) {
    k_mise_fill<<<ceil_div(h->g.G * h->g.G, 128), 128, 0, s>>>(h->g, out, axis);
    HOLD_LAUNCH_CHECK(h->ctx);
  }
  return HOLD_OK;
}

/* ---- marching cubes on a dense value grid (SURVEY §8f rank 4: the last step of generate_mesh, utils/meshing.py:51) ---- */
int hold_mc_mark(hold_ctx* ctx, int n0, int n1, int n2, const float* vol, float level, int32_t* edge_flags, int32_t* cell_ntri, void* stream) {
  HOLD_REQUIRE(ctx && vol && edge_flags && cell_ntri, "NULL argument");
  HOLD_REQUIRE(n0 >= 2 && n1 >= 2 && n2 >= 2, "grid must be at least 2 x 2 x 2");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  mc::Dims d{n0, n1, n2};
  const int64_t total = (int64_t)n0 * n1 * n2;
  k_mc_mark<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d, vol, level, edge_flags, cell_ntri);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_mc_emit(hold_ctx* ctx, int n0, int n1, int n2, const float* vol, float level, const int32_t* edge_flags, const int64_t* edge_vid,
                 const int64_t* cell_off, float* verts, int32_t* faces, void* stream) {
  HOLD_REQUIRE(ctx && vol && edge_flags && edge_vid && cell_off, "NULL argument");
  HOLD_REQUIRE(n0 >= 2 && n1 >= 2 && n2 >= 2, "grid must be at least 2 x 2 x 2");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  mc::Dims d{n0, n1, n2};
  const int64_t total = (int64_t)n0 * n1 * n2;
  k_mc_emit<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d, vol, level, edge_flags, edge_vid, cell_off, verts, faces);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

/* measurement hook (not in the public header): key 2 = accumulator compensation c of the tensor-core SDF chains (tools/exp_r2b.py) */
int hold_debug_set(hold_ctx* ctx, int key, int value) {
  if (!ctx) return HOLD_E_BADARG;
  if (key == 2) ctx->tc_acc_comp = value;
  else if (key == 3) ctx->sampler_passes = value;
  else return HOLD_E_BADARG;
  return HOLD_OK;
}

#ifdef HOLD_TC_PHASE_TIMING
/* measurement build only (tools/prof_mlp_phases.py): the tensor-core MLP kernels' phase clocks since the last call, summed over
 * the CTAs, as out[kTcMaxSteps layers][2 warpgroups][kPhSlots]; the device counters are zeroed. */
int hold_tc_phase_read(hold_ctx* ctx, unsigned long long* out) {
  if (!ctx || !out) return HOLD_E_BADARG;
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_CUDA(cudaDeviceSynchronize());
  static unsigned long long host[kPhMaxCtas][kTcMaxSteps][2][kPhSlots];
  HOLD_CUDA(cudaMemcpyFromSymbol(host, g_tc_phase, sizeof(host)));
  for (int i = 0; i < kTcMaxSteps * 2 * kPhSlots; ++i) {
    out[i] = 0;
    for (int c = 0; c < kPhMaxCtas; ++c) out[i] += (&host[c][0][0][0])[i];
  }
  void* dev = nullptr;
  HOLD_CUDA(cudaGetSymbolAddress(&dev, g_tc_phase));
  HOLD_CUDA(cudaMemset(dev, 0, sizeof(host)));
  return HOLD_OK;
}
#endif

/* debug/test hook (not in the public header): workspace slot pointers of the last call */
int hold_debug_ws_copy(hold_ctx* ctx, int slot, void* dst, size_t bytes) {
  if (!ctx || slot < 0 || slot >= WS_COUNT || ctx->ws[slot].bytes < bytes) return HOLD_E_BADARG;
  HOLD_CUDA(cudaDeviceSynchronize());
  HOLD_CUDA(cudaMemcpy(dst, ctx->ws[slot].p, bytes, cudaMemcpyDeviceToDevice));
  return HOLD_OK;
}

int hold_bg_set_weights(hold_ctx* ctx, const hold_mlp_weights* sdf, const hold_mlp_weights* rgb, int mlp_mode, void* stream) {
  HOLD_REQUIRE(ctx && sdf && rgb, "NULL argument");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  HOLD_REQUIRE(mlp_mode == HOLD_MLP_FP32 || mlp_mode == HOLD_MLP_TC, "bad mlp_mode");
  int rc;
  if ((rc = check_skip_net(sdf, kBgSdfShape)) || (rc = check_colour_net(rgb, kBgRgbShape))) return rc;
  const bool tc = mlp_mode == HOLD_MLP_TC;
  ctx->has_bg = false;   // until both nets are packed for this mode
  if ((rc = pack_skip_net(ctx, ctx->bg_sdf, sdf, kBgSdfShape, tc, s)) || (rc = pack_colour_net(ctx, ctx->bg_rgb, rgb, kBgRgbShape, tc, s))) return rc;
  ctx->bg_mlp_mode = mlp_mode;
  ctx->has_bg = true;
  return HOLD_OK;
}

// the bounding sphere is a per-node constant in the reference (same value for all nodes): take the first configured node's
static int bg_sphere(hold_ctx* ctx, float* r_sphere) {
  *r_sphere = 0.f;
  for (int n = 0; n < HOLD_MAX_NODES; ++n)
    if (ctx->nodes[n].configured) { *r_sphere = ctx->nodes[n].cfg.bounding_sphere; break; }
  HOLD_REQUIRE(*r_sphere > 0.f, "configure a node first (scene_bounding_sphere)");
  return HOLD_OK;
}

int hold_background(hold_ctx* ctx, int R, int B, const float* cam_loc, const float* ray_dirs, const float* frame_code,
                    const float* fg_bg_weights, float* bg_rgb, float* bg_rgb_only, float* bg_semantics, float* bg_z_vals,
                    void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  if (!ctx->has_bg) { set_error("background weights not set (hold_bg_set_weights)"); return HOLD_E_STATE; }
  HOLD_REQUIRE(R >= 0 && B >= 1, "bad R/B");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(R % B == 0, "R (%d) must be B (%d) frames x rays, frame-major", R, B);
  HOLD_REQUIRE(cam_loc && ray_dirs && frame_code && fg_bg_weights, "NULL argument");
  float r_sphere;
  if (int rc = bg_sphere(ctx, &r_sphere)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int rpf = R / B;
  const int rays_per_chunk = max(1, min(rpf, (1 << 20) / kBgN));
  const size_t cp = (size_t)rays_per_chunk * kBgN;
  WS(WS_BGSDF, float, cp, sdf_ws);
  WS(WS_BGFEAT, float, cp * kFeat, feat_ws);
  WS(WS_BGRGB, float, cp * 3, rgb_ws);
  for (int b = 0; b < B; ++b) {
    for (int r0 = 0; r0 < rpf; r0 += rays_per_chunk) {
      const int rn = min(rays_per_chunk, rpf - r0), P = rn * kBgN;
      const size_t ray0 = (size_t)b * rpf + r0;
      BgArgs a;
      memset(&a, 0, sizeof(a));
      a.P = P, a.pts_per_frame = P, a.cam = cam_loc + ray0 * 3, a.dirs = ray_dirs + ray0 * 3, a.frame_code = frame_code + (size_t)b * kBgFrame;
      a.r_sphere = r_sphere;
      simt_layers(ctx->bg_sdf, ctx->bg_sdf.n_layers, a);
      a.sdf = sdf_ws, a.feat = feat_ws;
      if (ctx->bg_mlp_mode == HOLD_MLP_TC) {
        int rc = tc_bg_launch(ctx, P, a.cam, a.dirs, a.frame_code, a.r_sphere, sdf_ws, feat_ws, rgb_ws, s);
        if (rc) return rc;
      } else {
        const int tiles = ceil_div(P, kTileRows);
        k_bg_mlp<BG_SDF><<<min(tiles, ctx->sm_count), 256, kBgSmemBytes, s>>>(a);
        HOLD_LAUNCH_CHECK(ctx);
        BgArgs c = a;
        simt_layers(ctx->bg_rgb, ctx->bg_rgb.n_layers, c);
        c.rgb = rgb_ws;
        k_bg_mlp<BG_RGB><<<min(tiles, ctx->sm_count), 256, kBgSmemBytes, s>>>(c);
        HOLD_LAUNCH_CHECK(ctx);
      }
      k_bg_composite<<<ceil_div(rn, 128), 128, 0, s>>>(rn, a.r_sphere, nullptr, sdf_ws, rgb_ws, fg_bg_weights + ray0,
                                                       bg_rgb ? bg_rgb + ray0 * 3 : nullptr, bg_rgb_only ? bg_rgb_only + ray0 * 3 : nullptr,
                                                       bg_semantics ? bg_semantics + ray0 * 4 : nullptr, bg_z_vals ? bg_z_vals + ray0 * kBgN : nullptr);
      HOLD_LAUNCH_CHECK(ctx);
    }
  }
  return HOLD_OK;
}

int hold_bg_encode(hold_ctx* ctx, int R, int B, const float* cam_loc, const float* ray_dirs, const float* jitter, float* bg_z_vals,
                   float* pe_pts, int ld_pts, float* pe_view, int ld_view, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(R >= 0 && B >= 1, "bad R/B");
  HOLD_REQUIRE(R % B == 0, "R (%d) must be B (%d) frames x rays, frame-major", R, B);
  HOLD_REQUIRE(ld_pts >= kBgEmbed && ld_view >= kBgView, "ld_pts (%d) must be >= %d and ld_view (%d) >= %d", ld_pts, kBgEmbed, ld_view, kBgView);
  HOLD_REQUIRE((size_t)R * kBgN <= (size_t)INT32_MAX, "R (%d) too large", R);
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(cam_loc && ray_dirs && bg_z_vals && pe_pts && pe_view, "NULL argument");
  float r_sphere;
  if (int rc = bg_sphere(ctx, &r_sphere)) return rc;
  k_bg_encode<<<ceil_div(R * kBgN, 128), 128, 0, (cudaStream_t)stream>>>(R, r_sphere, cam_loc, ray_dirs, jitter, bg_z_vals, pe_pts, ld_pts,
                                                                        pe_view, ld_view);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_bg_integrate(hold_ctx* ctx, int R, const float* bg_z_vals, const float* sdf, const float* rgb, const float* fg_bg_weights,
                      float* bg_rgb, float* bg_rgb_only, float* bg_semantics, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(R >= 0, "negative R");
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(bg_z_vals && sdf && rgb && fg_bg_weights, "NULL argument");
  k_bg_composite<<<ceil_div(R, 128), 128, 0, (cudaStream_t)stream>>>(R, 0.f, bg_z_vals, sdf, rgb, fg_bg_weights, bg_rgb, bg_rgb_only,
                                                                    bg_semantics, nullptr);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_bg_integrate_bwd(hold_ctx* ctx, int R, const float* bg_z_vals, const float* sdf, const float* rgb, const float* fg_bg_weights,
                          const float* g_bg_rgb, const float* g_bg_rgb_only, const float* g_bg_semantics, float* d_sdf, float* d_rgb,
                          float* d_fg_bg_weights, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  HOLD_REQUIRE(R >= 0 && R <= INT32_MAX / kBgN, "bad R (%d)", R);
  if (R == 0) return HOLD_OK;
  HOLD_REQUIRE(bg_z_vals && sdf && rgb && fg_bg_weights && d_sdf && d_rgb && d_fg_bg_weights, "NULL argument");
  k_bg_composite_bwd<<<ceil_div(R * kBgN, 128), 128, 0, (cudaStream_t)stream>>>(R, bg_z_vals, sdf, rgb, fg_bg_weights, g_bg_rgb, g_bg_rgb_only,
                                                                               g_bg_semantics, d_sdf, d_rgb, d_fg_bg_weights);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_sdf_eval(hold_ctx* ctx, int node, int P, const float* x_c, const float* embed_w, float* sdf, float* grad,
                  float* feat, void* stream) {
  int rc = check_node(ctx, node, true);
  if (rc) return rc;
  HOLD_REQUIRE(P >= 0, "negative P");
  if (P == 0) return HOLD_OK;
  HOLD_REQUIRE(x_c && sdf, "NULL argument");
  HOLD_REQUIRE((grad == nullptr) == (feat == nullptr), "grad and feat must be requested together");
  return launch_sdf(ctx, ctx->nodes[node], P, x_c, embed_w, sdf, grad, feat, nullptr, (cudaStream_t)stream);
}

int hold_linear(hold_ctx* ctx, int node, int mat, int P, const float* A, int lda, int kvalid, int add_bias, const float* in_scale,
                float* C, int ldc, int nvalid, void* stream) {
  HOLD_REQUIRE(ctx != nullptr, "ctx is NULL");
  HOLD_REQUIRE(P >= 0, "negative P");
  if (P == 0) return HOLD_OK;
  HOLD_REQUIRE(A && C, "NULL argument");
  LinearMat m;
  if (node == -1) {   // the background nets (hold_bg_set_weights with HOLD_MLP_TC)
    HOLD_CUDA(cudaSetDevice(ctx->device));
    HOLD_REQUIRE(ctx->has_bg, "hold_linear(node -1) needs tensor-core background weights (hold_bg_set_weights, HOLD_MLP_TC)");
    if (ctx->bg_mlp_mode != HOLD_MLP_TC) {
      set_error("hold_linear(node -1): the background weights were last set with HOLD_MLP_FP32; its tensor-core images are not current");
      return HOLD_E_STATE;
    }
    m = linear_mat(ctx->bg_sdf, ctx->bg_rgb, mat);
  } else {
    int rc = check_node(ctx, node, true);
    if (rc) return rc;
    m = linear_mat(ctx->nodes[node].sdf, ctx->nodes[node].rgb, mat);
  }
  HOLD_REQUIRE(m.img != nullptr, "hold_linear: unknown matrix id %d for node %d", mat, node);
  HOLD_REQUIRE(kvalid >= 1 && kvalid <= m.kmax && nvalid >= 1 && nvalid <= m.nmax, "hold_linear(%d): kvalid %d (max %d) / nvalid %d (max %d)", mat, kvalid,
               m.kmax, nvalid, m.nmax);
  HOLD_REQUIRE(!add_bias || m.bias != nullptr, "hold_linear(%d): this matrix has no bias", mat);
  return tc_launch_linear_img(ctx, m.img, add_bias ? m.bias : nullptr, m.nst, P, A, lda, kvalid, in_scale, C, ldc, nvalid, (cudaStream_t)stream);
}

int hold_wgrad(hold_ctx* ctx, int P, const float* D, int ldd, int N, const float* A, int lda, int K, const float* d_scale,
               const float* a_scale, float* out, int ldo, void* stream) {
  HOLD_REQUIRE(ctx && D && A && out, "NULL argument");
  HOLD_REQUIRE(P >= 0 && N >= 1 && N <= 256 && K >= 1 && K <= 256 && ldd >= N && lda >= K && ldo >= K, "hold_wgrad: N, K in [1, 256]");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  if (P == 0) {
    HOLD_CUDA(cudaMemset2DAsync(out, (size_t)ldo * sizeof(float), 0, (size_t)K * sizeof(float), N, s));
    return HOLD_OK;
  }
  // the partials' workspace has one size for every shape, so a captured call never sees it reallocated by a later call
  WS(WS_WGRAD, uint8_t, kWgPartBytes, part);
  WgArgs a;
  a.P = P, a.N = N, a.K = K, a.ldd = ldd, a.lda = lda, a.ldo = ldo, a.D = D, a.A = A, a.d_scale = d_scale, a.a_scale = a_scale;
  a.part = (float*)part, a.out = out, a.err = ctx->dev_err;
  const int splits = wgrad_splits(P, N);
  k_wgrad_tc<<<dim3(splits, ceil_div(N, kWgRowsD)), kWgThreads, kWgSmem, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  k_wgrad_sum<<<ceil_div(N * K, 32), kWgSumWarps * 32, 0, s>>>(a.part, splits, N, K, out, ldo);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_pow2_scale(hold_ctx* ctx, int P, int ncols, const float* x, int ld, float* scale_out, void* stream) {
  HOLD_REQUIRE(ctx && x && scale_out, "NULL argument");
  HOLD_REQUIRE(P >= 1 && ncols >= 1 && ld >= ncols, "bad sizes");
  HOLD_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  void* w = nullptr;
  int rc = ws_get(ctx, WS_AMAX, 256, &w);
  if (rc) return rc;
  // one word per call, rotating through the workspace so that back-to-back calls on a stream never share a counter in flight
  unsigned int* bits = (unsigned int*)w + (ctx->launches & 31);
  HOLD_CUDA(cudaMemsetAsync(bits, 0, sizeof(unsigned int), s));
  const size_t total = (size_t)P * ncols;
  k_absmax_bits<<<(int)std::min<size_t>((total + 255) / 256, (size_t)ctx->sm_count * 8), 256, 0, s>>>(P, ncols, x, ld, bits);
  HOLD_LAUNCH_CHECK(ctx);
  k_pow2_scale<<<1, 1, 0, s>>>(bits, scale_out);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_train_ew(hold_ctx* ctx, int op, int P, const hold_ew_args* args, void* stream) {
  HOLD_REQUIRE(ctx && args, "NULL argument");
  HOLD_REQUIRE(op >= 0 && op <= EW_RELU_BWD && P >= 0, "bad op / P");
  if (P == 0) return HOLD_OK;
  HOLD_CUDA(cudaSetDevice(ctx->device));
  EwArgs a;
  a.in0 = args->in0, a.in1 = args->in1, a.in2 = args->in2, a.out0 = args->out0, a.out1 = args->out1;
  a.ld_in0 = args->ld_in0, a.ld_in1 = args->ld_in1, a.ld_in2 = args->ld_in2, a.ld_out0 = args->ld_out0, a.ld_out1 = args->ld_out1;
  a.ncols = args->ncols, a.aux = args->aux;
  HOLD_REQUIRE(a.ncols >= 1 && a.ncols <= 320 && a.in0 && a.out0, "bad elementwise arguments");
  const size_t total = (size_t)P * (size_t)a.ncols;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->sm_count * 16);
  k_train_ew<<<blocks, 256, 0, (cudaStream_t)stream>>>(op, P, a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_rgb_eval(hold_ctx* ctx, int node, int B, int P, const float* x_c, const float* normals, const float* pose_cond,
                  const float* feat, const float* time_code, float* rgb, void* stream) {
  int rc = check_node(ctx, node, true);
  if (rc) return rc;
  HOLD_REQUIRE(B >= 1 && P >= 0, "bad sizes");
  if (P == 0) return HOLD_OK;
  HOLD_REQUIRE(P % B == 0, "P (%d) must be B (%d) frames x points, frame-major", P, B);
  HOLD_REQUIRE(x_c && normals && feat && rgb, "NULL argument");
  NodeState& ns = ctx->nodes[node];
  const bool hand = ns.cfg.kind == HOLD_KIND_HAND;
  cudaStream_t s = (cudaStream_t)stream;
  float* pe = nullptr;
  if (hand) {
    HOLD_REQUIRE(pose_cond != nullptr, "hand node needs pose_cond [B,45] (zeros give lin_pose's bias, texture_net.py:80-82)");
    WS(WS_PE, float, (size_t)B * 8, pe_ws);
    pe = pe_ws;
    k_pose_embed<<<ceil_div(B * 8, 64), 64, 0, s>>>(B, pose_cond, ns.lin_pose_w, ns.lin_pose_b, pe);
    HOLD_LAUNCH_CHECK(ctx);
  } else {
    HOLD_REQUIRE(time_code != nullptr, "object node needs time_code [B,32]");
  }
  return launch_rgb(ctx, ns, P, P / B, x_c, normals, pe, feat, hand ? nullptr : time_code, rgb, s);
}

int hold_forward_warp(hold_ctx* ctx, int node, int B, int P, const float* x_c, const hold_node_pose* pose, float* x_d,
                      int32_t* knn_idx, uint8_t* outlier_mask, void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  HOLD_REQUIRE(B >= 0 && P >= 0, "negative size");
  if (B * P == 0) return HOLD_OK;
  HOLD_REQUIRE(x_c && pose && x_d && pose->tfs, "NULL argument");
  NodeState& ns = ctx->nodes[node];
  dim3 grid(ceil_div(P, 128), B);
  cudaStream_t s = (cudaStream_t)stream;
  if (ns.cfg.kind == HOLD_KIND_HAND) {
    if (!ns.has_rig) { set_error("hand node has no rig (hold_node_set_rig)"); return HOLD_E_STATE; }
    k_inverse_warp<true, false, true><<<grid, 128, 0, s>>>(P, 1, 1, nullptr, nullptr, nullptr, x_c, pose->tfs, ns.cano_verts, ns.skin_w, x_d,
                                                           knn_idx, outlier_mask, nullptr, ctx->dev_err);
  } else {
    k_inverse_warp<false, false, true><<<grid, 128, 0, s>>>(P, 1, 1, nullptr, nullptr, nullptr, x_c, pose->tfs, nullptr, nullptr, x_d,
                                                            nullptr, nullptr, nullptr, ctx->dev_err);
  }
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

int hold_inverse_warp(hold_ctx* ctx, int node, int B, int P, const float* x, const hold_node_pose* pose, float* x_c,
                      int32_t* knn_idx, uint8_t* outlier_mask, void* stream) {
  int rc = check_node(ctx, node, false);
  if (rc) return rc;
  HOLD_REQUIRE(B >= 0 && P >= 0, "negative size");
  if (B * P == 0) return HOLD_OK;
  HOLD_REQUIRE(x && pose && x_c && pose->tfs, "NULL argument");
  return launch_inverse_warp(ctx, ctx->nodes[node], B, P, false, 1, 1, nullptr, nullptr, nullptr, x, pose, x_c, knn_idx,
                             outlier_mask, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
