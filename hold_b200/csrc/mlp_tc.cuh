// Tensor-core fused MLP chains on Hopper (sm_90a wgmma) — HOLD_MLP_TC.
//
// One persistent CTA per SM walks 128-row tiles through the whole layer chain:
//   * warps 0..7 : two consumer warpgroups, each owning 64 rows of the tile.  Per layer a warpgroup issues wgmma.mma_async
//                  m64n256k16 over the layer's weight stages into a [64 x 256] fp32 accumulator held in its registers (128 per
//                  thread), then runs the epilogue on those registers: bias + activation in fp32, split into fp16 hi/lo, and
//                  write the next layer's A operand (SW128 K-major) for its own 64 rows back to shared memory.  The two
//                  warpgroups share only the weight ring, so one warpgroup's epilogue overlaps the other's MMAs.
//   * warp 8     : (of a third warpgroup that hands its registers to the consumers through setmaxnreg) bulk-async (TMA engine) copies of pre-swizzled fp16 weight chunks L2 -> smem ring, mbarrier handshake
//                  (full: transaction count; empty: one arrival per consumer warp once its wgmma group has read the stage).
// Arithmetic: every fp32 operand x is split x = hi + lo (fp16 each: 11 + 11 mantissa bits) and each product is
// three MMAs (hi*hi + lo*hi + hi*lo, fp32 accumulate) — ~2^-21 relative per product (fp32-GEMM level), with an absolute floor
// of ~3e-8 where lo goes subnormal.  This is what the 1e-4 parity bar needs: an sdf error eps reaches the density as eps/beta^2
// (beta down to 1e-2), so plain bf16 (2^-9) and even a bf16 split (2^-16) do not meet it (SURVEY §7 "hard parts").  Range: |x|
// must stay below 65504 (activations/weights here are O(1e-3..1e2)).  The sdf / rgb heads (1 resp. 3 output rows) are fp32 dot
// products in the epilogue.  Gradients: reverse mode in the same kernel (MODE MLP_SDF_REV): the forward epilogues stash
// softplus'(z_l) as unorm16 (512 KB per CTA, L2-resident; quantisation step 1.5e-5 moves the gradient by <= 1.2e-5 of its
// scale, tests/test_cpu_stash_quant.py), the backward layers run over transposed weight images.
// Embeddings (tile prologue, skip layer) are inlined branch-free sin/cos (sincos_cw).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "embed_phases.h"
#include "mlp_simt.cuh"

namespace hold {

constexpr int kTcRows = 128;
constexpr int kTcStageBytes = 32768;      // one weight stage: [256 n x 32 k] fp16 hi (16 KB) + lo (16 KB)
constexpr int kTcAChunkBytes = 16384;     // one A chunk: [128 rows x 64 k] fp16
// Power-of-two operand scaling (exact): fp16 operands are fed to the tensor core as A * 2^6 and W * 2^10 so that
// the LOW halves of the hi/lo split stay in fp16's normal range for |a| >= 2e-3, |w| >= 1.2e-4 (unscaled, the low
// half of every |x| < 0.125 is subnormal and the split gains only 2x over bf16).  The accumulator is rescaled by 2^-16 in
// the epilogue's bias FMA.  Range: |a| < 1023, |w| < 64.
constexpr float kTcScaleA = 64.0f, kTcScaleW = 1024.0f, kTcUnscale = 1.0f / (64.0f * 1024.0f);
// Accumulator-truncation compensation of the Softplus chains: the tensor core adds into its fp32 accumulator with truncation
// (round toward zero), not round-to-nearest, so every layer of 48 accumulations (K = 256 x 3 passes) comes out shrunk by a few
// units of 2^-24 relative — a bias, not noise.  Undoing it in the epilogue's unscale multiply (free) lowers the sdf error, which
// is what the Laplace density needs at small beta (error amplification 1 / (2 beta^2), engine/density.py:21-26).  Measured on the
// H100 against float64 (tools/exp_r2b.py section 1, hand and object nets, reference init and perturbed): the mean sdf error crosses
// zero at c = 11.0 .. 12.9, and c = 12 lowers the max sdf error 4-7x against c = 0 (DESIGN.md §3.1).  hold_debug_set key 2
// overrides it for such measurements.
constexpr int kTcAccComp = 12;

constexpr int kTcMaxSteps = 17;
struct TcLayer {
  const uint8_t* wimg;  // pre-swizzled stage images, nst * 32 KB
  const float* bias;    // [256]
  int nst;              // number of 32-wide k stages
  int N;                // valid outputs
};

__global__ void k_scale_vec(const float* __restrict__ src, int n, float c, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = c * src[i];
}

struct TcMlp {
  uint8_t* sdf_img[HOLD_MAX_LAYERS] = {nullptr};
  uint8_t* rgb_img[HOLD_MAX_LAYERS] = {nullptr};
  uint8_t* sdf_imgT[HOLD_MAX_LAYERS] = {nullptr};  // W_l^T images of layers 0..7 for the reverse-mode gradient, 8: feature rows (training)
  uint8_t* rgb_imgT[6] = {nullptr};                // training backward: [0] W_0^T feature part, [1] W_0^T other inputs, [2..4] W_1..3^T
  int sdf_nst[HOLD_MAX_LAYERS], rgb_nst[HOLD_MAX_LAYERS];
  float* bias_s = nullptr;   // [13][256]: biases as the epilogues add them: SDF lin0..7 times kTcScaleA, lin8 (feature rows) plain, colour lin0..3 times kTcScaleA
};

struct TcArgs {
  int P, n_layers;
  TcLayer L[kTcMaxSteps];
  uint16_t* sig;  // reverse mode: per-CTA stash of softplus'(z_l) as unorm16, [grid][8 layers][128 rows x 256 columns]
  const float* w_last;
  const float* b_last;
  const float* xc;
  const float* embed_w;
  float* sdf;
  float* grad;
  float* feat;
  const float* normal;
  const float* pose_embed;
  const float* time_code;
  int pts_per_frame, k0;
  float* rgb;
  const SamplerState* st;
  int* err;
  const float* cam;          // background modes: ray origins / directions [R,3] of this frame chunk, its frame code [32]
  const float* dirs;
  const float* frame_code;
  float r_sphere;
  float unscale;             // accumulator -> value: kTcUnscale (times the accumulator compensation, hold_debug_set key 2)
  // MLP_LINEAR (hold_linear): C[P, nvalid] = A[P, kvalid] . W^T (+ bias): one layer against one packed image
  const float* lin_in;
  float* lin_out;
  const float* in_scale;     // device scalar s (a power of two) or NULL: A is fed as A / s, C comes out times s (keeps tiny gradients
                             // inside the fp16 hi/lo split's range)
  int lda, ldc, kvalid, nvalid;
  int passes;                // MMAs per product: 3 = hi*hi + lo*hi + hi*lo (always, in production); 2 / 1 only through the measurement
                             // hook hold_debug_set(ctx, 3, n) for the sampler rounds
};

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must surface as an error code, never as a hung GPU.  On a timeout the waiter
// records its tag in the device error word and raises the CTA's abort flag (shared memory); every other wait polls
// that flag, so the kernel drains in microseconds and hold_ctx_check() reports HOLD_E_STATE.
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, int* err, int tag, volatile int* abort_flag) {
  uint32_t done = 0;
  for (unsigned spin = 0; spin < (1u << 22); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return true;
    if ((spin & 63) == 63 && *abort_flag) return false;
  }
  if (err != nullptr) atomicOr(err, 0x100 | (tag << 12));
  *abort_flag = 1;
  return false;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// generic-proxy st.shared -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// One lane of a fully converged warp: the producer warp walks its loop with ALL lanes (warp-uniform control flow keeps the
// barrier addresses in uniform registers) and elects the issuing lane per bulk copy.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// Barrier over one warpgroup (named barrier `id`, 128 threads) that also returns whether `v` holds in every thread: the
// warpgroup leaves a pipeline together (wgmma is warpgroup-collective, so a partial exit would stall the rest).
__device__ __forceinline__ bool wg_all(bool v, int id) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.and.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r)
      : "r"((uint32_t)v), "r"(id)
      : "memory");
  return r != 0;
}

// wgmma shared-memory matrix descriptor (sm_90 GMMA format), K-major canonical layouts:
// start address >> 4 | LBO (=1, unused for swizzled K-major) | SBO = bytes between 8-row groups | layout type (bits 62-63)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t sbo_bytes, uint32_t layout_type) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout_type << 62;
  return d;
}
constexpr uint32_t kLayoutSW128 = 1, kLayoutSW64 = 2;

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, fp16 operands from shared memory (both K-major), fp32 accumulator in registers.
// Fragment of D in thread t of the warpgroup (warp w = t / 32, lane): d[4j + 2h + i] = D[16 w + lane / 4 + 8 h][8 j + 2 (lane % 4) + i].
__device__ __forceinline__ void wgmma_256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accum)
      : "memory");
}

// x = hi + lo: hi = fp16(x), lo = fp16(x - hi)
__device__ __forceinline__ void split8(const float* x, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 hh = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}
// byte offset of the 16-byte unit holding k = 8j..8j+7 of row r inside one [128 x 64] SW128 K-major A chunk
__device__ __forceinline__ uint32_t a_unit_off(int r, int j) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((j ^ (r & 7)) << 4));
}

__device__ __forceinline__ float mufu_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float mufu_lg2(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float mufu_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// kTcScaleA * Softplus(beta=100)(z) in its overflow-free form max(z,0) + log1p(exp(-|100 z|))/100 (two MUFU ops), from
// zs = kTcScaleA * z (the epilogue's bias FMA produces zs directly: accumulator scale and bias carry the power-of-two factor,
// so every value is bit-identical to scaling afterwards).  nn.Softplus' threshold branch (returns z for 100 z > 20) differs
// from this by < 2.1e-11.  u_out = exp(-|100 z|) for the derivative.
__device__ __forceinline__ float softplus100_scaled(float zs, float& u_out) {
  const float t = zs * (100.0f * 1.4426950408889634f / kTcScaleA);
  const float u = mufu_ex2(-fabsf(t));
  u_out = u;
  const float L = mufu_lg2(1.0f + u);
  return fmaf(L, 0.6931471805599453f * 0.01f * kTcScaleA, fmaxf(zs, 0.f));
}

// unorm16 stash of softplus' in [0, 1]: encode by the magic-number add (round to nearest, no F2I), decode by OR-ing the
// 16 bits into the mantissa of 2^23.  q = round(65535 s); decode returns q as a float (the caller folds 1/65535 into its scale).
__device__ __forceinline__ uint32_t unorm16_pack2(float s0, float s1) {
  const uint32_t b0 = __float_as_uint(fmaf(s0, 65535.0f, 8388608.0f)), b1 = __float_as_uint(fmaf(s1, 65535.0f, 8388608.0f));
  return __byte_perm(b0, b1, 0x5410);
}
__device__ __forceinline__ float unorm16_lo(uint32_t w) { return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7410)) - 8388608.0f; }
__device__ __forceinline__ float unorm16_hi(uint32_t w) { return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7432)) - 8388608.0f; }

struct Embed8 { float v[8]; uint32_t ok; };
template <int D, bool DERIV>
__device__ __forceinline__ Embed8 embed8(int e0, int n_embed, float x0, float x1, float x2, float x3, const float* __restrict__ ew) {
  Embed8 r;
  if (e0 >= n_embed || e0 + 8 <= 0) {   // no element of this group exists
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = 0.f;
    r.ok = 0;
    return r;
  }
  r.ok = embedn_inl<D, DERIV>(e0, n_embed, x0, x1, x2, x3, ew, r.v);
  return r;
}
// elements e0, e0 + 1 of the embedding (one accumulator column pair of the epilogue); returns the mask of those that exist
template <int D, bool DERIV>
__device__ __forceinline__ uint32_t embed2(int e0, int n_embed, const float (&pt)[4], const float* __restrict__ ew, float (&v)[2]) {
  if (e0 >= n_embed || e0 + 2 <= 0) {
    v[0] = v[1] = 0.f;
    return 0;
  }
  return embedn_inl<D, DERIV>(e0, n_embed, pt[0], pt[1], pt[2], pt[3], ew, v);
}

constexpr int kTcConsumers = 256;                     // two warpgroups: warps 0..7
constexpr int kTcThreadsTotal = kTcConsumers + 128;   // + the producer warpgroup (warp 8 issues the copies, 9..11 exit at once)
// registers per thread after the warpgroups' setmaxnreg: producer 40, consumers 232 (128 x 40 + 256 x 232 <= 64 K)
constexpr int kTcProducerRegs = 40, kTcConsumerRegs = 232;

template <int MODE>
struct TcCfg {
  static constexpr bool kColorLike = (MODE == MLP_COLOR || MODE == MLP_BG_RGB);   // ReLU chain with a 3-row sigmoid head
  static constexpr bool kWide = kColorLike || MODE == MLP_LINEAR;                  // first operand up to 320 wide
  static constexpr int kAChunks = kWide ? 5 : 4;   // 64-wide SW128 A chunks in smem
  static constexpr int kStages = kWide ? 2 : 3;
  static constexpr int kSmemA = 2 * kAChunks * kTcAChunkBytes;
  static constexpr int kSmemW = kStages * kTcStageBytes;
  static constexpr int kSmemBytes = kSmemA + kSmemW + 256 + 1024;  // + barriers (2 x 3, 8 B each) and the abort flag + 1 KB alignment slack
};

// Weight ring and A operand of one consumer warpgroup.
struct Pipe {
  uint32_t a_hi, a_lo;     // this warpgroup's 64 rows of A chunk 0 (hi / lo part), shared-space addresses
  uint32_t sW, bWFull, bWEmpty;
  uint32_t stage, phase;
  int ns, lane, bar_id;
  volatile int* abort_flag;
};

// All MMAs of layer l for this warpgroup: acc = A . W_l^T over the layer's k stages (PASSES MMAs per k16 step).  A stage is released
// to the producer when the wgmma group that read it has completed (one group in flight behind the one just issued).  PASSES is a
// template parameter so that no branch sits between the wgmmas on the accumulator (ptxas would serialise them with extra
// warpgroup.arrive instructions).
template <int PASSES>
__device__ __forceinline__ bool mma_layer_p(const TcArgs& a, Pipe& P, const int l, float (&acc)[128]) {
  const int nst = a.L[l].nst;
  uint32_t prev = 0;
  for (int s = 0; s < nst; ++s) {
    const bool got = mbar_wait(P.bWFull + 8 * P.stage, P.phase, a.err, 3, P.abort_flag);
    if (!wg_all(got, P.bar_id)) {
      wgmma_wait<0>();
      return false;
    }
    const uint32_t wb = P.sW + P.stage * kTcStageBytes;
    const int c = s >> 1;  // 64-wide A chunk holding this 32-k stage
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t koff = (uint32_t)(((s & 1) * 2 + j) * 32);  // bytes inside the 128-byte A row
      const uint64_t ahi = gmma_desc(P.a_hi + c * kTcAChunkBytes + koff, 1024, kLayoutSW128);
      const uint64_t alo = gmma_desc(P.a_lo + c * kTcAChunkBytes + koff, 1024, kLayoutSW128);
      const uint64_t whi = gmma_desc(wb + j * 32, 512, kLayoutSW64);
      const uint64_t wlo = gmma_desc(wb + 16384 + j * 32, 512, kLayoutSW64);
      wgmma_256(acc, ahi, whi, (s | j) != 0);
      if (PASSES >= 2) wgmma_256(acc, alo, whi, 1);
      if (PASSES >= 3) wgmma_256(acc, ahi, wlo, 1);
    }
    wgmma_commit();
    if (s > 0) {
      wgmma_wait<1>();
      __syncwarp();
      if (P.lane == 0) mbar_arrive(P.bWEmpty + 8 * prev);
    }
    prev = P.stage;
    if (++P.stage == (uint32_t)P.ns) { P.stage = 0; P.phase ^= 1; }
  }
  wgmma_wait<0>();
  __syncwarp();
  if (P.lane == 0) mbar_arrive(P.bWEmpty + 8 * prev);
  return true;
}
__device__ __forceinline__ bool mma_layer(const TcArgs& a, Pipe& P, const int l, float (&acc)[128]) {
  if (a.passes >= 3) return mma_layer_p<3>(a, P, l, acc);
  return (a.passes == 2) ? mma_layer_p<2>(a, P, l, acc) : mma_layer_p<1>(a, P, l, acc);
}

// Per-thread view of the accumulator fragment: rows r[0] and r[1] = r[0] + 8 of the tile, columns 8 j + 2 q + {0, 1}, j = 0..31.
struct Frag {
  uint8_t* a_row[2];     // generic pointer to row r[h] inside A chunk 0 (hi part), plus the thread's 4-byte slot
  int r7[2];             // r[h] & 7 (the SW128 swizzle of the row)
  uint32_t lo_off;       // hi -> lo part distance
  int q;
  int p[2];
  bool valid[2];
  float pt[2][4];        // the rows' points (embedding inputs of the skip columns)
  float head[2][3];
  float gz[2];           // reverse mode: d sdf / d z (head[h][1], head[h][2] hold d/dx, d/dy)
};

// two fp16 hi/lo pairs of the next layer's operand for accumulator columns c0 = 8 j + 2 q, c0 + 1 of row h
__device__ __forceinline__ void frag_store_a(const Frag& F, int h, int j, float o0, float o1) {
  uint32_t hi, lo;
  split2(o0, o1, hi, lo);
  uint8_t* dst = F.a_row[h] + (j >> 3) * kTcAChunkBytes + (((j & 7) ^ F.r7[h]) << 4);
  *reinterpret_cast<uint32_t*>(dst) = hi;
  *reinterpret_cast<uint32_t*>(dst + F.lo_off) = lo;
}

// One layer of a forward chain (every mode but the reverse-mode gradient and hold_linear), on the accumulator in registers:
//   HEAD : the 1- (sdf) or 3-row (colour) output head is accumulated from this layer's activations (fp32 dot products)
//   WRITE: the activations are the next MMA's operand (false on the chain's last MMA layer)
//   FEAT : the layer's outputs are the 256-d feature vector (no activation, stored to global memory)
//   SKIP : output columns >= a.L[l].N are the point's embedding (the skip connection into the next layer, shape_net.py:116-119)
// One specialised body per layer kind.  a.L[l].bias is pre-multiplied by kTcScaleA unless FEAT (TcMlp::bias_s).
template <int MODE, bool HEAD, bool WRITE, bool FEAT, bool SKIP>
__device__ __forceinline__ void epi_layer(const TcArgs& a, Frag& F, const int l, const float (&acc)[128]) {
  constexpr bool kColorLike = (MODE == MLP_COLOR || MODE == MLP_BG_RGB);
  const int N = a.L[l].N;
  const float* bias = a.L[l].bias;
  const float us = FEAT ? a.unscale : a.unscale * kTcScaleA;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c0 = 8 * j + 2 * F.q;
    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + c0));
    float2 w0, w1, w2;
    if (HEAD) {
      w0 = __ldg(reinterpret_cast<const float2*>(a.w_last + c0));
      if (kColorLike) {
        w1 = __ldg(reinterpret_cast<const float2*>(a.w_last + 256 + c0));
        w2 = __ldg(reinterpret_cast<const float2*>(a.w_last + 512 + c0));
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // accumulator -> pre-activation times kTcScaleA (undo the weight scaling, add the scaled bias); o is the next layer's operand,
      // i.e. the activation times kTcScaleA (FEAT: the plain output)
      const float z0 = fmaf(acc[4 * j + 2 * h], us, bv.x), z1 = fmaf(acc[4 * j + 2 * h + 1], us, bv.y);
      float o0, o1, e;
      if (FEAT) o0 = z0, o1 = z1;
      else if (kColorLike) o0 = fmaxf(z0, 0.f), o1 = fmaxf(z1, 0.f);
      else o0 = softplus100_scaled(z0, e), o1 = softplus100_scaled(z1, e);
      if (SKIP && 8 * j + 8 > N) {  // skip connection: embedding columns of layer 3's output
        float ev[2];
        const uint32_t ok = (MODE == MLP_BG_SDF) ? embed2<4, false>(c0 - N, kBgEmbed, F.pt[h], nullptr, ev)
                                                 : embed2<3, false>(c0 - N, kEmbed, F.pt[h], a.embed_w, ev);
        o0 = (c0 >= N) ? ((ok & 1u) ? kTcScaleA * ev[0] : 0.f) : o0;
        o1 = (c0 + 1 >= N) ? ((ok & 2u) ? kTcScaleA * ev[1] : 0.f) : o1;
      }
      if (HEAD) {
        F.head[h][0] += o0 * w0.x + o1 * w0.y;
        if (kColorLike) {
          F.head[h][1] += o0 * w1.x + o1 * w1.y;
          F.head[h][2] += o0 * w2.x + o1 * w2.y;
        }
      }
      if (FEAT) {
        if (F.valid[h]) *reinterpret_cast<float2*>(a.feat + (size_t)F.p[h] * kFeat + c0) = make_float2(o0, o1);
      } else if (WRITE) {
        frag_store_a(F, h, j, o0, o1);
      }
    }
  }
}

// Reverse-mode chain (MODE MLP_SDF_REV), one step = one accumulator: d sdf/d z_7 = w_sdf * s_7;  d sdf/d z_{l-1} = (g_l . W_l) * s_{l-1};
// the embedding columns (skip input of layer 4, input of layer 0) collect d sdf/d embed, chained with d embed/d x_c per column.
//   KIND 0: forward layer l = st (stashes s_l = softplus'(z_l));  SPEC 1: l = 3 (skip columns), SPEC 2: l = 7 (sdf head)
//   KIND 1: the feature layer (st = 8): writes the 256-d feature, seeds g_7 = w_sdf * s_7
//   KIND 2: backward layer l = 16 - st: operand of the next step = acc * s_{l-1};  SPEC 1: l = 4 (its columns >= 217 are d sdf/d embed)
//   KIND 3: st = 16: d sdf / d embed through layer 0's input, no operand
// Stash: s_l as unorm16 pairs, written and later read by the SAME thread (its fragment), L2 only (.cg), laid out so that a warp's
// 32 words of one (layer, column pair, row half) are contiguous: 512 KB per CTA.
template <int KIND, int SPEC>
__device__ __forceinline__ void rev_step(const TcArgs& a, Frag& F, uint32_t* sigw, const int st, const float (&acc)[128]) {
  constexpr float kInvQ = 1.0f / 65535.0f;
  const int l = (st <= 8) ? st : 16 - st;
  const float* bias = (KIND <= 1) ? a.L[st].bias : nullptr;
  // stash layer read by this step: s_7 for the feature layer's seed, s_{l-1} for backward layer l
  const int sl = (KIND == 1) ? 7 : l - 1;
  const float us = (KIND == 0) ? a.unscale * kTcScaleA : a.unscale;   // forward layers work on kTcScaleA * z (bias pre-scaled)
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c0 = 8 * j + 2 * F.q;
    float2 bv = make_float2(0.f, 0.f), wl = make_float2(0.f, 0.f);
    if (KIND <= 1) bv = __ldg(reinterpret_cast<const float2*>(bias + c0));
    if ((KIND == 0 && SPEC == 2) || KIND == 1) wl = __ldg(reinterpret_cast<const float2*>(a.w_last + c0));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float r0 = acc[4 * j + 2 * h], r1 = acc[4 * j + 2 * h + 1];
      float o0 = 0.f, o1 = 0.f;
      if (KIND == 0) {
        float e0, e1;
        const float z0 = fmaf(r0, us, bv.x), z1 = fmaf(r1, us, bv.y);
        o0 = softplus100_scaled(z0, e0), o1 = softplus100_scaled(z1, e1);
        const float q0 = mufu_rcp(1.0f + e0), q1 = mufu_rcp(1.0f + e1);
        __stcg(sigw + ((l * 32 + j) * 2 + h) * kTcConsumers, unorm16_pack2((z0 >= 0.f) ? q0 : e0 * q0, (z1 >= 0.f) ? q1 : e1 * q1));
        if (SPEC == 1 && 8 * j + 8 > 217) {
          float ev[2];
          const uint32_t ok = embed2<3, false>(c0 - 217, kEmbed, F.pt[h], a.embed_w, ev);
          o0 = (ok & 1u) ? kTcScaleA * ev[0] : o0;
          o1 = (ok & 2u) ? kTcScaleA * ev[1] : o1;
        }
        if (SPEC == 2) F.head[h][0] += o0 * wl.x + o1 * wl.y;
      } else {
        // softplus' of these 2 columns (times 65535; the scale is folded below)
        const uint32_t sq = (KIND == 3) ? 0u : __ldcg(sigw + ((sl * 32 + j) * 2 + h) * kTcConsumers);
        const float s0 = unorm16_lo(sq), s1 = unorm16_hi(sq);
        if (KIND == 1) {
          if (F.valid[h]) {   // the 256-d feature vector: written once, read once by the colour net -> streaming stores
            __stcs(reinterpret_cast<float2*>(a.feat + (size_t)F.p[h] * kFeat + c0), make_float2(fmaf(r0, us, bv.x), fmaf(r1, us, bv.y)));
          }
          // g_7 = w_sdf * s_7, times the operand scale
          o0 = (kTcScaleA * kInvQ) * wl.x * s0, o1 = (kTcScaleA * kInvQ) * wl.y * s1;
        } else {
          if (KIND == 2) {   // operand of the next backward layer: (acc * unscale) * s_{l-1}, times the operand scale (one constant)
            const float k2 = us * (kTcScaleA * kInvQ);
            o0 = (r0 * k2) * s0, o1 = (r1 * k2) * s1;
          }
          if ((KIND == 2 && SPEC == 1 && 8 * j + 8 > 217) || (KIND == 3 && 8 * j < 40)) {  // columns that are d sdf / d embed
            const int e0 = (KIND == 2) ? c0 - 217 : c0;
            float dv[2];
            const uint32_t ok = embed2<3, true>(e0, kEmbed, F.pt[h], a.embed_w, dv);
            const float rr[2] = {r0 * us, r1 * us};
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int ec = max(e0 + i, 0), d = ec - 3 * ((ec * 171) >> 9);
              const bool okc = (ok >> i) & 1u;
              const float je = okc ? rr[i] * dv[i] : 0.f;
              F.head[h][1] += (d == 0) ? je : 0.f;
              F.head[h][2] += (d == 1) ? je : 0.f;
              F.gz[h] += (d == 2) ? je : 0.f;
              if (KIND == 2 && okc) (i == 0 ? o0 : o1) = 0.f;
            }
          }
        }
      }
      if (KIND != 3) frag_store_a(F, h, j, o0, o1);
    }
  }
}

// Tile prologue of one consumer warpgroup: the layer-0 A operand of its 64 rows, in 8-column units (2 threads per row).
__device__ __forceinline__ void store_unit(uint8_t* gA_hi, uint8_t* gA_lo, int row, int u, const float (&x)[8]) {
  uint4 hi, lo;
  split8(x, hi, lo);
  const uint32_t off = (uint32_t)((u >> 3) * kTcAChunkBytes) + a_unit_off(row, u & 7);
  *reinterpret_cast<uint4*>(gA_hi + off) = hi;
  *reinterpret_cast<uint4*>(gA_lo + off) = lo;
}

template <int MODE>
__device__ __forceinline__ void prologue(const TcArgs& a, uint8_t* gA_hi, uint8_t* gA_lo, const int row, const int p, const int half) {
  constexpr bool kColorLike = (MODE == MLP_COLOR || MODE == MLP_BG_RGB);
  const bool valid = p < a.P;
  if (MODE == MLP_LINEAR) {
    // rows of a [P, lda] fp32 matrix, columns [0, kvalid) (zero padded to the image's K), optionally divided by *in_scale
    const float isc = (a.in_scale != nullptr) ? kTcScaleA / __ldg(a.in_scale) : kTcScaleA;
    const float* src = a.lin_in + (size_t)p * a.lda;
    const int nu = a.L[0].nst * 4;
#pragma unroll 1
    for (int u = half; u < nu; u += 2) {
      const int k0 = 8 * u;
      float x[8];
      if (valid && k0 + 8 <= a.kvalid) {
        const float4 f0 = __ldg(reinterpret_cast<const float4*>(src + k0)), f1 = __ldg(reinterpret_cast<const float4*>(src + k0) + 1);
        x[0] = f0.x, x[1] = f0.y, x[2] = f0.z, x[3] = f0.w, x[4] = f1.x, x[5] = f1.y, x[6] = f1.z, x[7] = f1.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = (valid && k0 + i < a.kvalid) ? __ldg(src + k0 + i) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] *= isc;
      store_unit(gA_hi, gA_lo, row, u, x);
    }
  } else if (MODE == MLP_BG_SDF) {
    // inverted-sphere point of sample p % 32 of ray p / 32 (background.py:63-68,102-135), PE-10 + frame code: 116 -> 128
    float p4[4] = {0.f, 0.f, 0.f, 0.f};
    if (valid) {
      const int ray = p / kBgN;
      const float o[3] = {a.cam[3 * ray], a.cam[3 * ray + 1], a.cam[3 * ray + 2]};
      const float d[3] = {a.dirs[3 * ray], a.dirs[3 * ray + 1], a.dirs[3 * ray + 2]};
      depth2pts_outside(o, d, bg_depth(p % kBgN, a.r_sphere), a.r_sphere, p4);
    }
    const int b = valid ? p / a.pts_per_frame : 0;
#pragma unroll 1
    for (int u = half; u < 16; u += 2) {
      float x[8];
      const int e0 = 8 * u;
      const Embed8 ev = embed8<4, false>(e0, kBgEmbed, p4[0], p4[1], p4[2], p4[3], nullptr);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int e = e0 + i;
        float v = ((ev.ok >> i) & 1u) ? ev.v[i] : 0.f;
        if (e >= kBgEmbed && e < kBgEmbed + kBgFrame) v = a.frame_code[b * kBgFrame + e - kBgEmbed];
        x[i] = kTcScaleA * v;
      }
      store_unit(gA_hi, gA_lo, row, u, x);
    }
  } else if (!kColorLike) {
    float px = 0.f, py = 0.f, pz = 0.f;
    if (valid) { px = a.xc[3 * (size_t)p], py = a.xc[3 * (size_t)p + 1], pz = a.xc[3 * (size_t)p + 2]; }
#pragma unroll 1
    for (int u = half; u < 8; u += 2) {
      float x[8];
      const Embed8 ev = embed8<3, false>(8 * u, kEmbed, px, py, pz, 0.f, a.embed_w);
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = ((ev.ok >> i) & 1u) ? kTcScaleA * ev.v[i] : 0.f;
      store_unit(gA_hi, gA_lo, row, u, x);
    }
  } else {
    const int b = valid ? p / a.pts_per_frame : 0;
#pragma unroll 1
    for (int u = half; u < 40; u += 2) {
      float x[8];
      const int k0 = 8 * u;
      if (k0 < kFeat) {
        if (valid) {
          const float4 f0 = *reinterpret_cast<const float4*>(a.feat + (size_t)p * kFeat + k0);
          const float4 f1 = *reinterpret_cast<const float4*>(a.feat + (size_t)p * kFeat + k0 + 4);
          x[0] = f0.x, x[1] = f0.y, x[2] = f0.z, x[3] = f0.w, x[4] = f1.x, x[5] = f1.y, x[6] = f1.z, x[7] = f1.w;
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) x[i] = 0.f;
        }
      } else {
        Embed8 ev;
        ev.ok = 0;
        if (MODE == MLP_BG_RGB) {
          const int ray = valid ? p / kBgN : 0;
          ev = embed8<3, false>(k0 - kFeat, kBgView, a.dirs[3 * ray], a.dirs[3 * ray + 1], a.dirs[3 * ray + 2], 0.f, nullptr);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int e = k0 + i - kFeat;  // [x_c(3), n(3), pose_embed(8), time_code(32)]; background: [view PE-4 (27), frame code (32)]
          float v = 0.f;
          if (MODE == MLP_BG_RGB) {
            if (valid) {
              if ((ev.ok >> i) & 1u) v = ev.v[i];
              else if (e >= kBgView && e < kBgView + kBgFrame) v = a.frame_code[b * kBgFrame + e - kBgView];
            }
          } else if (valid) {
            if (e < 3) v = a.xc[3 * (size_t)p + e];
            else if (e < 6) v = a.normal[3 * (size_t)p + e - 3];
            else if (e < 14) v = (a.pose_embed != nullptr) ? a.pose_embed[b * 8 + e - 6] : 0.f;
            else if (e < a.k0 - kFeat) v = a.time_code[b * 32 + e - 14];
          }
          x[i] = v;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] *= kTcScaleA;
      store_unit(gA_hi, gA_lo, row, u, x);
    }
  }
}

// sum over the 4 threads (lane % 4) that share a fragment row: fixed order, so the result does not depend on scheduling
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

template <int MODE>
__global__ void __launch_bounds__(kTcThreadsTotal, 1) k_mlp_tc(TcArgs a) {
  static_assert(MODE == MLP_SDF_ONLY || MODE == MLP_SDF_REV || MODE == MLP_COLOR || MODE == MLP_BG_SDF || MODE == MLP_BG_RGB || MODE == MLP_LINEAR, "chains built on wgmma");
  if (a.st != nullptr && a.st->done) return;
  using Cfg = TcCfg<MODE>;
  constexpr bool kColorLike = Cfg::kColorLike;
  constexpr int NA = Cfg::kAChunks, NS = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA_hi = base, sA_lo = base + NA * kTcAChunkBytes, sW = base + Cfg::kSmemA;
  const uint32_t sBar = sW + Cfg::kSmemW;
  const uint32_t bWFull = sBar, bWEmpty = sBar + 8 * NS, sAbort = sBar + 16 * NS;
  uint8_t* gen_base = smem_raw + (base - smem_u32(smem_raw));  // generic pointer to `base`
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  volatile int* abort_flag = reinterpret_cast<volatile int*>(gen_base + (sAbort - base));
  const int n_tiles = ceil_div(a.P, kTcRows);

  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(bWFull + 8 * i, 1); mbar_init(bWEmpty + 8 * i, kTcConsumers / 32); }  // empty: one arrival per consumer warp
    *abort_flag = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kTcConsumers / 32) {
    // ============================================================ weight producer (TMA engine, bulk async copies)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kTcProducerRegs));
    if (warp != kTcConsumers / 32) return;
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      for (int l = 0; l < a.n_layers; ++l) {
        const uint8_t* src = a.L[l].wimg;
        for (int s = 0; s < a.L[l].nst; ++s) {
          if (!__all_sync(0xffffffffu, mbar_wait(bWEmpty + 8 * stage, phase ^ 1, a.err, 1, abort_flag))) return;
          if (elect_one()) {
            mbar_expect_tx(bWFull + 8 * stage, kTcStageBytes);
            bulk_g2s(sW + stage * kTcStageBytes, src + (size_t)s * kTcStageBytes, kTcStageBytes, bWFull + 8 * stage);
          }
          __syncwarp();
          if (++stage == NS) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ============================================================ consumer warpgroups: MMAs + epilogue on their 64 rows
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTcConsumerRegs));
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  uint8_t* gA_hi = gen_base;
  uint8_t* gA_lo = gen_base + NA * kTcAChunkBytes;
  Pipe P;
  P.a_hi = sA_hi + wg * 64 * 128, P.a_lo = sA_lo + wg * 64 * 128;   // 64 rows x 128 bytes of every A chunk
  P.sW = sW, P.bWFull = bWFull, P.bWEmpty = bWEmpty, P.stage = 0, P.phase = 0, P.ns = NS, P.lane = lane, P.bar_id = 1 + wg;
  P.abort_flag = abort_flag;
  Frag F;
  F.q = lane & 3;
  F.lo_off = (uint32_t)(NA * kTcAChunkBytes);
  const int r_frag = wg * 64 + (tid >> 5) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_frag + 8 * h;
    F.r7[h] = r & 7;
    F.a_row[h] = gA_hi + (r >> 3) * 1024 + (r & 7) * 128 + 4 * F.q;
  }
  uint32_t* sigw = (MODE == MLP_SDF_REV) ? reinterpret_cast<uint32_t*>(a.sig) + (size_t)blockIdx.x * (8 * kTcRows * 256 / 2) + threadIdx.x : nullptr;
  float acc[128];

  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    // ---------------------------------------------------------- prologue: layer-0 A operand of this warpgroup's rows
    prologue<MODE>(a, gA_hi, gA_lo, wg * 64 + (tid & 63), tile * kTcRows + wg * 64 + (tid & 63), tid >> 6);
    fence_proxy_async();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      F.p[h] = tile * kTcRows + r_frag + 8 * h;
      F.valid[h] = F.p[h] < a.P;
      F.pt[h][0] = F.pt[h][1] = F.pt[h][2] = F.pt[h][3] = 0.f;
      F.head[h][0] = F.head[h][1] = F.head[h][2] = 0.f;
      F.gz[h] = 0.f;
      if (F.valid[h]) {
        const size_t p = (size_t)F.p[h];
        if (MODE == MLP_BG_SDF) {
          const int ray = (int)(p / kBgN);
          const float o[3] = {a.cam[3 * ray], a.cam[3 * ray + 1], a.cam[3 * ray + 2]};
          const float d[3] = {a.dirs[3 * ray], a.dirs[3 * ray + 1], a.dirs[3 * ray + 2]};
          depth2pts_outside(o, d, bg_depth((int)(p % kBgN), a.r_sphere), a.r_sphere, F.pt[h]);
        } else if (MODE == MLP_SDF_ONLY || MODE == MLP_SDF_REV) {
          F.pt[h][0] = a.xc[3 * p], F.pt[h][1] = a.xc[3 * p + 1], F.pt[h][2] = a.xc[3 * p + 2];
        }
      }
    }
    wg_all(true, P.bar_id);   // the operand is complete before any thread of the warpgroup issues the first MMA

    // ---------------------------------------------------------- layers: MMAs, then the epilogue on the accumulator
    bool ok = true;
    if (MODE == MLP_LINEAR) {
      // ======== one layer: C = acc * unscale (* in_scale) + bias, fp32 rows of [P, ldc], columns [0, nvalid) ========
      ok = mma_layer(a, P, 0, acc);
      if (!ok) break;
      const float* bias = a.L[0].bias;
      const float osc = (a.in_scale != nullptr) ? a.unscale * __ldg(a.in_scale) : a.unscale;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c0 = 8 * j + 2 * F.q;
        if (c0 >= a.nvalid) continue;
        float2 bv = make_float2(0.f, 0.f);
        if (bias != nullptr) bv = make_float2(__ldg(bias + c0), (c0 + 1 < a.nvalid) ? __ldg(bias + c0 + 1) : 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!F.valid[h]) continue;
          float* dst = a.lin_out + (size_t)F.p[h] * a.ldc + c0;
          const float o0 = fmaf(acc[4 * j + 2 * h], osc, bv.x), o1 = fmaf(acc[4 * j + 2 * h + 1], osc, bv.y);
          if (c0 + 1 < a.nvalid) *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
          else dst[0] = o0;
        }
      }
    } else if (MODE == MLP_SDF_REV) {
      // ======== reverse-mode gradient: 8 forward layers (stash softplus'), feature layer, 8 backward layers (rev_step) ========
      for (int st = 0; st < 17; ++st) {
        ok = mma_layer(a, P, st, acc);
        if (!ok) break;
        if (st < 8) {
          if (st == 3) rev_step<0, 1>(a, F, sigw, st, acc);
          else if (st == 7) rev_step<0, 2>(a, F, sigw, st, acc);
          else rev_step<0, 0>(a, F, sigw, st, acc);
        } else if (st == 8) {
          rev_step<1, 0>(a, F, sigw, st, acc);
        } else if (st < 16) {
          if (st == 12) rev_step<2, 1>(a, F, sigw, st, acc);
          else rev_step<2, 0>(a, F, sigw, st, acc);
        } else {
          rev_step<3, 0>(a, F, sigw, st, acc);
        }
        fence_proxy_async();
        wg_all(true, P.bar_id);   // the next layer's operand is complete
      }
      if (!ok) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float s = quad_sum(F.head[h][0]), gx = quad_sum(F.head[h][1]), gy = quad_sum(F.head[h][2]), gz = quad_sum(F.gz[h]);
        if (F.q == 0 && F.valid[h]) {
          const size_t p = (size_t)F.p[h];
          a.sdf[p] = s * (1.0f / kTcScaleA) + a.b_last[0];
          a.grad[3 * p] = gx, a.grad[3 * p + 1] = gy, a.grad[3 * p + 2] = gz;
        }
      }
    } else {
      for (int l = 0; l < a.n_layers; ++l) {
        ok = mma_layer(a, P, l, acc);
        if (!ok) break;
        const bool head_layer = kColorLike ? (l == a.n_layers - 1) : (l == 7);
        const bool last_mma = (l == a.n_layers - 1);
        if (MODE == MLP_BG_SDF && last_mma) epi_layer<MODE, false, false, true, false>(a, F, l, acc);           // the feature rows
        else if (MODE == MLP_BG_SDF && head_layer) epi_layer<MODE, true, true, false, false>(a, F, l, acc);
        else if (head_layer) epi_layer<MODE, true, false, false, false>(a, F, l, acc);
        else if (!kColorLike && l == 3) epi_layer<MODE, false, true, false, true>(a, F, l, acc);
        else epi_layer<MODE, false, true, false, false>(a, F, l, acc);
        fence_proxy_async();
        wg_all(true, P.bar_id);   // the next layer's operand is complete
      }
      if (!ok) break;
      // ---------------------------------------------------------- heads: sum over the 4 threads of each row
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float hs[3];
#pragma unroll
        for (int k = 0; k < (kColorLike ? 3 : 1); ++k) hs[k] = quad_sum(F.head[h][k]) * (1.0f / kTcScaleA);  // the head saw activations times kTcScaleA
        if (F.q == 0 && F.valid[h]) {
          const size_t p = (size_t)F.p[h];
          if (kColorLike) {
#pragma unroll
            for (int k = 0; k < 3; ++k) a.rgb[3 * p + k] = 1.0f / (1.0f + __expf(-(hs[k] + a.b_last[k])));
          } else {
            a.sdf[p] = hs[0] + a.b_last[0];
          }
        }
      }
    }
    // every thread of the warpgroup has finished with this tile's operand before the next tile's prologue overwrites it
    wg_all(true, P.bar_id);
  }
}

// ------------------------------------------------------------------------------------------------ packing
// One stage image = [256 n x 32 k] fp16 in the SW64 K-major canonical layout, hi part then lo part.
// W[n][k] = kTcScaleW * scale * fold(v, g)[row_off + n][colmap(k)];  colmap: k -> source column (or -1 => 0).
__global__ void k_tc_pack(const float* __restrict__ v, const float* __restrict__ g, int in_dim, int row_off, int N, int K,
                          int kpad, float scale, int perm_feat_first, uint8_t* __restrict__ img) {
  const int n = blockIdx.x;  // 0..255
  __shared__ float red[32];
  __shared__ float f_sh;
  float f = 0.f;
  const float* vr = v + (size_t)(row_off + (n < N ? n : 0)) * in_dim;
  if (g != nullptr) {
    float ss = 0.f;
    for (int k = threadIdx.x; k < in_dim; k += blockDim.x) ss += vr[k] * vr[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < blockDim.x / 32; ++w) tot += red[w];
      f_sh = g[row_off + (n < N ? n : 0)] / sqrtf(tot);
    }
    __syncthreads();
    f = f_sh;
  } else {
    f = 1.0f;
  }
  for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
    int src = k;
    if (perm_feat_first) {  // colour lin0: A order [feat(256) | x_c, n, pose(14) | time(32)] vs weight order [14 | 256 | 32];
      // background lin0: A order [feat(256) | view, frame (59)] vs weight order [59 | 256].  perm_feat_first = the leading width
      if (k < kFeat) src = perm_feat_first + k;
      else if (k < kFeat + perm_feat_first) src = k - kFeat;
      else src = k;
    }
    float w = (n < N && src < K) ? kTcScaleW * (scale * (vr[src] * f)) : 0.f;
    __half h = __float2half_rn(w);
    __half l = __float2half_rn(w - __half2float(h));
    const int st = k >> 5, kk = k & 31;
    const size_t off = (size_t)st * kTcStageBytes + (size_t)((n >> 3) * 512 + (n & 7) * 64 + ((((kk >> 3) ^ ((n >> 1) & 3))) << 4) + (kk & 7) * 2);
    *reinterpret_cast<__half*>(img + off) = h;
    *reinterpret_cast<__half*>(img + off + 16384) = l;
  }
}

// Transposed image for the reverse-mode gradient: B rows = input index k_in of layer l, K = output index n_out:
// WT[r][n_out] = kTcScaleW * scale * fold(v, g)[row_off + n_out][src(r)]  (zero outside [N_out) x valid sources).
// colmap: 0: src = r (r < K_in);  1: a first layer whose 256 feature inputs follow `lead` other inputs (colour lin0: lead = 14 [x_c, n,
//         pose]; background colour lin0: lead = 59 [view, frame code]), feature part: src = lead + r (r < 256);
//         2: the same layer's other inputs in the A operand's order [leading inputs | inputs after the features]: src = r (r < lead),
//         256 + r (256 + r < K_in)
__global__ void k_tc_pack_T(const float* __restrict__ v, const float* __restrict__ g, int in_dim, int row_off, int N_out, int K_in,
                            int colmap, int lead, float scale, uint8_t* __restrict__ img) {
  const int r = blockIdx.x;   // k_in, 0..255
  const int n = threadIdx.x;  // n_out, 0..255
  int src = -1;
  if (colmap == 0) src = (r < K_in) ? r : -1;
  else if (colmap == 1) src = lead + r;
  else src = (r < lead) ? r : ((256 + r < K_in) ? 256 + r : -1);
  float w = 0.f;
  if (n < N_out && src >= 0) {
    const float* vr = v + (size_t)(row_off + n) * in_dim;
    float f = 1.0f;
    if (g != nullptr) {
      float ss = 0.f;
      for (int k = 0; k < in_dim; ++k) ss += vr[k] * vr[k];
      f = g[row_off + n] / sqrtf(ss);
    }
    w = kTcScaleW * (scale * (vr[src] * f));
  }
  const __half h = __float2half_rn(w);
  const __half l = __float2half_rn(w - __half2float(h));
  const int st = n >> 5, kk = n & 31;
  const size_t off = (size_t)st * kTcStageBytes + (size_t)((r >> 3) * 512 + (r & 7) * 64 + ((((kk >> 3) ^ ((r >> 1) & 3))) << 4) + (kk & 7) * 2);
  *reinterpret_cast<__half*>(img + off) = h;
  *reinterpret_cast<__half*>(img + off + 16384) = l;
}

static int tc_init(hold_ctx*) {
  cudaError_t e;
  e = cudaFuncSetAttribute(k_mlp_tc<MLP_SDF_ONLY>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_SDF_ONLY>::kSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_tc<MLP_COLOR>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_COLOR>::kSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_tc<MLP_SDF_REV>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_SDF_REV>::kSmemBytes);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_tc<MLP_LINEAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<MLP_LINEAR>::kSmemBytes);
  if (e != cudaSuccess) { set_error("tensor-core MLP kernel attribute: %s", cudaGetErrorString(e)); return HOLD_E_CUDA; }
  return HOLD_OK;
}

static void tc_free(NodeState& ns) {
  if (!ns.tc) return;
  for (int l = 0; l < HOLD_MAX_LAYERS; ++l) {
    if (ns.tc->sdf_img[l]) cudaFree(ns.tc->sdf_img[l]);
    if (ns.tc->rgb_img[l]) cudaFree(ns.tc->rgb_img[l]);
    if (ns.tc->sdf_imgT[l]) cudaFree(ns.tc->sdf_imgT[l]);
    if (l < 6 && ns.tc->rgb_imgT[l]) cudaFree(ns.tc->rgb_imgT[l]);
  }
  if (ns.tc->bias_s) cudaFree(ns.tc->bias_s);
  delete ns.tc;
  ns.tc = nullptr;
}

static int tc_pack(hold_ctx* ctx, NodeState& ns, const hold_mlp_weights* sdf, const hold_mlp_weights* rgb, cudaStream_t s) {
  if (!ns.tc) ns.tc = new TcMlp();
  TcMlp& t = *ns.tc;
  for (int l = 0; l < 9; ++l) {
    const int K = (l == 0) ? kEmbed : kHidden, kpad = (l == 0) ? 64 : 256;
    const int N = (l == 3) ? kHidden - kEmbed : kHidden;
    const int row_off = (l == 8) ? 1 : 0;
    t.sdf_nst[l] = kpad / 32;
    if (!t.sdf_img[l]) HOLD_CUDA(cudaMalloc((void**)&t.sdf_img[l], (size_t)t.sdf_nst[l] * kTcStageBytes));
    const float scale = (l == 4) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    k_tc_pack<<<256, 128, 0, s>>>(sdf->weight_v[l], sdf->weight_g[l], sdf->in_dim[l], row_off, N, K, kpad, scale, 0, t.sdf_img[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int l = 0; l < 9; ++l) {  // W_l^T for the reverse-mode gradient (layers 7..0); l = 8: the feature rows (training backward)
    const int K_in = (l == 0) ? kEmbed : kHidden, N_out = (l == 3) ? kHidden - kEmbed : kHidden;
    if (!t.sdf_imgT[l]) HOLD_CUDA(cudaMalloc((void**)&t.sdf_imgT[l], (size_t)8 * kTcStageBytes));
    const float scale = (l == 4) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    k_tc_pack_T<<<256, 256, 0, s>>>(sdf->weight_v[l], sdf->weight_g[l], sdf->in_dim[l], l == 8 ? 1 : 0, N_out, K_in, 0, 0, scale, t.sdf_imgT[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int i = 0; i < 5; ++i) {  // colour net transposes for the training backward: lin0 in two parts (its K = 320 > 256), lin1..3
    const int l = (i < 2) ? 0 : i - 1;
    if (!t.rgb_imgT[i]) HOLD_CUDA(cudaMalloc((void**)&t.rgb_imgT[i], (size_t)8 * kTcStageBytes));
    k_tc_pack_T<<<256, 256, 0, s>>>(rgb->weight_v[l], rgb->weight_g[l], rgb->in_dim[l], 0, 256, rgb->in_dim[l], i == 0 ? 1 : (i == 1 ? 2 : 0), 14, 1.0f,
                                    t.rgb_imgT[i]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  if (!t.bias_s) HOLD_CUDA(cudaMalloc((void**)&t.bias_s, 13 * 256 * sizeof(float)));
  for (int l = 0; l < 13; ++l) {   // (the fp32 packing of this call has already written ns.sdf.bias / ns.rgb.bias on this stream)
    k_scale_vec<<<1, 256, 0, s>>>(l < 9 ? ns.sdf.bias[l] : ns.rgb.bias[l - 9], 256, l == 8 ? 1.0f : kTcScaleA, t.bias_s + 256 * l);
    HOLD_LAUNCH_CHECK(ctx);
  }
  for (int l = 0; l < 4; ++l) {
    const int K = (l == 0) ? rgb->in_dim[0] : 256, kpad = (l == 0) ? 320 : 256;
    t.rgb_nst[l] = kpad / 32;
    if (!t.rgb_img[l]) HOLD_CUDA(cudaMalloc((void**)&t.rgb_img[l], (size_t)t.rgb_nst[l] * kTcStageBytes));
    k_tc_pack<<<256, 128, 0, s>>>(rgb->weight_v[l], rgb->weight_g[l], rgb->in_dim[l], 0, 256, K, kpad, 1.0f, l == 0 ? 14 : 0, t.rgb_img[l]);
    HOLD_LAUNCH_CHECK(ctx);
  }
  return HOLD_OK;
}

// SDF net on P canonical points: sdf only (sampler rounds: 8 layers, sdf head), or sdf + d sdf / d x_c + 256-d feature
// (reverse mode: 8 forward layers, feature layer, 8 backward layers over the transposed images).
static int tc_launch_sdf(hold_ctx* ctx, NodeState& ns, int P, const float* xc, const float* embed_w, float* sdf, float* grad,
                         float* feat, const SamplerState* st, cudaStream_t s) {
  const bool rev = (grad != nullptr) || (feat != nullptr);
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.P = P, a.n_layers = rev ? 17 : 8;
  for (int l = 0; l < 9; ++l) {
    a.L[l].wimg = ns.tc->sdf_img[l], a.L[l].bias = ns.tc->bias_s + 256 * l, a.L[l].nst = ns.tc->sdf_nst[l], a.L[l].N = ns.sdf.N[l];
  }
  a.w_last = ns.sdf.w_last, a.b_last = ns.sdf.b_last;
  a.xc = xc, a.embed_w = embed_w, a.sdf = sdf, a.grad = grad, a.feat = feat, a.st = st, a.err = ctx->dev_err;
  a.passes = (st != nullptr && ctx->sampler_passes >= 1 && ctx->sampler_passes <= 3) ? ctx->sampler_passes : 3;
  a.unscale = kTcUnscale * (1.0f + (float)(ctx->tc_acc_comp >= 0 ? ctx->tc_acc_comp : kTcAccComp) * (1.0f / 16777216.0f));
  const int tiles = ceil_div(P, kTcRows), grid = min(tiles, ctx->sm_count);
  if (rev) {
    HOLD_REQUIRE(grad != nullptr && feat != nullptr, "sdf eval with gradient needs both grad and feat buffers");
    void* sig = nullptr;
    int rc = ws_get(ctx, 12 /* WS_SIG */, (size_t)grid * 8 * kTcRows * 256 * sizeof(uint16_t), &sig);
    if (rc) return rc;
    a.sig = (uint16_t*)sig;
    for (int i = 0; i < 8; ++i) {
      a.L[9 + i].wimg = ns.tc->sdf_imgT[7 - i], a.L[9 + i].bias = nullptr, a.L[9 + i].nst = 8, a.L[9 + i].N = 256;
    }
    k_mlp_tc<MLP_SDF_REV><<<grid, kTcThreadsTotal, TcCfg<MLP_SDF_REV>::kSmemBytes, s>>>(a);
  } else {
    k_mlp_tc<MLP_SDF_ONLY><<<grid, kTcThreadsTotal, TcCfg<MLP_SDF_ONLY>::kSmemBytes, s>>>(a);
  }
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

// hold_linear: C[P, nvalid] = A[P, kvalid] . M^T (+ bias) against one packed image (selection of the image: api.cu)
static int tc_launch_linear_img(hold_ctx* ctx, const uint8_t* img, const float* bias, int nst, int P, const float* A, int lda, int kvalid,
                                const float* in_scale, float* Cout, int ldc, int nvalid, cudaStream_t s) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.P = P, a.n_layers = 1;
  HOLD_REQUIRE(lda % 4 == 0 && ldc % 4 == 0 && ((uintptr_t)A & 15) == 0 && ((uintptr_t)Cout & 15) == 0, "hold_linear: rows must be 16-byte aligned");
  a.L[0].wimg = img, a.L[0].bias = bias, a.L[0].nst = nst, a.L[0].N = nvalid;
  a.passes = 3;
  a.lin_in = A, a.lda = lda, a.kvalid = kvalid, a.lin_out = Cout, a.ldc = ldc, a.nvalid = nvalid, a.in_scale = in_scale;
  a.err = ctx->dev_err, a.unscale = kTcUnscale * (1.0f + (float)(ctx->tc_acc_comp >= 0 ? ctx->tc_acc_comp : kTcAccComp) * (1.0f / 16777216.0f));
  const int tiles = ceil_div(P, kTcRows);
  k_mlp_tc<MLP_LINEAR><<<min(tiles, ctx->sm_count), kTcThreadsTotal, TcCfg<MLP_LINEAR>::kSmemBytes, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

static int tc_launch_rgb(hold_ctx* ctx, NodeState& ns, int P, int pts_per_frame, const float* xc, const float* normal,
                         const float* pe, const float* feat, const float* time_code, float* rgb, cudaStream_t s) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.P = P, a.n_layers = 4;
  for (int l = 0; l < 4; ++l) {
    a.L[l].wimg = ns.tc->rgb_img[l], a.L[l].bias = ns.tc->bias_s + 256 * (9 + l), a.L[l].nst = ns.tc->rgb_nst[l], a.L[l].N = 256;
  }
  a.w_last = ns.rgb.w_last, a.b_last = ns.rgb.b_last;
  a.xc = xc, a.normal = normal, a.pose_embed = pe, a.feat = const_cast<float*>(feat), a.time_code = time_code;
  a.pts_per_frame = pts_per_frame, a.k0 = ns.rgb.K[0], a.rgb = rgb, a.err = ctx->dev_err, a.unscale = kTcUnscale, a.passes = 3;
  int tiles = ceil_div(P, kTcRows);
  k_mlp_tc<MLP_COLOR><<<min(tiles, ctx->sm_count), kTcThreadsTotal, TcCfg<MLP_COLOR>::kSmemBytes, s>>>(a);
  HOLD_LAUNCH_CHECK(ctx);
  return HOLD_OK;
}

}  // namespace hold
