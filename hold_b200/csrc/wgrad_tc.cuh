// Weight-gradient reduction of the training backward on the tensor cores (SURVEY §8f rank 2): OUT[n, k] += sum_p D[p, n] * A[p, k]
// for row-major fp32 D [P, N <= 256] (a pre-activation gradient) and A [P, K <= 256] (the layer's input), fp32-level arithmetic.
//
// The contraction runs over the POINTS, so both MMA operands are the transposes D^T [n x p] and A^T [k x p]: the 8 warps read
// 32-point slabs with coalesced loads along n / k (lane = column), each lane collects 8 consecutive points of its column, splits
// them into fp16 hi/lo (operands pre-divided by power-of-two scales so that small gradients stay inside the split's range) and
// stores one 16-byte unit of the K-major SW64 canonical layout — the transposition happens in registers, the smem images are the
// same layout the weight stages of mlp_tc.cuh use.  Each CTA owns one 128-row block of n (blockIdx.y); its two warpgroups issue
// wgmma m64n256k16 (64 rows of n each, all 256 columns of k, K = 16 points, 3 passes hi*hi + lo*hi + hi*lo) into register
// accumulators while the next slab is loaded into the other half of a 2-stage smem ring.  Every CTA sweeps its share of the point
// slabs, then adds its partial to OUT with red.global.add.f32 (the order of those adds is not fixed: fp32 round-off level, far
// below the 1e-4 gradient bar).
#pragma once
#include "mlp_tc.cuh"

namespace hold {

constexpr int kWgPts = 32;                      // points per stage (K of the MMAs: two k16 steps)
constexpr int kWgRowsD = 128;                   // rows of n per CTA
constexpr int kWgImgD = kWgRowsD * kWgPts * 2;  // fp16 image [128 rows x 32 points] = 8 KB
constexpr int kWgImgA = 256 * kWgPts * 2;       // fp16 image [256 rows x 32 points] = 16 KB
constexpr int kWgStage = 2 * kWgImgD + 2 * kWgImgA;   // D^T hi | D^T lo | A^T hi | A^T lo
constexpr int kWgStages = 2;
constexpr int kWgThreads = 256;
constexpr int kWgSmem = kWgStages * kWgStage + 1024;

struct WgArgs {
  int P, N, K, ldd, lda, ldo;
  const float* D;
  const float* A;
  const float* d_scale;   // device scalars (powers of two) or NULL
  const float* a_scale;
  float* out;
  int* err;
};

// byte offset of element (row r, point kk) inside one [rows x 32] K-major SW64 image
__device__ __forceinline__ uint32_t wg_off(int r, int kk) {
  return (uint32_t)((r >> 3) * 512 + (r & 7) * 64 + ((((kk >> 3) ^ ((r >> 1) & 3))) << 4) + (kk & 7) * 2);
}

__global__ void __launch_bounds__(kWgThreads, 1) k_wgrad_tc(WgArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int n0 = blockIdx.y * kWgRowsD;
  const int n_slabs = ceil_div(a.P, kWgPts);
  const int my_slabs = (n_slabs > (int)blockIdx.x) ? (n_slabs - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  if (my_slabs == 0) return;
  const float dsc = kTcScaleA / ((a.d_scale != nullptr) ? __ldg(a.d_scale) : 1.0f);
  const float asc = kTcScaleW / ((a.a_scale != nullptr) ? __ldg(a.a_scale) : 1.0f);
  float acc[128];
  for (int i = 0; i < my_slabs; ++i) {
    const int slab = (int)blockIdx.x + i * (int)gridDim.x;
    const int p0 = slab * kWgPts;
    // 48 work units per slab: D^T (4 row blocks of 32 n) and A^T (8 row blocks of 32 k), x 4 groups of 8 points; 6 per warp
    float x[6][8];
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int wu = warp * 6 + u;
      const bool isA = wu >= 16;
      const int rb = isA ? (wu - 16) >> 2 : wu >> 2, grp = wu & 3;
      const int col = (isA ? 0 : n0) + rb * 32 + lane;   // n (D^T) or k (A^T)
      const float* src = isA ? a.A : a.D;
      const int ld = isA ? a.lda : a.ldd, ncol = isA ? a.K : a.N;
      const float sc = isA ? asc : dsc;
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int p = p0 + grp * 8 + t;
        x[u][t] = (p < a.P && col < ncol) ? __ldg(src + (size_t)p * ld + col) * sc : 0.f;
      }
    }
    __syncthreads();   // every warpgroup has waited for the MMAs of slab i - 2, which read this stage
    uint8_t* sb = gen_base + (i & 1) * kWgStage;
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int wu = warp * 6 + u;
      const bool isA = wu >= 16;
      const int rb = isA ? (wu - 16) >> 2 : wu >> 2, grp = wu & 3;
      uint4 hi, lo;
      split8(x[u], hi, lo);
      uint8_t* im = sb + (isA ? 2 * kWgImgD : 0);
      const int img_bytes = isA ? kWgImgA : kWgImgD;
      *reinterpret_cast<uint4*>(im + wg_off(rb * 32 + lane, grp * 8)) = hi;
      *reinterpret_cast<uint4*>(im + img_bytes + wg_off(rb * 32 + lane, grp * 8)) = lo;
    }
    fence_proxy_async();
    __syncthreads();
    const uint32_t s_base = base + (uint32_t)((i & 1) * kWgStage);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 2; ++j) {          // two k16 steps of the 32 points
      const uint64_t dhi = gmma_desc(s_base + wg * (64 * 64) + j * 32, 512, kLayoutSW64);   // this warpgroup's 64 rows of n
      const uint64_t dlo = gmma_desc(s_base + kWgImgD + wg * (64 * 64) + j * 32, 512, kLayoutSW64);
      const uint64_t ahi = gmma_desc(s_base + 2 * kWgImgD + j * 32, 512, kLayoutSW64);
      const uint64_t alo = gmma_desc(s_base + 2 * kWgImgD + kWgImgA + j * 32, 512, kLayoutSW64);
      wgmma_256(acc, dhi, ahi, (i | j) != 0);
      wgmma_256(acc, dlo, ahi, 1);
      wgmma_256(acc, dhi, alo, 1);
    }
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  // ============================================================ accumulator read-out: rows n of this warpgroup, columns k
  const float osc = ((a.d_scale != nullptr) ? __ldg(a.d_scale) : 1.0f) * ((a.a_scale != nullptr) ? __ldg(a.a_scale) : 1.0f) /
                    (kTcScaleA * kTcScaleW);
  const int nr = n0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = nr + 8 * h;
    if (n >= a.N) continue;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int k = 8 * j + 2 * (lane & 3) + t;
        if (k < a.K) atomicAdd(a.out + (size_t)n * a.ldo + k, acc[4 * j + 2 * h + t] * osc);
      }
    }
  }
}

static int wgrad_init() {
  cudaError_t e = cudaFuncSetAttribute(k_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem);
  if (e != cudaSuccess) { set_error("k_wgrad_tc attribute: %s", cudaGetErrorString(e)); return HOLD_E_CUDA; }
  return HOLD_OK;
}

}  // namespace hold
